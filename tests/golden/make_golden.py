"""Generate the golden vectors under tests/golden/ from the UNMODIFIED reference CUDA sources.

Run on a GPU machine where oracle/_ref/libr2ref.so has been built (oracle/build_ref.sh, with R2_REFERENCE_ROOT
naming the reference checkout):

    python tests/golden/make_golden.py /tmp/golden

and copy the resulting .npz files into tests/golden/.  Each file holds the inputs of one small scene and
what the reference produced for it: radii, tiles_touched, the sorted 64-bit keys and point list, the
image / volume, and the gradients for a fixed random dL.  tests/test_oracle_cpu.py::test_golden_vectors
checks the CPU oracle against them without a GPU.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from r2_gaussian_b200 import scene  # noqa: E402
import test_ref_gpu as R  # noqa: E402


def main(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    cases = [("raster_cone_trained", "cone", "trained", 400, 64, 0.9),
             ("raster_parallel_trained", "parallel", "trained", 300, 48, 2.1),
             ("raster_cone_init", "cone", "init", 500, 80, 4.0)]
    for name, beam, kind, P, n, ang in cases:
        sc = scene.cone_beam_scanner(n, 32) if beam == "cone" else scene.parallel_beam_scanner(n, 32)
        view = scene.make_view(sc, ang)
        cloud = scene.make_cloud(P, kind=kind, seed=P)
        dL = np.random.RandomState(P).randn(n, n).astype(np.float32)
        ref = R.run_ref_raster(cloud, view, dL)
        np.savez_compressed(
            os.path.join(out_dir, name + ".npz"), means=cloud.means, scales=cloud.scales, rots=cloud.rotations,
            dens=cloud.density, view=view.viewmatrix, proj=view.projmatrix, W=n, H=n, tanfovx=view.tanfovx,
            tanfovy=view.tanfovy, mode=view.mode, dL=dL, radii=ref["radii"], tiles_touched=ref["tiles_touched"],
            keys=ref["keys"], point_list=ref["point_list"], image=ref["image"],
            **{"g_" + k: v for k, v in ref["grads"].items()})
        print(name, "R =", ref["R"])
    vcases = [("voxel_cube24", (24, 24, 24), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0), 300),
              ("voxel_ragged", (20, 12, 28), (1.5, 1.0, 2.0), (0.1, -0.2, 0.05), 250)]
    for name, nV, sV, ctr, P in vcases:
        cloud = scene.make_cloud(P, kind="trained", seed=P)
        dL = np.random.RandomState(P).randn(*nV).astype(np.float32)
        ref = R.run_ref_voxel(cloud, nV, sV, ctr, dL)
        np.savez_compressed(
            os.path.join(out_dir, name + ".npz"), means=cloud.means, scales=cloud.scales, rots=cloud.rotations,
            dens=cloud.density, nVoxel=np.array(nV), sVoxel=np.array(sV, np.float32), center=np.array(ctr, np.float32),
            dL=dL, radii_x=ref["radii_x"], radii_y=ref["radii_y"], radii_z=ref["radii_z"],
            tiles_touched=ref["tiles_touched"], keys=ref["keys"], point_list=ref["point_list"], vol=ref["vol"],
            **{"g_" + k: v for k, v in ref["grads"].items()})
        print(name, "R =", ref["R"])


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "gpurun_out", "golden"))
