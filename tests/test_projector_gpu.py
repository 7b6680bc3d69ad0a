"""The volume projector on the GPU (r2_gaussian_b200.projector over r2x_volume_project) against the float64 oracle,
through the product path (query -> project vs render, project -> fdk vs the volume), and end to end through
`generate_data` and `initialize_pcd --recon_method fdk --evaluate`."""
import json
import math
import os
import re
import types

import numpy as np
import pytest

import fdk_cases as fc
import projector_cases as pc
from oracle import projector_oracle as po
from r2_gaussian_b200 import scene

pytestmark = pytest.mark.gpu

# fdk(project(vol)) against vol, 180 cone views of 128^2, 48^3 grid (measured 0.027 with the float64 oracles)
FDK_ROUND_TRIP_BOUND = 0.04


def _torch():
    import torch

    return torch


def _scanner(mode, det_hw, vox, s_voxel, off, accuracy):
    sc = fc.scanner(mode, 8, 8)
    sc["nDetector"] = list(det_hw)
    if mode == "cone":
        sc["sDetector"] = [3.0, 4.0]
    sc["nVoxel"], sc["sVoxel"], sc["offOrigin"] = list(vox), list(s_voxel), list(off)
    sc["accuracy"] = accuracy
    return sc


HALF_PI = math.pi / 2
ORACLE_CASES = {
    # H != W, neither a multiple of the 32 x 8 block; off-centre non-cubic grids with anisotropic voxels; uneven
    # angles that include exactly 0 and pi/2 (direction components exactly 0 for parallel beam); part of every
    # detector misses the box
    "cone_acc05": ("cone", (37, 52), (20, 28, 12), (1.6, 1.8, 1.2), (0.1, -0.2, 0.15), 0.5, (0.0, 0.4, HALF_PI, 2.2, 4.0)),
    "cone_acc025": ("cone", (24, 41), (13, 17, 22), (1.0, 1.4, 1.8), (-0.3, 0.2, 0.1), 0.25, (HALF_PI, 0.0, 3.3)),
    "cone_acc1": ("cone", (45, 30), (31, 9, 16), (1.8, 0.6, 1.5), (0.0, 0.35, -0.2), 1.0, (0.0, 1.3, HALF_PI, 5.9)),
    "parallel_acc05": ("parallel", (45, 30), (18, 10, 26), (1.4, 1.0, 1.8), (-0.15, 0.1, 0.05), 0.5,
                       (0.0, HALF_PI, 0.7, 3.0, math.pi)),
    "parallel_acc025": ("parallel", (33, 17), (11, 23, 14), (0.9, 1.5, 1.2), (0.2, 0.1, -0.25), 0.25, (HALF_PI, 0.0, 2.5)),
    "parallel_acc1": ("parallel", (20, 36), (25, 19, 9), (1.6, 1.2, 0.7), (-0.1, -0.3, 0.4), 1.0, (0.0, 1.9, HALF_PI)),
}


@pytest.mark.parametrize("name", sorted(ORACLE_CASES))
def test_cuda_matches_oracle(name):
    torch = _torch()
    from r2_gaussian_b200.projector import project

    mode, det, vox, sv, off, acc, angles = ORACLE_CASES[name]
    sc = _scanner(mode, det, vox, sv, off, acc)
    vol = np.random.RandomState(len(name)).uniform(0.0, 1.0, size=vox).astype(np.float32)
    got = project(torch.tensor(vol, device="cuda"), angles, sc).cpu().numpy()
    want = po.project_scene(vol, angles, sc)
    assert got.shape == (len(angles), *det)
    err = np.abs(got.astype(np.float64) - want).max()
    assert err <= 1e-5 * np.abs(want).max(), (err, np.abs(want).max())
    missed = want == 0.0
    assert 0 < missed.sum() < missed.size                            # some rays miss the box, some hit it
    assert (got[missed] == 0.0).all()                                 # a ray that misses gives exactly 0


def _cloud_tensors(cloud):
    torch = _torch()
    t = {k: torch.tensor(v, device="cuda") for k, v in
         (("xyz", cloud.means), ("dens", cloud.density), ("s", cloud.scales), ("r", cloud.rotations))}
    pcl = types.SimpleNamespace(get_xyz=t["xyz"], get_density=t["dens"], get_scaling=t["s"], get_rotation=t["r"])
    return pcl, types.SimpleNamespace(debug=False, compute_cov3D_python=False)


def _render(pcl, pipe, sc, angles):
    torch = _torch()
    from r2_gaussian_b200.render_query import render

    with torch.no_grad():
        return torch.stack([render(scene.camera_from_view(scene.make_view(sc, float(a))), pcl, pipe)["render"][0]
                            for a in angles])


def _query(pcl, pipe, sc):
    torch = _torch()
    from r2_gaussian_b200.render_query import query

    with torch.no_grad():
        return query(pcl, sc["offOrigin"], sc["nVoxel"], sc["sVoxel"], pipe)["vol"]


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_round_trip_query_project_render(mode):
    """project(query(cloud)) against render(cloud), with the cloud, sizes and bound of the CPU round trip; a flipped or
    transposed volume, or the negated angles, are far off."""
    from r2_gaussian_b200.projector import project

    pcl, pipe = _cloud_tensors(fc.round_trip_cloud())
    sc = fc.scanner(mode, pc.ROUND_TRIP_DET, pc.ROUND_TRIP_VOX)
    angles = list(pc.ROUND_TRIP_ANGLES)
    want = _render(pcl, pipe, sc, angles).cpu().numpy()
    vol = _query(pcl, pipe, sc)
    err = pc.rel_l2(project(vol, angles, sc).cpu().numpy(), want)
    assert err <= pc.ROUND_TRIP_BOUND, err
    torch = _torch()
    for name, v, a in pc.flipped_variants(vol.cpu().numpy(), angles):
        off = pc.rel_l2(project(torch.tensor(np.ascontiguousarray(v), device="cuda"), a, sc).cpu().numpy(), want)
        assert off >= 0.5, (name, off)


def test_round_trip_project_fdk():
    """fdk(project(vol)) against vol at 180 cone views: the projector and FDK are adjoint-consistent in geometry."""
    from r2_gaussian_b200.fdk import fdk
    from r2_gaussian_b200.projector import project

    pcl, pipe = _cloud_tensors(fc.round_trip_cloud())
    sc = fc.scanner("cone", fc.ROUND_TRIP_DET, fc.ROUND_TRIP_VOX)
    angles = fc.full_scan(180)
    vol = _query(pcl, pipe, sc)
    rec = fdk(project(vol, angles, sc), angles, sc).cpu().numpy()
    want = vol.cpu().numpy()
    err = pc.rel_l2(rec, want)
    assert err <= FDK_ROUND_TRIP_BOUND, err
    assert pc.rel_l2(rec[::-1], want) >= 0.5
    assert pc.rel_l2(rec[:, :, ::-1], want) >= 0.5


def test_deterministic():
    torch = _torch()
    from r2_gaussian_b200.projector import project

    sc = dict(fc.scanner("cone", 96, 40), accuracy=0.5)
    vol = torch.rand(40, 40, 40, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    angles = fc.full_scan(7)
    a, b = project(vol, angles, sc), project(vol, angles, sc)
    assert a.view(torch.int32).equal(b.view(torch.int32))           # bitwise, signed zeros included
    with pytest.raises(RuntimeError, match="CUDA"):
        project(vol.cpu(), angles, sc)


def test_project_512_cubed_grid():
    """512^3 volume (512 MiB), 1024^2 detector: a region of pixels whose rays cross the far (+x, +y, +z) part of the
    grid agrees with the oracle."""
    torch = _torch()
    from r2_gaussian_b200.projector import project

    sc = fc.scanner("cone", 1024, 512)
    angles = [math.pi / 4, 3.5]
    vol = torch.rand(512, 512, 512, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    projs = project(vol, angles, sc)
    host = vol.cpu().numpy()
    del vol
    r0, c0, n = 816, 816, 12                                          # ndc ~ (0.6, 0.6): rays through the top corner
    for i, a in enumerate(angles):
        o, d = po.rays(scene.make_view(sc, a))
        want = po.project_rays(host, o[r0:r0 + n, c0:c0 + n], d[r0:r0 + n, c0:c0 + n], True, sc["sVoxel"],
                               sc["offOrigin"], po.step_length(sc))
        got = projs[i, r0:r0 + n, c0:c0 + n].cpu().numpy()
        assert np.abs(want).min() > 0.0
        assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max(), i
    del projs
    torch.cuda.empty_cache()


# ---- generate_data end to end --------------------------------------------------------------------------------------

def _write_inputs(tmp_path, noise: bool):
    """A yml in physical units (sVoxel 4: scene scale 0.5) and vol_gt.npy = query(round_trip_cloud) on the scaled grid,
    with the detector and grid sizes of the round trip."""
    sc = scene.cone_beam_scanner(pc.ROUND_TRIP_DET, pc.ROUND_TRIP_VOX)
    phys = {k: (np.asarray(v, float) * 2.0).tolist() if k in ("DSD", "DSO", "sDetector", "sVoxel", "offOrigin",
                                                              "offDetector") else v for k, v in sc.items()}
    phys.update({"filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 30.0, "noise": noise,
                 "possion_noise": 100000, "gaussian_noise": [0, 10]})
    yml = tmp_path / ("noisy.yml" if noise else "clean.yml")
    lines = []
    for k, v in phys.items():
        lines.append(f"{k}: {json.dumps(v)}")                        # JSON values are valid YAML flow scalars/lists
    yml.write_text("\n".join(lines) + "\n")
    pcl, pipe = _cloud_tensors(fc.round_trip_cloud())
    vol_path = tmp_path / "vol.npy"
    if not vol_path.exists():
        np.save(vol_path, _query(pcl, pipe, sc).cpu().numpy())
    return yml, vol_path, sc, pcl, pipe


def _tree_bytes(root):
    out = {}
    for d, _, files in os.walk(root):
        for f in files:
            p = os.path.join(d, f)
            with open(p, "rb") as fh:
                out[os.path.relpath(p, root)] = fh.read()
    return out


def test_generate_data_end_to_end(tmp_path, capsys):
    from r2_gaussian_b200 import generate_data, initialize_pcd
    from r2_gaussian_b200.dataset import read_blender

    n_train, n_test = 24, 6
    yml, vol_path, sc, pcl, pipe = _write_inputs(tmp_path, noise=True)
    args = ["--vol", str(vol_path), "--scanner", str(yml), "--n_train", str(n_train), "--n_test", str(n_test)]
    case = generate_data.main(args + ["--output", str(tmp_path / "a")])
    again = generate_data.main(args + ["--output", str(tmp_path / "b")])
    assert os.path.basename(case) == "vol_cone"
    assert _tree_bytes(case) == _tree_bytes(again)                   # seeded: byte-identical
    other = generate_data.main(args + ["--output", str(tmp_path / "c"), "--seed", "1"])
    assert _tree_bytes(case)["proj_train/proj_train_0000.npy"] != _tree_bytes(other)["proj_train/proj_train_0000.npy"]
    assert "Generate data for case vol_cone complete!" in capsys.readouterr().out

    with open(os.path.join(case, "meta_data.json")) as f:
        meta = json.load(f)
    assert set(meta) >= {"scanner", "vol", "bbox", "proj_train", "proj_test"}
    assert meta["scanner"]["sVoxel"] == [4.0, 4.0, 4.0] and meta["vol"] == "vol_gt.npy"
    assert [fr["file_path"] for fr in meta["proj_test"]] == [f"proj_test/proj_test_{i:04d}.npy" for i in range(n_test)]
    info = read_blender(case)
    assert info.scene_scale == 0.5
    assert len(info.train_cameras) == n_train and len(info.test_cameras) == n_test
    start = math.radians(30.0)
    test_angles = np.array([c.angle for c in info.test_cameras])
    assert (np.diff(test_angles) >= 0).all() and (test_angles >= start).all() and (test_angles < start + 2 * math.pi).all()
    train_angles = np.array([c.angle for c in info.train_cameras])
    np.testing.assert_allclose(train_angles, start + np.arange(n_train) * 2 * math.pi / n_train, rtol=0, atol=1e-12)
    assert all((np.asarray(c.image) >= 0).all() for c in info.train_cameras)

    # the noise-free views match render(cloud) once read back in scene units
    yml_clean, *_ = _write_inputs(tmp_path, noise=False)
    clean = generate_data.main(["--vol", str(vol_path), "--scanner", str(yml_clean), "--n_train", str(n_train),
                                "--n_test", str(n_test), "--output", str(tmp_path / "clean")])
    info_clean = read_blender(clean)
    got = np.stack([c.image for c in info_clean.train_cameras])
    want = _render(pcl, pipe, sc, train_angles).cpu().numpy()
    err = pc.rel_l2(got, want)
    assert err <= pc.ROUND_TRIP_BOUND, err
    assert pc.rel_l2(np.stack([c.image for c in info.train_cameras]), got) > 0.0      # the noisy case differs

    capsys.readouterr()
    out = initialize_pcd.main(["--data", case, "--recon_method", "fdk", "--n_points", "400", "--evaluate"])
    assert os.path.exists(out)
    psnr = re.findall(r"3D PSNR for initial Gaussians: (\S+)", capsys.readouterr().out)
    assert len(psnr) == 1 and math.isfinite(float(psnr[0])), psnr


def test_generate_data_rejects_a_volume_of_the_wrong_shape(tmp_path):
    from r2_gaussian_b200 import generate_data

    yml, vol_path, *_ = _write_inputs(tmp_path, noise=False)
    bad = tmp_path / "bad.npy"
    np.save(bad, np.zeros((8, 8, 8), np.float32))
    with pytest.raises(SystemExit, match="nVoxel"):
        generate_data.main(["--vol", str(bad), "--scanner", str(yml), "--output", str(tmp_path / "out")])
    assert not os.path.exists(tmp_path / "out")
