"""The scene-view rasterizer on the GPU (r2x_scene_raster, `scene_view.render`):

    python scripts/gpu/scene_view_bench.py [--reps 10]

Cases, at 1000 x 800 (the visualize_scene default) from `scene_view.default_view`:
  * phantom_256_cams50: the mesh of mesh_bench's 256^3 phantom at level 0.5 (about 279k triangles) in scene units
    ([-1, 1]^3), the two boxes and the frame, and 50 cone-beam camera glyphs with 512^2 textured image planes -- the
    picture visualize_scene draws of a 50-view scene;
  * query_cloud_256: the mesh of a 256^3 query() volume of a 200k-Gaussian cloud (mesh_bench's, about 3.28 M triangles);
  * phantom_256_cams50_orbit36: the first case as a 36-frame orbit in one call.
Each case times the r2x_scene_raster call alone with CUDA events (primitives, records and outputs allocated once),
median of --reps after one warm-up call, an L2-sized buffer written between calls.  Prints one JSON line per case and
one with the card's name, power limit and SM clocks read in the same run."""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "scripts", "gpu"))


def scene_primitives(vol, level, n_cams):
    import numpy as np

    from r2_gaussian_b200 import scene, scene_view as sv
    from r2_gaussian_b200.mesh import marching_cubes
    n = vol.shape[0]
    cfg = {"offOrigin": [0.0, 0.0, 0.0], "sVoxel": [2.0, 2.0, 2.0], "nVoxel": [n, n, n]}
    verts, faces = marching_cubes(vol, level)
    parts = [sv.mesh_triangles(verts, faces, vol, cfg), sv.box((0, 0, 0), (2, 2, 2), sv.RED),
             sv.box((0, 0, 0), (2, 2, 2), sv.BLUE), sv.axes((0, 0, 0), 1.0)]
    sc = scene.cone_beam_scanner(512, n)
    rng = np.random.default_rng(0)
    for i, angle in enumerate(np.linspace(0, 2 * math.pi, n_cams + 1)[:-1]):
        cam = scene.camera_from_view(scene.make_view(sc, float(angle)))
        cam.image_width = cam.image_height = 512
        img = rng.random((512, 512)).astype(np.float32)
        parts.append(sv.camera_glyph(cam, 1.0, (i / n_cams, 0.0, 1.0 - i / n_cams), image=img))
    return sv.concat(*parts), int(faces.shape[0])


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    import numpy as np
    import torch

    import secondary
    from mesh_bench import cloud_volume, clocks, phantom
    from r2_gaussian_b200 import scene_view as sv
    from r2_gaussian_b200._lib import check, load

    if not torch.cuda.is_available():
        raise SystemExit("scene_view_bench needs a CUDA device")
    dev = torch.device("cuda")
    lib = load()
    flush = torch.empty(64 << 20, dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream

    def timed(fn):
        fn()
        ms = []
        for _ in range(a.reps):
            flush.fill_(1.0)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            e.synchronize()
            ms.append(s.elapsed_time(e))
        ms.sort()
        return ms[len(ms) // 2]

    W, H = 1000, 800
    phantom_prims = scene_primitives(phantom(256, 1), 0.5, 50)
    vol = cloud_volume(256)
    cloud_prims = scene_primitives(vol, 0.3 * float(vol.max()), 0)
    del vol
    cases = [("phantom_256_cams50", phantom_prims, 1), ("query_cloud_256", cloud_prims, 1),
             ("phantom_256_cams50_orbit36", phantom_prims, 36)]
    for name, (prims, n_tris), frames in cases:
        cam = sv.default_view(prims, W, H)
        cams = sv.scan_orbit(cam, frames) if frames > 1 else [cam]
        n, F = len(prims), len(cams)
        rec = torch.from_numpy(np.stack([c.record() for c in cams])).to(dev)
        lut = torch.tensor([[0.0, 0.0, 0.0], [1.0, 1.0, 1.0]], device=dev)
        tex = prims.textures
        n_tex, th, tw = (0, 1, 1) if tex is None else tuple(int(s) for s in tex.shape)
        nbytes = int(lib.r2x_scene_raster_scratch_bytes(n, F))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        keys = torch.empty((F, H, W), dtype=torch.int64, device=dev)
        rgb = torch.empty((F, H, W, 3), dtype=torch.float32, device=dev)
        bg = np.ones(3, np.float32)
        call = lambda: check(lib.r2x_scene_raster(stream, n, prims.pos.data_ptr(), prims.meta.data_ptr(),
                                                  prims.attr.data_ptr(), n_tex, th, tw,
                                                  None if tex is None else tex.data_ptr(), lut.data_ptr(), 2, F, H, W,
                                                  rec.data_ptr(), 0, sv.NEAR, bg.ctypes.data, keys.data_ptr(),
                                                  rgb.data_ptr(), scratch.data_ptr(), nbytes), "r2x_scene_raster")
        ms = timed(call)
        first = keys.clone()
        call()
        row = {"case": name, "triangles_mesh": n_tris, "primitives": n, "frames": F, "width": W, "height": H,
               "ms": ms, "ms_per_frame": ms / F, "primitive_frames_per_s": n * F / (ms * 1e-3),
               "covered_fraction": float((keys != -1).float().mean()), "reproducible": bool(torch.equal(first, keys)),
               "scratch_mb": nbytes / 2**20}
        if frames > 1:
            one = sv.render(prims, cams[5], return_keys=True)[1]
            row["orbit_frame_equals_single"] = bool(torch.equal(one[0], keys[5]))
        print(json.dumps(row), flush=True)
        del scratch, keys, rgb
        torch.cuda.empty_cache()
    print(json.dumps({**secondary.card(dev), **clocks()}))


if __name__ == "__main__":
    main()
