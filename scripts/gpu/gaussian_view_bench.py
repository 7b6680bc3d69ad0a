"""A trained model's Gaussians as ellipsoids on the GPU (r2x_scene_raster's ellipsoid kind, `visualize_scene
--gaussians`):

    python scripts/gpu/gaussian_view_bench.py [--reps 10]

Cases, at 1000 x 800 (the visualize_scene default) from `scene_view.default_view`: 100k and 500k Gaussians of a
trained-like cloud (`scene.make_cloud(..., kind="trained")`: random rotations, anisotropic scales) as one frame and as
a 36-frame orbit in one call.  Each case times the r2x_scene_raster call alone with CUDA events (records and outputs
allocated once), median of --reps after one warm-up call, an L2-sized buffer written between calls.  `select_ms` times
`gaussian_ellipsoids` (filter, stable sort by density, colours, records) on its own, the same way.  Prints one JSON
line per case and one with the card's name, power limit and SM clocks read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "scripts", "gpu"))


class CloudModel:
    """The accessors `gaussian_ellipsoids` reads, over a scene.Cloud on the device."""

    def __init__(self, cloud, dev):
        import torch
        t = lambda a: torch.as_tensor(a, device=dev)
        self.get_xyz, self.get_scaling = t(cloud.means), t(cloud.scales)
        self.get_rotation, self.get_density = t(cloud.rotations), t(cloud.density)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    import numpy as np
    import torch

    import secondary
    from mesh_bench import clocks
    from r2_gaussian_b200 import scene
    from r2_gaussian_b200 import scene_view as sv
    from r2_gaussian_b200._lib import check, load

    if not torch.cuda.is_available():
        raise SystemExit("gaussian_view_bench needs a CUDA device")
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
    for P in (100_000, 500_000):
        model = CloudModel(scene.make_cloud(P, kind="trained", seed=0), dev)
        select_ms = timed(lambda: sv.gaussian_ellipsoids(model, None, "density"))
        prims, _ = sv.gaussian_ellipsoids(model, None, "density")
        cam = sv.default_view(prims, W, H)
        for frames in (1, 36):
            cams = sv.scan_orbit(cam, frames) if frames > 1 else [cam]
            n, F = len(prims), len(cams)
            rec = torch.from_numpy(np.stack([c.record() for c in cams])).to(dev)
            lut = torch.tensor([[0.0, 0.0, 0.0], [1.0, 1.0, 1.0]], device=dev)
            nbytes = int(lib.r2x_scene_raster_scratch_bytes(n, F))
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            keys = torch.empty((F, H, W), dtype=torch.int64, device=dev)
            rgb = torch.empty((F, H, W, 3), dtype=torch.float32, device=dev)
            bg = np.ones(3, np.float32)
            call = lambda: check(lib.r2x_scene_raster(stream, n, prims.pos.data_ptr(), prims.meta.data_ptr(),
                                                      prims.attr.data_ptr(), 0, 1, 1, None, lut.data_ptr(), 2, F, H, W,
                                                      rec.data_ptr(), 0, sv.NEAR, bg.ctypes.data, keys.data_ptr(),
                                                      rgb.data_ptr(), scratch.data_ptr(), nbytes), "r2x_scene_raster")
            ms = timed(call)
            first = keys.clone()
            call()
            row = {"case": f"gaussians_{P // 1000}k" + (f"_orbit{F}" if F > 1 else ""), "gaussians": n, "frames": F,
                   "width": W, "height": H, "ms": ms, "ms_per_frame": ms / F, "select_ms": select_ms,
                   "covered_fraction": float((keys != -1).float().mean()),
                   "reproducible": bool(torch.equal(first, keys)), "scratch_mb": nbytes / 2**20}
            if F > 1:
                one = sv.render(prims, cams[5], return_keys=True)[1]
                row["orbit_frame_equals_single"] = bool(torch.equal(one[0], keys[5]))
            print(json.dumps(row), flush=True)
            del scratch, keys, rgb, first
            torch.cuda.empty_cache()
    print(json.dumps({**secondary.card(dev), **clocks()}))


if __name__ == "__main__":
    main()
