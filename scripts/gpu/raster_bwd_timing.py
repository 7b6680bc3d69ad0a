"""Time the rasterizer's backward render kernel (raster_render_bwd2_kernel) on the bench scene: 100k Gaussians,
512x512 cone beam, init-like and trained-like clouds.

    python scripts/gpu/raster_bwd_timing.py [--reps 200] [--rounds 5]

The kernel's own device time from torch.profiler (the per-Gaussian chain and the rest of
_C.rasterize_gaussians_backward are left out), averaged over the launches the profiler recorded of `reps` backward calls per round, a 256 MiB memset between calls so
that every call starts from a cold L2; one JSON line per cloud with the per-round means (us per call) and their median.
To compare two builds, run it on both trees alternately from one shell command (A B A B ...), so that both see the
same clocks and neighbours.

Taking the backward's row moments about the column nearest each Gaussian's centre instead of the tile's column 0
(exact-path pixels re-centred, fast-path run sums rebased once per instance) measured, on an H100 80GB HBM3 at 700 W,
raster_render_bwd2_kernel, alternating builds: init 171.7 / 170.2 -> 170.6 us, trained 207.5 / 205.8 -> 206.0 us
(before -> after): within noise.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "tests"))

import util  # noqa: E402
from r2_gaussian_b200 import _C, scene  # noqa: E402


def _kernel_us(prof, name):
    tot, n = 0.0, 0
    for e in prof.key_averages():
        if name in e.key:
            tot += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            n += e.count
    return tot / max(n, 1), n


def main():
    from torch.profiler import ProfilerActivity, profile

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    view = scene.make_view(scene.cone_beam_scanner(512, 256), 0.3)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for kind in ("init", "trained"):
        cloud = scene.make_cloud(100000, kind=kind, seed=0)
        fwd = util.ours_raster_forward(cloud, view, export=False)
        t = fwd["t"]
        geom, binning, img = fwd["state"]
        radii = torch.tensor(fwd["radii"], device="cuda")
        dL = torch.rand((1, 512, 512), device="cuda") + 0.5
        call = lambda: _C.rasterize_gaussians_backward(
            t["means"], radii, t["scales_in"], t["rots_in"], 1.0, t["cov_in"], t["view"], t["proj"], view.tanfovx,
            view.tanfovy, dL, t["campos"], geom, fwd["R"], binning, img, view.mode, False)
        for _ in range(10):
            call()
        torch.cuda.synchronize()
        rounds = []
        for _ in range(args.rounds):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    flush.zero_()
                    call()
                torch.cuda.synchronize()
            us, n = _kernel_us(prof, "raster_render_bwd2")
            assert n >= 0.9 * args.reps, f"expected {args.reps} raster_render_bwd2 launches, profiled {n}"
            rounds.append(us)
        print(json.dumps(dict(cloud=kind, num_rendered=int(fwd["R"]), kernel="raster_render_bwd2_kernel",
                              median_us=float(np.median(rounds)), rounds_us=[round(x, 2) for x in rounds],
                              gpu=torch.cuda.get_device_name())))


if __name__ == "__main__":
    main()
