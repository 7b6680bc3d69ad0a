#!/usr/bin/env python
"""Device time of the headline rasterizer backward with and without the view- / projection-matrix gradients (the
bench.py scene: 100k Gaussians, init-like, seed 0, 512x512 cone beam, 50 views cycled).

    python scripts/gpu/pose_grad_bench.py [--steps 200] [--warmup 20] [--out FILE]

One forward per view (kept), then the two backward variants alternate step by step -- r2x_raster_backward and
r2x_raster_backward_pose -- each timed with CUDA events after an L2 flush (256 MiB memset), as in forward_breakdown.py.
A second, profiled pass (torch.profiler, CUDA activities) gives the per-kernel split of both.  Prints one JSON object
with the card and its power limit."""
from __future__ import annotations

import argparse
import json
import os
import sys

HERE_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, HERE_ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    from forward_breakdown import card
    from r2_gaussian_b200 import _C, scene

    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    views = scene.make_views(scene.cone_beam_scanner(512, 256), 50)
    cloud = scene.make_cloud(100_000, kind="init", seed=0)
    t = lambda a: torch.tensor(a, device=dev)
    means, scales, rots, dens = t(cloud.means), t(cloud.scales), t(cloud.rotations), t(cloud.density)
    empty = torch.empty(0, device=dev)
    dL = torch.rand((1, 512, 512), device=dev)
    fwd = []
    for v in views:
        tv, tp, tc = t(v.viewmatrix), t(v.projmatrix), t(v.campos)
        R, _, radii, geom, binning, img = _C.rasterize_gaussians(means, dens, scales, rots, 1.0, empty, tv, tp, v.tanfovx,
                                                                 v.tanfovy, 512, 512, tc, False, v.mode, False)
        fwd.append((tv, tp, tc, v, R, radii, geom, binning, img))

    def backward(i, matrices):
        tv, tp, tc, v, R, radii, geom, binning, img = fwd[i % len(fwd)]
        fn = _C.rasterize_gaussians_backward_matrices if matrices else _C.rasterize_gaussians_backward
        return fn(means, radii, scales, rots, 1.0, empty, tv, tp, v.tanfovx, v.tanfovy, dL, tc, geom, R, binning, img,
                  v.mode, False)

    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for i in range(args.warmup):
        backward(i, False)
        backward(i, True)
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for i in range(args.steps):
        for m in ((False, True) if i % 2 == 0 else (True, False)):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            backward(i, m)
            b.record()
            torch.cuda.synchronize()
            times[m].append(a.elapsed_time(b) * 1000.0)

    def split(matrices):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(args.steps):
                backward(i, matrices)
            torch.cuda.synchronize()
        rows = {}
        for e in prof.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            dur = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            r = rows.setdefault(e.name, [0, 0.0])
            r[0] += 1
            r[1] += float(dur)
        return [{"name": n, "launches_per_backward": c / args.steps, "us_per_backward": tot / args.steps}
                for n, (c, tot) in sorted(rows.items(), key=lambda kv: -kv[1][1])]

    plain, pose = np.array(times[False]), np.array(times[True])
    out = dict(card(), workload="bench.py scene: 100000 Gaussians (init-like, seed 0), 512x512 cone beam, 50 views",
               steps=args.steps, l2_flushed=True,
               backward_us={"plain_mean": float(plain.mean()), "plain_median": float(np.median(plain)),
                            "matrices_mean": float(pose.mean()), "matrices_median": float(np.median(pose))},
               overhead_us_median=float(np.median(pose) - np.median(plain)),
               kernels_plain=split(False), kernels_matrices=split(True),
               timing="CUDA events around one backward call after an L2 flush, the two variants alternating; kernel "
                      "split from torch.profiler CUDA activity durations in a separate pass")
    s = json.dumps(out)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
