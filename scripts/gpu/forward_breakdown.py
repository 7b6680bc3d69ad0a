#!/usr/bin/env python
"""Per-kernel device time of the headline forward projection (the bench.py scene: 100k Gaussians, init-like, seed 0,
512x512 cone beam, 50 views cycled), measured with torch.profiler (CUDA activities).

    python scripts/gpu/forward_breakdown.py [--steps 200] [--warmup 20] [--no-flush] [--no-pdl] [--root DIR] [--out FILE]

Each forward goes through RasterEngine (r2x_raster_forward_async), like the bench's timed steps; as there, L2 is flushed
(256 MiB memset) before every forward unless --no-flush is given.  The flush kernel is listed on its own row and left
out of the forward's total.  The forward's kernels use programmatic dependent launch, so a kernel's recorded duration
starts while it still waits for its predecessor and the durations overlap; --no-pdl launches them one after the other,
which gives each kernel's own time.  --root imports r2_gaussian_b200 from another checkout, so two builds can be
compared with the same script.  Prints one JSON object: the card, its power limit, and the mean device time per launch
of every kernel and memset in the forward, in microseconds."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

HERE_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card() -> dict:
    import torch

    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"] = float(q[0])
        info["sm_clock_max_mhz"] = float(q[1])
    except Exception as e:  # informational
        info["power_limit_w"] = None
        info["nvidia_smi_error"] = str(e)
    return info


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--no-flush", action="store_true", help="do not flush L2 between forwards")
    ap.add_argument("--root", default=HERE_ROOT, help="checkout whose r2_gaussian_b200 is imported")
    ap.add_argument("--out", default=None, help="also write the JSON object to this file")
    ap.add_argument("--no-pdl", action="store_true",
                    help="launch without programmatic dependent launch (R2X_NO_PDL=1), so that no kernel becomes resident "
                         "before its predecessor ends and the per-kernel durations do not overlap")
    args = ap.parse_args()
    if args.no_pdl:
        os.environ["R2X_NO_PDL"] = "1"
    sys.path.insert(0, os.path.abspath(args.root))

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile

    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.engine import RasterEngine

    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    sc = scene.cone_beam_scanner(512, 256)
    views = scene.make_views(sc, 50)
    cloud = scene.make_cloud(100_000, kind="init", seed=0)
    t = lambda a: torch.tensor(a, device=dev)
    means, scales, rots, dens = t(cloud.means), t(cloud.scales), t(cloud.rotations), t(cloud.density)
    dv = [(t(v.viewmatrix), t(v.projmatrix), t(v.campos), v.tanfovx, v.tanfovy, v.mode) for v in views]
    eng = RasterEngine(cloud.P, 512, 512, dev)
    Rs = []
    for i in range(len(dv)):        # provision the capacity as bench.py does
        while True:
            eng.forward(means, dens, scales, rots, *dv[i])
            if eng.check():
                break
        Rs.append(eng.num_rendered())
    eng._reserve(int(max(Rs) * 1.25) + 4096)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def step(i):
        if not args.no_flush:
            flush.zero_()
        eng.forward(means, dens, scales, rots, *dv[i % len(dv)])

    for i in range(args.warmup):
        step(i)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(args.steps):
            step(i)
        torch.cuda.synchronize()
    assert eng.check(), "instance capacity overflowed"

    rows = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = e.name
        dur = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        r = rows.setdefault(name, [0, 0.0])
        r[0] += 1
        r[1] += float(dur)
    flush_names = [n for n in rows if not args.no_flush and rows[n][0] == args.steps and
                   ("fill" in n.lower() or "elementwise" in n.lower()) and "r2x" not in n and "raster" not in n]
    kernels = []
    for name, (n, tot) in sorted(rows.items(), key=lambda kv: -kv[1][1]):
        kernels.append({"name": name, "launches_per_forward": n / args.steps, "us_per_launch": tot / n,
                        "us_per_forward": tot / args.steps, "l2_flush": name in flush_names})
    fwd = sum(k["us_per_forward"] for k in kernels if not k["l2_flush"])
    short = {"raster_preprocess_kernel": 0.0, "direct_scan_kernel": 0.0, "direct_fill_kernel": 0.0, "render": 0.0}
    for k in kernels:
        for key in ("raster_preprocess_kernel", "direct_scan_kernel", "direct_fill_kernel"):
            if key in k["name"]:
                short[key] += k["us_per_forward"]
        if "raster_render" in k["name"]:
            short["render"] += k["us_per_forward"]
    out = dict(card(), workload="bench.py scene: 100000 Gaussians (init-like, seed 0), 512x512 cone beam, 50 views",
               root=os.path.abspath(args.root), steps=args.steps, l2_flushed=not args.no_flush, pdl=not args.no_pdl,
               num_rendered_mean=float(np.mean(Rs)), forward_device_us=fwd,
               front_end_us=short["raster_preprocess_kernel"] + short["direct_scan_kernel"] + short["direct_fill_kernel"],
               summary_us=short, kernels=kernels,
               timing="torch.profiler CUDA activity durations, mean over the profiled forwards")
    s = json.dumps(out)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
