#!/usr/bin/env python
"""Batched views against a loop of single views: device time of projecting one cloud into N views (default 50).

    python scripts/gpu/views_bench.py [--views 50] [--steps 20] [--warmup 5] [--out FILE]

Two scenes: 50k init-like Gaussians on a 256x256 cone-beam detector, and the bench.py scene (100k, 512x512 cone).
For each, with persistent workspaces and no host synchronisation inside the timed window:
  loop     N x RasterEngine.forward (r2x_raster_forward_async), one view after the other;
           forward + backward: each forward followed by r2x_raster_backward of that view;
  batched  one RasterEngine.forward_views (r2x_raster_forward_views_async) of the N views;
           forward + backward: followed by one r2x_raster_backward_views.
The variants alternate step by step and each step is timed with CUDA events after warm-up.  The batched images are
checked bit for bit against the loop's before timing.  Prints one JSON object with the card and its power limit."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


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


def run_scene(name, P, n_det, n_views, steps, warmup) -> dict:
    import torch

    from r2_gaussian_b200 import _C, engine, scene
    from r2_gaussian_b200._lib import check

    sc = scene.cone_beam_scanner(n_det, 256)
    views = scene.make_views(sc, n_views)
    cloud = scene.make_cloud(P, kind="init", seed=0)
    dev = torch.device("cuda")
    means = torch.tensor(cloud.means, device=dev); dens = torch.tensor(cloud.density, device=dev)
    scales = torch.tensor(cloud.scales, device=dev); rots = torch.tensor(cloud.rotations, device=dev)
    vm = torch.stack([torch.tensor(v.viewmatrix, device=dev) for v in views])
    pm = torch.stack([torch.tensor(v.projmatrix, device=dev) for v in views])
    campos = torch.zeros(3, device=dev)
    v0 = views[0]
    W, H, N = v0.image_width, v0.image_height, n_views
    tx, ty, mode = v0.tanfovx, v0.tanfovy, v0.mode
    dL = torch.randn((N, H, W), device=dev, generator=torch.Generator("cuda").manual_seed(0))

    single = engine.RasterEngine(P, W, H)
    batched = engine.RasterEngine(P, W, H)
    lib = single.lib
    # provision both workspaces: the loop's for the largest view, the batch's for all views at once
    loop_img = torch.empty((N, 1, H, W), device=dev)
    for v in range(N):
        while True:
            single.forward(means, dens, scales, rots, vm[v], pm[v], campos, tx, ty, mode, out=loop_img[v])
            if single.check():
                break
    while True:
        batched.forward_views(means, dens, scales, rots, vm, pm, tx, ty, mode)
        if batched.check():
            break
    torch.cuda.synchronize()
    assert batched.forward_views(means, dens, scales, rots, vm, pm, tx, ty, mode).view(torch.int32).equal(
        loop_img[:, 0].contiguous().view(torch.int32)), "batched images differ from the single-view loop"

    f32 = dict(dtype=torch.float32, device=dev)
    g1 = [torch.empty((P, k), **f32) for k in (3, 1, 1, 3, 6, 3, 4)]
    gN = [torch.empty((N, P, 3), **f32)] + [torch.empty((P, k), **f32) for k in (1, 3, 6, 3, 4)]
    s1 = _C.RASTER.bwd_scratch(single.capacity, dev)
    sN = _C.RASTER.bwd_scratch(batched.capacity, dev)
    stream = lambda: torch.cuda.current_stream(dev).cuda_stream
    p = lambda t: t.data_ptr()

    def loop(backward: bool):
        for v in range(N):
            single.forward(means, dens, scales, rots, vm[v], pm[v], campos, tx, ty, mode, out=loop_img[v])
            if backward:
                check(lib.r2x_raster_backward(stream(), P, single.capacity, W, H, p(means), p(scales), 1.0, p(rots),
                                              None, p(vm[v]), p(pm[v]), None, tx, ty, p(single.radii), p(single.geom),
                                              p(single.binning), p(single.img), p(s1), p(dL[v]), *map(p, g1), mode, 0),
                      "r2x_raster_backward")

    def batch(backward: bool):
        batched.forward_views(means, dens, scales, rots, vm, pm, tx, ty, mode)
        if backward:
            geom, img, radii, _ = batched._views[N]
            check(lib.r2x_raster_backward_views(stream(), P, N, batched.capacity, W, H, p(means), p(scales), 1.0,
                                                p(rots), p(vm), p(pm), tx, ty, p(radii), p(geom), p(batched.binning),
                                                p(img), p(sN), p(dL), *map(p, gN), mode, 0),
                  "r2x_raster_backward_views")

    out = {"scene": name, "P": P, "W": W, "H": H, "views": N, "R_batched": batched.num_rendered()}
    for backward in (False, True):
        times = {"loop": [], "batched": []}
        for step in range(warmup + steps):
            for label, fn in (("loop", loop), ("batched", batch)):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn(backward)
                b.record()
                b.synchronize()
                if step >= warmup:
                    times[label].append(a.elapsed_time(b))
        assert single.check() and batched.check(), "a timed forward overflowed its workspace"
        key = "forward_backward" if backward else "forward"
        lo = sorted(times["loop"])[len(times["loop"]) // 2]
        ba = sorted(times["batched"])[len(times["batched"]) // 2]
        out[key] = {"loop_ms_median": round(lo, 3), "batched_ms_median": round(ba, 3),
                    "loop_ms_min": round(min(times["loop"]), 3), "batched_ms_min": round(min(times["batched"]), 3),
                    "speedup_median": round(lo / ba, 3)}
    return out


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=50)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("views_bench.py needs a CUDA device")
    res = {"card": card(), "steps": args.steps, "warmup": args.warmup, "scenes": []}
    for name, P, n_det in (("50k_256_cone", 50_000, 256), ("bench_100k_512_cone", 100_000, 512)):
        res["scenes"].append(run_scene(name, P, n_det, args.views, args.steps, args.warmup))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
