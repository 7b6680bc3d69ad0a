#!/usr/bin/env python
"""Cost of pose refinement in the native training step: `NativeTrainStep` with and without `pose=` on the bench.py
scene (100k Gaussians, init-like, seed 0, 512x512 cone beam, 50 views cycled, TV crop 32^3).

    python scripts/gpu/pose_train_bench.py [--steps 200] [--warmup 20] [--out FILE]

Two models and two steps, one with a PoseCorrection over the 50 views (view 0 anchored) and one without, alternate
iteration by iteration in the same process.  Every call starts from a synchronised GPU, so that the host time of the
call is its enqueue time; a ~2 ms spin kernel queued ahead of it keeps the GPU busy until the whole iteration is
enqueued, so the CUDA events around the call give the device time of one iteration without host gaps.
Prints one JSON object with the card and its power limit."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

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

    from forward_breakdown import card
    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.gaussian_model import GaussianModel
    from r2_gaussian_b200.optim import FusedAdam
    from r2_gaussian_b200.pose import PoseCorrection
    from r2_gaussian_b200.train_step import NativeTrainStep
    from r2_gaussian_b200.trainer import OptimizationParams

    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    views = scene.make_views(scene.cone_beam_scanner(512, 256), 50)
    cams = []
    for v in views:
        c = scene.camera_from_view(v)
        c.projection_matrix = torch.tensor(scene.projection_matrix(v.FoVx, v.FoVy, v.mode).T.copy(), device=dev)
        cams.append(c)
    cloud = scene.make_cloud(100_000, kind="init", seed=0)
    g = torch.Generator(device="cuda").manual_seed(0)
    gts = [torch.rand((1, 512, 512), device=dev, generator=g) * 0.5 for _ in cams]
    rng = np.random.RandomState(0)
    tv_n, tv_s = [32, 32, 32], [0.25, 0.25, 0.25]          # 32 voxels of the 256^3 grid over sVoxel 2
    centres = [tuple(rng.uniform(-0.85, 0.85, 3)) for _ in range(args.warmup + args.steps)]

    def model():
        gm = GaussianModel(np.array([0.0005, 0.5]) * 2.0)
        gm.create_from_pcd(cloud.means, cloud.density, 1.0)
        gm.training_setup(OptimizationParams())
        return gm

    corr = PoseCorrection(len(cams), device=dev)
    pose_opt = FusedAdam([{"params": [corr.omega], "lr": 1e-3}, {"params": [corr.nu], "lr": 5e-3}], lr=0.0, eps=1e-15)
    steps = {False: NativeTrainStep(model(), 0.25, 0.05, tv_n, tv_s),
             True: NativeTrainStep(model(), 0.25, 0.05, tv_n, tv_s, pose=(corr, pose_opt), pose_anchor=0)}
    dev_us, host_us = {False: [], True: []}, {False: [], True: []}
    for i in range(args.warmup + args.steps):
        k = i % len(cams)
        for pose in ((False, True) if i % 2 == 0 else (True, False)):
            step = steps[pose]
            step.flush()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(4_000_000)        # ~2 ms of GPU work ahead of the call: no host gap inside the events
            a.record()
            t0 = time.perf_counter()
            step(cams[k], gts[k], centres[i], **({"view": k} if pose else {}))
            t1 = time.perf_counter()
            b.record()
            torch.cuda.synchronize()
            if i >= args.warmup:
                dev_us[pose].append(a.elapsed_time(b) * 1000.0)
                host_us[pose].append((t1 - t0) * 1e6)
    for s in steps.values():
        s.flush()
    stats = lambda x: {"mean": float(np.mean(x)), "median": float(np.median(x))}
    out = dict(card(), workload="bench.py scene: 100000 Gaussians (init-like, seed 0), 512x512 cone beam, 50 views, "
                                "TV crop 32^3, NativeTrainStep", steps=args.steps, warmup=args.warmup,
               device_us={"plain": stats(dev_us[False]), "pose": stats(dev_us[True])},
               host_enqueue_us={"plain": stats(host_us[False]), "pose": stats(host_us[True])},
               device_overhead_us_median=float(np.median(dev_us[True]) - np.median(dev_us[False])),
               host_overhead_us_median=float(np.median(host_us[True]) - np.median(host_us[False])),
               repeated_iterations={"plain": steps[False].repeats, "pose": steps[True].repeats},
               timing="each call after a synchronise and a ~2 ms spin kernel; CUDA events around the call (device), "
                      "perf_counter around it (host enqueue); the two variants alternate")
    s = json.dumps(out)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
