#!/usr/bin/env python
"""Learning the horizontal detector offset in training: cost of `NativeTrainStep(detector=...)` per iteration, and
recovery of a known shift through `trainer --detector_offset_refine`.

    python scripts/gpu/detector_offset_bench.py [--steps 200] [--warmup 20] [--recovery 2000]
                                                [--rates 5e-2:5e-4 ...] [--out FILE]

Speed: the bench.py scene (100k Gaussians, init-like, seed 0, 512x512 cone beam, 50 views, TV crop 32^3) at B = 1 and
B = 4, each without and with the detector offset.  One model and one step per variant; the variants alternate
iteration by iteration in the same process.  Every call starts from a synchronised GPU, so that the host time of the
call is its enqueue time; a ~2 ms spin kernel queued ahead of it keeps the GPU busy until the whole iteration is
enqueued, so the CUDA events around the call give the device time of one iteration without host gaps.

Recovery (`--recovery K`, 0 skips it): the generate_data scene of the end-to-end tests (48^3 volume, 96^2 cone beam,
24 train / 6 test views, no noise), as generated and with every projection moved 3 columns towards larger index,
each initialised by FDK of its own views, trained K iterations from seed 0 without the switch and with it at every
`--rates init:final` pair: the offset reached, psnr_3d and the training time.
Prints one JSON object with the card and its power limit."""
from __future__ import annotations

import argparse
import json
import os
import pathlib
import re
import shutil
import sys
import tempfile
import time

HERE_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, HERE_ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def speed(args, P, det, seed, batches):
    import numpy as np
    import torch

    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.detector import DetectorOffset
    from r2_gaussian_b200.gaussian_model import GaussianModel
    from r2_gaussian_b200.optim import FusedAdam
    from r2_gaussian_b200.train_step import NativeTrainStep
    from r2_gaussian_b200.trainer import OptimizationParams

    dev = torch.device("cuda", 0)
    cams = [scene.camera_from_view(v) for v in scene.make_views(scene.cone_beam_scanner(det, 256), 50)]
    cloud = scene.make_cloud(P, kind="init", seed=seed)
    g = torch.Generator(device="cuda").manual_seed(0)
    gts = torch.rand((len(cams), det, det), device=dev, generator=g) * 0.5
    rng = np.random.RandomState(0)
    tv_n, tv_s = [32, 32, 32], [0.25, 0.25, 0.25]
    centres = [tuple(rng.uniform(-0.85, 0.85, 3)) for _ in range(args.warmup + args.steps)]

    def model():
        gm = GaussianModel(np.array([0.0005, 0.5]) * 2.0)
        gm.create_from_pcd(cloud.means, cloud.density, 1.0)
        gm.training_setup(OptimizationParams())
        return gm

    def detector():
        d = DetectorOffset(dev)
        return d, FusedAdam([d.offset], lr=1e-2, eps=1e-15)

    variants = [(B, on) for B in batches for on in (False, True)]
    steps = {v: NativeTrainStep(model(), 0.25, 0.05, tv_n, tv_s, **({"detector": detector()} if v[1] else {}))
             for v in variants}
    dev_us, host_us = {v: [] for v in variants}, {v: [] for v in variants}
    for i in range(args.warmup + args.steps):
        order = variants[i % len(variants):] + variants[:i % len(variants)]     # rotate which variant goes first
        for v in order:
            B = v[0]
            idx = [(i * B + j) % len(cams) for j in range(B)]
            cam = cams[idx[0]] if B == 1 else [cams[j] for j in idx]
            gt = gts[idx[0]:idx[0] + 1] if B == 1 else gts[idx]
            step = steps[v]
            step.flush()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(4_000_000)        # ~2 ms of GPU work ahead of the call: no host gap inside the events
            a.record()
            t0 = time.perf_counter()
            step(cam, gt, centres[i])
            t1 = time.perf_counter()
            b.record()
            torch.cuda.synchronize()
            if i >= args.warmup:
                dev_us[v].append(a.elapsed_time(b) * 1000.0)
                host_us[v].append((t1 - t0) * 1e6)
    for s in steps.values():
        s.flush()
    med = lambda x: float(np.median(x))
    rows = {}
    for B in batches:
        off, on = (B, False), (B, True)
        rows[f"B={B}"] = {"device_us_per_iteration_without": med(dev_us[off]), "device_us_per_iteration_with": med(dev_us[on]),
                          "device_us_added": med(dev_us[on]) - med(dev_us[off]),
                          "host_enqueue_us_without": med(host_us[off]), "host_enqueue_us_with": med(host_us[on]),
                          "host_enqueue_us_added": med(host_us[on]) - med(host_us[off]),
                          "repeated_iterations": steps[off].repeats + steps[on].repeats}
    return {"workload": f"bench.py scene: {P} Gaussians (init-like, seed {seed}), {det}x{det} cone beam, 50 views, "
                        f"TV crop 32^3", "medians": rows}


def kernel_times(args, P, det, seed, batches, n_it=30):
    """Device time of each detector-offset kernel per iteration (torch.profiler, a run of its own after the timed one):
    what the added device time of the step is made of, apart from launch gaps."""
    import numpy as np
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.detector import DetectorOffset
    from r2_gaussian_b200.gaussian_model import GaussianModel
    from r2_gaussian_b200.optim import FusedAdam
    from r2_gaussian_b200.train_step import NativeTrainStep
    from r2_gaussian_b200.trainer import OptimizationParams

    dev = torch.device("cuda", 0)
    cams = [scene.camera_from_view(v) for v in scene.make_views(scene.cone_beam_scanner(det, 256), 50)]
    cloud = scene.make_cloud(P, kind="init", seed=seed)
    gts = torch.rand((len(cams), det, det), device=dev, generator=torch.Generator(device="cuda").manual_seed(0)) * 0.5
    out = {}
    for B in batches:
        gm = GaussianModel(np.array([0.0005, 0.5]) * 2.0)
        gm.create_from_pcd(cloud.means, cloud.density, 1.0)
        gm.training_setup(OptimizationParams())
        d = DetectorOffset(dev)
        step = NativeTrainStep(gm, 0.25, 0.05, [32, 32, 32], [0.25, 0.25, 0.25],
                               detector=(d, FusedAdam([d.offset], lr=1e-2, eps=1e-15)))

        def one(i):
            idx = [(i * B + j) % len(cams) for j in range(B)]
            step(cams[idx[0]] if B == 1 else [cams[j] for j in idx],
                 gts[idx[0]:idx[0] + 1] if B == 1 else gts[idx], (0.0, 0.0, 0.0))
        for i in range(10):
            one(i)
        step.flush()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(n_it):
                one(10 + i)
            step.flush()
            torch.cuda.synchronize()
        tot = {}
        for e in prof.events():
            m = re.search(r"(detector_offset_\w+_kernel|adam_kernel)", e.name)
            if e.device_type == DeviceType.CUDA and m:
                key = m.group(1)
                t, n = tot.get(key, (0.0, 0))
                tot[key] = (t + e.device_time, n + 1)     # device_time in us
        out[f"B={B}"] = {k: {"us_per_iteration": t / n_it, "launches_per_iteration": n / n_it} for k, (t, n) in tot.items()}
    return out


def recovery(iterations, rates):
    from r2_gaussian_b200 import trainer

    sys.path.insert(0, os.path.join(HERE_ROOT, "tests"))
    from detector_cases import SHIFT, recovery_scenes, train    # the recipe of the recovery test

    tmp = pathlib.Path(tempfile.mkdtemp(prefix="detector_recovery_"))
    try:
        scenes = recovery_scenes(tmp)
        out = {"workload": f"generate_data scene: 48^3 volume, 96x96 cone beam, 24 train / 6 test views, no noise, "
                           f"FDK init of 2000 points; every projection moved {SHIFT} columns towards larger index; "
                           f"{iterations} iterations from seed 0", "runs": []}
        for name in ("shifted", "plain"):
            path, init = scenes[name]
            for rate in [None] + rates:
                det = trainer.DetectorParams(detector_offset_refine=rate is not None,
                                             **({} if rate is None else dict(detector_offset_lr_init=rate[0],
                                                                             detector_offset_lr_final=rate[1])))
                h = train(path, init, "", det, iterations)
                ev = h["eval"][iterations]
                out["runs"].append({"scene": name, "rates": rate, "offset_px": h.get("detector_offset_px"),
                                    "psnr_3d": float(ev["psnr_3d"]), "ssim_3d": float(ev["ssim_3d"]),
                                    "psnr_2d_test": float(ev["psnr_2d_test"]), "train_seconds": h["train_seconds"]})
                print(json.dumps(out["runs"][-1]), file=sys.stderr)
        return out
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--recovery", type=int, default=2000, help="iterations of each recovery run (0: skip them)")
    ap.add_argument("--rates", nargs="+", default=None,
                    help="detector learning rates init:final of the recovery runs (default: DetectorParams')")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from forward_breakdown import card
    from r2_gaussian_b200.trainer import DetectorParams

    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    torch.cuda.set_device(0)
    rates = [tuple(float(x) for x in r.split(":")) for r in args.rates] if args.rates else \
        [(DetectorParams.detector_offset_lr_init, DetectorParams.detector_offset_lr_final)]
    out = dict(card(), steps=args.steps, warmup=args.warmup,
               timing="each call after a synchronise and a ~2 ms spin kernel; CUDA events around the call (device), "
                      "perf_counter around it (host enqueue); the variants alternate; medians")
    if args.steps > 0:
        out["speed"] = speed(args, 100_000, 512, 0, [1, 4])
        print(json.dumps(out["speed"]), file=sys.stderr)
        out["kernel_times"] = kernel_times(args, 100_000, 512, 0, [1, 4])
        print(json.dumps(out["kernel_times"]), file=sys.stderr)
    if args.recovery > 0:
        out["recovery"] = recovery(args.recovery, rates)
    s = json.dumps(out)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
