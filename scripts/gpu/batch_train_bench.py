#!/usr/bin/env python
"""Training on B views per optimizer step: speed of `NativeTrainStep` with a list of cameras, and reconstruction
quality of `trainer --batch_size`.

    python scripts/gpu/batch_train_bench.py [--steps 200] [--warmup 20] [--quality 2000] [--out FILE]

Speed, two workloads: the bench.py scene (100k Gaussians, init-like, seed 0, 512x512 cone beam, 50 views, TV crop 32^3)
at B = 1, 2, 4, and 50k Gaussians (seed 3) at 256x256 at B = 1, 4, 16 (16 views of 256^2 are the most the direct
binning path of the stacked tile grid takes).  One model and one step per B; the variants alternate iteration by
iteration in the same process.  Every call starts from a synchronised GPU, so that the host time of the call is its
enqueue time; a ~2 ms spin kernel queued ahead of it keeps the GPU busy until the whole iteration is enqueued, so the
CUDA events around the call give the device time of one iteration without host gaps.  Reported per iteration and per
view (iteration / B).

Quality (`--quality K`, 0 skips it): the generate_data scene of the end-to-end tests (48^3 volume, 96^2 cone beam, 24
train / 6 test views, FDK initialisation of 2000 points) trained by the trainer at B = 1 for K iterations and at B = 4
for K / 4 iterations (the same number of views seen), with psnr_3d / ssim_3d and wall time, and the metrics of the
FDK initialisation itself.
Prints one JSON object with the card and its power limit."""
from __future__ import annotations

import argparse
import json
import os
import pathlib
import random
import sys
import tempfile
import time

HERE_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, HERE_ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def speed(args, name, P, det, seed, batches, tv_s):
    import numpy as np
    import torch

    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.gaussian_model import GaussianModel
    from r2_gaussian_b200.train_step import NativeTrainStep
    from r2_gaussian_b200.trainer import OptimizationParams

    dev = torch.device("cuda", 0)
    cams = [scene.camera_from_view(v) for v in scene.make_views(scene.cone_beam_scanner(det, 256), 50)]
    cloud = scene.make_cloud(P, kind="init", seed=seed)
    g = torch.Generator(device="cuda").manual_seed(0)
    gts = torch.rand((len(cams), det, det), device=dev, generator=g) * 0.5
    rng = np.random.RandomState(0)
    tv_n = [32, 32, 32]
    centres = [tuple(rng.uniform(-0.85, 0.85, 3)) for _ in range(args.warmup + args.steps)]

    def model():
        gm = GaussianModel(np.array([0.0005, 0.5]) * 2.0)
        gm.create_from_pcd(cloud.means, cloud.density, 1.0)
        gm.training_setup(OptimizationParams())
        return gm

    steps = {B: NativeTrainStep(model(), 0.25, 0.05, tv_n, tv_s) for B in batches}
    dev_us, host_us = {B: [] for B in batches}, {B: [] for B in batches}
    for i in range(args.warmup + args.steps):
        order = batches[i % len(batches):] + batches[:i % len(batches)]      # rotate which variant goes first
        for B in order:
            idx = [(i * B + j) % len(cams) for j in range(B)]
            cam = cams[idx[0]] if B == 1 else [cams[j] for j in idx]
            gt = gts[idx[0]:idx[0] + 1] if B == 1 else gts[idx]
            step = steps[B]
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
                dev_us[B].append(a.elapsed_time(b) * 1000.0)
                host_us[B].append((t1 - t0) * 1e6)
    for s in steps.values():
        s.flush()
    med = lambda x: float(np.median(x))
    rows = {}
    for B in batches:
        rows[f"B={B}"] = {"device_us_per_iteration": med(dev_us[B]), "device_us_per_view": med(dev_us[B]) / B,
                          "host_enqueue_us_per_iteration": med(host_us[B]),
                          "host_enqueue_us_per_view": med(host_us[B]) / B,
                          "device_mean_us_per_iteration": float(np.mean(dev_us[B])),
                          "views_per_second_device": B / (med(dev_us[B]) * 1e-6),
                          "repeated_iterations": steps[B].repeats}
    b1 = rows["B=1"]["device_us_per_view"]
    for B in batches:
        rows[f"B={B}"]["device_speedup_per_view_vs_B1"] = b1 / rows[f"B={B}"]["device_us_per_view"]
    return {"workload": name, "medians": rows}


def quality(iterations):
    import numpy as np
    import torch

    from r2_gaussian_b200 import generate_data, initialize_pcd, trainer
    from r2_gaussian_b200.dataset import Scene
    from r2_gaussian_b200.gaussian_model import GaussianModel

    sys.path.insert(0, os.path.join(HERE_ROOT, "tests"))
    from test_projector_gpu import _write_inputs     # the scene of the end-to-end tests (48^3 volume, 96^2 detector)

    tmp = pathlib.Path(tempfile.mkdtemp(prefix="batch_quality_"))
    yml, vol_path, *_ = _write_inputs(tmp, noise=False)
    path = generate_data.main(["--vol", str(vol_path), "--scanner", str(yml), "--n_train", "24", "--n_test", "6",
                               "--output", str(tmp / "data")])
    init = initialize_pcd.main(["--data", path, "--recon_method", "fdk", "--n_points", "2000",
                                "--output", str(tmp / "init.npy")])
    model0, opt0, pipe0 = trainer.ModelParams(source_path=path, ply_path=init), trainer.OptimizationParams(), \
        trainer.PipelineParams()
    sc = Scene(path, "", shuffle=False)
    gm = GaussianModel(trainer.derived_settings(sc.scanner_cfg, model0, opt0)["scale_bound"])
    pts = np.load(init)
    gm.create_from_pcd(pts[:, :3], pts[:, 3:4], 1.0)
    ev0 = trainer.evaluate(sc, gm, pipe0)
    out = {"workload": f"generate_data scene: 48^3 volume, 96x96 cone beam, 24 train / 6 test views, FDK init of "
                       f"2000 points; B = 1 for {iterations} iterations against B = 4 for {iterations // 4}",
           "fdk_init": {"psnr_3d": float(ev0["psnr_3d"]), "ssim_3d": float(ev0["ssim_3d"])}}
    for B, it in ((1, iterations), (4, iterations // 4)):
        random.seed(0); np.random.seed(0); torch.manual_seed(0)
        model = trainer.ModelParams(source_path=path, model_path="", ply_path=init)
        opt = trainer.OptimizationParams(iterations=it)
        hist = trainer.training(model, opt, trainer.PipelineParams(), {it}, log=lambda *a: None, batch_size=B)
        ev = hist["eval"][it]
        out[f"B={B}"] = {"iterations": it, "views_seen": it * B, "psnr_3d": float(ev["psnr_3d"]),
                         "ssim_3d": float(ev["ssim_3d"]), "train_seconds": hist["train_seconds"],
                         "seconds_with_eval": hist["seconds"], "gaussians": hist["gaussians"]}
    return out


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--quality", type=int, default=2000, help="B = 1 iterations of the quality run (0: skip it)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from forward_breakdown import card

    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    torch.cuda.set_device(0)
    out = dict(card(), steps=args.steps, warmup=args.warmup,
               timing="each call after a synchronise and a ~2 ms spin kernel; CUDA events around the call (device), "
                      "perf_counter around it (host enqueue); the variants alternate; medians",
               speed=[speed(args, "bench.py scene: 100000 Gaussians (init-like, seed 0), 512x512 cone beam, 50 views, "
                                  "TV crop 32^3", 100_000, 512, 0, [1, 2, 4], [0.25, 0.25, 0.25]),
                      speed(args, "50000 Gaussians (init-like, seed 3), 256x256 cone beam, 50 views, TV crop 32^3",
                            50_000, 256, 3, [1, 4, 16], [0.25, 0.25, 0.25])])
    if args.quality > 0:
        out["quality"] = quality(args.quality)
    s = json.dumps(out)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
