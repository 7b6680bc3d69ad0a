"""Cost and benefit of FDK's truncation pad (r2x_fdk_pad through fdk.fdk(pad=...)):

    python scripts/gpu/fdk_pad_bench.py [--reps 20] [--train_iterations 1500] [--out DIR]

  * cost: the 50-view 512^2 -> 256^3 cone-beam circle (scripts/secondary.py's fdk row) at pad 0 (r2x_fdk), 0.25, 0.5
    and 1, Ram-Lak and Hann.  `call` is the whole r2x_fdk / r2x_fdk_pad call; `filter` is the same call onto a 1^3
    grid, whose backprojection (one thread, 50 views) is negligible next to the filter stage.  The variants run
    alternately; each time is the median of --reps calls timed with CUDA events after a warm-up.
  * benefit: the truncated and the untruncated scene of tests/test_fdk_pad_gpu.py (the same phantom with a detector
    covering 64 % of its lateral shadow, and all of it), reconstructed by `recon --methods fdk [--fdk_pad F]`, scored
    with psnr_3d and SSIM inside the field of view (the voxels every train view projects onto the detector; SSIM as
    metrics.metric_vol's with both volumes set to 0 outside it) and over the whole grid.  Then `initialize_pcd
    --recon_method fdk [--fdk_pad 0.5]` and --train_iterations of training from each initializer, scored by `test`.
Prints one JSON line with the card name and power limit (nvidia-smi)."""
from __future__ import annotations

import argparse
import json
import math
import os
import pathlib
import random
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

PADS = (0.0, 0.25, 0.5, 1.0)


def _median_ms(fns: dict, reps: int) -> dict:
    import torch
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():          # alternate the variants
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b))
    return {k: float(np.median(v)) for k, v in times.items()}


def cost(reps: int) -> dict:
    import torch

    from r2_gaussian_b200 import _lib, scene
    from r2_gaussian_b200.fdk import pad_pixels
    lib, dev = _lib.load(), torch.device("cuda")
    sc = scene.cone_beam_scanner(512, 256)
    N, H, W, n = 50, 512, 512, 256
    angles = np.linspace(0.0, 2.0 * math.pi, N + 1)[:-1]
    views = [scene.make_view(sc, float(t)) for t in angles]
    vm = torch.tensor(np.stack([v.viewmatrix.reshape(16) for v in views]), device=dev)
    pm = torch.tensor(np.stack([v.projmatrix.reshape(16) for v in views]), device=dev)
    projs = torch.rand(N, H, W, device=dev, generator=torch.Generator(dev).manual_seed(0))
    vol, one = torch.empty(n, n, n, device=dev), torch.empty(1, 1, 1, device=dev)
    nbytes = int(lib.r2x_fdk_scratch_bytes(N, H, W))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    tx, ty, dso = float(views[0].tanfovx), float(views[0].tanfovy), float(sc["DSO"])

    def call(window, pad, grid, out):
        def run():
            args = (torch.cuda.current_stream(dev).cuda_stream, N, H, W, projs.data_ptr(), vm.data_ptr(),
                    pm.data_ptr(), tx, ty, 1, 0.0, 0.0, window, None, 0.0, dso, *grid, out.data_ptr(),
                    scratch.data_ptr(), nbytes)
            L = pad_pixels(pad, W)
            _lib.check(lib.r2x_fdk_pad(*args, L) if pad > 0 else lib.r2x_fdk(*args), "fdk")
        return run

    big, small = (n, n, n, 2.0, 2.0, 2.0, 0.0, 0.0, 0.0), (1, 1, 1, 2.0, 2.0, 2.0, 0.0, 0.0, 0.0)
    res = {}
    for fname, window in (("ram_lak", 0x000), ("hann", 0x400)):
        fns = {}
        for pad in PADS:
            fns[f"call_pad{pad:g}"] = call(window, pad, big, vol)
            fns[f"filter_pad{pad:g}"] = call(window, pad, small, one)
        res[fname] = _median_ms(fns, reps)
    return res


def _in_field(gt, pred, fov) -> dict:
    import fdk_pad_oracle as fpo
    from r2_gaussian_b200.metrics import metric_vol
    return {"psnr_3d_fov": fpo.psnr_in(gt, pred, fov),
            "ssim_3d_fov": metric_vol(np.where(fov, gt, 0.0).astype(np.float32),
                                      np.where(fov, pred, 0.0).astype(np.float32), "ssim")[0],
            "psnr_3d": metric_vol(gt, pred, "psnr")[0], "ssim_3d": metric_vol(gt, pred, "ssim")[0]}


def benefit(tmp: pathlib.Path, iterations: int) -> dict:
    import torch
    import yaml

    from r2_gaussian_b200 import initialize_pcd, recon, test, trainer
    from test_fdk_pad_gpu import TRUNCATED_W, WIDE_W, scene_field_of_view, write_truncation_scene
    res = {}
    for label, w in (("truncated", TRUNCATED_W), ("untruncated", WIDE_W)):
        src = write_truncation_scene(tmp, w)
        fov = scene_field_of_view(src)
        row = {"detector_width": w, "fov_fraction": float(fov.mean())}
        for pad in PADS:
            out = tmp / f"recon_{label}_{pad:g}"
            recon.main(["-s", src, "-m", str(out), "--methods", "fdk"] + (["--fdk_pad", str(pad)] if pad else []))
            gt, pred = np.load(out / "fdk" / "ct_gt.npy"), np.load(out / "fdk" / "ct_pred.npy")
            row[f"fdk_pad{pad:g}"] = _in_field(gt, pred, fov)
        for pad in (0.0, 0.5):
            init = initialize_pcd.main(["--data", src, "--recon_method", "fdk", "--output",
                                        str(tmp / f"init_{label}_{pad:g}.npy")]
                                       + (["--fdk_pad", str(pad)] if pad else []))
            model = tmp / f"model_{label}_{pad:g}"
            random.seed(0); np.random.seed(0); torch.manual_seed(0)
            it = str(iterations)
            trainer.main(["-s", src, "-m", str(model), "--ply_path", init, "--iterations", it, "--test_iterations", it,
                          "--save_iterations", it])
            test.main(["-m", str(model), "--skip_render_train", "--skip_render_test"])
            with open(model / "test" / f"iter_{iterations}" / "eval3d.yml") as f:
                ev = yaml.safe_load(f)
            row[f"train_from_pad{pad:g}"] = {k: float(ev[k]) for k in ("psnr_3d", "ssim_3d")}
        res[label] = row
    return res


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--train_iterations", type=int, default=1500)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "cost_ms": cost(a.reps)}
    with tempfile.TemporaryDirectory() as tmp:
        res["benefit"] = benefit(pathlib.Path(tmp), a.train_iterations)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "fdk_pad_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
