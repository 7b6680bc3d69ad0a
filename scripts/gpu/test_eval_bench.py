"""Time evaluation: the torch metrics (`metric_vol`, `metric_proj`) against the device metrics (`volume_metrics`,
`projection_metrics`), and the whole `python -m r2_gaussian_b200.test` on a generated scene.

    python scripts/gpu/test_eval_bench.py [--out DIR] [--reps 3]

Cases: metric_vol (ssim) against volume_metrics at 256^3 and 512^3; metric_proj (psnr + ssim) against
projection_metrics on 150 views of 512^2; the test driver on a 128^3 generate_data scene (50 train and 50 test views
of 256^2) after a short training run, its rendering, metrics and file writing timed apart.  Each timing is the median
of --reps runs after one warm-up run, between CUDA events (metrics) or a host clock around synchronised phases (the
driver).  Prints the largest difference between the old and new scores, the card name and power limit, and one JSON
line; with --out, writes it to DIR/test_eval_bench.json."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from r2_gaussian_b200 import metrics  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn, reps):
    """(median ms over reps after one warm-up, last result) between CUDA events."""
    out = fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times)), out


def phantom(shape, seed):
    gen = torch.Generator("cuda").manual_seed(seed)
    grids = torch.meshgrid(*[torch.linspace(-1, 1, n, device="cuda") for n in shape], indexing="ij")
    gt = torch.clamp(1.0 - sum(g * g for g in grids), min=0) + 0.05 * torch.rand(shape, generator=gen, device="cuda")
    pred = gt + 0.1 * torch.randn(shape, generator=gen, device="cuda")
    return gt.float().contiguous(), pred.float().contiguous()


def volume_case(n, reps):
    gt, pred = phantom((n, n, n), n)
    t_old, old = timed(lambda: metrics.metric_vol(gt, pred, "ssim"), reps)
    t_new, new = timed(lambda: metrics.volume_metrics(gt, pred), reps)
    diff = max(abs(old[0] - new["ssim_3d"]), *(abs(o - new[f"ssim_3d_{k}"]) for o, k in zip(old[1], "xyz")))
    return {"case": f"volume_{n}^3", "metric_vol_ssim_ms": t_old, "volume_metrics_ms": t_new,
            "speedup": t_old / t_new, "max_abs_ssim_diff": diff,
            "psnr_diff": abs(metrics.metric_vol(gt, pred, "psnr")[0] - new["psnr_3d"])}


def projection_case(N, HW, reps):
    gt, pred = phantom((N, HW, HW), N)
    hwn = (gt.permute(1, 2, 0), pred.permute(1, 2, 0))
    t_old, old = timed(lambda: (metrics.metric_proj(*hwn, "psnr"), metrics.metric_proj(*hwn, "ssim")), reps)
    t_new, new = timed(lambda: metrics.projection_metrics(gt, pred), reps)
    dp = max(abs(a - b) for a, b in zip(old[0][1], new["psnr_2d_projs"]))
    ds = max(abs(a - b) for a, b in zip(old[1][1], new["ssim_2d_projs"]))
    return {"case": f"projections_{N}x{HW}^2", "metric_proj_psnr_ssim_ms": t_old, "projection_metrics_ms": t_new,
            "speedup": t_old / t_new, "max_abs_psnr_diff": dp, "max_abs_ssim_diff": ds}


def driver_case(workdir, reps):
    """generate_data -> initialize_pcd -> trainer (300 iterations) -> the test driver, timed per phase."""
    from r2_gaussian_b200 import generate_data, initialize_pcd, scene, trainer
    from r2_gaussian_b200 import test as evaltest
    vol, _ = phantom((128, 128, 128), 3)
    vol = torch.clamp(vol, min=0).cpu().numpy()
    np.save(os.path.join(workdir, "vol.npy"), vol)
    sc = scene.cone_beam_scanner(256, 128)
    sc.update({"filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0, "noise": False})
    with open(os.path.join(workdir, "scanner.yml"), "w") as f:
        f.write("".join(f"{k}: {json.dumps(v)}\n" for k, v in sc.items()))
    src = generate_data.main(["--vol", os.path.join(workdir, "vol.npy"),
                              "--scanner", os.path.join(workdir, "scanner.yml"), "--n_train", "50", "--n_test", "50", "--output", os.path.join(workdir, "data")])
    init = initialize_pcd.main(["--data", src, "--n_points", "50000", "--output", os.path.join(workdir, "init.npy")])
    model = os.path.join(workdir, "model")
    trainer.main(["-s", src, "-m", model, "--ply_path", init, "--iterations", "300", "--test_iterations", "300",
                  "--save_iterations", "300"])
    runs = [evaltest.main(["-m", model, "--quiet"]) for _ in range(reps + 1)][1:]
    sec = {k: float(np.median([r["seconds"][k] for r in runs])) for k in runs[0]["seconds"]}
    ev = runs[-1]
    return {"case": "test_driver_128^3_50+50x256^2", **{f"{k}_s": v for k, v in sec.items()},
            "total_s": sum(sec.values()), "psnr_3d": ev["eval3d"]["psnr_3d"], "ssim_3d": ev["eval3d"]["ssim_3d"]}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default=None, help="directory for test_eval_bench.json (default: print only)")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    torch.cuda.init()
    res = {"card": card(), "tf32_convolutions": torch.backends.cudnn.allow_tf32, "cases": []}
    for n in (256, 512):
        res["cases"].append(volume_case(n, a.reps))
        print(res["cases"][-1], flush=True)
    res["cases"].append(projection_case(150, 512, a.reps))
    print(res["cases"][-1], flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        res["cases"].append(driver_case(tmp, a.reps))
    print(res["cases"][-1], flush=True)
    print(f"card: {res['card']}")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "test_eval_bench.json"), "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
