"""Cost and quality of the short-scan FDK (r2x_fdk with R2X_FDK_PARKER) against the plain one (R2X_FDK_PLAIN):

    python scripts/gpu/fdk_short_scan_bench.py [--reps 20] [--out DIR]

Time: the fdk row of scripts/secondary.py (50 seeded cone-beam views of 512^2 into 256^3), the plain call on the full
circle and the short-scan call on 220 degrees, alternated, each timed with CUDA events (median of --reps).  The filter
kernels (fdk_filter_kernel<R2X_FDK_PLAIN>, fdk_filter_kernel<R2X_FDK_PARKER>) and the backprojection are timed in a
separate torch.profiler run.  Quality: recon_baselines.py's seeded 256^3 phantom and noisy cone-beam scanner, 50 train views at 220 degrees
reconstructed by plain and short-scan FDK, and 82 train views on the full circle (the same view density) by plain FDK;
3D PSNR / SSIM against the phantom.  Prints one JSON line with the card name and power limit."""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "scripts", "gpu"))

ARC_DEG, N_VIEWS = 220.0, 50


def timing(dev, reps: int) -> dict:
    import torch

    from r2_gaussian_b200 import _lib, scene
    from r2_gaussian_b200.fdk import R2X_FDK_PARKER, R2X_FDK_PLAIN, short_scan_views

    lib = _lib.load()
    sc = scene.cone_beam_scanner(512, 256)
    N, H, W, n = N_VIEWS, 512, 512, 256
    projs = torch.rand(N, H, W, device=dev, generator=torch.Generator(dev).manual_seed(0))
    vol = torch.empty(n, n, n, device=dev)
    nbytes = int(lib.r2x_fdk_scratch_bytes(N, H, W))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    grid = (n, n, n, 2.0, 2.0, 2.0, 0.0, 0.0, 0.0)

    def mats(angles):
        views = [scene.make_view(sc, float(a)) for a in angles]
        return (views[0], torch.tensor(np.stack([v.viewmatrix.reshape(16) for v in views]), device=dev),
                torch.tensor(np.stack([v.projmatrix.reshape(16) for v in views]), device=dev))

    v0, vm_full, pm_full = mats(np.linspace(0.0, 2.0 * math.pi, N + 1)[:-1])
    short_angles = np.linspace(0.0, math.radians(ARC_DEG), N + 1)[:-1]
    _, vm_short, pm_short = mats(short_angles)
    vw_host, arc = short_scan_views(short_angles, v0.mode, v0.tanfovx)
    vw = torch.tensor(vw_host.astype(np.float32), device=dev)
    tx, ty, dso = float(v0.tanfovx), float(v0.tanfovy), float(sc["DSO"])
    stream = lambda: torch.cuda.current_stream(dev).cuda_stream
    tail = (dso, *grid, vol.data_ptr(), scratch.data_ptr(), nbytes)

    def plain():
        _lib.check(lib.r2x_fdk(stream(), N, H, W, projs.data_ptr(), vm_full.data_ptr(), pm_full.data_ptr(), tx, ty, 1,
                               0.0, 0.0, R2X_FDK_PLAIN, None, 0.0, *tail), "r2x_fdk")

    def short():
        _lib.check(lib.r2x_fdk(stream(), N, H, W, projs.data_ptr(), vm_short.data_ptr(), pm_short.data_ptr(), tx, ty, 1,
                               0.0, 0.0, R2X_FDK_PARKER, vw.data_ptr(), float(arc), *tail), "r2x_fdk")

    for f in (plain, short, plain, short):                  # warm-up of both shapes
        f()
    torch.cuda.synchronize(dev)
    ms = {"plain": [], "short": []}
    for _ in range(reps):
        for name, f in (("plain", plain), ("short", short)):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            f()
            e.record()
            e.synchronize()
            ms[name].append(s.elapsed_time(e))
    row = {name + "_call_ms": float(np.median(v)) for name, v in ms.items()}
    row["call_spread_ms"] = {name: [float(min(v)), float(max(v))] for name, v in ms.items()}

    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            plain()
            short()
        torch.cuda.synchronize(dev)
    kernels = {}
    for ev in prof.key_averages():
        for key in ("fdk_filter_kernel<1>", "fdk_filter_kernel<0>", "fdk_backproject_kernel"):
            if key in ev.key:
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
                k = kernels.setdefault(key, [0.0, 0])
                k[0] += t
                k[1] += ev.count
                break
    for key, (t_us, count) in kernels.items():
        row[key + "_ms"] = t_us / count / 1e3
    if "fdk_filter_kernel<0>_ms" in row and "fdk_filter_kernel<1>_ms" in row:
        row["filter_ratio"] = row["fdk_filter_kernel<1>_ms"] / row["fdk_filter_kernel<0>_ms"]
    row["call_ratio"] = row["short_call_ms"] / row["plain_call_ms"]
    return row


def quality(out: str) -> dict:
    import torch
    import yaml

    import recon_baselines
    from r2_gaussian_b200 import generate_data
    from r2_gaussian_b200.dataset import read_scene
    from r2_gaussian_b200.fdk import fdk
    from r2_gaussian_b200.metrics import metric_vol

    vol_path = os.path.join(out, "phantom.npy")
    np.save(vol_path, recon_baselines.phantom())
    res, cases = {}, {}
    for label, deg, n_train, short in (("plain_220", ARC_DEG, N_VIEWS, False), ("short_scan_220", ARC_DEG, N_VIEWS, True),
                                       ("plain_360", 360.0, round(N_VIEWS * 360.0 / ARC_DEG), False)):
        if deg not in cases:
            yml = os.path.join(out, f"scanner_{int(deg)}.yml")
            with open(yml, "w") as f:
                yaml.safe_dump(dict(recon_baselines.SCANNER, totalAngle=deg), f)
            cases[deg] = generate_data.main(["--vol", vol_path, "--scanner", yml, "--output",
                                             os.path.join(out, f"data_{int(deg)}"), "--n_train", str(n_train),
                                             "--n_test", "1"])
        case = cases[deg]
        info = read_scene(case, eval=False)
        b = torch.from_numpy(np.stack([np.asarray(c.image, np.float32) for c in info.train_cameras])).cuda()
        pred = fdk(b, [c.angle for c in info.train_cameras], info.scanner_cfg, short_scan=short).cpu().numpy()
        gt = np.asarray(info.vol, np.float32)
        res[label] = {"views": n_train, "arc_deg": deg, "psnr_3d": float(metric_vol(gt, pred, "psnr")[0]),
                      "ssim_3d": float(metric_vol(gt, pred, "ssim")[0])}
        print(label, res[label], flush=True)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="scenes (default: a new temporary directory)")
    a = ap.parse_args()
    import torch

    import secondary

    if not torch.cuda.is_available():
        raise SystemExit("fdk_short_scan_bench needs a CUDA device")
    dev = torch.device("cuda")
    out = a.out or tempfile.mkdtemp(prefix="fdk_short_scan_")
    os.makedirs(out, exist_ok=True)
    row = {"workload": f"FDK, {N_VIEWS} cone-beam views of 512x512 (DSD 7, DSO 5) -> 256^3: r2x_fdk(R2X_FDK_PLAIN) on 360 "
                       f"degrees against r2x_fdk(R2X_FDK_PARKER) on {ARC_DEG:g} degrees", **timing(dev, a.reps)}
    row["quality"] = quality(out)
    print(json.dumps({**row, **secondary.card(dev)}))


if __name__ == "__main__":
    main()
