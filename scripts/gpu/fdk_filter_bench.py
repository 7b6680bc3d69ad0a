"""Cost and quality of FDK's windowed ramp filters (r2x_fdk's filter field) against the Ram-Lak filter:

    python scripts/gpu/fdk_filter_bench.py [--reps 20] [--out DIR] [--skip_quality]

Time: the fdk row of scripts/secondary.py (50 seeded cone-beam views of 512^2 into 256^3 on the full circle), one
r2x_fdk call per filter, the five filters alternated call by call, each call timed with CUDA events (median of --reps
after a warm-up of every filter).  The filter kernels (fdk_filter_kernel<0> for Ram-Lak, fdk_window_kernel<0, F> for
the windows) and the backprojection are timed in a separate torch.profiler run.  Quality: recon_baselines.py's seeded
256^3 phantom and noisy cone-beam scanner (Poisson 1e4 + Gaussian (0, 10)), 50 train views, reconstructed with each
filter, 3D PSNR / SSIM against the phantom; and the 3D PSNR of the initialize_pcd cloud (--recon_method fdk,
--evaluate) from Ram-Lak and from Hann FDK on the noisy 48^3 scene of tests/test_tv_recon_gpu.py.  Prints one JSON line
with the card name and power limit."""
from __future__ import annotations

import argparse
import json
import math
import os
import re
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "scripts", "gpu"))

N_VIEWS = 50


def timing(dev, reps: int) -> dict:
    import torch

    from r2_gaussian_b200 import _lib, scene
    from r2_gaussian_b200.fdk import FILTERS, R2X_FDK_PLAIN

    lib = _lib.load()
    sc = scene.cone_beam_scanner(512, 256)
    N, H, W, n = N_VIEWS, 512, 512, 256
    projs = torch.rand(N, H, W, device=dev, generator=torch.Generator(dev).manual_seed(0))
    vol = torch.empty(n, n, n, device=dev)
    nbytes = int(lib.r2x_fdk_scratch_bytes(N, H, W))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    views = [scene.make_view(sc, float(a)) for a in np.linspace(0.0, 2.0 * math.pi, N + 1)[:-1]]
    vm = torch.tensor(np.stack([v.viewmatrix.reshape(16) for v in views]), device=dev)
    pm = torch.tensor(np.stack([v.projmatrix.reshape(16) for v in views]), device=dev)
    tx, ty, dso = float(views[0].tanfovx), float(views[0].tanfovy), float(sc["DSO"])

    def call(name):
        def f():
            _lib.check(lib.r2x_fdk(torch.cuda.current_stream(dev).cuda_stream, N, H, W, projs.data_ptr(), vm.data_ptr(),
                                   pm.data_ptr(), tx, ty, 1, 0.0, 0.0, R2X_FDK_PLAIN | (FILTERS.index(name) << 8), None,
                                   0.0, dso, n, n, n, 2.0, 2.0, 2.0, 0.0, 0.0, 0.0, vol.data_ptr(), scratch.data_ptr(),
                                   nbytes), "r2x_fdk")
        return f

    calls = {name: call(name) for name in FILTERS}
    for _ in range(2):                                       # warm-up of every filter
        for f in calls.values():
            f()
    torch.cuda.synchronize(dev)
    ms = {name: [] for name in FILTERS}
    for _ in range(reps):
        for name, f in calls.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            f()
            e.record()
            e.synchronize()
            ms[name].append(s.elapsed_time(e))
    row = {"call_ms": {name: float(np.median(v)) for name, v in ms.items()},
           "call_spread_ms": {name: [float(min(v)), float(max(v))] for name, v in ms.items()}}
    row["call_ratio_to_ram_lak"] = {name: row["call_ms"][name] / row["call_ms"]["ram_lak"] for name in FILTERS}

    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            for f in calls.values():
                f()
        torch.cuda.synchronize(dev)
    kernels = {}
    for ev in prof.key_averages():
        m = re.search(r"(fdk_filter_kernel<0>|fdk_window_kernel<0, (\d+)>|fdk_backproject_kernel)", ev.key)
        if not m:
            continue
        key = "ram_lak" if m.group(1).startswith("fdk_filter") else (
            "backproject" if m.group(2) is None else FILTERS[int(m.group(2)) >> 8])
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        k = kernels.setdefault(key, [0.0, 0])
        k[0] += t
        k[1] += ev.count
    row["kernel_ms"] = {key: t_us / count / 1e3 for key, (t_us, count) in kernels.items()}
    if "ram_lak" in row["kernel_ms"]:
        row["filter_kernel_ratio_to_ram_lak"] = {k: v / row["kernel_ms"]["ram_lak"] for k, v in row["kernel_ms"].items()
                                                 if k in FILTERS}
    return row


def quality(out: str) -> dict:
    import torch
    import yaml

    import recon_baselines
    from r2_gaussian_b200 import generate_data
    from r2_gaussian_b200.dataset import read_scene
    from r2_gaussian_b200.fdk import FILTERS, fdk
    from r2_gaussian_b200.metrics import metric_vol

    vol_path = os.path.join(out, "phantom.npy")
    np.save(vol_path, recon_baselines.phantom())
    yml = os.path.join(out, "scanner.yml")
    with open(yml, "w") as f:
        yaml.safe_dump(recon_baselines.SCANNER, f)
    case = generate_data.main(["--vol", vol_path, "--scanner", yml, "--output", os.path.join(out, "data"),
                               "--n_train", str(N_VIEWS), "--n_test", "1"])
    info = read_scene(case, eval=False)
    b = torch.from_numpy(np.stack([np.asarray(c.image, np.float32) for c in info.train_cameras])).cuda()
    angles = [c.angle for c in info.train_cameras]
    gt = np.asarray(info.vol, np.float32)
    res = {}
    for name in FILTERS:
        pred = fdk(b, angles, info.scanner_cfg, filter=name).cpu().numpy()
        res[name] = {"psnr_3d": float(metric_vol(gt, pred, "psnr")[0]), "ssim_3d": float(metric_vol(gt, pred, "ssim")[0])}
        print(name, res[name], flush=True)
    return res


def init_cloud(out: str) -> dict:
    """3D PSNR of the initialize_pcd cloud (2000 points) from Ram-Lak and from Hann FDK on the noisy 48^3 scene."""
    import contextlib
    import io
    import pathlib

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_projector_gpu import _write_inputs

    from r2_gaussian_b200 import generate_data, initialize_pcd

    tmp = pathlib.Path(out) / "noisy48"
    tmp.mkdir(parents=True, exist_ok=True)
    yml, vol_path, *_ = _write_inputs(tmp, noise=True)
    case = generate_data.main(["--vol", str(vol_path), "--scanner", str(yml), "--n_train", "24", "--n_test", "6",
                               "--output", str(tmp / "data")])
    res = {}
    for name in ("ram_lak", "hann"):
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            initialize_pcd.main(["--data", case, "--recon_method", "fdk", "--fdk_filter", name, "--n_points", "2000",
                                 "--evaluate", "--output", str(tmp / f"init_{name}.npy")])
        res[name] = float(re.findall(r"3D PSNR for initial Gaussians: (\S+)", buf.getvalue())[0])
        print("init", name, res[name], flush=True)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="scenes (default: a new temporary directory)")
    ap.add_argument("--skip_quality", action="store_true")
    a = ap.parse_args()
    import torch

    import secondary

    if not torch.cuda.is_available():
        raise SystemExit("fdk_filter_bench needs a CUDA device")
    dev = torch.device("cuda")
    out = a.out or tempfile.mkdtemp(prefix="fdk_filter_")
    os.makedirs(out, exist_ok=True)
    row = {"workload": f"FDK, {N_VIEWS} cone-beam views of 512x512 (DSD 7, DSO 5) -> 256^3, full circle: r2x_fdk with "
                       "each filter", **secondary.card(dev), **timing(dev, a.reps)}
    if not a.skip_quality:
        row["quality_256_noisy"] = quality(out)
        row["init_cloud_psnr_48_noisy"] = init_cloud(out)
    print(json.dumps({**row, **secondary.card(dev)}))


if __name__ == "__main__":
    main()
