"""Where the time of a real-scan scene build goes: copy-in and preparation of a 721-view scan on the GPU, the FDK of
all views, the same preparation on the host, and the `.mat` decode of a few full-size files.

    python scripts/gpu/real_data_bench.py [--views 721] [--H0 2368] [--W0 2240] [--chunk 32] [--nvox 256]

The scan is never written out: its views come from two pinned host sets of `chunk` seeded float64 views used in turn
(30 GB of distinct full-size views would not fit a shared host), so every chunk still crosses PCIe; H0 x W0 is a
stand-in for a full resolution frame (the FIPS frame size itself is not checked here).  Timed with CUDA events:
  * h2d_s / prepare_s: the chunked copy of the float64 views and r2x_projection_prepare, summed over the chunks;
  * fdk_s: fdk.fdk of all prepared views into nvox^3;
  * host_prepare_s_per_view: the numpy chain (tests/real_data_oracle.py; with cv2.resize when cv2 imports) of one view;
  * mat_decode_s_per_view: scipy.io.loadmat of 4 full-size files written to a temporary directory.
Prints one JSON line with the card name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=721)
    ap.add_argument("--H0", type=int, default=2368)
    ap.add_argument("--W0", type=int, default=2240)
    ap.add_argument("--subsample", type=int, default=4)
    ap.add_argument("--chunk", type=int, default=32)
    ap.add_argument("--nvox", type=int, default=256)
    a = ap.parse_args()
    import numpy as np
    import scipy.io
    import torch

    import real_data_oracle as oracle
    from r2_gaussian_b200 import generate_real_data as grd
    from r2_gaussian_b200.dataset import scale_scanner
    from r2_gaussian_b200.fdk import fdk

    if not torch.cuda.is_available():
        raise SystemExit("real_data_bench needs a CUDA device")
    rng = np.random.default_rng(0)
    frame = rng.normal(0.4, 0.7, (a.H0, a.W0)) * 8.0
    ring = min(a.views, 2 * a.chunk)
    host = torch.empty((ring, a.H0, a.W0), dtype=torch.float64, pin_memory=True)
    for v in range(ring):
        host[v].numpy()[...] = frame + 1e-3 * v
    H, W = grd.prepared_shape(a.H0, a.W0, a.subsample)
    stack = torch.empty((a.views, H, W), dtype=torch.float32, device="cuda")
    dev = torch.empty((a.chunk, a.H0, a.W0), dtype=torch.float64, device="cuda")
    grd.prepare(dev[:1].zero_(), a.subsample, 400.0, 50, out=stack[:1])    # warm-up
    torch.cuda.synchronize()

    h2d_ms = prep_ms = 0.0
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    t0 = time.perf_counter()
    for c0 in range(0, a.views, a.chunk):
        n = min(a.chunk, a.views - c0)
        ev[0].record()
        h0 = (c0 // a.chunk) % 2 * a.chunk
        dev[:n].copy_(host[h0:h0 + n], non_blocking=True)
        ev[1].record()
        grd.prepare(dev[:n], a.subsample, 400.0, 50, out=stack[c0:c0 + n])
        ev[2].record()
        ev[2].synchronize()
        h2d_ms += ev[0].elapsed_time(ev[1])
        prep_ms += ev[1].elapsed_time(ev[2])
    wall_s = time.perf_counter() - t0
    last = a.views - 1
    for v, h in ((0, 0), (last, (last // a.chunk) % 2 * a.chunk + last % a.chunk)):
        assert stack[v].cpu().numpy().tobytes() == oracle.prepare(host[h].numpy(), a.subsample, 400.0, 50).tobytes()

    dd = 0.05 * 4 / 1000 * 50
    cfg = {"mode": "cone", "DSD": 553.74 / 1000 * 50, "DSO": 410.66 / 1000 * 50, "nDetector": [H, W],
           "sDetector": [H * dd, W * dd], "nVoxel": [a.nvox] * 3, "sVoxel": [2.0] * 3, "offOrigin": [0.0] * 3,
           "offDetector": [0.0, 0.0], "accuracy": 0.5, "filter": None}
    scale = scale_scanner(cfg)
    angles = np.linspace(0, 2 * np.pi, a.views, endpoint=False)
    fdk(stack[:8] * scale, angles[:8], cfg)
    torch.cuda.synchronize()
    ev[0].record()
    fdk(stack * scale, angles, cfg)
    ev[1].record()
    ev[1].synchronize()
    fdk_ms = ev[0].elapsed_time(ev[1])

    t0 = time.perf_counter()
    for _ in range(3):
        oracle.prepare(frame, a.subsample, 400.0, 50)
    host_numpy_s = (time.perf_counter() - t0) / 3
    cv2_s = None
    if oracle.reference_chain(frame[:16, :16], a.subsample, 400.0, 50) is not None:
        t0 = time.perf_counter()
        for _ in range(3):
            oracle.reference_chain(frame, a.subsample, 400.0, 50)
        cv2_s = (time.perf_counter() - t0) / 3

    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for k in range(4):
            paths.append(os.path.join(tmp, f"v{k}.mat"))
            scipy.io.savemat(paths[-1], {"img": frame + k})
        t0 = time.perf_counter()
        for p in paths:
            scipy.io.loadmat(p)["img"]
        mat_s = (time.perf_counter() - t0) / len(paths)

    in_bytes = a.views * a.H0 * a.W0 * 8
    print(json.dumps({
        "card": card(), "views": a.views, "frame": [a.H0, a.W0], "prepared": [H, W], "chunk": a.chunk,
        "h2d_s": round(h2d_ms / 1e3, 4), "h2d_GB_per_s": round(in_bytes / (h2d_ms / 1e3) / 1e9, 2),
        "prepare_s": round(prep_ms / 1e3, 4), "prepare_input_GB_per_s": round(in_bytes / (prep_ms / 1e3) / 1e9, 1),
        "copy_and_prepare_wall_s": round(wall_s, 3), "fdk_s": round(fdk_ms / 1e3, 4), "fdk_nvox": a.nvox,
        "host_numpy_prepare_s_per_view": round(host_numpy_s, 4),
        "host_cv2_prepare_s_per_view": None if cv2_s is None else round(cv2_s, 4),
        "mat_decode_s_per_view": round(mat_s, 4),
        "mat_decode_s_all_views_est": round(mat_s * a.views, 1),
    }))


if __name__ == "__main__":
    main()
