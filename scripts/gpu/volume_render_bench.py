"""Volume rendering on the GPU (r2x_volume_render, `volume_render.render`):

    python scripts/gpu/volume_render_bench.py [--reps 10] [--no-oracle]

Cases: a seeded ellipsoid phantom (three overlapping ellipsoids plus 2 % noise, clipped to [0, 1]) at 256^3 and 512^3,
rendered at 800 x 1000 (plot_volume.py's window) from `default_camera`, composite and MIP, one frame and a 36-frame
orbit.  Each case is timed with CUDA events around the render call, median of --reps after one warm-up call.  The
samples are counted on the host from the geometry (tests/volume_render_oracle.py's ray set-up: floor((s_out - s_in) /
step) + 1 per ray that meets the box); composite rays may stop early, so for composite that count is an upper bound
on the samples taken.  Also printed: the numpy oracle's CPU time for one composite frame at 256^3 (for scale), and
one JSON line with the card's name, power limit and SM clocks read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def clocks() -> dict:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=20)
        sm, smax = (float(x) for x in r.stdout.strip().splitlines()[0].split(","))
        return {"sm_clock_mhz": sm, "max_sm_clock_mhz": smax}
    except Exception:
        return {"sm_clock_mhz": None, "max_sm_clock_mhz": None}


def phantom(n, seed):
    import torch
    g = torch.linspace(-1, 1, n, device="cuda")
    X, Y, Z = torch.meshgrid(g, g, g, indexing="ij")
    vol = torch.zeros((n, n, n), device="cuda")
    for (cx, cy, cz), (a, b, c), w in (((0.0, 0.0, 0.0), (0.7, 0.55, 0.6), 0.6), ((0.25, -0.1, 0.2), (0.3, 0.25, 0.35), 0.4),
                                       ((-0.3, 0.2, -0.25), (0.2, 0.3, 0.2), -0.3)):
        q = ((X - cx) / a) ** 2 + ((Y - cy) / b) ** 2 + ((Z - cz) / c) ** 2
        vol += w * torch.clamp(1 - q, min=0)
    gen = torch.Generator("cuda").manual_seed(seed)
    return (vol + 0.02 * torch.randn(vol.shape, generator=gen, device="cuda")).clamp(0, 1).contiguous()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    import numpy as np
    import torch

    import secondary
    import volume_render_oracle as vo
    from r2_gaussian_b200 import volume_render as vr

    if not torch.cuda.is_available():
        raise SystemExit("volume_render_bench needs a CUDA device")
    dev = torch.device("cuda")
    W, H, step = 800, 1000, 0.5

    def timed(fn):
        fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(a.reps):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            e.synchronize()
            ms.append(s.elapsed_time(e))
        ms.sort()
        return ms[len(ms) // 2]

    for n, seed in ((256, 1), (512, 2)):
        vol = phantom(n, seed)
        cam = vr.default_camera(vol.shape, W, H)
        for frames in (1, 36):
            cams = vr.orbit(cam, frames) if frames > 1 else [cam]
            samples = 0
            for c in cams:
                _, _, s0, s1, meets = vo.ray_setup(c.record(), H, W, False, vol.shape)
                samples += int(vo.sample_counts(s0, s1, meets, step).sum())
            for mode in ("composite", "mip"):
                ms = timed(lambda: vr.render(vol, cams, mode=mode, step=step))
                out = vr.render(vol, cams, mode=mode, step=step)
                row = {"case": f"phantom_{n}", "mode": mode, "frames": frames, "width": W, "height": H,
                       "ms": ms, "ms_per_frame": ms / frames, "samples": samples,
                       "samples_per_s": samples / (ms * 1e-3), "mean_alpha": float(out[..., 3].mean())}
                if mode == "composite" and frames == 1 and n == 256 and not a.no_oracle:
                    host = vol.cpu().numpy()
                    t0 = time.perf_counter()
                    want = vo.render(host, [cam], step=step)
                    row["oracle_cpu_s"] = time.perf_counter() - t0
                    row["oracle_max_err"] = float(np.abs(out.cpu().numpy() - want).max())
                print(json.dumps(row), flush=True)
                del out
        del vol
        torch.cuda.empty_cache()
    print(json.dumps({**secondary.card(dev), **clocks()}))


if __name__ == "__main__":
    main()
