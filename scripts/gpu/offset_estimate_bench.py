#!/usr/bin/env python
"""Time `detector.estimate_offset` (the conjugate-ray search: two launches of r2x_detector_offset_cost, one host read
each).

    python scripts/gpu/offset_estimate_bench.py [--repeat 20] [--out FILE]

Cases: the closed-form blob projections of tests/offset_estimate_oracle.py, evaluated on the GPU, shifted 2.4 px, at
50 and 721 (cone) or 720 (parallel) views of 512^2: cone beam (mid-plane only) and parallel beam (every row of the views pi apart), default search (+-128 px coarse,
129 fine candidates).  Each case is run once to warm up, then `--repeat` times with a device synchronise before and
after; the median and the spread of the host time are reported, with the estimate's error.  Prints one JSON object
with the card and its power limit."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def project(torch, blob_rows, angles, sc, sigma):
    """The closed-form blob projections of tests/offset_estimate_oracle.py, evaluated on the GPU in float64."""
    H, W = int(sc["nDetector"][0]), int(sc["nDetector"][1])
    du, dv = sc["sDetector"][1] / W, sc["sDetector"][0] / H
    f64 = dict(dtype=torch.float64, device="cuda")
    b = torch.tensor(angles, **f64)[:, None, None]
    u = (du * (torch.arange(W, **f64) - (W - 1) / 2 - sigma))[None, None, :]
    v = (dv * (torch.arange(H, **f64) - (H - 1) / 2))[None, :, None]
    cb, sb = torch.cos(b), torch.sin(b)
    radial = torch.stack([cb, sb, torch.zeros_like(cb)], -1)
    e = torch.stack([-sb, cb, torch.zeros_like(cb)], -1)
    z = torch.tensor([0.0, 0.0, 1.0], **f64)
    if sc["mode"] == "parallel":
        o = u[..., None] * e - v[..., None] * z + sc["DSO"] * radial
        d = (-radial).expand_as(o)
    else:
        o = (sc["DSO"] * radial).expand(len(angles), H, W, 3)
        d = -sc["DSD"] * radial + u[..., None] * e - v[..., None] * z
        d = d / d.norm(dim=-1, keepdim=True)
    out = torch.zeros(o.shape[:-1], **f64)
    for x, y, zc, s, amp in blob_rows:
        w = torch.tensor([x, y, zc], **f64) - o
        along = (w * d).sum(-1)
        dist2 = ((w * w).sum(-1) - along * along).clamp_min(0.0)
        out += amp * (2 * 3.141592653589793) ** 0.5 * s * torch.exp(-dist2 / (2 * s * s))
    return out.float()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch

    import offset_estimate_oracle as oo
    from r2_gaussian_b200 import detector, scene
    bl = oo.blobs(9, seed=0, radius=0.5)
    res = {"card": card(), "cases": []}
    for mode in ("cone", "parallel"):
        sc = scene.cone_beam_scanner(512, 64) if mode == "cone" else scene.parallel_beam_scanner(512, 64)
        for n in (50, 720 if mode == "parallel" else 721):
            ang = np.linspace(0, 2 * np.pi, n + 1)[:-1] + 0.3
            p = torch.cat([project(torch, bl, ang[k:k + 16], sc, 2.4) for k in range(0, n, 16)])
            est = detector.estimate_offset(p, ang, sc)
            times = []
            for _ in range(a.repeat):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                est = detector.estimate_offset(p, ang, sc)
                torch.cuda.synchronize()
                times.append(time.perf_counter() - t0)
            t = np.array(times) * 1e3
            res["cases"].append({"mode": mode, "views": n, "detector": 512, "n_pairs": est["n_pairs"],
                                 "samples_per_candidate": est["n_samples"], "candidates": len(est["coarse"][0]) +
                                 len(est["fine"][0]), "median_ms": float(np.median(t)), "min_ms": float(t.min()),
                                 "max_ms": float(t.max()), "error_px": est["offset_px"] - 2.4})
            print(json.dumps(res["cases"][-1]), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
