"""Cost of the offset detector (`use_offDetector=True`) in the projector, the backprojector and FDK, and of the half-fan
weights in the FDK filter:

    python scripts/gpu/detector_geometry_bench.py [--reps 20]

Workloads of scripts/secondary.py: project = a seeded 256^3 volume into 150 cone-beam views of 512^2; backproject and
fdk = 50 cone-beam views of 512^2 into 256^3.  Each pair of variants (centred / offset by (2.4, -1.7) pixels; for the
filter, offset FDK without / with half-fan weights at a quarter-width offset) is alternated call by call, each call
timed with CUDA events after a 256 MiB L2 flush, median of --reps.  A torch.profiler pass then sums the device time of
each kernel over 5 calls per variant.  Prints one JSON line with the card name and power limit."""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

SHIFT = (2.4, -1.7)


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "?"
    except Exception:
        return "?"


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args(argv)

    import torch

    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.fdk import fdk
    from r2_gaussian_b200.projector import CTOperator

    dev = torch.device("cuda", 0)
    gen = torch.Generator(dev).manual_seed(0)
    sc = scene.cone_beam_scanner(512, 256)
    du = sc["sDetector"][1] / 512

    def offset(t_u, t_v):
        return dict(sc, offDetector=[t_u * du, t_v * du])

    off = offset(*SHIFT)
    quarter = offset(128.0, 0.0)
    vol = torch.rand(256, 256, 256, device=dev, generator=gen)
    a150 = np.linspace(0.0, 2.0 * math.pi, 151)[:-1]
    a50 = np.linspace(0.0, 2.0 * math.pi, 51)[:-1]
    projs = torch.rand(50, 512, 512, device=dev, generator=gen)
    A = {"centred": CTOperator(a150, sc, dev), "offset": CTOperator(a150, off, dev, use_offDetector=True)}
    At = {"centred": CTOperator(a50, sc, dev), "offset": CTOperator(a50, off, dev, use_offDetector=True)}
    pairs = {
        "project": {k: (lambda op=op: op.A(vol)) for k, op in A.items()},
        "backproject": {k: (lambda op=op: op.At(projs)) for k, op in At.items()},
        "fdk": {"centred": lambda: fdk(projs, a50, sc), "offset": lambda: fdk(projs, a50, off, use_offDetector=True)},
        "fdk_half_fan": {"offset": lambda: fdk(projs, a50, quarter, use_offDetector=True),
                         "half_fan": lambda: fdk(projs, a50, quarter, use_offDetector=True, half_fan=True)},
    }
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    out = {"card": _card(), "protocol": "median of per-call CUDA-event times, variants alternated, 256 MiB L2 flush "
                                        "before each call", "reps": a.reps}
    for name, variants in pairs.items():
        for f in list(variants.values()) * 2:                               # warm-up
            f()
        torch.cuda.synchronize(dev)
        ms = {k: [] for k in variants}
        for _ in range(a.reps):
            for k, f in variants.items():
                flush.zero_()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                f()
                e.record()
                e.synchronize()
                ms[k].append(s.elapsed_time(e))
        out[name] = {k + "_ms": float(np.median(v)) for k, v in ms.items()}
        out[name]["spread_ms"] = {k: [float(min(v)), float(max(v))] for k, v in ms.items()}
        keys = list(variants)
        out[name]["ratio"] = out[name][keys[1] + "_ms"] / out[name][keys[0] + "_ms"]

    from torch.profiler import ProfilerActivity, profile

    kernels = {}
    for name, variants in pairs.items():
        for k, f in variants.items():
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    f()
                torch.cuda.synchronize(dev)
            for ev in prof.key_averages():
                if ev.device_type is not None and "kernel" in ev.key and ev.key != "at::native":
                    t = getattr(ev, "device_time_total", None)
                    if t is None:
                        t = ev.cuda_time_total
                    if t > 0:
                        kernels.setdefault(f"{name}/{k}", {})[ev.key[:60]] = round(t / 5 / 1e3, 4)   # ms per call
    out["kernels_ms_per_call"] = kernels
    print(json.dumps(out))


if __name__ == "__main__":
    main()
