"""The TV prox kernel (r2x_tv_prox) at 256^3, and its share of one FISTA-TV iteration:

    python scripts/gpu/tv_prox_bench.py [--n 256] [--reps 10]

Times `tv.tv_denoise` at 1 and 21 inner iterations with CUDA events, a 256 MB buffer written before each timed call so
that L2 starts cold; (t21 - t1) / 20 is the time of one inner iteration.  The design moves 40 bytes per voxel per
steady inner iteration (two dual fields of 12 bytes read, v read, one dual field written), which over the H100 SXM's
3.35 TB/s is the HBM floor printed beside it.  Then one A and one A^T (CTOperator, 50 cone views of 512^2 onto the same
grid, the scene of recon_baselines.py) and the 20-iteration prox, whose ratio is the prox's share of a FISTA-TV
iteration (which also runs one more A for its history).  Prints one JSON line with the card name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

BYTES_PER_VOXEL = 40
HBM_BYTES_PER_S = 3.35e12


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=256)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    import torch

    import fdk_cases as fc
    import secondary
    from r2_gaussian_b200.projector import CTOperator
    from r2_gaussian_b200.tv import tv_denoise

    if not torch.cuda.is_available():
        raise SystemExit("tv_prox_bench needs a CUDA device")
    dev = torch.device("cuda")
    n = a.n
    g = torch.Generator("cuda").manual_seed(0)
    v = torch.rand((n, n, n), device=dev, generator=g) - 0.2
    flush = torch.empty(64 << 20, dtype=torch.float32, device=dev)

    def timed(fn, reps):
        fn()                                                            # warm-up of this shape
        ms = []
        for _ in range(reps):
            flush.fill_(1.0)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            e.synchronize()
            ms.append(s.elapsed_time(e))
        ms.sort()
        return ms[len(ms) // 2]

    w = 0.02
    t1 = timed(lambda: tv_denoise(v, w, 1), a.reps)
    t21 = timed(lambda: tv_denoise(v, w, 21), a.reps)
    t20 = timed(lambda: tv_denoise(v, w, 20), a.reps)
    inner_us = (t21 - t1) / 20 * 1e3
    floor_us = BYTES_PER_VOXEL * n ** 3 / HBM_BYTES_PER_S * 1e6

    sc = fc.scanner("cone", 512, n)
    op = CTOperator(fc.full_scan(50), sc, dev)
    x = torch.rand((n, n, n), device=dev, generator=g)
    y = op.A(x)
    tA = timed(lambda: op.A(x), max(3, a.reps // 3))
    tAt = timed(lambda: op.At(y), max(3, a.reps // 3))
    iter_ms = tA + tAt + tA + t20
    print(json.dumps({
        "n": n, "prox_1_ms": t1, "prox_20_ms": t20, "prox_21_ms": t21, "inner_iteration_us": inner_us,
        "hbm_floor_us": floor_us, "floor_share": floor_us / inner_us,
        "A_ms_50x512": tA, "At_ms_50x512": tAt,
        "prox20_share_of_fista_iteration": t20 / iter_ms, "fista_iteration_ms": iter_ms,
        **secondary.card(dev)}))


if __name__ == "__main__":
    main()
