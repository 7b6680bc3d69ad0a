"""cp_tv (Chambolle-Pock for min TV(x) s.t. |A x - b| <= epsilon, x >= 0) on the noisy scene of recon_baselines.py:

    python scripts/gpu/cp_tv_bench.py [--out DIR] [--curve 25,50,100,200,400] [--reps 5] [--power_iters 20]
                                      [--no_fista]

The seeded 256^3 ellipsoid phantom -> `generate_data` (the reference's cone-beam scanner, 512^2 detector, Poisson 1e4 +
Gaussian (0, 10) noise, 50 train and 100 test views), then on the 50 train views:
- the time of each part of one iteration with CUDA events (medians of --reps, L2 flushed by a 256 MB write before each
  call): A, A^T, the step kernel (r2x_tv_cp_step at 256^3), the data dual with the rest of the projection-space
  work (torch ops and two float64 norms, which synchronise the host) and the history's TV; the step kernel's 44
  bytes per voxel over the H100 SXM's data-sheet 3.35 TB/s is the HBM floor printed beside it;
- the convergence curve: one cp_tv_solve run to max(--curve) iterations at the default epsilon (0.15 |A FDK(b) - b|),
  3D PSNR / SSIM, residual / epsilon and TV at each listed iteration (a run of N iterations has the first N iterates
  of a longer one, bit for bit);
- `recon.cp_tv` at its defaults end to end (epsilon included), wall time and 3D PSNR / SSIM, and `recon.fista_tv` at
  its defaults on the same views for comparison (skipped with --no_fista);
- the Schur bound L that both use against --power_iters power iterations on A^T A from a seeded start.
Prints one JSON line with the card name and power limit; the scene goes under DIR."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "scripts", "gpu"))

STEP_BYTES_PER_VOXEL = 44
HBM_BYTES_PER_S = 3.35e12


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="scene directory (default: a new temporary directory)")
    ap.add_argument("--curve", default="25,50,100,200,400", help="iterations at which to score the iterate ('' skips)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--power_iters", type=int, default=20)
    ap.add_argument("--no_fista", action="store_true")
    a = ap.parse_args()
    import torch
    import yaml

    import secondary
    from r2_gaussian_b200 import generate_data, recon
    from r2_gaussian_b200.dataset import read_scene
    from r2_gaussian_b200.metrics import metric_vol
    from r2_gaussian_b200.projector import CTOperator
    from r2_gaussian_b200.tv import tv_cp_step, tv_value
    from recon_baselines import SCANNER, phantom

    if not torch.cuda.is_available():
        raise SystemExit("cp_tv_bench needs a CUDA device")
    if a.out is None:
        import tempfile

        a.out = tempfile.mkdtemp(prefix="cp_tv_bench_")
    os.makedirs(a.out, exist_ok=True)
    vol_path = os.path.join(a.out, "phantom.npy")
    np.save(vol_path, phantom())
    yml = os.path.join(a.out, "cone_beam.yml")
    with open(yml, "w") as f:
        yaml.safe_dump(SCANNER, f)
    case = generate_data.main(["--vol", vol_path, "--scanner", yml, "--output", os.path.join(a.out, "data"),
                               "--n_train", "50", "--n_test", "100"])
    info = read_scene(case, eval=False)
    cfg = info.scanner_cfg
    dev = torch.device("cuda")
    b = torch.from_numpy(np.stack([np.asarray(c.image, np.float32) for c in info.train_cameras])).to(dev)
    angles = [c.angle for c in info.train_cameras]
    vol_gt = np.asarray(info.vol, np.float32)
    op = CTOperator(angles, cfg, dev)
    n = op.nvox
    nvox = int(np.prod(n))

    def score(x):
        pred = x.cpu().numpy()
        return float(metric_vol(vol_gt, pred, "psnr")[0]), float(metric_vol(vol_gt, pred, "ssim")[0])

    # ---- the parts of one iteration
    flush = torch.empty(64 << 20, dtype=torch.float32, device=dev)

    def timed(fn):
        fn()                                                            # warm-up of this shape
        ms = []
        for _ in range(a.reps):
            flush.fill_(1.0)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            e.synchronize()
            ms.append(s.elapsed_time(e))
        ms.sort()
        return ms[len(ms) // 2]

    g = torch.Generator("cuda").manual_seed(0)
    x = torch.rand(n, device=dev, generator=g)
    xbar = torch.rand(n, device=dev, generator=g)
    p = torch.rand((3,) + n, device=dev, generator=g) * 0.1
    y = op.A(x)
    grad = op.At(y)
    tau, sigma, nu = recon.cp_step_sizes(2.5)

    def projection_space():
        """cp_tv_solve's projection-space work of one iteration: the data dual, q, the history's residual and A xbar."""
        v = y.sub(b).add_(y)
        norm = recon._dot(v, v) ** 0.5
        q = v.mul_(0.5).mul(sigma)
        r = y.sub(b)
        return q, recon._dot(r, r), y.mul(2.0).sub_(y), norm

    parts = {"A_ms": timed(lambda: op.A(x)), "At_ms": timed(lambda: op.At(y)),
             "step_ms": timed(lambda: tv_cp_step(x, xbar, p, grad, tau, sigma, nu, True)),
             "data_dual_ms": timed(projection_space), "tv_value_ms": timed(lambda: tv_value(x))}
    parts["iteration_ms"] = sum(parts.values())
    floor_ms = STEP_BYTES_PER_VOXEL * nvox / HBM_BYTES_PER_S * 1e3
    parts.update({"step_bytes_per_voxel": STEP_BYTES_PER_VOXEL, "step_hbm_floor_ms": floor_ms,
                  "step_floor_share": floor_ms / parts["step_ms"]})
    print(f"parts {parts}", flush=True)
    del x, xbar, p, y, grad

    # ---- convergence curve at the default epsilon
    eps = recon.cp_tv_epsilon(b, angles, cfg)
    L = recon.schur_lipschitz(b, op.A, op.At, n)
    curve = {}
    marks = sorted({int(t) for t in a.curve.split(",") if t.strip()})
    if marks:
        kept = {}
        count = [0]

        def tv_keep(v):
            count[0] += 1
            if count[0] in marks:
                kept[count[0]] = v.clone()
            return tv_value(v)

        _, hist = recon.cp_tv_solve(b, op.A, op.At, n, marks[-1], eps, L, True, tv=tv_keep)
        for k in marks:
            ps, ss = score(kept.pop(k))
            curve[k] = {"psnr_3d": ps, "ssim_3d": ss, "residual_over_epsilon": hist[k - 1]["residual"] / eps,
                        "tv": hist[k - 1]["tv"]}
            print(f"cp_tv iteration {k}: {curve[k]}", flush=True)

    # ---- the defaults end to end, and FISTA-TV on the same views
    rows = {}
    methods = [("cp_tv", lambda: recon.cp_tv(b, angles, cfg))]
    if not a.no_fista:
        methods.append(("fista_tv", lambda: recon.fista_tv(b, angles, cfg)))
    for name, fn in methods:
        torch.cuda.synchronize()
        t0 = time.time()
        x, hist = fn()
        torch.cuda.synchronize()
        dt = time.time() - t0
        ps, ss = score(x)
        rows[name] = {"psnr_3d": ps, "ssim_3d": ss, "duration (sec)": dt, "iterations": len(hist)}
        if name == "cp_tv":
            rows[name].update({"epsilon": eps, "residual_over_epsilon": hist[-1]["residual"] / eps})
        print(f"{name}: {rows[name]}", flush=True)

    lip = {"schur": L}
    if a.power_iters:
        v = torch.rand(n, device=dev, generator=torch.Generator("cuda").manual_seed(0))
        est = 0.0
        for _ in range(a.power_iters):
            v = v / torch.linalg.vector_norm(v)
            v = op.At(op.A(v))
            est = float(torch.linalg.vector_norm(v))
        lip.update({"power_iteration": est, "iters": a.power_iters, "ratio": L / est})
    print(json.dumps({"nvox": list(n), "views": len(angles), "parts": parts, "curve": curve, "defaults": rows,
                      "lipschitz": lip, "cp_niter": recon.CP_NITER, **secondary.card(dev)}))


if __name__ == "__main__":
    main()
