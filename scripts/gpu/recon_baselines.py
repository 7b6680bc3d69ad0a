"""The traditional-reconstruction baselines at the reference's synthetic sizes, end to end on one GPU:

    python scripts/gpu/recon_baselines.py [--out DIR] [--methods fdk,sart,cgls,fista_tv] [--fista_lambdas 1e-3,3e-3]
                                          [--power_iters 20]

A seeded phantom of random ellipsoids (256^3, densities in [0, 1]) -> `generate_data` with the reference's cone-beam
scanner (DSD 7, DSO 5, 512^2 detector of size 4, 2^3 volume, accuracy 0.5, Poisson 1e4 + Gaussian (0, 10) noise),
50 train and 100 test views -> `python -m r2_gaussian_b200.recon`.  Prints the top-level eval_3d.yml (3D PSNR / SSIM
and wall time per method) and the card name and power limit; the scene and the outputs go under DIR.
`--fista_lambdas` also runs FISTA-TV (default iterations) at each listed lmbda on the same views and reports 3D PSNR /
SSIM and wall time per value (how FISTA_LAMBDA was chosen); `--power_iters K` reports the Schur bound L that FISTA-TV
uses against K power iterations on A^T A from a seeded start (a lower estimate of |A|^2)."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

SCANNER = {"mode": "cone", "filter": None, "DSD": 7.0, "DSO": 5.0, "nDetector": [512, 512], "sDetector": [4.0, 4.0],
           "nVoxel": [256, 256, 256], "sVoxel": [2.0, 2.0, 2.0], "offOrigin": [0, 0, 0], "offDetector": [0, 0],
           "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0, "noise": True, "possion_noise": 10000,
           "gaussian_noise": [0, 10]}


def phantom(n: int = 256, count: int = 12, seed: int = 0) -> np.ndarray:
    """A body ellipsoid of density 0.3 holding `count` seeded rotated ellipsoids; clipped to [0, 1]."""
    rng = np.random.RandomState(seed)
    x = (np.arange(n) + 0.5) * 2.0 / n - 1.0
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    P = np.stack([X, Y, Z], -1)
    vol = np.where((X / 0.8) ** 2 + (Y / 0.65) ** 2 + (Z / 0.85) ** 2 <= 1.0, 0.3, 0.0)
    for _ in range(count):
        c = rng.uniform(-0.45, 0.45, 3)
        r = rng.uniform(0.06, 0.25, 3)
        q = rng.randn(4)
        q /= np.linalg.norm(q)
        w, a, b, d = q
        R = np.array([[1 - 2 * (b * b + d * d), 2 * (a * b - w * d), 2 * (a * d + w * b)],
                      [2 * (a * b + w * d), 1 - 2 * (a * a + d * d), 2 * (b * d - w * a)],
                      [2 * (a * d - w * b), 2 * (b * d + w * a), 1 - 2 * (a * a + b * b)]])
        L = ((P - c) @ R / r) ** 2
        vol = vol + np.where(L.sum(-1) <= 1.0, rng.uniform(-0.2, 0.6), 0.0)
    return np.clip(vol, 0.0, 1.0).astype(np.float32)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="scene and outputs (default: a new temporary directory)")
    ap.add_argument("--methods", default="fdk,sart,cgls")
    ap.add_argument("--fista_lambdas", default="", help="comma-separated lmbda values for a FISTA-TV sweep")
    ap.add_argument("--power_iters", type=int, default=0)
    a = ap.parse_args()
    if a.out is None:
        import tempfile

        a.out = tempfile.mkdtemp(prefix="recon_baselines_")
    import torch
    import yaml

    import secondary
    from r2_gaussian_b200 import generate_data, recon

    os.makedirs(a.out, exist_ok=True)
    vol_path = os.path.join(a.out, "phantom.npy")
    np.save(vol_path, phantom())
    yml = os.path.join(a.out, "cone_beam.yml")
    with open(yml, "w") as f:
        yaml.safe_dump(SCANNER, f)
    case = generate_data.main(["--vol", vol_path, "--scanner", yml, "--output", os.path.join(a.out, "data"),
                               "--n_train", "50", "--n_test", "100"])
    report = recon.main(["-s", case, "-m", os.path.join(a.out, "trad"), "--methods", a.methods])
    extra = {}
    if a.fista_lambdas or a.power_iters:
        import time

        from r2_gaussian_b200.dataset import read_scene
        from r2_gaussian_b200.metrics import metric_vol
        from r2_gaussian_b200.projector import CTOperator

        info = read_scene(case, eval=False)
        cfg = info.scanner_cfg
        b = torch.from_numpy(np.stack([np.asarray(c.image, np.float32) for c in info.train_cameras])).cuda()
        angles = [c.angle for c in info.train_cameras]
        vol_gt = np.asarray(info.vol, np.float32)
        sweep = {}
        for lam in [float(t) for t in a.fista_lambdas.split(",") if t.strip()]:
            torch.cuda.synchronize()
            t0 = time.time()
            x, hist = recon.fista_tv(b, angles, cfg, lmbda=lam)
            torch.cuda.synchronize()
            dt = time.time() - t0
            pred = x.cpu().numpy()
            sweep[lam] = {"psnr_3d": float(metric_vol(vol_gt, pred, "psnr")[0]),
                          "ssim_3d": float(metric_vol(vol_gt, pred, "ssim")[0]), "duration (sec)": dt,
                          "F_first": hist[0]["F"], "F_last": hist[-1]["F"]}
            print(f"fista_tv lmbda {lam:g}: {sweep[lam]}")
        extra["fista_sweep"] = sweep
        if a.power_iters:
            op = CTOperator(angles, cfg, b.device)
            L = recon.schur_lipschitz(b, op.A, op.At, op.nvox)
            x = torch.rand(op.nvox, device=b.device, generator=torch.Generator("cuda").manual_seed(0))
            est = 0.0
            for _ in range(a.power_iters):
                x = x / torch.linalg.vector_norm(x)
                x = op.At(op.A(x))
                est = float(torch.linalg.vector_norm(x))
            extra["lipschitz"] = {"schur": L, "power_iteration": est, "iters": a.power_iters, "ratio": L / est}
    print(json.dumps({"recon": report, **extra, **secondary.card(torch.device("cuda"))}))


if __name__ == "__main__":
    main()
