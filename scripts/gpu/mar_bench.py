"""Cost and effect of metal artifact reduction (r2x_mar_inpaint, `mar.reduce_metal`, `recon --mar`):

    python scripts/gpu/mar_bench.py [--reps 20] [--out DIR] [--json FILE] [--skip_quality]

Time: `mar.inpaint` out of place with the trace output, without and with a prior, on 50 x 512^2 and 721 x 560^2
stacks (a 5 % random trace dilated by 1), median of --reps CUDA-event timings after two warm-up calls, with L2 flushed
(a 256 MiB write) before each; each against the HBM floor of the bytes the kernel must move (p and m read, out
written, the trace written: 13 bytes per sample, 17 with the prior read) at the H100 SXM's 3.35 TB/s data-sheet
bandwidth.  Then a whole `reduce_metal` call (FDK, mask projection, inpainting; NMAR adds the second FDK, the prior's
projection and the second inpainting) on 50 views of 512^2 -> 256^3, median of 3 host-clock timings ending in a device
synchronise.
Quality, on cone-beam metal scenes of tests/mar_cases.py (64^3 grid, 64^2 detector, 60 train views): a sweep of
TRACE_TAU x TRACE_DILATE with the true mask and of the metal threshold, scored by NMAR's FDK psnr_3d_outside_metal
(always against the true mask, so thresholds compare); then `recon --mar` li / nmar and without, for fdk and cgls, on
the photon-starved scene (metal 3.0, I0 = 1e4), a weak-artifact scene (metal 1.0, no noise) and the ideal monochromatic
scene; and a 1000-iteration training on the starved scene and on its `reduce_metal` correction, each scored outside
the metal (the corrected one with the metal of the uncorrected FDK reinserted).
Prints one JSON line with the card's name, power limit and SM clocks, read in the same call."""
from __future__ import annotations

import argparse
import contextlib
import io
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

SHAPES = [(50, 512, 512), (721, 560, 560)]
HBM_BYTES_PER_S = 3.35e12
TAUS = (0.1, 0.25, 0.5, 1.0, 2.0)
DILATES = (0, 1, 2, 3)
THRESHOLDS = (0.4, 0.6, 1.0, 1.5, 2.0)


def clocks() -> dict:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=20)
        sm, mx = (float(v) for v in r.stdout.strip().splitlines()[0].split(","))
        return {"sm_clock_mhz": sm, "max_sm_clock_mhz": mx}
    except Exception:
        return {"sm_clock_mhz": None, "max_sm_clock_mhz": None}


def timing(dev, reps: int) -> dict:
    import torch

    from r2_gaussian_b200.mar import inpaint

    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    rows = {}
    for n, H, W in SHAPES:
        g = torch.Generator(dev).manual_seed(0)
        p = torch.rand((n, H, W), device=dev, generator=g)
        m = (torch.rand((n, H, W), device=dev, generator=g) < 0.05).to(torch.float32)
        P = torch.rand((n, H, W), device=dev, generator=g) + 0.5
        out = torch.empty_like(p)
        tr = torch.empty((n, H, W), dtype=torch.uint8, device=dev)
        for label, prior, nbytes in (("li", None, 13), ("nmar", P, 17)):
            for _ in range(2):
                inpaint(p, m, 0.5, 1, prior, out=out, trace=tr)
            torch.cuda.synchronize(dev)
            ms = []
            for _ in range(reps):
                flush.zero_()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                inpaint(p, m, 0.5, 1, prior, out=out, trace=tr)
                e.record()
                e.synchronize()
                ms.append(s.elapsed_time(e))
            t = float(np.median(ms))
            floor_ms = nbytes * n * H * W / HBM_BYTES_PER_S * 1e3
            key = f"{label} {n}x{H}x{W}"
            rows[key] = {"call_ms": t, "spread_ms": [float(min(ms)), float(max(ms))], "hbm_floor_ms": floor_ms,
                         "achieved_gb_s": nbytes * n * H * W / t / 1e6, "floor_over_time": floor_ms / t}
            print(key, rows[key], flush=True)
        del p, m, P, out, tr
        torch.cuda.empty_cache()
    return rows


def reduce_timing(dev) -> dict:
    import torch

    import mar_cases
    from r2_gaussian_b200.mar import reduce_metal
    from r2_gaussian_b200.projector import project
    from r2_gaussian_b200.scene import cone_beam_scanner

    sc = cone_beam_scanner(512, 256)
    cfg = dict(sc, dVoxel=[2.0 / 256] * 3, dDetector=[4.0 / 512] * 2)
    tissue, metal, mask = mar_cases.phantom(256)
    ang = np.linspace(0, 2 * np.pi, 50, endpoint=False)
    p_t = project(torch.from_numpy(tissue).to(dev), ang, cfg)
    p_m = project(torch.from_numpy(metal).to(dev), ang, cfg)
    p = mar_cases.polychromatic(p_t, p_m, 6.0, 1e4, np.random.default_rng(0))
    res = {}
    for method in ("li", "nmar"):
        reduce_metal(p, ang, cfg, method=method, mask=mask)
        ts = []
        for _ in range(3):
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            reduce_metal(p, ang, cfg, method=method, mask=mask)
            torch.cuda.synchronize(dev)
            ts.append((time.perf_counter() - t0) * 1e3)
        res[f"reduce_metal {method} 50x512^2 -> 256^3 ms"] = float(np.median(ts))
        print(method, res, flush=True)
    return res


def _quiet(fn, *a, **k):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*a, **k)


def _recon_scores(path, mask_path, tmp, methods="fdk,cgls"):
    from r2_gaussian_b200 import recon

    import mar_oracle as mo

    out = {}
    plain = _quiet(recon.main, ["-s", path, "-m", os.path.join(tmp, "plain"), "--methods", methods])
    gt = np.load(os.path.join(path, "vol_gt.npy"))
    mask = np.load(mask_path)
    for m in methods.split(","):
        ct = np.load(os.path.join(tmp, "plain", m, "ct_pred.npy"))
        out[f"{m}"] = mo.psnr_outside_metal(gt, ct, mask)
        out[f"{m} psnr_3d"] = plain[m]["psnr_3d"]
    for mar in ("li", "nmar"):
        r = _quiet(recon.main, ["-s", path, "-m", os.path.join(tmp, mar), "--methods", methods, "--mar", mar,
                                "--metal_mask", mask_path])
        for m in methods.split(","):
            out[f"{m}+{mar}"] = r[m]["psnr_3d_outside_metal"]
    return out


def quality(tmp) -> dict:
    import torch

    import mar_cases
    import mar_oracle as mo
    from r2_gaussian_b200 import mar
    from r2_gaussian_b200.dataset import read_scene
    from r2_gaussian_b200.fdk import fdk

    res = {}
    scenes = {"starved": dict(metal_density=3.0, I0=1e4), "weak": dict(metal_density=1.0, I0=None),
              "mono": dict(metal_density=3.0, mono=True)}
    paths = {}
    for name, kw in scenes.items():
        path, tissue, metal, mask = mar_cases.metal_scene(os.path.join(tmp, name), **kw)
        np.save(os.path.join(tmp, f"{name}_mask.npy"), mask)
        paths[name] = (path, os.path.join(tmp, f"{name}_mask.npy"))

    # sweep on the starved scene, NMAR FDK scored against the true mask
    path, mask_path = paths["starved"]
    mask = np.load(mask_path)
    info = read_scene(path)
    cfg = info.scanner_cfg
    p = torch.from_numpy(np.stack([c.image for c in info.train_cameras]).astype(np.float32)).cuda()
    ang = [c.angle for c in info.train_cameras]
    gt = info.vol

    def score(r):
        return mo.psnr_outside_metal(gt, fdk(r.projs, ang, cfg).cpu().numpy(), mask)

    sweep = {}
    for tau in TAUS:
        for d in DILATES:
            sweep[f"tau {tau} dilate {d}"] = score(mar.reduce_metal(p, ang, cfg, mask=mask, trace_tau=tau,
                                                                    trace_dilate=d))
    res["sweep_trace"] = sweep
    print("sweep_trace", sweep, flush=True)
    vol0 = fdk(p, ang, cfg)
    thr = {"fdk_max": float(vol0.max())}
    for t in THRESHOLDS:
        try:
            r = mar.reduce_metal(p, ang, cfg, threshold=t)
            thr[f"threshold {t}"] = {"psnr_outside_true_metal": score(r), "metal_voxels": int(r.mask.sum()),
                                     "true_metal_voxels": int(mask.sum())}
        except ValueError as e:
            thr[f"threshold {t}"] = str(e)
    res["sweep_threshold"] = thr
    print("sweep_threshold", thr, flush=True)

    for name, (path, mask_path) in paths.items():
        res[f"recon_{name}"] = _recon_scores(path, mask_path, os.path.join(tmp, f"recon_{name}"))
        print(f"recon_{name}", res[f"recon_{name}"], flush=True)

    res["train_starved"] = training(paths["starved"], tmp)
    print("train_starved", res["train_starved"], flush=True)
    return res


def training(scene, tmp, iterations: int = 1000) -> dict:
    import torch

    import mar_oracle as mo
    from r2_gaussian_b200 import initialize_pcd, reduce_metal as rm, trainer
    from r2_gaussian_b200.dataset import read_scene
    from r2_gaussian_b200.fdk import fdk

    path, mask_path = scene
    mask = np.load(mask_path)
    fixed = _quiet(rm.main, ["-s", path, "--output", os.path.join(tmp, "starved_nmar"), "--metal_mask", mask_path])
    info = read_scene(path)
    p = torch.from_numpy(np.stack([c.image for c in info.train_cameras]).astype(np.float32)).cuda()
    vol0 = fdk(p, [c.angle for c in info.train_cameras], info.scanner_cfg).cpu().numpy()
    out = {}
    for label, src in (("uncorrected", path), ("nmar", fixed)):
        init = _quiet(initialize_pcd.main, ["--data", src, "--recon_method", "fdk", "--n_points", "20000",
                                            "--output", os.path.join(tmp, f"init_{label}.npy")])
        random.seed(0); np.random.seed(0); torch.manual_seed(0)
        mp = os.path.join(tmp, f"train_{label}")
        model = trainer.ModelParams(source_path=src, model_path=mp, ply_path=init)
        _quiet(trainer.training, model, trainer.OptimizationParams(iterations=iterations), trainer.PipelineParams(),
               {iterations}, {iterations}, log=lambda *a: None)
        vol = np.load(os.path.join(mp, "point_cloud", f"iteration_{iterations}", "vol_pred.npy"))
        if label == "nmar":
            vol = mo.reinsert(vol, vol0, mask)
        out[label] = mo.psnr_outside_metal(info.vol, vol, mask)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None, help="scenes (default: a new temporary directory)")
    ap.add_argument("--json", default=None, help="also write the JSON line to this file")
    ap.add_argument("--skip_quality", action="store_true")
    a = ap.parse_args()
    import torch

    import secondary

    if not torch.cuda.is_available():
        raise SystemExit("mar_bench needs a CUDA device")
    dev = torch.device("cuda")
    out = a.out or tempfile.mkdtemp(prefix="mar_")
    os.makedirs(out, exist_ok=True)
    row = {"workload": "r2x_mar_inpaint and reduce_metal", **secondary.card(dev), **clocks(),
           "time": timing(dev, a.reps), "reduce_metal": reduce_timing(dev)}
    if not a.skip_quality:
        row["quality"] = quality(out)
    line = json.dumps({**row, **secondary.card(dev), "clocks_after": clocks()})
    print(line)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
