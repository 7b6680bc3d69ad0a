"""Cost and effect of stripe removal (r2x_remove_stripes, `stripes.remove_stripes`):

    python scripts/gpu/stripes_bench.py [--reps 10] [--out DIR] [--json FILE] [--skip_quality]

Time: one in-place call, at the default window and at sarepy's 21, at 721 x 560^2 (a FIPS scene at proj_subsample
4), 150 x 512^2 and 721 x 2368 x 2240 (a FIPS scan at full resolution, past 2^31 samples), median of --reps CUDA-event
timings after two warm-up calls, each against the floor of 8 bytes per sample (one read and one write of every float)
at the H100 SXM's 3.35 TB/s data-sheet bandwidth.  A torch.profiler run splits the first shape into the sort pass and
the median pass.
Quality, at the default window (`stripes.DEFAULT_SIZE`) unless swept: FDK psnr_3d / SSIM on the seeded 48^3 scene of
tests/test_eval_gpu.py and on recon_baselines.py's noisy 256^3 phantom with 50 views, each clean, striped (constant
per-pixel offsets of 5 % of the largest projection value on 10 % of the detector columns, the same in every view),
striped + removed and clean + removed -- the last is the cost of removing stripes that are not there; the same four
cases for a 1000-iteration `trainer` run on the 48^3 scene; a sweep of the window, 3 / 5 / 7 / 11 / 21 / 41, over the
striped and the clean 48^3 and 256^3 scenes with FDK; and the pseudo-GT psnr_3d against the phantom of
`generate_real_data [--remove_stripes K]` on the 90-view FIPS-format scan of tests/test_real_data_gpu.py (a 64-pixel
detector), clean and with the stripes of tests/test_stripes_gpu.py, for K = 3, 5 and 21.  The corrected scenes are
written by `python -m r2_gaussian_b200.remove_stripes`, as a user would.
Prints one JSON line with the card's name and power limit, read in the same call."""
from __future__ import annotations

import argparse
import contextlib
import io
import json
import os
import pathlib
import random
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "scripts", "gpu"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

SHAPES = [(721, 560, 560), (150, 512, 512), (721, 2368, 2240)]
HBM_BYTES_PER_S = 3.35e12
SWEEP = (3, 5, 7, 11, 21, 41)
FIPS_SIZES = (None, 3, 5, 21)


def timing(dev, reps: int) -> dict:
    import torch

    from r2_gaussian_b200.stripes import DEFAULT_SIZE, remove_stripes

    rows = {}
    for K, (n, H, W) in [(K, s) for K in sorted({DEFAULT_SIZE, 21}) for s in SHAPES]:
        x = torch.rand((n, H, W), device=dev, generator=torch.Generator(dev).manual_seed(0))
        for _ in range(2):
            remove_stripes(x, K, out=x)
        torch.cuda.synchronize(dev)
        ms = []
        for _ in range(reps if n * H * W < 2 ** 31 else max(3, reps // 3)):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            remove_stripes(x, K, out=x)
            e.record()
            e.synchronize()
            ms.append(s.elapsed_time(e))
        floor_ms = 8.0 * n * H * W / HBM_BYTES_PER_S * 1e3
        rows[f"K{K} {n}x{H}x{W}"] = {"call_ms": float(np.median(ms)), "spread_ms": [float(min(ms)), float(max(ms))],
                                     "hbm_floor_ms": floor_ms, "floor_over_time": floor_ms / float(np.median(ms))}
        print(f"K{K} {n}x{H}x{W}", rows[f"K{K} {n}x{H}x{W}"], flush=True)
        del x
        torch.cuda.empty_cache()

    from torch.profiler import ProfilerActivity, profile

    n, H, W = SHAPES[0]
    x = torch.rand((n, H, W), device=dev, generator=torch.Generator(dev).manual_seed(0))
    remove_stripes(x, 21, out=x)
    torch.cuda.synchronize(dev)
    for K in sorted({DEFAULT_SIZE, 21}):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                remove_stripes(x, K, out=x)
            torch.cuda.synchronize(dev)
        split = {}
        for ev in prof.key_averages():
            for name in ("stripes_sort_kernel", "stripes_median_kernel"):
                if name in ev.key:
                    t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
                    split[name] = t / ev.count / 1e3
        rows[f"K{K} {n}x{H}x{W}"]["kernel_ms"] = split
    return rows


def _quiet(fn, *args, **kw):
    with contextlib.redirect_stdout(io.StringIO()):
        return fn(*args, **kw)


def fdk_score(scene: str) -> dict:
    import torch

    from r2_gaussian_b200.dataset import read_scene
    from r2_gaussian_b200.fdk import fdk
    from r2_gaussian_b200.metrics import metric_vol

    info = read_scene(scene, eval=False)
    b = torch.from_numpy(np.stack([np.asarray(c.image, np.float32) for c in info.train_cameras])).cuda()
    pred = fdk(b, [c.angle for c in info.train_cameras], info.scanner_cfg).cpu().numpy()
    gt = np.asarray(info.vol, np.float32)
    return {"psnr_3d": float(metric_vol(gt, pred, "psnr")[0]), "ssim_3d": float(metric_vol(gt, pred, "ssim")[0])}


def striped_copy(clean: str, out: str, seed: int) -> str:
    from test_stripes_gpu import _add_stripes

    with open(os.path.join(clean, "meta_data.json")) as f:
        meta = json.load(f)
    rels = [fr["file_path"] for s in ("proj_train", "proj_test") for fr in meta[s]]
    views = [np.load(os.path.join(clean, r)) for r in rels]
    amp = 0.05 * float(max(v.max() for v in views))
    for r, v in zip(rels, _add_stripes(views, 0.1, np.random.default_rng(seed), amp)):
        os.makedirs(os.path.dirname(os.path.join(out, r)), exist_ok=True)
        np.save(os.path.join(out, r), v)
    for f in ("meta_data.json", meta["vol"]):
        shutil.copyfile(os.path.join(clean, f), os.path.join(out, f))
    return out


def four_cases(clean: str, root: str) -> dict:
    from r2_gaussian_b200.remove_stripes import remove_scene_stripes
    from r2_gaussian_b200.stripes import DEFAULT_SIZE as size

    striped = striped_copy(clean, os.path.join(root, "striped"), 8)
    return {"clean": clean, "striped": striped,
            "striped_removed": _quiet(remove_scene_stripes, striped, os.path.join(root, f"striped_k{size}"), size),
            "clean_removed": _quiet(remove_scene_stripes, clean, os.path.join(root, f"clean_k{size}"), size)}


def train_score(scene: str, root: str) -> float:
    import torch

    from r2_gaussian_b200 import initialize_pcd, trainer

    init = _quiet(initialize_pcd.main, ["--data", scene, "--n_points", "5000",
                                        "--output", os.path.join(root, os.path.basename(scene) + "_init.npy")])
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    model = trainer.ModelParams(source_path=scene, model_path="", ply_path=init)
    hist = trainer.training(model, trainer.OptimizationParams(iterations=1000), trainer.PipelineParams(), {1000},
                            set(), log=lambda *a: None)
    return float(hist["eval"][1000]["psnr_3d"])


def quality(out: str) -> dict:
    import yaml

    import recon_baselines
    from r2_gaussian_b200 import generate_data
    from r2_gaussian_b200.remove_stripes import remove_scene_stripes
    from test_projector_gpu import _write_inputs

    res = {}
    tmp = pathlib.Path(out) / "s48"
    tmp.mkdir(parents=True, exist_ok=True)
    yml, vol_path, *_ = _write_inputs(tmp, noise=False)
    clean48 = _quiet(generate_data.main, ["--vol", str(vol_path), "--scanner", str(yml), "--n_train", "24",
                                          "--n_test", "6", "--output", str(tmp / "clean")])
    cases48 = four_cases(clean48, str(tmp))
    res["fdk_48"] = {k: fdk_score(v) for k, v in cases48.items()}
    print("fdk_48", res["fdk_48"], flush=True)

    t256 = pathlib.Path(out) / "s256"
    t256.mkdir(parents=True, exist_ok=True)
    np.save(t256 / "phantom.npy", recon_baselines.phantom())
    with open(t256 / "scanner.yml", "w") as f:
        yaml.safe_dump(recon_baselines.SCANNER, f)
    clean256 = _quiet(generate_data.main, ["--vol", str(t256 / "phantom.npy"), "--scanner", str(t256 / "scanner.yml"),
                                           "--output", str(t256 / "clean"), "--n_train", "50", "--n_test", "1"])
    res["fdk_256_noisy"] = {k: fdk_score(v) for k, v in four_cases(clean256, str(t256)).items()}
    print("fdk_256_noisy", res["fdk_256_noisy"], flush=True)

    res["train_48_psnr_3d"] = {k: train_score(v, str(tmp)) for k, v in cases48.items()}
    print("train_48", res["train_48_psnr_3d"], flush=True)

    cases256 = {"clean": clean256, "striped": os.path.join(str(t256), "striped")}
    for label, cases, root in (("sweep_fdk_48", cases48, tmp), ("sweep_fdk_256_noisy", cases256, t256)):
        res[label] = {K: {name: fdk_score(_quiet(remove_scene_stripes, cases[name], str(root / f"sweep_{name}_{K}"), K))
                          for name in ("striped", "clean")} for K in SWEEP}
        print(label, res[label], flush=True)
    res["fips_pseudo_gt_psnr_3d"] = fips(pathlib.Path(out) / "fips")
    print("fips", res["fips_pseudo_gt_psnr_3d"], flush=True)
    return res


def fips(tmp) -> dict:
    """Pseudo-GT psnr_3d of generate_real_data [--remove_stripes K] on the clean and the striped FIPS-format scan."""
    import scipy.io

    import real_data_oracle as rdo
    from r2_gaussian_b200 import generate_real_data as grd
    from r2_gaussian_b200.metrics import metric_vol
    from test_real_data_gpu import _fips_scan
    from test_stripes_gpu import fips_stripes

    tmp.mkdir(parents=True, exist_ok=True)
    scan, phantom = _fips_scan(tmp)
    names = sorted(f for f in os.listdir(scan) if f.endswith(".mat"))
    raw = [scipy.io.loadmat(os.path.join(scan, f))["img"] for f in names]
    rdo.write_fips_case(str(tmp / "striped"), fips_stripes(raw), 0.0, 4.0, dsd=553.74, dso=410.66, pixel=1.0 / 4)
    res = {}
    for name, data in (("clean", scan), ("striped", str(tmp / "striped"))):
        for K in FIPS_SIZES:
            args = ["--data", data, "--n_train", "30", "--n_test", "20", "--nVoxel", "48", "48", "48",
                    "--output", str(tmp / f"{name}_{K}"), *(["--remove_stripes", str(K)] if K else [])]
            p = _quiet(grd.main, args)
            res[f"{name} K={K}"] = float(metric_vol(phantom, np.load(os.path.join(p, "vol_gt.npy")), "psnr")[0])
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="scenes (default: a new temporary directory)")
    ap.add_argument("--json", default=None, help="also write the JSON line to this file")
    ap.add_argument("--skip_quality", action="store_true")
    a = ap.parse_args()
    import torch

    import secondary

    if not torch.cuda.is_available():
        raise SystemExit("stripes_bench needs a CUDA device")
    dev = torch.device("cuda")
    out = a.out or tempfile.mkdtemp(prefix="stripes_")
    os.makedirs(out, exist_ok=True)
    row = {"workload": "r2x_remove_stripes in place, window 21", **secondary.card(dev), "time": timing(dev, a.reps)}
    if not a.skip_quality:
        row["quality"] = quality(out)
    line = json.dumps({**row, **secondary.card(dev)})
    print(line)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
