"""Real cone-beam scan -> scene -- the reference's `data_generator/real_dataset/generate_data.py`, without TIGRE or cv2.

    python -m r2_gaussian_b200.generate_real_data --data <processed scan dir> --output DIR
        [--proj_subsample 4] [--proj_rescale 400] [--object_scale 50] [--n_test 100] [--n_train 75]
        [--nVoxel 256 256 256] [--sVoxel 2 2 2] [--offOrigin 0 0 0] [--offDetector 0 0] [--accuracy 0.5]
        [--remove_stripes K]

The input is a processed FIPS scan (pine, seashell, walnut): a `config.txt` and one `.mat` per view whose `img` holds the
line integrals.  Step by step:
  * `config.txt` is read with the reference's substring rules (`read_config`); lengths become `/ 1000 * object_scale`
    and the pixel pitch is multiplied by `proj_subsample`.  A missing key is refused by name.
  * The angles are arange(AngleFirst, AngleLast, AngleInterval) + [AngleLast] degrees (`scan_angles`); their count and
    NumberImages must both equal the number of `.mat` files.
  * Train views are linspace(0, n - 1, n_train) cast to int, test views n_test of the others drawn by
    random.Random(0).sample and sorted (`split_ids`): the reference's ids, without touching the global `random` state.
  * Every view goes through `prepare` (r2x_projection_prepare on the GPU: scale, clamp, move up 5 rows, cv2's
    INTER_LINEAR resize and the centre crop), `chunk` views per call, into one float32 stack kept on the device;
    `proj_all/`, `proj_train/` and `proj_test/` get the reference's file names.
  * `--remove_stripes K` (off by default) corrects ring artifacts in that stack of all views before anything is
    written: `stripes.remove_stripes` with a median window of K columns.  The train and test views, `proj_all/` and
    the pseudo ground truth then all come from the corrected projections.
  * The pseudo ground truth `vol_gt.npy` is `fdk.fdk` of all views in scene units (with `use_offDetector` when
    `--offDetector` is not zero, as the reference hands it to TIGRE's FDK), negatives set to 0; an existing file is
    kept.  `meta_data.json` has the reference's keys and scanner fields.

Differences from the reference: the volume is named under `"vol"` (what its own scene reader and `dataset.read_blender`
read) as well as under its `"ct"`; when the resized height and width differ by exactly 1 nothing is cropped (its
`off:-off` slice is empty there); the pseudo ground truth is this project's FDK, not TIGRE's, so scores against it are
not comparable bit for bit with published ones.  Dependencies: numpy, scipy (`loadmat`) and torch with this package's
CUDA library.
"""
from __future__ import annotations

import argparse
import copy
import glob
import json
import os
import random

import numpy as np

DEFAULT_CHUNK = 32          # views per r2x_projection_prepare call (the float64 staging buffer holds this many)

# config.txt key -> name used here; checked in this order, the first substring that matches a line wins
_CONFIG_KEYS = (("NumberImages", "n_proj"), ("AngleInterval", "angle_interval"), ("AngleFirst", "angle_first"),
                ("AngleLast", "angle_last"), ("DistanceSourceDetector", "DSD"), ("DistanceSourceOrigin", "DSO"),
                ("PixelSize", "dDetector"))


def read_config(path: str, proj_subsample: int, object_scale: float) -> dict:
    """The scan geometry of a `config.txt` with the reference's rules: a line counts for the first key (in
    _CONFIG_KEYS order) it contains, `PixelSize` not when it also contains `PixelSizeUnit`, the value is what follows
    the last '='; a key seen twice keeps its last value.  DSD, DSO and dDetector are in metres times object_scale,
    dDetector also times proj_subsample."""
    raw = {}
    with open(path) as f:
        for line in f.readlines():
            for key, name in _CONFIG_KEYS:
                if key in line and not (key == "PixelSize" and "PixelSizeUnit" in line):
                    raw[name] = line.split("=")[-1]
                    break
    missing = [key for key, name in _CONFIG_KEYS if name not in raw]
    if missing:
        raise ValueError(f"{path}: no {', '.join(missing)} line")
    return {"n_proj": int(raw["n_proj"]), "angle_interval": float(raw["angle_interval"]),
            "angle_first": float(raw["angle_first"]), "angle_last": float(raw["angle_last"]),
            "DSD": float(raw["DSD"]) / 1000 * object_scale, "DSO": float(raw["DSO"]) / 1000 * object_scale,
            "dDetector": float(raw["dDetector"]) * proj_subsample / 1000 * object_scale}


def scan_angles(cfg: dict) -> np.ndarray:
    """Radians: arange(first, last, interval) and then last, in degrees, times pi / 180."""
    deg = np.concatenate([np.arange(cfg["angle_first"], cfg["angle_last"], cfg["angle_interval"]), [cfg["angle_last"]]])
    return deg / 180.0 * np.pi


def split_ids(n_proj: int, n_train: int, n_test: int):
    """(train_ids, test_ids) as the reference draws them after random.seed(0), from a private generator."""
    if n_train < 1 or n_test < 0:
        raise ValueError(f"--n_train must be at least 1 and --n_test at least 0, got {n_train} and {n_test}")
    if n_train + n_test > n_proj:
        raise ValueError(f"--n_train {n_train} + --n_test {n_test} views asked of a scan with {n_proj}")
    train_ids = np.linspace(0, n_proj - 1, n_train).astype(int)
    rest = np.setdiff1d(np.arange(n_proj), train_ids).tolist()
    return train_ids, sorted(random.Random(0).sample(rest, n_test))


def prepared_shape(H0: int, W0: int, subsample: int):
    """(H, W) that `prepare` makes of H0 x W0 images."""
    import ctypes as C

    from ._lib import check, load

    hw = (C.c_int * 2)()
    check(load().r2x_projection_prepare_shape(int(H0), int(W0), int(subsample), hw), "r2x_projection_prepare_shape")
    return int(hw[0]), int(hw[1])


def prepare(img, subsample: int, proj_rescale: float, object_scale: float, out=None):
    """r2x_projection_prepare of a CUDA float64 [n, H0, W0] tensor into a CUDA float32 [n, H, W] one (`out`, a
    contiguous tensor of that shape, or a new one), on the current stream."""
    import torch

    from ._lib import check, load

    if not isinstance(img, torch.Tensor) or img.device.type != "cuda" or img.dtype != torch.float64 or img.dim() != 3:
        raise ValueError("prepare: img must be a CUDA float64 [n, H0, W0] tensor")
    img = img.contiguous()
    n, H0, W0 = (int(s) for s in img.shape)
    H, W = prepared_shape(H0, W0, subsample)
    if out is None:
        out = torch.empty((n, H, W), dtype=torch.float32, device=img.device)
    if tuple(out.shape) != (n, H, W) or out.dtype != torch.float32 or not out.is_contiguous() or out.device != img.device:
        raise ValueError(f"prepare: out must be a contiguous float32 {[n, H, W]} tensor on {img.device}")
    with torch.cuda.device(img.device):
        stream = torch.cuda.current_stream(img.device).cuda_stream
        rc = load().r2x_projection_prepare(stream, n, H0, W0, int(subsample), img.data_ptr(), float(proj_rescale),
                                           float(object_scale), out.data_ptr())
    check(rc, "r2x_projection_prepare")
    return out


def load_mat(path: str) -> np.ndarray:
    import scipy.io

    return np.asarray(scipy.io.loadmat(path)["img"], np.float64)


def prepare_files(paths, subsample: int, proj_rescale: float, object_scale: float, chunk: int = DEFAULT_CHUNK):
    """Load the `.mat` files `chunk` at a time into pinned host memory, prepare each chunk on the GPU and return the
    float32 [len(paths), H, W] stack on the device."""
    import torch

    if chunk < 1:
        raise ValueError(f"chunk must be at least 1, got {chunk}")
    first = load_mat(paths[0])
    if first.ndim != 2:
        raise ValueError(f"{paths[0]}: img has shape {first.shape}, expected a 2-D image")
    H0, W0 = first.shape
    H, W = prepared_shape(H0, W0, subsample)
    stack = torch.empty((len(paths), H, W), dtype=torch.float32, device="cuda")
    host = torch.empty((min(chunk, len(paths)), H0, W0), dtype=torch.float64, pin_memory=True)
    dev = torch.empty_like(host, device="cuda")
    for c0 in range(0, len(paths), chunk):
        part = paths[c0:c0 + chunk]
        torch.cuda.current_stream().synchronize()      # the previous chunk's copy has left the staging buffer
        for k, p in enumerate(part):
            img = first if c0 + k == 0 else load_mat(p)
            if img.shape != (H0, W0):
                raise ValueError(f"{p}: img is {img.shape[0]}x{img.shape[1]}, the scan's first view {H0}x{W0}")
            host[k].numpy()[...] = img
        dev[:len(part)].copy_(host[:len(part)], non_blocking=True)
        prepare(dev[:len(part)], subsample, proj_rescale, object_scale, out=stack[c0:c0 + len(part)])
    return stack


def pseudo_ground_truth(stack, angles, scanner_cfg: dict):
    """fdk.fdk of every view in scene units (projections times scene_scale, as `dataset.read_blender` scales them),
    through the detector offset when it is not zero, negatives set to 0: a CUDA float32 [nx, ny, nz] tensor."""
    import torch

    from .dataset import scale_scanner
    from .fdk import fdk

    scaled = copy.deepcopy(scanner_cfg)
    scene_scale = scale_scanner(scaled)
    off = any(float(v) != 0.0 for v in scanner_cfg["offDetector"])
    vol = fdk(stack * scene_scale, angles, scaled, use_offDetector=off)
    return torch.where(vol < 0, torch.zeros_like(vol), vol)


def generate(data: str, output: str, proj_subsample: int = 4, proj_rescale: float = 400.0, object_scale: float = 50,
             n_test: int = 100, n_train: int = 75, nVoxel=(256, 256, 256), sVoxel=(2.0, 2.0, 2.0),
             offOrigin=(0.0, 0.0, 0.0), offDetector=(0.0, 0.0), accuracy: float = 0.5,
             chunk: int = DEFAULT_CHUNK, remove_stripes: int | None = None) -> str:
    import torch

    from .stripes import check_size

    if proj_subsample < 1:
        raise ValueError(f"--proj_subsample must be at least 1, got {proj_subsample}")
    if remove_stripes is not None:
        check_size(remove_stripes)
    cfg = read_config(os.path.join(data, "config.txt"), proj_subsample, object_scale)
    angles = scan_angles(cfg)
    paths = sorted(glob.glob(os.path.join(data, "*.mat")))
    if not paths:
        raise ValueError(f"{data}: no .mat files")
    if len(angles) != len(paths) or cfg["n_proj"] != len(paths):
        raise ValueError(f"{data}: {len(paths)} .mat files, but config.txt gives {len(angles)} angles and "
                         f"NumberImages = {cfg['n_proj']}")
    train_ids, test_ids = split_ids(cfg["n_proj"], n_train, n_test)
    if not torch.cuda.is_available():
        raise RuntimeError("generate_real_data needs a CUDA device: the projections are prepared and reconstructed "
                           "on the GPU, with no CPU fallback")

    stack = prepare_files(paths, proj_subsample, proj_rescale, object_scale, chunk)
    if remove_stripes is not None:
        from .stripes import remove_stripes as _remove_stripes

        _remove_stripes(stack, check_size(remove_stripes, stack.shape[2]), out=stack)
    names = [os.path.basename(p).split(".")[0] for p in paths]
    splits = {"proj_train": set(int(i) for i in train_ids), "proj_test": set(test_ids)}
    frames = {"proj_train": [], "proj_test": []}
    for d in ("proj_all", *frames):
        os.makedirs(os.path.join(output, d), exist_ok=True)
    host = stack.cpu().numpy()
    for i, name in enumerate(names):
        np.save(os.path.join(output, "proj_all", name + ".npy"), host[i])
        for split, ids in splits.items():
            if i in ids:
                rel = os.path.join(split, name + ".npy")
                np.save(os.path.join(output, rel), host[i])
                frames[split].append({"file_path": rel, "angle": float(angles[i])})
                break

    nDetector = [int(host.shape[1]), int(host.shape[2])]
    nVoxel, sVoxel = [int(v) for v in nVoxel], [float(v) for v in sVoxel]
    offOrigin, offDetector = [float(v) for v in offOrigin], [float(v) for v in offDetector]
    scanner_cfg = {
        "mode": "cone",
        "DSD": cfg["DSD"],
        "DSO": cfg["DSO"],
        "nDetector": nDetector,
        "sDetector": (np.array(nDetector) * np.array(cfg["dDetector"])).tolist(),
        "nVoxel": nVoxel,
        "sVoxel": sVoxel,
        "offOrigin": offOrigin,
        "offDetector": offDetector,
        "accuracy": float(accuracy),
        "totalAngle": cfg["angle_last"] - cfg["angle_first"],
        "startAngle": cfg["angle_first"],
        "noise": True,
        "filter": None,
    }
    gt_path = os.path.join(output, "vol_gt.npy")
    if not os.path.exists(gt_path):
        np.save(gt_path, pseudo_ground_truth(stack, angles, scanner_cfg).cpu().numpy())
    bbox = np.array([np.array(offOrigin) - np.array(sVoxel) / 2, np.array(offOrigin) + np.array(sVoxel) / 2]).tolist()
    meta = {"scanner": scanner_cfg, "vol": "vol_gt.npy", "ct": "vol_gt.npy", "radius": 1.0, "bbox": bbox,
            "proj_train": frames["proj_train"], "proj_test": frames["proj_test"]}
    with open(os.path.join(output, "meta_data.json"), "w", encoding="utf-8") as f:
        json.dump(meta, f, indent=4)
    print(f"Data saved in {output}")
    return output


def main(argv=None) -> str:
    ap = argparse.ArgumentParser(description="Build a scene from a processed real cone-beam scan")
    ap.add_argument("--data", required=True, type=str, help="Path to the processed scan (config.txt and *.mat).")
    ap.add_argument("--output", required=True, type=str, help="Path to output.")
    ap.add_argument("--proj_subsample", default=4, type=int, help="subsample projections pixels")
    ap.add_argument("--proj_rescale", default=400.0, type=float,
                    help="rescale projection values to fit density to around [0,1]")
    ap.add_argument("--object_scale", default=50, type=int,
                    help="Rescale the whole scene to similar scales as the synthetic data")
    ap.add_argument("--n_test", default=100, type=int, help="number of test")
    ap.add_argument("--n_train", default=75, type=int, help="number of train")
    ap.add_argument("--nVoxel", nargs="+", default=[256, 256, 256], type=int, help="voxel dimension")
    ap.add_argument("--sVoxel", nargs="+", default=[2.0, 2.0, 2.0], type=float, help="volume size")
    ap.add_argument("--offOrigin", nargs="+", default=[0.0, 0.0, 0.0], type=float, help="offOrigin")
    ap.add_argument("--offDetector", nargs="+", default=[0.0, 0.0], type=float, help="offDetector")
    ap.add_argument("--accuracy", default=0.5, type=float, help="accuracy")
    ap.add_argument("--remove_stripes", default=None, type=int, metavar="K",
                    help="remove ring artifacts from all views before writing them: sorting-based stripe removal with "
                         "a median window of K detector columns (odd, 1 to 255; off by default)")
    a = ap.parse_args(argv)
    return generate(a.data, a.output, a.proj_subsample, a.proj_rescale, a.object_scale, a.n_test, a.n_train,
                    a.nVoxel, a.sVoxel, a.offOrigin, a.offDetector, a.accuracy, remove_stripes=a.remove_stripes)


if __name__ == "__main__":
    main()
