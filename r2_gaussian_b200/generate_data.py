"""Synthetic CT scene from a volume -- the reference's `data_generator/synthetic_dataset/generate_data.py`.

    python -m r2_gaussian_b200.generate_data --vol X.npy --scanner cone_beam.yml --output DIR
        [--n_train 50] [--n_test 100] [--seed 0]

Reads the scanner configuration (the reference's yml format), projects the volume on the GPU with
`projector.project` (the reference uses TIGRE's `Ax`) at the train angles linspace(0, totalAngle, n_train + 1)[:-1]
+ startAngle and at n_test sorted random test angles over the full circle + startAngle, adds noise to the train views if
the configuration asks for it, and writes `<output>/<volume name>_<mode>/` (`meta_data.json`, `proj_train/`,
`proj_test/`, `vol_gt.npy`) with the reference's file names and the yml's own units.

Differences from the reference: the noise and the test angles come from one `numpy.random.RandomState(--seed)`, drawn
in the reference's order (train noise first, then test angles), where the reference uses numpy's unseeded global
generator; the projector is defined by render()'s geometry, not bit-identical to TIGRE's; `offDetector` must be zero.
"""
from __future__ import annotations

import argparse
import copy
import os

import numpy as np


def add_noise(projs: np.ndarray, I0: float, gaussian, rng: np.random.RandomState) -> np.ndarray:
    """Poisson + Gaussian noise on a stack of line integrals, the model TIGRE's `CTnoise.add` implements, restated from
    TIGRE's published code (not checked against TIGRE, which is not part of this build):
    m = max over the whole stack, I = Poisson(I0 exp(-p / m)) + Normal(gaussian[0], gaussian[1]), I <= 0 -> 1e-6,
    p' = -log(I / I0) m.  Negative results are then clamped to 0, as the reference's generator does."""
    p = np.asarray(projs, np.float64)
    m = float(p.max())
    inten = rng.poisson(I0 * np.exp(-p / m)).astype(np.float64)
    inten = inten + rng.normal(float(gaussian[0]), float(gaussian[1]), p.shape)
    inten[inten <= 0] = 1e-6
    out = (-np.log(inten / I0) * m).astype(np.float32)
    out[out < 0.0] = 0.0
    return out


def train_angles(cfg: dict, n_train: int) -> np.ndarray:
    return (np.linspace(0, cfg["totalAngle"] / 180 * np.pi, n_train + 1)[:-1] + cfg["startAngle"] / 180 * np.pi)


def draw_test_angles(cfg: dict, n_test: int, rng: np.random.RandomState) -> np.ndarray:
    return np.sort(rng.rand(n_test) * 2.0 * np.pi) + cfg["startAngle"] / 180 * np.pi    # the full circle, always


def shift_projections(case_path: str, columns: int, empty: float = 1e-6) -> None:
    """Move every train and test projection of a generated case `columns` columns (> 0: towards larger column index,
    < 0: towards smaller), filling with zeros -- what a horizontal detector offset of -columns pixels does to the data
    (`detector.py` for the sign).  The columns that fall off must be empty: each view's are at most `empty` times its
    maximum (the projector leaves float32 round-off of ~1e-9 outside the object), else ValueError and nothing written."""
    import json

    k = int(columns)
    if k == 0:
        return
    with open(os.path.join(case_path, "meta_data.json")) as f:
        meta = json.load(f)
    paths = [os.path.join(case_path, fr["file_path"]) for split in ("proj_train", "proj_test") for fr in meta[split]]
    out = []
    for p in paths:
        a = np.load(p)
        if abs(k) >= a.shape[-1]:
            raise ValueError(f"shift_projections: {k} columns is not less than the detector width {a.shape[-1]}")
        lost = a[..., -k:] if k > 0 else a[..., :-k]
        if float(np.abs(lost).max()) > empty * float(np.abs(a).max()):
            raise ValueError(f"shift_projections: {p}: the {abs(k)} columns that would fall off are not empty")
        b = np.zeros_like(a)
        if k > 0:
            b[..., k:] = a[..., :-k]
        else:
            b[..., :k] = a[..., -k:]
        out.append((p, b))
    for p, b in out:
        np.save(p, b)


def main(argv=None) -> str:
    ap = argparse.ArgumentParser(description="Data generator parameters")
    ap.add_argument("--vol", required=True, type=str, help="Path to volume.")
    ap.add_argument("--scanner", required=True, type=str, help="Path to scanner configuration.")
    ap.add_argument("--output", required=True, type=str, help="Path to output.")
    ap.add_argument("--n_train", default=50, type=int, help="Number of projections for training.")
    ap.add_argument("--n_test", default=100, type=int, help="Number of projections for evaluation.")
    ap.add_argument("--seed", default=0, type=int, help="Seed of the noise and of the test angles.")
    a = ap.parse_args(argv)

    import torch
    import yaml

    from .dataset import scale_scanner, write_blender
    from .projector import project

    if not torch.cuda.is_available():
        raise SystemExit("generate_data needs a CUDA device: the projector runs on the GPU and has no CPU fallback")
    if a.n_train < 1 or a.n_test < 1:
        raise SystemExit("--n_train and --n_test must be at least 1")
    with open(a.scanner) as f:
        cfg = yaml.safe_load(f)
    vol_name = os.path.basename(a.vol)[:-4]
    case_name = f"{vol_name}_{cfg['mode']}"
    print(f"Generate data for case {case_name}")
    vol = np.load(a.vol).astype(np.float32)
    if tuple(vol.shape) != tuple(int(n) for n in cfg["nVoxel"]):
        raise SystemExit(f"volume {a.vol} has shape {tuple(vol.shape)}, the scanner's nVoxel is {list(cfg['nVoxel'])}")
    scaled = copy.deepcopy(cfg)
    scene_scale = scale_scanner(scaled)
    rng = np.random.RandomState(a.seed)

    dvol = torch.from_numpy(vol).cuda()
    angles_train = train_angles(cfg, a.n_train)
    projs_train = (project(dvol, angles_train, scaled) / scene_scale).cpu().numpy()
    if cfg.get("noise", False):
        projs_train = add_noise(projs_train, cfg["possion_noise"], cfg["gaussian_noise"], rng)
    angles_test = draw_test_angles(cfg, a.n_test, rng)
    projs_test = (project(dvol, angles_test, scaled) / scene_scale).cpu().numpy()

    case_path = os.path.join(a.output, case_name)
    write_blender(case_path, cfg, list(zip(angles_train, projs_train)), list(zip(angles_test, projs_test)), vol)
    print(f"Generate data for case {case_name} complete!")
    return case_path


if __name__ == "__main__":
    main()
