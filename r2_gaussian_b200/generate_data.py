"""Synthetic CT scene from a volume -- the reference's `data_generator/synthetic_dataset/generate_data.py`.

    python -m r2_gaussian_b200.generate_data --vol X.npy --scanner cone_beam.yml --output DIR
        [--n_train 50] [--n_test 100] [--seed 0] [--use_offDetector] [--helical_travel Z | --view_geometry FILE.json]

Reads the scanner configuration (the reference's yml format), projects the volume on the GPU with
`projector.project` (the reference uses TIGRE's `Ax`) at the train angles linspace(0, totalAngle, n_train + 1)[:-1]
+ startAngle and at n_test sorted random test angles over the full circle + startAngle, adds noise to the train views if
the configuration asks for it, and writes `<output>/<volume name>_<mode>/` (`meta_data.json`, `proj_train/`,
`proj_test/`, `vol_gt.npy`) with the reference's file names and the yml's own units.

Differences from the reference: the noise and the test angles come from one `numpy.random.RandomState(--seed)`, drawn
in the reference's order (train noise first, then test angles), where the reference uses numpy's unseeded global
generator; the projector is defined by render()'s geometry, not bit-identical to TIGRE's.  A scanner whose
`offDetector` is not zero is refused unless `--use_offDetector` is given, which projects through the offset detector
(`projector.project(..., use_offDetector=True)`, TIGRE's `geo.offDetector`; the convention is
`scene.detector_shift`'s).  The reference's real-data generator takes the same offset on its command line; here it is
the scanner file's `offDetector` ([u, v], in the file's units), written unchanged into `meta_data.json`, so the scene
is then reconstructed and trained with the same switch.

Per-view geometry (`scene.view_scanner`; the scene is then used with `--use_view_geometry`):
  * `--helical_travel Z` moves the volume along the rotation axis during the train arc, a helical scan:
    offOrigin_z(beta) = offOrigin_z + Z ((beta - startAngle) / totalAngle - 1/2), in the scanner file's units, with
    totalAngle free to exceed 360 (several turns).  The test angles are drawn over the same arc, and every frame is
    written with its `offOrigin`.
  * `--view_geometry FILE.json` takes any other table, e.g. a calibration: {"train": [...], "test": [...]} with one
    dict per view of `scene.VIEW_KEYS` overrides (DSO, DSD, offOrigin [x, y, z], offDetector [u, v]; file units).
    Each list must hold --n_train / --n_test entries.  The frames are written with their overrides.
Either projects through the per-view table (`projector.project(..., view_geometry=...)`), which implies
`--use_offDetector`.
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


def helical_offsets(cfg: dict, angles, travel: float) -> list[dict]:
    """{"offOrigin": [x, y, z]} per angle (radians) of a helical scan: the scanner's offOrigin with z moved by
    travel ((beta - startAngle) / totalAngle - 1/2), beta the angle in degrees."""
    off = [float(v) for v in cfg.get("offOrigin", [0.0, 0.0, 0.0])]
    frac = (np.degrees(np.asarray(angles, np.float64)) - float(cfg["startAngle"])) / float(cfg["totalAngle"]) - 0.5
    return [{"offOrigin": [off[0], off[1], off[2] + float(travel) * float(f)]} for f in frac]


def draw_arc_angles(cfg: dict, n_test: int, rng: np.random.RandomState) -> np.ndarray:
    """n_test sorted random angles (radians) over the train arc [startAngle, startAngle + totalAngle)."""
    return np.sort(rng.rand(n_test) * (cfg["totalAngle"] / 180 * np.pi)) + cfg["startAngle"] / 180 * np.pi


def read_view_geometry(path: str, n_train: int, n_test: int) -> dict:
    """The {"train": [...], "test": [...]} override file of --view_geometry, after the refusals."""
    import json

    from .scene import VIEW_KEYS

    with open(path) as f:
        table = json.load(f)
    if not isinstance(table, dict) or set(table) != {"train", "test"}:
        raise SystemExit(f"--view_geometry {path}: expected an object with the keys 'train' and 'test'")
    for split, n in (("train", n_train), ("test", n_test)):
        rows = table[split]
        if not isinstance(rows, list) or len(rows) != n:
            raise SystemExit(f"--view_geometry {path}: {split} holds {len(rows) if isinstance(rows, list) else '?'} "
                             f"entries, --n_{split} is {n}")
        for i, row in enumerate(rows):
            unknown = sorted(set(row) - set(VIEW_KEYS)) if isinstance(row, dict) else ["(not an object)"]
            if unknown:
                raise SystemExit(f"--view_geometry {path}: {split}[{i}] has unknown keys {unknown} "
                                 f"(supported: {', '.join(VIEW_KEYS)})")
            for k, size in (("offOrigin", 3), ("offDetector", 2)):
                if k in row and np.asarray(row[k]).shape != (size,):
                    raise SystemExit(f"--view_geometry {path}: {split}[{i}].{k} must hold {size} numbers")
    return table


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
    ap.add_argument("--use_offDetector", default=False, action="store_true",
                    help="Project through the scanner's offDetector (else a non-zero offDetector is refused).")
    ap.add_argument("--helical_travel", default=None, type=float,
                    help="Move the volume this far along z (scanner units) over the train arc: a helical scan.")
    ap.add_argument("--view_geometry", default=None, type=str,
                    help="JSON file {\"train\": [...], \"test\": [...]} of per-view DSO, DSD, offOrigin, offDetector.")
    a = ap.parse_args(argv)

    import torch
    import yaml

    from .dataset import frame_geometry, scale_scanner, write_blender
    from .projector import project

    with open(a.scanner) as f:
        cfg = yaml.safe_load(f)
    if a.helical_travel is not None and a.view_geometry is not None:
        raise SystemExit("--helical_travel and --view_geometry cannot be combined: give the helix in the file")
    if a.helical_travel is not None and not np.isfinite(a.helical_travel):
        raise SystemExit(f"--helical_travel must be finite, got {a.helical_travel}")
    table = read_view_geometry(a.view_geometry, a.n_train, a.n_test) if a.view_geometry else None
    per_view = table is not None or a.helical_travel is not None
    off = [float(v) for v in cfg.get("offDetector", [0.0, 0.0])]
    if any(v != 0.0 for v in off) and not (a.use_offDetector or per_view):
        raise SystemExit(f"the scanner's offDetector is {off}: pass --use_offDetector to project through the offset "
                         "detector (and use it again to reconstruct and train on the scene)")
    if not torch.cuda.is_available():
        raise SystemExit("generate_data needs a CUDA device: the projector runs on the GPU and has no CPU fallback")
    if a.n_train < 1 or a.n_test < 1:
        raise SystemExit("--n_train and --n_test must be at least 1")
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
    rows = {"train": table["train"] if table else None, "test": table["test"] if table else None}
    if a.helical_travel is not None:
        rows["train"] = helical_offsets(cfg, angles_train, a.helical_travel)

    def views(split):   # the split's overrides in scene units (frame_geometry), or None: the scalar path
        return None if rows[split] is None else [frame_geometry(r, scene_scale) for r in rows[split]]

    projs_train = (project(dvol, angles_train, scaled, a.use_offDetector, views("train")) / scene_scale).cpu().numpy()
    if cfg.get("noise", False):
        projs_train = add_noise(projs_train, cfg["possion_noise"], cfg["gaussian_noise"], rng)
    if a.helical_travel is not None:
        angles_test = draw_arc_angles(cfg, a.n_test, rng)
        rows["test"] = helical_offsets(cfg, angles_test, a.helical_travel)
    else:
        angles_test = draw_test_angles(cfg, a.n_test, rng)
    projs_test = (project(dvol, angles_test, scaled, a.use_offDetector, views("test")) / scene_scale).cpu().numpy()

    def frames(angles, projs, split):
        if rows[split] is None:
            return list(zip(angles, projs))
        return list(zip(angles, projs, rows[split]))

    case_path = os.path.join(a.output, case_name)
    write_blender(case_path, cfg, frames(angles_train, projs_train, "train"), frames(angles_test, projs_test, "test"),
                  vol)
    print(f"Generate data for case {case_name} complete!")
    return case_path


if __name__ == "__main__":
    main()
