"""Float64 oracles of the per-view geometry operators, composed one view at a time from the existing ones: each view is
the scalar oracle of `scene.view_scanner`'s scanner for that view (its own view matrix, FoV, detector offset and DSO),
and the backprojections and FDK volumes of the views are summed.  Also small scenes with per-view frames for the CPU
tests."""
from __future__ import annotations

import json
import math
import os

import numpy as np

import ct_edge_cases as ct
import offset_detector_oracle as oo
from oracle import fdk_oracle
from r2_gaussian_b200 import scene


def view_scanners(sc: dict, geometry) -> list[dict]:
    return [scene.view_scanner(sc, g or {}) for g in geometry]


def views(sc: dict, angles, geometry) -> list[scene.View]:
    return [scene.make_view(c, float(a), True) for c, a in zip(view_scanners(sc, geometry), angles)]


def project(volume, angles, sc: dict, geometry) -> np.ndarray:
    """[N, H, W]: view v is the offset-detector oracle of its own scanner."""
    out = [ct.project_views(volume, [v], sc, *scene.detector_shift(c))
           for v, c in zip(views(sc, angles, geometry), view_scanners(sc, geometry))]
    return np.concatenate(out)


def backproject(y, angles, sc: dict, geometry) -> np.ndarray:
    """The sum over views of each view's exact transpose."""
    y = np.asarray(y, np.float64)
    out = 0.0
    for i, (v, c) in enumerate(zip(views(sc, angles, geometry), view_scanners(sc, geometry))):
        out = out + ct.backproject_views(y[i:i + 1], [v], sc, *scene.detector_shift(c))
    return out


def filtered(projs, angles, sc: dict, geometry) -> np.ndarray:
    """[N, H, W]: each view through the offset oracle's filter with its own FoV, offset and DSO."""
    p = np.asarray(projs, np.float64)
    out = [oo.filter_projections(p[i:i + 1], v.tanfovx, v.tanfovy, v.mode, float(c["DSO"]), *scene.detector_shift(c))
           for i, (v, c) in enumerate(zip(views(sc, angles, geometry), view_scanners(sc, geometry)))]
    return np.concatenate(out)


def fdk(projs, angles, sc: dict, geometry) -> np.ndarray:
    """(pi / N) sum over views of each view's filtered backprojection with its own (DSO / z)^2 weight."""
    q = filtered(projs, angles, sc, geometry)
    vs, cs = views(sc, angles, geometry), view_scanners(sc, geometry)
    out = 0.0
    for i, (v, c) in enumerate(zip(vs, cs)):
        # fdk_oracle.backproject of one view scales by pi / 1
        out = out + fdk_oracle.backproject(q[i:i + 1], [v.viewmatrix], [v.projmatrix], v.mode, float(c["DSO"]),
                                           sc["nVoxel"], sc["sVoxel"], sc["offOrigin"])
    return out / len(vs)


def jittered(n: int, sc: dict, seed: int = 3, px: float = 2.0, rel: float = 0.02) -> list[dict]:
    """Per-view calibration overrides (scene units): offDetector_u within +-px pixels, DSO and DSD within +-rel."""
    rng = np.random.RandomState(seed)
    du = float(sc["sDetector"][1]) / float(sc["nDetector"][1])
    off = [float(v) for v in sc.get("offDetector", [0.0, 0.0])]
    return [{"DSO": float(sc["DSO"]) * (1.0 + rel * rng.uniform(-1, 1)),
             "DSD": float(sc["DSD"]) * (1.0 + rel * rng.uniform(-1, 1)),
             "offDetector": [off[0] + px * du * rng.uniform(-1, 1), off[1]]} for _ in range(n)]


def helix(n: int, sc: dict, travel: float) -> list[dict]:
    """offOrigin overrides moving the volume `travel` along z over n views (scene units)."""
    off = [float(v) for v in sc["offOrigin"]]
    return [{"offOrigin": [off[0], off[1], off[2] + travel * (i / n - 0.5)]} for i in range(n)]


def write_scene(path: str, scanner: dict, frames: list[tuple[float, dict]], n_test: int = 0,
                vol_shape=(4, 4, 4)) -> str:
    """A blender scene whose train frames are (angle, overrides); the projections are zeros of the detector's shape."""
    os.makedirs(os.path.join(path, "proj_train"), exist_ok=True)
    os.makedirs(os.path.join(path, "proj_test"), exist_ok=True)
    H, W = (int(v) for v in scanner["nDetector"])
    meta = {"scanner": scanner, "vol": "vol_gt.npy", "proj_train": [], "proj_test": []}
    np.save(os.path.join(path, "vol_gt.npy"), np.zeros(vol_shape, np.float32))
    for split, fr in (("train", frames), ("test", frames[:n_test])):
        for i, (angle, over) in enumerate(fr):
            rel = os.path.join(f"proj_{split}", f"{i:04d}.npy")
            np.save(os.path.join(path, rel), np.zeros((H, W), np.float32))
            meta[f"proj_{split}"].append({"file_path": rel, "angle": float(angle), **over})
    with open(os.path.join(path, "meta_data.json"), "w") as f:
        json.dump(meta, f)
    return path


def file_scanner(n_detector: int = 8, n_voxel: int = 4) -> dict:
    """A cone-beam scanner in file units (scene_scale 0.5)."""
    return {"mode": "cone", "DSD": 14.0, "DSO": 10.0, "nDetector": [n_detector, n_detector], "sDetector": [8.0, 8.0],
            "nVoxel": [n_voxel] * 3, "sVoxel": [4.0, 4.0, 4.0], "offOrigin": [0.0, 0.0, 0.0],
            "offDetector": [0.0, 0.0], "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0,
            "filter": None}


ANGLES = (0.0, 0.7, math.pi / 2, 2.5, 4.1)
