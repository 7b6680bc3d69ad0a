"""Shared inputs of the FDK tests (tests/test_fdk_cpu.py, tests/test_fdk_gpu.py): an analytic ball phantom and an
off-centre, anisotropic, randomly rotated Gaussian cloud whose projections and volume both come from the rasterizer /
voxelizer conventions."""
from __future__ import annotations

import math

import numpy as np

from r2_gaussian_b200 import scene

# (mode, views) -> bound on the relative L2 error of fdk(render(cloud)) against query(cloud) on the 48^3 grid
ROUND_TRIP_BOUNDS = {("cone", 180): 0.03, ("cone", 50): 0.07, ("parallel", 180): 0.06, ("parallel", 50): 0.08}
ROUND_TRIP_DET, ROUND_TRIP_VOX = 128, 48


def scanner(mode: str, n_detector: int, n_voxel: int) -> dict:
    sc = scene.cone_beam_scanner(n_detector, n_voxel) if mode == "cone" else scene.parallel_beam_scanner(n_detector, n_voxel)
    sc["dDetector"] = (np.asarray(sc["sDetector"], float) / np.asarray(sc["nDetector"], float)).tolist()
    sc["dVoxel"] = (np.asarray(sc["sVoxel"], float) / np.asarray(sc["nVoxel"], float)).tolist()
    return sc


def full_scan(n_views: int) -> np.ndarray:
    return np.linspace(0.0, 2.0 * math.pi, n_views + 1)[:-1]


def ball_projections(sc: dict, angles, radius: float = 0.5) -> np.ndarray:
    """Exact chord lengths through a uniform ball of density 1 centred at the origin, per detector pixel centre."""
    out = []
    for a in angles:
        v = scene.make_view(sc, float(a))
        H, W = v.image_height, v.image_width
        nx = (2.0 * np.arange(W) + 1.0) / W - 1.0
        ny = (2.0 * np.arange(H) + 1.0) / H - 1.0
        c2w = np.linalg.inv(v.viewmatrix.astype(np.float64).T)           # viewmatrix is stored transposed
        if v.mode == scene.MODE_CONE:
            d = np.stack(np.broadcast_arrays(nx[None, :] * v.tanfovx, ny[:, None] * v.tanfovy, 1.0), -1)
            o = np.broadcast_to(c2w[:3, 3], d.shape)
        else:
            d = np.broadcast_to(np.array([0.0, 0.0, 1.0]), (H, W, 3))
            o = np.stack(np.broadcast_arrays(nx[None, :], ny[:, None], 0.0), -1)
            o = o @ c2w[:3, :3].T + c2w[:3, 3]
        d = d @ c2w[:3, :3].T
        d = d / np.linalg.norm(d, axis=-1, keepdims=True)
        t = -(o * d).sum(-1)
        dist2 = ((o + t[..., None] * d) ** 2).sum(-1)
        out.append(2.0 * np.sqrt(np.maximum(radius * radius - dist2, 0.0)))
    return np.asarray(out, np.float32)


def round_trip_cloud(seed: int = 7, P: int = 60) -> scene.Cloud:
    """Anisotropic, randomly rotated Gaussians around an off-centre point, all well inside the volume of interest."""
    rng = np.random.RandomState(seed)
    centre = np.array([0.22, -0.12, 0.18])
    means = (centre + rng.uniform(-0.38, 0.38, size=(P, 3))).astype(np.float32)
    scales = rng.uniform(0.05, 0.14, size=(P, 3)).astype(np.float32)
    q = rng.randn(P, 4)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    dens = rng.uniform(0.4, 1.2, size=(P, 1)).astype(np.float32)
    return scene.Cloud(means, scales, q.astype(np.float32), dens, {"kind": "fdk-round-trip", "seed": seed})


def rel_l2(a, b) -> float:
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))
