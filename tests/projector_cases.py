"""Shared inputs of the projector tests (tests/test_projector_cpu.py, tests/test_projector_gpu.py)."""
from __future__ import annotations

import math

import numpy as np

import fdk_cases as fc
from r2_gaussian_b200 import scene

# relative L2 of the oracle against exact chord lengths, ball of radius 0.5 sampled at the centres of a 64^3 grid
# (measured 0.028 cone, 0.021 parallel)
BALL_BOUND = 0.04
# relative L2 of project(voxel(cloud)) against raster(cloud) on ROUND_TRIP_VOX^3 / ROUND_TRIP_DET^2
# (measured 0.011 cone, 0.010 parallel with the oracle)
ROUND_TRIP_BOUND = 0.02
ROUND_TRIP_DET, ROUND_TRIP_VOX = 96, 48
ROUND_TRIP_ANGLES = (0.0, 0.9, math.pi / 2, 2.6, 4.4)


def ball_volume(n: int, radius: float = 0.5) -> np.ndarray:
    """Indicator of a centred ball sampled at the voxel centres of an n^3 grid over [-1, 1]^3."""
    x = (np.arange(n) + 0.5) * 2.0 / n - 1.0
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    return (X * X + Y * Y + Z * Z <= radius * radius).astype(np.float32)


def flipped_variants(vol: np.ndarray, angles):
    """(name, volume, angles) that a wrong axis order, orientation or angle sign would produce."""
    return [("flip x", vol[::-1], angles), ("flip y", vol[:, ::-1], angles), ("flip z", vol[:, :, ::-1], angles),
            ("transpose x y", vol.transpose(1, 0, 2), angles), ("negative angle", vol, [-a for a in angles])]


def raster_views(cloud: scene.Cloud, sc: dict, angles) -> np.ndarray:
    """The C rasterizer oracle's projections of a cloud."""
    from oracle import r2_oracle as orc

    out = []
    for a in angles:
        v = scene.make_view(sc, float(a))
        out.append(orc.raster_forward(cloud.means, cloud.scales, cloud.rotations, cloud.density, v.viewmatrix,
                                      v.projmatrix, v.image_width, v.image_height, v.tanfovx, v.tanfovy,
                                      v.mode)["image"])
    return np.stack(out)


rel_l2 = fc.rel_l2
