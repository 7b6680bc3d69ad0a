"""Float64 NumPy statement of the offset-detector projector, backprojector and FDK (with half-fan weights) that
`r2_gaussian_b200.projector` / `fdk` run on the GPU with `use_offDetector=True`.

TEST INFRASTRUCTURE ONLY: imported by tests/, never by the product package.

It builds on the centred statements (oracle/projector_oracle.py, tests/backproject_oracle.py, oracle/fdk_oracle.py),
which are unchanged; a shift of (0, 0) gives their results.  (t_u, t_v) = `scene.detector_shift(scanner_cfg)`.

1. Rays.  Pixel (row i, column j) takes the centred projector's ray at ndc ((2j+1)/W - 1 + 2 t_u/W,
   (2i+1)/H - 1 - 2 t_v/H): the centred detector's fractional pixel (i - t_v, j + t_u).
2. Projection and its transpose: the centred oracle's integral and np.add.at over those rays.
3. FDK.  Cosine weight (cone) at the offset ndc; optional half-fan weight w(a_j) with a_j = ndc_x(j) * (tan_fovx or 1),
   delta = (1 - 2|t_u|/W) * (tan_fovx or 1), sigma = sign(t_u), w = 2 sin^2(pi/4 (1 + sigma a / delta)) for
   |a| <= delta, 2 for sigma a > delta; the centred ramp filter; the centred backprojection through the offset
   matrices (`scene.make_view(..., use_offDetector=True)`), scale pi / N.
"""
from __future__ import annotations

import math

import numpy as np
from scipy.signal import fftconvolve

import backproject_oracle as bo
from oracle import fdk_oracle
from oracle import projector_oracle as po


def ndc(H: int, W: int, t_u: float = 0.0, t_v: float = 0.0):
    """(ndc_x [W], ndc_y [H]) of the pixel centres of a detector offset by (t_u, t_v) pixels."""
    return ((2.0 * np.arange(W) + 1.0) / W - 1.0 + 2.0 * t_u / W,
            (2.0 * np.arange(H) + 1.0) / H - 1.0 - 2.0 * t_v / H)


def rays(view, t_u: float = 0.0, t_v: float = 0.0):
    """po.rays of a `scene.View` whose detector is offset by (t_u, t_v) pixels."""
    H, W = view.image_height, view.image_width
    ndx, ndy = ndc(H, W, t_u, t_v)
    c2w = np.linalg.inv(view.viewmatrix.astype(np.float64).T)
    if view.mode == 1:
        d = np.stack(np.broadcast_arrays(ndx[None, :] * view.tanfovx, ndy[:, None] * view.tanfovy, 1.0), -1)
        o = np.broadcast_to(c2w[:3, 3], d.shape)
    else:
        d = np.broadcast_to(np.array([0.0, 0.0, 1.0]), (H, W, 3))
        o = np.stack(np.broadcast_arrays(ndx[None, :], ndy[:, None], 0.0), -1) @ c2w[:3, :3].T + c2w[:3, 3]
    d = d @ c2w[:3, :3].T
    return np.ascontiguousarray(o), d / np.linalg.norm(d, axis=-1, keepdims=True)


def project_scene(volume, angles, scanner_cfg: dict) -> np.ndarray:
    """project(volume, angles, scanner_cfg, use_offDetector=True) in float64: [N, H, W]."""
    from r2_gaussian_b200.scene import detector_shift, make_view

    t_u, t_v = detector_shift(scanner_cfg)
    step = po.step_length(scanner_cfg)
    out = []
    for a in angles:
        view = make_view(scanner_cfg, float(a))
        o, d = rays(view, t_u, t_v)
        out.append(po.project_rays(volume, o, d, view.mode == 1, scanner_cfg["sVoxel"], scanner_cfg["offOrigin"], step))
    return np.stack(out)


def backproject_scene(projs, angles, scanner_cfg: dict) -> np.ndarray:
    """The exact transpose of `project_scene`: [nx, ny, nz] float64."""
    from r2_gaussian_b200.scene import detector_shift, make_view

    t_u, t_v = detector_shift(scanner_cfg)
    step = po.step_length(scanner_cfg)
    shape = tuple(int(v) for v in scanner_cfg["nVoxel"])
    out = np.zeros(shape)
    for v, a in enumerate(angles):
        view = make_view(scanner_cfg, float(a))
        o, d = rays(view, t_u, t_v)
        out += bo.backproject_rays(projs[v], o, d, view.mode == 1, shape, scanner_cfg["sVoxel"],
                                   scanner_cfg["offOrigin"], step)
    return out


def half_fan_weight(a, t_u: float, W: int, fan: float):
    """Wang's weight w(a) of the fan coordinate a (see the module docstring)."""
    delta = (1.0 - 2.0 * abs(t_u) / W) * fan
    x = math.copysign(1.0, t_u) * np.asarray(a, np.float64) / delta
    return np.where(x >= 1.0, 2.0, np.where(x <= -1.0, 0.0, 2.0 * np.sin(0.25 * math.pi * (1.0 + x)) ** 2))


def filter_projections(projs, tan_fovx: float, tan_fovy: float, mode: int, dso: float, t_u: float, t_v: float,
                       half_fan: bool = False) -> np.ndarray:
    p = np.asarray(projs, dtype=np.float64)
    N, H, W = p.shape
    ndx, ndy = ndc(H, W, t_u, t_v)
    if mode == 1:
        a, b = ndx * tan_fovx, ndy * tan_fovy
        p = p / np.sqrt(1.0 + a[None, None, :] ** 2 + b[None, :, None] ** 2)
    if half_fan:
        p = p * half_fan_weight(ndx * (tan_fovx if mode == 1 else 1.0), t_u, W, tan_fovx if mode == 1 else 1.0)
    D = fdk_oracle.ramp_pitch(W, tan_fovx, mode, dso)
    k = np.arange(-(W - 1), W).astype(np.float64)
    odd = np.abs(k) % 2 == 1
    h = np.zeros(2 * W - 1)
    h[odd] = -1.0 / (math.pi ** 2 * k[odd] ** 2 * D * D)
    h[W - 1] = 1.0 / (4.0 * D * D)
    return fftconvolve(p, h[None, None, :], mode="full", axes=2)[..., W - 1:2 * W - 1] * D


def fdk_scene(projs, angles, scanner_cfg: dict, half_fan: bool = False) -> np.ndarray:
    """fdk(projs, angles, scanner_cfg, use_offDetector=True, half_fan=half_fan) in float64."""
    from r2_gaussian_b200.scene import detector_shift, make_view

    t_u, t_v = detector_shift(scanner_cfg)
    views = [make_view(scanner_cfg, float(a), use_offDetector=True) for a in angles]
    v0, dso = views[0], float(scanner_cfg["DSO"])
    q = filter_projections(projs, v0.tanfovx, v0.tanfovy, v0.mode, dso, t_u, t_v, half_fan)
    return fdk_oracle.backproject(q, [v.viewmatrix for v in views], [v.projmatrix for v in views], v0.mode, dso,
                                  scanner_cfg["nVoxel"], scanner_cfg["sVoxel"], scanner_cfg["offOrigin"])
