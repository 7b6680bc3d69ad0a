"""Float64 NumPy statement of FDK with the truncation pad, which `r2_gaussian_b200.fdk.fdk(pad=...)` runs on the GPU
(r2x_fdk_pad; the model is stated in include/r2x.h).

TEST INFRASTRUCTURE ONLY: imported by tests/, never by the product package.

Per detector row, after step 1 (the cosine weight and any Parker weight), with r[0 .. W-1] the weighted row and a pad
of L pixels (0 <= L <= W):

    e[i] = r[i]                                          0 <= i < W
    e[-k] = t_k r[k-1],  e[W-1+k] = t_k r[W-k]           k = 1 .. L,  t_k = (1 + cos(pi k / (L + 1))) / 2
    q[j] = (1 / D) sum_{i=-L}^{W-1+L} h[j-i] e[i]        0 <= j < W

with the taps h of tests/fdk_window_oracle.py and its isocentre pitch D.  Step 1 and the backprojection are the
existing oracles' (tests/fdk_window_oracle.py, tests/fdk_short_scan_oracle.py, oracle/fdk_oracle.py); with L = 0 this
module gives their results.
"""
from __future__ import annotations

import math

import numpy as np
from scipy.signal import fftconvolve

import fdk_short_scan_oracle as sso
import fdk_window_oracle as fwo
import offset_detector_oracle as oo
from oracle import fdk_oracle


def taper(L: int) -> np.ndarray:
    """t_1 .. t_L."""
    k = np.arange(1, L + 1, dtype=np.float64)
    return 0.5 * (1.0 + np.cos(math.pi * k / (L + 1)))


def extend(rows, L: int) -> np.ndarray:
    """e[-L .. W-1+L] of every row of `rows` [..., W]: the rows with their rolled-off mirrors on both sides."""
    r = np.asarray(rows, np.float64)
    W = r.shape[-1]
    if not 0 <= L <= W:
        raise ValueError(f"pad {L} outside [0, {W}]")
    t = taper(L)
    left = t[::-1] * r[..., :L][..., ::-1]            # e[-L] .. e[-1] = t_L r[L-1] .. t_1 r[0]
    right = t * r[..., W - L:][..., ::-1]             # e[W] .. e[W-1+L] = t_1 r[W-1] .. t_L r[W-L]
    return np.concatenate([left, r, right], axis=-1)


def weight_rows(projs, tan_fovx: float, tan_fovy: float, mode: int, t_u: float = 0.0, t_v: float = 0.0,
                weights=None) -> np.ndarray:
    """Step 1: the cosine weight (cone) at the ndc of a detector offset by (t_u, t_v) pixels, times `weights`."""
    p = np.asarray(projs, dtype=np.float64)
    N, H, W = p.shape
    ndx, ndy = oo.ndc(H, W, t_u, t_v)
    if mode == 1:
        p = p / np.sqrt(1.0 + (ndx * tan_fovx)[None, None, :] ** 2 + (ndy * tan_fovy)[None, :, None] ** 2)
    if weights is not None:
        p = p * weights
    return p


def filter_rows(rows, name: str, L: int, D: float) -> np.ndarray:
    """Step 2 on weighted rows [..., W]: the extension by L, the convolution with `name`'s taps, q[0 .. W-1] / D."""
    W = np.shape(rows)[-1]
    e = extend(rows, L)
    h = fwo.taps(name, np.arange(-(W - 1 + L), W + L))
    full = fftconvolve(e, np.broadcast_to(h, (1,) * (e.ndim - 1) + h.shape), mode="full", axes=-1)
    return full[..., W - 1 + 2 * L:2 * W - 1 + 2 * L] / D


def filter_projections(projs, name: str, L: int, tan_fovx: float, tan_fovy: float, mode: int, dso: float,
                       t_u: float = 0.0, t_v: float = 0.0, weights=None) -> np.ndarray:
    """Steps 1-2 with a pad of L pixels."""
    W = int(np.shape(projs)[2])
    p = weight_rows(projs, tan_fovx, tan_fovy, mode, t_u, t_v, weights)
    return filter_rows(p, name, L, fdk_oracle.ramp_pitch(W, tan_fovx, mode, dso))


def fdk_scene(projs, angles, scanner_cfg: dict, name: str = "ram_lak", L: int = 0, short_scan: bool = False,
              use_offDetector: bool = False) -> np.ndarray:
    """fdk(projs, angles, scanner_cfg, short_scan, use_offDetector, filter=name, pad=...) with a pad of L pixels,
    in float64."""
    from r2_gaussian_b200.fdk import short_scan_views
    from r2_gaussian_b200.scene import detector_shift, make_view

    t_u, t_v = detector_shift(scanner_cfg) if use_offDetector else (0.0, 0.0)
    views = [make_view(scanner_cfg, float(a), use_offDetector) for a in angles]
    v0, dso = views[0], float(scanner_cfg["DSO"])
    W = int(np.shape(projs)[2])
    weights, scale = None, 1.0
    if short_scan:
        vw, arc = short_scan_views(angles, v0.mode, v0.tanfovx)
        w = sso.parker_weights(vw[:, :1], sso.fan_angles(W, v0.tanfovx, v0.mode)[None, :], arc)
        weights, scale = (w * vw[:, 1:])[:, None, :], len(views) / math.pi
    q = filter_projections(projs, name, L, v0.tanfovx, v0.tanfovy, v0.mode, dso, t_u, t_v, weights)
    return scale * fdk_oracle.backproject(q, [v.viewmatrix for v in views], [v.projmatrix for v in views], v0.mode,
                                          dso, scanner_cfg["nVoxel"], scanner_cfg["sVoxel"], scanner_cfg["offOrigin"])


def field_of_view(scanner_cfg: dict, angles, use_offDetector: bool = False) -> np.ndarray:
    """Bool [nx, ny, nz]: the voxels whose centre every view projects onto the detector (pixel coordinates in
    (-0.5, W - 0.5) x (-0.5, H - 0.5), the rasterizer's ndc -> pixel mapping)."""
    from r2_gaussian_b200.scene import make_view

    nx, ny, nz = (int(v) for v in scanner_cfg["nVoxel"])
    H, W = (int(v) for v in scanner_cfg["nDetector"])
    s = np.asarray(scanner_cfg["sVoxel"], np.float64)
    c = np.asarray(scanner_cfg["offOrigin"], np.float64)
    axes = [c[i] - 0.5 * s[i] + (np.arange(n) + 0.5) * s[i] / n for i, n in enumerate((nx, ny, nz))]
    X, Y, Z = np.meshgrid(*axes, indexing="ij")
    pts = np.stack([X.ravel(), Y.ravel(), Z.ravel(), np.ones(X.size)], 1)
    inside = np.ones(X.size, bool)
    for a in angles:
        pm = np.asarray(make_view(scanner_cfg, float(a), use_offDetector).projmatrix, np.float64).reshape(4, 4)
        hom = pts @ pm                                       # row vector times the column-major matrix
        px = (hom[:, 0] / hom[:, 3]) * (0.5 * W) + 0.5 * (W - 1)
        py = (hom[:, 1] / hom[:, 3]) * (0.5 * H) + 0.5 * (H - 1)
        inside &= (hom[:, 3] > 0) & (px > -0.5) & (px < W - 0.5) & (py > -0.5) & (py < H - 0.5)
    return inside.reshape(nx, ny, nz)


def psnr_in(gt, pred, mask) -> float:
    """metrics.metric_vol's psnr_3d (pixel_max 1) over the voxels of `mask`."""
    d = np.asarray(gt, np.float64)[mask] - np.asarray(pred, np.float64)[mask]
    return float(10.0 * np.log10(1.0 / np.mean(d * d)))
