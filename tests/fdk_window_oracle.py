"""Float64 NumPy statement of FDK with a windowed ramp filter, which `r2_gaussian_b200.fdk.fdk(filter=...)` runs on the
GPU (r2x_fdk's filter field).

TEST INFRASTRUCTURE ONLY: imported by tests/, never by the product package.

The band-limited Ram-Lak taps of oracle/fdk_oracle.py, in units of 1/D, are the inverse DTFT of the ramp,
h[k] = (1 / 2 pi^2) int_0^pi w Wn(w) cos(w k) dw with Wn = 1.  A windowed filter keeps that definition and that
normalisation with TIGRE's window Wn at frequency scale 1 (the windows of MATLAB's iradon):

    name         Wn(w), w in [0, pi]     h[k]
    ram_lak      1                       1/4 at 0, -1 / (pi^2 k^2) at odd k, 0 at even k != 0
    shepp_logan  sin(w/2) / (w/2)        -2 / (pi^2 (4k^2 - 1))
    cosine       cos(w/2)                -(-1)^k / (pi (4k^2 - 1)) - (1/(2k+1)^2 + 1/(2k-1)^2) / pi^2
    hamming      0.54 + 0.46 cos w       0.54 h_RL[k] + 0.23 (h_RL[k-1] + h_RL[k+1])
    hann         (1 + cos w) / 2         0.5 h_RL[k] + 0.25 (h_RL[k-1] + h_RL[k+1])

The filter is the linear convolution of each weighted row with h over the whole row (0 beyond it), divided by the
isocentre pitch D.  Everything else is the unwindowed FDK's: the cosine weight at the (offset) ndc, the redundancy
weights applied per pixel before the filter (Parker's of tests/fdk_short_scan_oracle.py, scale 1 instead of pi / N;
Wang's half-fan weights of tests/offset_detector_oracle.py), the pitch, and oracle/fdk_oracle.py's backprojection.
With "ram_lak" this module gives those three oracles' results.
"""
from __future__ import annotations

import math

import numpy as np
from scipy.signal import fftconvolve

import fdk_short_scan_oracle as sso
import offset_detector_oracle as oo
from oracle import fdk_oracle

FILTERS = ("ram_lak", "shepp_logan", "cosine", "hamming", "hann")

# Wn(w) of each filter, for the integral definition
WINDOWS = {
    "ram_lak": lambda w: np.ones_like(w),
    "shepp_logan": lambda w: np.sinc(w / (2.0 * math.pi)),           # np.sinc(x) = sin(pi x) / (pi x)
    "cosine": lambda w: np.cos(w / 2.0),
    "hamming": lambda w: 0.54 + 0.46 * np.cos(w),
    "hann": lambda w: 0.5 * (1.0 + np.cos(w)),
}


def ram_lak_taps(k) -> np.ndarray:
    k = np.abs(np.asarray(k, np.int64))
    odd = k % 2 == 1
    return np.where(k == 0, 0.25, np.where(odd, -1.0 / (math.pi ** 2 * np.maximum(k, 1).astype(float) ** 2), 0.0))


def taps(name: str, k) -> np.ndarray:
    """h[k] in units of 1/D (the closed forms of the table above) at integer offsets `k` (any sign)."""
    k = np.abs(np.asarray(k, np.int64))
    kf = k.astype(np.float64)
    if name == "ram_lak":
        return ram_lak_taps(k)
    if name == "shepp_logan":
        return -2.0 / (math.pi ** 2 * (4.0 * kf ** 2 - 1.0))
    if name == "cosine":
        sign = np.where(k % 2 == 0, 1.0, -1.0)
        return -sign / (math.pi * (4.0 * kf ** 2 - 1.0)) - (1.0 / (2 * kf + 1) ** 2 + 1.0 / (2 * kf - 1) ** 2) / math.pi ** 2
    if name in ("hamming", "hann"):
        c0, c1 = (0.54, 0.23) if name == "hamming" else (0.5, 0.25)
        return c0 * ram_lak_taps(k) + c1 * (ram_lak_taps(k - 1) + ram_lak_taps(k + 1))
    raise ValueError(f"unknown filter {name!r}")


def filter_projections(projs, name: str, tan_fovx: float, tan_fovy: float, mode: int, dso: float, t_u: float = 0.0,
                       t_v: float = 0.0, weights=None) -> np.ndarray:
    """Steps 1-2: cosine weight (cone) at the ndc of a detector offset by (t_u, t_v) pixels, times `weights` (the
    redundancy weights, broadcast against [N, H, W]; None for none), then the filter `name` along each row."""
    p = np.asarray(projs, dtype=np.float64)
    N, H, W = p.shape
    ndx, ndy = oo.ndc(H, W, t_u, t_v)
    if mode == 1:
        p = p / np.sqrt(1.0 + (ndx * tan_fovx)[None, None, :] ** 2 + (ndy * tan_fovy)[None, :, None] ** 2)
    if weights is not None:
        p = p * weights
    h = taps(name, np.arange(-(W - 1), W))
    D = fdk_oracle.ramp_pitch(W, tan_fovx, mode, dso)
    return fftconvolve(p, h[None, None, :], mode="full", axes=2)[..., W - 1:2 * W - 1] / D


def fdk_scene(projs, angles, scanner_cfg: dict, name: str = "ram_lak", short_scan: bool = False,
              use_offDetector: bool = False, half_fan: bool = False) -> np.ndarray:
    """fdk(projs, angles, scanner_cfg, short_scan, use_offDetector, half_fan, filter=name) in float64."""
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
    if half_fan:
        fan = v0.tanfovx if v0.mode == 1 else 1.0
        weights = oo.half_fan_weight(oo.ndc(1, W, t_u, t_v)[0] * fan, t_u, W, fan)
    q = filter_projections(projs, name, v0.tanfovx, v0.tanfovy, v0.mode, dso, t_u, t_v, weights)
    return scale * fdk_oracle.backproject(q, [v.viewmatrix for v in views], [v.projmatrix for v in views], v0.mode,
                                          dso, scanner_cfg["nVoxel"], scanner_cfg["sVoxel"], scanner_cfg["offOrigin"])
