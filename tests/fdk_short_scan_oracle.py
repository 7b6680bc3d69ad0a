"""Float64 NumPy statement of the short-scan FDK that `r2_gaussian_b200.fdk.fdk(short_scan=True)` runs on the GPU
(Parker 1982, in the overscan form of Silver 2000).  It reuses the plain FDK's filter and backprojection from
oracle/fdk_oracle.py, whose (pi / N) scale assumes every ray is measured twice (a full scan, or a 180-degree parallel
scan) and so reconstructs a cone-beam short scan as if it were a full one.

TEST INFRASTRUCTURE ONLY: imported by tests/, never by the product package.

Inputs are the views' angles theta_v (radians, any order) and the fan angle of detector column j:
gamma_j = -atan(ndc_x(j) tan_fovx) for cone beam, with ndc_x(j) = (2j + 1)/W - 1, and 0 for parallel beam.  The sign:
make_view puts the source at (DSO cos t, DSO sin t, 0) and the detector's u axis along (-sin t, cos t, 0), the direction
of rotation, so the ray through u leaves the source at angle t + pi - atan(u / DSD); with gamma signed as above, the
conjugate of ray (beta, gamma) is (beta + pi + 2 gamma, -gamma).
  a. Arc: reduce theta_v mod 2 pi and sort; the largest circular gap between neighbours marks the start theta_start of
     the scan.  beta_v = (theta_v - theta_start) mod 2 pi, D = max(beta) / (N - 1); each view stands for an interval of
     width D around it, so beta'_v = beta_v + D/2 and the arc is B = max(beta) + D (linspace(0, R, n + 1)[:-1]: B = R).
  b. Intervals: dbeta_v runs between the midpoints of the sorted beta' (0 and B at the ends); views at the same angle
     share their interval equally.
  c. Parker weights with delta = (B - pi)/2: w = sin^2(pi/4 beta' / (delta - gamma)) for 0 <= beta' < 2(delta - gamma),
     1 up to pi - 2 gamma, sin^2(pi/4 (pi + 2 delta - beta') / (delta + gamma)) up to pi + 2 delta = B, 0 beyond.
     A ray and its conjugate have weights summing to 1.
  d. P' = w(beta'_v, gamma_j) dbeta_v P before the cosine weight, then the plain FDK's filter unchanged, then its
     backprojection with scale 1 instead of pi / N.  With w = 1/2 and dbeta = 2 pi / N this is the plain FDK.
It needs pi + 2 atan(tan_fovx) <= B < 2 pi (cone; pi <= B < 2 pi parallel) and N >= 2; `r2_gaussian_b200.fdk`
refuses anything else.  Steps a-b are `r2_gaussian_b200.fdk.short_scan_views`, which this oracle calls; the tests pin
them against hand-derived cases.
"""
from __future__ import annotations

import math

import numpy as np

from oracle.fdk_oracle import backproject, filter_projections


def fan_angles(W: int, tan_fovx: float, mode: int) -> np.ndarray:
    """gamma_j: -atan(ndc_x(j) tan_fovx) for cone beam, 0 for parallel beam."""
    if mode != 1:
        return np.zeros(W)
    return -np.arctan(((2.0 * np.arange(W) + 1.0) / W - 1.0) * tan_fovx)


def parker_weights(beta, gamma, arc: float) -> np.ndarray:
    """Step c: w(beta', gamma) for every pair of the broadcast shapes of `beta` and `gamma`."""
    beta, gamma = np.broadcast_arrays(np.asarray(beta, np.float64), np.asarray(gamma, np.float64))
    delta = 0.5 * (arc - math.pi)
    lo, hi = delta - gamma, delta + gamma
    rise = beta < 2.0 * lo
    fall = ~rise & (beta >= math.pi - 2.0 * gamma) & (beta < arc)
    w = np.where(beta < math.pi - 2.0 * gamma, 1.0, 0.0)
    w = np.where(rise, np.sin(0.25 * math.pi * beta / np.where(rise, lo, 1.0)) ** 2, w)
    return np.where(fall, np.sin(0.25 * math.pi * (arc - beta) / np.where(fall, hi, 1.0)) ** 2, w)


def fdk_short_scan_scene(projs, angles, scanner_cfg: dict) -> np.ndarray:
    """The short-scan FDK (steps a-d) on a scanner dict and one angle per view, geometry from scene.make_view."""
    from r2_gaussian_b200.fdk import short_scan_views
    from r2_gaussian_b200.scene import make_view

    views = [make_view(scanner_cfg, float(a)) for a in angles]
    v0 = views[0]
    p = np.asarray(projs, np.float64)
    vw, arc = short_scan_views(angles, v0.mode, v0.tanfovx)
    w = parker_weights(vw[:, :1], fan_angles(p.shape[2], v0.tanfovx, v0.mode)[None, :], arc)      # [N, W]
    p = p * (w * vw[:, 1:])[:, None, :]
    dso = float(scanner_cfg["DSO"])
    q = filter_projections(p, v0.tanfovx, v0.tanfovy, v0.mode, dso)
    vol = backproject(q, [v.viewmatrix for v in views], [v.projmatrix for v in views], v0.mode, dso,
                      scanner_cfg["nVoxel"], scanner_cfg["sVoxel"], scanner_cfg["offOrigin"])
    return vol * (len(views) / math.pi)                                              # scale 1 instead of pi / N
