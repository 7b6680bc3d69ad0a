"""Float64 NumPy statement of the FDK reconstruction that `r2_gaussian_b200.fdk` runs on the GPU.

TEST INFRASTRUCTURE ONLY: imported by tests/, never by the product package.

All lengths are in the scene-scaled units of `dataset.read_scene` (volume of interest [-1,1]^3, projections already
multiplied by scene_scale).  projs[N,H,W] holds N views of H rows (v) by W columns (u); viewmatrices / projmatrices are
the rasterizer's per-view matrices (`scene.make_view`: 16 floats, column-major flat).

1. Cosine weight (cone only): P'(u,v) = P(u,v) * DSD / sqrt(DSD^2 + u^2 + v^2) at the pixel centres; with
   u / DSD = ndc_x * tan_fovx this is 1 / sqrt(1 + (ndc_x tan_fovx)^2 + (ndc_y tan_fovy)^2).
2. Ramp filter along each row: band-limited Ram-Lak taps at the isocentre pitch D (cone: dDetector_u * DSO / DSD =
   2 tan_fovx DSO / W; parallel: the rasterizer's parallel detector spans ndc [-1,1] = scene [-1,1], so D = 2 / W),
   h[0] = 1/(4 D^2), h[k odd] = -1/(pi^2 k^2 D^2), h[k even != 0] = 0, linear (zero-padded) convolution over the whole
   row, times D.
3. Voxel-driven backprojection: voxel centres center - s/2 + (i + 1/2) d per axis, projected with the same matrices and
   ndc -> pixel mapping as the rasterizer, bilinear sample of the filtered view (0 outside the detector), cone
   magnification U = DSO / z_view (0 where z_view <= 0; parallel U = 1), vol = (pi / N) sum_i U_i^2 Q_i(px_i, py_i).
   Cone-beam short scans get no Parker weights.
"""
from __future__ import annotations

import math

import numpy as np
from scipy.signal import fftconvolve


def ramp_pitch(W: int, tan_fovx: float, mode: int, dso: float) -> float:
    return 2.0 * tan_fovx * dso / W if mode == 1 else 2.0 / W


def filter_projections(projs, tan_fovx: float, tan_fovy: float, mode: int, dso: float) -> np.ndarray:
    p = np.asarray(projs, dtype=np.float64)
    N, H, W = p.shape
    if mode == 1:
        a = ((2.0 * np.arange(W) + 1.0) / W - 1.0) * tan_fovx
        b = ((2.0 * np.arange(H) + 1.0) / H - 1.0) * tan_fovy
        p = p / np.sqrt(1.0 + a[None, None, :] ** 2 + b[None, :, None] ** 2)
    D = ramp_pitch(W, tan_fovx, mode, dso)
    k = np.arange(-(W - 1), W).astype(np.float64)
    odd = np.abs(k) % 2 == 1
    h = np.zeros(2 * W - 1)
    h[odd] = -1.0 / (math.pi ** 2 * k[odd] ** 2 * D * D)
    h[W - 1] = 1.0 / (4.0 * D * D)
    q = fftconvolve(p, h[None, None, :], mode="full", axes=2)[..., W - 1:2 * W - 1]
    return q * D


def voxel_centres(nVoxel, sVoxel, center):
    return [np.asarray(center[a], np.float64) - sVoxel[a] / 2.0 + (np.arange(nVoxel[a]) + 0.5) * (sVoxel[a] / nVoxel[a])
            for a in range(3)]


def _row(m, r, X, Y, Z):
    return m[r] * X + m[4 + r] * Y + m[8 + r] * Z + m[12 + r]


def backproject(q, viewmatrices, projmatrices, mode: int, dso: float, nVoxel, sVoxel, center) -> np.ndarray:
    q = np.asarray(q, dtype=np.float64)
    N, H, W = q.shape
    xs, ys, zs = voxel_centres(nVoxel, sVoxel, center)
    X, Y, Z = np.meshgrid(xs, ys, zs, indexing="ij")
    vol = np.zeros(X.shape, np.float64)
    qp = np.pad(q, ((0, 0), (1, 1), (1, 1)))          # one zero pixel around the detector
    for i in range(N):
        vm = np.asarray(viewmatrices[i], np.float64).reshape(16)
        pm = np.asarray(projmatrices[i], np.float64).reshape(16)
        pw = 1.0 / (_row(pm, 3, X, Y, Z) + 1e-7)      # the rasterizer's homogeneous divide
        px = ((_row(pm, 0, X, Y, Z) * pw + 1.0) * W - 1.0) * 0.5
        py = ((_row(pm, 1, X, Y, Z) * pw + 1.0) * H - 1.0) * 0.5
        if mode == 1:
            zv = _row(vm, 2, X, Y, Z)
            ok = zv > 0
            U2 = np.where(ok, (dso / np.where(ok, zv, 1.0)) ** 2, 0.0)
        else:
            U2 = np.ones_like(X)
        x0, y0 = np.floor(px), np.floor(py)
        fx, fy = px - x0, py - y0
        inside = (x0 >= -1) & (x0 <= W - 1) & (y0 >= -1) & (y0 <= H - 1)
        xi = np.clip(x0, -1, W - 1).astype(np.int64) + 1
        yi = np.clip(y0, -1, H - 1).astype(np.int64) + 1
        qi = qp[i]
        s = ((1 - fy) * ((1 - fx) * qi[yi, xi] + fx * qi[yi, xi + 1]) +
             fy * ((1 - fx) * qi[yi + 1, xi] + fx * qi[yi + 1, xi + 1]))
        vol += np.where(inside, U2 * s, 0.0)
    return vol * (math.pi / N)


def fdk(projs, viewmatrices, projmatrices, tan_fovx, tan_fovy, mode, dso, nVoxel, sVoxel, center) -> np.ndarray:
    q = filter_projections(projs, tan_fovx, tan_fovy, mode, dso)
    return backproject(q, viewmatrices, projmatrices, mode, dso, nVoxel, sVoxel, center)


def fdk_scene(projs, angles, scanner_cfg: dict) -> np.ndarray:
    """The oracle on a scanner dict (as `read_scene` returns it) and one angle per view, geometry from scene.make_view."""
    from r2_gaussian_b200.scene import make_view

    views = [make_view(scanner_cfg, float(a)) for a in angles]
    v0 = views[0]
    return fdk(projs, [v.viewmatrix for v in views], [v.projmatrix for v in views], v0.tanfovx, v0.tanfovy, v0.mode,
               float(scanner_cfg["DSO"]), scanner_cfg["nVoxel"], scanner_cfg["sVoxel"], scanner_cfg["offOrigin"])
