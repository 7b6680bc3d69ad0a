"""A float64 numpy statement of the scene view's ellipsoid kind (include/r2x.h, "ellipsoid"), operation for operation:
the pixel box, the ray-quadric hit and the depth give the kernel's keys bit for bit, and the shading its colours.  The
other kinds go through tests/scene_view_oracle.py, so lists that mix ellipsoids with triangles and lines can be
checked.  numpy's element-wise float64 operations round once each, as the kernel's explicit round-to-nearest
intrinsics do; every expression below keeps the header's order.

    keys, rgb = raster(pos, meta, attr, tex, lut, cams, H, W, parallel, near, background, window=None)

`window=(y0, y1, x0, x1)` restricts the work to those rows and columns (exclusive ends), as in scene_view_oracle.
"""
from __future__ import annotations

import numpy as np

import scene_view_oracle as so

ELLIPSOID = 4


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def rotation(q):
    """build_rotation's matrix of quaternions (w, x, y, z) float32 [n, 4], normalised in float64: [n, 3, 3]."""
    q = np.asarray(q, np.float32).reshape(-1, 4).astype(np.float64)
    w, x, y, z = q.T
    m = np.sqrt(((w * w + x * x) + y * y) + z * z)
    w, x, y, z = w / m, x / m, y / m, z / m
    R = np.empty((len(q), 3, 3))
    R[:, 0, 0] = 1.0 - 2.0 * (y * y + z * z)
    R[:, 0, 1] = 2.0 * (x * y - w * z)
    R[:, 0, 2] = 2.0 * (x * z + w * y)
    R[:, 1, 0] = 2.0 * (x * y + w * z)
    R[:, 1, 1] = 1.0 - 2.0 * (x * x + z * z)
    R[:, 1, 2] = 2.0 * (y * z - w * x)
    R[:, 2, 0] = 2.0 * (x * z - w * y)
    R[:, 2, 1] = 2.0 * (y * z + w * x)
    R[:, 2, 2] = 1.0 - 2.0 * (x * x + y * y)
    return R


def _local(R, k, v):
    """diag(k) R^T v, element-wise over leading dimensions."""
    return np.stack([((R[..., 0, j] * v[..., 0] + R[..., 1, j] * v[..., 1]) + R[..., 2, j] * v[..., 2]) * k[..., j]
                     for j in range(3)], -1)


class Ellipsoids:
    """Centres c, semi-axes s, inverses k = 1 / s and rotations R of the ellipsoid rows."""

    def __init__(self, pos, attr):
        pos = np.asarray(pos, np.float64).reshape(-1, 3, 3)
        self.c, self.s = pos[:, 0].copy(), pos[:, 1].copy()
        self.k = 1.0 / self.s
        self.R = rotation(np.asarray(attr, np.float32).reshape(-1, 12)[:, 3:7])

    def take(self, i):
        out = Ellipsoids.__new__(Ellipsoids)
        out.c, out.s, out.k, out.R = self.c[i], self.s[i], self.k[i], self.R[i]
        return out


def boxes(k: so.Cam, near, E: Ellipsoids):
    """(x0, x1, y0, y1) int64 per ellipsoid, the clamped pixel box of the header (x0 > x1 or y0 > y1: nothing)."""
    d = E.c - np.asarray(k.P)
    cc = [_dot(d, np.asarray(v)) for v in (k.r, k.u, k.f)]
    rows = (k.r, k.u, k.f)
    M = np.empty((len(E.c), 3, 3))
    for i in range(3):
        for j in range(3):
            M[:, i, j] = ((rows[i][0] * E.R[:, 0, j] + rows[i][1] * E.R[:, 1, j]) + rows[i][2] * E.R[:, 2, j]) * E.s[:, j]
    S = lambda a, b: (M[:, a, 0] * M[:, b, 0] + M[:, a, 1] * M[:, b, 1]) + M[:, a, 2] * M[:, b, 2]
    W, H, p = k.W, k.H, k.p
    szz = S(2, 2)
    sz = np.sqrt(szz)
    nothing = (cc[2] + sz) < near
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if k.parallel:
            sx, sy = np.sqrt(S(0, 0)), np.sqrt(S(1, 1))
            lx, hx = 0.5 * W + (cc[0] - sx) / p, 0.5 * W + (cc[0] + sx) / p
            ly, hy = 0.5 * H - (cc[1] + sy) / p, 0.5 * H - (cc[1] - sy) / p
            whole = np.zeros(len(sz), bool)
        else:
            a2 = cc[2] * cc[2] - szz
            whole = ~((cc[2] - sz) >= near) | ~(a2 > 0.0)

            def tangent(cx, sxz, sxx):
                b1, c0 = cx * cc[2] - sxz, cx * cx - sxx
                dd = np.sqrt(np.fmax(b1 * b1 - a2 * c0, 0.0))
                return (b1 - dd) / a2, (b1 + dd) / a2

            lo, hi = tangent(cc[0], S(0, 2), S(0, 0))
            lx, hx = 0.5 * W + lo / p, 0.5 * W + hi / p
            lo, hi = tangent(cc[1], S(1, 2), S(1, 1))
            ly, hy = 0.5 * H - hi / p, 0.5 * H - lo / p
        x0 = np.fmin(np.fmax(np.floor(lx) - 1.0, 0.0), float(W))
        x1 = np.fmax(np.fmin(np.floor(hx) + 1.0, W - 1.0), -1.0)
        y0 = np.fmin(np.fmax(np.floor(ly) - 1.0, 0.0), float(H))
        y1 = np.fmax(np.fmin(np.floor(hy) + 1.0, H - 1.0), -1.0)
    box = np.stack([x0, x1, y0, y1], 1).astype(np.int64)
    box[whole] = (0, W - 1, 0, H - 1)
    box[nothing] = (0, -1, 0, -1)
    return box


def rays(k: so.Cam, xs, ys):
    """(O, D) float64 [M, 3] of pixel arrays xs, ys."""
    a, b = so.pixel_ab(k, xs, ys)
    a, b = a[:, None], b[:, None]
    P, f, r, u = (np.asarray(v)[None] for v in (k.P, k.f, k.r, k.u))
    if k.parallel:
        return (P + a * r) + b * u, np.broadcast_to(f, a.shape[:1] + (3,))
    return np.broadcast_to(P, a.shape[:1] + (3,)), (f + a * r) + b * u


def hit(E: Ellipsoids, O, D, near):
    """(covered, z) of rays O + t D against ellipsoids E, element-wise."""
    e, g = _local(E.R, E.k, O - E.c), _local(E.R, E.k, D)
    A, B, C = _dot(g, g), _dot(g, e), _dot(e, e) - 1.0
    disc = B * B - A * C
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        h = -(B + np.copysign(np.sqrt(disc), B))
        t1 = h / A
        t2 = np.where(h != 0.0, C / h, t1)
    lo, hi = np.fmin(t1, t2), np.fmax(t1, t2)
    covered = (disc >= 0.0) & (hi >= near)
    return covered, np.where(lo >= near, lo, hi)


def shade(E: Ellipsoids, O, D, z, base):
    """The headlight colour float32 [M, 3] at the hit H = O + z D with the normal R diag(1/s^2) R^T (H - c)."""
    v = (O + z[:, None] * D) - E.c
    m = _local(E.R, E.k, v) * E.k
    n = np.stack([(E.R[:, i, 0] * m[:, 0] + E.R[:, i, 1] * m[:, 1]) + E.R[:, i, 2] * m[:, 2] for i in range(3)], 1)
    nn, dd = _dot(n, n), _dot(D, D)
    with np.errstate(divide="ignore", invalid="ignore"):
        lam = np.where(nn > 0.0, np.fmin(np.abs(_dot(n, D) / np.sqrt(nn * dd)), 1.0), 0.0)
    s = so.AMBIENT + (1.0 - so.AMBIENT) * lam
    return (np.asarray(base, np.float32).astype(np.float64) * s[:, None]).astype(np.float32)


def _pairs(box, window):
    """(prim, x, y) int64 of every pixel of every box clipped to the window."""
    wy0, wy1, wx0, wx1 = window
    x0, x1 = np.maximum(box[:, 0], wx0), np.minimum(box[:, 1], wx1 - 1)
    y0, y1 = np.maximum(box[:, 2], wy0), np.minimum(box[:, 3], wy1 - 1)
    live = np.nonzero((x0 <= x1) & (y0 <= y1))[0]
    nx, ny = (x1 - x0 + 1)[live], (y1 - y0 + 1)[live]
    n = nx * ny
    prim = np.repeat(live, n)
    j = np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
    nxr = np.repeat(nx, n)
    return prim, x0[prim] + j % nxr, y0[prim] + j // nxr


def ellipsoid_keys(k: so.Cam, near, E: Ellipsoids, ids, window):
    """(flat pixel index, key uint64) of every covered pixel of ellipsoids E (ids: their rows in the list)."""
    prim, xs, ys = _pairs(boxes(k, near, E), window)
    O, D = rays(k, xs, ys)
    cov, z = hit(E.take(prim), O, D, near)
    d = so.clamp_depth(z[cov], near)
    key = (d.view(np.uint32).astype(np.uint64) << np.uint64(32)) | ids[prim[cov]].astype(np.uint64)
    return ys[cov] * k.W + xs[cov], key


def raster(pos, meta, attr, tex, lut, cams, H, W, parallel, near, background, window=None):
    pos = np.asarray(pos, np.float64).reshape(-1, 3, 3)
    meta = np.asarray(meta, np.int32).reshape(-1, 2)
    attr = np.asarray(attr, np.float32).reshape(-1, 12)
    recs = np.asarray(cams, np.float32).reshape(-1, 16)
    F = len(recs)
    ell = meta[:, 0] == ELLIPSOID
    keys = np.full((F, H, W), so.EMPTY, np.uint64)
    other = np.nonzero(~ell)[0]
    if len(other):
        k2, _ = so.raster(pos[other], meta[other], attr[other], tex, lut, recs, H, W, parallel, near, background,
                          window)
        hitk = k2 != so.EMPTY
        remap = other.astype(np.uint64)[(k2[hitk] & np.uint64(0xFFFFFFFF)).astype(np.int64)]
        keys[hitk] = (k2[hitk] & ~np.uint64(0xFFFFFFFF)) | remap
    cams = [so.Cam(r, H, W, bool(parallel)) for r in recs]
    ids = np.nonzero(ell)[0]
    if len(ids):
        E = Ellipsoids(pos[ids], attr[ids])
        for f, k in enumerate(cams):
            px, key = ellipsoid_keys(k, near, E, ids, window if window is not None else (0, H, 0, W))
            flat = keys[f].reshape(-1)
            np.minimum.at(flat, px, key)
    rgb = so.resolve(keys, pos, meta, attr, tex, lut, cams, near, background)
    for f, k in enumerate(cams):
        fy, fx = np.nonzero(keys[f] != so.EMPTY)
        sel = (keys[f, fy, fx] & np.uint64(0xFFFFFFFF)).astype(np.int64)
        e = meta[sel, 0] == ELLIPSOID
        if e.any():
            fy, fx, sel = fy[e], fx[e], sel[e]
            Es = Ellipsoids(pos[sel], attr[sel])
            O, D = rays(k, fx, fy)
            _, z = hit(Es, O, D, near)
            rgb[f, fy, fx] = shade(Es, O, D, z, attr[sel, 0:3])
    return keys, rgb
