"""A float64 / int64 numpy statement of the scene-view rasterizer (include/r2x.h, "scene view"), operation for
operation: the clipping, snapping, edge functions, line distance and depth give the kernel's keys bit for bit, and the
shading its colours.  Python floats and numpy float64 element-wise operations round every operation once, as the
kernel's explicit round-to-nearest intrinsics do.

    keys, rgb = raster(pos, meta, attr, tex, lut, cams, H, W, parallel, near, background)

`cams` are the float32 camera records (volume_render.Camera.record()).  `window=(y0, y1, x0, x1)` restricts the work to
those rows and columns (exclusive ends); pixels outside it stay empty and are not meaningful.
"""
from __future__ import annotations

import math

import numpy as np

FLAT, MESH, TEXTURED, LINE = 0, 1, 2, 3
GUARD = 1048576.0
AMBIENT = 0.25
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


class Cam:
    def __init__(self, rec, H, W, parallel):
        r = [float(v) for v in np.asarray(rec, np.float32)]
        self.P, self.f, self.r, self.u, self.p = r[0:3], r[3:6], r[6:9], r[9:12], r[12]
        self.H, self.W, self.parallel = H, W, parallel


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def to_cam(k: Cam, X):
    d = [float(X[0]) - k.P[0], float(X[1]) - k.P[1], float(X[2]) - k.P[2]]
    return [_dot(d, k.r), _dot(d, k.u), _dot(d, k.f)]


def _plane(k: Cam, near, j, c):
    if j == 0:
        return c[2] - near
    g = GUARD * k.p if k.parallel else (GUARD * k.p) * c[2]
    s = c[(j - 1) >> 1] if j in (1, 3) else -c[(j - 1) >> 1]
    return g - s


def _cut(a, b, da, db):
    t = da / (da - db)
    return [a[i] + t * (b[i] - a[i]) for i in range(3)]


def _project(k: Cam, c):
    den = k.p if k.parallel else c[2] * k.p
    return 0.5 * k.W + c[0] / den, 0.5 * k.H - c[1] / den


def _snap(s):
    return int(np.rint(s * 256.0))


def clip_triangle(k: Cam, near, V):
    poly = [list(v) for v in V]
    for j in range(5):
        if not poly:
            break
        out = []
        n = len(poly)
        for i in range(n):
            a, b = poly[i], poly[(i + 1) % n]
            da, db = _plane(k, near, j, a), _plane(k, near, j, b)
            if da >= 0.0:
                out.append(a)
            if (da >= 0.0) != (db >= 0.0):
                out.append(_cut(a, b, da, db) if da >= 0.0 else _cut(b, a, db, da))
        poly = out
    return poly if len(poly) >= 3 else []


def clip_segment(k: Cam, near, a, b):
    for j in range(5):
        da, db = _plane(k, near, j, a), _plane(k, near, j, b)
        if da < 0.0 and db < 0.0:
            return None
        if da < 0.0:
            a = _cut(b, a, db, da)
        elif db < 0.0:
            b = _cut(a, b, da, db)
    return a, b


def geometry(k: Cam, near, pos_i, kind, width):
    """The primitive in one frame: dict with the clamped pixel box and what the pixel test needs, or None."""
    if kind == LINE:
        a, b = to_cam(k, pos_i[0]), to_cam(k, pos_i[1])
        ab = clip_segment(k, near, a, b)
        if ab is None:
            return None
        a, b = ab
        ax, ay = (_snap(s) / 256.0 for s in _project(k, a))
        bx, by = (_snap(s) / 256.0 for s in _project(k, b))
        r = 0.5 * float(np.float32(width))
        g = {"line": True, "a": (ax, ay), "b": (bx, by), "za": a[2], "zb": b[2], "r": r}
        g["x0"] = int(max(math.ceil((min(ax, bx) - r) - 0.5), 0.0))
        g["x1"] = int(min(math.floor((max(ax, bx) + r) - 0.5), float(k.W - 1)))
        g["y0"] = int(max(math.ceil((min(ay, by) - r) - 0.5), 0.0))
        g["y1"] = int(min(math.floor((max(ay, by) + r) - 0.5), float(k.H - 1)))
        return g
    V = [to_cam(k, pos_i[v]) for v in range(3)]
    poly = clip_triangle(k, near, V)
    if not poly:
        return None
    S = [tuple(_snap(s) for s in _project(k, c)) for c in poly]
    xs, ys = [s[0] for s in S], [s[1] for s in S]
    e1 = [V[1][i] - V[0][i] for i in range(3)]
    e2 = [V[2][i] - V[0][i] for i in range(3)]
    n = [e1[1] * e2[2] - e1[2] * e2[1], e1[2] * e2[0] - e1[0] * e2[2], e1[0] * e2[1] - e1[1] * e2[0]]
    return {"line": False, "S": S, "n": n, "c": _dot(n, V[0]), "V": V,
            "x0": max((min(xs) - 128 + 255) >> 8, 0), "x1": min((max(xs) - 128) >> 8, k.W - 1),
            "y0": max((min(ys) - 128 + 255) >> 8, 0), "y1": min((max(ys) - 128) >> 8, k.H - 1)}


def _edge_in(a, b, px, py):
    dx, dy = b[0] - a[0], b[1] - a[1]
    e = dx * (py - a[1]) - dy * (px - a[0])
    top_left = dy < 0 or (dy == 0 and dx > 0)
    return (e > 0) | ((e == 0) & top_left)


def pixel_ab(k: Cam, x, y):
    """a = ((x + 1/2) - W/2) p, b = ((H/2 - y) - 1/2) p, element-wise over integer arrays."""
    x = np.asarray(x, np.float64)
    y = np.asarray(y, np.float64)
    return ((x + 0.5) - 0.5 * k.W) * k.p, ((0.5 * k.H - y) - 0.5) * k.p


def tri_depth(k: Cam, n, c, a, b):
    if k.parallel:
        return ((c - n[0] * a) - n[1] * b) / n[2]
    return c / ((n[0] * a + n[1] * b) + n[2])


def cover(k: Cam, g, xs, ys):
    """(covered mask, depth float64) at pixel arrays xs, ys (int64)."""
    if g["line"]:
        (ax, ay), (bx, by), r = g["a"], g["b"], g["r"]
        cx, cy = xs.astype(np.float64) + 0.5, ys.astype(np.float64) + 0.5
        dx, dy, ex, ey = bx - ax, by - ay, cx - ax, cy - ay
        L = dx * dx + dy * dy
        if L > 0.0:
            with np.errstate(invalid="ignore"):
                t = np.fmin(np.fmax((ex * dx + ey * dy) / L, 0.0), 1.0)
        else:
            t = np.zeros_like(cx)
        qx, qy = ex - t * dx, ey - t * dy
        m = (qx * qx + qy * qy) <= r * r
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            if k.parallel:
                z = g["za"] + t * (g["zb"] - g["za"])
            else:
                z = 1.0 / ((1.0 - t) / g["za"] + t / g["zb"])
        return m, z
    px, py = 256 * xs + 128, 256 * ys + 128
    S = g["S"]
    m = np.zeros(xs.shape, bool)
    for v in range(1, len(S) - 1):
        A, B, C = S[0], S[v], S[v + 1]
        area = (B[0] - A[0]) * (C[1] - A[1]) - (B[1] - A[1]) * (C[0] - A[0])
        if area == 0:
            continue
        if area < 0:
            B, C = C, B
        m |= _edge_in(A, B, px, py) & _edge_in(B, C, px, py) & _edge_in(C, A, px, py)
    a, b = pixel_ab(k, xs, ys)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        z = tri_depth(k, g["n"], g["c"], a, b)
    return m, z


def clamp_depth(z, near):
    z = np.where(z >= near, z, near)          # NaN -> near
    with np.errstate(over="ignore"):
        return z.astype(np.float32)


def _candidates(cams, near, pos, window, H, W):
    """Primitives that may touch the window in some frame: all of them, unless the window is given, in which case a
    vectorized pass drops those wholly in front of the near plane, inside the guard band and off the window."""
    n = len(pos)
    if window is None:
        return [np.arange(n)] * len(cams)
    y0, y1, x0, x1 = window
    out = []
    for k in cams:
        P = np.asarray(k.P)
        d = pos - P
        c = [(d[..., 0] * rr[0] + d[..., 1] * rr[1]) + d[..., 2] * rr[2] for rr in (k.r, k.u, k.f)]
        den = k.p if k.parallel else c[2] * k.p
        with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
            sx, sy = 0.5 * W + c[0] / den, 0.5 * H - c[1] / den
        safe = (c[2] >= near * 2).all(1) & (np.abs(sx - 0.5 * W) < GUARD / 2).all(1) & \
               (np.abs(sy - 0.5 * H) < GUARD / 2).all(1)
        # conservative box: the snap moves a point by at most 1/512 pixel; lines add their half width in the caller
        pad = 64.0
        hit = (sx.max(1) + pad >= x0) & (sx.min(1) - pad <= x1) & (sy.max(1) + pad >= y0) & (sy.min(1) - pad <= y1)
        out.append(np.nonzero(~safe | hit)[0])
    return out


def raster(pos, meta, attr, tex, lut, cams, H, W, parallel, near, background, window=None):
    pos = np.asarray(pos, np.float64).reshape(-1, 3, 3)
    meta = np.asarray(meta, np.int32).reshape(-1, 2)
    attr = np.asarray(attr, np.float32).reshape(-1, 12)
    cams = [Cam(r, H, W, bool(parallel)) for r in np.asarray(cams, np.float32).reshape(-1, 16)]
    F = len(cams)
    keys = np.full((F, H, W), EMPTY, np.uint64)
    wy0, wy1, wx0, wx1 = window if window is not None else (0, H, 0, W)
    for f, (k, ids) in enumerate(zip(cams, _candidates(cams, near, pos, window, H, W))):
        for i in ids.tolist():
            g = geometry(k, near, pos[i], int(meta[i, 0]), attr[i, 3])
            if g is None:
                continue
            x0, x1 = max(g["x0"], wx0), min(g["x1"], wx1 - 1)
            y0, y1 = max(g["y0"], wy0), min(g["y1"], wy1 - 1)
            if x0 > x1 or y0 > y1:
                continue
            ys, xs = np.mgrid[y0:y1 + 1, x0:x1 + 1]
            ys, xs = ys.ravel().astype(np.int64), xs.ravel().astype(np.int64)
            m, z = cover(k, g, xs, ys)
            if not m.any():
                continue
            d = clamp_depth(z[m], near)
            key = (d.view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.uint64(i)
            keys[f, ys[m], xs[m]] = np.minimum(keys[f, ys[m], xs[m]], key)
    rgb = resolve(keys, pos, meta, attr, tex, lut, cams, near, background)
    return keys, rgb


def lut_colour(lut, t):
    """The volume renderer's LUT map in float32 without FMA, t float32 [M] -> [M, 3]."""
    lut = np.asarray(lut, np.float32).reshape(-1, 3)
    K = len(lut)
    if K == 1:
        return np.repeat(lut[:1], len(t), 0)
    pos = t * np.float32(K - 1)
    j = np.minimum(np.floor(pos).astype(np.int64), K - 2)
    w = (pos - j.astype(np.float32))[:, None]
    return (np.float32(1) - w) * lut[j] + w * lut[j + 1]


def resolve(keys, pos, meta, attr, tex, lut, cams, near, background):
    F, H, W = keys.shape
    rgb = np.empty((F, H, W, 3), np.float32)
    rgb[:] = np.asarray(background, np.float32)
    for f, k in enumerate(cams):
        fy, fx = np.nonzero(keys[f] != EMPTY)
        if not len(fy):
            continue
        ids = (keys[f, fy, fx] & np.uint64(0xFFFFFFFF)).astype(np.int64)
        kind = meta[ids, 0]
        at = attr[ids]
        col = at[:, 0:3].astype(np.float32).copy()
        tri = (kind == MESH) | (kind == TEXTURED)
        if tri.any():
            sel = np.nonzero(tri)[0]
            col[sel] = _shade(k, near, pos[ids[sel]], meta[ids[sel]], at[sel], fx[sel], fy[sel], tex, lut)
        rgb[f, fy, fx] = col
    return rgb


def _shade(k: Cam, near, X, meta, at, xs, ys, tex, lut):
    P = np.asarray(k.P)
    V = []
    for v in range(3):
        d = X[:, v] - P
        V.append(np.stack([(d[:, 0] * rr[0] + d[:, 1] * rr[1]) + d[:, 2] * rr[2] for rr in (k.r, k.u, k.f)], 1))
    e1, e2 = V[1] - V[0], V[2] - V[0]
    n = np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                  e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)
    dot = lambda a, b: (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]
    c = dot(n, V[0])
    a, b = pixel_ab(k, xs, ys)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        z = tri_depth(k, [n[:, 0], n[:, 1], n[:, 2]], c, a, b)
    z = np.where(z >= near, z, near)
    Pt = np.stack([a, b, z], 1) if k.parallel else np.stack([a * z, b * z, z], 1)
    n2 = dot(n, n)
    w = np.full((len(xs), 3), 1.0 / 3.0)
    ok = n2 > 0.0
    for v in range(3):
        A, B = V[(v + 1) % 3] - Pt, V[(v + 2) % 3] - Pt
        cr = np.stack([A[:, 1] * B[:, 2] - A[:, 2] * B[:, 1], A[:, 2] * B[:, 0] - A[:, 0] * B[:, 2],
                       A[:, 0] * B[:, 1] - A[:, 1] * B[:, 0]], 1)
        with np.errstate(divide="ignore", invalid="ignore"):
            w[ok, v] = (dot(n, cr) / n2)[ok]
    out = np.empty((len(xs), 3), np.float32)
    mesh = meta[:, 0] == MESH
    if mesh.any():
        at64 = at.astype(np.float64)
        N = (w[:, 0:1] * at64[:, 3:6] + w[:, 1:2] * at64[:, 6:9]) + w[:, 2:3] * at64[:, 9:12]
        f, r, u = (np.asarray(v) for v in (k.f, k.r, k.u))
        D = np.broadcast_to(f, N.shape) if k.parallel else (f + a[:, None] * r) + b[:, None] * u
        nn, dd = dot(N, N), dot(D, D)
        with np.errstate(divide="ignore", invalid="ignore"):
            lam = np.where(nn > 0.0, np.fmin(np.abs(dot(N, D) / np.sqrt(nn * dd)), 1.0), 0.0)
        shade = AMBIENT + (1.0 - AMBIENT) * lam
        out[mesh] = (at64[:, 0:3] * shade[:, None]).astype(np.float32)[mesh]
    txd = ~mesh
    if txd.any():
        at64 = at.astype(np.float64)
        tu = (w[:, 0] * at64[:, 3] + w[:, 1] * at64[:, 5]) + w[:, 2] * at64[:, 7]
        tv = (w[:, 0] * at64[:, 4] + w[:, 1] * at64[:, 6]) + w[:, 2] * at64[:, 8]
        tex = np.asarray(tex, np.float32)
        th, tw = tex.shape[1:]
        with np.errstate(invalid="ignore"):
            j = np.fmin(np.fmax(np.floor(tu * tw), 0.0), tw - 1.0).astype(np.int64)
            i = np.fmin(np.fmax(np.floor(tv * th), 0.0), th - 1.0).astype(np.int64)
        val = tex[meta[txd, 1], i[txd], j[txd]]
        t = np.fmin(np.fmax(val, np.float32(0)), np.float32(1))          # NaN -> 0
        out[txd] = lut_colour(lut, t)
    return out
