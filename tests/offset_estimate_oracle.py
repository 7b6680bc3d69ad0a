"""Float64 oracle of the detector-offset estimate (`detector.estimate_offset`, r2x_detector_offset_cost), written from
the geometry, not from the kernel: the conjugate pairs by brute force over ordered view pairs, the samples and the cost
in numpy float64, the same coarse / fine / parabola search, and a closed-form projector of isotropic 3-D Gaussian
blobs whose line integrals make the redundancy identity exact.

Geometry (scene.make_view / angle2pose): the source of view beta sits at DSO (cos beta, sin beta, 0) and looks at the
origin; image columns run along e(beta) = (-sin beta, cos beta, 0), image rows along -z.  Column c of an image whose
rotation axis sits sigma columns right of the detector centre sees detector coordinate u = du (c - (W - 1) / 2 - sigma);
row r sees v = dv (r - (H - 1) / 2 - t_v) (v along -z).
"""
from __future__ import annotations

import math

import numpy as np

FINE = 64


# ---- closed-form projections of Gaussian blobs -----------------------------------------------------------------------

def blobs(n=9, seed=0, radius=0.7, zmax=0.3, sizes=(0.06, 0.2)):
    """[n, 5] rows (x, y, z, size, amplitude) of isotropic Gaussians amp exp(-|p - c|^2 / (2 size^2))."""
    rng = np.random.RandomState(seed)
    r = radius * np.sqrt(rng.rand(n))
    a = rng.rand(n) * 2 * np.pi
    return np.stack([r * np.cos(a), r * np.sin(a), rng.uniform(-zmax, zmax, n), rng.uniform(*sizes, n),
                     rng.uniform(0.5, 1.5, n)], axis=1)


def ray(beta, u, v, mode, DSD, DSO):
    """(origin [..., 3], unit direction [..., 3]) of the ray at detector coordinates (u, v) of view beta."""
    beta, u, v = np.broadcast_arrays(np.asarray(beta, np.float64), np.asarray(u, np.float64), np.asarray(v, np.float64))
    cb, sb = np.cos(beta), np.sin(beta)
    radial = np.stack([cb, sb, np.zeros_like(cb)], -1)
    e = np.stack([-sb, cb, np.zeros_like(cb)], -1)
    z = np.stack([np.zeros_like(cb)] * 2 + [np.ones_like(cb)], -1)
    if mode == "parallel":
        o = u[..., None] * e - v[..., None] * z + DSO * radial
        d = -radial
    else:
        o = DSO * radial
        p = o - DSD * radial + u[..., None] * e - v[..., None] * z
        d = p - o
        d = d / np.linalg.norm(d, axis=-1, keepdims=True)
    return o, d


def line_integral(blob_rows, beta, u, v, mode, DSD, DSO):
    """The exact integral of the blobs along the ray (beta, u, v): amp sqrt(2 pi) size exp(-dist^2 / (2 size^2))."""
    o, d = ray(beta, u, v, mode, DSD, DSO)
    out = np.zeros(o.shape[:-1])
    for x, y, zc, s, amp in blob_rows:
        w = np.array([x, y, zc]) - o
        along = (w * d).sum(-1)
        dist2 = (w * w).sum(-1) - along * along
        out += amp * math.sqrt(2 * math.pi) * s * np.exp(-np.maximum(dist2, 0.0) / (2 * s * s))
    return out


def project(blob_rows, angles, scanner, sigma=0.0, t_v=0.0):
    """[N, H, W] float64 images of the blobs whose rotation axis sits `sigma` columns right of the detector centre."""
    H, W = int(scanner["nDetector"][0]), int(scanner["nDetector"][1])
    du = scanner["sDetector"][1] / W
    dv = scanner["sDetector"][0] / H
    b = np.asarray(angles, np.float64)[:, None, None]
    u = du * (np.arange(W)[None, None, :] - (W - 1) / 2 - sigma)
    v = dv * (np.arange(H)[None, :, None] - (H - 1) / 2 - t_v)
    return line_integral(blob_rows, b, u, v, scanner["mode"], scanner["DSD"], scanner["DSO"])


def project_point(p, beta, mode, DSD, DSO):
    """Detector coordinate u of the world point p in view beta."""
    cb, sb = math.cos(beta), math.sin(beta)
    e = np.array([-sb, cb, 0.0])
    if mode == "parallel":
        return float(np.dot(p, e))
    rel = np.asarray(p, np.float64) - DSO * np.array([cb, sb, 0.0])
    depth = -float(np.dot(rel, [cb, sb, 0.0]))
    return DSD * float(np.dot(rel, e)) / depth


# ---- pairs, samples, cost --------------------------------------------------------------------------------------------

def pairs(angles, scanner, reach, angle_tol=1e-4):
    """[(i, j, dbeta)] with i < j: ordered pairs enumerated one by one, each unordered pair kept once."""
    W = int(scanner["nDetector"][1])
    du = scanner["sDetector"][1] / W
    out = []
    n = len(angles)
    for i in range(n):
        for j in range(n):
            if i == j:
                continue
            d = (float(angles[j]) - float(angles[i])) % (2 * math.pi)
            if scanner["mode"] == "parallel":
                ok = abs(d - math.pi) <= angle_tol
            else:
                ok = 0.0 < d and abs(scanner["DSD"] * math.tan((math.pi - d) / 2) / du) <= reach
            if ok and i < j:
                out.append((i, j, d))
    return out


def partner(beta, gamma):
    """The conjugate (beta', gamma') of the cone-beam mid-plane ray (beta, gamma): (beta + pi - 2 gamma, -gamma)."""
    return beta + math.pi - 2.0 * gamma, -gamma


def _lerp(projs, r, c, v):
    """Bilinear value of projs [N, H, W] in views v at (r, c) arrays (valid positions only)."""
    _, H, W = projs.shape
    r0 = np.floor(r).astype(np.int64)
    c0 = np.floor(c).astype(np.int64)
    fr, fc = r - r0, c - c0
    r1, c1 = np.minimum(r0 + 1, H - 1), np.minimum(c0 + 1, W - 1)
    top = (1 - fc) * projs[v, r0, c0] + fc * projs[v, r0, c1]
    bot = (1 - fc) * projs[v, r1, c0] + fc * projs[v, r1, c1]
    return (1 - fr) * top + fr * bot


def samples(projs, table, scanner, sigma, t_v=0.0, rows=None):
    """(a, b) float64 arrays of the valid conjugate samples at shift sigma."""
    N, H, W = projs.shape
    du = scanner["sDetector"][1] / W
    if scanner["mode"] == "cone":                       # one sample per pair: all pairs at once
        i, j, d = (np.array(x) for x in zip(*table))
        t = scanner["DSD"] * np.tan((math.pi - d) / 2) / du
        r = np.full(t.shape, (H - 1) / 2 + t_v)
        ci, cj = (W - 1) / 2 + t + sigma, (W - 1) / 2 - t + sigma
        ok = (ci >= 0) & (ci <= W - 1) & (cj >= 0) & (cj <= W - 1) & (r >= 0) & (r <= H - 1)
        return _lerp(projs, r[ok], ci[ok], i[ok]), _lerp(projs, r[ok], cj[ok], j[ok])
    A, B = [], []
    lo, hi = (0, H) if rows is None else rows
    m = np.arange(W, dtype=np.float64)
    r = np.repeat(np.arange(lo, hi, dtype=np.float64), W)
    ci = np.tile(m + sigma, hi - lo)
    cj = np.tile((W - 1 - m) + sigma, hi - lo)
    ok = (ci >= 0) & (ci <= W - 1) & (cj >= 0) & (cj <= W - 1)
    for i, j, d in table:                               # parallel beam: every column of every row
        A.append(_lerp(projs, r[ok], ci[ok], i))
        B.append(_lerp(projs, r[ok], cj[ok], j))
    return np.concatenate(A), np.concatenate(B)


def cost_terms(projs, table, scanner, sigmas, t_v=0.0, rows=None):
    """(num, den, count) per candidate sigma."""
    p = np.asarray(projs, np.float64)
    out = []
    for s in sigmas:
        a, b = samples(p, table, scanner, float(s), t_v, rows)
        out.append((float(((a - b) ** 2).sum()), float((a * a + b * b).sum()), int(a.size)))
    num, den, cnt = (np.array(x) for x in zip(*out))
    return num, den, cnt


def estimate(projs, angles, scanner, t_u=0.0, t_v=0.0, max_shift=None, angle_tol=1e-4, rows=None):
    """The search of detector.estimate_offset in float64: -> (s, cost curve dict)."""
    N, H, W = projs.shape
    M = int(math.ceil(W / 4 if max_shift is None else max_shift))
    table = pairs(angles, scanner, (W - 1) / 2 + M + 1 + abs(t_u), angle_tol)
    if not table:
        raise ValueError("no conjugate pairs")
    coarse = np.arange(-M, M + 1, dtype=np.float64)
    num, den, _ = cost_terms(projs, table, scanner, coarse - t_u, t_v, rows)
    cc = np.where(den > 0, num / np.where(den > 0, den, 1), np.inf)
    k = int(np.argmin(cc))
    if k in (0, len(coarse) - 1):
        raise ValueError("minimum on the edge")
    fine = coarse[k] + np.arange(-FINE, FINE + 1) / FINE
    num, den, cnt = cost_terms(projs, table, scanner, fine - t_u, t_v, rows)
    fc = np.where(den > 0, num / np.where(den > 0, den, 1), np.inf)
    j = int(np.argmin(fc))
    y0, y1, y2 = fc[j - 1], fc[j], fc[j + 1]
    curv = y0 - 2 * y1 + y2
    s = fine[j] + (0.5 * (y0 - y2) / curv / FINE if curv > 0 else 0.0)
    return float(s), {"table": table, "coarse": (coarse, cc), "fine": (fine, fc), "n_samples": int(cnt[j])}
