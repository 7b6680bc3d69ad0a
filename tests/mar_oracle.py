"""numpy restatement of r2x_mar_inpaint (include/r2x.h), op for op in float32, and a float64 restatement of the host
rules of `mar.reduce_metal`: segmentation, the NMAR prior's classes, reinsertion and the score outside the metal."""
from __future__ import annotations

import numpy as np


def trace_row(m: np.ndarray, tau: float, d: int) -> np.ndarray:
    """t[c] = any(m[k] > tau) for k in [c - d, c + d] clipped to the row, by direct search."""
    W = m.shape[0]
    t0 = np.asarray(m, np.float32) > np.float32(tau)
    return np.array([t0[max(0, c - d):min(W, c + d + 1)].any() for c in range(W)], bool)


CANONICAL_NAN = np.array([0x7FFFFFFF], np.uint32).view(np.float32)[0]


def _arith(x):
    """A result of float32 arithmetic as the GPU gives it: a NaN is the canonical 0x7FFFFFFF, whatever NaN went in."""
    x = np.asarray(x, np.float32)
    return np.where(np.isnan(x), CANONICAL_NAN, x).astype(np.float32)


def inpaint_row(p, m, tau, d, P=None, eps=1e-3):
    """(out, t) of one row, float32 throughout."""
    p = np.asarray(p, np.float32)
    W = p.shape[0]
    t = trace_row(m, tau, d)
    out = p.copy()
    if P is not None:
        P = np.asarray(P, np.float32)
        e = np.float32(eps)
        Pe = np.where(P > e, P, e).astype(np.float32)       # a NaN P gives eps
        with np.errstate(all="ignore"):
            q = _arith(p / Pe)
    else:
        q = p
    good = np.flatnonzero(~t)
    for c in np.flatnonzero(t):
        left, right = good[good < c], good[good > c]
        if len(left) and len(right):
            l, r = int(left[-1]), int(right[0])
            with np.errstate(all="ignore"):
                s = np.float32(c - l) / np.float32(r - l)
                v = _arith(q[l] + np.float32(s * np.float32(q[r] - q[l])))
        elif len(left):
            v = q[int(left[-1])]
        elif len(right):
            v = q[int(right[0])]
        elif P is not None:
            v = np.float32(1.0)
        else:
            continue
        with np.errstate(all="ignore"):
            out[c] = _arith(v * Pe[c]) if P is not None else v
    return out, t


def inpaint(p, m, tau, d, P=None, eps=1e-3, rows=None):
    """The model on a stack [n, H, W]; `rows` restricts it to those detector rows (out[:, rows])."""
    p, m = np.asarray(p, np.float32), np.asarray(m, np.float32)
    rows = range(p.shape[1]) if rows is None else rows
    out = np.empty((p.shape[0], len(rows), p.shape[2]), np.float32)
    trace = np.empty(out.shape, np.uint8)
    for v in range(p.shape[0]):
        for i, r in enumerate(rows):
            o, t = inpaint_row(p[v, r], m[v, r], tau, d, None if P is None else P[v, r], eps)
            out[v, i], trace[v, i] = o, t
    return out, trace


# ---- reduce_metal's host rules, float64 ------------------------------------------------------------------------------

def segment(fdk_vol, threshold):
    return np.asarray(fdk_vol, np.float32) > np.float32(threshold)


def nmar_prior(x, mask, air=0.5, bone=1.5, floor=0.1):
    """The NMAR prior of mar.nmar_prior: s = the lower median of the non-metal voxels above floor * their maximum;
    below air * s -> 0, tissue [air s, bone s) and metal -> the tissue mean, at or above bone * s kept."""
    x = np.asarray(x, np.float32)
    x64 = x.astype(np.float64)
    keep = ~mask
    top = x64[keep].max()
    sel = np.sort(x64[keep & (x64 > floor * top)])
    s = sel[(len(sel) - 1) // 2]
    tissue = keep & (x64 >= air * s) & (x64 < bone * s)
    mean = x64[tissue].mean()
    prior = np.where(x64 < air * s, 0.0, x64)
    prior = np.where(tissue | mask, mean, prior)
    return prior.astype(np.float32), s, mean


def reinsert(volume, fdk_with_metal, mask):
    return np.where(mask, fdk_with_metal, volume)


def dilate(mask, k=2):
    """mask dilated by k voxels in every direction (the (2k + 1)^3 cube)."""
    out = mask.copy()
    padded = np.pad(mask, k)
    nx, ny, nz = mask.shape
    for a in range(2 * k + 1):
        for b in range(2 * k + 1):
            for c in range(2 * k + 1):
                out |= padded[a:a + nx, b:b + ny, c:c + nz]
    return out


def psnr_outside_metal(gt, pred, mask, k=2):
    out = ~dilate(mask, k)
    g, x = np.asarray(gt, np.float64)[out], np.asarray(pred, np.float64)[out]
    mse = np.mean((g - x) ** 2)
    return 10.0 * np.log10(g.max() ** 2 / mse)
