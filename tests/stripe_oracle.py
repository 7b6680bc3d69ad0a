"""numpy restatement of r2x_remove_stripes (include/r2x.h), op for op: key, sort by (key, view), the rank-h key of each
reflected window of columns, put back.  Exact: every output is an input value."""
from __future__ import annotations

import numpy as np
from scipy.ndimage import median_filter


def key(x: np.ndarray) -> np.ndarray:
    u = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def unkey(k: np.ndarray) -> np.ndarray:
    k = np.asarray(k, np.uint32)
    return np.where(k & np.uint32(0x80000000), k & np.uint32(0x7FFFFFFF), ~k).astype(np.uint32).view(np.float32)


def reflect_index(W: int, h: int) -> np.ndarray:
    """Column read for j = -h .. W - 1 + h: -j - 1 left of 0, 2W - 1 - j right of W - 1 (needs h <= W)."""
    j = np.arange(-h, W + h)
    return np.where(j < 0, -j - 1, np.where(j >= W, 2 * W - 1 - j, j))


def sinogram(S: np.ndarray, K: int) -> np.ndarray:
    """The model on one sinogram S[n views, W columns] (float32)."""
    n, W = S.shape
    h = K // 2
    assert K % 2 == 1 and h <= W
    keys = key(S)
    words = (keys.astype(np.uint64) << np.uint64(32)) | np.arange(n, dtype=np.uint64)[:, None]
    order = np.argsort(words, axis=0)                                  # words are unique: the sort is (key, v)
    T = np.take_along_axis(keys, order, axis=0)
    win = np.lib.stride_tricks.sliding_window_view(T[:, reflect_index(W, h)], K, axis=1)   # [n, W, K]
    M = np.sort(win, axis=2)[:, :, h]
    out = np.empty((n, W), np.uint32)
    np.put_along_axis(out, order, M, axis=0)
    return unkey(out)


def remove_stripes(stack: np.ndarray, K: int, rows=None) -> np.ndarray:
    """The model on in[n, H, W]; with `rows`, only those rows, as [n, len(rows), W]."""
    stack = np.asarray(stack, np.float32)
    rows = range(stack.shape[1]) if rows is None else rows
    return np.stack([sinogram(stack[:, r, :], K) for r in rows], axis=1)


def sarepy(S: np.ndarray, K: int) -> np.ndarray:
    """sarepy's remove_stripe_based_sorting with the 1-D window: stable argsort over the views, median_filter of
    size (1, K) with mode="reflect", inverse permutation."""
    idx = np.argsort(S, axis=0, kind="stable")
    T = np.take_along_axis(S, idx, axis=0)
    M = median_filter(T, size=(1, K), mode="reflect")
    out = np.empty_like(S)
    np.put_along_axis(out, idx, M, axis=0)
    return out
