"""A float64 statement of the rasterizer's and the voxelizer's forwards, per pixel and per voxel, to judge the float32
kernels element by element (tests/test_forward_float64_gpu.py; tests/test_forward_float64_cpu.py checks the statement).

The suite's image checks share one bar, 1e-5 of the image maximum.  CT projections have a wide dynamic range: a pixel
at 1e-4 of the maximum can be 10 % wrong under that bar, yet the training loss is per pixel and evaluation scores the
volume voxel by voxel.  The kernels' own arithmetic has errors relative to each (Gaussian, pixel) pair -- exponent-2
domain, log2 w folded into the exponent, alpha advanced by multiplicative forward differences from an anchor up to 3
pixels back (render_fast_8, voxel_fast_8) -- so it is judged per pixel, against the float64 sum of the same pairs.

From the forward's own stage outputs (xy, conic_opacity, mu, the tile lists; xyz_vol, conic_opacity for the voxelizer),
each pixel gets, over the Gaussians of its tile:
  S64      the float64 sum of alpha = w exp(power) over the decided pairs, plus half of each borderline pair (the band
           rule of grad_float64: alpha within BAND of the cut, or power within BAND of 0 relative to its terms);
  absw     sum over the decided pairs of |alpha| (1 + L / POWER_WEIGHT), L = the power's terms |A dx^2 / 2| + |C dy^2 / 2|
           + |B dx dy| plus |log2 w|: the fast paths carry w in the exponent (rasterizer: log2 w, voxelizer: log2 rho),
           so each term's rounding is relative to L, as in the backward's statement;
  abs_all  sum of |alpha| over the decided and the borderline pairs; border = sum over the borderline pairs;
  n, n_border, and n_chain, the longest chain of float32 additions any term of the pixel goes through.
The bar is
    |got - S64| <= C_BAR u absw + u n_chain abs_all + border / 2
(the terms' own rounding, the summation's, and the pairs neither side can decide).

n_chain.  A float32 sum whose partial sums start from exact zeros is within u d sum|t| of the exact sum, d the depth of
the deepest term in its addition tree, and d <= n - 1 for any tree of n terms.  The C oracle adds the terms of a pixel
one by one in depth order: n_chain = n - 1.  The rasterizer's render kernel deals a chunk's Gaussians to RW_SLICES
slices (slice s takes chunk positions j = s mod RW_SLICES), adds the slices in fixed order and then the tile's chunks
in chunk order: n_chain = min(n - 1, max over chunks and slices of that pixel's terms in one slice + RW_SLICES +
chunks).  The voxelizer's chunk size is decided on the device from R (and overridden by two-level binning), so its
chain is not stated tightly here: n_chain = n - 1.

Every constant of the kernels is read from the CUDA sources (regime_cases.py).

Measured on an H100 80GB HBM3 (700 W) with tests/test_forward_float64_gpu.py: no kernel needed a fix.  Over pixels
without a borderline pair the worst element is 0.36x the bar (the anchor case: A2 = 2, log2 w = 20, first contributing
pixel at the end of a run), 0.23x on the dynamic-range cloud's faint pixels, 0.21x on the radix path and at most 0.30x
for the voxelizer; a pixel holding a borderline pair can reach ~1x, since half that pair is its bar.
"""
from __future__ import annotations

import numpy as np

import regime_cases as rc
from grad_float64 import ALPHA_CUT, BAND, C_BAR, POWER_WEIGHT, U, VALPHA_CUT, VBAND, tile_rect, voxel_cube  # noqa: F401

RW_SLICES = rc._constexpr("RW_SLICES", rc._source("r2x_raster.cu"), {})
VR_SLICES = rc._constexpr("VR_SLICES", rc._source("r2x_voxel.cu"), {})
PLAN_CHUNK = rc.K["PLAN_CHUNK"]
FAINT = 1e-4          # a judged pixel below this fraction of the image maximum is "faint"
KEYS = ("S64", "absw", "abs_all", "border", "n", "n_border", "n_chain")


def _empty(shape):
    out = {k: np.zeros(shape) for k in KEYS[:4]}
    out.update({k: np.zeros(shape, np.int64) for k in KEYS[4:]})
    return out


def _plan_slices(n_list, chunk=PLAN_CHUNK):
    """(chunk, position in chunk) of every entry of a tile list of n_list, as plan_slice cuts it: ceil(n / chunk)
    chunks of equal length (+-1), the first `rem` one longer."""
    nch = max(1, -(-n_list // chunk))
    q, rem = divmod(n_list, nch)
    lens = np.full(nch, q) + (np.arange(nch) < rem)
    ch = np.repeat(np.arange(nch), lens)
    pos = np.arange(n_list) - np.repeat(np.cumsum(lens) - lens, lens)
    return ch, pos, nch


def _tiles(ranges, tiles):
    live = np.nonzero(ranges[:, 1] > ranges[:, 0])[0]
    return live if tiles is None else np.intersect1d(live, np.asarray(tiles, np.int64))


def _tile_terms(alpha, power, L, cut, band_rel):
    """Decided / borderline masks of a tile's pairs [terms, pixels] (grad_float64's band rule)."""
    inside = (power <= 0.0) & (alpha >= cut)
    border = (np.abs(alpha - cut) <= band_rel * cut) | (np.abs(power) <= band_rel * L + 1e-300)
    border &= alpha >= (1 - band_rel) * cut
    return inside & ~border, border


def _accumulate(out, sel, alpha, L, dec, border, chain, flags=None, ids=None):
    a = np.abs(alpha)
    for name, f in (flags or {}).items():       # contributing pairs of the flagged Gaussians, per element
        out["count_" + name][sel] = ((dec | border) & f[ids, None]).sum(0)
    out["S64"][sel] = np.where(dec, alpha, 0.0).sum(0) + 0.5 * np.where(border, alpha, 0.0).sum(0)
    out["absw"][sel] = np.where(dec, a * (1.0 + L / POWER_WEIGHT), 0.0).sum(0)
    out["abs_all"][sel] = np.where(dec | border, a, 0.0).sum(0)
    out["border"][sel] = np.where(border, a, 0.0).sum(0)
    n = dec.sum(0)
    nb = border.sum(0)
    out["n"][sel] = n
    out["n_border"][sel] = nb
    out["n_chain"][sel] = np.minimum(np.maximum(n + nb - 1, 0), chain)


def raster_statement(xy, conic_opacity, mu, ranges, point_list, W, H, chain="kernel", flags=None, tiles=None):
    """Per pixel [H, W] arrays of KEYS.  chain: 'kernel' (the render kernel's slices and chunks, point_list in the
    kernel's order) or 'oracle' (one sequential sum: n - 1).  flags: {name: [P] bool}, adds per pixel 'count_<name>',
    the contributing pairs of the flagged Gaussians.  tiles: only these tiles (default: every tile)."""
    out = _empty((H, W))
    for name in flags or {}:
        out["count_" + name] = np.zeros((H, W), np.int64)
    gx = (W + 15) // 16
    lw_all = np.log2(np.maximum((conic_opacity[:, 3] * mu).astype(np.float32).astype(np.float64), 1e-300))
    for t in _tiles(ranges, tiles):
        a, b = (int(v) for v in ranges[t])
        ids = point_list[a:b].astype(np.int64)
        tx, ty = t % gx, t // gx
        ys, xs = np.mgrid[ty * 16:min(H, ty * 16 + 16), tx * 16:min(W, tx * 16 + 16)]
        p = xy[ids].astype(np.float64)
        co = conic_opacity[ids].astype(np.float64)
        w = (conic_opacity[ids, 3] * mu[ids]).astype(np.float32).astype(np.float64)
        dx = p[:, 0, None] - xs.reshape(1, -1)
        dy = p[:, 1, None] - ys.reshape(1, -1)
        ta, tc, tb = 0.5 * co[:, 0, None] * dx * dx, 0.5 * co[:, 2, None] * dy * dy, co[:, 1, None] * dx * dy
        power = -(ta + tc) - tb
        alpha = w[:, None] * np.exp(np.minimum(power, 0.0))
        Lp = np.abs(ta) + np.abs(tc) + np.abs(tb)
        dec, border = _tile_terms(alpha, power, Lp, ALPHA_CUT, BAND)
        L = Lp + np.abs(lw_all[ids])[:, None]
        if chain == "kernel":
            ch, pos, nch = _plan_slices(len(ids))
            live = (dec | border).astype(np.int64)
            key = ch * RW_SLICES + pos % RW_SLICES
            per = np.zeros((nch * RW_SLICES, live.shape[1]), np.int64)
            np.add.at(per, key, live)
            c = per.max(0) + RW_SLICES + nch
        else:
            c = np.iinfo(np.int64).max
        _accumulate(out, (ys.reshape(-1), xs.reshape(-1)), alpha, L, dec, border, c, flags, ids)
    return out


def voxel_statement(xyz_vol, conic_opacity, ranges, point_list, nV, flags=None, tiles=None):
    """Per voxel [nx, ny, nz] arrays of KEYS (n_chain = n - 1, see the module's docstring); flags, tiles as for
    raster_statement."""
    out = _empty(tuple(nV))
    for name in flags or {}:
        out["count_" + name] = np.zeros(tuple(nV), np.int64)
    g = [-(-n // 8) for n in nV]
    rho_all = conic_opacity[:, 6].astype(np.float64)
    lw_all = np.log2(np.maximum(rho_all, 1e-300))
    for t in _tiles(ranges, tiles):
        a, b = (int(v) for v in ranges[t])
        ids = point_list[a:b].astype(np.int64)
        tx, ty, tz = t % g[0], (t // g[0]) % g[1], t // (g[0] * g[1])
        vx, vy, vz = np.meshgrid(*[np.arange(k * 8, min(n, k * 8 + 8)) for k, n in zip((tx, ty, tz), nV)],
                                 indexing="ij")
        vx, vy, vz = vx.reshape(-1), vy.reshape(-1), vz.reshape(-1)
        p = xyz_vol[ids].astype(np.float64)
        c = conic_opacity[ids].astype(np.float64)
        dx, dy, dz = (p[:, k, None] - (v[None] + 0.5) for k, v in enumerate((vx, vy, vz)))
        terms = [0.5 * c[:, 0, None] * dx * dx, 0.5 * c[:, 3, None] * dy * dy, 0.5 * c[:, 5, None] * dz * dz,
                 c[:, 1, None] * dx * dy, c[:, 2, None] * dx * dz, c[:, 4, None] * dy * dz]
        power = -sum(terms)
        Lp = sum(np.abs(x) for x in terms)
        alpha = rho_all[ids, None] * np.exp(np.minimum(power, 0.0))
        dec, border = _tile_terms(alpha, power, Lp, VALPHA_CUT, VBAND)
        _accumulate(out, (vx, vy, vz), alpha, Lp + np.abs(lw_all[ids])[:, None], dec, border, np.iinfo(np.int64).max,
                    flags, ids)
    return out


def bar(st):
    return C_BAR * U * st["absw"] + U * st["n_chain"] * st["abs_all"] + 0.5 * st["border"]


def ratio(got, st):
    """|got - S64| / bar per element: <= 1 passes.  An element no pair reaches has a zero bar: it must be exactly 0."""
    return np.abs(np.asarray(got, np.float64) - st["S64"]) / (bar(st) + 1e-300)


def old_bar_ratio(got, st):
    """The suite's image bar, 1e-5 max|image| + 1e-7, as a ratio (<= 1 passes)."""
    return np.abs(np.asarray(got, np.float64) - st["S64"]).max() / (1e-5 * np.abs(st["S64"]).max() + 1e-7)


def judged(st):
    """Elements some pair reaches."""
    return (st["n"] + st["n_border"]) > 0


def faint(st):
    return judged(st) & (st["S64"] < FAINT * st["S64"].max())
