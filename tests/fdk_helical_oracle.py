"""Float64 NumPy statement of the helical FDK that `r2_gaussian_b200.fdk.fdk(helical=True)` runs on the GPU
(r2x_fdk_helical; Tang et al. 2006, "A three-dimensional-weighted cone beam filtered backprojection (CB-FBP) algorithm
for image reconstruction in volumetric CT -- helical scanning", Phys. Med. Biol. 51:855).

TEST INFRASTRUCTURE ONLY: imported by tests/, never by the product package.

  a. Helix (`fdk.helix_views`, which this oracle calls): the views sorted into increasing unwrapped angle beta_v, their
     quadrature intervals dbeta_v, the arc [beta_lo, beta_hi), the source height z_s(beta) = z0 + h beta and the
     rotation centre (c_x, c_y): the source of angle beta sits at (DSO cos beta + c_x, DSO sin beta + c_y, z_s(beta)).
  b. Filter: the plain FDK's cosine weight and ramp filter (tests/fdk_window_oracle.py, any window).
  c. Conjugates of voxel x at view beta: d = x - source in-plane, L = |d|, gamma = the angle from the central ray
     -(cos beta, sin beta) to d, counter-clockwise (so the source at beta + pi + 2 gamma lies on the same line: the
     Parker note's convention); zin = L cos(gamma).  K = {(beta + 2 pi m, zin)} u {(beta + pi + 2 gamma + 2 pi m,
     2 DSO cos^2(gamma) - zin)} over the m with beta_lo <= beta_k < beta_hi (a conjugate whose depth is <= 0 is
     dropped), each at detector row nu_k = (Z - z_s(beta_k)) / (depth_k tan_fovy).  zin <= 0: weight 0.
  d. W_Q(nu) = 0 for |nu| >= 1, else 1 for |nu| <= Q, else cos^2(pi/2 (|nu| - Q) / (1 - Q));
     w = W_Q(nu_0) / sum_K W_Q(nu_k) (0 where W_Q(nu_0) = 0).
  e. vol = sum_v dbeta_v w U^2 Qf_v(px, py), sampled as oracle/fdk_oracle.py's backprojection samples (bilinear,
     0 outside the detector, U = DSO / z_view, 0 for z_view <= 0).
"""
from __future__ import annotations

import math

import numpy as np

import fdk_window_oracle as fwo
from oracle import fdk_oracle


def wq(nu, q: float) -> np.ndarray:
    """Step d's W_Q."""
    a = np.abs(np.asarray(nu, np.float64))
    band = np.cos(0.5 * math.pi * (a - q) / (1.0 - q)) ** 2 if q < 1.0 else np.ones_like(a)
    return np.where(a >= 1.0, 0.0, np.where(a <= q, 1.0, band))


def conjugate_geometry(beta, X, Y, dso: float, c_x: float, c_y: float):
    """(zin, gamma, zc): the view's depth L cos(gamma), the signed fan angle and the conjugate's depth
    2 DSO cos^2(gamma) - zin, at the in-plane points (X, Y)."""
    cb, sb = math.cos(beta), math.sin(beta)
    ddx, ddy = X - (dso * cb + c_x), Y - (dso * sb + c_y)
    zin = -(cb * ddx + sb * ddy)
    sg = sb * ddx - cb * ddy
    gam = np.arctan2(sg, zin)
    l2 = zin * zin + sg * sg
    return zin, gam, 2.0 * dso * zin * zin / np.where(l2 > 0, l2, 1.0) - zin


def candidates(beta, gam, zin, zc, hx):
    """[(beta_k, depth_k)] of step c as lists of broadcast arrays, with a mask of the candidates that exist."""
    arc_turns = int(math.ceil((hx.beta_hi - hx.beta_lo) / (2.0 * math.pi))) + 1
    out = []
    for m in range(-arc_turns, arc_turns + 1):
        for base, depth in ((np.full_like(gam, beta + 2.0 * math.pi * m), zin),
                            (beta + math.pi + 2.0 * gam + 2.0 * math.pi * m, zc)):
            ok = (base >= hx.beta_lo) & (base < hx.beta_hi) & (depth > 0)
            out.append((base, depth, ok))
    return out


def weights(beta, X, Y, Z, hx, dso: float, tany: float, q: float) -> np.ndarray:
    """w(beta, x) of step d at the voxel centres (X, Y, Z)."""
    zin, gam, zc = conjugate_geometry(beta, X, Y, dso, hx.c_x, hx.c_y)
    pos = zin > 0
    zin_s = np.where(pos, zin, 1.0)
    nu0 = (Z - (hx.z0 + hx.h * beta)) / (zin_s * tany)
    w0 = np.where(pos, wq(nu0, q), 0.0)
    total = np.zeros(np.broadcast(X, Y, Z).shape)
    for bk, depth, ok in candidates(beta, gam, zin, zc, hx):
        nu = (Z - (hx.z0 + hx.h * bk)) / (np.where(ok, depth, 1.0) * tany)
        total = total + np.where(ok & pos, wq(nu, q), 0.0)
    return np.where(w0 > 0, w0 / np.where(total > 0, total, 1.0), 0.0)


def sample(qi, vm, pm, dso: float, X, Y, Z) -> np.ndarray:
    """U^2 Qf(px, py) of one view at the voxel centres, as oracle/fdk_oracle.py's backprojection samples it."""
    H, W = qi.shape
    qp = np.pad(qi, ((1, 1), (1, 1)))
    row = fdk_oracle._row
    vm, pm = np.asarray(vm, np.float64).reshape(16), np.asarray(pm, np.float64).reshape(16)
    pw = 1.0 / (row(pm, 3, X, Y, Z) + 1e-7)
    px = ((row(pm, 0, X, Y, Z) * pw + 1.0) * W - 1.0) * 0.5
    py = ((row(pm, 1, X, Y, Z) * pw + 1.0) * H - 1.0) * 0.5
    zv = row(vm, 2, X, Y, Z)
    ok = zv > 0
    U2 = np.where(ok, (dso / np.where(ok, zv, 1.0)) ** 2, 0.0)
    x0, y0 = np.floor(px), np.floor(py)
    fx, fy = px - x0, py - y0
    inside = (x0 >= -1) & (x0 <= W - 1) & (y0 >= -1) & (y0 <= H - 1)
    xi = np.clip(x0, -1, W - 1).astype(np.int64) + 1
    yi = np.clip(y0, -1, H - 1).astype(np.int64) + 1
    s = ((1 - fy) * ((1 - fx) * qp[yi, xi] + fx * qp[yi, xi + 1]) +
         fy * ((1 - fx) * qp[yi + 1, xi] + fx * qp[yi + 1, xi + 1]))
    return np.where(inside, U2 * s, 0.0)


def fdk_helical_scene(projs, angles, scanner_cfg: dict, view_geometry, q: float, name: str = "ram_lak") -> np.ndarray:
    """fdk(projs, angles, scanner_cfg, view_geometry=view_geometry, helical=True, helical_q=q, filter=name) in
    float64 (steps a-e)."""
    from r2_gaussian_b200.fdk import helix_views
    from r2_gaussian_b200.projector import view_table

    hx = helix_views(angles, scanner_cfg, view_geometry)
    angles = np.asarray(angles, np.float64)
    views, table = view_table(angles[hx.order], scanner_cfg, [view_geometry[i] for i in hx.order])
    p = np.asarray(projs, np.float64)[hx.order]
    tanx, tany, dso = float(table[0, 0]), float(table[0, 1]), float(table[0, 4])
    qf = fwo.filter_projections(p, name, tanx, tany, 1, dso)
    xs, ys, zs = fdk_oracle.voxel_centres(scanner_cfg["nVoxel"], scanner_cfg["sVoxel"], scanner_cfg["offOrigin"])
    X, Y, Z = np.meshgrid(xs, ys, zs, indexing="ij")
    vol = np.zeros(X.shape)
    flat = vol.reshape(-1)
    Xf, Yf, Zf = X.reshape(-1), Y.reshape(-1), Z.reshape(-1)
    for i, v in enumerate(views):
        # the voxels the view reaches (|nu_0| < 1); every other voxel has w = 0
        b = float(hx.beta[i])
        zin, _, _ = conjugate_geometry(b, Xf, Yf, dso, hx.c_x, hx.c_y)
        idx = np.nonzero((zin > 0) & (np.abs(Zf - (hx.z0 + hx.h * b)) < np.where(zin > 0, zin, 0.0) * tany))[0]
        if idx.size == 0:
            continue
        x, y, z = Xf[idx], Yf[idx], Zf[idx]
        w = weights(b, x, y, z, hx, dso, tany, q)
        flat[idx] += hx.dbeta[i] * w * sample(qf[i], v.viewmatrix, v.projmatrix, dso, x, y, z)
    return vol


def helix_case(n_views: int, turns: float, travel: float, nvox=(12, 11, 20), ndet=(9, 13), svox=(1.0, 1.0, 2.0),
               sdet=(0.9, 2.6), start: float = 0.3, dso: float = 5.0, dsd: float = 7.0, off=(0.05, -0.04, 0.1)):
    """(scanner, angles, per-view overrides) of a helix: n_views angles over `turns` turns from `start`, the volume
    moved by travel * (i / n - 1/2) along z (as generate_data --helical_travel), scene units."""
    sc = {"mode": "cone", "DSD": dsd, "DSO": dso, "nDetector": list(ndet), "sDetector": list(sdet),
          "nVoxel": list(nvox), "sVoxel": list(svox), "offOrigin": list(off), "offDetector": [0.0, 0.0]}
    angles = start + np.linspace(0.0, 2.0 * math.pi * turns, n_views + 1)[:-1]
    geo = [{"offOrigin": [off[0], off[1], off[2] + travel * (i / n_views - 0.5)]} for i in range(n_views)]
    return sc, angles, geo
