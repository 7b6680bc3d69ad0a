"""A float64 statement of the rasterizer's and the voxelizer's backwards, per Gaussian, to judge the float32 kernels
element by element.  The rasterizer is described here; the voxelizer's statement (voxel_moments, make_voxel_chain)
follows the same plan with 10 moments over its tile cube.

Two layers, as the kernels split the work:

* Screen space (raster_moments).  X-ray rendering is additive, so a Gaussian's gradient depends on its own
  (Gaussian, pixel) pairs only: every pixel of the Gaussian's tile rectangle, alpha and both skip rules of the
  reference evaluated in float64 from the forward's own stage outputs (xy, conic_opacity, mu, radii).  Per Gaussian it
  returns the six moments m = (S0, Sx, Sy, Sxx, Sxy, Syy) = sums over the contributing pairs of t (1, dx, dy, dx^2,
  dx dy, dy^2) with t = dL/dpixel * G, and the same sums over |t f| (the absolute moments, each pair weighted for the
  rounding of its power, POWER_WEIGHT).
* The chain (make_chain).  The reference's backward equations from the moments to dL/dmean2D, dL/dopacity, dL/dmu,
  dL/dmean3D, dL/dcov3D, dL/dscale and dL/drot, in float64 torch, with what the kernels deliberately keep: the 1e-7
  regularisations (of det2^2, mu and the projective w), x_grad_mul / y_grad_mul at the 1.3 tanfov clamp, the
  parallel-beam constant J, scale_modifier (dL/dscale is with respect to the modified scale, as the reference's) and
  the cov3D_precomp path.
* The matrix gradients (make_pose_chain).  The same chain (_chain_core) continued to one Gaussian's contribution to
  dL/dviewmatrix and dL/dprojmatrix in the layout of the rasterizer's pose rows, with the same frozen decisions; its
  inputs are those of make_chain and PNK more rounding knobs.  tests/test_pose_grad_float64_cpu.py checks it against
  autograd of a float64 forward and against central differences where the clamp is active.

The bar (reference).  The chain is linear in the moments.  A float32 kernel that sums the pairs and runs the chain
well is off from y64 by a small multiple of u = 2^-24 of
    |dy/dm| |m|_abs          (the sums: each term rounded, no cancellation beyond that of the terms themselves)
  + |dy/dp| |p|              (the chain: its inputs p -- the cloud, the stage outputs, the two matrices and unit
                              factors on its main intermediates, NK -- each perturbed by a unit roundoff: what the
                              float32 chain's own rounding looks like)
so the test is |y_kernel - y64| <= C_BAR u (|dy/dm| |m|_abs + |dy/dp| |p|) + band_y, one constant C_BAR for every
output.  band_y holds the pairs neither side can decide (BAND below).

A Gaussian whose 2-D covariance is nearly singular (det2 = a d - b^2 cancelling, COND_MAX) has an ill-conditioned
chain: it is not held to this bar, but counted (the oracle tests still cover it).

Measured on an H100 (700 W) with tests/test_grad_float64_gpu.py: about the tile's column 0, the backward's exact path
(sub-pixel conics) was off by up to 496x this bar in dL/dmean2D, 261x in dL/dmean3D, 28x in dL/dscale, 5.7x in
dL/drot and 4.6x in dL/dcov3D; with the
moments about the column nearest the centre, the worst element over every case is 0.29x (fast path) and 0.08x (exact).
The voxelizer's fast path keeps its z moments about the tile's voxel 0 (dz0 <= 8): its worst element over the voxel
sweeps (dz0 across the whole tile, fast and exact conics) and trained clouds is 0.87x, so it is left as it is.
"""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -24
C_BAR = 64.0
# A pair is borderline when its float64 alpha lies within BAND (relative) of the 1e-5 cut, or its power within BAND of
# 0 relative to the power's terms.  The kernels decide such pairs with the reference's float32 expression (or with
# ex2.approx, relative error 2^-22, on a q whose rounding is a few u of its terms, |q| <= 17 + log2 w for a
# contributing pair): together well under 1e-6 of alpha, so outside 1e-5 the float32 and the float64 decisions agree.
# A borderline pair enters the moments at half weight and half of its absolute terms enter the bar.
BAND = 1e-5
ALPHA_CUT = 1e-5
# A float32 kernel evaluates each pair's power from float32 terms: t carries a relative error of a few u times the
# power's terms L = |A dx^2 / 2| + |C dy^2 / 2| + |B dx dy| (up to ~20 at the cut).  The absolute moments weight each
# pair by 1 + L / POWER_WEIGHT: C_BAR u / POWER_WEIGHT = 4 u per unit of L.
POWER_WEIGHT = 16.0
COND_MAX = 1e3                     # (a d + b^2) / |a d - b^2| of the 2-D covariance above this: not held to the bar
LOG2E = 1.4426950408889634
OUT_KEYS = ("dL_dmean2D", "dL_dopacity", "dL_dmu", "dL_dmean3D", "dL_dcov3D", "dL_dscale", "dL_drot")
OUT_DIMS = {"dL_dmean2D": 2, "dL_dopacity": 1, "dL_dmu": 1, "dL_dmean3D": 3, "dL_dcov3D": 6, "dL_dscale": 3,
            "dL_drot": 4}
# mean, scale, rot, cov3D, conic, rho, mu, view, proj, then NK rounding knobs (all 1): factors on the chain's float32
# intermediates M (9), Sigma (6), hat (6), det2, det3 and mu, so that |dy/dknob| is what one rounding of each costs
NK = 9 + 6 + 6 + 3
NP = 3 + 3 + 4 + 6 + 3 + 1 + 1 + 16 + 16 + NK


def _f32(x):
    return np.float32(x)


def tile_rect(px, py, radius, W, H):
    """The preprocess's tile rectangle (x0, y0, x1, y1) in tiles, float32 as the forward forms it."""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    rf, x, y, s = _f32(radius), _f32(px), _f32(py), _f32(0.0625)
    x0 = min(gx, max(0, int(_f32(x - rf) * s)))
    y0 = min(gy, max(0, int(_f32(y - rf) * s)))
    x1 = min(gx, max(0, int(_f32(_f32(_f32(x + rf) + _f32(16.0)) + _f32(-1.0)) * s)))
    y1 = min(gy, max(0, int(_f32(_f32(_f32(y + rf) + _f32(16.0)) + _f32(-1.0)) * s)))
    return x0, y0, x1, y1


def raster_moments(xy, conic_opacity, mu, radii, dL):
    """Float64 moments of every Gaussian from the forward's stage outputs -> dict of [P, 6] arrays:
    m (signed, borderline pairs at half weight), a (absolute, decided pairs), b (absolute, borderline pairs),
    and [P] arrays n_pairs, n_border, n_near_cut (pixels within 1e-4 of the cut: the rows the fast path redoes)."""
    H, W = dL.shape
    P = len(radii)
    m = np.zeros((P, 6)); a = np.zeros((P, 6)); b = np.zeros((P, 6))
    n_pairs = np.zeros(P, np.int64); n_border = np.zeros(P, np.int64); n_near = np.zeros(P, np.int64)
    dL = dL.astype(np.float64)
    for g in np.nonzero(radii > 0)[0]:
        x0, y0, x1, y1 = tile_rect(xy[g, 0], xy[g, 1], radii[g], W, H)
        if x1 <= x0 or y1 <= y0:
            continue
        xs = np.arange(16 * x0, min(16 * x1, W), dtype=np.float64)
        ys = np.arange(16 * y0, min(16 * y1, H), dtype=np.float64)
        dx = float(xy[g, 0]) - xs[None, :]
        dy = float(xy[g, 1]) - ys[:, None]
        A, B, C, rho = (float(v) for v in conic_opacity[g])
        w = rho * float(mu[g])
        ta, tc, tb = 0.5 * A * dx * dx, 0.5 * C * dy * dy, B * dx * dy
        power = -(ta + tc) - tb
        G = np.exp(np.minimum(power, 0.0))
        alpha = w * G
        inside = (power <= 0.0) & (alpha >= ALPHA_CUT)
        border = (np.abs(alpha - ALPHA_CUT) <= BAND * ALPHA_CUT) | (
            np.abs(power) <= BAND * (np.abs(ta) + np.abs(tc) + np.abs(tb)) + 1e-300)
        border &= (alpha >= (1 - BAND) * ALPHA_CUT)      # a pair far below the cut never contributes
        sl = dL[int(ys[0]):int(ys[-1]) + 1, int(xs[0]):int(xs[-1]) + 1]
        t = sl * np.exp(power)                           # G at a pair with power > 0 only matters when borderline
        f = [np.ones_like(dx * dy), dx + 0 * dy, dy + 0 * dx, dx * dx + 0 * dy, dx * dy, dy * dy + 0 * dx]
        dec = inside & ~border
        wt = 1.0 + (np.abs(ta) + np.abs(tc) + np.abs(tb)) / POWER_WEIGHT
        for k in range(6):
            tf = t * f[k]
            m[g, k] = tf[dec].sum() + 0.5 * tf[border].sum()
            a[g, k] = (np.abs(tf) * wt)[dec].sum()
            b[g, k] = np.abs(tf[border]).sum()
        n_pairs[g] = int(dec.sum())
        n_border[g] = int(border.sum())
        n_near[g] = int((np.abs(alpha / ALPHA_CUT - 1.0) <= 1e-4).sum())
    return dict(m=m, a=a, b=b, n_pairs=n_pairs, n_border=n_border, n_near_cut=n_near)


# ---- the chain -----------------------------------------------------------------------------------------------------
def _quat_rot(q):
    import torch

    r, x, y, z = q[0], q[1], q[2], q[3]
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)]),
        torch.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)]),
        torch.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)])])


def _sym6(c):
    import torch

    return torch.stack([torch.stack([c[0], c[1], c[2]]), torch.stack([c[1], c[3], c[4]]),
                        torch.stack([c[2], c[4], c[5]])])


def _six(S):
    """Upper triangle (00, 01, 02, 11, 12, 22) of a symmetric 3x3."""
    import torch

    return torch.stack([S[0, 0], S[0, 1], S[0, 2], S[1, 1], S[1, 2], S[2, 2]])


def _adj_det(S):
    """Cofactor matrix and determinant of a symmetric 3x3, as polynomials (no pivoting: smooth for forward-mode)."""
    import torch

    a, b, c, d, e, f = S[0, 0], S[0, 1], S[0, 2], S[1, 1], S[1, 2], S[2, 2]
    K = torch.stack([torch.stack([d * f - e * e, c * e - b * f, b * e - c * d]),
                     torch.stack([c * e - b * f, a * f - c * c, b * c - a * e]),
                     torch.stack([b * e - c * d, b * c - a * e, a * d - b * b])])
    return K, a * K[0, 0] + b * K[0, 1] + c * K[0, 2]


def _sigma6(s, q):
    R = _quat_rot(q)
    return _six(R @ (s * s).diag() @ R.T)


def _chain_core(m, p, W, H, tanfovx, tanfovy, mode, scale_modifier, precomp, eps):
    """The reference's backward of one Gaussian from its moments m to dL/dhat and dL/dt (zero in parallel beam), and
    the intermediates the 3-D mean and the matrix gradients go on from, as a dict.  eps: the backward's two 1e-7
    regularisations, of det2^2 and of mu (0 gives the exact derivative of the frozen forward)."""
    import torch

    hx, hy = W / (2.0 * tanfovx), H / (2.0 * tanfovy)
    S0, Sx, Sy, Sxx, Sxy, Syy = m[0], m[1], m[2], m[3], m[4], m[5]
    mean, sc, q, c6 = p[0:3], p[3:6], p[6:10], p[10:16]
    A, B, Cc, rho, mu = p[16], p[17], p[18], p[19], p[20]
    view, proj = p[21:37], p[37:53]
    kM, kV, kh, kd2, kd3, kmu = p[53:62].reshape(3, 3), p[62:68], p[68:74], p[74], p[75], p[76]
    w = rho * mu
    g2x = w * (-A * Sx - B * Sy) * (0.5 * W)
    g2y = w * (-Cc * Sy - B * Sx) * (0.5 * H)
    dcx, dcy, dcz = -0.5 * w * Sxx, -w * Sxy, -0.5 * w * Syy
    dmu = rho * S0
    dop = mu * S0
    s_eff = scale_modifier * sc
    V = _sym6(kV * (c6 if precomp else _sigma6(s_eff, q)))
    V4 = view.reshape(4, 4)                          # V4[k][r] = view[4k + r]
    Rv = V4[:3, :3].T                                # t = Rv mean + V4[3, :3]
    t = Rv @ mean + V4[3, :3]
    tx, ty, tz = t[0], t[1], t[2]
    zero, one = torch.zeros_like(tz), torch.ones_like(tz)
    if mode == 1:
        limx, limy = 1.3 * tanfovx, 1.3 * tanfovy
        txtz, tytz = tx / tz, ty / tz
        xgm = ((txtz >= -limx) & (txtz <= limx)).to(t.dtype)
        ygm = ((tytz >= -limy) & (tytz <= limy)).to(t.dtype)
        tx = tz * txtz.clamp(-limx, limx)
        ty = tz * tytz.clamp(-limy, limy)
        l = torch.sqrt(tx * tx + ty * ty + tz * tz)
        J = torch.stack([torch.stack([hx / tz, zero, -hx * tx / (tz * tz)]),
                         torch.stack([zero, hy / tz, -hy * ty / (tz * tz)]),
                         torch.stack([tx / l, ty / l, tz / l])])
    else:
        J = torch.stack([torch.stack([hx + zero, zero, zero]), torch.stack([zero, hy + zero, zero]),
                         torch.stack([zero, zero, one])])
    M = kM * (J @ Rv)
    hat = _sym6(kh * _six(M @ V @ M.T))
    a, b, d = hat[0, 0], hat[0, 1], hat[1, 1]
    det2 = kd2 * (a * d - b * b)
    K, det3 = _adj_det(hat)
    det3 = kd3 * det3
    musq = 2 * math.pi * det3 / det2
    muv = kmu * torch.sqrt(torch.clamp(musq, min=0.0))
    inv = 1.0 / (det2 * det2 + eps)
    adj = torch.stack([torch.stack([d, -b]), torch.stack([-b, a])])
    Gc = torch.stack([torch.stack([dcx, 0.5 * dcy]), torch.stack([0.5 * dcy, dcz])])
    T = adj @ Gc @ adj
    pi_mu = math.pi / (muv + eps)
    ratio = det3 / det2
    ddet3 = torch.stack([K[0, 0], 2 * K[0, 1], 2 * K[0, 2], K[1, 1], 2 * K[1, 2], K[2, 2]])
    ddet2 = torch.stack([d, -2 * b, zero, a, zero, zero])
    dh = pi_mu * (ddet3 - ratio * ddet2) / det2 * dmu
    dh = dh + torch.stack([-inv * T[0, 0], -inv * (T[0, 1] + T[1, 0]), zero, -inv * T[1, 1], zero, zero])
    D = torch.stack([torch.stack([dh[0], 0.5 * dh[1], 0.5 * dh[2]]),
                     torch.stack([0.5 * dh[1], dh[3], 0.5 * dh[4]]),
                     torch.stack([0.5 * dh[2], 0.5 * dh[4], dh[5]])])
    dt = torch.zeros_like(mean)
    if mode == 1:
        dJ = 2.0 * (D @ M @ V) @ Rv.T                # dL/dJ = (dL/dM) Rv^T, dL/dM = 2 D M V
        rz = 1.0 / tz
        rl, rl3 = 1.0 / l, 1.0 / (l * l * l)
        tdot = tx * dJ[2, 0] + ty * dJ[2, 1] + tz * dJ[2, 2]
        dtx = xgm * (-hx * rz * rz * dJ[0, 2] + rl * dJ[2, 0] - rl3 * tx * tdot)
        dty = ygm * (-hy * rz * rz * dJ[1, 2] + rl * dJ[2, 1] - rl3 * ty * tdot)
        dtz = (-rz * rz * (hx * dJ[0, 0] + hy * dJ[1, 1]) + 2 * rz ** 3 * (hx * tx * dJ[0, 2] + hy * ty * dJ[1, 2])
               + rl * dJ[2, 2] - rl3 * tz * tdot)
        dt = torch.stack([dtx, dty, dtz])
    P4 = proj.reshape(4, 4)                          # P4[k][r] = proj[4k + r]
    hom = P4[:3, :].T @ mean + P4[3, :]
    m_w = 1.0 / (hom[3] + 1e-7)                      # the forward's own 1e-7 (not a regularisation of the backward)
    return dict(g2x=g2x, g2y=g2y, dop=dop, dmu=dmu, mean=mean, sc=sc, q=q, s_eff=s_eff, V=V, Rv=Rv, J=J, M=M, D=D,
                dt=dt, P4=P4, hom=hom, m_w=m_w)


def make_chain(W, H, tanfovx, tanfovy, mode, scale_modifier=1.0, precomp=False):
    """chain(m [6], p [NP]) -> y (the outputs of OUT_KEYS concatenated), for one Gaussian, float64 torch."""
    import torch
    from torch.func import grad

    def chain(m, p):
        c = _chain_core(m, p, W, H, tanfovx, tanfovy, mode, scale_modifier, precomp, 1e-7)
        g2x, g2y, M, D, P4, m_w, q, s_eff = c["g2x"], c["g2y"], c["M"], c["D"], c["P4"], c["m_w"], c["q"], c["s_eff"]
        G3 = M.T @ D @ M                                 # dL/dSigma, full symmetric
        dcov = torch.stack([G3[0, 0], 2 * G3[0, 1], 2 * G3[0, 2], G3[1, 1], 2 * G3[1, 2], G3[2, 2]])
        dmean = c["Rv"].T @ c["dt"]
        mul1, mul2 = c["hom"][0] * m_w * m_w, c["hom"][1] * m_w * m_w
        dmean = dmean + torch.stack([(P4[k, 0] * m_w - P4[k, 3] * mul1) * g2x + (P4[k, 1] * m_w - P4[k, 3] * mul2) * g2y
                                     for k in range(3)])
        if precomp:
            ds, dr = torch.zeros(3, dtype=m.dtype), torch.zeros(4, dtype=m.dtype)
        else:
            ds = grad(lambda s: (dcov * _sigma6(s, q)).sum())(s_eff)
            dr = grad(lambda qq: (dcov * _sigma6(s_eff, qq)).sum())(q)
        return torch.cat([torch.stack([g2x, g2y, c["dop"], c["dmu"]]), dmean, dcov, ds, dr])

    return chain


# ---- the matrix gradients ------------------------------------------------------------------------------------------
# One Gaussian's contribution to dL/dviewmatrix and dL/dprojmatrix, laid out as the rasterizer's pose rows (POSE_N = 24
# floats, include/r2x.h): pose[3a + b] = dL/dview[4a + b] (a < 4: a = 3 is the translation column), pose[12 + 3a + j]
# = dL/dproj[4a + (0, 1, 3)[j]].  With the chain's D = dL/dhat and dt = dL/dt (x_grad_mul / y_grad_mul, J at the
# clamped t, the parallel-beam constant J):
#     t_b = sum_a view[4a + b] p_a + view[12 + b]          -> dt_b p_a,  dt_b
#     M[i][a] = sum_b J[i][b] view[4a + b]                 -> sum_i (2 D M Sigma)[i][a] J[i][b]
#     ndc = (hom_x, hom_y) / (hom_w + 1e-7), hom = P^T [p, 1] -> g2x m_w, g2y m_w, -(g2x hom_x + g2y hom_y) m_w^2
# times [p, 1]_a.  Four more rounding knobs (PNK, after the chain's NP inputs) are unit factors on the two view terms
# and on m_w and the w term: the float32 sums of the kernel round each of them.
POSE_N = 24
PNK = 4
POSE_KEYS = ("view_rot", "view_trans", "proj")
POSE_SLICES = {"view_rot": slice(0, 9), "view_trans": slice(9, 12), "proj": slice(12, 24)}


def make_pose_chain(W, H, tanfovx, tanfovy, mode, scale_modifier=1.0, precomp=False, eps=1e-7):
    """chain(m [6], p [NP + PNK]) -> the POSE_N matrix-gradient contributions of one Gaussian, float64 torch.
    eps = 0: the exact derivative of the frozen forward (no regularisations)."""
    import torch

    def chain(m, p):
        c = _chain_core(m, p[:NP], W, H, tanfovx, tanfovy, mode, scale_modifier, precomp, eps)
        kt, kM, kw, kgw = p[NP], p[NP + 1], p[NP + 2], p[NP + 3]
        mean, dt, J = c["mean"], c["dt"], c["J"]
        dM = 2.0 * (c["D"] @ c["M"] @ c["V"])           # dL/dM
        rot = kt * (mean[:, None] * dt[None, :]) + kM * (dM.T @ J)    # [a][b]
        m_w = kw * c["m_w"]
        hom = c["hom"]
        gw = kgw * -(c["g2x"] * hom[0] + c["g2y"] * hom[1]) * m_w * m_w
        ph = torch.cat([mean, torch.ones_like(mean[:1])])
        pj = ph[:, None] * torch.stack([c["g2x"] * m_w, c["g2y"] * m_w, gw])[None, :]    # [a][j]
        return torch.cat([rot.reshape(9), dt, pj.reshape(12)])

    return chain


def pose_chain_inputs(*args):
    """chain_inputs(...) followed by the PNK pose knobs (all 1): [P, NP + PNK]."""
    p = chain_inputs(*args)
    return np.concatenate([p, np.ones((len(p), PNK))], 1)


def chain_inputs(means, scales, rots, cov3D, conic_opacity, mu, view, proj):
    """[P, NP] float64 chain inputs (missing scales / rots / cov3D: zeros)."""
    P = len(means)
    z = lambda k: np.zeros((P, k))
    cols = [means, z(3) if scales is None else scales, z(4) if rots is None else rots, z(6) if cov3D is None else cov3D,
            conic_opacity[:, :3], conic_opacity[:, 3:4], np.asarray(mu).reshape(P, 1),
            np.tile(np.asarray(view, np.float64).reshape(1, 16), (P, 1)),
            np.tile(np.asarray(proj, np.float64).reshape(1, 16), (P, 1)), np.ones((P, NK))]
    return np.concatenate([np.asarray(c, np.float64).reshape(P, -1) for c in cols], 1)


def reference(mom, p, chain, idx):
    """For the Gaussians idx: y64 [n, ny], the bar [n, ny] (without C_BAR u) and the band [n, ny]."""
    import torch
    from torch.func import jacfwd, vmap

    m = torch.tensor(mom["m"][idx], dtype=torch.float64)
    pt = torch.tensor(p[idx], dtype=torch.float64)
    y = vmap(chain)(m, pt)
    Jm = vmap(jacfwd(chain, argnums=0))(m, pt).abs()    # exact: the chain is linear in m
    Jp = vmap(jacfwd(chain, argnums=1))(m, pt).abs()
    a = torch.tensor(mom["a"][idx]); b = torch.tensor(mom["b"][idx])
    bar = (Jm @ a[:, :, None])[..., 0] + (Jp @ pt.abs()[:, :, None])[..., 0]
    band = 0.5 * (Jm @ b[:, :, None])[..., 0]
    return y.numpy(), bar.numpy(), band.numpy()


def split(y):
    """[n, ny] -> dict of OUT_KEYS."""
    out, o = {}, 0
    for k in OUT_KEYS:
        out[k] = y[:, o:o + OUT_DIMS[k]]
        o += OUT_DIMS[k]
    return out


def kernel_rows(g, idx):
    """The kernel's (or oracle's) gradients of the Gaussians idx, concatenated in the chain's output order."""
    return np.concatenate([np.asarray(g[k], np.float64).reshape(len(g[k]), -1)[idx][:, :OUT_DIMS[k]]
                           for k in OUT_KEYS], 1)


def cond2(conic_opacity):
    """(a d + b^2) / |a d - b^2| of the 2-D covariance, from its conic (the same ratio for the inverse)."""
    A, B, C = (conic_opacity[:, k].astype(np.float64) for k in range(3))
    return (A * C + B * B) / np.maximum(np.abs(A * C - B * B), 1e-300)


def compare(y_got, y64, bar, band):
    """Per element |got - y64| / (C_BAR u bar + band): <= 1 passes."""
    return np.abs(y_got - y64) / (C_BAR * U * bar + band + 1e-300)


def fast_path(conic_opacity, mu):
    """The preprocess's choice of render path (fast = forward differences) from the stage outputs, as it makes it."""
    co = conic_opacity.astype(np.float32)
    conx, cony, conz, rho = co[:, 0], co[:, 1], co[:, 2], co[:, 3]
    w = (rho * mu.astype(np.float32)).astype(np.float32)
    A2 = (conx * np.float32(0.5 * LOG2E)).astype(np.float32)
    with np.errstate(divide="ignore"):
        lw = np.where(w > 0, np.log2(w.astype(np.float64)), -np.inf).astype(np.float32)
    pd = (conx > 0) & (conz > 0) & ((conx * conz - cony * cony).astype(np.float32) > np.float32(1e-4) * conx * conz)
    return ~(w > 0) | (pd & (A2 <= 2) & (lw <= 20) & (lw >= -100))


# ---- the voxelizer ---------------------------------------------------------------------------------------------------
# The voxelizer's backward, stated the same way: 10 moments per Gaussian, (S0, Sx, Sy, Sz, Sxx, Sxy, Sxz, Syy, Syz, Szz)
# over the voxels of its tile cube, d = xyz_vol - (voxel index + 1/2), cut alpha = rho G >= 1e-6.  The voxelizer's
# backward decides every pair with its own float32 q (no reference fall-back), whose rounding is a few u of the power's
# terms (up to ~35 at the cut): VBAND = 1e-5 relative, as BAND, is wide enough for that and for ex2.approx.
VALPHA_CUT = 1e-6
VBAND = 1e-5
VOUT_KEYS = ("dL_dopacity", "dL_dmean3D", "dL_dcov3D", "dL_dscale", "dL_drot")
VOUT_DIMS = {"dL_dopacity": 1, "dL_dmean3D": 3, "dL_dcov3D": 6, "dL_dscale": 3, "dL_drot": 4}
# scale, rot, cov3D, rho, then VNK rounding knobs: factors on the voxel-space covariance (6) and its determinant
VNK = 6 + 1
VNP = 3 + 4 + 6 + 1 + VNK


def voxel_cube(xyz, rx, ry, rz, nV):
    """The preprocess's tile cube (x0, y0, z0, x1, y1, z1) in 8-voxel tiles, float32 as the forward forms it."""
    out = []
    for p, r, n in zip(xyz, (rx, ry, rz), nV):
        g = (n + 7) // 8
        p, r, s = _f32(p), _f32(r), _f32(0.125)
        lo = min(g, max(0, int(_f32(p - r) * s)))
        hi = min(g, max(0, int(_f32(_f32(_f32(p + r) + _f32(8.0)) + _f32(-1.0)) * s)))
        out.append((lo, hi))
    return [o[0] for o in out] + [o[1] for o in out]


def voxel_moments(xyz_vol, conic_opacity, radii, nV, dL):
    """Float64 moments of every Gaussian from the voxelizer forward's stage outputs (radii = (rx, ry, rz) arrays)
    -> dict of [P, 10] arrays m, a, b and [P] arrays n_pairs, n_border (as raster_moments)."""
    rx, ry, rz = radii
    P = len(rx)
    m = np.zeros((P, 10)); a = np.zeros((P, 10)); b = np.zeros((P, 10))
    n_pairs = np.zeros(P, np.int64); n_border = np.zeros(P, np.int64)
    dL = dL.astype(np.float64)
    for g in np.nonzero((rx > 0) & (ry > 0) & (rz > 0))[0]:
        x0, y0, z0, x1, y1, z1 = voxel_cube(xyz_vol[g], rx[g], ry[g], rz[g], nV)
        if x1 <= x0 or y1 <= y0 or z1 <= z0:
            continue
        ax = [np.arange(8 * lo, min(8 * hi, n), dtype=np.float64) for lo, hi, n in
              ((x0, x1, nV[0]), (y0, y1, nV[1]), (z0, z1, nV[2]))]
        dx = float(xyz_vol[g, 0]) - (ax[0][:, None, None] + 0.5)
        dy = float(xyz_vol[g, 1]) - (ax[1][None, :, None] + 0.5)
        dz = float(xyz_vol[g, 2]) - (ax[2][None, None, :] + 0.5)
        c = [float(v) for v in conic_opacity[g]]
        terms = [0.5 * c[0] * dx * dx, 0.5 * c[3] * dy * dy, 0.5 * c[5] * dz * dz, c[1] * dx * dy, c[2] * dx * dz,
                 c[4] * dy * dz]
        power = -sum(terms)
        L = sum(np.abs(t) for t in terms)
        alpha = c[6] * np.exp(np.minimum(power, 0.0))
        inside = (power <= 0.0) & (alpha >= VALPHA_CUT)
        border = (np.abs(alpha - VALPHA_CUT) <= VBAND * VALPHA_CUT) | (np.abs(power) <= VBAND * L + 1e-300)
        border &= alpha >= (1 - VBAND) * VALPHA_CUT
        sl = dL[int(ax[0][0]):int(ax[0][-1]) + 1, int(ax[1][0]):int(ax[1][-1]) + 1, int(ax[2][0]):int(ax[2][-1]) + 1]
        t = sl * np.exp(power)
        one = np.ones_like(dx * dy * dz)
        f = [one, dx * one, dy * one, dz * one, dx * dx * one, dx * dy * one, dx * dz * one, dy * dy * one,
             dy * dz * one, dz * dz * one]
        dec = inside & ~border
        wt = 1.0 + L / POWER_WEIGHT
        for k in range(10):
            tf = t * f[k]
            m[g, k] = tf[dec].sum() + 0.5 * tf[border].sum()
            a[g, k] = (np.abs(tf) * wt)[dec].sum()
            b[g, k] = np.abs(tf[border]).sum()
        n_pairs[g] = int(dec.sum())
        n_border[g] = int(border.sum())
    return dict(m=m, a=a, b=b, n_pairs=n_pairs, n_border=n_border)


def make_voxel_chain(nV, sV, scale_modifier=1.0, precomp=False):
    """chain(m [10], p [VNP]) -> y (the outputs of VOUT_KEYS concatenated), one Gaussian, float64 torch: the
    reference's voxelizer backward with its 1e-7 regularisation of det^2, the mean gradient times dVoxel (as the
    reference's), scale_modifier and the cov3D_precomp path."""
    import torch
    from torch.func import grad

    dv = [float(np.float32(s) / np.float32(n)) for s, n in zip(sV, nV)]
    Dm = torch.diag(torch.tensor([1.0 / d for d in dv], dtype=torch.float64))
    dvt = torch.tensor(dv, dtype=torch.float64)

    def chain(m, p):
        S0 = m[0]
        S1 = m[1:4]
        g6 = -p[13] * torch.stack([0.5 * m[4], m[5], m[6], 0.5 * m[7], m[8], 0.5 * m[9]])
        sc, q, c6, rho = p[0:3], p[3:7], p[7:13], p[13]
        kS, kdet = p[14:20], p[20]
        s_eff = scale_modifier * sc
        Sig = _sym6(c6 if precomp else _sigma6(s_eff, q))
        Sv = _sym6(kS * _six(Dm @ Sig @ Dm))
        K, det0 = _adj_det(Sv)
        det = kdet * det0
        inv = K / det0
        dmean = rho * -(inv @ S1) * dvt
        Gf = torch.stack([torch.stack([g6[0], 0.5 * g6[1], 0.5 * g6[2]]),
                          torch.stack([0.5 * g6[1], g6[3], 0.5 * g6[4]]),
                          torch.stack([0.5 * g6[2], 0.5 * g6[4], g6[5]])])
        dSv = -(K @ Gf @ K) / (det * det + 1e-7)
        dS = Dm @ dSv @ Dm
        dcov = torch.stack([dS[0, 0], 2 * dS[0, 1], 2 * dS[0, 2], dS[1, 1], 2 * dS[1, 2], dS[2, 2]])
        if precomp:
            ds, dr = torch.zeros(3, dtype=m.dtype), torch.zeros(4, dtype=m.dtype)
        else:
            ds = grad(lambda s: (dcov * _sigma6(s, q)).sum())(s_eff)
            dr = grad(lambda qq: (dcov * _sigma6(s_eff, qq)).sum())(q)
        return torch.cat([S0[None], dmean, dcov, ds, dr])

    return chain


def voxel_chain_inputs(scales, rots, cov3D, conic_opacity):
    P = len(conic_opacity)
    z = lambda k: np.zeros((P, k))
    cols = [scales, z(4) if rots is None else rots, z(6) if cov3D is None else cov3D, conic_opacity[:, 6:7],
            np.ones((P, VNK))]
    return np.concatenate([np.asarray(c, np.float64).reshape(P, -1) for c in cols], 1)


def voxel_split(y):
    out, o = {}, 0
    for k in VOUT_KEYS:
        out[k] = y[:, o:o + VOUT_DIMS[k]]
        o += VOUT_DIMS[k]
    return out


def voxel_kernel_rows(g, idx):
    return np.concatenate([np.asarray(g[k], np.float64).reshape(len(g[k]), -1)[idx] for k in VOUT_KEYS], 1)


def voxel_cond(cov3D, nV, sV):
    """(sum of |terms| of det) / |det| of the voxel-space covariance: above COND_MAX not held to the bar."""
    dv = np.array([float(np.float32(s) / np.float32(n)) for s, n in zip(sV, nV)])
    c = np.asarray(cov3D, np.float64)
    a, b, cc = c[:, 0] / dv[0] ** 2, c[:, 1] / (dv[0] * dv[1]), c[:, 2] / (dv[0] * dv[2])
    d, e, f = c[:, 3] / dv[1] ** 2, c[:, 4] / (dv[1] * dv[2]), c[:, 5] / dv[2] ** 2
    terms = [a * d * f, 2 * b * cc * e, a * e * e, f * b * b, d * cc * cc]
    det = terms[0] + terms[1] - terms[2] - terms[3] - terms[4]
    return sum(np.abs(t) for t in terms) / np.maximum(np.abs(det), 1e-300)


def voxel_fast_path(conic_opacity):
    """The voxelizer preprocess's choice of the fast (forward differences along z) backward path."""
    co = conic_opacity.astype(np.float32)
    inv, rho = co[:, :6], co[:, 6]
    m01 = (inv[:, 0] * inv[:, 3] - inv[:, 1] * inv[:, 1]).astype(np.float32)
    det3 = (inv[:, 0] * (inv[:, 3] * inv[:, 5] - inv[:, 4] * inv[:, 4]) - inv[:, 1] * (inv[:, 1] * inv[:, 5] - inv[:, 4] * inv[:, 2])
            + inv[:, 2] * (inv[:, 1] * inv[:, 4] - inv[:, 3] * inv[:, 2])).astype(np.float32)
    pd = (inv[:, 0] > 0) & (inv[:, 3] > 0) & (inv[:, 5] > 0) & (m01 > np.float32(1e-4) * inv[:, 0] * inv[:, 3]) & (
        det3 > np.float32(1e-4) * inv[:, 0] * inv[:, 3] * inv[:, 5])
    F2 = (inv[:, 5] * np.float32(0.5 * LOG2E)).astype(np.float32)
    with np.errstate(divide="ignore"):
        lw = np.where(rho > 0, np.log2(rho.astype(np.float64)), -np.inf)
    return ~(rho > 0) | (pd & (F2 <= 2) & (lw <= 20) & (lw >= -100))
