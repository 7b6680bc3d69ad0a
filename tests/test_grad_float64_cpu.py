"""The float64 statements of the rasterizer's and the voxelizer's backwards (grad_float64.py) checked before it judges a kernel: it agrees
with the CPU oracle to within the oracle's own float32 error, its chain is the true derivative of the textbook forward,
and its bar tells a moment sum that cancels from one that does not."""
import numpy as np
import pytest

import grad_float64 as g64
import textbook
import util
from r2_gaussian_b200 import scene

torch = pytest.importorskip("torch")


def dl_ramp(H, W, seed):
    """Positive: a ramp with noise, so that no moment sum cancels."""
    r = np.random.RandomState(seed)
    ys, xs = np.mgrid[0:H, 0:W]
    return (1.0 + 0.5 * (xs + ys) / (W + H) + 0.25 * r.rand(H, W)).astype(np.float32)


def dl_signed(H, W, seed):
    return np.random.RandomState(seed).randn(H, W).astype(np.float32)


def _oracle_case(name, dl_fn, scale_modifier=1.0, precomp=False):
    cloud, view = util.case(name)
    cov = textbook.sigma3(cloud.scales, cloud.rotations)[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].astype(
        np.float32) if precomp else None
    kw = dict(scale_modifier=scale_modifier, cov3D_precomp=cov)
    fwd = util.oracle_raster_forward(cloud, view, **kw)
    dL = dl_fn(view.image_height, view.image_width, 3)
    got = util.oracle_raster_backward(cloud, view, fwd, dL, **kw)
    return cloud, view, fwd, dL, got, cov


@pytest.mark.parametrize("dl_fn", [dl_ramp, dl_signed], ids=["ramp", "signed"])
@pytest.mark.parametrize("name", ["cone_trained_small", "parallel_trained_small", "cone_trained_ragged"])
def test_float64_statement_agrees_with_the_oracle(name, dl_fn):
    cloud, view, fwd, dL, got, _ = _oracle_case(name, dl_fn)
    _check(cloud, view, fwd, dL, got, None, 1.0)


@pytest.mark.parametrize("variant", ["modifier0.5", "modifier1.6", "cov3D_precomp"])
def test_float64_statement_agrees_with_the_oracle_variants(variant):
    mod = {"modifier0.5": 0.5, "modifier1.6": 1.6}.get(variant, 1.0)
    cloud, view, fwd, dL, got, cov = _oracle_case("cone_trained_small", dl_ramp, mod, variant == "cov3D_precomp")
    _check(cloud, view, fwd, dL, got, cov, mod)


def _check(cloud, view, fwd, dL, got, cov, mod):
    mom = g64.raster_moments(fwd["xy"], fwd["conic_opacity"], fwd["mu"], fwd["radii"], dL)
    chain = g64.make_chain(view.image_width, view.image_height, view.tanfovx, view.tanfovy, view.mode, mod,
                           precomp=cov is not None)
    p = g64.chain_inputs(cloud.means, None if cov is not None else cloud.scales,
                         None if cov is not None else cloud.rotations, cov, fwd["conic_opacity"], fwd["mu"],
                         view.viewmatrix, view.projmatrix)
    well = g64.cond2(fwd["conic_opacity"]) <= g64.COND_MAX
    idx = np.nonzero((fwd["radii"] > 0) & (mom["n_pairs"] > 0) & well)[0]
    assert len(idx) >= 100
    y64, bar, band = g64.reference(mom, p, chain, idx)
    r = g64.compare(g64.kernel_rows(got, idx), y64, bar, band)
    assert np.isfinite(r).all()
    worst = {k: float(v.max()) for k, v in g64.split(r).items()}
    print("oracle, worst per output in units of the bar:", {k: f"{v:.3g}" for k, v in worst.items()})
    assert max(worst.values()) <= 1.0, worst


def test_chain_is_the_derivative_of_the_textbook_forward():
    """Where the regularisations are negligible, the chain applied to the moments of a loss equals torch float64
    autograd of the textbook forward's image (the cut and rectangles held fixed as masks)."""
    cloud, view = util.case("cone_trained_small")
    fwd = util.oracle_raster_forward(cloud, view)
    dL = dl_signed(view.image_height, view.image_width, 4)
    W, H = view.image_width, view.image_height
    vis = np.nonzero(fwd["radii"] > 0)[0][:200]
    mom = g64.raster_moments(fwd["xy"][vis], fwd["conic_opacity"][vis], fwd["mu"][vis], fwd["radii"][vis], dL)
    # the float64 forward: the projection restated in torch, the contributing pairs as the masks raster_moments found
    T = lambda a: torch.tensor(np.asarray(a, np.float64)[vis], requires_grad=True)
    means, scales, rots, dens = T(cloud.means), T(cloud.scales), T(cloud.rotations), T(cloud.density)
    view_t = torch.tensor(view.viewmatrix, dtype=torch.float64)
    proj_t = torch.tensor(view.projmatrix, dtype=torch.float64)
    img = _textbook_image_torch(means, scales, rots, dens[:, 0], view_t, proj_t, view, fwd, vis)
    (img * torch.tensor(dL, dtype=torch.float64)).sum().backward()
    chain = g64.make_chain(W, H, view.tanfovx, view.tanfovy, view.mode)
    # the chain on the textbook's own float64 stage values (conic, rho, mu), not the float32 ones
    st = _textbook_stage(means.detach(), scales.detach(), rots.detach(), dens.detach()[:, 0], view_t, proj_t, view)
    co = torch.cat([st["conic"], dens.detach()], 1).numpy()
    mom = g64.raster_moments(st["xy"].numpy(), co, st["mu"].numpy(), fwd["radii"][vis], dL)
    p = g64.chain_inputs(means.detach().numpy(), scales.detach().numpy(), rots.detach().numpy(), None, co,
                         st["mu"].numpy(), view.viewmatrix, view.projmatrix)
    y, _, _ = g64.reference(mom, p, chain, np.arange(len(vis)))
    out = g64.split(y)
    for name, want in (("dL_dmean3D", means.grad), ("dL_dscale", scales.grad), ("dL_drot", rots.grad),
                       ("dL_dopacity", dens.grad)):
        want = want.numpy().reshape(len(vis), -1)
        err = np.abs(out[name] - want).max() / np.abs(want).max()
        assert err <= 1e-6, (name, err)


def _textbook_stage(means, scales, rots, dens, view_t, proj_t, view):
    W, H = view.image_width, view.image_height
    hx, hy = W / (2 * view.tanfovx), H / (2 * view.tanfovy)
    V4 = view_t.reshape(4, 4)
    Rv = V4[:3, :3].T
    t = means @ Rv.T + V4[3, :3]
    P4 = proj_t.reshape(4, 4)
    hom = means @ P4[:3, :] + P4[3, :]
    ndc = hom[:, :2] / (hom[:, 3:4] + 1e-7)
    xy = torch.stack([((ndc[:, 0] + 1) * W - 1) * 0.5, ((ndc[:, 1] + 1) * H - 1) * 0.5], 1)
    tx, ty, tz = t[:, 0], t[:, 1], t[:, 2]
    limx, limy = 1.3 * view.tanfovx, 1.3 * view.tanfovy
    tx = tz * (tx / tz).clamp(-limx, limx)
    ty = tz * (ty / tz).clamp(-limy, limy)
    l = torch.sqrt(tx * tx + ty * ty + tz * tz)
    z = torch.zeros_like(tz)
    J = torch.stack([torch.stack([hx / tz, z, -hx * tx / tz ** 2], -1), torch.stack([z, hy / tz, -hy * ty / tz ** 2], -1),
                     torch.stack([tx / l, ty / l, tz / l], -1)], 1)
    r, x, y, zq = rots[:, 0], rots[:, 1], rots[:, 2], rots[:, 3]
    R = torch.stack([torch.stack([1 - 2 * (y * y + zq * zq), 2 * (x * y - r * zq), 2 * (x * zq + r * y)], -1),
                     torch.stack([2 * (x * y + r * zq), 1 - 2 * (x * x + zq * zq), 2 * (y * zq - r * x)], -1),
                     torch.stack([2 * (x * zq - r * y), 2 * (y * zq + r * x), 1 - 2 * (x * x + y * y)], -1)], 1)
    Sig = R @ torch.diag_embed(scales ** 2) @ R.transpose(1, 2)
    M = J @ Rv
    hat = M @ Sig @ M.transpose(1, 2)
    a, b, d = hat[:, 0, 0], hat[:, 0, 1], hat[:, 1, 1]
    det2 = a * d - b * b
    mu = torch.sqrt(2 * np.pi * torch.linalg.det(hat) / det2)
    return dict(xy=xy, conic=torch.stack([d / det2, -b / det2, a / det2], 1), mu=mu)


def _textbook_image_torch(means, scales, rots, dens, view_t, proj_t, view, fwd, vis):
    W, H = view.image_width, view.image_height
    st = _textbook_stage(means, scales, rots, dens, view_t, proj_t, view)
    img = torch.zeros(H, W, dtype=torch.float64)
    for i, g in enumerate(vis):
        x0, y0, x1, y1 = g64.tile_rect(fwd["xy"][g, 0], fwd["xy"][g, 1], fwd["radii"][g], W, H)
        xs = torch.arange(16 * x0, min(16 * x1, W), dtype=torch.float64)
        ys = torch.arange(16 * y0, min(16 * y1, H), dtype=torch.float64)
        dx = st["xy"][i, 0] - xs[None, :]
        dy = st["xy"][i, 1] - ys[:, None]
        A, B, C = st["conic"][i]
        power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
        alpha = dens[i] * st["mu"][i] * torch.exp(power)
        keep = ((power <= 0) & (alpha >= g64.ALPHA_CUT)).detach()
        img[16 * y0:16 * y0 + len(ys), 16 * x0:16 * x0 + len(xs)] += torch.where(keep, alpha, torch.zeros_like(alpha))
    return img


# ---- sharpness: the bar tells the tile-origin moment shift from the re-centred one ---------------------------------
def _emulate_exact_path(dxb, dyb, A2, B2, C2, dL, gcut, recentre):
    """float32 numpy emulation of the exact path's per-instance moments (Horner per pixel, column moments summed per
    row, then over rows, shifted to dx once): about tile column 0, or about c0 = clamp(rint(dxb), 0, 15)."""
    f = np.float32

    def fma(a, b, c):
        return (a.astype(np.float64) * b + c).astype(f)

    n = len(dxb)
    c0 = np.clip(np.rint(dxb), 0, 15).astype(f) if recentre else np.zeros(n, f)
    S0 = np.zeros(n, f); N1 = np.zeros(n, f); N2 = np.zeros(n, f)
    for ry in range(16):
        dy = (dyb - f(ry)).astype(f)
        bdy = (B2 * dy).astype(f)
        cdy2 = ((C2 * dy).astype(f) * dy).astype(f)
        M0 = np.zeros(n, f); M1 = np.zeros(n, f); M2 = np.zeros(n, f)
        for c in range(16):
            dx = (dxb - f(c)).astype(f)
            G = np.exp2(-fma(dx, fma(A2, dx, bdy), cdy2).astype(np.float64)).astype(f)
            t = np.where(G >= gcut, (dL[:, ry, c] * G).astype(f), f(0))
            cc = (f(c) - c0).astype(f)
            M0 = (M0 + t).astype(f); M1 = fma(t, cc, M1); M2 = fma(t, (cc * cc).astype(f), M2)
        S0 = (S0 + M0).astype(f); N1 = (N1 + M1).astype(f); N2 = (N2 + M2).astype(f)
    d = (dxb - c0).astype(f)
    return S0, fma(d, S0, -N1), fma(d, fma(d, S0, (f(-2) * N1).astype(f)), N2)


@pytest.mark.parametrize("sigma", [0.25, 0.4, 0.6])
def test_bar_separates_tile_origin_moments_from_recentred_ones(sigma):
    """Sub-pixel Gaussians centred at every quarter column of a tile (and just outside it), one tile row of moments:
    the tile-origin shift misses the bar of C_BAR u |m|_abs, the shift about the nearest column meets it."""
    r = np.random.RandomState(int(sigma * 100))
    dxb = np.repeat(np.arange(-2.0, 17.0, 0.25), 4).astype(np.float32)
    n = len(dxb)
    dyb = r.uniform(3, 12, n).astype(np.float32)
    th = r.uniform(0, np.pi, n)
    sx, sy = sigma * np.ones(n), sigma * r.uniform(1.0, 1.5, n)
    c, s = np.cos(th), np.sin(th)
    a, b, d = c * c * sx ** 2 + s * s * sy ** 2, c * s * (sx ** 2 - sy ** 2), s * s * sx ** 2 + c * c * sy ** 2
    det = a * d - b * b
    A2 = (0.5 * d / det * g64.LOG2E).astype(np.float32)
    B2 = (-b / det * g64.LOG2E).astype(np.float32)
    C2 = (0.5 * a / det * g64.LOG2E).astype(np.float32)
    dL = r.uniform(1.0, 1.5, (n, 16, 16)).astype(np.float32)
    gcut = np.float32(2.0 ** -16.6)
    # float64 moments of the same pairs (same conic, same cut)
    dx = dxb[:, None, None].astype(np.float64) - np.arange(16.0)[None, None, :]
    dy = dyb[:, None, None].astype(np.float64) - np.arange(16.0)[None, :, None]
    G = np.exp2(-(A2[:, None, None] * dx * dx + B2[:, None, None] * dx * dy + C2[:, None, None] * dy * dy))
    t = np.where(G >= gcut, dL * G, 0.0)
    want = [(t * f).sum((1, 2)) for f in (1.0, dx, dx * dx)]
    # the absolute moments as raster_moments forms them for the bar: each pair weighted for the rounding of its power
    L = np.log(2.0) * (np.abs(A2[:, None, None] * dx * dx) + np.abs(B2[:, None, None] * dx * dy)
                       + np.abs(C2[:, None, None] * dy * dy))
    absm = [(np.abs(t * f) * (1.0 + L / g64.POWER_WEIGHT)).sum((1, 2)) for f in (1.0, dx, dx * dx)]
    worst = {}
    live = absm[0] > 0                       # a centre 2 columns outside the tile: no pair of this row contributes
    assert live.sum() >= 0.9 * n
    for recentre in (False, True):
        got = _emulate_exact_path(dxb, dyb, A2, B2, C2, dL, gcut, recentre)
        assert all((gv[~live] == 0).all() for gv in got)
        worst[recentre] = max(float((np.abs(gv - w) / (g64.C_BAR * g64.U * am))[live].max())
                              for gv, w, am in zip(got, want, absm))
    print(f"sigma {sigma}: tile origin {worst[False]:.3g} x the bar, nearest column {worst[True]:.3g} x the bar")
    assert worst[False] > 1.0
    assert worst[True] <= 0.5


# ---- the voxelizer ----------------------------------------------------------------------------------------------------
VGRIDS = {"full32": ((32, 32, 32), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0)),
          "ragged": ((20, 36, 28), (1.3, 2.0, 1.7), (0.1, -0.05, 0.2))}


def voxel_judge(cloud, grid, fwd, dL, got, mod=1.0, cov=None):
    """Per-element comparison of a voxelizer backward's gradients with the float64 statement -> (ratios [n, 17] in
    units of the bar, compared Gaussians, Gaussians with an ill-conditioned voxel covariance)."""
    nV, sV, _ = grid
    radii = (fwd["radii_x"], fwd["radii_y"], fwd["radii_z"])
    mom = g64.voxel_moments(fwd["xyz_vol"], fwd["conic_opacity"], radii, nV, dL)
    chain = g64.make_voxel_chain(nV, sV, mod, precomp=cov is not None)
    p = g64.voxel_chain_inputs(cloud.scales, None if cov is not None else cloud.rotations, cov, fwd["conic_opacity"])
    c3 = cov if cov is not None else textbook.sigma3(cloud.scales, cloud.rotations, mod)[
        :, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    live = (radii[0] > 0) & (mom["n_pairs"] > 0)
    well = g64.voxel_cond(c3, nV, sV) <= g64.COND_MAX
    idx = np.nonzero(live & well)[0]
    y64, bar, band = g64.reference(mom, p, chain, idx)
    r = g64.compare(g64.voxel_kernel_rows(got, idx), y64, bar, band)
    return r, idx, int((live & ~well).sum()), mom


@pytest.mark.parametrize("dl_kind", ["ramp", "signed"])
@pytest.mark.parametrize("grid", ["full32", "ragged"])
def test_voxel_float64_statement_agrees_with_the_oracle(grid, dl_kind):
    nV, sV, ctr = VGRIDS[grid]
    cloud = scene.make_cloud(1500, kind="trained", seed=nV[1])
    fwd = util.oracle_voxel_forward(cloud, nV, sV, ctr)
    r = np.random.RandomState(9)
    dL = (1.0 + r.rand(*nV) if dl_kind == "ramp" else r.randn(*nV)).astype(np.float32)
    got = util.oracle_voxel_backward(cloud, nV, sV, fwd, dL)
    ratio, idx, ill, _ = voxel_judge(cloud, VGRIDS[grid], fwd, dL, got)
    assert np.isfinite(ratio).all()
    worst = {k: float(v.max()) for k, v in g64.voxel_split(ratio).items()}
    print(f"oracle voxel {grid}: {len(idx)} compared, {ill} ill-conditioned;", {k: f"{v:.3g}" for k, v in worst.items()})
    assert len(idx) >= 500 and max(worst.values()) <= 1.0, worst
