"""GPU parity at the code-path boundaries of the rasterizer and the voxelizer, on the engineered inputs of
tests/regime_cases.py (whose sides tests/test_regimes_cpu.py checks on the CPU), at small and partial CTA counts, from
inputs that cannot take the TMA loads, and for the asynchronous capacity contract.

The bars are those of test_raster_gpu.py / test_voxel_gpu.py: per-Gaussian stage outputs and tile lists bit-exact, the
image / volume within 1e-5 of its scale (+1e-7), gradients within util.assert_grads_close's defaults.  One exception,
stated where it applies: a tile whose list holds thousands of Gaussians is compared against a float64 sum."""
import numpy as np
import pytest

import regime_cases as rc
import util
from r2_gaussian_b200 import scene

pytestmark = pytest.mark.gpu

CASES = {c.name: c for c in rc.engineered_cases()}
RASTER = [n for n, c in CASES.items() if c.kind == "raster"]
# Not compared on the GPU: the voxel det-ratio straddle.  A conic 1e-4 from singular is ill-conditioned in float32 (the
# quadratic form's terms are ~1e5 times the power along the needle), and the kernel's Horner evaluation and the oracle's
# differ by up to ~1e-4 of the volume's scale there, beyond the 1e-5 bar; the CPU test still checks its sides.
VOXEL = [n for n, c in CASES.items() if c.kind == "voxel" and n != "voxel_fast_det"]
RASTER_GRADS = ["dL_dmean2D", "dL_dopacity", "dL_dmu", "dL_dmean3D", "dL_dcov3D", "dL_dscale", "dL_drot"]
VOXEL_GRADS = ["dL_dopacity", "dL_dmean3D", "dL_dcov3D", "dL_dscale", "dL_drot"]
U = 2.0 ** -24   # unit roundoff of float32


def _crowded_bound(alpha, cut, scale):
    """Bar for a pixel / voxel summed from many float32 terms, against the float64 sum of the same terms.

    `alpha` [terms, pixels] holds the float64 alphas of every Gaussian of the tile at every pixel of it.  The oracle adds
    the terms in depth order, the kernel in id order in chunks whose partial sums are then added: each is a float32 sum
    of the same n terms, within (n - 1) u sum|term| of the exact sum whatever the order.  On top of that the bar keeps
    the suite's per-pixel 1e-5 of the image scale (+1e-7), and allows one cut-sized term for every pair that lies within
    the bwd_row_careful band of the alpha cut, where float32 may decide the cut either way."""
    keep = alpha >= cut
    S = np.where(keep, alpha, 0.0).sum(axis=0)
    n = keep.sum(axis=0)
    band = (np.abs(alpha / cut - 1.0) <= rc.K["CAREFUL_HI"] - 1.0).sum(axis=0)
    return S, np.maximum(n - 1, 0) * U * S + 1e-5 * scale + 1e-7 + band * cut * rc.K["CAREFUL_HI"]


def _raster_tile_alphas(orc, tile, W, H):
    gx = -(-W // rc.RASTER_TILE)
    tx, ty = tile % gx, tile // gx
    a, b = orc["ranges"][tile]
    ids = orc["point_list"][a:b]
    ys, xs = np.mgrid[ty * 16:min(H, ty * 16 + 16), tx * 16:min(W, tx * 16 + 16)]
    xy, co = orc["xy"][ids].astype(np.float64), orc["conic_opacity"][ids].astype(np.float64)
    w = (orc["conic_opacity"][ids, 3] * orc["mu"][ids]).astype(np.float32).astype(np.float64)
    dx = xy[:, 0, None] - xs.reshape(1, -1)
    dy = xy[:, 1, None] - ys.reshape(1, -1)
    power = -0.5 * (co[:, 0, None] * dx * dx + co[:, 2, None] * dy * dy) - co[:, 1, None] * dx * dy
    alpha = np.where(power <= 0, w[:, None] * np.exp(np.minimum(power, 0)), 0.0)
    return alpha, (ys.reshape(-1), xs.reshape(-1))


def _voxel_tile_alphas(orc, tile, nV):
    g = rc.tile_grid(nV)
    tx, ty, tz = tile % g[0], (tile // g[0]) % g[1], tile // (g[0] * g[1])
    a, b = orc["ranges"][tile]
    ids = orc["point_list"][a:b]
    vx, vy, vz = np.meshgrid(*[np.arange(t * 8, min(n, t * 8 + 8)) for t, n in zip((tx, ty, tz), nV)], indexing="ij")
    vx, vy, vz = vx.reshape(-1), vy.reshape(-1), vz.reshape(-1)
    p = orc["xyz_vol"][ids].astype(np.float64)
    co = orc["conic_opacity"][ids].astype(np.float64)
    dx, dy, dz = (p[:, k, None] - (v[None] + 0.5) for k, v in enumerate((vx, vy, vz)))
    power = (-0.5 * (co[:, 0, None] * dx * dx + co[:, 3, None] * dy * dy + co[:, 5, None] * dz * dz)
             - co[:, 1, None] * dx * dy - co[:, 2, None] * dx * dz - co[:, 4, None] * dy * dz)
    alpha = np.where(power <= 0, co[:, 6, None] * np.exp(np.minimum(power, 0)), 0.0)
    return alpha, (vx, vy, vz)


def assert_raster_forward(ours, orc, W, H, crowded=()):
    assert ours["R"] == orc["R"]
    np.testing.assert_array_equal(ours["radii"], orc["radii"])
    np.testing.assert_array_equal(ours["tiles_touched"], orc["tiles_touched"])
    vis = orc["radii"] > 0
    for k in ("depth", "xy", "conic_opacity", "mu"):
        np.testing.assert_array_equal(ours[k][vis].view(np.uint32), orc[k][vis].view(np.uint32), err_msg=k)
    np.testing.assert_array_equal(ours["point_offsets"], np.cumsum(orc["tiles_touched"]).astype(np.uint32))
    assert util.key_multiset_equal(ours["keys"], orc["keys"])
    _assert_lists(ours, orc)
    scale = float(np.abs(orc["image"]).max()) if orc["R"] else 1.0
    err = np.abs(ours["image"].astype(np.float64) - orc["image"])
    for t in crowded:
        alpha, (ys, xs) = _raster_tile_alphas(orc, t, W, H)
        S, bar = _crowded_bound(alpha, 2.0 ** -rc.K["Q_CUT"], scale)
        got = ours["image"][ys, xs].astype(np.float64)
        print(f"crowded tile {t}: {alpha.shape[0]} Gaussians, max |ours - f64| / bar = "
              f"{(np.abs(got - S) / bar).max():.3g}, max |ours - oracle| = {err[ys, xs].max():.3g} (scale {scale:.3g})")
        assert np.all(np.abs(got - S) <= bar), f"crowded tile {t}"
        err[ys, xs] = 0.0
    assert err.max() <= 1e-5 * scale + 1e-7, f"image error {err.max()} vs scale {scale}"


def assert_voxel_forward(ours, orc, nV, crowded=()):
    assert ours["R"] == orc["R"]
    for k in ("radii_x", "radii_y", "radii_z", "tiles_touched"):
        np.testing.assert_array_equal(ours[k], orc[k])
    vis = orc["tiles_touched"] > 0
    for k in ("xyz_vol", "depth"):
        np.testing.assert_array_equal(ours[k][vis].view(np.uint32), orc[k][vis].view(np.uint32), err_msg=k)
    np.testing.assert_allclose(ours["conic_opacity"][vis], orc["conic_opacity"][vis], rtol=2e-6, atol=0)
    assert util.key_multiset_equal(ours["keys"], orc["keys"])
    _assert_lists(ours, orc)
    scale = float(np.abs(orc["vol"]).max()) if orc["R"] else 1.0
    err = np.abs(ours["vol"].astype(np.float64) - orc["vol"])
    for t in crowded:
        alpha, idx = _voxel_tile_alphas(orc, t, nV)
        S, bar = _crowded_bound(alpha, 2.0 ** -rc.K["VQ_CUT"], scale)
        got = ours["vol"][idx].astype(np.float64)
        print(f"crowded tile {t}: {alpha.shape[0]} Gaussians, max |ours - f64| / bar = "
              f"{(np.abs(got - S) / bar).max():.3g}, max |ours - oracle| = {err[idx].max():.3g} (scale {scale:.3g})")
        assert np.all(np.abs(got - S) <= bar), f"crowded tile {t}"
        err[idx] = 0.0
    assert err.max() <= 1e-5 * scale + 1e-7, f"volume error {err.max()} vs scale {scale}"


def _assert_lists(ours, orc):
    np.testing.assert_array_equal(ours["ranges"], orc["ranges"])
    for t in np.nonzero(orc["ranges"][:, 1] > orc["ranges"][:, 0])[0]:
        a, b = orc["ranges"][t]
        mine = ours["point_list"][a:b]
        assert np.all(np.diff(mine.astype(np.int64)) > 0), f"tile {t}: list not strictly ascending"
        np.testing.assert_array_equal(mine, np.sort(orc["point_list"][a:b]), err_msg=f"tile {t}")


def _raster_both(cloud, view, crowded=(), seed=7, needles=()):
    """Forward and backward against the oracle.  The gradients of `needles` (conics 1e-4 from singular, whose gradients
    two float32 evaluations cannot agree on to 2e-4) are required to be finite, not compared; every other Gaussian's are
    compared at util.assert_grads_close's defaults."""
    W, H = view.image_width, view.image_height
    ours = util.ours_raster_forward(cloud, view)
    orc = util.oracle_raster_forward(cloud, view)
    assert_raster_forward(ours, orc, W, H, crowded)
    dL = np.random.RandomState(seed).randn(H, W).astype(np.float32)
    g = util.ours_raster_backward(cloud, view, ours, dL)
    go = util.oracle_raster_backward(cloud, view, orc, dL)
    for k in RASTER_GRADS:
        assert np.all(np.isfinite(g[k])), f"{k}: not finite"
    rows = np.setdiff1d(np.arange(cloud.P), np.asarray(needles, np.int64))
    util.assert_grads_close({k: g[k][rows] for k in g}, {k: go[k][rows] for k in go}, RASTER_GRADS)
    return orc


def _voxel_both(cloud, grid, crowded=(), seed=11):
    nV, sV, ctr = grid
    ours = util.ours_voxel_forward(cloud, nV, sV, ctr)
    orc = util.oracle_voxel_forward(cloud, nV, sV, ctr)
    assert_voxel_forward(ours, orc, nV, crowded)
    dL = np.random.RandomState(seed).randn(*nV).astype(np.float32)
    g = util.ours_voxel_backward(cloud, nV, sV, ctr, ours, dL)
    go = util.oracle_voxel_backward(cloud, nV, sV, orc, dL)
    util.assert_grads_close(g, go, VOXEL_GRADS)
    return orc


@pytest.mark.parametrize("name", RASTER)
def test_raster_engineered_case(name):
    case = CASES[name]
    orc = _raster_both(case.cloud, case.view, case.crowded, needles=case.needles)
    rc.check_case(case, orc)   # and it still exercised what it is named after


@pytest.mark.parametrize("name", VOXEL)
def test_voxel_engineered_case(name):
    case = CASES[name]
    orc = _voxel_both(case.cloud, case.grid, case.crowded)
    rc.check_case(case, orc)


@pytest.mark.parametrize("P", [1, 255, 256, 257])
def test_partial_and_single_ctas(P):
    """P around one preprocess / direct_fill CTA: a full CTA, a partial one, a full one plus a single Gaussian."""
    cloud = scene.make_cloud(P, kind="trained", seed=P)
    orc = _raster_both(cloud, rc.parallel_view(96, 80))
    reg = rc.regime(orc, (80, 96))
    assert len(reg["cta_total"]) == -(-P // rc.K["DIRECT_BLOCK"]) and reg["R"] > 0
    _voxel_both(cloud, ((24, 20, 28), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0)))


def _unaligned(x):
    """A copy of x whose storage starts 4 bytes past an allocation (so never 16-byte aligned)."""
    import torch
    buf = torch.empty(x.numel() + 1, dtype=x.dtype, device=x.device)
    y = buf[1:].view(x.shape)
    y.copy_(x)
    assert y.data_ptr() % 16 == 4
    return y


def test_unaligned_inputs_take_the_plain_loads_bit_identically():
    """The preprocess kernels stage full CTAs with TMA only from 16-byte-aligned inputs; from inputs at a 4-byte offset
    every CTA takes the plain loads.  Both must give the same bits."""
    import torch
    from r2_gaussian_b200 import _C

    cloud = scene.make_cloud(1000, kind="trained", seed=5)   # 3 full CTAs and a partial one
    view = rc.cone_view(128, 128)
    t = util.to_torch(cloud, view)
    u = {k: _unaligned(t[k]) for k in ("means", "dens", "scales", "rots")}
    e = torch.Tensor([])

    def raster(m):
        R, color, radii, *_ = _C.rasterize_gaussians(m["means"], m["dens"], m["scales"], m["rots"], 1.0, e, t["view"],
                                                     t["proj"], view.tanfovx, view.tanfovy, 128, 128, t["campos"],
                                                     False, view.mode, False)
        return R, color.cpu().numpy(), radii.cpu().numpy()

    def voxel(m):
        R, vol, rx, ry, rz, *_ = _C.voxelize_gaussians(m["means"], m["dens"], m["scales"], m["rots"], 1.0, e, 40, 36, 32,
                                                       2.0, 2.0, 2.0, 0.0, 0.0, 0.0, False, False)
        return R, vol.cpu().numpy(), rx.cpu().numpy(), ry.cpu().numpy(), rz.cpu().numpy()

    for f in (raster, voxel):
        a, b = f(t), f(u)
        assert a[0] == b[0] and a[0] > 0
        for x, y in zip(a[1:], b[1:]):
            np.testing.assert_array_equal(x.view(np.uint32), y.view(np.uint32))


GUARD = 64 * 1024
CAPACITY_CASES = {
    "raster_direct": ("raster", "cone_trained_small", None),
    "raster_radix": ("raster", "cone_trained_bigdet", None),
    "voxel_direct": ("voxel", ((32, 32, 32), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0)), None),
    "voxel_two_level": ("voxel", ((144, 136, 136), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0)), None),
    "voxel_radix": ("voxel", ((144, 136, 136), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0)), "radix"),
}


@pytest.mark.parametrize("name", list(CAPACITY_CASES))
def test_async_capacity_contract_with_guard(name, monkeypatch):
    """The asynchronous forward never touches memory beyond the binning buffer of the provisioned capacity: with
    capacity R - 1 it reports (R, overflow) and with capacity R (R, 0) and the oracle's output, and in both cases a
    guard region of a fixed pattern right after the buffer is left as it was."""
    import torch
    from r2_gaussian_b200.engine import RasterEngine, VoxelEngine

    kind, what, binning = CAPACITY_CASES[name]
    if binning:
        monkeypatch.setenv("R2X_VOXEL_BINNING", binning)
    else:
        monkeypatch.delenv("R2X_VOXEL_BINNING", raising=False)
    if kind == "raster":
        cloud, view = util.case(what)
        ref = util.oracle_raster_forward(cloud, view)
        t = util.to_torch(cloud, view)
        eng = RasterEngine(cloud.P, view.image_width, view.image_height, "cuda", capacity=1)
        args = (t["means"], t["dens"], t["scales"], t["rots"], t["view"], t["proj"], t["campos"], view.tanfovx,
                view.tanfovy, view.mode)
        want = ref["image"]
        assert rc.binning_path((view.image_height, view.image_width)) == name.split("_", 1)[1]
    else:
        nV, sV, ctr = what
        cloud = scene.make_cloud(1200, kind="trained", seed=9)
        ref = util.oracle_voxel_forward(cloud, nV, sV, ctr)
        t = util.to_torch(cloud, None)
        eng = VoxelEngine(cloud.P, nV, "cuda", capacity=1)
        args = (t["means"], t["dens"], t["scales"], t["rots"], sV, ctr)
        want = ref["vol"]
        assert binning or rc.binning_path(nV) == name.split("_", 1)[1]
    R = ref["R"]
    assert R > 1
    pattern = (torch.arange(GUARD, device="cuda") * 37 + 11).remainder(256).to(torch.uint8)
    for cap, ov in ((R - 1, 1), (R, 0)):
        nbytes = eng.lib.r2x_binning_bytes(cap)
        buf = torch.empty(nbytes + GUARD, dtype=torch.uint8, device="cuda")
        buf[nbytes:] = pattern
        eng.capacity, eng.binning = cap, buf[:nbytes]
        eng.status.zero_()
        out = eng.forward(*args)
        torch.cuda.synchronize()
        assert [int(v) for v in eng.status.cpu()] == [R, ov], (cap, eng.status.cpu())
        assert torch.equal(buf[nbytes:], pattern), f"capacity {cap}: bytes past the binning buffer were written"
        if not ov:
            got = out[0] if kind == "raster" else out
            err = np.abs(got.cpu().numpy().astype(np.float64) - want).max()
            assert err <= 1e-5 * np.abs(want).max() + 1e-7
