"""Every per-Gaussian gradient of the rasterizer's and the voxelizer's backwards element by element against its float64 statement
(grad_float64.py), on the kernels' own stage outputs.

Adam scales each element's step by that element's own gradient history, so small and faint Gaussians need a small error
of their own, not one relative to the array's largest element.  The engineered sweeps put Gaussians of 0.15 to 12 px at
every column of a tile, at sub-pixel offsets and just outside it, so that both render paths of the backward (the exact
path of narrow conics, the forward-difference fast path and its careful rows) and the partial tiles of a ragged detector
see them; realistic clouds, both beams, the 1.3 tanfov clamp, scale_modifier, cov3D_precomp and a batched-views call
complete the cases.  The voxelizer's sweeps step the centre through every voxel of a tile along z, at fast and
exact conics, on the full32 and ragged grids.  Each test prints its worst error per output and regime in units of the bar, and asserts a minimum
number of compared Gaussians per regime so that none drops out silently."""
import numpy as np
import pytest

import grad_float64 as g64
import util
from r2_gaussian_b200 import scene
from test_grad_float64_cpu import dl_ramp, dl_signed

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

SIGMAS = (0.15, 0.25, 0.4, 0.6, 0.8, 1.2, 2.0, 4.0, 8.0)
OFFSETS = np.r_[np.repeat(np.arange(16.0), 3) + np.tile([0.0, 0.25, 0.5], 16), -1.5, -0.5, 16.25, 17.5]


def _view(beam, n):
    sc = scene.cone_beam_scanner(n, 64) if beam == "cone" else scene.parallel_beam_scanner(n, 64)
    return scene.make_view(sc, 0.9)


def _unproject(view, px, py):
    """World points on the plane through the origin facing the source that project to pixel (px, py)."""
    P4 = view.projmatrix.astype(np.float64)                     # hom = [p, 1] @ P4
    W, H = view.image_width, view.image_height
    nx, ny = (2 * px + 1) / W - 1, (2 * py + 1) / H - 1
    n = view.campos.astype(np.float64) / np.linalg.norm(view.campos)
    out = np.zeros((len(px), 3))
    for i in range(len(px)):
        A = np.stack([P4[:3, 0] - nx[i] * P4[:3, 3], P4[:3, 1] - ny[i] * P4[:3, 3], n])
        rhs = -np.array([P4[3, 0] - nx[i] * P4[3, 3], P4[3, 1] - ny[i] * P4[3, 3], 0.0])
        out[i] = np.linalg.solve(A, rhs)
    return out


def _sweep_cloud(view, seed, clamp=False):
    """Gaussians at every column offset of OFFSETS, one tile apart, at each sigma of SIGMAS (in pixels), isotropic and
    anisotropic (rotated); the last tile column of a ragged detector is a partial tile.  clamp: large Gaussians centred
    beyond 1.3 tanfov on both sides that still reach the image."""
    r = np.random.RandomState(seed)
    W, H = view.image_width, view.image_height
    gx, gy = -(-W // 16), -(-H // 16)
    px, py, sig, ani = [], [], [], []
    k = 0
    for s in SIGMAS:
        for aniso in (False, True):
            for o in OFFSETS:
                tx, ty = k % gx, (k // gx) % gy
                k += 1
                px.append(16 * tx + o)
                py.append(16 * ty + r.uniform(2, 14))
                sig.append(s)
                ani.append(aniso)
    if clamp:
        for side in (-1, 1):
            for i in range(24):
                px.append(W / 2 + side * (0.65 * W + 4 + 8 * (i % 3)) - 0.5)
                py.append(r.uniform(0, H))
                sig.append(9.0 + (i % 4))
                ani.append(bool(i % 2))
    n_dim = len(px)
    for i in range(16):                           # density so high that log2 w > 20: the exact path at a wide conic
        px.append(r.uniform(8, W - 8)); py.append(r.uniform(8, H - 8)); sig.append(1.0 + 0.1 * i); ani.append(bool(i % 2))
    px, py, sig, ani = (np.asarray(a) for a in (px, py, sig, ani))
    means = _unproject(view, px, py)
    if view.mode == 1:
        depth = np.linalg.norm(view.campos.astype(np.float64))
        per_px = depth * 2 * view.tanfovx / W
    else:
        per_px = 2 * view.tanfovx / W
    n = len(px)
    ratio = np.where(ani, r.uniform(1.5, 3.0, n), 1.0)
    scales = (per_px * sig)[:, None] * np.stack([np.ones(n), ratio, r.uniform(0.8, 1.2, n)], 1)
    q = r.randn(n, 4)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    dens = r.uniform(0.5, 2.0, (n, 1))
    dens[n_dim:] = 3e8
    f = np.float32
    return scene.Cloud(means.astype(f), scales.astype(f), q.astype(f), dens.astype(f))


def _regimes(fwd, view, mom, cloud=None):
    """Boolean masks of the compared Gaussians by regime."""
    co, mu = fwd["conic_opacity"], fwd["mu"]
    fast = g64.fast_path(co, mu)
    A2 = co[:, 0].astype(np.float64) * 0.5 * g64.LOG2E
    W = view.image_width
    px = fwd["xy"][:, 0]
    right = np.array([g64.tile_rect(fwd["xy"][g, 0], fwd["xy"][g, 1], fwd["radii"][g], W, view.image_height)[2]
                      for g in range(len(px))])
    partial = (W % 16 != 0) & (right == -(-W // 16))
    sub = np.sqrt(np.maximum(1.0 / np.maximum(co[:, 0].astype(np.float64), 1e-30), 0)) < 1.0   # sigma_x < 1 px
    out = {"exact": ~fast, "fast": fast, "careful": fast & (mom["n_near_cut"] > 0), "partial_tile": partial,
           "subpixel": sub, "narrow_A2>2": A2 > 2, "exact_by_density": ~fast & (A2 <= 2)}
    if view.mode == 1:
        t = cloud.means.astype(np.float64) @ view.viewmatrix[:3, :3].astype(np.float64) + view.viewmatrix[3, :3]
        out["clamp"] = (np.abs(t[:, 0] / t[:, 2]) > 1.3 * view.tanfovx) | (np.abs(t[:, 1] / t[:, 2]) > 1.3 * view.tanfovy)
    return out


def _judge(label, got, fwd, view, cloud, dL, mod=1.0, cov=None, min_count=None):
    mom = g64.raster_moments(fwd["xy"], fwd["conic_opacity"], fwd["mu"], fwd["radii"], dL)
    chain = g64.make_chain(view.image_width, view.image_height, view.tanfovx, view.tanfovy, view.mode, mod,
                           precomp=cov is not None)
    p = g64.chain_inputs(cloud.means, None if cov is not None else cloud.scales,
                         None if cov is not None else cloud.rotations, cov, fwd["conic_opacity"], fwd["mu"],
                         view.viewmatrix, view.projmatrix)
    live = (fwd["radii"] > 0) & (mom["n_pairs"] > 0)
    well = g64.cond2(fwd["conic_opacity"]) <= g64.COND_MAX
    idx = np.nonzero(live & well)[0]
    y64, bar, band = g64.reference(mom, p, chain, idx)
    r = g64.split(g64.compare(g64.kernel_rows(got, idx), y64, bar, band))
    assert all(np.isfinite(v).all() for v in r.values()), f"{label}: a gradient or its statement is not finite"
    reg = {k: v[idx] for k, v in _regimes(fwd, view, mom, cloud).items()}
    counts = {k: int(v.sum()) for k, v in reg.items()}
    print(f"\n{label}: {len(idx)} Gaussians compared, {int((live & ~well).sum())} with cond(2-D cov) > "
          f"{g64.COND_MAX:g} not held to the bar; per regime {counts}")
    worst = 0.0
    for k, v in r.items():
        per = {name: float(v[m].max()) if m.any() else 0.0 for name, m in reg.items()}
        print(f"  {k:12s} worst {float(v.max()):.3g} x bar; " + ", ".join(f"{n} {x:.3g}" for n, x in per.items()))
        worst = max(worst, float(v.max()))
    for name, n in (min_count or {}).items():
        assert counts[name] >= n, f"{label}: regime {name} has {counts[name]} Gaussians, expected >= {n}"
    assert worst <= 1.0, f"{label}: worst element {worst:.3g} x its bar"
    return r


@pytest.mark.parametrize("dl_kind", ["ramp", "signed"])
@pytest.mark.parametrize("beam,n", [("cone", 128), ("parallel", 128), ("cone", 100)], ids=["cone", "parallel", "ragged"])
def test_sweep_gradients_per_element_against_float64(beam, n, dl_kind, monkeypatch):
    monkeypatch.setenv("R2X_SPECULATIVE", "0")
    view = _view(beam, n)
    cloud = _sweep_cloud(view, seed=n, clamp=(beam == "cone"))
    dL = (dl_ramp if dl_kind == "ramp" else dl_signed)(view.image_height, view.image_width, 11)
    fwd = util.ours_raster_forward(cloud, view)
    got = util.ours_raster_backward(cloud, view, fwd, dL)
    mc = {"exact": 150, "fast": 300, "careful": 2, "subpixel": 300, "narrow_A2>2": 150, "exact_by_density": 8}
    if beam == "cone":
        mc["clamp"] = 8
    if n % 16:
        mc["partial_tile"] = 20
    _judge(f"sweep {beam} {n}px, dL {dl_kind}", got, fwd, view, cloud, dL, min_count=mc)


@pytest.mark.parametrize("variant", ["modifier0.5", "modifier1.6", "cov3D_precomp"])
def test_sweep_variants_per_element_against_float64(variant, monkeypatch):
    monkeypatch.setenv("R2X_SPECULATIVE", "0")
    view = _view("cone", 128)
    cloud = _sweep_cloud(view, seed=5)
    mod = {"modifier0.5": 0.5, "modifier1.6": 1.6}.get(variant, 1.0)
    cov = None
    if variant == "cov3D_precomp":
        import textbook
        cov = textbook.sigma3(cloud.scales, cloud.rotations)[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].astype(np.float32)
    dL = dl_ramp(view.image_height, view.image_width, 12)
    fwd = util.ours_raster_forward(cloud, view, cov3D_precomp=cov, scale_modifier=mod)
    got = util.ours_raster_backward(cloud, view, fwd, dL)
    _judge(f"sweep {variant}", got, fwd, view, cloud, dL, mod, cov, min_count={"exact": 100, "fast": 200})


@pytest.mark.parametrize("dl_kind", ["ramp", "signed"])
@pytest.mark.parametrize("name", ["cone_trained_small", "cone_trained_ragged"])
def test_realistic_cloud_gradients_per_element_against_float64(name, dl_kind):
    cloud, view = util.case(name)
    dL = (dl_ramp if dl_kind == "ramp" else dl_signed)(view.image_height, view.image_width, 13)
    fwd = util.ours_raster_forward(cloud, view)
    got = util.ours_raster_backward(cloud, view, fwd, dL)
    _judge(f"{name}, dL {dl_kind}", got, fwd, view, cloud, dL, min_count={"fast": 500, "careful": 20})


def test_batched_views_gradients_per_element_against_float64(monkeypatch):
    """rasterize_views_backward: each view's dL/dmean2D against that view's float64 statement, and the gradients summed
    over the views against the sum of the views' statements (with the sum of their bars)."""
    from r2_gaussian_b200 import _C

    monkeypatch.setenv("R2X_SPECULATIVE", "0")
    sc = scene.cone_beam_scanner(128, 64)
    views = [scene.make_view(sc, a) for a in (0.9, 2.1, 4.0)]
    cloud = _sweep_cloud(views[0], seed=3)
    dL = np.stack([dl_ramp(128, 128, 20 + v) for v in range(len(views))])
    t = util.to_torch(cloud, None)
    V = torch.tensor(np.stack([v.viewmatrix for v in views]), device="cuda")
    Pm = torch.tensor(np.stack([v.projmatrix for v in views]), device="cuda")
    v0 = views[0]
    R, _, radii, geom, binning, img = _C.rasterize_views(t["means"], t["dens"], t["scales"], t["rots"], 1.0, V, Pm,
                                                         v0.tanfovx, v0.tanfovy, 128, 128, v0.mode)
    g = _C.rasterize_views_backward(t["means"], radii, t["scales"], t["rots"], 1.0, V, Pm, v0.tanfovx, v0.tanfovy,
                                    torch.tensor(dL, device="cuda"), geom, R, binning, img, v0.mode)
    g = [x.cpu().numpy() for x in g]
    radii = radii.cpu().numpy()
    P = cloud.P
    y_sum, bar_sum, band_sum = np.zeros((P, 20)), np.zeros((P, 20)), np.zeros((P, 20))
    held = np.ones(P, bool)
    for v, view in enumerate(views):
        fwd = util.ours_raster_forward(cloud, view)       # the single-view stage outputs: bit for bit the batched ones
        assert np.array_equal(fwd["radii"], radii[v])
        mom = g64.raster_moments(fwd["xy"], fwd["conic_opacity"], fwd["mu"], fwd["radii"], dL[v])
        chain = g64.make_chain(128, 128, view.tanfovx, view.tanfovy, view.mode)
        p = g64.chain_inputs(cloud.means, cloud.scales, cloud.rotations, None, fwd["conic_opacity"], fwd["mu"],
                             view.viewmatrix, view.projmatrix)
        live = (fwd["radii"] > 0) & (mom["n_pairs"] > 0)
        held &= (g64.cond2(fwd["conic_opacity"]) <= g64.COND_MAX) | ~live
        idx = np.nonzero(live)[0]
        y64, bar, band = g64.reference(mom, p, chain, idx)
        ok = g64.cond2(fwd["conic_opacity"][idx]) <= g64.COND_MAX
        r = g64.compare(np.asarray(g[0][v], np.float64)[idx, :2], y64[:, :2], bar[:, :2], band[:, :2])[ok]
        print(f"view {v}: dL_dmean2D worst {r.max():.3g} x bar over {int(ok.sum())} Gaussians")
        assert r.max() <= 1.0
        y_sum[idx] += y64; bar_sum[idx] += bar; band_sum[idx] += band
    # batched outputs: opacity, mean3D, cov3D, scale, rot -> chain columns 2, 4..19 (no mean2D, no mu)
    got = np.concatenate([g[1].reshape(P, -1), g[2], g[3], g[4], g[5]], 1).astype(np.float64)
    sel = np.nonzero(held & (bar_sum[:, 2] > 0))[0]
    cols = [2] + list(range(4, 20))
    r = g64.compare(got[sel], y_sum[sel][:, cols], bar_sum[sel][:, cols], band_sum[sel][:, cols])
    print(f"summed over {len(views)} views: worst {r.max():.3g} x bar over {len(sel)} Gaussians")
    assert len(sel) >= 500 and r.max() <= 1.0


# ---- the voxelizer ----------------------------------------------------------------------------------------------------
from test_grad_float64_cpu import VGRIDS, voxel_judge  # noqa: E402

VSIGMAS = (0.3, 0.45, 0.6, 0.8, 1.2, 2.0, 4.0)
ZOFFSETS = np.r_[np.repeat(np.arange(8.0), 3) + np.tile([0.0, 0.25, 0.5], 8), -1.5, -0.5, 8.25, 9.5]


def _voxel_sweep_cloud(grid, seed):
    """Gaussians whose z centre steps through every voxel of an 8-voxel tile at offsets 0, 1/4, 1/2 and just outside
    it (dz0 across the whole tile), at each sigma of VSIGMAS (voxels along z), isotropic and anisotropic (rotated),
    one x-y tile apart; plus a few of density above 2^20 (the exact path through log2 rho)."""
    nV, sV, ctr = grid
    r = np.random.RandomState(seed)
    dv = np.array(sV, np.float64) / np.array(nV)
    g = [-(-n // 8) for n in nV]
    vox, sig, ani, dens = [], [], [], []
    k = 0
    for s in VSIGMAS:
        for aniso in (False, True):
            for o in ZOFFSETS:
                tx, ty, tz = k % g[0], (k // g[0]) % g[1], (k // (g[0] * g[1])) % g[2]
                k += 1
                vox.append((8 * tx + r.uniform(2, 6), 8 * ty + r.uniform(2, 6), 8 * tz + o))
                sig.append(s); ani.append(aniso); dens.append(r.uniform(0.5, 2.0))
    for i in range(16):
        vox.append((r.uniform(4, nV[0] - 4), r.uniform(4, nV[1] - 4), r.uniform(4, nV[2] - 4)))
        sig.append(1.0 + 0.1 * i); ani.append(bool(i % 2)); dens.append(3e6)
    vox, sig, ani = np.asarray(vox), np.asarray(sig), np.asarray(ani)
    n = len(sig)
    means = vox * dv - 0.5 * np.array(sV) + np.array(ctr)
    ratio = np.where(ani, r.uniform(1.5, 3.0, n), 1.0)
    scales = (sig * dv.min())[:, None] * np.stack([ratio, r.uniform(0.8, 1.2, n), np.ones(n)], 1)
    q = np.where(ani[:, None], r.randn(n, 4), np.array([[1.0, 0, 0, 0]]))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    f = np.float32
    return scene.Cloud(means.astype(f), scales.astype(f), q.astype(f), np.asarray(dens).reshape(-1, 1).astype(f))


def _voxel_check(label, cloud, grid, dL, min_count, mod=1.0, cov=None):
    nV, sV, ctr = grid
    fwd = util.ours_voxel_forward(cloud, nV, sV, ctr, cov3D_precomp=cov, scale_modifier=mod)
    got = util.ours_voxel_backward(cloud, nV, sV, ctr, fwd, dL)
    ratio, idx, ill, mom = voxel_judge(cloud, grid, fwd, dL, got, mod, cov)
    assert np.isfinite(ratio).all(), f"{label}: a gradient or its statement is not finite"
    fast = g64.voxel_fast_path(fwd["conic_opacity"])[idx]
    czz = fwd["conic_opacity"][idx, 5].astype(np.float64)
    reg = {"fast": fast, "exact": ~fast, "exact_by_density": ~fast & (czz * 0.5 * g64.LOG2E <= 2),
           "subvoxel_z": 1.0 / np.sqrt(czz) < 1.0}
    counts = {k: int(v.sum()) for k, v in reg.items()}
    print(f"\n{label}: {len(idx)} Gaussians compared, {ill} with an ill-conditioned voxel covariance not held to the "
          f"bar; per regime {counts}")
    worst = 0.0
    for k, v in g64.voxel_split(ratio).items():
        per = {name: float(v[m].max()) if m.any() else 0.0 for name, m in reg.items()}
        print(f"  {k:12s} worst {float(v.max()):.3g} x bar; " + ", ".join(f"{n} {x:.3g}" for n, x in per.items()))
        worst = max(worst, float(v.max()))
    for name, n in min_count.items():
        assert counts[name] >= n, f"{label}: regime {name} has {counts[name]} Gaussians, expected >= {n}"
    assert worst <= 1.0, f"{label}: worst element {worst:.3g} x its bar"


@pytest.mark.parametrize("dl_kind", ["ramp", "signed"])
@pytest.mark.parametrize("grid", ["full32", "ragged"])
def test_voxel_sweep_gradients_per_element_against_float64(grid, dl_kind, monkeypatch):
    monkeypatch.setenv("R2X_SPECULATIVE", "0")
    nV = VGRIDS[grid][0]
    cloud = _voxel_sweep_cloud(VGRIDS[grid], seed=nV[1])
    r = np.random.RandomState(21)
    dL = (1.0 + r.rand(*nV) if dl_kind == "ramp" else r.randn(*nV)).astype(np.float32)
    _voxel_check(f"voxel sweep {grid}, dL {dl_kind}", cloud, VGRIDS[grid], dL,
                 {"fast": 150, "exact": 80, "exact_by_density": 8, "subvoxel_z": 80})


@pytest.mark.parametrize("variant", ["modifier0.5", "modifier1.6", "cov3D_precomp"])
def test_voxel_sweep_variants_per_element_against_float64(variant, monkeypatch):
    monkeypatch.setenv("R2X_SPECULATIVE", "0")
    grid = VGRIDS["full32"]
    cloud = _voxel_sweep_cloud(grid, seed=4)
    mod = {"modifier0.5": 0.5, "modifier1.6": 1.6}.get(variant, 1.0)
    cov = None
    if variant == "cov3D_precomp":
        import textbook
        cov = textbook.sigma3(cloud.scales, cloud.rotations)[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].astype(np.float32)
    dL = (1.0 + np.random.RandomState(22).rand(*grid[0])).astype(np.float32)
    _voxel_check(f"voxel sweep {variant}", cloud, grid, dL, {"fast": 100, "exact": 50}, mod, cov)


@pytest.mark.parametrize("dl_kind", ["ramp", "signed"])
@pytest.mark.parametrize("grid", ["full32", "ragged"])
def test_voxel_realistic_cloud_gradients_per_element_against_float64(grid, dl_kind):
    nV = VGRIDS[grid][0]
    cloud = scene.make_cloud(1500, kind="trained", seed=nV[1])
    r = np.random.RandomState(23)
    dL = (1.0 + r.rand(*nV) if dl_kind == "ramp" else r.randn(*nV)).astype(np.float32)
    _voxel_check(f"voxel {grid} trained cloud, dL {dl_kind}", cloud, VGRIDS[grid], dL, {"fast": 500})
