"""The rasterizer's image and the voxelizer's volume pixel by pixel against their float64 statement (forward_float64.py),
on the kernels' own stage outputs, and the render-only entry points bit for bit against the forward.

A bar relative to the image maximum says little about faint pixels; the per-pixel bar holds every pixel to the error
its own terms allow.  The cases put Gaussians at every column of a tile and sub-pixel offsets (both render paths,
partial tiles), at the fast-path limits (A2 = 2, log2 w = 20 and -100, the determinant ratio), at the anchor limit of
the multiplicative forward differences, over a wide dynamic range (faint pixels below 1e-4 of the maximum), in crowded
tiles of several work-plan chunks, on the radix path, with scale_modifier, cov3D_precomp, the raw-parameter forward and
a batched-views call.  Each case prints its worst |got - S64| / bar per regime and asserts a minimum number of judged
pixels per regime, so that none drops out silently.  Pixels reached by a Gaussian whose 2-D covariance is
ill-conditioned (grad_float64.COND_MAX) are counted, not judged."""
import numpy as np
import pytest

import forward_float64 as f64
import grad_float64 as g64
import regime_cases as rc
import textbook
import util
from r2_gaussian_b200 import scene
from test_grad_float64_cpu import VGRIDS

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

L2E = g64.LOG2E


# ---- judging ----------------------------------------------------------------------------------------------------------
def _report(label, r, regimes, held, mins, st):
    counts = {k: int((m & held).sum()) for k, m in regimes.items()}
    worst = {k: float(r[m & held].max(initial=0.0)) for k, m in regimes.items()}
    clean = held & (st["n_border"] == 0)     # a borderline pair alone can take a pixel to ~1x: half of it is the bar
    print(f"\n{label}: {int(held.sum())} judged, per regime " + ", ".join(
        f"{k} {counts[k]} (worst {worst[k]:.3g} x bar)" for k in regimes)
        + f"; without a borderline pair worst {float(r[clean].max(initial=0.0)):.3g} x bar")
    for k, n in mins.items():
        assert counts[k] >= n, f"{label}: regime {k} has {counts[k]} judged elements, expected >= {n}"
    w = float(r[held].max(initial=0.0))
    assert w <= 1.0, f"{label}: worst element {w:.3g} x its bar"
    return worst


def judge_raster(label, image, fwd, W, H, mins, tiles=None):
    """image [H, W] against the statement of the stage outputs fwd (xy, conic_opacity, mu, ranges, point_list)."""
    co, mu = fwd["conic_opacity"], fwd["mu"]
    fast = g64.fast_path(co, mu)
    flags = {"fast": fast, "exact": ~fast, "ill": g64.cond2(co) > g64.COND_MAX}
    st = f64.raster_statement(fwd["xy"], co, mu, fwd["ranges"], fwd["point_list"], W, H, "kernel", flags, tiles)
    image = np.asarray(image, np.float64)
    judged = f64.judged(st)
    if tiles is None:
        assert np.all(image[~judged] == 0.0), f"{label}: a pixel no pair reaches is not 0"
    held = judged & (st["count_ill"] == 0)
    n_list = (fwd["ranges"][:, 1] - fwd["ranges"][:, 0]).astype(np.int64)
    gx = (W + 15) // 16
    crowded = np.zeros((H, W), bool)
    for t in np.nonzero(n_list > f64.PLAN_CHUNK)[0]:
        crowded[(t // gx) * 16:(t // gx) * 16 + 16, (t % gx) * 16:(t % gx) * 16 + 16] = True
    regimes = {"fast": st["count_fast"] > 0, "exact": st["count_exact"] > 0, "crowded": judged & crowded,
               "faint": f64.faint(st)}
    print(f"\n{label}: {int((judged & ~held).sum())} pixels reached by an ill-conditioned conic, not judged")
    return _report(label, f64.ratio(image, st), regimes, held, mins, st)


def judge_voxel(label, vol, fwd, nV, mins, tiles=None):
    co = fwd["conic_opacity"]
    fast = g64.voxel_fast_path(co)
    flags = {"fast": fast, "exact": ~fast}
    st = f64.voxel_statement(fwd["xyz_vol"], co, fwd["ranges"], fwd["point_list"], nV, flags, tiles)
    vol = np.asarray(vol, np.float64)
    judged = f64.judged(st)
    if tiles is None:
        assert np.all(vol[~judged] == 0.0), f"{label}: a voxel no pair reaches is not 0"
    g = [-(-n // 8) for n in nV]
    n_list = (fwd["ranges"][:, 1] - fwd["ranges"][:, 0]).astype(np.int64)
    crowded = np.zeros(tuple(nV), bool)
    for t in np.nonzero(n_list > f64.PLAN_CHUNK)[0]:
        tx, ty, tz = t % g[0], (t // g[0]) % g[1], t // (g[0] * g[1])
        crowded[8 * tx:8 * tx + 8, 8 * ty:8 * ty + 8, 8 * tz:8 * tz + 8] = True
    regimes = {"fast": st["count_fast"] > 0, "exact": st["count_exact"] > 0, "crowded": judged & crowded,
               "faint": f64.faint(st)}
    return _report(label, f64.ratio(vol, st), regimes, judged, mins, st)


# ---- raster cases -----------------------------------------------------------------------------------------------------
def _par_px(view):
    """World length of one pixel of a parallel-beam view."""
    return 2.0 * view.tanfovx / view.image_width


def _dens_for(cloud, view, lw):
    """Densities that give the Gaussians of `cloud` log2 w = lw (w = rho mu, mu from the float64 textbook)."""
    mu = textbook.project(cloud.means, cloud.scales, cloud.rotations, view.viewmatrix, view.projmatrix,
                          view.image_width, view.image_height, view.tanfovx, view.tanfovy, view.mode)["mu"]
    return (2.0 ** np.asarray(lw, np.float64) / mu).astype(np.float32).reshape(-1, 1)


def _axis_scales(view, sx_px, sy_px, n):
    """Scales along view x / view y of a parallel view (in pixels), a thin depth extent."""
    ax = rc.view_axes(view)
    sc = np.full((n, 3), 0.01)
    sc[:, ax[0]] = np.asarray(sx_px) * _par_px(view)
    sc[:, ax[1]] = np.asarray(sy_px) * _par_px(view)
    return sc


def dynamic_range_cloud(view, seed=31):
    """A few bright Gaussians with log2 w just under and just over 20 (the fast-path limit) over a field of faint ones
    whose w runs from 1e-5 to 1e-2: most of the field's pixels lie below 1e-4 of the image maximum."""
    r = np.random.RandomState(seed)
    W, H = view.image_width, view.image_height
    nb, nf = 8, 600
    bright = rc.make(rc.world_at_pixel(view, r.uniform(10, W - 10, nb), r.uniform(10, H - 10, nb)),
                     _axis_scales(view, r.uniform(1.5, 4, nb), r.uniform(1.5, 4, nb), nb))
    bright.density[:] = _dens_for(bright, view, np.where(np.arange(nb) % 2, 20.05, 19.95))
    faint = rc.make(rc.world_at_pixel(view, r.uniform(0, W, nf), r.uniform(0, H, nf), 5.0 + r.uniform(-0.3, 0.3, nf)),
                    _axis_scales(view, r.uniform(0.4, 4, nf), r.uniform(0.4, 4, nf), nf))
    faint.density[:] = _dens_for(faint, view, np.log2(10.0 ** r.uniform(-5, -2, nf)))
    return rc.concat(bright, faint)


def anchor_cloud(view, seed=33):
    """Fast-path Gaussians at A2 = 2 (just under) and log2 w = 20 (just under) whose first contributing pixel of the row
    through the centre is the last of a 4-pixel run, so that the run's anchor, 3 pixels further out, has the largest q
    the fast path allows; and wide Gaussians of tiny A2 whose runs start far from the centre."""
    r = np.random.RandomState(seed)
    W, H = view.image_width, view.image_height
    gx, gy = W // 16, H // 16
    a2, lw = 1.999, 19.99
    ext = np.sqrt((rc.K["Q_CUT"] + lw) / a2)            # |dx| of the last contributing pixel on the centre row
    sx = np.sqrt(0.5 * L2E / a2)                         # A2 = log2(e) / (2 sx^2), sx in pixels
    px, py = [], []
    for i in range(64):
        tx, ty, run = 1 + i % (gx - 2), 1 + (i // (gx - 2)) % (gy - 2), 4 * (i % 4)
        px.append(16 * tx + run + 3 + ext - 0.02 - 0.3 * r.rand() * (i % 2))
        py.append(16 * ty + r.randint(2, 14))            # an integer row: dy = 0 on the centre row
    n = len(px)
    narrow = rc.make(rc.world_at_pixel(view, np.array(px), np.array(py), 5.0 + r.uniform(-0.3, 0.3, n)),
                     _axis_scales(view, np.full(n, sx), r.uniform(0.7, 3.0, n), n))
    narrow.density[:] = _dens_for(narrow, view, np.full(n, lw))
    m = 24
    wide = rc.make(rc.world_at_pixel(view, r.uniform(0, W, m), r.uniform(0, H, m), 5.0 + r.uniform(-0.3, 0.3, m)),
                   _axis_scales(view, r.uniform(8, 14, m), r.uniform(0.6, 2.0, m), m))
    wide.density[:] = _dens_for(wide, view, np.where(np.arange(m) % 2, 19.99, r.uniform(0, 12, m)))
    return rc.concat(narrow, wide)


def _sweep(beam, n):
    from test_grad_float64_gpu import _sweep_cloud, _view

    view = _view(beam, n)
    return _sweep_cloud(view, seed=n, clamp=(beam == "cone")), view


def _engineered(name):
    case = {c.name: c for c in rc.raster_fastpath_cases()}[name]
    return case.cloud, case.view


def crowded_cloud(view, seed=35):
    """1500 Gaussians of 0.5 to 4 px over the central 48 x 48 pixels of a 64 x 64 detector, w from 1e-4 to 10: every
    tile's list spans several work-plan chunks."""
    r = np.random.RandomState(seed)
    n = 1500
    c = rc.make(rc.world_at_pixel(view, r.uniform(8, 56, n), r.uniform(8, 56, n), 5.0 + r.uniform(-0.3, 0.3, n)),
                _axis_scales(view, r.uniform(0.5, 4, n), r.uniform(0.5, 4, n), n))
    c.density[:] = _dens_for(c, view, np.log2(10.0 ** r.uniform(-4, 1, n)))
    return c


def _crowded():
    view = rc.parallel_view(64, 64)
    return crowded_cloud(view), view


RASTER_CASES = {
    # name: (cloud, view builder, forward keywords, minimum judged pixels per regime)
    "sweep_cone": (lambda: _sweep("cone", 128), {}, {"fast": 6000, "exact": 5000, "faint": 10000}),
    "sweep_parallel": (lambda: _sweep("parallel", 128), {}, {"fast": 5000, "exact": 8000, "faint": 10000}),
    "sweep_ragged": (lambda: _sweep("cone", 100), {}, {"fast": 2500, "exact": 5000, "faint": 5000}),
    "dynamic_range": (lambda: (dynamic_range_cloud(rc.parallel_view(128, 128)), rc.parallel_view(128, 128)), {},
                      {"fast": 10000, "exact": 2500, "faint": 10000}),
    "fast_a2": (lambda: _engineered("raster_fast_a2"), {}, {"fast": 50000, "exact": 500}),
    "fast_lw_max": (lambda: _engineered("raster_fast_lw_max"), {}, {"fast": 50000, "exact": 50000}),
    "fast_lw_min": (lambda: _engineered("raster_fast_lw_min"), {}, {"fast": 50000}),
    "fast_det": (lambda: _engineered("raster_fast_det"), {}, {"fast": 40000}),
    "anchor": (lambda: (anchor_cloud(rc.parallel_view(128, 128)), rc.parallel_view(128, 128)), {},
               {"fast": 10000, "faint": 5000}),
    "cone_init_small": (lambda: util.case("cone_init_small"), {}, {"fast": 16000, "crowded": 8000}),
    "cone_trained_small": (lambda: util.case("cone_trained_small"), {}, {"fast": 16000, "crowded": 8000}),
    "parallel_trained_small": (lambda: util.case("parallel_trained_small"), {}, {"fast": 9000, "crowded": 8000}),
    "cone_trained_ragged": (lambda: util.case("cone_trained_ragged"), {}, {"fast": 10000, "crowded": 5000}),
    "cone_trained_mid": (lambda: util.case("cone_trained_mid"), {}, {"fast": 60000, "crowded": 40000, "faint": 400}),
    "crowded": (_crowded, {}, {"fast": 3000, "exact": 1000, "crowded": 3000}),
    "radix": (lambda: util.case("det_272x3856"), {}, {"fast": 200000, "crowded": 90000, "faint": 8000}),
    "modifier0.5": (lambda: util.case("cone_trained_small"), {"scale_modifier": 0.5},
                    {"fast": 16000, "exact": 10, "crowded": 5000, "faint": 100}),
    "cov3D_precomp": (lambda: util.case("cone_trained_small"), {"cov3D_precomp": True},
                      {"fast": 16000, "crowded": 8000}),
}


def _cov(cloud):
    return textbook.sigma3(cloud.scales, cloud.rotations)[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].astype(np.float32)


@pytest.mark.parametrize("name", list(RASTER_CASES))
def test_raster_image_per_pixel_against_float64(name, monkeypatch):
    monkeypatch.setenv("R2X_SPECULATIVE", "0")
    build, kw, mins = RASTER_CASES[name]
    cloud, view = build()
    kw = dict(kw)
    if kw.pop("cov3D_precomp", False):
        kw["cov3D_precomp"] = _cov(cloud)
    fwd = util.ours_raster_forward(cloud, view, **kw)
    judge_raster(name, fwd["image"], fwd, view.image_width, view.image_height, mins)


def test_raw_parameter_forward_per_pixel_against_float64(monkeypatch):
    """fused.rasterize_raw (the activations folded into the preprocess) on the density sweep of test_activations_gpu.
    With grad enabled the call is speculative once its shape has a capacity hint, and a hint left by another test of the
    same shape can be too small; the synchronous forward re-runs until its binning buffer fits, so the image and the
    exported lists are always those of a complete forward."""
    monkeypatch.setenv("R2X_SPECULATIVE", "0")
    from r2_gaussian_b200 import fused
    from r2_gaussian_b200.rasterization import GaussianRasterizationSettings
    from test_activations_gpu import N, VIEWS, _lattice, _sweep

    raw, bound, _ = _sweep("density", "cone")
    v = VIEWS["cone"]
    f = lambda a: torch.tensor(a, device="cuda")
    s = GaussianRasterizationSettings(v.image_height, v.image_width, v.tanfovx, v.tanfovy, 1.0, f(v.viewmatrix),
                                      f(v.projmatrix), f(v.campos), False, v.mode, False)
    pars = dict({k: f(x).requires_grad_(True) for k, x in raw.items()}, scale_bound=bound)   # keeps the saved state
    xyz = f(_lattice("cone"))
    out, _ = fused.rasterize_raw(xyz, torch.zeros_like(xyz), pars, s)
    fn = out.grad_fn
    st = util.raster_export(N, v.image_width, v.image_height, fn.num_rendered, *fn.saved_tensors[4:7])
    judge_raster("raw density sweep, cone", out.detach()[0].cpu().numpy(), st, v.image_width, v.image_height,
                 {"fast": 3000})


def test_batched_views_image_per_pixel_against_float64():
    """rasterize_views: view 1 of 3 against the statement of view 1's single-view stage outputs (the batched images are
    bit for bit single-view renders, tests/test_views_gpu.py)."""
    from r2_gaussian_b200 import _C

    sc = scene.cone_beam_scanner(128, 64)
    views = [scene.make_view(sc, a) for a in (0.9, 2.1, 4.0)]
    cloud, _ = util.case("cone_trained_small")
    t = util.to_torch(cloud, None)
    V = torch.tensor(np.stack([v.viewmatrix for v in views]), device="cuda")
    Pm = torch.tensor(np.stack([v.projmatrix for v in views]), device="cuda")
    v1 = views[1]
    R, imgs, radii, *_ = _C.rasterize_views(t["means"], t["dens"], t["scales"], t["rots"], 1.0, V, Pm, v1.tanfovx,
                                            v1.tanfovy, 128, 128, v1.mode)
    fwd = util.ours_raster_forward(cloud, v1)
    assert np.array_equal(fwd["radii"], radii[1].cpu().numpy())
    judge_raster("views 1 of 3", imgs[1].cpu().numpy(), fwd, 128, 128, {"fast": 10000})


# ---- voxel cases ------------------------------------------------------------------------------------------------------
def voxel_dynamic_range_cloud(grid, seed=41):
    """Bright Gaussians with log2 rho just under and just over 20 over a field of faint ones, rho 1e-6 to 1e-3."""
    nV, sV, _ = grid
    r = np.random.RandomState(seed)
    dv = sV[0] / nV[0]
    nb, nf = 6, 500
    bright = rc.make(rc.voxel_world(grid, r.uniform(4, np.array(nV) - 4, (nb, 3))), r.uniform(1.0, 2.5, (nb, 3)) * dv,
                     dens=2.0 ** np.where(np.arange(nb) % 2, 20.05, 19.95))
    faint = rc.make(rc.voxel_world(grid, r.uniform(0, np.array(nV), (nf, 3))), r.uniform(0.4, 3.0, (nf, 3)) * dv,
                    dens=10.0 ** r.uniform(-6, -3, nf))
    return rc.concat(bright, faint)


def _voxel_sweep(grid_name):
    from test_grad_float64_gpu import _voxel_sweep_cloud

    grid = VGRIDS[grid_name]
    return _voxel_sweep_cloud(grid, seed=grid[0][1]), grid


TWO_LEVEL = ((144, 136, 136), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0))
VOXEL_CASES = {
    "sweep_full32": (lambda: _voxel_sweep("full32"), {"fast": 30000, "exact": 30000, "faint": 8000}),
    "sweep_ragged": (lambda: _voxel_sweep("ragged"), {"fast": 18000, "exact": 18000, "faint": 5000}),
    "dynamic_range": (lambda: (voxel_dynamic_range_cloud(VGRIDS["full32"]), VGRIDS["full32"]),
                      {"fast": 30000, "exact": 15000, "faint": 20000}),
    "two_level": (lambda: (scene.make_cloud(1200, kind="trained", seed=9), TWO_LEVEL),
                  {"fast": 2500000, "crowded": 250000}),
}


@pytest.mark.parametrize("name", list(VOXEL_CASES))
def test_voxel_volume_per_voxel_against_float64(name, monkeypatch):
    monkeypatch.setenv("R2X_SPECULATIVE", "0")
    monkeypatch.delenv("R2X_VOXEL_BINNING", raising=False)
    build, mins = VOXEL_CASES[name]
    cloud, (nV, sV, ctr) = build()
    if name == "two_level":
        assert rc.binning_path(nV) == "two_level"
    fwd = util.ours_voxel_forward(cloud, nV, sV, ctr)
    judge_voxel(name, fwd["vol"], fwd, nV, mins)


def voxel_crowded_case():
    """regime_cases.voxel_counts_case (filler Gaussians, every alpha below the cut, make R large: chunks of 2 segments),
    with 1500 more Gaussians of 0.5 to 2 voxels (0.85 to 1.2 along z: the fast path) in its first two z layers over
    2 x 2 tiles: each of those tiles holds several chunks of two segments.  Every Gaussian above the cut lies in the
    first two z layers of tiles."""
    case = rc.voxel_counts_case()
    r = np.random.RandomState(43)
    n = 1500
    pv = np.c_[r.uniform(24, 40, (n, 2)), r.uniform(3, 5, n)]
    dv = case.grid[1][0] / case.grid[0][0]
    sc = np.c_[r.uniform(0.5, 2.0, (n, 2)), r.uniform(0.85, 1.2, n)] * dv
    cluster = rc.make(rc.voxel_world(case.grid, pv), sc, dens=10.0 ** r.uniform(-3, 0.5, n))
    return rc.concat(case.cloud, cluster), case.grid


def test_voxel_crowded_tiles_per_voxel_against_float64():
    """Only the first two z layers of tiles are stated (the fillers make the whole grid costly on the CPU); the rest of
    the volume must be exactly 0."""
    cloud, (nV, sV, ctr) = voxel_crowded_case()
    fwd = util.ours_voxel_forward(cloud, nV, sV, ctr)
    g = [-(-n // 8) for n in nV]
    n_list = (fwd["ranges"][:, 1] - fwd["ranges"][:, 0]).astype(np.int64)
    print(f"\nvoxel crowded: R = {fwd['R']}, largest tile list {int(n_list.max())}")
    judge_voxel("voxel crowded", fwd["vol"], fwd, nV, {"fast": 2000, "crowded": 1000}, tiles=np.arange(2 * g[0] * g[1]))
    assert np.all(fwd["vol"][:, :, 16:] == 0.0)


# ---- render-only, bit for bit -----------------------------------------------------------------------------------------
def _assert_render_only(eng, want, label):
    for i in range(3):
        got = eng.render_only(out=torch.full_like(want, float("nan")))
        torch.cuda.synchronize()
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), f"{label}: render_only call {i} differs"


RASTER_RENDER_ONLY = {
    "direct": (lambda: util.case("cone_trained_small"), None),
    "radix": (lambda: util.case("cone_trained_bigdet"), None),
    "crowded": (_crowded, None),
    "capacity_64R": (lambda: util.case("cone_trained_small"), "64R"),
    "grown": (lambda: util.case("cone_trained_small"), 1),
}


@pytest.mark.parametrize("name", list(RASTER_RENDER_ONLY))
def test_raster_render_only_is_the_forward_bit_for_bit(name):
    """RasterEngine.render_only (the work plan rewound, the render kernel relaunched with R = capacity, so on another
    grid than the forward's) equals the forward's image, three calls in a row."""
    from r2_gaussian_b200.engine import RasterEngine

    build, cap = RASTER_RENDER_ONLY[name]
    cloud, view = build()
    t = util.to_torch(cloud, view)
    args = (t["means"], t["dens"], t["scales"], t["rots"], t["view"], t["proj"], t["campos"], view.tanfovx,
            view.tanfovy, view.mode)
    eng = RasterEngine(cloud.P, view.image_width, view.image_height, "cuda", capacity=None if cap == "64R" else cap)
    R = eng.fit(*args)
    if cap == "64R":
        eng._reserve(64 * R)
        eng.forward(*args)
        assert eng.check()
    if cap == 1:
        assert eng.capacity >= R > 1
    want = eng.out.clone()
    torch.cuda.synchronize()
    print(f"\nraster {name}: R = {R}, capacity {eng.capacity}")
    _assert_render_only(eng, want, f"raster {name}")


VOXEL_RENDER_ONLY = {
    "direct": (VGRIDS["full32"], None, None),
    "two_level": (TWO_LEVEL, None, None),
    "radix": (TWO_LEVEL, "radix", None),
    "capacity_64R": (VGRIDS["full32"], None, "64R"),
    "grown": (VGRIDS["ragged"], None, 1),
}


@pytest.mark.parametrize("name", list(VOXEL_RENDER_ONLY) + ["crowded"])
def test_voxel_render_only_is_the_forward_bit_for_bit(name, monkeypatch):
    from r2_gaussian_b200.engine import VoxelEngine

    if name == "crowded":
        cloud, (nV, sV, ctr) = voxel_crowded_case()
        binning, cap = None, None
    else:
        (nV, sV, ctr), binning, cap = VOXEL_RENDER_ONLY[name]
        cloud = scene.make_cloud(1200, kind="trained", seed=9)
    if binning:
        monkeypatch.setenv("R2X_VOXEL_BINNING", binning)
    else:
        monkeypatch.delenv("R2X_VOXEL_BINNING", raising=False)
    t = util.to_torch(cloud, None)
    args = (t["means"], t["dens"], t["scales"], t["rots"], sV, ctr)
    eng = VoxelEngine(cloud.P, nV, "cuda", capacity=None if cap == "64R" else cap)
    R = eng.fit(*args)
    if cap == "64R":
        eng._reserve(64 * R)
        eng.forward(*args)
        assert eng.check()
    if cap == 1:
        assert eng.capacity >= R > 1
    want = eng.out.clone()
    torch.cuda.synchronize()
    print(f"\nvoxel {name}: R = {R}, capacity {eng.capacity}")
    _assert_render_only(eng, want, f"voxel {name}")
