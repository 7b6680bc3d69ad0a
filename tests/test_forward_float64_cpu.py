"""The float64 statement of the forwards (forward_float64.py) checked before it judges a kernel: it agrees with the
textbook math, the CPU oracle's image and volume meet its per-pixel bar, and the bar catches errors of the kind the
render kernels could make -- small relative to a pixel, invisible next to the image maximum."""
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

RASTER_CASES = ["cone_trained_small", "parallel_trained_small", "cone_trained_ragged"]


def _sorted_lists(fwd):
    """The oracle's tile lists (depth order) in the render kernel's order: ascending Gaussian id per tile."""
    pl = fwd["point_list"].copy()
    for a, b in fwd["ranges"]:
        pl[a:b] = np.sort(pl[a:b])
    return pl


def _raster(fwd, view, chain="oracle", pl=None):
    return f64.raster_statement(fwd["xy"], fwd["conic_opacity"], fwd["mu"], fwd["ranges"],
                                fwd["point_list"] if pl is None else pl, view.image_width, view.image_height, chain)


def _voxel(fwd, nV):
    return f64.voxel_statement(fwd["xyz_vol"], fwd["conic_opacity"], fwd["ranges"], fwd["point_list"], nV)


# ---- the statement against independent math -------------------------------------------------------------------------
def test_raster_statement_agrees_with_the_textbook():
    """textbook.render_bruteforce, one Gaussian at a time over its tile rectangle, on the oracle's stage outputs: equal
    to ~1e-12 of the pixel's absolute sum wherever no pair is borderline."""
    cloud, view = util.case("cone_trained_small")
    fwd = util.oracle_raster_forward(cloud, view)
    W, H = view.image_width, view.image_height
    st = _raster(fwd, view)
    img = np.zeros((H, W))
    w = (fwd["conic_opacity"][:, 3] * fwd["mu"]).astype(np.float32).astype(np.float64)
    for g in np.nonzero(fwd["radii"] > 0)[0]:
        x0, y0, x1, y1 = g64.tile_rect(fwd["xy"][g, 0], fwd["xy"][g, 1], fwd["radii"][g], W, H)
        if x1 <= x0 or y1 <= y0:
            continue
        X0, Y0, X1, Y1 = 16 * x0, 16 * y0, min(16 * x1, W), min(16 * y1, H)
        xy = fwd["xy"][g:g + 1].astype(np.float64) - [X0, Y0]
        img[Y0:Y1, X0:X1] += textbook.render_bruteforce(xy, fwd["conic_opacity"][g:g + 1, :3].astype(np.float64),
                                                        w[g:g + 1], X1 - X0, Y1 - Y0)
    clean = st["n_border"] == 0
    err = np.abs(st["S64"] - img)[clean] / (st["abs_all"][clean] + 1e-300)
    print(f"raster: {int(clean.sum())} pixels without a borderline pair, worst {err.max():.3g} of sum|t|")
    assert clean.sum() > 0.9 * H * W and err.max() <= 1e-12
    assert (st["n"] > 0).sum() > 0.5 * H * W


def test_voxel_statement_agrees_with_a_per_gaussian_sum():
    """Gaussian by Gaussian over its tile cube (the other loop order of the per-tile statement): equal to ~1e-12."""
    nV, sV, ctr = VGRIDS["ragged"]
    cloud = scene.make_cloud(1500, kind="trained", seed=nV[1])
    fwd = util.oracle_voxel_forward(cloud, nV, sV, ctr)
    st = _voxel(fwd, nV)
    vol = np.zeros(nV)
    co = fwd["conic_opacity"].astype(np.float64)
    for g in np.nonzero(fwd["tiles_touched"] > 0)[0]:
        x0, y0, z0, x1, y1, z1 = g64.voxel_cube(fwd["xyz_vol"][g], fwd["radii_x"][g], fwd["radii_y"][g],
                                                fwd["radii_z"][g], nV)
        ax = [np.arange(8 * lo, min(8 * hi, n)) + 0.5 for lo, hi, n in ((x0, x1, nV[0]), (y0, y1, nV[1]), (z0, z1, nV[2]))]
        X, Y, Z = np.meshgrid(*ax, indexing="ij")
        d = [float(fwd["xyz_vol"][g, k]) - v for k, v in enumerate((X, Y, Z))]
        M = np.array([[co[g, 0], co[g, 1], co[g, 2]], [co[g, 1], co[g, 3], co[g, 4]], [co[g, 2], co[g, 4], co[g, 5]]])
        power = -0.5 * sum(M[i, j] * d[i] * d[j] for i in range(3) for j in range(3))
        a = co[g, 6] * np.exp(np.minimum(power, 0.0))
        vol[8 * x0:8 * x0 + X.shape[0], 8 * y0:8 * y0 + X.shape[1], 8 * z0:8 * z0 + X.shape[2]] += np.where(
            (power <= 0) & (a >= g64.VALPHA_CUT), a, 0.0)
    clean = st["n_border"] == 0
    err = np.abs(st["S64"] - vol)[clean] / (st["abs_all"][clean] + 1e-300)
    print(f"voxel: {int(clean.sum())} voxels without a borderline pair, worst {err.max():.3g} of sum|t|")
    assert clean.sum() > 0.9 * vol.size and err.max() <= 1e-12
    assert (st["n"] > 0).sum() > 0.3 * vol.size


# ---- the oracle meets the bar ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", RASTER_CASES)
def test_oracle_image_meets_the_per_pixel_bar(name):
    cloud, view = util.case(name)
    fwd = util.oracle_raster_forward(cloud, view)
    st = _raster(fwd, view, "oracle")
    r = f64.ratio(fwd["image"], st)
    faint = f64.faint(st)
    print(f"oracle {name}: worst {r.max():.3g} x bar over {int(f64.judged(st).sum())} pixels, "
          f"faint ({int(faint.sum())}) {r[faint].max(initial=0):.3g}")
    assert r.max() <= 1.0


@pytest.mark.parametrize("grid", ["full32", "ragged"])
def test_oracle_volume_meets_the_per_voxel_bar(grid):
    nV, sV, ctr = VGRIDS[grid]
    cloud = scene.make_cloud(1500, kind="trained", seed=nV[1])
    fwd = util.oracle_voxel_forward(cloud, nV, sV, ctr)
    st = _voxel(fwd, nV)
    r = f64.ratio(fwd["vol"], st)
    faint = f64.faint(st)
    print(f"oracle voxel {grid}: worst {r.max():.3g} x bar over {int(f64.judged(st).sum())} voxels, "
          f"faint ({int(faint.sum())}) {r[faint].max(initial=0):.3g}")
    assert r.max() <= 1.0


# ---- sensitivity: the bar catches a render kernel that is subtly wrong ---------------------------------------------
f32 = np.float32
CUT = f32(g64.ALPHA_CUT)


def _fma(a, b, c):
    return (np.asarray(a, np.float64) * b + c).astype(f32)


def _ex2(x):
    with np.errstate(over="ignore"):
        return np.exp2(np.asarray(x, np.float64)).astype(f32)


def _emulate_image(fwd, pl, W, H, mutation=None):
    """float32 numpy emulation of the forward render: per tile, each Gaussian's 16 rows by render_fast_16 (two halves
    of render_fast_8: q0 and d0 at the anchors dx0 and dx0 - 4, alpha advanced by E *= D, D *= K, the cut tested on
    alpha itself) or render_exact_8, summed per slice of each chunk, the slices and then the chunks in order.
    mutation: None, 'cut_on_G' (the cut tested on G = alpha / w), 'faint_scaled' (the terms of Gaussians with w below
    1e-3 of the brightest scaled by 1 + 2e-4), 'K_bf16' (K = exp2f(-(2 A2 truncated to bf16)))."""
    co = fwd["conic_opacity"].astype(f32)
    L2E = f32(1.4426950408889634)
    A2 = (co[:, 0] * f32(0.5 * L2E)).astype(f32)
    B2 = (co[:, 1] * L2E).astype(f32)
    C2 = (co[:, 2] * f32(0.5 * L2E)).astype(f32)
    w = (co[:, 3] * fwd["mu"].astype(f32)).astype(f32)
    with np.errstate(divide="ignore"):
        lw = np.where(w > 0, np.log2(w.astype(np.float64)), -np.inf).astype(f32)
    twoA2 = (A2 + A2).astype(f32)
    if mutation == "K_bf16":
        twoA2 = (twoA2.view(np.uint32) & np.uint32(0xFFFF0000)).view(f32)
    K = _ex2(-twoA2.astype(np.float64))
    fast = g64.fast_path(fwd["conic_opacity"], fwd["mu"])
    scale = np.where(w < 1e-3 * w.max(), 1.0 + 2e-4, 1.0) if mutation == "faint_scaled" else np.ones(len(w))
    img = np.zeros((H, W), f32)
    gx = (W + 15) // 16
    for t in np.nonzero(fwd["ranges"][:, 1] > fwd["ranges"][:, 0])[0]:
        a, b = (int(v) for v in fwd["ranges"][t])
        ids = pl[a:b].astype(np.int64)
        x0, y0 = f32(16 * (t % gx)), f32(16 * (t // gx))
        n = len(ids)
        x, y = fwd["xy"][ids, 0].astype(f32)[:, None], fwd["xy"][ids, 1].astype(f32)[:, None]
        a2, b2, c2, k_, l_, w_ = (v[ids][:, None] for v in (A2, B2, C2, K, lw, w))
        dy = (y - (y0 + np.arange(16, dtype=f32))[None]).astype(f32)            # [n, 16 rows]
        bdy = (b2 * dy).astype(f32)
        terms = np.zeros((n, 16, 16))
        # fast path
        cdy2 = _fma((c2 * dy).astype(f32), dy, -l_)
        aa2 = (a2 + a2).astype(f32)
        e0 = (a2 - bdy).astype(f32)
        for half in (0, 8):
            dx0 = (x - (x0 + f32(half))).astype(f32)
            for run in (0, 1):
                DX = (dx0 - f32(4 * run)).astype(f32)
                Q = _fma(DX, _fma(a2, DX, bdy), cdy2)
                Dd = _fma(-aa2, DX, e0)
                E, D = _ex2(-Q.astype(np.float64)), _ex2(-Dd.astype(np.float64))
                with np.errstate(invalid="ignore", over="ignore"):
                    for k in range(4):
                        if k:
                            E = (E * D).astype(f32)
                            if k < 3:
                                D = (D * k_).astype(f32)
                        test = E / w_ if mutation == "cut_on_G" else E
                        terms[:, :, half + 4 * run + k] = np.where(test >= CUT, E, 0.0)
        # exact path
        cdy2e = ((c2 * dy).astype(f32) * dy).astype(f32)
        qmax = (f32(rc.K["Q_CUT"]) + l_).astype(f32)
        ex = ~fast[ids]
        for col in range(16):
            dx = (x - (x0 + f32(col))).astype(f32)
            q = _fma(dx, _fma(a2, dx, bdy), cdy2e)
            ok = (q >= 0) & (q <= qmax) & ~np.signbit(q)
            terms[ex, :, col] = np.where(ok, w_ * _ex2(-q.astype(np.float64)).astype(np.float64), 0.0)[ex]
        terms *= scale[ids][:, None, None]
        # the kernel's order: slices of each chunk, then the slices in order, then the chunks in chunk order
        ch, pos, nch = f64._plan_slices(n)
        tile = np.zeros((16, 16), f32)
        for c in range(nch):
            part = np.zeros((f64.RW_SLICES, 16, 16), f32)
            for j in np.nonzero(ch == c)[0]:
                s = pos[j] % f64.RW_SLICES
                part[s] = (part[s] + terms[j]).astype(f32)
            v = part[0]
            for s in range(1, f64.RW_SLICES):
                v = (v + part[s]).astype(f32)
            tile = v if c == 0 else (tile + v).astype(f32)
        ys, xs = int(y0), int(x0)
        img[ys:ys + 16, xs:xs + 16] = tile[:min(16, H - ys), :min(16, W - xs)]
    return img


@pytest.fixture(scope="module")
def sweep():
    from test_grad_float64_gpu import _sweep_cloud, _view

    view = _view("cone", 128)
    cloud = _sweep_cloud(view, seed=128, clamp=True)
    fwd = util.oracle_raster_forward(cloud, view)
    pl = _sorted_lists(fwd)
    st = _raster(fwd, view, "kernel", pl)
    return fwd, pl, view, st


def test_emulated_render_kernel_meets_the_bar(sweep):
    fwd, pl, view, st = sweep
    img = _emulate_image(fwd, pl, view.image_width, view.image_height)
    r = f64.ratio(img, st)
    faint = f64.faint(st)
    print(f"emulated kernel: worst {r.max():.3g} x bar, faint ({int(faint.sum())}) {r[faint].max():.3g}; "
          f"old bar {f64.old_bar_ratio(img, st):.3g}")
    assert r.max() <= 1.0 and faint.sum() >= 200


@pytest.mark.parametrize("mutation", ["cut_on_G", "faint_scaled", "K_bf16"])
def test_bar_catches_what_the_image_maximum_hides(sweep, mutation):
    """Each mutation of the emulated render kernel stays within the suite's 1e-5 max|image| bar and misses the
    per-pixel bar."""
    fwd, pl, view, st = sweep
    img = _emulate_image(fwd, pl, view.image_width, view.image_height, mutation)
    r = f64.ratio(img, st)
    old = f64.old_bar_ratio(img, st)
    print(f"{mutation}: per-pixel bar {r.max():.3g} x ({int((r > 1).sum())} pixels over), old bar {old:.3g} x")
    assert old <= 1.0
    assert r.max() > 1.0
