"""The rasterizer's view- and projection-matrix gradients (r2x_raster_backward_pose) against their float64 statement
(grad_float64.make_pose_chain), Gaussian by Gaussian, and the two consumers of matrix-sized gradients at their launch
limits.

1. Per Gaussian.  The backward writes one row of POSE_N partial sums per 256 Gaussians; a culled Gaussian (behind the
   camera, radius 0) contributes exactly 0.  So a cloud with one live Gaussian per 256-slot and 255 culled ones turns
   every row into one Gaussian's float32 contribution, all in one call.  Each is held element by element to the
   module bar of grad_float64 (C_BAR u (|dy/dm| |m|_abs + |dy/dp| |p|) + band): the sweeps of
   test_grad_float64_gpu (every tile column, 0.15-12 px, ragged detector), both beams, scale_modifier, cov3D_precomp,
   Gaussians past the 1.3 tanfov clamp in x, in y and in both, and a scene 10^3 from the origin.  The raw-activation
   call gives the plain call's rows bit for bit.  Every call's dL/dview / dL/dproj is the float64 sum of its rows,
   rounded once (1 ulp: the lane order is not fsum's).
2. Sums at the row limits: P = 1, 255, 256, 257, 256 * 32 +- 1 and realistic clouds against the float64 sum of the
   float64 contributions, with the float32 row reduction added to the bar; at P = 10^6 the sum of the rows.
3. r2x_detector_offset_grad across its block-size and grid limits, and r2x_pose_grad across its zero-fill blocks, the
   series switch, theta near pi and large nu.

Measured on an H100 (700 W): the worst element of the per-Gaussian sweeps is 0.28x the bar (parallel 128 px,
rotation block); Gaussians past the clamp 0.02x; the scene 10^3 from the origin 0.17x in cone beam and 0.89x in
parallel beam (rotation block and projection, where dt_b p_a + 2 (dM^T J)_ab and g2 m_w p_a carry the size of the far
means); the sums at the row limits and of the realistic clouds stay below 0.01x their bar.  Each of these mutations of
the kernel fails at least one test here: the factor 2 of pose[3a + b] dropped, J from the unclamped t, x_grad_mul left
out of dt_pose, the w term of the projection set to 0, pose[13 + 3a] and pose[14 + 3a] swapped, the rows summed in
float32."""
import math

import numpy as np
import pytest

import grad_float64 as g64
import util
from r2_gaussian_b200 import scene
from test_grad_float64_cpu import dl_ramp, dl_signed
from test_grad_float64_gpu import _regimes, _sweep_cloud, _unproject

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
SLOT = 256     # Gaussians per row of pose partial sums


def _view(beam, n, angle=0.9):
    sc = scene.cone_beam_scanner(n, 64) if beam == "cone" else scene.parallel_beam_scanner(n, 64)
    return scene.make_view(sc, angle)


def _translated(view, cloud, c):
    """The same scene moved by c: every mean and the camera (world -> camera composed with a translation by -c)."""
    Tr = np.eye(4)
    Tr[:3, 3] = -np.asarray(c, np.float64)
    vm = (Tr.T @ view.viewmatrix.astype(np.float64)).astype(np.float32)
    pm = (Tr.T @ view.projmatrix.astype(np.float64)).astype(np.float32)
    v = scene.View(**{**view.__dict__, "viewmatrix": vm, "projmatrix": pm,
                      "campos": (view.campos.astype(np.float64) + c).astype(np.float32)})
    moved = scene.Cloud((cloud.means.astype(np.float64) + c).astype(np.float32), cloud.scales, cloud.rotations,
                        cloud.density)
    return v, moved


def _spread(cloud, view):
    """Gaussian i of `cloud` at slot SLOT * i; every other slot holds a Gaussian behind the camera (culled)."""
    n = cloud.P
    behind = (2.0 * view.campos.astype(np.float64)).astype(np.float32)
    means = np.repeat(behind[None], SLOT * n, 0)
    scales = np.full((SLOT * n, 3), 0.01, np.float32)
    rots = np.tile(np.array([[1, 0, 0, 0]], np.float32), (SLOT * n, 1))
    dens = np.ones((SLOT * n, 1), np.float32)
    means[::SLOT], scales[::SLOT], rots[::SLOT], dens[::SLOT] = cloud.means, cloud.scales, cloud.rotations, cloud.density
    return scene.Cloud(means, scales, rots, dens)


class _Capture:
    """Keeps the device buffers `_C._u8` hands out, to read the pose rows back from the backward's own scratch."""

    def __init__(self, monkeypatch):
        from r2_gaussian_b200 import _C
        self.bufs, orig = [], _C._u8

        def u8(nbytes, dev):
            t = orig(nbytes, dev)
            self.bufs.append(t)
            return t
        monkeypatch.setattr(_C, "_u8", u8)

    def rows(self, P):
        from r2_gaussian_b200._lib import load
        nb = int(load().r2x_raster_backward_pose_scratch_bytes(P))
        buf = [t for t in self.bufs if t.numel() == nb][-1]
        self.bufs.clear()
        off = (-buf.data_ptr()) % 256
        n = (max(P, 1) + SLOT - 1) // SLOT
        return buf[off:off + 4 * g64.POSE_N * n].view(torch.float32).reshape(n, g64.POSE_N).cpu().numpy()


def _pose_backward(cap, cloud, view, fwd, dL):
    """r2x_raster_backward_pose on a forward of util.ours_raster_forward -> (rows, dL/dview [16], dL/dproj [16])."""
    from r2_gaussian_b200 import _C
    t = fwd["t"]
    geom, binning, img = fwd["state"]
    radii = torch.tensor(fwd["radii"], device=DEV)
    out = _C.rasterize_gaussians_backward_matrices(
        t["means"], radii, t["scales_in"], t["rots_in"], fwd["scale_modifier"], t["cov_in"] if t["cov_in"].numel()
        else None, t["view"], t["proj"], view.tanfovx, view.tanfovy, torch.tensor(dL, device=DEV)[None], t["campos"],
        geom, fwd["R"], binning, img, view.mode, False)
    torch.cuda.synchronize()
    return cap.rows(cloud.P), out[7].reshape(16).cpu().numpy(), out[8].reshape(16).cpu().numpy()


def _flat_pose(gv, gp):
    """dL/dview [16], dL/dproj [16] -> the POSE_N layout."""
    return np.r_[[gv[4 * a + b] for a in range(4) for b in range(3)],
                 [gp[4 * a + (0, 1, 3)[j]] for a in range(4) for j in range(3)]]


def _assert_sum_of_rows(rows, gv, gp):
    """Each matrix gradient is the float64 sum of its column of rows, rounded once (within 1 ulp), and the entries the
    rasterizer never reads are 0."""
    want = np.array([math.fsum(rows[:, k].astype(np.float64)) for k in range(g64.POSE_N)])
    got = _flat_pose(gv, gp).astype(np.float64)
    ulp = np.spacing(np.abs(want.astype(np.float32))).astype(np.float64)
    assert (np.abs(got - want) <= ulp).all(), np.abs(got - want) / ulp
    assert not gv[3::4].any() and not gp[2::4].any()


def _judge(label, rows, gv, gp, fwd, view, spread, cloud, dL, mod=1.0, cov=None, min_count=None):
    """Row i (Gaussian i of `cloud`, slot SLOT i) against its float64 statement, element by element."""
    _assert_sum_of_rows(rows, gv, gp)
    live_slot = np.arange(cloud.P) * SLOT
    sub = {k: fwd[k][live_slot] for k in ("xy", "conic_opacity", "mu", "radii")}
    assert (fwd["radii"][np.setdiff1d(np.arange(spread.P), live_slot)] == 0).all()
    mom = g64.raster_moments(sub["xy"], sub["conic_opacity"], sub["mu"], sub["radii"], dL)
    chain = g64.make_pose_chain(view.image_width, view.image_height, view.tanfovx, view.tanfovy, view.mode, mod,
                                precomp=cov is not None)
    p = g64.pose_chain_inputs(cloud.means, None if cov is not None else cloud.scales,
                              None if cov is not None else cloud.rotations, cov, sub["conic_opacity"], sub["mu"],
                              view.viewmatrix, view.projmatrix)
    live = (sub["radii"] > 0) & (mom["n_pairs"] > 0)
    well = g64.cond2(sub["conic_opacity"]) <= g64.COND_MAX
    assert not rows[sub["radii"] <= 0].any(), f"{label}: a culled Gaussian contributes"
    idx = np.nonzero(live & well)[0]
    y64, bar, band = g64.reference(mom, p, chain, idx)
    r = g64.compare(rows[idx].astype(np.float64), y64, bar, band)
    assert np.isfinite(r).all(), f"{label}: a contribution or its statement is not finite"
    reg = {k: v[idx] for k, v in _regimes(sub, view, mom, cloud).items()}
    counts = {k: int(v.sum()) for k, v in reg.items()}
    print(f"\n{label}: {len(idx)} Gaussians compared, {int((live & ~well).sum())} with cond(2-D cov) > "
          f"{g64.COND_MAX:g} not held to the bar; per regime {counts}")
    worst = 0.0
    for k in g64.POSE_KEYS:
        v = r[:, g64.POSE_SLICES[k]]
        per = {name: float(v[m].max()) if m.any() else 0.0 for name, m in reg.items()}
        print(f"  {k:10s} worst {float(v.max()):.3g} x bar; " + ", ".join(f"{n} {x:.3g}" for n, x in per.items()))
        worst = max(worst, float(v.max()))
    for name, n in (min_count or {}).items():
        assert counts[name] >= n, f"{label}: regime {name} has {counts[name]} Gaussians, expected >= {n}"
    assert worst <= 1.0, f"{label}: worst element {worst:.3g} x its bar"
    return y64, bar, band


def _sweep_run(monkeypatch, cloud, view, dL, mod=1.0, cov=None):
    monkeypatch.setenv("R2X_SPECULATIVE", "0")
    cap = _Capture(monkeypatch)
    spread = _spread(cloud, view)
    cov_s = None
    if cov is not None:
        cov_s = np.tile(np.array([[1e-4, 0, 0, 1e-4, 0, 1e-4]], np.float32), (spread.P, 1))
        cov_s[::SLOT] = cov
    fwd = util.ours_raster_forward(spread, view, cov3D_precomp=cov_s, scale_modifier=mod)
    rows, gv, gp = _pose_backward(cap, spread, view, fwd, dL)
    return rows, gv, gp, fwd, spread


# ---- 1. per Gaussian -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dl_kind", ["ramp", "signed"])
@pytest.mark.parametrize("beam,n", [("cone", 128), ("parallel", 128), ("cone", 100)], ids=["cone", "parallel", "ragged"])
def test_sweep_pose_contributions_per_gaussian_against_float64(beam, n, dl_kind, monkeypatch):
    view = _view(beam, n)
    cloud = _sweep_cloud(view, seed=n, clamp=(beam == "cone"))
    dL = (dl_ramp if dl_kind == "ramp" else dl_signed)(view.image_height, view.image_width, 11)
    rows, gv, gp, fwd, spread = _sweep_run(monkeypatch, cloud, view, dL)
    mc = {"exact": 150, "fast": 300, "subpixel": 300, "narrow_A2>2": 150, "exact_by_density": 8}
    if beam == "cone":
        mc["clamp"] = 8
    if n % 16:
        mc["partial_tile"] = 20
    _judge(f"pose sweep {beam} {n}px, dL {dl_kind}", rows, gv, gp, fwd, view, spread, cloud, dL, min_count=mc)


@pytest.mark.parametrize("variant", ["modifier0.5", "modifier1.6", "cov3D_precomp"])
def test_sweep_pose_variants_per_gaussian_against_float64(variant, monkeypatch):
    view = _view("cone", 128)
    cloud = _sweep_cloud(view, seed=5)
    mod = {"modifier0.5": 0.5, "modifier1.6": 1.6}.get(variant, 1.0)
    cov = None
    if variant == "cov3D_precomp":
        import textbook
        cov = textbook.sigma3(cloud.scales, cloud.rotations)[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].astype(np.float32)
    dL = dl_ramp(128, 128, 12)
    rows, gv, gp, fwd, spread = _sweep_run(monkeypatch, cloud, view, dL, mod, cov)
    _judge(f"pose sweep {variant}", rows, gv, gp, fwd, view, spread, cloud, dL, mod, cov,
           min_count={"exact": 100, "fast": 200})


def _clamp_sweep_cloud(view, seed):
    """Broad Gaussians centred past 1.3 tanfov in x, in y and in both (x_grad_mul / y_grad_mul = 0, J at the clamped t)
    that still reach the image, at several sizes and shapes; -> (cloud, which coordinate is clamped)."""
    r = np.random.RandomState(seed)
    W, H = view.image_width, view.image_height
    px, py, sig, kind = [], [], [], []
    for side in (-1, 1):
        for i in range(16):
            ox = W / 2 + side * (0.65 * W + 2 + 6 * r.rand()) - 0.5
            oy = H / 2 + side * (0.65 * H + 2 + 6 * r.rand()) - 0.5
            s = 8.0 + 6 * r.rand()
            for k, (x, y) in (("x", (ox, r.uniform(8, H - 8))), ("y", (r.uniform(8, W - 8), oy)),
                              ("xy", (ox, H - 1 - oy))):
                px.append(x); py.append(y); sig.append(s); kind.append(k)
    px, py, sig = np.asarray(px), np.asarray(py), np.asarray(sig)
    means = _unproject(view, px, py)
    per_px = np.linalg.norm(view.campos.astype(np.float64)) * 2 * view.tanfovx / W
    n = len(px)
    scales = (per_px * sig)[:, None] * np.stack([np.ones(n), r.uniform(1.0, 2.0, n), r.uniform(0.8, 1.2, n)], 1)
    q = r.randn(n, 4)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    f = np.float32
    return scene.Cloud(means.astype(f), scales.astype(f), q.astype(f), r.uniform(0.5, 2, (n, 1)).astype(f)), np.array(kind)


@pytest.mark.parametrize("dl_kind", ["ramp", "signed"])
def test_clamped_gaussians_pose_contributions_against_float64(dl_kind, monkeypatch):
    view = _view("cone", 128)
    cloud, kind = _clamp_sweep_cloud(view, 17)
    t = cloud.means.astype(np.float64) @ view.viewmatrix[:3, :3].astype(np.float64) + view.viewmatrix[3, :3]
    cx = np.abs(t[:, 0] / t[:, 2]) > 1.3 * view.tanfovx
    cy = np.abs(t[:, 1] / t[:, 2]) > 1.3 * view.tanfovy
    assert (cx == np.isin(kind, ["x", "xy"])).all() and (cy == np.isin(kind, ["y", "xy"])).all()
    dL = (dl_ramp if dl_kind == "ramp" else dl_signed)(128, 128, 14)
    rows, gv, gp, fwd, spread = _sweep_run(monkeypatch, cloud, view, dL)
    _judge(f"pose clamp sweep, dL {dl_kind}", rows, gv, gp, fwd, view, spread, cloud, dL, min_count={"clamp": 60})
    # every kind reaches the image, so each of the three clamp cases is compared
    live = fwd["radii"][::SLOT] > 0
    for k in ("x", "y", "xy"):
        assert (live & (kind == k)).sum() >= 16, k


@pytest.mark.parametrize("beam", ["cone", "parallel"])
def test_far_scene_pose_contributions_against_float64(beam, monkeypatch):
    """Means ~10^3 from the origin: the rotation block is dt_b p_a + 2 (dM^T J)_ab with |p| ~ 10^3, which cancels to
    the size of a scene at the origin."""
    base = _view(beam, 128)
    cloud0 = _sweep_cloud(base, seed=8)
    view, cloud = _translated(base, cloud0, np.array([700.0, -500.0, 600.0]))
    assert np.abs(cloud.means).min() > 400
    dL = dl_ramp(128, 128, 15)
    rows, gv, gp, fwd, spread = _sweep_run(monkeypatch, cloud, view, dL)
    _judge(f"pose far scene {beam}", rows, gv, gp, fwd, view, spread, cloud, dL, min_count={"fast": 200})


def _exact_quaternions(n, seed):
    """Unit quaternions whose float32 normalisation is exact (integer quadruples of norm 3, 5, 9 and 2; the
    components are k / norm with k a power of two or 0), with random signs and orders."""
    base = [(1, 2, 2, 0), (1, 2, 2, 4), (1, 4, 8, 0), (2, 0, 0, 0), (0, 0, 2, 0)]
    r = np.random.RandomState(seed)
    out = np.zeros((n, 4), np.float32)
    for i in range(n):
        q = np.array(base[i % len(base)], np.float32)[r.permutation(4)] * r.choice([-1, 1], 4)
        out[i] = q
    return out


@pytest.mark.parametrize("beam", ["cone", "parallel"])
def test_raw_activation_call_gives_the_plain_rows_bit_for_bit(beam, monkeypatch):
    """r2x_raster_backward_pose with act (raw scales / rotations / density) against the plain call on the activated
    cloud: the same image, the same rows and the same matrix gradients, bit for bit."""
    from r2_gaussian_b200 import fused
    from r2_gaussian_b200.rasterization import GaussianRasterizationSettings, rasterize_gaussians_matrices
    monkeypatch.setenv("R2X_SPECULATIVE", "0")
    view = _view(beam, 128)
    c0 = _sweep_cloud(view, seed=9)
    raw_q = _exact_quaternions(c0.P, 3)
    spread = _spread(scene.Cloud(c0.means, c0.scales, raw_q, c0.density), view)
    raw_s = torch.tensor(np.log(spread.scales), device=DEV)
    d = spread.density.astype(np.float64)          # softplus(x) = x above 20: such densities are their own raw value
    raw_d = torch.tensor(np.where(d > 20, d, np.log(np.expm1(np.minimum(d, 20)))).astype(np.float32), device=DEV)
    raw_r = torch.tensor(spread.rotations, device=DEV)
    act_s, act_d = torch.exp(raw_s), torch.nn.functional.softplus(raw_d)
    act_r = raw_r / raw_r.norm(dim=1, keepdim=True)
    assert torch.equal(act_r * raw_r.norm(dim=1, keepdim=True), raw_r)      # exact normalisation
    dL = torch.tensor(dl_signed(128, 128, 16), device=DEV)[None]
    cap = _Capture(monkeypatch)
    out = []
    for raw in (True, False):
        means = torch.tensor(spread.means, device=DEV, requires_grad=True)
        m2 = torch.zeros_like(means, requires_grad=True)
        tv = torch.tensor(view.viewmatrix, device=DEV, requires_grad=True)
        tp = torch.tensor(view.projmatrix, device=DEV, requires_grad=True)
        st = GaussianRasterizationSettings(128, 128, view.tanfovx, view.tanfovy, 1.0, tv.detach(), tp.detach(),
                                           torch.tensor(view.campos, device=DEV), False, view.mode, False)
        if raw:
            rawp = {"density": raw_d, "scaling": raw_s, "rotation": raw_r, "scale_bound": None}
            img, _ = fused.rasterize_raw_matrices(means, m2, rawp, tv, tp, st)
        else:
            img, _ = rasterize_gaussians_matrices(means, m2, act_d, act_s, act_r, None, tv, tp, st)
        img.backward(dL)
        torch.cuda.synchronize()
        out.append((img.detach(), cap.rows(spread.P), tv.grad.clone(), tp.grad.clone()))
    (i0, r0, v0, p0), (i1, r1, v1, p1) = out
    assert torch.equal(i0.view(torch.int32), i1.view(torch.int32)), "the activated cloud is not the raw one's"
    live = np.abs(r1).sum(1) > 0
    print(f"\nraw {beam}: {int(live.sum())} live rows of {len(r1)}")
    assert live.sum() >= 500
    assert np.array_equal(r0.view(np.int32), r1.view(np.int32))
    assert torch.equal(v0.view(torch.int32), v1.view(torch.int32)) and torch.equal(p0.view(torch.int32), p1.view(torch.int32))


# ---- 2. sums at the row limits ---------------------------------------------------------------------------------------

def _sum_check(label, cap, cloud, view, dL):
    """dL/dview, dL/dproj of the whole cloud against the float64 sum of the float64 contributions.  Bar per entry:
    sum over the Gaussians of (C_BAR u bar + band) -- each contribution as held above -- plus the float32 reduction of
    each row, at most 255 additions of partials no larger than the row's sum |contribution| (256 u sum |y|), plus the
    final rounding (1 ulp).  Gaussians not held to the per-Gaussian bar (cond2) enter with 256 u |y| more."""
    fwd = util.ours_raster_forward(cloud, view)
    rows, gv, gp = _pose_backward(cap, cloud, view, fwd, dL)
    _assert_sum_of_rows(rows, gv, gp)
    mom = g64.raster_moments(fwd["xy"], fwd["conic_opacity"], fwd["mu"], fwd["radii"], dL)
    chain = g64.make_pose_chain(view.image_width, view.image_height, view.tanfovx, view.tanfovy, view.mode)
    p = g64.pose_chain_inputs(cloud.means, cloud.scales, cloud.rotations, None, fwd["conic_opacity"], fwd["mu"],
                              view.viewmatrix, view.projmatrix)
    idx = np.nonzero((fwd["radii"] > 0) & (mom["n_pairs"] + mom["n_border"] > 0))[0]
    got = _flat_pose(gv, gp).astype(np.float64)
    if len(idx) == 0:
        assert not got.any()
        return 0
    y64, bar, band = g64.reference(mom, p, chain, idx)
    ill = g64.cond2(fwd["conic_opacity"][idx]) > g64.COND_MAX
    want = np.array([math.fsum(y64[:, k]) for k in range(g64.POSE_N)])
    per = g64.C_BAR * g64.U * bar + band + np.where(ill[:, None], 256 * g64.U * np.abs(y64), 0.0)
    rowsum = np.zeros_like(y64)
    np.add.at(rowsum, idx // SLOT, np.abs(y64))
    tol = per.sum(0) + 256 * g64.U * rowsum.sum(0) + np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    r = np.abs(got - want) / tol
    print(f"{label}: {len(idx)} Gaussians, {len(rows)} rows; worst " +
          ", ".join(f"{k} {float(r[g64.POSE_SLICES[k]].max()):.3g}" for k in g64.POSE_KEYS) + " x bar")
    assert r.max() <= 1.0, (label, r)
    return len(idx)


@pytest.mark.parametrize("beam", ["cone", "parallel"])
def test_pose_sums_at_the_row_limits_against_float64(beam, monkeypatch):
    monkeypatch.setenv("R2X_SPECULATIVE", "0")
    cap = _Capture(monkeypatch)
    view = _view(beam, 512, 2.3)
    dL = dl_signed(512, 512, 17)
    n = 0
    for P in (1, 255, 256, 257, SLOT * 32 - 1, SLOT * 32 + 1):
        n += _sum_check(f"{beam} P={P}", cap, scene.make_cloud(P, kind="trained", seed=P), view, dL)
    assert n >= 8000


@pytest.mark.parametrize("name", ["cone_trained_small", "cone_trained_ragged"])
def test_pose_sums_of_realistic_clouds_against_float64(name, monkeypatch):
    cap = _Capture(monkeypatch)
    cloud, view = util.case(name)
    assert _sum_check(name, cap, cloud, view, dl_ramp(view.image_height, view.image_width, 18)) >= 1000


@pytest.mark.parametrize("beam", ["cone", "parallel"])
def test_pose_sum_of_a_million_gaussians_is_the_sum_of_its_rows(beam, monkeypatch):
    """P = 10^6 (3907 rows, the last one partial): the matrix gradients are the float64 sum of the rows rounded once,
    and a second call is bit for bit the first."""
    cap = _Capture(monkeypatch)
    view = _view(beam, 512, 0.6)
    cloud = scene.make_cloud(1_000_000, kind="trained", seed=19)
    dL = dl_signed(512, 512, 19)
    fwd = util.ours_raster_forward(cloud, view, export=False)
    a = _pose_backward(cap, cloud, view, fwd, dL)
    b = _pose_backward(cap, cloud, view, fwd, dL)
    assert a[0].shape == (3907, g64.POSE_N)
    _assert_sum_of_rows(*a)
    assert (np.abs(a[0]).sum(1) > 0).all()
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.int32), y.view(np.int32))


# ---- 3. the consumers at their launch limits -------------------------------------------------------------------------

KPER = 2048            # r2x_detector.cu: kPerBlock = 8 * 256
KMAX = 1024            # kMaxBlocks


@pytest.mark.parametrize("N", [0, 1, KPER - 1, KPER, KPER + 1, KPER * KMAX - 1, KPER * KMAX, KPER * KMAX + 1,
                               3 * KPER * KMAX + 12345])
def test_detector_offset_grad_at_its_launch_limits(N):
    """dL/ds = (2 / W) sum of dL_dmean2D[..., 0] over N = P n_views rows, against the float64 sum rounded once."""
    from r2_gaussian_b200.detector import DetectorOffset
    n_views = 3 if N % 3 == 0 and N > 0 else 1
    P = N // n_views
    g = torch.randn((n_views, P, 3), device=DEV, generator=torch.Generator("cuda").manual_seed(N)) + 0.25
    det = DetectorOffset(DEV)
    W = 384
    got = det.grad_from(g, W).clone()
    want = 2.0 / W * math.fsum(g[..., 0].double().cpu().numpy().reshape(-1).tolist())
    sp = float(np.spacing(np.float32(abs(want))))
    print(f"N={N}: {float(got):.9g} vs {want:.12g}")
    if N == 0:
        assert float(got) == 0.0
    else:
        assert abs(float(got) - want) <= sp, (float(got), want, sp)


def _pose_cases():
    """(omega, nu) in float64: theta^2 just either side of the series switch (1e-2), near pi, and large nu."""
    rng = np.random.RandomState(23)
    out = []
    for theta, nu in ((0.1 * (1 - 1e-6), 0.1), (0.1 * (1 + 1e-6), 0.1), (math.pi - 1e-3, 0.5), (math.pi * (1 - 1e-7), 2.0),
                      (0.3, 300.0), (1e-3, 1e3)):
        ax = rng.randn(3)
        ax /= np.linalg.norm(ax)
        out.append(((ax * theta).astype(np.float32), (rng.randn(3) * nu).astype(np.float32)))
    th2 = [float(np.sum(w.astype(np.float64) ** 2)) for w, _ in out]
    assert th2[0] < 1e-2 < th2[1]
    return out


@pytest.mark.parametrize("n_views", [1, 42, 43, 1000])
def test_pose_grad_at_its_launch_limits_against_float64_autograd(n_views):
    from test_pose_train_gpu import _camera, _corrections
    cam = _camera(0.9, det=128)
    g = torch.Generator("cuda").manual_seed(n_views)
    gv = torch.randn((4, 4), device=DEV, generator=g)
    gp = torch.randn((4, 4), device=DEV, generator=g)
    i = n_views - 1
    for k, (w, v) in enumerate(_pose_cases()):
        for anchor in (-1, i, 0 if i else -1):
            c32, c64 = _corrections(n_views, i, w, v)
            out = c32.device_camera(cam, i, anchor=anchor)
            g32 = torch.autograd.grad((out.world_view_transform, out.full_proj_transform), (c32.omega, c32.nu), (gv, gp))
            rows = [j for j in range(n_views) if j != i]
            for name, x in zip(("omega", "nu"), g32):
                assert x.shape == (n_views, 3)
                assert torch.count_nonzero(x[rows]) == 0, (k, name)
            if anchor == i:
                assert torch.count_nonzero(g32[0]) == 0 and torch.count_nonzero(g32[1]) == 0, k
                continue
            rv, rf = c64.matrices(cam, i)
            g64_ = torch.autograd.grad((rv, rf), (c64.omega, c64.nu), (gv.double(), gp.double()))
            for name, x, r in zip(("omega", "nu"), g32, g64_):
                r_i = r[i].detach()
                bound = 2 * np.spacing(np.abs(r_i.float().cpu().numpy())).astype(np.float64) + 1e-7 * float(r_i.abs().max())
                err = np.abs(x[i].double().cpu().numpy() - r_i.cpu().numpy())
                assert (err <= bound).all(), (n_views, k, anchor, name, x[i], r_i)
                assert torch.count_nonzero(x[i]) > 0, (k, name)
