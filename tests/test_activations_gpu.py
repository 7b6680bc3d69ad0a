"""The folded activations (fused.py: softplus, bounded sigmoid / exp and normalize inside the preprocess kernels,
gradients with respect to the RAW parameters from the per-Gaussian backward kernels) element by element against
float64, and scale_modifier != 1 through every path that takes it.

Adam scales each parameter's step by that parameter's own gradient history, so what training needs is a small RELATIVE
error per element, also on the Gaussians whose gradients are small: the bars here are per element, not tied to the
largest gradient of the array.  The engineered clouds sweep one raw parameter at a time across a lattice; the raw path
runs next to the plain path (the kernels on the activated values) and, wherever both forwards left bit-identical stage
outputs, the two gradients differ by the activation factor alone."""
import types

import numpy as np
import pytest

import util
from r2_gaussian_b200 import scene

torch = pytest.importorskip("torch")
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                      # unit roundoff of float32
N = 256                             # Gaussians per engineered cloud
NV, SV, CTR = (64, 64, 64), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0)
BOUND = (0.002, 0.3)                # scale range of the bounded-sigmoid sweep
VIEWS = {"cone": scene.make_view(scene.cone_beam_scanner(256, 64), 0.4),
         "parallel": scene.make_view(scene.parallel_beam_scanner(256, 64), 0.4)}
# |q| = 1 exactly, so q * 2^k is normalised exactly in float32 by the kernel and by F.normalize alike
HURWITZ = np.array([(1, 0, 0, 0), (.5, .5, .5, .5), (.5, -.5, .5, .5), (.5, .5, -.5, .5), (.5, .5, .5, -.5),
                    (0, 1, 0, 0), (.5, -.5, -.5, .5), (0, 0, 0, 1)], np.float32)
ROT_K = np.r_[np.arange(-20, 21), -41, -45]       # 2^-41, 2^-45: |q| below F.normalize's 1e-12 clamp
INF = np.inf
# bucket edges of each sweep, over the swept raw value (rotation: the exponent k)
EDGES = {"density": [-14, -11, -9, -6.9, 0, 20, 26], "scale_exp": [-INF, np.log(1e-2), np.log(5e-2), INF],
         "scale_sigmoid": [-INF, -4, 4, INF], "rotation": [-INF, -21, 0, INF]}


def _lattice(backend):
    if backend == "voxel":
        # 8 x 8 x 4 voxel indices + a quarter voxel (off every sample point), inside the 64^3 grid
        i = np.arange(8) * 8 + 4.25
        ix, iy, iz = np.meshgrid(i, i, np.arange(4) * 16 + 8.25, indexing="ij")
        return (np.stack([ix, iy, iz], -1).reshape(-1, 3) * (SV[0] / NV[0]) - 1.0).astype(np.float32)
    # 16 x 16 in the plane through the origin that faces the source
    c = VIEWS[backend].campos.astype(np.float64)
    e1 = np.cross([0.0, 0.0, 1.0], c / np.linalg.norm(c))
    e1 /= np.linalg.norm(e1)
    uu, vv = np.meshgrid(np.linspace(-0.8, 0.8, 16), np.linspace(-0.8, 0.8, 16), indexing="ij")
    return (uu.reshape(-1, 1) * e1 + vv.reshape(-1, 1) * np.array([0.0, 0.0, 1.0])).astype(np.float32)


def _sweep(param, backend):
    """Raw parameters of an engineered cloud with `param` swept across the lattice and the others fixed
    -> (raw dict of float32 arrays, scale_bound, swept value of each compared element)."""
    i = np.arange(N)
    dens = np.zeros((N, 1), np.float32)                               # softplus(0) = 0.69
    scal = np.log(np.tile(np.float32([[0.045, 0.03, 0.02]]), (N, 1)))
    rot = HURWITZ[i % len(HURWITZ)]
    bound = None

    def three(s):   # each axis takes the sweep in a different order
        return np.stack([s, np.roll(s, N // 3), np.roll(s, 2 * N // 3)], 1).astype(np.float32)

    if param == "density":
        # torch's softplus switches to the identity for x > 20; -90 and -104: denormal and zero rho
        dens[:, 0] = np.r_[np.linspace(-16, 25, N - 5), 19.999998, 20.0, 20.000002, -90.0, -104.0]
        if backend != "voxel":
            # the rasterizer cuts pairs with rho mu e^power < 1e-5: mu of about 1.5 keeps Gaussians down to raw -11.9
            scal[:] = np.log(np.float32(0.6))
        key = dens[:, 0]
    elif param == "scale_exp":
        scal = three(np.linspace(np.log(2e-3), np.log(0.3), N))
        key = scal
    elif param == "scale_sigmoid":
        scal, bound = three(np.linspace(-12.0, 12.0, N)), BOUND
        key = scal
    else:
        k = ROT_K[i % len(ROT_K)]
        rot = (HURWITZ[i % len(HURWITZ)] * np.exp2(k)[:, None]).astype(np.float32)
        key = k
    return dict(density=dens, scaling=scal.astype(np.float32), rotation=rot), bound, key


def _scale_c(bound):
    """hi - lo as the kernel forms it: float(hi) - float(lo).  GaussianModel's scaling activation multiplies by
    float(hi - lo), which can be one ulp away (not for BOUND); the plain path here takes the kernel's value so that both
    paths get identical scales."""
    return float(np.float32(bound[1]) - np.float32(bound[0])), float(np.float32(bound[0]))


def _activated(raw, bound):
    """The plain path's inputs, on the device: F.softplus, the scales by the kernel's formula, F.normalize."""
    t = {k: torch.tensor(v, device="cuda") for k, v in raw.items()}
    if bound is None:
        sc = torch.exp(t["scaling"])
    else:
        c, lo = _scale_c(bound)
        sc = torch.sigmoid(t["scaling"]) * c + lo
    return F.softplus(t["density"]), sc, F.normalize(t["rotation"])


def _dL(backend, seed=5):
    """Positive (1 + 0.5 U): the moment sums have no cancellation, their sign is fixed."""
    shape = NV if backend == "voxel" else (VIEWS[backend].image_height, VIEWS[backend].image_width)
    return (1.0 + 0.5 * np.random.RandomState(seed).rand(*shape)).astype(np.float32)


STAGE = {"raster": ("xy", "conic_opacity", "mu", "depth"), "voxel": ("xyz_vol", "conic_opacity", "depth")}
RADII = {"raster": ("radii",), "voxel": ("radii_x", "radii_y", "radii_z")}


def _run_raw(backend, means, raw, bound, m, dL):
    """fused.rasterize_raw / voxelize_raw (what render() / query() run) -> (stage outputs, raw gradients)."""
    from r2_gaussian_b200 import fused
    from r2_gaussian_b200.rasterization import GaussianRasterizationSettings
    from r2_gaussian_b200.voxelization import GaussianVoxelizationSettings

    t = {k: torch.tensor(v, device="cuda", requires_grad=True) for k, v in raw.items()}
    pars = dict(t, scale_bound=bound)
    xyz = torch.tensor(means, device="cuda")
    if backend == "voxel":
        s = GaussianVoxelizationSettings(m, *NV, *SV, *CTR, False, False)
        out, radii = fused.voxelize_raw(xyz, pars, s)
        fn = out.grad_fn                                     # ctx of _VoxelizeRaw: its saved forward state
        st = util.voxel_export(N, NV, fn.num_rendered, *fn.saved_tensors[6:9])
        st.update({k: r.cpu().numpy() for k, r in zip(RADII["voxel"], radii)})
        dLt = torch.tensor(dL, device="cuda")
    else:
        v = VIEWS[backend]
        f = lambda a: torch.tensor(a, device="cuda")
        s = GaussianRasterizationSettings(v.image_height, v.image_width, v.tanfovx, v.tanfovy, m, f(v.viewmatrix),
                                          f(v.projmatrix), f(v.campos), False, v.mode, False)
        out, radii = fused.rasterize_raw(xyz, torch.zeros_like(xyz), pars, s)
        fn = out.grad_fn                                     # ctx of _RasterizeRaw
        st = util.raster_export(N, v.image_width, v.image_height, fn.num_rendered, *fn.saved_tensors[4:7])
        st["radii"] = radii.cpu().numpy()
        dLt = torch.tensor(dL, device="cuda")[None]
    out.backward(dLt)
    return st, {k: x.grad.cpu().numpy() for k, x in t.items()}


def _run_plain(backend, means, raw, bound, m, dL):
    """The kernels on the activated values -> (cloud, stage outputs, gradients w.r.t. the activated values)."""
    rho, sc, rot = _activated(raw, bound)
    cloud = scene.Cloud(means, sc.cpu().numpy(), rot.cpu().numpy(), rho.cpu().numpy())
    if backend == "voxel":
        fwd = util.ours_voxel_forward(cloud, NV, SV, CTR, scale_modifier=m)
        return cloud, fwd, util.ours_voxel_backward(cloud, NV, SV, CTR, fwd, dL)
    fwd = util.ours_raster_forward(cloud, VIEWS[backend], scale_modifier=m)
    return cloud, fwd, util.ours_raster_backward(cloud, VIEWS[backend], fwd, dL)


def _same_state(kind, a, b):
    """Visible Gaussians whose stage outputs the two forwards left bit for bit identical -> (same, visible)."""
    vis = np.ones(N, bool)
    same = np.ones(N, bool)
    for k in RADII[kind]:
        vis &= b[k] > 0
        same &= a[k] == b[k]
    for k in STAGE[kind]:
        same &= (a[k].reshape(N, -1).view(np.uint32) == b[k].reshape(N, -1).view(np.uint32)).all(1)
    return same & vis, vis


def _buckets(param, key, live):
    return np.histogram(np.asarray(key, np.float64)[live], bins=EDGES[param])[0]


# Elements with a nonzero gradient in each bucket of EDGES, the smallest count over the three scale modifiers (the CPU
# oracle on the same clouds).  The alpha cuts set the first density bucket: at modifier 1 the rasterizer keeps
# Gaussians down to raw -11.9 (0.5: -11.1), the voxelizer down to -13.5; modifier 0.5 halves the smallest voxelizer
# scales to a third of a voxel, and most of those pass no sample point.
MIN_COUNT = {
    ("density", "cone"): [1, 12, 13, 42, 123, 33], ("density", "parallel"): [1, 12, 13, 42, 123, 33],
    ("density", "voxel"): [14, 12, 13, 42, 123, 33],
    ("scale_exp", "cone"): [246, 246, 276], ("scale_exp", "parallel"): [246, 246, 276],
    ("scale_exp", "voxel"): [180, 180, 210],
    ("scale_sigmoid", "cone"): [255, 255, 258], ("scale_sigmoid", "parallel"): [255, 255, 258],
    ("scale_sigmoid", "voxel"): [51, 51, 54],
    ("rotation", "cone"): [10, 120, 126], ("rotation", "parallel"): [10, 120, 126],
    ("rotation", "voxel"): [10, 120, 126],
}


@pytest.mark.parametrize("modifier", [1.0, 0.5, 1.6])
@pytest.mark.parametrize("backend", ["cone", "parallel", "voxel"])
@pytest.mark.parametrize("param", ["density", "scale_exp", "scale_sigmoid", "rotation"])
def test_raw_gradients_per_element_against_float64(param, backend, modifier, monkeypatch):
    # one synchronous forward per call: a speculative one may overflow a capacity hint left by another sweep
    monkeypatch.setenv("R2X_SPECULATIVE", "0")
    kind = "voxel" if backend == "voxel" else "raster"
    means = _lattice(backend)
    raw, bound, key = _sweep(param, backend)
    dL = _dL(backend)
    st_raw, g_raw = _run_raw(backend, means, raw, bound, modifier, dL)
    cloud, st_plain, g_plain = _run_plain(backend, means, raw, bound, modifier, dL)
    same, vis = _same_state(kind, st_raw, st_plain)
    # the exp-mode scales and the normalised Hurwitz rotations are bit-equal in both paths; the sigmoid-mode scales too,
    # with hi - lo formed as the kernel forms it (_scale_c)
    assert vis.sum() >= 0.9 * N and same.sum() >= 0.9 * vis.sum(), (int(same.sum()), int(vis.sum()))

    if param == "density":
        gp, gr = g_plain["dL_dopacity"][:, 0].astype(np.float64), g_raw["density"][:, 0].astype(np.float64)
        x = raw["density"][:, 0].astype(np.float64)
        # forward rho (conic_opacity w) against F.softplus on the device, to the bit, also where it is denormal / zero
        rho = st_raw["conic_opacity"][:, -1]
        want = F.softplus(torch.tensor(raw["density"], device="cuda")).cpu().numpy()[:, 0]
        ulps = np.abs(rho.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
        assert ulps[vis].max() <= 1, f"forward rho: {ulps[vis].max()} ulp from F.softplus"
        assert vis[-2:].all() and 0.0 < want[-2] < np.finfo(np.float32).tiny and want[-1] == 0.0
        live = same & (gp != 0)
        ref = gp * (1.0 / (1.0 + np.exp(-x)))                              # softplus' = sigmoid, float64
        err = np.abs(gr - ref) / np.abs(np.where(live, ref, 1.0))
        # measured on an H100 (400 W): at most 1.6e-7 over all sweeps; with 1 - expf(-rho) in place of -expm1f(-rho) the
        # worst Gaussian was off by 1.3e-2 (rasterizer, raw -12.2) and 2.4e-2 (voxelizer, raw -13.0)
        worst = f"relative error {err[live].max():.3g} at raw {x[live][err[live].argmax()]:.4g}"
        assert err[live].max() <= 2e-6, f"raw density: {worst}"
        assert (gr[same & (gp == 0)] == 0).all()                          # below the alpha cut: 0 on both paths
    elif param.startswith("scale"):
        gp, gr = g_plain["dL_dscale"].astype(np.float64), g_raw["scaling"].astype(np.float64)
        x = raw["scaling"].astype(np.float64)
        live = same[:, None] & (gp != 0)
        if param == "scale_exp":
            ref = gp * np.exp(x)
            err = np.abs(gr - ref) / np.abs(np.where(live, ref, 1.0))
            worst = f"relative error {err[live].max():.3g}"
            # measured on an H100 (400 W): at most 1.7e-7
            assert err[live].max() <= 2e-6, f"exp-mode scale: {worst}"
        else:
            # torch's float32 chain (mul backward, then sigmoid backward (g (1 - y)) y): the reference's own
            # cancellation in 1 - y, kept for parity.  Measured on an H100 (400 W): at most 3 ulp from that chain, and
            # 8.9e-3 relative from float64 (the chain's own error at raw 12, where 1 - y is 6e-6)
            c, lo = _scale_c(bound)
            s = torch.tensor(raw["scaling"], device="cuda", requires_grad=True)
            (torch.sigmoid(s) * c + lo).backward(torch.tensor(g_plain["dL_dscale"], device="cuda"))
            gt = s.grad.cpu().numpy()
            ulps = np.abs(gr - gt) / np.spacing(np.abs(gt).astype(np.float32)).astype(np.float64)
            assert ulps[live].max() <= 4, f"sigmoid-mode scale: {ulps[live].max()} ulp from torch's chain"
            y = 1.0 / (1.0 + np.exp(-x))
            ref = gp * (np.float64(np.float32(bound[1])) - np.float64(np.float32(bound[0]))) * y * (1.0 - y)
            rel = np.abs(gr - ref) / np.abs(np.where(live, ref, 1.0))
            worst = f"{ulps[live].max():.0f} ulp from torch's chain, relative error from float64 {rel[live].max():.3g}"
        assert (gr[same[:, None] & (gp == 0)] == 0).all()
    else:
        gp, gr = g_plain["dL_drot"].astype(np.float64), g_raw["rotation"].astype(np.float64)
        q = raw["rotation"].astype(np.float64)
        n = np.linalg.norm(q, axis=1, keepdims=True)
        eps = np.float64(np.float32(1e-12))
        qh = q / n
        proj = (gp - qh * (qh * gp).sum(1, keepdims=True)) / n            # d normalize: (I - q^ q^T) g / |q|
        ref = np.where(n >= eps, proj, gp / eps)                          # clamped: q / 1e-12, no projection
        gn = np.linalg.norm(gp, axis=1)
        live = same & (gn > 0)
        err = np.abs(gr - ref).max(1) / (U * gn / np.maximum(n[:, 0], eps))
        # measured on an H100 (400 W): at most 0.92 u |dL/dq^| / |q|; projecting below the clamp as well was off by
        # 3.5e6 u (0.2 |dL/dq^| / 1e-12)
        worst = f"{err[live].max():.3g} u |dL/dq^| / |q|"
        assert err[live].max() <= 8, f"rotation: {worst}"
    counts = _buckets(param, key, live)
    print(f"{param}, {backend}, modifier {modifier}: {worst}; compared per bucket {counts.tolist()}")
    assert (counts >= MIN_COUNT[param, backend]).all(), counts.tolist()


# ---- scale_modifier != 1 against the oracle ------------------------------------------------------------------------
@pytest.mark.parametrize("modifier", [0.5, 1.6])
@pytest.mark.parametrize("name", ["cone_trained_small", "parallel_trained_small"])
def test_raster_scale_modifier_matches_oracle(name, modifier):
    cloud, view = util.case(name)
    ours = util.ours_raster_forward(cloud, view, scale_modifier=modifier)
    orc = util.oracle_raster_forward(cloud, view, scale_modifier=modifier)
    assert ours["R"] == orc["R"]
    np.testing.assert_array_equal(ours["radii"], orc["radii"])
    np.testing.assert_array_equal(ours["tiles_touched"], orc["tiles_touched"])
    vis = orc["radii"] > 0
    for k in ("xy", "depth", "conic_opacity", "mu"):
        np.testing.assert_array_equal(ours[k][vis].view(np.uint32), orc[k][vis].view(np.uint32), err_msg=k)
    assert util.key_multiset_equal(ours["keys"], orc["keys"])
    np.testing.assert_array_equal(ours["ranges"], orc["ranges"])
    scale = float(np.abs(orc["image"]).max())
    assert np.abs(ours["image"].astype(np.float64) - orc["image"]).max() <= 1e-5 * scale + 1e-7
    dL = np.random.RandomState(7).randn(view.image_height, view.image_width).astype(np.float32)
    g = util.ours_raster_backward(cloud, view, ours, dL)
    go = util.oracle_raster_backward(cloud, view, orc, dL, scale_modifier=modifier)
    util.assert_grads_close(g, go, ["dL_dmean2D", "dL_dopacity", "dL_dmu", "dL_dmean3D", "dL_dcov3D", "dL_dscale",
                                    "dL_drot"])


@pytest.mark.parametrize("modifier", [0.5, 1.6])
@pytest.mark.parametrize("grid", [((32, 32, 32), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0)),
                                  ((20, 36, 28), (1.3, 2.0, 1.7), (0.1, -0.05, 0.2))], ids=["full32", "ragged"])
def test_voxel_scale_modifier_matches_oracle(grid, modifier):
    """The bounding radius comes from the unmodified scales (as the reference's): above 1 the footprint is cut there."""
    nV, sV, ctr = grid
    cloud = scene.make_cloud(1500, kind="trained", seed=nV[1])
    ours = util.ours_voxel_forward(cloud, nV, sV, ctr, scale_modifier=modifier)
    orc = util.oracle_voxel_forward(cloud, nV, sV, ctr, scale_modifier=modifier)
    assert ours["R"] == orc["R"]
    for k in ("radii_x", "radii_y", "radii_z", "tiles_touched"):
        np.testing.assert_array_equal(ours[k], orc[k], err_msg=k)
    vis = orc["tiles_touched"] > 0
    for k in ("xyz_vol", "depth"):
        np.testing.assert_array_equal(ours[k][vis].view(np.uint32), orc[k][vis].view(np.uint32), err_msg=k)
    assert util.key_multiset_equal(ours["keys"], orc["keys"])
    np.testing.assert_array_equal(ours["ranges"], orc["ranges"])
    np.testing.assert_allclose(ours["conic_opacity"][vis], orc["conic_opacity"][vis], rtol=2e-6, atol=0)
    scale = float(np.abs(orc["vol"]).max())
    assert np.abs(ours["vol"].astype(np.float64) - orc["vol"]).max() <= 1e-5 * scale + 1e-7
    dL = np.random.RandomState(11).randn(*nV).astype(np.float32)
    g = util.ours_voxel_backward(cloud, nV, sV, ctr, ours, dL)
    go = util.oracle_voxel_backward(cloud, nV, sV, orc, dL, scale_modifier=modifier)
    util.assert_grads_close(g, go, ["dL_dopacity", "dL_dmean3D", "dL_dcov3D", "dL_dscale", "dL_drot"])


def test_native_train_step_at_a_scale_modifier_is_the_autograd_iteration():
    """NativeTrainStep(scaling_modifier=0.7) against render() / query() at 0.7 + the fused losses + autograd +
    FusedAdam: parameters and Adam moments bit for bit."""
    from r2_gaussian_b200 import losses
    from r2_gaussian_b200.render_query import query, render
    from r2_gaussian_b200.train_step import NativeTrainStep
    from test_train_gpu import _make_model, _train_inputs

    pipe = types.SimpleNamespace(compute_cov3D_python=False, debug=False)
    cams, gts, centres = _train_inputs()
    lam_d, lam_tv, n_it, mod = 0.25, 0.05, 5, 0.7
    tv_n, tv_s = [32, 32, 32], [0.5, 0.5, 0.5]
    a, _, _ = _make_model(n=5000, seed=17)
    b, _, _ = _make_model(n=5000, seed=17)
    step = NativeTrainStep(b, lam_d, lam_tv, tv_n, tv_s, scaling_modifier=mod)
    for i in range(1, n_it + 1):
        k = i % len(cams)
        a.update_learning_rate(i); b.update_learning_rate(i)
        pkg = render(cams[k], a, pipe, scaling_modifier=mod)
        total = losses.image_loss(pkg["render"], gts[k], lam_d)["total"]
        total = total + lam_tv * losses.tv_3d_loss(query(a, centres[k], tv_n, tv_s, pipe, scaling_modifier=mod)["vol"],
                                                   "mean")
        total.backward()
        with torch.no_grad():
            a.update_max_radii(pkg["radii"], pkg["visibility_filter"])
            a.add_densification_stats(pkg["viewspace_points"], pkg["visibility_filter"])
        a.optimizer.step()
        a.optimizer.zero_grad(set_to_none=True)
        res = step(cams[k], gts[k], centres[k])
        if i == n_it:
            assert abs(step.total_loss() - total.item()) <= 1e-6 * abs(total.item())
            assert torch.equal(res["radii"], pkg["radii"])
    step.flush()
    for name in ("_xyz", "_density", "_scaling", "_rotation"):
        pa, pb = getattr(a, name), getattr(b, name)
        assert torch.equal(pa, pb), name
        sa, sb = a.optimizer.state[pa], b.optimizer.state[pb]
        assert torch.equal(sa["exp_avg"], sb["exp_avg"]) and torch.equal(sa["exp_avg_sq"], sb["exp_avg_sq"]), name
    assert torch.equal(a.max_radii2D, b.max_radii2D)
