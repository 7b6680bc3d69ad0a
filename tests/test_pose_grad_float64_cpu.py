"""The float64 statement of each Gaussian's view- and projection-matrix gradient contribution
(grad_float64.make_pose_chain) checked on its own, without the kernel:

1. against autograd of test_pose_gpu._restated_image (a float64 torch forward, alpha-cut mask frozen), Gaussian by
   Gaussian, in cone and parallel beam, with scale_modifier and with cov3D_precomp, where no Gaussian reaches the
   1.3 tanfov clamp;
2. against central differences of a float64 forward whose clamped view-space coordinate is frozen (the convention the
   kernel keeps: x_grad_mul / y_grad_mul, J at the clamped t), with Gaussians past the clamp in x, in y and in both;
3. the 1e-7 regularisations: with eps = 1e-7 the statement moves from the exact derivative by what they account for.

The statement is compared with eps = 0 (the exact derivative of the frozen forward); the kernel is judged against the
eps = 1e-7 statement, which is what it computes."""
import math

import numpy as np
import pytest

import grad_float64 as g64
import textbook
from r2_gaussian_b200 import scene
from test_grad_float64_cpu import dl_ramp, dl_signed

torch = pytest.importorskip("torch")

# the 24 pose entries as (matrix, flat index): view[4a + b] (a < 4, b < 3), then proj[4a + (0, 1, 3)[j]]
POSE_ENTRIES = [("view", 4 * a + b) for a in range(4) for b in range(3)] + \
               [("proj", 4 * a + (0, 1, 3)[j]) for a in range(4) for j in range(3)]


def _view(mode, n=64, angle=1.1):
    sc = scene.cone_beam_scanner(n, 64) if mode == 1 else scene.parallel_beam_scanner(n, 64)
    return scene.make_view(sc, angle)


def _tiny_cloud(P, seed):
    from test_pose_gpu import _tiny_cloud
    return _tiny_cloud(P, seed)


def _forward(view16, proj16, mean, Sig, rho, view, frozen=None):
    """One Gaussian's screen-space quantities in float64: (px, py, A, B, C, mu, clamp constants).  Cone beam: a view-space
    coordinate past 1.3 tanfov is clamped, and `frozen` (the constants of a base evaluation) holds the clamped value
    fixed, as the backward does."""
    W, H = view.image_width, view.image_height
    V4, P4 = view16.reshape(4, 4), proj16.reshape(4, 4)
    ph = np.r_[mean, 1.0]
    t = ph @ V4[:, :3]
    hom = ph @ P4
    pw = 1.0 / (hom[3] + 1e-7)
    px = ((hom[0] * pw + 1) * W - 1) * 0.5
    py = ((hom[1] * pw + 1) * H - 1) * 0.5
    fx, fy = W / (2 * view.tanfovx), H / (2 * view.tanfovy)
    consts = [None, None]
    if view.mode == 1:
        tx, ty, tz = t
        lim = (1.3 * view.tanfovx, 1.3 * view.tanfovy)
        tt = [tx, ty]
        for k in range(2):
            r = tt[k] / tz
            if abs(r) > lim[k]:
                consts[k] = tz * math.copysign(lim[k], r) if frozen is None else frozen[k]
                tt[k] = consts[k]
        tx, ty = tt
        ln = math.sqrt(tx * tx + ty * ty + tz * tz)
        J = np.array([[fx / tz, 0, -fx * tx / tz ** 2], [0, fy / tz, -fy * ty / tz ** 2], [tx / ln, ty / ln, tz / ln]])
    else:
        J = np.diag([fx, fy, 1.0])
    M = J @ V4[:3, :3].T
    hat = M @ Sig @ M.T
    a, b, d = hat[0, 0], hat[0, 1], hat[1, 1]
    det2 = a * d - b * b
    mu = math.sqrt(2 * math.pi * np.linalg.det(hat) / det2)
    return px, py, d / det2, -b / det2, a / det2, mu, consts


def _pixels(view):
    ys, xs = np.mgrid[0:view.image_height, 0:view.image_width].astype(np.float64)
    return xs, ys


def _loss(fw, rho, dL, mask, view):
    px, py, A, B, C, mu = fw[:6]
    xs, ys = _pixels(view)
    dx, dy = px - xs, py - ys
    power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
    return float((dL * rho * mu * np.exp(power))[mask].sum())


def _mask_and_moments(fw, rho, dL, view):
    """The contributing pixels of the whole image (power <= 0, alpha >= 1e-5) and the six moments over them."""
    px, py, A, B, C, mu = fw[:6]
    xs, ys = _pixels(view)
    dx, dy = px - xs, py - ys
    power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
    mask = (power <= 0) & (rho * mu * np.exp(power) >= 1e-5)
    t = dL * np.exp(power)
    m = np.array([(t * f)[mask].sum() for f in (1.0, dx, dy, dx * dx, dx * dy, dy * dy)])
    return mask, m


def _statement(view, cloud, g, fw, m, mod=1.0, precomp=False, eps=0.0):
    px, py, A, B, C, mu = fw[:6]
    co = np.array([[A, B, C, float(cloud.density[g, 0])]])
    cov = None
    if precomp:
        cov = textbook.sigma3(cloud.scales[g:g + 1], cloud.rotations[g:g + 1], mod)[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    p = g64.pose_chain_inputs(cloud.means[g:g + 1].astype(np.float64), None if precomp else cloud.scales[g:g + 1],
                              None if precomp else cloud.rotations[g:g + 1], cov, co, np.array([mu]),
                              view.viewmatrix, view.projmatrix)
    chain = g64.make_pose_chain(view.image_width, view.image_height, view.tanfovx, view.tanfovy, view.mode, mod,
                                precomp=precomp, eps=eps)
    return chain(torch.tensor(m), torch.tensor(p[0])).numpy()


def _flat(mats):
    """{view: [16], proj: [16]} -> the 24 pose entries."""
    return np.array([mats[k][i] for k, i in POSE_ENTRIES])


def _per_gaussian(view, cloud, dL, mod=1.0, precomp=False):
    """-> list of (statement with eps = 0, autograd of _restated_image, the Gaussian's base quantities)."""
    from test_pose_gpu import _restated_image
    out = []
    v16, p16 = view.viewmatrix.astype(np.float64).reshape(16), view.projmatrix.astype(np.float64).reshape(16)
    for g in range(cloud.P):
        one = scene.Cloud(cloud.means[g:g + 1], cloud.scales[g:g + 1], cloud.rotations[g:g + 1], cloud.density[g:g + 1])
        Sig = textbook.sigma3(one.scales, one.rotations, mod)[0]
        rho = float(cloud.density[g, 0])
        fw = _forward(v16, p16, cloud.means[g].astype(np.float64), Sig, rho, view)
        mask, m = _mask_and_moments(fw, rho, dL, view)
        if not mask.any():
            continue
        V = torch.tensor(view.viewmatrix, dtype=torch.float64, requires_grad=True)
        Pf = torch.tensor(view.projmatrix, dtype=torch.float64, requires_grad=True)
        rs = _RestatedScaled(one, mod)
        img, _, _ = _restated_image(rs, V, Pf, view, torch.tensor(mask)[None])
        (img * torch.tensor(dL, dtype=torch.float64)).sum().backward()
        ag = _flat({"view": V.grad.reshape(16).numpy(), "proj": Pf.grad.reshape(16).numpy()})
        assert float(V.grad[:, 3].abs().max()) == 0.0 and float(Pf.grad[:, 2].abs().max()) == 0.0
        out.append((_statement(view, cloud, g, fw, m, mod, precomp), ag, (fw, m)))
    return out


class _RestatedScaled:
    """A one-Gaussian cloud for _restated_image with scale_modifier folded into its scales (the restatement has none)."""

    def __init__(self, one, mod):
        self.means, self.rotations, self.density = one.means, one.rotations, one.density
        self.scales = (one.scales.astype(np.float64) * mod) if mod != 1.0 else one.scales


def _worst(rows):
    return max(float(np.abs(s - a).max() / max(np.abs(a).max(), 1e-300)) for s, a, _ in rows)


@pytest.mark.parametrize("dl", ["ramp", "signed"])
@pytest.mark.parametrize("mode", [1, 0], ids=["cone", "parallel"])
def test_statement_is_autograd_of_the_restated_forward_per_gaussian(mode, dl):
    view = _view(mode)
    cloud = _tiny_cloud(24, 4 + mode)
    dL = (dl_ramp if dl == "ramp" else dl_signed)(64, 64, 7).astype(np.float64)
    rows = _per_gaussian(view, cloud, dL)
    assert len(rows) >= 20
    worst = _worst(rows)
    print(f"mode {mode}, dL {dl}: {len(rows)} Gaussians, worst |statement - autograd| / max = {worst:.3g}")
    assert worst <= 1e-9


@pytest.mark.parametrize("variant", ["modifier0.5", "modifier1.6", "cov3D_precomp"])
def test_statement_variants_are_autograd_of_the_restated_forward(variant):
    view = _view(1)
    cloud = _tiny_cloud(16, 9)
    mod = {"modifier0.5": 0.5, "modifier1.6": 1.6}.get(variant, 1.0)
    dL = dl_ramp(64, 64, 8).astype(np.float64)
    rows = _per_gaussian(view, cloud, dL, mod, precomp=(variant == "cov3D_precomp"))
    assert len(rows) >= 12
    assert _worst(rows) <= 1e-9, _worst(rows)


def _clamp_cloud(view, seed):
    """Broad Gaussians centred past 1.3 tanfov in x, in y and in both (and a few inside), that still reach the image."""
    from test_grad_float64_gpu import _unproject
    r = np.random.RandomState(seed)
    W, H = view.image_width, view.image_height
    out_x = lambda side: W / 2 + side * (0.65 * W + 3 + 3 * r.rand()) - 0.5
    out_y = lambda side: H / 2 + side * (0.65 * H + 3 + 3 * r.rand()) - 0.5
    px, py, where = [], [], []
    for side in (-1, 1):
        for _ in range(3):
            px.append(out_x(side)); py.append(r.uniform(8, H - 8)); where.append("x")
            px.append(r.uniform(8, W - 8)); py.append(out_y(side)); where.append("y")
            px.append(out_x(side)); py.append(out_y(-side)); where.append("xy")
    for _ in range(4):
        px.append(r.uniform(8, W - 8)); py.append(r.uniform(8, H - 8)); where.append("none")
    means = _unproject(view, np.array(px), np.array(py))
    per_px = np.linalg.norm(view.campos.astype(np.float64)) * 2 * view.tanfovx / W
    n = len(px)
    scales = per_px * r.uniform(9, 12, (n, 1)) * np.stack([np.ones(n), r.uniform(1.0, 1.8, n), r.uniform(0.8, 1.2, n)], 1)
    q = r.randn(n, 4)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    f = np.float32
    return scene.Cloud(means.astype(f), scales.astype(f), q.astype(f), r.uniform(0.5, 2, (n, 1)).astype(f)), where


def test_statement_is_the_central_difference_of_the_frozen_clamp_forward():
    view = _view(1)
    cloud, where = _clamp_cloud(view, 3)
    dL = dl_signed(64, 64, 9).astype(np.float64)
    v16, p16 = view.viewmatrix.astype(np.float64).reshape(16), view.projmatrix.astype(np.float64).reshape(16)
    seen = {"x": 0, "y": 0, "xy": 0, "none": 0}
    worst = 0.0
    for g in range(cloud.P):
        Sig = textbook.sigma3(cloud.scales[g:g + 1], cloud.rotations[g:g + 1])[0]
        rho = float(cloud.density[g, 0])
        mean = cloud.means[g].astype(np.float64)
        fw = _forward(v16, p16, mean, Sig, rho, view)
        kind = {(True, False): "x", (False, True): "y", (True, True): "xy", (False, False): "none"}[
            (fw[6][0] is not None, fw[6][1] is not None)]
        assert kind == where[g], (g, kind, where[g])
        mask, m = _mask_and_moments(fw, rho, dL, view)
        if mask.sum() < 4:
            continue
        seen[kind] += 1
        stmt = _statement(view, cloud, g, fw, m)
        cd = np.zeros(len(POSE_ENTRIES))
        for e, (mat, i) in enumerate(POSE_ENTRIES):
            h = 1e-5 * max(1.0, abs((v16 if mat == "view" else p16)[i]))
            vals = []
            for s in (1, -1):
                v, p = v16.copy(), p16.copy()
                (v if mat == "view" else p)[i] += s * h
                vals.append(_loss(_forward(v, p, mean, Sig, rho, view, frozen=fw[6]), rho, dL, mask, view))
            cd[e] = (vals[0] - vals[1]) / (2 * h)
        err = float(np.abs(stmt - cd).max() / np.abs(cd).max())
        worst = max(worst, err)
        assert err <= 1e-6, (g, kind, err, stmt, cd)
        if kind != "none":   # the clamped coordinate carries no gradient of its own: J's row of t / |t| still does
            assert np.abs(cd).max() > 0
    print(f"clamp sweep: compared per kind {seen}, worst |statement - central difference| / max = {worst:.3g}")
    assert min(seen.values()) >= 2, seen


def test_regularisations_move_the_statement_by_their_own_size():
    """eps = 1e-7 against eps = 0: the difference is what 1e-7 / det2^2 and 1e-7 / mu account for, and is not 0."""
    view = _view(1)
    cloud = _tiny_cloud(12, 2)
    dL = dl_ramp(64, 64, 3).astype(np.float64)
    v16, p16 = view.viewmatrix.astype(np.float64).reshape(16), view.projmatrix.astype(np.float64).reshape(16)
    for g in range(cloud.P):
        Sig = textbook.sigma3(cloud.scales[g:g + 1], cloud.rotations[g:g + 1])[0]
        rho = float(cloud.density[g, 0])
        fw = _forward(v16, p16, cloud.means[g].astype(np.float64), Sig, rho, view)
        mask, m = _mask_and_moments(fw, rho, dL, view)
        if not mask.any():
            continue
        exact = _statement(view, cloud, g, fw, m)
        reg = _statement(view, cloud, g, fw, m, eps=1e-7)
        A, B, C, mu = fw[2:6]
        det2 = 1.0 / (A * C - B * B)                 # of the 2-D covariance
        rel = 1e-7 / det2 ** 2 + 1e-7 / mu
        d = np.abs(reg - exact)
        assert d.max() > 0 and d.max() <= 4 * rel * np.abs(exact).max() + 1e-300, (g, d.max(), rel)
