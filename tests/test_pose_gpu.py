"""View- and projection-matrix gradients of the rasterizer backward, and per-view pose refinement with them.

1. requesting the matrix gradients changes no other output or gradient, bit for bit, and they are reproducible;
2. / 3. translating / rotating the world through the view matrix equals moving the means, so the matrix gradients
   chained to that motion equal the reference-pinned mean gradients summed over the Gaussians;
4. a float64 torch restatement of the forward (alpha-cut mask and tile rectangles frozen) differentiated by autograd;
5. fitting `PoseCorrection` to perturbed views recovers the poses;
6. an overflowed speculative forward still raises CapacityOverflow from the backward.
"""
import math
import types

import numpy as np
import pytest
import torch

import textbook
from r2_gaussian_b200 import _C, fused, scene
from r2_gaussian_b200.pose import PoseCorrection, se3_exp
from r2_gaussian_b200.rasterization import (GaussianRasterizationSettings, GaussianRasterizer,
                                            rasterize_gaussians_matrices)
from r2_gaussian_b200.render_query import render

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def _view(mode, n, angle):
    sc = scene.cone_beam_scanner(n, 64) if mode == 1 else scene.parallel_beam_scanner(n, 64)
    return scene.make_view(sc, angle)


def _settings(view, t_view, t_proj):
    return GaussianRasterizationSettings(view.image_height, view.image_width, view.tanfovx, view.tanfovy, 1.0, t_view,
                                         t_proj, torch.tensor(view.campos, device=DEV), False, view.mode, False)


def _dl(H, W, seed=0):
    """dL/dimage: a ramp (coherent gradients, no cancellation in the sums) plus seeded noise."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    return (xs / W + 0.5 * ys / H + 0.25 + 0.1 * torch.randn(H, W, generator=g))[None].to(DEV)


def _leaves(cloud, raw=False):
    t = lambda a: torch.tensor(a, device=DEV, requires_grad=True)
    if raw:   # raw parameters whose activations are the cloud's
        d = torch.tensor(cloud.density, dtype=torch.float64)
        return dict(means=t(cloud.means), dens=t(torch.log(torch.expm1(d)).float().numpy()),
                    scales=t(np.log(cloud.scales)), rots=t(cloud.rotations))
    return dict(means=t(cloud.means), dens=t(cloud.density), scales=t(cloud.scales), rots=t(cloud.rotations))


def _run(cloud, view, matrices, raw=False, dL=None):
    """One forward + backward; -> (image, radii, {leaf: grad}, view.grad | None, proj.grad | None)."""
    p = _leaves(cloud, raw)
    m2 = torch.zeros_like(p["means"], requires_grad=True)
    tv = torch.tensor(view.viewmatrix, device=DEV, requires_grad=matrices)
    tp = torch.tensor(view.projmatrix, device=DEV, requires_grad=matrices)
    s = _settings(view, tv.detach(), tp.detach())
    if raw:
        rawp = {"density": p["dens"], "scaling": p["scales"], "rotation": p["rots"], "scale_bound": None}
        if matrices:
            img, radii = fused.rasterize_raw_matrices(p["means"], m2, rawp, tv, tp, s)
        else:
            img, radii = fused.rasterize_raw(p["means"], m2, rawp, s)
    elif matrices:
        img, radii = rasterize_gaussians_matrices(p["means"], m2, p["dens"], p["scales"], p["rots"], None, tv, tp, s)
    else:
        img, radii = GaussianRasterizer(s)(p["means"], m2, p["dens"], p["scales"], p["rots"])
    img.backward(_dl(view.image_height, view.image_width) if dL is None else dL)
    torch.cuda.synchronize()
    grads = {k: v.grad for k, v in p.items()}
    grads["means2D"] = m2.grad
    return img.detach(), radii, grads, tv.grad, tp.grad


def _bits(x):
    return x.contiguous().view(torch.int32)


# ---- 1. nothing changes without matrix gradients ---------------------------------------------------------------------

@pytest.mark.parametrize("raw", [False, True], ids=["plain", "raw"])
@pytest.mark.parametrize("mode", [1, 0], ids=["cone512", "parallel512"])
def test_matrix_gradients_change_nothing_else(mode, raw):
    cloud = scene.make_cloud(100_000, kind="init", seed=0)
    view = _view(mode, 512, 0.9)
    img0, radii0, g0, v0, p0 = _run(cloud, view, False, raw)
    img1, radii1, g1, v1, p1 = _run(cloud, view, True, raw)
    img2, radii2, g2, v2, p2 = _run(cloud, view, True, raw)
    assert v0 is None and p0 is None
    assert torch.equal(_bits(img0), _bits(img1)) and torch.equal(radii0, radii1)
    for k in g0:
        assert torch.equal(_bits(g0[k]), _bits(g1[k])), k
    assert torch.equal(_bits(v1), _bits(v2)) and torch.equal(_bits(p1), _bits(p2))
    assert torch.count_nonzero(v1) > 0 and torch.count_nonzero(p1) > 0
    # entries the rasterizer never reads: the bottom row of the view matrix, row 2 of the projection matrix
    assert torch.count_nonzero(v1[:, 3]) == 0 and torch.count_nonzero(p1[:, 2]) == 0
    assert torch.isfinite(v1).all() and torch.isfinite(p1).all()


def test_empty_cloud_gives_zero_matrix_gradients():
    cloud = scene.make_cloud(8, kind="init", seed=0)
    empty = scene.Cloud(cloud.means[:0], cloud.scales[:0], cloud.rotations[:0], cloud.density[:0])
    img, radii, _, gv, gp = _run(empty, _view(1, 64, 0.3), True)
    assert torch.count_nonzero(img) == 0 and radii.numel() == 0
    assert gv.shape == (4, 4) and gp.shape == (4, 4)
    assert torch.count_nonzero(gv) == 0 and torch.count_nonzero(gp) == 0


# ---- 2. / 3. translation and rotation identities ---------------------------------------------------------------------

def _chain(view, gv, gp):
    """(dL/dd, dL/domega) at 0 of the world motions T -> T Tr(d) and T -> T Rot(omega), from the matrix gradients.
    T = world->camera = viewmatrix^T, F = full projection = projmatrix^T (the matrices are stored transposed)."""
    T, F = view.viewmatrix.astype(np.float64).T, view.projmatrix.astype(np.float64).T
    GT, GF = gv.double().cpu().numpy().T, gp.double().cpu().numpy().T
    dd = T[:, :3].T @ GT[:, 3] + F[:, :3].T @ GF[:, 3]
    dw = np.zeros(3)
    for k in range(3):
        e = np.zeros(3)
        e[k] = 1.0
        Kk = _hat(e)
        dw[k] = (GT[:, :3] * (T[:, :3] @ Kk)).sum() + (GF[:, :3] * (F[:, :3] @ Kk)).sum()
    return dd, dw


def _hat(w):
    return np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]], dtype=np.float64)


@pytest.mark.parametrize("kind", ["init", "trained"])
@pytest.mark.parametrize("mode", [1, 0], ids=["cone", "parallel"])
def test_translation_and_rotation_identities(mode, kind):
    cloud = scene.make_cloud(100_000, kind=kind, seed=3)
    view = _view(mode, 512, 2.1)
    _, _, g, gv, gp = _run(cloud, view, True)
    dd, dw = _chain(view, gv, gp)
    G = g["means"].double().cpu().numpy()
    want_d = G.sum(0)
    assert np.linalg.norm(dd - want_d) <= 1e-4 * np.linalg.norm(want_d), (dd, want_d)
    # rotation: rotating the world leaves a covariance unchanged only when it is isotropic
    iso = type(cloud)(cloud.means, np.repeat(cloud.scales[:, :1], 3, axis=1), cloud.rotations, cloud.density)
    _, _, g, gv, gp = _run(iso, view, True)
    _, dw = _chain(view, gv, gp)
    want_w = np.cross(iso.means.astype(np.float64), g["means"].double().cpu().numpy()).sum(0)
    assert np.linalg.norm(dw - want_w) <= 1e-4 * np.linalg.norm(want_w), (dw, want_w)


# ---- 4. float64 restatement ------------------------------------------------------------------------------------------

def _tiny_cloud(P, seed):
    rng = np.random.RandomState(seed)
    means = (rng.rand(P, 3) - 0.5).astype(np.float32) * 0.9
    scales = rng.uniform(0.02, 0.09, size=(P, 3)).astype(np.float32)
    q = rng.randn(P, 4)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    dens = rng.uniform(0.2, 1.0, size=(P, 1)).astype(np.float32)
    return scene.Cloud(means, scales, q.astype(np.float32), dens)


def _restated_image(cloud, V, Pf, view, mask):
    """Image of the cloud in float64 torch, differentiable in the flat-layout matrices V (view) and Pf (projection).
    `mask` [P,H,W] (pairs that contribute) is held fixed; returns (image, mask computed at these matrices)."""
    H, W = view.image_height, view.image_width
    m = torch.tensor(cloud.means, dtype=torch.float64)
    T, F = V.T, Pf.T
    ph = torch.cat([m, torch.ones(len(m), 1, dtype=torch.float64)], 1)
    t = (ph @ T.T)[:, :3]
    hom = ph @ F.T
    ndc = hom[:, :2] / (hom[:, 3:4] + 1e-7)
    px = ((ndc[:, 0] + 1) * W - 1) * 0.5
    py = ((ndc[:, 1] + 1) * H - 1) * 0.5
    fx, fy = W / (2 * view.tanfovx), H / (2 * view.tanfovy)
    z = torch.zeros(len(m), dtype=torch.float64)
    if view.mode == 0:
        J = torch.tensor([[fx, 0, 0], [0, fy, 0], [0, 0, 1.0]], dtype=torch.float64).expand(len(m), 3, 3)
    else:
        tx, ty, tz = t[:, 0], t[:, 1], t[:, 2]
        assert (tx.abs() / tz < 1.3 * view.tanfovx).all() and (ty.abs() / tz < 1.3 * view.tanfovy).all()
        ln = torch.sqrt(tx * tx + ty * ty + tz * tz)
        J = torch.stack([torch.stack([fx / tz, z, -fx * tx / tz ** 2], -1),
                         torch.stack([z, fy / tz, -fy * ty / tz ** 2], -1),
                         torch.stack([tx / ln, ty / ln, tz / ln], -1)], -2)
    Mx = J @ T[:3, :3]
    Sig = torch.tensor(textbook.sigma3(cloud.scales, cloud.rotations))
    hat = Mx @ Sig @ Mx.transpose(1, 2)
    a, b, d = hat[:, 0, 0], hat[:, 0, 1], hat[:, 1, 1]
    det2 = a * d - b * b
    mu = torch.sqrt(2 * math.pi * torch.linalg.det(hat) / det2)
    A, B, C = d / det2, -b / det2, a / det2
    w = torch.tensor(cloud.density[:, 0], dtype=torch.float64) * mu
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    dx = px[:, None, None] - xs
    dy = py[:, None, None] - ys
    power = -0.5 * (A[:, None, None] * dx * dx + C[:, None, None] * dy * dy) - B[:, None, None] * dx * dy
    alpha = w[:, None, None] * torch.exp(power)
    live = ((power <= 0) & (alpha >= 1e-5)).detach()
    return (torch.where(mask, alpha, torch.zeros_like(alpha))).sum(0), live, (px.detach(), py.detach())


def _rect_mask(px, py, radii, W, H):
    """[P,H,W] pixels inside each Gaussian's tile rectangle (the preprocess's, from its radius)."""
    gx, gy = (W + 15) // 16, (H + 15) // 16
    P = len(radii)
    out = torch.zeros(P, H, W, dtype=torch.bool)
    for g in range(P):
        r = float(radii[g])
        if r <= 0:
            continue
        x0 = min(gx, max(0, int((px[g] - r) / 16))); x1 = min(gx, max(0, int((px[g] + r + 15) / 16)))
        y0 = min(gy, max(0, int((py[g] - r) / 16))); y1 = min(gy, max(0, int((py[g] + r + 15) / 16)))
        out[g, y0 * 16:y1 * 16, x0 * 16:x1 * 16] = True
    return out


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("mode", [1, 0], ids=["cone64", "parallel64"])
def test_matrix_gradients_match_float64_restatement(mode, seed):
    cloud = _tiny_cloud(48 + 16 * (seed - 1), seed)
    view = _view(mode, 64, 0.4 + seed)
    dL = _dl(64, 64, seed)
    img, radii, _, gv, gp = _run(cloud, view, True, dL=dL)
    V = torch.tensor(view.viewmatrix, dtype=torch.float64, requires_grad=True)
    Pf = torch.tensor(view.projmatrix, dtype=torch.float64, requires_grad=True)
    with torch.no_grad():
        _, live, (px, py) = _restated_image(cloud, V, Pf, view, torch.ones(1, dtype=torch.bool))
    mask = live & _rect_mask(px, py, radii.cpu().numpy(), 64, 64)
    ref, _, _ = _restated_image(cloud, V, Pf, view, mask)
    err = (ref - img[0].double().cpu()).abs().max()
    assert err <= 1e-4 * ref.abs().max(), err
    (ref * dL[0].double().cpu()).sum().backward()
    for got, want in ((gv, V.grad), (gp, Pf.grad)):
        got, want = got.double().cpu(), want
        bound = 2e-4 * want.abs() + 2e-5 * want.abs().max()
        assert ((got - want).abs() <= bound).all(), (got, want)


# ---- 5. pose recovery end to end -------------------------------------------------------------------------------------

class _Model:
    """A frozen cloud with the attributes render() reads; `raw_parameters` selects the folded-activation path."""

    def __init__(self, cloud, fused_path):
        t = lambda a: torch.tensor(a, device=DEV)
        self.get_xyz, self.get_density = t(cloud.means), t(cloud.density)
        self.get_scaling, self.get_rotation = t(cloud.scales), t(cloud.rotations)
        if fused_path:
            d = torch.tensor(cloud.density, dtype=torch.float64)
            self._raw = {"density": torch.log(torch.expm1(d)).float().to(DEV), "scaling": torch.log(self.get_scaling),
                         "rotation": self.get_rotation, "scale_bound": None}
            self.raw_parameters = lambda: self._raw

    def get_covariance(self, mod=1.0):
        S = torch.tensor(textbook.sigma3(self.get_scaling.cpu().numpy(), self.get_rotation.cpu().numpy(), mod))
        return S[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].float().to(DEV)


class _Pipe:
    def __init__(self, cov3D_python=False):
        self.debug, self.compute_cov3D_python = False, cov3D_python


def _camera(view):
    wvt = torch.tensor(view.viewmatrix, device=DEV)
    proj = torch.tensor(scene.projection_matrix(view.FoVx, view.FoVy, view.mode).T.copy(), device=DEV)
    full = wvt.unsqueeze(0).bmm(proj.unsqueeze(0)).squeeze(0).contiguous()
    return types.SimpleNamespace(world_view_transform=wvt, projection_matrix=proj, full_proj_transform=full,
                                 camera_center=torch.tensor(view.campos, device=DEV), image_height=view.image_height,
                                 image_width=view.image_width, FoVx=view.FoVx, FoVy=view.FoVy, mode=view.mode)


def test_render_fills_matrix_gradients_on_every_path():
    """render() with a corrected camera: the fused-activation path, the plain path and compute_cov3D_python agree."""
    cloud = scene.make_cloud(20_000, kind="trained", seed=5)
    cam = _camera(_view(1, 256, 1.3))
    out = []
    for fused_path, cov_py in ((True, False), (False, False), (False, True)):
        corr = PoseCorrection(1, device=DEV)
        img = render(corr(cam, 0), _Model(cloud, fused_path), _Pipe(cov_py))["render"]
        (img * _dl(256, 256)).sum().backward()
        out.append(torch.cat([corr.omega.grad[0], corr.nu.grad[0]]).double().cpu())
    assert torch.count_nonzero(out[0]) == 6
    for o in out[1:]:
        assert torch.allclose(o, out[0], rtol=1e-3, atol=1e-4 * float(out[0].abs().max())), (o, out[0])


def test_pose_recovery_end_to_end():
    torch.manual_seed(0)
    cloud = scene.make_cloud(20_000, kind="trained", seed=11)
    model, pipe = _Model(cloud, True), _Pipe()
    sc = scene.cone_beam_scanner(256, 64)
    views = scene.make_views(sc, 24)
    true_cams = [_camera(v) for v in views]
    with torch.no_grad():
        targets = [render(c, model, pipe)["render"] for c in true_cams]
    rng = np.random.RandomState(7)
    n = len(views)
    axis = rng.randn(n, 3); axis /= np.linalg.norm(axis, axis=1, keepdims=True)
    shift = rng.randn(n, 3); shift /= np.linalg.norm(shift, axis=1, keepdims=True)
    w_p = torch.tensor(axis * math.radians(0.5))
    n_p = torch.tensor(shift * 0.01 * sc["DSO"])
    cams = []
    for c, w, v in zip(true_cams, w_p, n_p):   # perturbed camera: T_p = exp(xi_p) T
        E = se3_exp(w, v).to(DEV)
        wvt = (E @ c.world_view_transform.double().T).T.float().contiguous()
        full = wvt.unsqueeze(0).bmm(c.projection_matrix.unsqueeze(0)).squeeze(0).contiguous()
        cams.append(types.SimpleNamespace(**dict(vars(c), world_view_transform=wvt, full_proj_transform=full)))
    corr = PoseCorrection(n, device=DEV)
    steps = 400
    opt = torch.optim.Adam([{"params": [corr.omega], "lr": 2e-3}, {"params": [corr.nu], "lr": 1e-2}])
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda s: 0.01 ** (s / steps))

    def errors():   # the fitted correction should undo the perturbation: xi = -xi_p
        w = (corr.omega.detach().double().cpu() + w_p).norm(dim=1).mean().item()
        v = (corr.nu.detach().double().cpu() + n_p).norm(dim=1).mean().item()
        return w, v

    w0, v0 = errors()
    losses = []
    for _ in range(steps):
        opt.zero_grad()
        total = 0.0
        for i in range(n):
            img = render(corr(cams[i], i), model, pipe)["render"]
            loss = (img - targets[i]).abs().mean()
            loss.backward()
            total += loss.item()
        losses.append(total / n)
        opt.step()
        sched.step()
    w1, v1 = errors()
    assert w1 < 0.1 * w0 and v1 < 0.1 * v0, (w0, w1, v0, v1)
    assert losses[-1] <= 0.1 * losses[0], (losses[0], losses[-1])


# ---- 6. capacity ----------------------------------------------------------------------------------------------------

def test_overflowed_speculative_forward_raises_with_matrix_gradients():
    cloud = scene.make_cloud(3000, kind="trained", seed=4)
    view = _view(1, 128, 0.8)
    key = _C.raster_key(DEV, cloud.P, view.image_width, view.image_height)
    _C._Workspace.hints.pop(key, None)
    _run(cloud, view, True)                               # first call of the shape: synchronous, sets the hint
    big = type(cloud)(cloud.means, np.clip(cloud.scales * 6.0, 0, 0.9).astype(np.float32), cloud.rotations,
                      cloud.density)
    with pytest.raises(_C.CapacityOverflow):
        _run(big, view, True)
    img, _, g, gv, gp = _run(big, view, True)              # the hint was raised: the repeat fits
    _C._Workspace.hints.pop(key, None)
    img_s, _, g_s, gv_s, gp_s = _run(big, view, True)      # synchronous reference run
    assert torch.equal(img, img_s) and torch.equal(gv, gv_s) and torch.equal(gp, gp_s)
    assert torch.equal(g["means"], g_s["means"])
