"""Training on B views per iteration: the raw-parameter batched rasterizer, the batched loss and statistics kernels,
`NativeTrainStep` with a list of cameras and `trainer --batch_size`.

1. r2x_raster_forward_views_async_raw: image v and radii[v] bit for bit the single-view raw forward of view v (both
   binning paths, parallel beam, a ragged detector, views that cull different Gaussians, P = 0, a repeated overflow);
2. r2x_raster_backward_views_raw: every raw gradient the view-order float32 sum of the single-view raw backwards,
   dL/dmean2D per view bit for bit;
3. r2x_image_loss_views / r2x_densify_stats_views bit for bit the single-view calls, the guarded no-op included;
4. NativeTrainStep at B = 4 is the autograd batched iteration bit for bit, with and without TV;
5. the batched objective is the loop of single-view render() iterations plus B lambda_tv TV (1e-6 relative);
6. an overflowed batched iteration changes nothing and is repeated once with the same views;
7. at B = 1 the trainer launches the kernels of the parent commit;
8. a generate_data scene trained at B = 4 beats its FDK initialisation by at least 3 dB of psnr_3d.
"""
import json
import math
import os
import random
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import util
from r2_gaussian_b200 import _C, scene
from r2_gaussian_b200._lib import ActivationDesc, load
from r2_gaussian_b200.fused import rasterize_raw
from r2_gaussian_b200.rasterization import GaussianRasterizationSettings

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BOUND = (0.0005, 1.0)


def _bit_equal(a, b):
    return a.shape == b.shape and a.contiguous().view(torch.int32).equal(b.contiguous().view(torch.int32))


def _raw_inputs(cloud, views):
    """Raw parameters whose activations (softplus, bounded sigmoid, normalize) give back about the cloud's."""
    t = util.to_torch(cloud, None)
    lo, hi = BOUND
    p = ((t["scales"] - lo) / (hi - lo)).clamp(1e-4, 1 - 1e-4)
    raw = {"means": t["means"], "dens": torch.log(torch.expm1(t["dens"].clamp_min(1e-4))),
           "scales": torch.log(p / (1 - p)), "rots": t["rots"] * 1.7}
    raw["views"] = torch.stack([torch.tensor(v.viewmatrix, device="cuda") for v in views])
    raw["projs"] = torch.stack([torch.tensor(v.projmatrix, device="cuda") for v in views])
    act = ActivationDesc()
    act.scale_mode, act.scale_lo, act.scale_hi = 1, lo, hi
    return raw, act


def _settings(view, t, v):
    return GaussianRasterizationSettings(view.image_height, view.image_width, view.tanfovx, view.tanfovy, 1.0,
                                         t["views"][v], t["projs"][v], torch.zeros(3, device="cuda"), False, view.mode,
                                         False)


def _single(t, act, view, v, dL=None):
    """Single-view raw forward (fused.rasterize_raw) and, with dL, its raw gradients."""
    leaves = [t[k].detach().clone().requires_grad_(dL is not None) for k in ("means", "dens", "scales", "rots")]
    m2 = torch.zeros((t["means"].shape[0], 3), device="cuda", requires_grad=dL is not None)
    raw = {"density": leaves[1], "scaling": leaves[2], "rotation": leaves[3],
           "scale_bound": (act.scale_lo, act.scale_hi)}
    image, radii = rasterize_raw(leaves[0], m2, raw, _settings(view, t, v))
    out = dict(image=image[0].detach(), radii=radii)
    if dL is not None:
        g = torch.autograd.grad(image, [m2] + leaves, dL[v:v + 1])
        out.update(zip(("mean2D", "mean3D", "opacity", "scale", "rot"), g))
    return out


def _batched(t, act, views, dL=None):
    v0 = views[0]
    R, images, radii, geom, binning, img = _C.rasterize_views_raw(
        t["means"], t["dens"], t["scales"], t["rots"], 1.0, t["views"], t["projs"], v0.tanfovx, v0.tanfovy,
        v0.image_height, v0.image_width, v0.mode, act)
    out = dict(images=images, radii=radii, R=int(R))
    if dL is not None:
        g = _C.rasterize_views_raw_backward(t["means"], radii, t["scales"], t["rots"], 1.0, t["views"], t["projs"],
                                            v0.tanfovx, v0.tanfovy, dL, geom, R, binning, img, v0.mode, act)
        out.update(zip(("mean2D", "opacity", "mean3D", "cov3D", "scale", "rot"), g))
    return out


def _dL(views, seed=0):
    gen = torch.Generator("cuda").manual_seed(seed)
    return torch.randn((len(views), views[0].image_height, views[0].image_width), device="cuda", generator=gen)


def _check(cloud, views, backward=True, seed=0):
    t, act = _raw_inputs(cloud, views)
    dL = _dL(views, seed) if backward else None
    b = _batched(t, act, views, dL)
    acc = None
    for v, view in enumerate(views):
        s = _single(t, act, view, v, dL)
        assert _bit_equal(b["images"][v], s["image"]), f"view {v}: image differs from the single-view raw render"
        assert b["radii"][v].equal(s["radii"]), f"view {v}: radii differ"
        if backward:
            assert _bit_equal(b["mean2D"][v], s["mean2D"]), f"view {v}: dL/dmean2D"
            g = {k: s[k].reshape(b[k].shape) for k in ("opacity", "mean3D", "scale", "rot")}
            acc = g if acc is None else {k: acc[k] + g[k] for k in acc}
    if backward:
        for k, want in acc.items():
            assert _bit_equal(b[k], want), f"{k}: not the view-ordered float32 sum of the single-view raw gradients"
    return b


def _bench_scene():
    return scene.make_cloud(100_000, kind="init", seed=0), scene.make_views(scene.cone_beam_scanner(512, 256), 50)


def _mid_scene():
    return scene.make_cloud(50_000, kind="init", seed=3), scene.make_views(scene.cone_beam_scanner(256, 256), 50)


# ---- 1 / 2. raw batched rasterizer -----------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 4])
def test_bench_scene_raw_bits(n):
    cloud, views = _bench_scene()
    _check(cloud, views[::12][:n], backward=(n == 4))


@pytest.mark.parametrize("n", [16, 20], ids=["direct", "radix"])
def test_50k_256_raw_bits(n):
    cloud, views = _mid_scene()
    _check(cloud, views[::3][:n] if n == 16 else views[:n], backward=(n == 20), seed=n)


def test_parallel_beam_raw_bits():
    sc = scene.parallel_beam_scanner(96, 64)
    _check(scene.make_cloud(2000, kind="trained", seed=5), [scene.make_view(sc, a) for a in (0.1, 1.3, 2.9, 4.4)])


def test_ragged_detector_raw_bits():
    sc = scene.cone_beam_scanner(200, 64)
    sc["nDetector"] = [200, 136]
    sc["sDetector"] = [4.0 * 200 / 512 * 2, 4.0 * 136 / 512 * 2]
    _check(scene.make_cloud(3000, kind="trained", seed=7), [scene.make_view(sc, a) for a in (0.2, 0.9, 2.5)], seed=1)


def test_culled_in_some_views_only_raw_bits():
    cloud = scene.make_cloud(3000, kind="trained", seed=11)
    cloud.means[:64] = np.float32([6.0, 0.0, 0.0]) + 0.05 * cloud.means[:64]
    sc = scene.cone_beam_scanner(128, 64)
    b = _check(cloud, [scene.make_view(sc, a) for a in (0.0, math.pi, 0.5 * math.pi)], seed=2)
    r = b["radii"][:, :64]
    assert (r[0] == 0).all() and (r[1] > 0).any(), "the case does not cull in some views only"


def test_empty_cloud_raw():
    sc = scene.cone_beam_scanner(64, 32)
    views = [scene.make_view(sc, a) for a in (0.0, 1.0)]
    t, act = _raw_inputs(scene.make_cloud(1, kind="trained", seed=0), views)
    for k in ("means", "dens", "scales", "rots"):
        t[k] = t[k][:0]
    b = _batched(t, act, views, _dL(views))
    assert b["R"] == 0 and b["images"].abs().sum().item() == 0 and b["radii"].shape == (2, 0)
    assert b["mean2D"].shape == (2, 0, 3) and b["opacity"].shape == (0, 1)


def test_repeated_overflow_raw():
    """A far too small capacity hint overflows and the call re-runs; twice in a row, each time the single-view bits."""
    cloud, views = _mid_scene()
    views = views[:6]
    t, act = _raw_inputs(cloud, views)
    key = _C.views_key(t["means"].device, cloud.P, len(views), views[0].image_width, views[0].image_height)
    results = []
    for _ in range(2):
        _C._Workspace.hints[key] = 1
        results.append(_batched(t, act, views))
    assert _bit_equal(results[0]["images"], results[1]["images"]) and results[0]["radii"].equal(results[1]["radii"])
    for v, view in enumerate(views):
        s = _single(t, act, view, v)
        assert _bit_equal(results[0]["images"][v], s["image"]) and results[0]["radii"][v].equal(s["radii"])


# ---- 3. batched loss and statistics ------------------------------------------------------------------------------------

@pytest.mark.parametrize("hw", [(128, 128), (136, 200)])
@pytest.mark.parametrize("with_grad", [True, False])
def test_image_loss_views_is_the_single_image_call(hw, with_grad):
    lib = load()
    H, W = hw
    N = 4
    g = torch.Generator("cuda").manual_seed(3)
    x = torch.rand((N, H, W), device="cuda", generator=g)
    y = torch.rand((N, H, W), device="cuda", generator=g)
    st = torch.cuda.current_stream().cuda_stream
    nb = lib.r2x_image_loss_views_scratch_bytes(N, H, W)
    scratch = torch.empty(nb, dtype=torch.uint8, device="cuda")
    out = torch.full((N, 3), float("nan"), device="cuda")
    grad = torch.full((N, H, W), float("nan"), device="cuda")
    assert lib.r2x_image_loss_views(st, N, H, W, x.data_ptr(), y.data_ptr(), 1.0, 0.25, out.data_ptr(),
                                    grad.data_ptr() if with_grad else None, scratch.data_ptr(), nb) == 0
    n1 = lib.r2x_image_loss_scratch_bytes(H, W)
    s1 = torch.empty(n1, dtype=torch.uint8, device="cuda")
    for v in range(N):
        o1 = torch.empty(3, device="cuda")
        g1 = torch.empty((H, W), device="cuda")
        assert lib.r2x_image_loss(st, H, W, x[v].data_ptr(), y[v].data_ptr(), 1.0, 0.25, o1.data_ptr(),
                                  g1.data_ptr() if with_grad else None, s1.data_ptr(), n1) == 0
        assert _bit_equal(out[v], o1), v
        if with_grad:
            assert _bit_equal(grad[v], g1), v
    if not with_grad:
        assert torch.isnan(grad).all()


@pytest.mark.parametrize("guarded", [False, True])
def test_densify_stats_views_is_n_sequential_calls(guarded):
    lib = load()
    N, P = 5, 70_001
    g = torch.Generator("cuda").manual_seed(4)
    radii = (torch.randint(-3, 12, (N, P), device="cuda", generator=g)).int()
    g2 = torch.randn((N, P, 3), device="cuda", generator=g) * 1e-3
    base = [torch.rand(P, device="cuda", generator=g) * 4, torch.rand(P, device="cuda", generator=g) * 1e-2,
            torch.randint(0, 9, (P,), device="cuda", generator=g).float()]
    status = torch.tensor([123, 1 if guarded else 0], dtype=torch.int32, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    got = [b.clone() for b in base]
    assert lib.r2x_densify_stats_views(st, N, P, radii.data_ptr(), g2.data_ptr(), *(x.data_ptr() for x in got),
                                       status.data_ptr(), None) == 0
    want = [b.clone() for b in base]
    for v in range(N):
        assert lib.r2x_densify_stats(st, P, radii[v].data_ptr(), g2[v].data_ptr(), *(x.data_ptr() for x in want),
                                     status.data_ptr(), None) == 0
    for a, b, b0 in zip(got, want, base):
        assert _bit_equal(a, b)
        if guarded:
            assert _bit_equal(a, b0)
    if not guarded:
        assert not _bit_equal(got[1], base[1])


# ---- 4 / 5 / 6. the batched training iteration ------------------------------------------------------------------------

B = 4


def _inputs(n_cams=8):
    from test_train_gpu import _train_inputs
    cams, gts, centres = _train_inputs(n_cams=n_cams)
    for k, c in enumerate(cams):
        c.uid = k
    return cams, gts, centres


def _batch(cams, gts, i):
    idx = [(B * i + j) % len(cams) for j in range(B)]
    return [cams[j] for j in idx], torch.stack([gts[j] for j in idx])


def _autograd_batch_iteration(gm, cams, gts, centre, lam_d, lam_tv, use_tv, tv_n, tv_s):
    """The trainer's autograd batched iteration (trainer.render_batch, the fused losses, FusedAdam)."""
    from r2_gaussian_b200 import losses, trainer
    from r2_gaussian_b200.render_query import query
    pipe = types.SimpleNamespace(compute_cov3D_python=False, debug=False)
    pkg = trainer.render_batch(cams, gm)
    per_view = [losses.image_loss(pkg["render"][v], gts[v], lambda_dssim=lam_d)["total"] for v in range(len(cams))]
    total, tv = sum(per_view), None
    if use_tv:
        tv = losses.tv_3d_loss(query(gm, centre, tv_n, tv_s, pipe)["vol"], "mean")
        total = total + (len(cams) * lam_tv) * tv
    total.backward()
    with torch.no_grad():
        for v in range(len(cams)):
            seen = pkg["radii"][v] > 0
            gm.update_max_radii(pkg["radii"][v], seen)
            gm.add_densification_stats(trainer._ViewGrad(pkg["viewspace_points"].grad[v]), seen)
    gm.optimizer.step()
    gm.optimizer.zero_grad(set_to_none=True)
    return pkg, torch.stack([x.detach() for x in per_view]), tv


def _assert_models_equal(a, b, steps):
    for name in ("_xyz", "_density", "_scaling", "_rotation"):
        ga, gb = getattr(a, name), getattr(b, name)
        assert _bit_equal(ga, gb), name
        sa, sb = a.optimizer.state[ga], b.optimizer.state[gb]
        assert _bit_equal(sa["exp_avg"], sb["exp_avg"]) and _bit_equal(sa["exp_avg_sq"], sb["exp_avg_sq"]), name
        assert float(sa["step"]) == float(sb["step"]) == steps
    for name in ("max_radii2D", "xyz_gradient_accum", "denom"):
        assert _bit_equal(getattr(a, name), getattr(b, name)), name


@pytest.mark.parametrize("use_tv", [True, False])
def test_native_batch_step_is_the_autograd_batch_iteration(use_tv):
    from r2_gaussian_b200.train_step import NativeTrainStep
    from test_train_gpu import _make_model
    cams, gts, centres = _inputs()
    lam_d, lam_tv, n_it = 0.25, 0.05, 7
    tv_n, tv_s = [32, 32, 32], [0.5, 0.5, 0.5]
    a, _, _ = _make_model(n=5000, seed=11)
    b, _, _ = _make_model(n=5000, seed=11)
    step = NativeTrainStep(b, lam_d, lam_tv if use_tv else 0.0, tv_n, tv_s)
    for i in range(1, n_it + 1):
        bc, bg = _batch(cams, gts, i)
        centre = centres[i % len(centres)]
        a.update_learning_rate(i); b.update_learning_rate(i)
        pkg, per_view, tv = _autograd_batch_iteration(a, bc, bg, centre, lam_d, lam_tv, use_tv, tv_n, tv_s)
        res = step(bc, bg, centre)
        if i == n_it:
            assert _bit_equal(res["render"], pkg["render"].detach()) and res["radii"].equal(pkg["radii"])
            assert _bit_equal(res["loss"][:, 2], per_view)
            want = float(per_view.double().mean()) + (lam_tv * float(tv.detach()) if use_tv else 0.0)
            assert abs(step.total_loss() - want) <= 1e-6 * abs(want)
    step.flush()
    assert step.repeats == 0
    _assert_models_equal(a, b, n_it)
    assert float(b.denom.max()) > n_it          # several views of one iteration count separately


def test_batch_objective_is_the_loop_of_single_view_iterations():
    """Raw gradients of one batched iteration against render() + image_loss per view and B lambda_tv TV, summed by
    autograd in its own order (1e-6 relative: the summation order differs)."""
    from r2_gaussian_b200 import losses
    from r2_gaussian_b200.render_query import query, render
    from test_train_gpu import _make_model
    cams, gts, centres = _inputs()
    bc, bg = _batch(cams, gts, 0)
    lam_d, lam_tv, tv_n, tv_s = 0.25, 0.05, [32, 32, 32], [0.5, 0.5, 0.5]
    pipe = types.SimpleNamespace(compute_cov3D_python=False, debug=False)
    a, _, _ = _make_model(n=5000, seed=12)
    b, _, _ = _make_model(n=5000, seed=12)
    from r2_gaussian_b200 import trainer
    pkg = trainer.render_batch(bc, a)
    total = sum(losses.image_loss(pkg["render"][v], bg[v], lam_d)["total"] for v in range(B))
    total = total + (B * lam_tv) * losses.tv_3d_loss(query(a, centres[0], tv_n, tv_s, pipe)["vol"], "mean")
    total.backward()
    loop = 0
    for v in range(B):
        loop = loop + losses.image_loss(render(bc[v], b, pipe)["render"], bg[v], lam_d)["total"]
    loop = loop + B * lam_tv * losses.tv_3d_loss(query(b, centres[0], tv_n, tv_s, pipe)["vol"], "mean")
    loop.backward()
    assert abs(float(total) - float(loop)) <= 1e-6 * abs(float(loop))
    for name in ("_xyz", "_density", "_scaling", "_rotation"):
        got, want = getattr(a, name).grad, getattr(b, name).grad
        scale = want.abs().max().item()
        assert scale > 0 and (got - want).abs().max().item() <= 1e-6 * scale, name


def test_overflowed_batch_changes_nothing_and_repeats_once():
    from r2_gaussian_b200.train_step import NativeTrainStep
    from test_train_gpu import _make_model
    cams, gts, centres = _inputs()
    a, _, _ = _make_model(n=5000, seed=13)
    b, _, _ = _make_model(n=5000, seed=13)
    sa = NativeTrainStep(a, 0.25, 0.05, [32, 32, 32], [0.5, 0.5, 0.5])
    sb = NativeTrainStep(b, 0.25, 0.05, [32, 32, 32], [0.5, 0.5, 0.5])
    for i in (1, 2):
        bc, bg = _batch(cams, gts, i)
        a.update_learning_rate(i); sa(bc, bg, centres[i])
    sa.flush()
    bc, bg = _batch(cams, gts, 1)
    b.update_learning_rate(1); sb(bc, bg, centres[1]); sb.flush()
    lib = sb.lib
    sb.cap_r = 4096
    sb.binning_r = torch.empty(lib.r2x_binning_bytes(4096), dtype=torch.uint8, device="cuda")
    sb.scratch_r = torch.empty(lib.r2x_raster_bwd_scratch_bytes(4096), dtype=torch.uint8, device="cuda")
    saved = dict(_C._Workspace.hints)
    _C._Workspace.hints[sb.key_r] = 1
    sb._provision = lambda: None
    b.update_learning_rate(2)
    before = [getattr(b, k).clone() for k in ("_xyz", "_density", "max_radii2D", "xyz_gradient_accum", "denom")]
    bc, bg = _batch(cams, gts, 2)
    sb(bc, bg, centres[2])
    torch.cuda.synchronize()
    for x, k in zip(before, ("_xyz", "_density", "max_radii2D", "xyz_gradient_accum", "denom")):
        assert _bit_equal(x, getattr(b, k)), k
    del sb._provision
    sb.cap_r = 0
    sb.flush()
    assert sb.repeats == 1
    _C._Workspace.hints.update({k: v for k, v in saved.items() if k == sb.key_r})
    _assert_models_equal(a, b, 2)


# ---- 7. B = 1: the parent's launches -----------------------------------------------------------------------------------

def test_trainer_at_batch_size_one_issues_the_parent_kernels(tmp_path):
    from test_pose_train_gpu import PARENT_KERNELS, PARENT_SEQUENCE
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path)], capture_output=True, text=True,
                       env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-4000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    assert [PARENT_KERNELS[k] for k in PARENT_SEQUENCE] == names


def _trainer_kernel_sequence_b1(workdir):
    """test_pose_train_gpu's 6-iteration trainer run, with batch_size=1 passed explicitly."""
    import test_pose_train_gpu as tp
    from r2_gaussian_b200 import trainer
    real = trainer.training
    trainer.training = lambda *a, **k: real(*a, batch_size=1, **k)
    try:
        return tp._trainer_kernel_sequence(workdir)
    finally:
        trainer.training = real


# ---- 8. end to end -----------------------------------------------------------------------------------------------------

E2E_ITERATIONS = 500       # x 4 views


def test_batch_training_beats_the_fdk_initialisation(tmp_path):
    from r2_gaussian_b200 import generate_data, initialize_pcd, trainer
    from r2_gaussian_b200.dataset import Scene
    from r2_gaussian_b200.gaussian_model import GaussianModel
    from test_projector_gpu import _write_inputs
    yml, vol_path, *_ = _write_inputs(tmp_path, noise=False)
    path = generate_data.main(["--vol", str(vol_path), "--scanner", str(yml), "--n_train", "24", "--n_test", "6",
                               "--output", str(tmp_path / "data")])
    init = initialize_pcd.main(["--data", path, "--recon_method", "fdk", "--n_points", "2000",
                                "--output", str(tmp_path / "init.npy")])
    model = trainer.ModelParams(source_path=path, model_path=str(tmp_path / "out"), ply_path=init)
    opt = trainer.OptimizationParams(iterations=E2E_ITERATIONS)
    pipe = trainer.PipelineParams()
    sc = Scene(path, "", shuffle=False)
    gm = GaussianModel(trainer.derived_settings(sc.scanner_cfg, model, opt)["scale_bound"])
    pts = np.load(init)
    gm.create_from_pcd(pts[:, :3], pts[:, 3:4], 1.0)
    p0 = trainer.evaluate(sc, gm, pipe, with_ssim=False)["psnr_3d"]
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    hist = trainer.training(model, opt, pipe, {E2E_ITERATIONS}, log=lambda *a: None, batch_size=4)
    p1 = hist["eval"][E2E_ITERATIONS]["psnr_3d"]
    print(f"psnr_3d {p0:.3f} (FDK initialisation) -> {p1:.3f} after {E2E_ITERATIONS} x 4 views")
    assert p1 >= p0 + 3.0, (p0, p1)


if __name__ == "__main__":
    print(json.dumps(_trainer_kernel_sequence_b1(sys.argv[1])))
