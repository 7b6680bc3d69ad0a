"""Pose refinement in training: the device pose kernels and both training paths that use them.

1. r2x_pose_apply against `PoseCorrection(dtype=float64).matrices()` rounded to float32 (1 ulp), bit for bit at zero;
2. r2x_pose_grad against autograd through the same float64 statement (2 ulps), other rows and the anchor exactly 0;
3. `NativeTrainStep(pose=...)` is the autograd iteration through `device_camera` / render / FusedAdam, bit for bit;
4. an iteration repeated after a capacity overflow moves the poses once;
5. `trainer --pose_refine` recovers seeded angle errors of a generate_data scene and reconstructs it better;
6. without `--pose_refine` a trainer run launches the kernels it launched before pose refinement existed.
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

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _camera(angle, det=128, mode=1):
    from r2_gaussian_b200 import scene
    sc = scene.cone_beam_scanner(det, 64) if mode == 1 else scene.parallel_beam_scanner(det, 64)
    v = scene.make_view(sc, angle)
    wvt = torch.tensor(v.viewmatrix, device=DEV)
    proj = torch.tensor(scene.projection_matrix(v.FoVx, v.FoVy, v.mode).T.copy(), device=DEV)
    full = wvt.unsqueeze(0).bmm(proj.unsqueeze(0)).squeeze(0).contiguous()
    return types.SimpleNamespace(world_view_transform=wvt, projection_matrix=proj, full_proj_transform=full,
                                 camera_center=torch.tensor(v.campos, device=DEV), image_height=v.image_height,
                                 image_width=v.image_width, FoVx=v.FoVx, FoVy=v.FoVy, mode=v.mode)


def _twists():
    """(omega, nu) float32: zero, theta^2 just below / above the series switch at 1e-2, small, theta around 0.3."""
    rng = np.random.RandomState(5)
    out = [(np.zeros(3, np.float32), np.zeros(3, np.float32))]
    for theta in (0.1 * (1 - 1e-5), 0.1 * (1 + 1e-5), 1e-4, 0.05, 0.29, 0.3, 0.31):
        axis = rng.randn(3)
        axis /= np.linalg.norm(axis)
        out.append(((axis * theta).astype(np.float32), (rng.randn(3) * 0.1).astype(np.float32)))
    th2 = [float(np.sum(w.astype(np.float64) ** 2)) for w, _ in out]
    assert th2[1] < 1e-2 < th2[2]
    return out


def _corrections(n, i, w, v):
    from r2_gaussian_b200.pose import PoseCorrection
    c32 = PoseCorrection(n, device=DEV)
    c64 = PoseCorrection(n, device=DEV, dtype=torch.float64)
    with torch.no_grad():
        c32.omega[i] = torch.from_numpy(w)
        c32.nu[i] = torch.from_numpy(v)
        c64.omega.copy_(c32.omega.double())
        c64.nu.copy_(c32.nu.double())
    return c32, c64


def _ulps(got, ref64):
    """|got - ref| in units of the float32 spacing at |ref| (ref rounded to float32)."""
    ref32 = ref64.float().cpu().numpy()
    sp = np.spacing(np.abs(ref32)).astype(np.float64)
    return np.abs(got.double().cpu().numpy() - ref64.cpu().numpy()) / sp


# ---- 1. apply kernel -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", [1, 0], ids=["cone", "parallel"])
def test_apply_kernel_matches_float64_statement(mode):
    cam = _camera(0.7, mode=mode)
    for k, (w, v) in enumerate(_twists()):
        c32, c64 = _corrections(3, 1, w, v)
        got = c32.device_camera(cam, 1)
        ref_v, ref_f = c64.matrices(cam, 1)
        torch.cuda.synchronize()
        for name, g, r in (("view", got.world_view_transform, ref_v), ("full", got.full_proj_transform, ref_f)):
            assert g.dtype == torch.float32 and g.shape == (4, 4)
            # 1 ulp of the float64 value: both round the same float64 expression once
            assert torch.equal(g, r.float()) or _ulps(g, r.detach()).max() <= 1.0, (k, name, g, r)
        if k == 0:
            for name in ("world_view_transform", "full_proj_transform"):
                assert torch.equal(getattr(got, name).view(torch.int32), getattr(cam, name).view(torch.int32)), name
            assert got.camera_center is cam.camera_center
    # rows other than i leave their camera alone too (zero twist)
    other = c32.device_camera(cam, 0)
    assert torch.equal(other.world_view_transform.view(torch.int32), cam.world_view_transform.view(torch.int32))


# ---- 2. gradient kernel ----------------------------------------------------------------------------------------------

def _captured_matrix_gradients(cam):
    """dL/dview, dL/dfull of a real rasterizer backward (a trained cloud, a ramp-plus-noise dL/dimage)."""
    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.pose import PoseCorrection
    from r2_gaussian_b200.render_query import render
    from test_pose_gpu import _dl, _Model, _Pipe
    cloud = scene.make_cloud(20_000, kind="trained", seed=5)
    c = PoseCorrection(1, device=DEV)(cam, 0)
    c.world_view_transform.retain_grad()
    c.full_proj_transform.retain_grad()
    img = render(c, _Model(cloud, True), _Pipe())["render"]
    (img * _dl(cam.image_height, cam.image_width)).sum().backward()
    gv, gp = c.world_view_transform.grad.clone(), c.full_proj_transform.grad.clone()
    assert torch.count_nonzero(gv) > 0 and torch.count_nonzero(gp) > 0
    return gv, gp


def test_grad_kernel_matches_autograd_in_float64():
    cam = _camera(1.3, det=256)
    gv, gp = _captured_matrix_gradients(cam)
    n, i = 5, 3
    for k, (w, v) in enumerate(_twists()):
        c32, c64 = _corrections(n, i, w, v)
        out = c32.device_camera(cam, i, anchor=0)
        g32 = torch.autograd.grad((out.world_view_transform, out.full_proj_transform), (c32.omega, c32.nu), (gv, gp))
        rv, rf = c64.matrices(cam, i)
        g64 = torch.autograd.grad((rv, rf), (c64.omega, c64.nu), (gv.double(), gp.double()))
        for name, g, r in zip(("omega", "nu"), g32, g64):
            assert g.dtype == torch.float32 and g.shape == (n, 3)
            rows = [j for j in range(n) if j != i]
            assert torch.count_nonzero(g[rows]) == 0, (k, name)
            r_i, g_i = r[i].detach(), g[i]
            bound = 2 * np.spacing(np.abs(r_i.float().cpu().numpy())).astype(np.float64) + 1e-7 * float(r_i.abs().max())
            assert (np.abs(g_i.double().cpu().numpy() - r_i.cpu().numpy()) <= bound).all(), (k, name, g_i, r_i)
            assert torch.count_nonzero(g_i) > 0, (k, name)
        # the anchor's row is always 0, also when it is the rendered view; anchor -1: no anchor
        out = c32.device_camera(cam, i, anchor=i)
        g = torch.autograd.grad((out.world_view_transform, out.full_proj_transform), (c32.omega, c32.nu), (gv, gp))
        assert torch.count_nonzero(g[0]) == 0 and torch.count_nonzero(g[1]) == 0
        out = c32.device_camera(cam, i, anchor=-1)
        g = torch.autograd.grad((out.world_view_transform, out.full_proj_transform), (c32.omega, c32.nu), (gv, gp))
        assert torch.equal(g[0], g32[0]) and torch.equal(g[1], g32[1])


# ---- 3. native step == autograd iteration ------------------------------------------------------------------------------

def _pose_pair(n, seed=3):
    from r2_gaussian_b200.optim import FusedAdam
    from r2_gaussian_b200.pose import PoseCorrection
    out = []
    rng = np.random.RandomState(seed)
    w0, v0 = rng.randn(n, 3) * 0.01, rng.randn(n, 3) * 0.02
    w0[0] = v0[0] = 0.0
    for _ in range(2):
        corr = PoseCorrection(n, device=DEV)
        with torch.no_grad():
            corr.omega.copy_(torch.tensor(w0)); corr.nu.copy_(torch.tensor(v0))
        opt = FusedAdam([{"params": [corr.omega], "lr": 1e-3}, {"params": [corr.nu], "lr": 5e-3}], lr=0.0, eps=1e-15)
        out.append((corr, opt))
    return out


def _with_projection(cams):
    from r2_gaussian_b200 import scene
    for c in cams:
        c.projection_matrix = torch.tensor(scene.projection_matrix(c.FoVx, c.FoVy, c.mode).T.copy(), device=DEV)
    return cams


def _assert_pose_equal(pa, oa, pb, ob, steps):
    for name in ("omega", "nu"):
        a, b = getattr(pa, name), getattr(pb, name)
        assert torch.equal(a, b), name
        sa, sb = oa.state[a], ob.state[b]
        assert torch.equal(sa["exp_avg"], sb["exp_avg"]) and torch.equal(sa["exp_avg_sq"], sb["exp_avg_sq"]), name
        assert float(sa["step"]) == float(sb["step"]) == steps, name


@pytest.mark.parametrize("use_tv", [True, False])
def test_native_pose_step_is_the_autograd_iteration(use_tv):
    from r2_gaussian_b200 import losses
    from r2_gaussian_b200.render_query import query, render
    from r2_gaussian_b200.train_step import NativeTrainStep
    from test_train_gpu import _make_model, _train_inputs
    pipe = types.SimpleNamespace(compute_cov3D_python=False, debug=False)
    cams, gts, centres = _train_inputs()
    cams = _with_projection(cams)
    lam_d, lam_tv, n_it = 0.25, 0.05, 7
    tv_n, tv_s = [32, 32, 32], [0.5, 0.5, 0.5]
    a, _, _ = _make_model(n=5000, seed=11)
    b, _, _ = _make_model(n=5000, seed=11)
    (pa, oa), (pb, ob) = _pose_pair(len(cams))
    w_start = pa.omega.detach().clone()
    step = NativeTrainStep(b, lam_d, lam_tv if use_tv else 0.0, tv_n, tv_s, pose=(pb, ob), pose_anchor=0)
    for i in range(1, n_it + 1):
        k = i % len(cams)
        a.update_learning_rate(i); b.update_learning_rate(i)
        pkg = render(pa.device_camera(cams[k], k, 0), a, pipe)
        total = losses.image_loss(pkg["render"], gts[k], lam_d)["total"]
        if use_tv:
            total = total + lam_tv * losses.tv_3d_loss(query(a, centres[k], tv_n, tv_s, pipe)["vol"], "mean")
        total.backward()
        with torch.no_grad():
            a.update_max_radii(pkg["radii"], pkg["visibility_filter"])
            a.add_densification_stats(pkg["viewspace_points"], pkg["visibility_filter"])
        a.optimizer.step(); a.optimizer.zero_grad(set_to_none=True)
        oa.step(); oa.zero_grad(set_to_none=True)
        res = step(cams[k], gts[k], centres[k], view=k)
        if i == n_it:
            assert abs(step.total_loss() - float(total)) <= 1e-6 * abs(float(total))
            assert torch.equal(res["radii"], pkg["radii"])
    step.flush()
    assert step.repeats == 0
    for name in ("_xyz", "_density", "_scaling", "_rotation"):
        ga, gb = getattr(a, name), getattr(b, name)
        assert torch.equal(ga, gb), name
        sa, sb = a.optimizer.state[ga], b.optimizer.state[gb]
        assert torch.equal(sa["exp_avg"], sb["exp_avg"]) and torch.equal(sa["exp_avg_sq"], sb["exp_avg_sq"]), name
        assert float(sa["step"]) == float(sb["step"]) == n_it
    assert torch.equal(a.max_radii2D, b.max_radii2D) and torch.equal(a.denom, b.denom)
    _assert_pose_equal(pa, oa, pb, ob, n_it)
    moved = (pb.omega != w_start).any(dim=1)
    assert bool(moved[1:].all()) and not bool(moved[0]) and torch.count_nonzero(pb.omega[0]) == 0


# ---- 4. overflow repeat ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("starve", ["both", "tv"])
def test_native_pose_step_repeats_an_overflowed_iteration_once(starve):
    from r2_gaussian_b200 import _C
    from r2_gaussian_b200.train_step import NativeTrainStep
    from test_train_gpu import _make_model, _train_inputs
    cams, gts, centres = _train_inputs(n_cams=2)
    cams = _with_projection(cams)
    a, _, _ = _make_model(n=5000, seed=13)
    b, _, _ = _make_model(n=5000, seed=13)
    (pa, oa), (pb, ob) = _pose_pair(2, seed=4)
    sa = NativeTrainStep(a, 0.25, 0.05, [32, 32, 32], [0.5, 0.5, 0.5], pose=(pa, oa), pose_anchor=-1)
    sb = NativeTrainStep(b, 0.25, 0.05, [32, 32, 32], [0.5, 0.5, 0.5], pose=(pb, ob), pose_anchor=-1)
    for i in (1, 2):
        a.update_learning_rate(i); sa(cams[i % 2], gts[i % 2], centres[i % 2], view=i % 2)
    sa.flush()
    b.update_learning_rate(1); sb(cams[1], gts[1], centres[1], view=1); sb.flush()
    lib = sb.lib
    if starve == "both":
        sb.cap_r = 4096
        sb.binning_r = torch.empty(lib.r2x_binning_bytes(4096), dtype=torch.uint8, device="cuda")
        sb.scratch_r = torch.empty(lib.r2x_raster_bwd_scratch_bytes(4096), dtype=torch.uint8, device="cuda")
    sb.cap_v = 4096
    sb.binning_v = torch.empty(lib.r2x_binning_bytes(4096), dtype=torch.uint8, device="cuda")
    sb.scratch_v = torch.empty(lib.r2x_voxel_bwd_scratch_bytes(4096), dtype=torch.uint8, device="cuda")
    saved = dict(_C._Workspace.hints)
    if starve == "both":
        _C._Workspace.hints[sb.key_r] = 1
    _C._Workspace.hints[sb.key_v] = 1
    sb._provision = lambda: None
    b.update_learning_rate(2)
    before = (b._xyz.clone(), pb.omega.detach().clone(), pb.nu.detach().clone())
    sb(cams[0], gts[0], centres[0], view=0)
    torch.cuda.synchronize()
    assert torch.equal(before[0], b._xyz)
    assert torch.equal(before[1], pb.omega) and torch.equal(before[2], pb.nu)    # guarded by the TV forward too
    del sb._provision
    sb.cap_r = sb.cap_v = 0
    sb.flush()
    assert sb.repeats == 1
    _C._Workspace.hints.update({k: v for k, v in saved.items() if k in (sb.key_r, sb.key_v)})
    for name in ("_xyz", "_density", "_scaling", "_rotation"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    _assert_pose_equal(pa, oa, pb, ob, 2)
    assert not torch.equal(before[1], pb.omega)


# ---- 5. recovery through the trainer -----------------------------------------------------------------------------------

RECOVERY_ITERATIONS = 2000


@pytest.fixture(scope="module")
def perturbed_scene(tmp_path_factory):
    """The generate_data scene of test_recon_gpu (48^3, 24 train / 6 test views of 96^2) whose meta_data.json gives train
    views 1-23 seeded angle errors of up to +-1 degree (view 0 exact), initialised by FDK from the perturbed angles."""
    from r2_gaussian_b200 import generate_data, initialize_pcd
    from test_projector_gpu import _write_inputs
    tmp = tmp_path_factory.mktemp("pose_scene")
    yml, vol_path, *_ = _write_inputs(tmp, noise=False)
    path = generate_data.main(["--vol", str(vol_path), "--scanner", str(yml), "--n_train", "24", "--n_test", "6",
                               "--output", str(tmp / "data")])
    meta_path = os.path.join(path, "meta_data.json")
    with open(meta_path) as f:
        meta = json.load(f)
    true = np.array([fr["angle"] for fr in meta["proj_train"]])
    err = np.radians(np.concatenate([[0.0], np.random.RandomState(2026).uniform(-1.0, 1.0, len(true) - 1)]))
    for fr, e in zip(meta["proj_train"], err):
        fr["angle"] = float(fr["angle"] + e)
    with open(meta_path, "w") as f:
        json.dump(meta, f, indent=1)
    init = initialize_pcd.main(["--data", path, "--recon_method", "fdk", "--n_points", "2000",
                                 "--output", str(tmp / "init.npy")])
    return path, true, init


def _train(path, init, out, refine):
    from r2_gaussian_b200 import trainer
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    model = trainer.ModelParams(source_path=path, model_path=str(out), ply_path=init)
    opt = trainer.OptimizationParams(iterations=RECOVERY_ITERATIONS)
    it = RECOVERY_ITERATIONS
    return trainer.training(model, opt, trainer.PipelineParams(), {it}, {it}, log=lambda *a: None,
                            pose_params=trainer.PoseParams(pose_refine=refine))


def _pose_errors(wvts, angles, dso):
    """Per view: rotation angle of T' T_true^-1 (rad) and distance between the camera centres (scene units)."""
    from r2_gaussian_b200.scene import angle2pose
    rot, centre = [], []
    for wvt, ang in zip(wvts, angles):
        T = np.asarray(wvt, np.float64).T
        Tt = np.linalg.inv(angle2pose(dso, float(ang)))
        dR = T[:3, :3] @ Tt[:3, :3].T
        rot.append(math.acos(min(1.0, max(-1.0, (np.trace(dR) - 1) / 2))))
        centre.append(np.linalg.norm(-T[:3, :3].T @ T[:3, 3] + Tt[:3, :3].T @ Tt[:3, 3]))
    return np.array(rot), np.array(centre)


@pytest.mark.xfail(strict=True, raises=AssertionError, reason="finding (H100, default pose learning rates): the train-view PSNR rises but the "
                   "mean rotation error stays at 0.53 deg (from 0.54), the camera-centre error doubles (0.047 -> 0.094) "
                   "and psnr_3d falls (39.6 -> 27.3); lower rates down to 1/30 only limit the damage.  The bars stay as "
                   "fixed; strict, so a change that makes them hold is noticed")
def test_pose_refine_recovers_angle_errors_through_the_trainer(perturbed_scene, tmp_path):
    path, true, init = perturbed_scene
    plain = _train(path, init, tmp_path / "plain", False)
    refined = _train(path, init, tmp_path / "pose", True)
    assert "pose" not in plain
    assert not os.path.exists(tmp_path / "plain" / "point_cloud" / f"iteration_{RECOVERY_ITERATIONS}" / "train_poses.npz")
    sc = refined["scene"]
    dso = sc.scanner_cfg["DSO"]
    nominal = [c.world_view_transform.cpu().numpy() for c in sc.getTrainCameras()]
    saved = np.load(tmp_path / "pose" / "point_cloud" / f"iteration_{RECOVERY_ITERATIONS}" / "train_poses.npz")
    assert saved["world_view_transform"].shape == (24, 4, 4) and saved["omega"].shape == (24, 3)
    assert np.array_equal(saved["angle"], np.array([c.angle for c in sc.getTrainCameras()]))
    assert np.count_nonzero(saved["omega"][0]) == 0 and np.count_nonzero(saved["nu"][0]) == 0
    r0, c0 = _pose_errors(nominal, true, dso)
    r1, c1 = _pose_errors(saved["world_view_transform"], true, dso)
    p_plain = plain["eval"][RECOVERY_ITERATIONS]["psnr_3d"]
    p_pose = refined["eval"][RECOVERY_ITERATIONS]["psnr_3d"]
    print(f"rotation error {np.degrees(r0[1:].mean()):.4f} -> {np.degrees(r1[1:].mean()):.4f} deg, camera centre "
          f"{c0[1:].mean():.5f} -> {c1[1:].mean():.5f}, psnr_3d {p_plain:.3f} (nominal poses) {p_pose:.3f} (refined), "
          f"2d train {plain['eval'][RECOVERY_ITERATIONS]['psnr_2d_train']:.3f} -> "
          f"{refined['eval'][RECOVERY_ITERATIONS]['psnr_2d_train']:.3f}")
    assert r1[1:].mean() <= 0.5 * r0[1:].mean(), (r0[1:].mean(), r1[1:].mean())
    assert c1[1:].mean() <= 0.5 * c0[1:].mean(), (c0[1:].mean(), c1[1:].mean())
    assert p_pose > p_plain, (p_plain, p_pose)


# ---- 6. pose off: the same launches ------------------------------------------------------------------------------------

# Recorded from the trainer as it was before pose refinement (same script, `_trainer_kernel_sequence`): the distinct
# kernel names, and the launch order as indices into them.
PARENT_KERNELS = [
    "void gemmSN_NN_kernel<float, 128, 2, 4, 8, 4, 4, false, cublasGemvTensorStridedBatched<float const>, cublasGemvTensorStridedBatched<float const>, cublasGemvTensorStridedBatched<float> >(cublasGemmSmallNParams<cublasGemvTensorStridedBatched<float const>, cublasGemvTensorStridedBatched<float const>, cublasGemvTensorStridedBatched<float>, float>)",
    "void at::native::vectorized_elementwise_kernel<4, at::native::FillFunctor<float>, std::array<char*, 1ul> >(int, at::native::FillFunctor<float>, std::array<char*, 1ul>)",
    "void at::native::elementwise_kernel<128, 2, at::native::gpu_kernel_impl_nocast<at::native::FillFunctor<float> >(at::TensorIteratorBase&, at::native::FillFunctor<float> const&)::{lambda(int)#1}>(int, at::native::gpu_kernel_impl_nocast<at::native::FillFunctor<float> >(at::TensorIteratorBase&, at::native::FillFunctor<float> const&)::{lambda(int)#1})",
    "void at::native::elementwise_kernel<128, 2, at::native::gpu_kernel_impl_nocast<at::native::direct_copy_kernel_cuda(at::TensorIteratorBase&)::{lambda()#3}::operator()() const::{lambda()#7}::operator()() const::{lambda(float)#1}>(at::TensorIteratorBase&, at::native::direct_copy_kernel_cuda(at::TensorIteratorBase&)::{lambda()#3}::operator()() const::{lambda()#7}::operator()() const::{lambda(float)#1} const&)::{lambda(int)#1}>(int, at::native::gpu_kernel_impl_nocast<at::native::direct_copy_kernel_cuda(at::TensorIteratorBase&)::{lambda()#3}::operator()() const::{lambda()#7}::operator()() const::{lambda(float)#1}>(at::TensorIteratorBase&, at::native::direct_copy_kernel_cuda(at::TensorIteratorBase&)::{lambda()#3}::operator()() const::{lambda()#7}::operator()() const::{lambda(float)#1} const&)::{lambda(int)#1})",
    "xxtrf4_set_info_ker(int, int*)",
    "void getrf_pivot<getrf_params_<float, 32, 1, 32, 32, 1> >(int, int, int, void*, int, long*, int, getrf_params_<float, 32, 1, 32, 32, 1>::data_type*, unsigned int*, unsigned int*, getrf_params_<float, 32, 1, 32, 32, 1>::data_type*, unsigned int, unsigned int, unsigned int, int*)",
    "void ipiv_lower_small<float, 32>(int, void*, int, long*, int, int)",
    "void create_pivot_v2<32>(int, int*, long*, int)",
    "void ipiv_lower_diag<float, 32>(int, void*, int, int*, int)",
    "void ipiv_64_to_32_ker<128>(long, long const*, int*)",
    "void (anonymous namespace)::elementwise_kernel_with_index<int, at::native::arange_cuda_out(c10::Scalar const&, c10::Scalar const&, c10::Scalar const&, at::Tensor&)::{lambda()#1}::operator()() const::{lambda()#4}::operator()() const::{lambda(long)#1}>(int, at::native::arange_cuda_out(c10::Scalar const&, c10::Scalar const&, c10::Scalar const&, at::Tensor&)::{lambda()#1}::operator()() const::{lambda()#4}::operator()() const::{lambda(long)#1}, function_traits<at::native::arange_cuda_out(c10::Scalar const&, c10::Scalar const&, c10::Scalar const&, at::Tensor&)::{lambda()#1}::operator()() const::{lambda()#4}::operator()() const::{lambda(long)#1}>::result_type*)",
    "void laswp_kernel<float, false>(int, float* const*, int, int, int, int const*, int, int, int)",
    "void trsm_batch_left_lower_kernel<float>(cublasTrsmBatchParams<float>, float const* const*, float* const*, float const*, float)",
    "void trsm_batch_left_upper_kernel<float>(cublasTrsmBatchParams<float>, float const* const*, float* const*, float const*, float)",
    "void at::native::unrolled_elementwise_kernel<at::native::direct_copy_kernel_cuda(at::TensorIteratorBase&)::{lambda()#3}::operator()() const::{lambda()#11}::operator()() const::{lambda(bool)#1}, std::array<char*, 2ul>, 4, TrivialOffsetCalculator<1, unsigned int>, TrivialOffsetCalculator<1, unsigned int>, at::native::memory::LoadWithCast<1>, at::native::memory::StoreWithCast<1> >(int, at::native::direct_copy_kernel_cuda(at::TensorIteratorBase&)::{lambda()#3}::operator()() const::{lambda()#11}::operator()() const::{lambda(bool)#1}, std::array<char*, 2ul>, TrivialOffsetCalculator<1, unsigned int>, TrivialOffsetCalculator<1, unsigned int>, at::native::memory::LoadWithCast<1>, at::native::memory::StoreWithCast<1>)",
    "r2x::knn_init_kernel(unsigned int*)",
    "r2x::knn_bbox_kernel(int, float const*, unsigned int*)",
    "r2x::knn_count_kernel(int, float const*, unsigned int const*, int, unsigned int*)",
    "r2x::scan_kernel(int, unsigned int const*, unsigned int*, unsigned long long*, unsigned int*, int)",
    "r2x::knn_scatter_kernel(int, float const*, unsigned int const*, int, unsigned int*, unsigned int const*, float4*)",
    "r2x::knn_query_kernel(int, unsigned int const*, int, unsigned int const*, float4 const*, float*)",
    "void at::native::vectorized_elementwise_kernel<4, at::native::(anonymous namespace)::launch_clamp_scalar(at::TensorIteratorBase&, c10::Scalar, c10::Scalar, at::native::detail::ClampLimits)::{lambda()#1}::operator()() const::{lambda()#7}::operator()() const::{lambda(float)#1}, std::array<char*, 2ul> >(int, at::native::(anonymous namespace)::launch_clamp_scalar(at::TensorIteratorBase&, c10::Scalar, c10::Scalar, at::native::detail::ClampLimits)::{lambda()#1}::operator()() const::{lambda()#7}::operator()() const::{lambda(float)#1}, std::array<char*, 2ul>)",
    "void at::native::vectorized_elementwise_kernel<4, at::native::sqrt_kernel_cuda(at::TensorIteratorBase&)::{lambda()#2}::operator()() const::{lambda()#2}::operator()() const::{lambda(float)#1}, std::array<char*, 2ul> >(int, at::native::sqrt_kernel_cuda(at::TensorIteratorBase&)::{lambda()#2}::operator()() const::{lambda()#2}::operator()() const::{lambda(float)#1}, std::array<char*, 2ul>)",
    "void at::native::vectorized_elementwise_kernel<4, at::native::CUDAFunctorOnSelf_add<float>, std::array<char*, 2ul> >(int, at::native::CUDAFunctorOnSelf_add<float>, std::array<char*, 2ul>)",
    "void at::native::vectorized_elementwise_kernel<4, at::native::BUnaryFunctor<float, float, float, at::native::binary_internal::MulFunctor<float> >, std::array<char*, 2ul> >(int, at::native::BUnaryFunctor<float, float, float, at::native::binary_internal::MulFunctor<float> >, std::array<char*, 2ul>)",
    "void at::native::vectorized_elementwise_kernel<4, at::native::CUDAFunctorOnOther_add<float>, std::array<char*, 2ul> >(int, at::native::CUDAFunctorOnOther_add<float>, std::array<char*, 2ul>)",
    "void at::native::vectorized_elementwise_kernel<4, at::native::BinaryFunctor<float, float, float, at::native::binary_internal::DivFunctor<float> >, std::array<char*, 3ul> >(int, at::native::BinaryFunctor<float, float, float, at::native::binary_internal::DivFunctor<float> >, std::array<char*, 3ul>)",
    "void at::native::vectorized_elementwise_kernel<4, at::native::log_kernel_cuda(at::TensorIteratorBase&)::{lambda()#2}::operator()() const::{lambda()#2}::operator()() const::{lambda(float)#1}, std::array<char*, 2ul> >(int, at::native::log_kernel_cuda(at::TensorIteratorBase&)::{lambda()#2}::operator()() const::{lambda()#2}::operator()() const::{lambda(float)#1}, std::array<char*, 2ul>)",
    "void at::native::vectorized_elementwise_kernel<4, at::native::FillFunctor<int>, std::array<char*, 1ul> >(int, at::native::FillFunctor<int>, std::array<char*, 1ul>)",
    "r2x::raster_preprocess_kernel(int, float const*, float const*, float, float const*, float const*, float const*, float const*, float const*, int, int, float, float, float, float, int, int, int, int*, r2x::RasterGeom, r2x::DirectBin, int, r2x::Activation)",
    "r2x::direct_scan_kernel(r2x::DirectBin, uint2*, r2x::TilePlan, unsigned int*, long long, unsigned int*)",
    "r2x::direct_fill_kernel(int, unsigned short const*, unsigned int const*, unsigned int*, r2x::DirectBin, r2x::TilePlan, unsigned int*, int, int, unsigned int const*, int)",
    "r2x::raster_render_ws_kernel(int, int, int, uint2 const*, unsigned int const*, float4 const*, r2x::TilePlan, float*)",
    "r2x::ssim_stats_kernel(int, int, float const*, float const*, r2x::SsimWindow, float*, float*)",
    "r2x::ssim_reduce_kernel(int, float const*, float, float, float, float*)",
    "r2x::ssim_grad_kernel(int, int, float const*, float const*, r2x::SsimWindow, float const*, float, float, float, float*)",
    "r2x::voxel_preprocess_kernel(int, float const*, float const*, float, float const*, float const*, float const*, r2x::VoxelGrid, int, int*, int*, int*, r2x::VoxelGeom, r2x::DirectBin, int, r2x::Activation)",
    "r2x::voxel_render_kernel(r2x::VoxelGrid, uint2 const*, unsigned int const*, float4 const*, r2x::TilePlan, float*)",
    "r2x::tv3d_kernel(int, int, int, float const*, float, float*, float*)",
    "r2x::tv3d_reduce_kernel(int, float const*, float, float*)",
    "void at::native::vectorized_elementwise_kernel<4, at::native::AUnaryFunctor<float, float, float, at::native::binary_internal::MulFunctor<float> >, std::array<char*, 2ul> >(int, at::native::AUnaryFunctor<float, float, float, at::native::binary_internal::MulFunctor<float> >, std::array<char*, 2ul>)",
    "r2x::voxel_render_bwd_kernel(r2x::VoxelGrid, uint2 const*, unsigned int const*, unsigned int const*, r2x::VoxelGeom, float4 const*, r2x::TilePlan, float const*, float4*)",
    "r2x::voxel_gauss_bwd_kernel(int, int const*, int const*, int const*, float const*, float, float const*, float const*, r2x::VoxelGrid, r2x::VoxelGeom, long long, unsigned int const*, float4 const*, float*, float*, float*, float*, float*, r2x::Activation)",
    "r2x::raster_render_bwd2_kernel(int, int, int, uint2 const*, unsigned int const*, unsigned int const*, r2x::RasterGeom, float4 const*, float4 const*, float const*, r2x::TilePlan, float const*, float4*, int)",
    "void r2x::raster_gauss_bwd_kernel<false>(int, float const*, int const*, float const*, float, float const*, float const*, float const*, float const*, int, int, float, float, float, float, int, r2x::RasterGeom, long long, unsigned int const*, float4 const*, float*, float*, float*, float*, float*, float*, float*, r2x::Activation, float*)",
    "r2x::densify_stats_kernel(int, int const*, float const*, float*, float*, float*, unsigned int const*, unsigned int const*)",
    "r2x::adam_kernel(r2x::AdamPack, float, float, float, float, float, float)",
    "void at::native::vectorized_elementwise_kernel<4, at::native::(anonymous namespace)::softplus_kernel(at::TensorIteratorBase&, c10::Scalar const&, c10::Scalar const&)::{lambda()#1}::operator()() const::{lambda()#2}::operator()() const::{lambda(float)#1}, std::array<char*, 2ul> >(int, at::native::(anonymous namespace)::softplus_kernel(at::TensorIteratorBase&, c10::Scalar const&, c10::Scalar const&)::{lambda()#1}::operator()() const::{lambda()#2}::operator()() const::{lambda(float)#1}, std::array<char*, 2ul>)",
]
PARENT_SEQUENCE = [
    0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 10, 11, 12, 13, 14, 3, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 10, 11, 12, 13, 14, 3, 0,
    1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 10, 11, 12, 13, 14, 3, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 10, 11, 12, 13, 14, 3, 0, 1,
    2, 3, 4, 5, 6, 7, 8, 9, 10, 10, 11, 12, 13, 14, 3, 15, 16, 17, 18, 19, 20, 21, 22, 21, 23, 24, 21, 25, 26, 27, 3, 1,
    2, 1, 1, 1, 1, 28, 1, 1, 28, 1, 1, 1, 1, 1, 1, 1, 1, 1, 29, 30, 31, 32, 33, 34, 35, 36, 30, 31, 37, 38, 39, 40, 41,
    42, 43, 44, 45, 46, 47, 29, 30, 31, 32, 33, 34, 35, 36, 30, 31, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47, 29, 30,
    31, 32, 33, 34, 35, 36, 30, 31, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47, 29, 30, 31, 32, 33, 34, 35, 36, 30, 31,
    37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47, 29, 30, 31, 32, 33, 34, 35, 36, 30, 31, 37, 38, 39, 40, 41, 42, 43, 44,
    45, 46, 47, 29, 30, 31, 32, 33, 34, 35, 36, 30, 31, 37, 38, 39, 40, 41, 42, 43, 44, 45, 47
]


def _trainer_kernel_sequence(workdir):
    """Kernel names, in launch order, of a 6-iteration trainer run (TV on, no densification, no saves) on a small
    synthetic scene, in a fresh process so no capacity hint of another test changes the path."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from r2_gaussian_b200 import scene, trainer
    from r2_gaussian_b200.dataset import write_blender
    rng = np.random.RandomState(0)
    sc = scene.cone_beam_scanner(32, 16)
    sc.update({"filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0, "noise": False})
    frames = [(0.4 * k, rng.rand(32, 32).astype(np.float32)) for k in range(5)]
    src = os.path.join(workdir, "scene")
    write_blender(src, sc, frames[:4], frames[4:], rng.rand(16, 16, 16).astype(np.float32))
    pts = np.concatenate([rng.uniform(-0.8, 0.8, (3000, 3)), rng.uniform(0.05, 0.5, (3000, 1))], 1)
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    model = trainer.ModelParams(source_path=src, model_path="")
    opt = trainer.OptimizationParams(iterations=6)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        trainer.training(model, opt, trainer.PipelineParams(), init_points=pts, log=lambda *a: None)
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA), key=lambda e: e.time_range.start)
    return [e.name for e in ev if not e.name.startswith(("Memcpy", "Memset"))]


def test_trainer_without_pose_refine_issues_the_same_kernels(tmp_path):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path)], capture_output=True, text=True,
                       env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-4000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    assert len(names) > 6 * 10
    assert [PARENT_KERNELS[k] for k in PARENT_SEQUENCE] == names


if __name__ == "__main__":
    print(json.dumps(_trainer_kernel_sequence(sys.argv[1])))
