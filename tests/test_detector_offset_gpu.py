"""The horizontal detector offset: the device kernels and both training paths that use them.

1. r2x_detector_offset_apply: s = 0 bit for bit; within 1 float32 ulp of a float64 torch statement;
2. geometry and sign: render() with the shifted matrices is the nominal render moved s columns towards larger index;
3. r2x_detector_offset_grad: against a float64 sum, against the matrix gradients of r2x_raster_backward_pose, against
   central differences; bitwise reproducible; a batch of views is the sum of its single views;
4. `NativeTrainStep(detector=...)` is the autograd iteration bit for bit (B = 1 and B = 4, with and without TV), and
   an iteration repeated after a capacity overflow moves the offset once;
5. the trainer: without the switch the same kernel launches as before; a resumed checkpoint ends where the
   uninterrupted run ends; `--detector_offset_refine` recovers a 3-column shift of a generate_data scene.
"""
import json
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
ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))


def _bits(x):
    return x.contiguous().view(torch.int32)


def _cameras(n, mode=1, det=128):
    from r2_gaussian_b200 import scene
    sc = scene.cone_beam_scanner(det, 64) if mode == 1 else scene.parallel_beam_scanner(det, 64)
    cams = []
    for k in range(n):
        v = scene.make_view(sc, 0.3 + 0.83 * k)
        c = scene.camera_from_view(v)
        c.view = v
        cams.append(c)
    return cams


def _float64_shift(full, s, W):
    f = full.double()
    out = f.clone()
    out[..., :, 0] = f[..., :, 0] + (2.0 * s / W) * f[..., :, 3]
    return out


# ---- 1. apply kernel -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [1, 7])
@pytest.mark.parametrize("mode", [1, 0], ids=["cone", "parallel"])
def test_apply_kernel_is_exact_at_zero_and_within_one_ulp(mode, n):
    from r2_gaussian_b200.detector import DetectorOffset
    cams = _cameras(n, mode)
    W = int(cams[0].image_width)
    det = DetectorOffset(DEV)
    out = det.cameras(cams)
    for c, o in zip(cams, out):
        assert torch.equal(_bits(o.full_proj_transform), _bits(c.full_proj_transform))
        assert o.world_view_transform is c.world_view_transform
    full = torch.stack([c.full_proj_transform for c in cams])
    for s in (3.0, -1.37, 0.25, 1e-6, 250.5):
        with torch.no_grad():
            det.offset.fill_(s)
        got = det.apply(full, W)
        ref = _float64_shift(full, float(np.float32(s)), W)
        ref32 = ref.float()
        sp = torch.from_numpy(np.spacing(np.abs(ref32.cpu().numpy())).astype(np.float64)).to(DEV)
        assert ((got.double() - ref).abs() <= sp).all(), s
        # only the x row changes; the others are copied
        for j in (1, 2, 3):
            assert torch.equal(_bits(got[..., :, j]), _bits(full[..., :, j]))
        one = det.camera(cams[-1]).full_proj_transform
        assert torch.equal(_bits(one), _bits(got[-1]))


# ---- 2. geometry and sign --------------------------------------------------------------------------------------------

def _centred_cloud(mode):
    from r2_gaussian_b200 import scene
    return scene.make_cloud(4000, kind="trained", seed=3, s_voxel=(1.0, 1.0, 1.0) if mode == 1 else (0.8, 0.8, 0.8))


def _render(cloud, cam):
    from r2_gaussian_b200.render_query import render
    from test_pose_gpu import _Model, _Pipe
    return render(cam, _Model(cloud, True), _Pipe())


def _shifted_and_moved(mode, s):
    """(render with offset s, nominal render moved s columns towards larger index, image maximum) in float64."""
    from r2_gaussian_b200.detector import DetectorOffset
    cloud = _centred_cloud(mode)
    cam = _cameras(1, mode)[0]
    with torch.no_grad():
        base = _render(cloud, cam)["render"][0].double()
    assert float(base[:, -16:].abs().max()) == 0.0 and float(base[:, :16].abs().max()) == 0.0   # clear of the edges
    det = DetectorOffset(DEV)
    with torch.no_grad():
        det.offset.fill_(float(s))
        img = _render(cloud, det.camera(cam))["render"][0].double()
    moved = torch.zeros_like(base)
    moved[:, s:] = base[:, :-s]
    return img, moved, base


@pytest.mark.parametrize("mode", [1, 0], ids=["cone", "parallel"])
def test_an_integer_offset_moves_the_render_towards_larger_column_index(mode):
    """s = 16 (one whole tile): the nominal render moved 16 columns within 1e-5 max + 1e-7, away from the left 16
    columns.  s = 3: the shift that best matches the two images is +3 (sign and size of the map), and the images agree
    within 0.5 % of the maximum; the 1e-5 bar at s = 3 is the strict expected failure below."""
    for s, bar in ((16, 1e-5), (3, 5e-3)):
        img, moved, base = _shifted_and_moved(mode, s)
        err = float((img - moved)[:, s:].abs().max())
        top = float(base.abs().max())
        print(f"mode {mode} s {s}: max error {err:.3g} of max {top:.4g}")
        assert err <= bar * top + 1e-7, (s, err, top)
        miss = {k: float((img[:, 20:-20] - torch.roll(base, k, 1)[:, 20:-20]).abs().sum()) for k in range(s - 6, s + 7)}
        assert min(miss, key=miss.get) == s, miss


@pytest.mark.xfail(strict=True, raises=AssertionError, reason="finding (H100): at s = 3 the render with the offset "
                   "differs from the nominal render moved 3 columns by 0.0101 of a maximum of 4.70 (cone) and 0.0071 of "
                   "3.80 (parallel), against the bar 1e-5 max + 1e-7.  The 16-pixel tile rectangles of the 3-sigma radii "
                   "fall differently after a shift that is not a whole tile, so a pixel just beyond a Gaussian's radius "
                   "is rendered in one geometry and not in the other (up to e^-4.5 of its peak); at s = 16 the bar "
                   "holds (1.4e-6).  The bar stays as fixed; strict, so a change that makes it hold is noticed")
@pytest.mark.parametrize("mode", [1, 0], ids=["cone", "parallel"])
def test_a_three_column_offset_is_the_moved_render_within_1e5_of_max(mode):
    img, moved, base = _shifted_and_moved(mode, 3)
    err = float((img - moved)[:, 3:].abs().max())
    top = float(base.abs().max())
    print(f"mode {mode} s 3: max error {err:.3g} of max {top:.4g}")
    assert err <= 1e-5 * top + 1e-7, (err, top)


# ---- 3. gradient kernel ----------------------------------------------------------------------------------------------

def _view_and_grad(cloud, cam, s, dl_seed=0):
    """Render `cam` shifted by s with a ramp-plus-noise dL/dimage; -> (dL_dmean2D [P,3], dL/dfull [4,4], full')."""
    from r2_gaussian_b200 import fused
    from r2_gaussian_b200.detector import DetectorOffset
    from r2_gaussian_b200.rasterization import GaussianRasterizationSettings
    from test_pose_gpu import _dl, _leaves
    det = DetectorOffset(DEV)
    with torch.no_grad():
        det.offset.fill_(s)
    v = cam.view
    full = det.camera(cam).full_proj_transform.clone().requires_grad_(True)
    tv = cam.world_view_transform.clone().requires_grad_(True)
    p = _leaves(cloud, True)
    m2 = torch.zeros_like(p["means"], requires_grad=True)
    st = GaussianRasterizationSettings(v.image_height, v.image_width, v.tanfovx, v.tanfovy, 1.0, tv.detach(),
                                       full.detach(), torch.tensor(v.campos, device=DEV), False, v.mode, False)
    rawp = {"density": p["dens"], "scaling": p["scales"], "rotation": p["rots"], "scale_bound": None}
    img, _ = fused.rasterize_raw_matrices(p["means"], m2, rawp, tv, full, st)
    img.backward(_dl(v.image_height, v.image_width, dl_seed))
    torch.cuda.synchronize()
    return m2.grad.detach(), full.grad.detach(), det


@pytest.mark.parametrize("mode", [1, 0], ids=["cone", "parallel"])
def test_grad_kernel_against_float64_sum_and_the_matrix_gradients(mode):
    from r2_gaussian_b200 import scene
    cloud = scene.make_cloud(20_000, kind="trained", seed=5)
    cam = _cameras(1, mode, det=256)[0]
    W = int(cam.image_width)
    g2, gfull, det = _view_and_grad(cloud, cam, 0.7)
    got = float(det.grad_from(g2, W))
    ref = float(2.0 / W * g2[:, 0].double().sum())
    assert got != 0.0 and abs(got - ref) <= 1e-6 * abs(ref), (got, ref)
    # the same derivative through the matrix gradients: d full[k][0] / ds = (2 / W) full[k][3]
    chain = float((gfull[:, 0].double() * (2.0 / W) * cam.full_proj_transform[:, 3].double()).sum())
    print(f"mode {mode}: dL/ds {got:.6g}, float64 sum {ref:.6g}, through dL/dprojmatrix {chain:.6g}")
    assert abs(got - chain) <= 1e-4 * abs(chain), (got, chain)


def test_grad_kernel_agrees_with_central_differences():
    """The loss sum(dL * image) through render() at s +- h, h = 0.25 px, on a smooth scene (a few hundred broad
    Gaussians).  The per-Gaussian gradient convention holds cull, radii and tile rectangles fixed, which the finite
    difference does not, so the bar is loose: 5 % relative."""
    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.detector import DetectorOffset
    from test_pose_gpu import _dl
    cloud = scene.make_cloud(400, kind="init", seed=7, s_voxel=(1.0, 1.0, 1.0))
    cam = _cameras(1, 1)[0]
    W = int(cam.image_width)
    dl = _dl(cam.image_height, W, 3)
    s0, h = 0.4, 0.25
    g2, _, det = _view_and_grad(cloud, cam, s0, dl_seed=3)
    got = float(det.grad_from(g2, W))

    def loss(s):
        d = DetectorOffset(DEV)
        with torch.no_grad():
            d.offset.fill_(s)
            return float((_render(cloud, d.camera(cam))["render"].double() * dl.double()).sum())
    fd = (loss(s0 + h) - loss(s0 - h)) / (2 * h)
    print(f"dL/ds kernel {got:.6g}, central difference {fd:.6g}")
    assert abs(got - fd) <= 0.05 * abs(fd), (got, fd)


def test_grad_kernel_is_reproducible_and_a_batch_is_the_sum_of_its_views():
    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.detector import DetectorOffset
    from test_pose_gpu import _dl
    det = DetectorOffset(DEV)
    # bitwise reproducible, on a size that takes the full stage-one grid
    g = torch.randn((4, 300_000, 3), device=DEV, generator=torch.Generator("cuda").manual_seed(1))
    a = det.grad_from(g, 512).clone()
    b = det.grad_from(g, 512).clone()
    assert torch.equal(_bits(a), _bits(b)) and det.offset.grad.shape == (1,)
    ref = 2.0 / 512 * g[..., 0].double().sum()
    assert abs(float(a) - float(ref)) <= 1e-6 * abs(float(ref))
    # B = 4 views rendered in one batched call: the view-order sum of the single-view values
    from r2_gaussian_b200 import trainer
    from test_train_gpu import _make_model
    gm, _, _ = _make_model(n=5000, seed=21)
    cams = _cameras(4, 1)
    W = int(cams[0].image_width)
    with torch.no_grad():
        det.offset.fill_(1.5)
    pkg = trainer.render_batch(det.cameras(cams), gm)
    dls = torch.stack([_dl(c.image_height, W, k)[0] for k, c in enumerate(cams)])
    (pkg["render"] * dls).sum().backward()
    batched = float(det.grad_from(pkg["viewspace_points"].grad, W))
    singles = []
    pipe = types.SimpleNamespace(compute_cov3D_python=False, debug=False)
    from r2_gaussian_b200.render_query import render
    for k, c in enumerate(cams):
        gm.optimizer.zero_grad(set_to_none=True)
        p = render(det.camera(c), gm, pipe)
        (p["render"][0] * dls[k]).sum().backward()
        singles.append(float(det.grad_from(p["viewspace_points"].grad, W)))
    want = sum(singles)
    print(f"batched {batched:.7g}, single views {singles}")
    assert abs(batched - want) <= 1e-6 * sum(abs(x) for x in singles), (batched, singles)
    # an empty cloud gives 0
    assert float(det.grad_from(torch.zeros((0, 3), device=DEV), W)) == 0.0


# ---- 4. native step == autograd iteration ----------------------------------------------------------------------------

def _detector_pair(s0=0.4):
    from r2_gaussian_b200.detector import DetectorOffset
    from r2_gaussian_b200.optim import FusedAdam
    out = []
    for _ in range(2):
        det = DetectorOffset(DEV)
        with torch.no_grad():
            det.offset.fill_(s0)
        out.append((det, FusedAdam([det.offset], lr=2e-2, eps=1e-15)))
    return out


def _assert_detector_equal(da, oa, db, ob, steps):
    assert torch.equal(_bits(da.offset.detach()), _bits(db.offset.detach()))
    sa, sb = oa.state[da.offset], ob.state[db.offset]
    assert torch.equal(_bits(sa["exp_avg"]), _bits(sb["exp_avg"]))
    assert torch.equal(_bits(sa["exp_avg_sq"]), _bits(sb["exp_avg_sq"]))
    assert float(sa["step"]) == float(sb["step"]) == steps


def _assert_models_equal(a, b, steps):
    for name in ("_xyz", "_density", "_scaling", "_rotation"):
        ga, gb = getattr(a, name), getattr(b, name)
        assert torch.equal(_bits(ga), _bits(gb)), name
        sa, sb = a.optimizer.state[ga], b.optimizer.state[gb]
        assert torch.equal(sa["exp_avg"], sb["exp_avg"]) and torch.equal(sa["exp_avg_sq"], sb["exp_avg_sq"]), name
        assert float(sa["step"]) == float(sb["step"]) == steps
    for name in ("max_radii2D", "xyz_gradient_accum", "denom"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name


@pytest.mark.parametrize("use_tv", [True, False], ids=["tv", "no-tv"])
@pytest.mark.parametrize("B", [1, 4])
def test_native_detector_step_is_the_autograd_iteration(B, use_tv):
    from r2_gaussian_b200 import losses, trainer
    from r2_gaussian_b200.render_query import query, render
    from r2_gaussian_b200.train_step import NativeTrainStep
    from test_train_gpu import _make_model, _train_inputs
    pipe = types.SimpleNamespace(compute_cov3D_python=False, debug=False)
    cams, gts, centres = _train_inputs(n_cams=8)
    W = int(cams[0].image_width)
    lam_d, lam_tv, n_it = 0.25, 0.05, 7
    tv_n, tv_s = [32, 32, 32], [0.5, 0.5, 0.5]
    a, _, _ = _make_model(n=5000, seed=11)
    b, _, _ = _make_model(n=5000, seed=11)
    (da, oa), (db, ob) = _detector_pair()
    s_start = float(da.offset)
    step = NativeTrainStep(b, lam_d, lam_tv if use_tv else 0.0, tv_n, tv_s, detector=(db, ob))
    for i in range(1, n_it + 1):
        idx = [(B * i + j) % len(cams) for j in range(B)]
        bc, bg = [cams[j] for j in idx], torch.stack([gts[j] for j in idx])
        centre = centres[i % len(centres)]
        a.update_learning_rate(i); b.update_learning_rate(i)
        if B == 1:
            pkg = render(da.camera(bc[0]), a, pipe)
            total = losses.image_loss(pkg["render"], bg[0], lam_d)["total"]
        else:
            pkg = trainer.render_batch(da.cameras(bc), a)
            total = sum(losses.image_loss(pkg["render"][v], bg[v], lambda_dssim=lam_d)["total"] for v in range(B))
        if use_tv:
            total = total + (B * lam_tv) * losses.tv_3d_loss(query(a, centre, tv_n, tv_s, pipe)["vol"], "mean")
        total.backward()
        with torch.no_grad():
            g = pkg["viewspace_points"].grad
            da.grad_from(g, W)
            if B == 1:
                a.update_max_radii(pkg["radii"], pkg["visibility_filter"])
                a.add_densification_stats(pkg["viewspace_points"], pkg["visibility_filter"])
            else:
                for v in range(B):
                    seen = pkg["radii"][v] > 0
                    a.update_max_radii(pkg["radii"][v], seen)
                    a.add_densification_stats(trainer._ViewGrad(g[v]), seen)
        a.optimizer.step(); a.optimizer.zero_grad(set_to_none=True)
        oa.step(); oa.zero_grad(set_to_none=True)
        res = step(bc if B > 1 else bc[0], bg if B > 1 else bg[0], centre)
        if i == n_it:
            assert torch.equal(res["radii"], pkg["radii"])
    step.flush()
    assert step.repeats == 0
    _assert_models_equal(a, b, n_it)
    _assert_detector_equal(da, oa, db, ob, n_it)
    assert float(db.offset) != s_start


@pytest.mark.parametrize("B", [1, 4])
def test_native_detector_step_repeats_an_overflowed_iteration_once(B):
    from r2_gaussian_b200 import _C
    from r2_gaussian_b200.train_step import NativeTrainStep
    from test_train_gpu import _make_model, _train_inputs
    cams, gts, centres = _train_inputs(n_cams=4)
    batch = lambda i: ([cams[(i + j) % 4] for j in range(B)], torch.stack([gts[(i + j) % 4] for j in range(B)]))
    arg = lambda i: (batch(i)[0], batch(i)[1]) if B > 1 else (cams[i % 4], gts[i % 4])
    a, _, _ = _make_model(n=5000, seed=13)
    b, _, _ = _make_model(n=5000, seed=13)
    (da, oa), (db, ob) = _detector_pair(0.0)
    sa = NativeTrainStep(a, 0.25, 0.05, [32, 32, 32], [0.5, 0.5, 0.5], detector=(da, oa))
    sb = NativeTrainStep(b, 0.25, 0.05, [32, 32, 32], [0.5, 0.5, 0.5], detector=(db, ob))
    for i in (1, 2):
        a.update_learning_rate(i); sa(*arg(i), centres[i])
    sa.flush()
    b.update_learning_rate(1); sb(*arg(1), centres[1]); sb.flush()
    lib = sb.lib
    sb.cap_r = 4096
    sb.binning_r = torch.empty(lib.r2x_binning_bytes(4096), dtype=torch.uint8, device="cuda")
    sb.scratch_r = torch.empty(lib.r2x_raster_bwd_scratch_bytes(4096), dtype=torch.uint8, device="cuda")
    saved = dict(_C._Workspace.hints)
    _C._Workspace.hints[sb.key_r] = 1
    sb._provision = lambda: None
    b.update_learning_rate(2)
    before = (b._xyz.clone(), db.offset.detach().clone())
    sb(*arg(2), centres[2])
    torch.cuda.synchronize()
    assert torch.equal(before[0], b._xyz) and torch.equal(before[1], db.offset)
    del sb._provision
    sb.cap_r = 0
    sb.flush()
    assert sb.repeats == 1
    _C._Workspace.hints.update({k: v for k, v in saved.items() if k == sb.key_r})
    for name in ("_xyz", "_density", "_scaling", "_rotation"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    _assert_detector_equal(da, oa, db, ob, 2)
    assert not torch.equal(before[1], db.offset)


# ---- 5. the trainer --------------------------------------------------------------------------------------------------

def _small_scene(workdir):
    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.dataset import write_blender
    rng = np.random.RandomState(0)
    sc = scene.cone_beam_scanner(32, 16)
    sc.update({"filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0, "noise": False})
    frames = [(0.4 * k, rng.rand(32, 32).astype(np.float32)) for k in range(5)]
    src = os.path.join(workdir, "scene")
    write_blender(src, sc, frames[:4], frames[4:], rng.rand(16, 16, 16).astype(np.float32))
    pts = np.concatenate([rng.uniform(-0.8, 0.8, (3000, 3)), rng.uniform(0.05, 0.5, (3000, 1))], 1)
    return src, pts


def _kernel_sequence(workdir):
    """The kernel names of test_pose_train_gpu's 6-iteration trainer run, with the detector settings passed off."""
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    from r2_gaussian_b200 import trainer
    src, pts = _small_scene(workdir)
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    model = trainer.ModelParams(source_path=src, model_path="")
    opt = trainer.OptimizationParams(iterations=6)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        trainer.training(model, opt, trainer.PipelineParams(), init_points=pts, log=lambda *a: None,
                         detector_params=trainer.DetectorParams())
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA), key=lambda e: e.time_range.start)
    return [e.name for e in ev if not e.name.startswith(("Memcpy", "Memset"))]


def test_trainer_without_the_switch_issues_the_same_kernels(tmp_path):
    from test_pose_train_gpu import PARENT_KERNELS, PARENT_SEQUENCE
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path)], capture_output=True, text=True,
                       env=env, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-4000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    assert not any("detector_offset" in n for n in names)
    assert [PARENT_KERNELS[k] for k in PARENT_SEQUENCE] == names


def _run_small(src, pts, out, iterations, refine, checkpoint_iterations=(), start=None, B=1, rng=None):
    from r2_gaussian_b200 import trainer
    if rng is None:
        random.seed(0); np.random.seed(0); torch.manual_seed(0)
    else:
        random.setstate(rng[0]); np.random.set_state(rng[1]); torch.set_rng_state(rng[2])
    model = trainer.ModelParams(source_path=src, model_path=str(out))
    opt = trainer.OptimizationParams(iterations=iterations)
    return trainer.training(model, opt, trainer.PipelineParams(), {iterations}, {iterations},
                            set(checkpoint_iterations), start, init_points=pts, log=lambda *a: None, batch_size=B,
                            detector_params=trainer.DetectorParams(detector_offset_refine=refine))


@pytest.mark.parametrize("B", [1, 2])
def test_checkpoint_resume_ends_equal_and_refuses_the_other_setting(tmp_path, monkeypatch, B):
    """A run of 12 iterations checkpointed at 8 (4 train views: the camera stack is empty there, as after a resume)
    against the run resumed from that checkpoint with the host RNG states of that moment: the same offset, offset Adam
    state and Gaussians, bit for bit.  Resuming with the other setting raises."""
    import yaml
    src, pts = _small_scene(str(tmp_path))
    states, save = {}, torch.save

    def save_and_snapshot(obj, path, *a, **k):
        states[os.path.basename(str(path))] = (random.getstate(), np.random.get_state(), torch.get_rng_state())
        return save(obj, path, *a, **k)
    monkeypatch.setattr(torch, "save", save_and_snapshot)
    full = _run_small(src, pts, tmp_path / "full", 12, True, checkpoint_iterations=(8,), B=B)
    monkeypatch.setattr(torch, "save", save)
    ck = str(tmp_path / "full" / "ckpt" / "chkpnt8.pth")
    payload = torch.load(ck, weights_only=False)
    assert len(payload) == 5 and payload[3] is None and set(payload[4]) == {"offset", "optimizer"}
    resumed = _run_small(src, pts, tmp_path / "resumed", 12, True, start=ck, B=B, rng=states["chkpnt8.pth"])
    da, db = full["detector"], resumed["detector"]
    assert float(da.offset) != 0.0
    assert torch.equal(_bits(da.offset.detach()), _bits(db.offset.detach()))
    for name in ("_xyz", "_density", "_scaling", "_rotation"):
        assert torch.equal(_bits(getattr(full["model"], name)), _bits(getattr(resumed["model"], name))), name
    doc = yaml.safe_load(open(tmp_path / "full" / "point_cloud" / "iteration_12" / "detector_offset.yml"))
    cfg = full["scene"].scanner_cfg
    assert doc["offset_px"] == float(da.offset.detach()[0])
    assert doc["offset_scene"] == pytest.approx(doc["offset_px"] * cfg["sDetector"][1] / cfg["nDetector"][1], rel=1e-6)
    assert "larger column index" in doc["sign_convention"]
    with pytest.raises(RuntimeError, match="detector_offset_refine"):
        _run_small(src, pts, tmp_path / "other", 12, False, start=ck, B=B)
    _run_small(src, pts, tmp_path / "plain", 4, False, checkpoint_iterations=(2,), B=B)
    with pytest.raises(RuntimeError, match="detector_offset_refine"):
        _run_small(src, pts, tmp_path / "other2", 4, True, start=str(tmp_path / "plain" / "ckpt" / "chkpnt2.pth"), B=B)


# ---- recovery through the trainer ------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def shifted_scenes(tmp_path_factory):
    from detector_cases import recovery_scenes
    return recovery_scenes(tmp_path_factory.mktemp("detector_scene"))


def test_detector_offset_recovers_a_three_column_shift_through_the_trainer(shifted_scenes, tmp_path):
    from r2_gaussian_b200 import trainer
    from detector_cases import ITERATIONS as it, SHIFT, train
    runs = {}
    for scene_name in ("shifted", "plain"):
        path, init = shifted_scenes[scene_name]
        for refine in (False, True):
            h = train(path, init, tmp_path / f"{scene_name}_{refine}",
                      trainer.DetectorParams(detector_offset_refine=refine))
            runs[scene_name, refine] = (h["eval"][it]["psnr_3d"], h.get("detector_offset_px"), h["train_seconds"])
    for k, v in runs.items():
        print(f"{k}: psnr_3d {v[0]:.3f}, offset {v[1]}, train {v[2]:.2f} s")
    assert not os.path.exists(tmp_path / "shifted_False" / "point_cloud" / f"iteration_{it}" / "detector_offset.yml")
    assert os.path.exists(tmp_path / "shifted_True" / "point_cloud" / f"iteration_{it}" / "detector_offset.yml")
    p_sh_off, _, _ = runs["shifted", False]
    p_sh_on, s_sh, _ = runs["shifted", True]
    p_pl_off, _, _ = runs["plain", False]
    p_pl_on, s_pl, _ = runs["plain", True]
    assert abs(s_sh - SHIFT) <= 0.1, s_sh
    assert p_sh_on >= p_sh_off + 3.0, (p_sh_off, p_sh_on)
    assert p_sh_on >= p_pl_off - 1.5, (p_pl_off, p_sh_on)
    assert abs(s_pl) <= 0.1, s_pl
    assert abs(p_pl_on - p_pl_off) <= 0.3, (p_pl_off, p_pl_on)


if __name__ == "__main__":
    print(json.dumps(_kernel_sequence(sys.argv[1])))
