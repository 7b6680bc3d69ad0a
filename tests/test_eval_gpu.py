"""Device-side evaluation (`metrics.volume_metrics` / `projection_metrics`) and `python -m r2_gaussian_b200.test` on
the GPU.

1. Metrics: the counted slices equal metric_vol / metric_proj's exactly; every per-slice SSIM is within 1e-5 of a
   float64 statement of `metrics.ssim` (with the kernel's float32 taps), the aggregates within 1e-5 of the torch
   functions (float32 convolutions, TF32 off) and PSNR within 1e-4 dB; empty volumes raise ZeroDivisionError, an
   all-zero prediction gives metric_proj's non-finite values; two calls give the same bits; one device-to-host copy
   per call; the kernel's N and H limits are met by chunking and transposing.
2. End to end on a 48^3 generate_data scene: the written volume and renders are bit for bit the trainer's saved volume
   and `render()`, the scores agree with the trainer's `eval/` files, with and without pose / detector corrections,
   `--iteration -1` picks the last save and each `--skip_*` flag removes exactly its files."""
import math
import os
import shutil

import numpy as np
import pytest
import torch
import torch.nn.functional as F
import yaml

import train_edge_cases as te
from r2_gaussian_b200 import metrics

pytestmark = pytest.mark.gpu

SSIM_BAR = 1e-5
PSNR_BAR = 1e-4


@pytest.fixture(autouse=True)
def _float32_convolutions():
    """The torch functions are compared in float32: cuDNN may otherwise pick TF32 convolutions (10-bit mantissa)."""
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = old


def ssim64_rows(x, y, chunk=64):
    """Mean SSIM of each pair of [N, H, W] images in float64: `metrics.ssim` with the 11-tap window taken as the outer
    product of the kernel's float32 taps (separable), zero padding, C1 = 0.01^2, C2 = 0.03^2."""
    g = torch.tensor(te.ssim_taps(), dtype=torch.float64, device=x.device)
    gv, gh = g.reshape(1, 1, 11, 1), g.reshape(1, 1, 1, 11)
    conv = lambda t: F.conv2d(F.conv2d(t, gv, padding=(5, 0)), gh, padding=(0, 5))
    out = []
    for s in range(0, x.shape[0], chunk):
        a, b = x[s:s + chunk, None].double(), y[s:s + chunk, None].double()
        mu1, mu2 = conv(a), conv(b)
        s11, s22, s12 = conv(a * a) - mu1 * mu1, conv(b * b) - mu2 * mu2, conv(a * b) - mu1 * mu2
        C1, C2 = 0.01 ** 2, 0.03 ** 2
        m = ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s11 + s22 + C2))
        out.append(m.mean(dim=(1, 2, 3)))
    return torch.cat(out)


def _phantom(shape, seed, zero_border=True):
    """A smooth non-negative volume with noise, and slices whose maximum is 0 at the low end of each long axis."""
    gen = torch.Generator("cuda").manual_seed(seed)
    grids = torch.meshgrid(*[torch.linspace(-1, 1, n, device="cuda") for n in shape], indexing="ij")
    r2 = sum(g * g for g in grids)
    vol = torch.clamp(1.0 - r2, min=0) + 0.05 * torch.rand(shape, generator=gen, device="cuda")
    if zero_border:
        for ax, n in enumerate(shape):
            if n > 2:
                vol.select(ax, 0).zero_()
    return vol.float().contiguous()


def _noisy(vol, seed, scale=0.1):
    gen = torch.Generator("cuda").manual_seed(seed)
    return (vol + scale * torch.randn(vol.shape, generator=gen, device="cuda")).float().contiguous()


def _torch_counted(stack_along_axis0):
    return [bool(s.max() > 0) for s in stack_along_axis0]


VOLUMES = [(20, 36, 28), (1, 11, 17), (5, 12, 17), (17, 1, 11), (12, 5, 1), (11, 17, 5), (256, 256, 256)]


def _check_volume(shape, seed=0):
    gt = _phantom(shape, seed)
    pred = _noisy(gt, seed + 1)
    parts = metrics.volume_slice_scores(gt, pred)
    got = metrics.volume_metrics(gt, pred)
    want_psnr = metrics.metric_vol(gt, pred, "psnr")[0]
    want_ssim, want_axes = metrics.metric_vol(gt, pred, "ssim")
    assert abs(got["psnr_3d"] - want_psnr) <= PSNR_BAR, (got["psnr_3d"], want_psnr)
    worst = 0.0
    for axis in range(3):
        g, p = gt.movedim(axis, 0), pred.movedim(axis, 0)
        rows, counted = parts[1 + 2 * axis], parts[2 + 2 * axis]
        assert counted.bool().tolist() == _torch_counted(g), (shape, axis)
        err = (rows - ssim64_rows(g, p)).abs().max().item()
        worst = max(worst, err)
        assert err <= SSIM_BAR, (shape, axis, err)
        assert abs(got[f"ssim_3d_{'xyz'[axis]}"] - want_axes[axis]) <= SSIM_BAR, (shape, axis)
    assert abs(got["ssim_3d"] - want_ssim) <= SSIM_BAR
    return worst


@pytest.mark.parametrize("shape", VOLUMES, ids=lambda s: "x".join(map(str, s)))
def test_volume_metrics_against_metric_vol_and_float64(shape):
    worst = _check_volume(shape)
    print(f"{shape}: worst per-slice |ssim - ssim64| {worst:.3g}")


def test_volume_metrics_at_512_cubed():
    worst = _check_volume((512, 512, 512), seed=5)
    print(f"512^3: worst per-slice |ssim - ssim64| {worst:.3g}")


def _views(N, H=560, W=560, seed=0):
    gen = torch.Generator("cuda").manual_seed(seed)
    y = torch.linspace(-1, 1, H, device="cuda")[:, None]
    x = torch.linspace(-1, 1, W, device="cuda")[None, :]
    amp = 0.5 + torch.rand(N, 1, 1, generator=gen, device="cuda")
    base = torch.clamp(1.0 - (x * x + y * y), min=0)[None] * amp
    gt = (base + 0.02 * torch.rand(N, H, W, generator=gen, device="cuda")).float()
    pred = (gt * 1.1 + 0.05 * torch.randn(N, H, W, generator=gen, device="cuda")).float()
    if N > 2:
        gt[1].zero_()                   # a view that is not counted
    return gt.contiguous(), pred.contiguous()


@pytest.mark.parametrize("N", [1, 150, 721])
def test_projection_metrics_against_metric_proj_and_float64(N):
    gt, pred = _views(N, seed=N)
    got = metrics.projection_metrics(gt, pred)
    psnr_v, ssim_v, counted = metrics.projection_view_scores(gt, pred)
    hwn = (gt.permute(1, 2, 0), pred.permute(1, 2, 0))
    want_psnr, want_psnr_l = metrics.metric_proj(*hwn, "psnr")
    want_ssim, want_ssim_l = metrics.metric_proj(*hwn, "ssim")
    assert counted.bool().tolist() == _torch_counted(gt)
    assert len(got["psnr_2d_projs"]) == len(got["ssim_2d_projs"]) == N
    assert [v == 0.0 for v in got["ssim_2d_projs"]] == [v == 0.0 for v in want_ssim_l]
    assert max(abs(a - b) for a, b in zip(got["psnr_2d_projs"], want_psnr_l)) <= PSNR_BAR
    assert abs(got["psnr_2d"] - want_psnr) <= PSNR_BAR
    a = gt / gt.amax(dim=(1, 2), keepdim=True)
    b = pred / pred.amax(dim=(1, 2), keepdim=True)
    keep = counted.bool()
    err = (ssim_v[keep] - ssim64_rows(a[keep], b[keep])).abs().max().item()
    assert err <= SSIM_BAR, err
    assert max(abs(x - y) for x, y in zip(got["ssim_2d_projs"], want_ssim_l)) <= SSIM_BAR
    assert abs(got["ssim_2d"] - want_ssim) <= SSIM_BAR
    print(f"N={N}: worst per-view |ssim - ssim64| {err:.3g}")


def test_empty_volumes_and_stacks():
    shape = (9, 13, 7)
    border = torch.zeros(shape, device="cuda")
    border[0], border[-1] = 0.7, 0.3          # non-zero only in two slices of axis 0
    border[:, 0] += 0.2
    pred = _noisy(border, 2)
    got = metrics.volume_metrics(border, pred)
    want_ssim, want_axes = metrics.metric_vol(border, pred, "ssim")
    parts = metrics.volume_slice_scores(border, pred)
    for axis in range(3):
        assert parts[2 + 2 * axis].bool().tolist() == _torch_counted(border.movedim(axis, 0))
        assert abs(got[f"ssim_3d_{'xyz'[axis]}"] - want_axes[axis]) <= SSIM_BAR
    zero = torch.zeros(shape, device="cuda")
    with pytest.raises(ZeroDivisionError):
        metrics.metric_vol(zero, pred, "ssim")
    with pytest.raises(ZeroDivisionError):
        metrics.volume_metrics(zero, pred)
    with pytest.raises(ZeroDivisionError):
        metrics.metric_proj(zero.permute(1, 2, 0), pred.permute(1, 2, 0), "psnr")
    with pytest.raises(ZeroDivisionError):
        metrics.projection_metrics(zero, pred)


def test_an_all_zero_prediction_gives_metric_projs_non_finite_values():
    gt, pred = _views(4, 64, 48, seed=3)
    pred[2].zero_()
    got = metrics.projection_metrics(gt, pred)
    hwn = (gt.permute(1, 2, 0), pred.permute(1, 2, 0))
    for metric in ("psnr", "ssim"):
        agg, per = metrics.metric_proj(*hwn, metric)
        mine = got[f"{metric}_2d_projs"]
        assert math.isnan(per[2]) and math.isnan(mine[2]), (metric, per[2], mine[2])
        assert all(math.isfinite(v) for i, v in enumerate(mine) if i != 2)
        assert math.isnan(agg) and math.isnan(got[f"{metric}_2d"])


def test_two_calls_give_the_same_bits_and_chunking_changes_none(monkeypatch):
    gt = _phantom((40, 33, 50), 7)
    pred = _noisy(gt, 8)
    a, b = metrics.volume_metrics(gt, pred), metrics.volume_metrics(gt, pred)
    assert a == b
    g2, p2 = _views(30, 70, 90, seed=4)
    c, d = metrics.projection_metrics(g2, p2), metrics.projection_metrics(g2, p2)
    assert c == d
    monkeypatch.setattr(metrics, "VIEWS_MAX_N", 7)
    assert metrics.volume_metrics(gt, pred) == a and metrics.projection_metrics(g2, p2) == c
    monkeypatch.setattr(metrics, "VIEWS_MAX_N", 65535)
    monkeypatch.setattr(metrics, "SSIM_SCRATCH_BYTES", 1)      # one image per call
    assert metrics.volume_metrics(gt, pred) == a and metrics.projection_metrics(g2, p2) == c


def test_one_device_to_host_copy_per_call():
    from torch.profiler import ProfilerActivity, profile
    gt = _phantom((24, 31, 18), 9)
    pred = _noisy(gt, 10)
    g2, p2 = _views(5, 40, 30, seed=6)
    metrics.volume_metrics(gt, pred), metrics.projection_metrics(g2, p2)     # warm
    for fn, args in ((metrics.volume_metrics, (gt, pred)), (metrics.projection_metrics, (g2, p2))):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn(*args)
            torch.cuda.synchronize()
        d2h = [e for e in prof.events() if "DtoH" in e.name or "Device -> Pageable" in e.name]
        gpu_d2h = [e for e in d2h if e.device_type == torch.autograd.DeviceType.CUDA]
        assert len(gpu_d2h) == 1, (fn.__name__, [e.name for e in d2h])


def test_the_kernel_limits_are_met_by_chunking_and_transposing():
    # 65 537 slices along axis 0: two calls of the kernel (N <= 65535)
    gt = _phantom((65537, 2, 3), 11, zero_border=False)
    pred = _noisy(gt, 12)
    parts = metrics.volume_slice_scores(gt, pred)
    got = metrics.volume_metrics(gt, pred)
    for axis in range(3):
        g, p = gt.movedim(axis, 0), pred.movedim(axis, 0)
        ref = ssim64_rows(g.contiguous(), p.contiguous(), chunk=4096)
        assert (parts[1 + 2 * axis] - ref).abs().max().item() <= SSIM_BAR, axis
        assert abs(got[f"ssim_3d_{'xyz'[axis]}"] - ref.mean().item()) <= SSIM_BAR, axis
    # an image taller than 65535 16-row tiles: run transposed
    H = metrics.IMAGE_MAX_H + 1
    g2 = _phantom((2, H, 2), 13, zero_border=False)
    p2 = _noisy(g2, 14)
    psnr_v, ssim_v, counted = metrics.projection_view_scores(g2, p2)
    a = g2 / g2.amax(dim=(1, 2), keepdim=True)
    b = p2 / p2.amax(dim=(1, 2), keepdim=True)
    assert (ssim_v - ssim64_rows(a, b)).abs().max().item() <= SSIM_BAR


def test_refusals_on_the_device():
    v = torch.rand(4, 5, 6, device="cuda")
    for fn in (metrics.volume_metrics, metrics.projection_metrics):
        with pytest.raises(TypeError, match="float32"):
            fn(v.double(), v.double())
        with pytest.raises(ValueError, match="shapes differ"):
            fn(v, v[:, :, :5].contiguous())
        with pytest.raises(ValueError, match="3-D"):
            fn(v[0], v[0])
        with pytest.raises(RuntimeError, match="CUDA"):
            fn(v, v.cpu())


# ---- 2. the driver end to end -------------------------------------------------------------------------------------------

ITERS = (150, 300)


@pytest.fixture(scope="module")
def scene_48(tmp_path_factory):
    """A 48^3 generate_data scene (24 train and 6 test views of 96^2) and a random initial cloud."""
    from r2_gaussian_b200 import generate_data, initialize_pcd
    from test_projector_gpu import _write_inputs
    tmp = tmp_path_factory.mktemp("eval_scene")
    yml, vol_path, *_ = _write_inputs(tmp, noise=False)
    src = generate_data.main(["--vol", str(vol_path), "--scanner", str(yml), "--n_train", "24", "--n_test", "6",
                              "--output", str(tmp / "data")])
    init = initialize_pcd.main(["--data", src, "--n_points", "5000", "--output", str(tmp / "init.npy")])
    return src, init


def _train(scene_48, out, *flags):
    from r2_gaussian_b200 import trainer
    src, init = scene_48
    it = [str(i) for i in ITERS]
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False          # the trainer's metric_vol / metric_proj in float32 too
    trainer.main(["-s", src, "-m", str(out), "--ply_path", init, "--iterations", it[-1], "--test_iterations", *it,
                  "--save_iterations", *it, *flags])
    torch.backends.cudnn.allow_tf32 = old
    return out


@pytest.fixture(scope="module")
def models(scene_48, tmp_path_factory):
    root = tmp_path_factory.mktemp("eval_models")
    return {"plain": _train(scene_48, root / "plain"),
            "pose": _train(scene_48, root / "pose", "--pose_refine"),
            "detector": _train(scene_48, root / "detector", "--detector_offset_refine")}


def _files(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


def _load(path):
    with open(path) as f:
        return yaml.safe_load(f)


def _eval_against_trainer(model, res, n):
    ev_dir = os.path.join(model, "eval", f"iter_{n:06d}")
    t3 = _load(os.path.join(ev_dir, "eval3d.yml"))
    mine3 = _load(os.path.join(res["path"], "eval3d.yml"))
    assert list(mine3) == ["psnr_3d", "ssim_3d", "ssim_3d_x", "ssim_3d_y", "ssim_3d_z"]
    assert abs(mine3["psnr_3d"] - t3["psnr_3d"]) <= PSNR_BAR and abs(mine3["ssim_3d"] - t3["ssim_3d"]) <= SSIM_BAR
    for split, n_views in (("train", 24), ("test", 6)):
        t2 = _load(os.path.join(ev_dir, f"eval2d_render_{split}.yml"))
        mine2 = _load(os.path.join(res["path"], f"eval2d_render_{split}.yml"))
        assert list(mine2) == ["psnr_2d", "ssim_2d", "psnr_2d_projs", "ssim_2d_projs"]
        assert len(mine2["psnr_2d_projs"]) == len(mine2["ssim_2d_projs"]) == n_views
        assert abs(mine2["psnr_2d"] - t2["psnr_2d"]) <= PSNR_BAR, (split, mine2["psnr_2d"], t2["psnr_2d"])
        assert abs(mine2["ssim_2d"] - t2["ssim_2d"]) <= SSIM_BAR, (split, mine2["ssim_2d"], t2["ssim_2d"])
    return mine3


def _renders_are_render(model, res, settings, iteration):
    """Each written prediction is bit for bit render() of its view with the evaluation's cameras."""
    from r2_gaussian_b200 import test as evaltest
    from r2_gaussian_b200.dataset import Scene
    from r2_gaussian_b200.gaussian_model import GaussianModel
    from r2_gaussian_b200.render_query import render
    from r2_gaussian_b200.trainer import PipelineParams, evaluation_cameras
    scene = Scene(settings["source_path"], str(model), shuffle=False, device="cuda")
    g = GaussianModel(None)
    it_dir = os.path.join(model, "point_cloud", f"iteration_{iteration}")
    g.load_ply(os.path.join(it_dir, "point_cloud.pickle"))
    pose, det = evaltest.correction_modules(it_dir, scene)
    pipe = PipelineParams()
    with torch.no_grad():
        for split, cams in evaluation_cameras(scene, pose, det):
            for i, c in enumerate(cams):
                want = render(c, g, pipe)["render"][0].cpu().numpy()
                got = np.load(os.path.join(res["path"], f"render_{split}", f"{i:05d}_pred.npy"))
                gt = np.load(os.path.join(res["path"], f"render_{split}", f"{i:05d}_gt.npy"))
                assert got.dtype == np.float32 and got.shape == want.shape
                assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (split, i)
                assert np.array_equal(gt, c.original_image[0].cpu().numpy()), (split, i)
    return scene, g, pipe


def test_the_driver_matches_the_trainers_save_and_scores(models):
    from r2_gaussian_b200 import test as evaltest
    model = str(models["plain"])
    res = evaltest.main(["-m", model, "--quiet"])
    n = ITERS[-1]
    assert res["iteration"] == n and res["path"] == os.path.join(model, "test", f"iter_{n}")
    saved = np.load(os.path.join(model, "point_cloud", f"iteration_{n}", "vol_pred.npy"))
    mine = np.load(os.path.join(res["path"], "vol_pred.npy"))
    assert np.array_equal(mine.view(np.uint32), saved.view(np.uint32))
    vg = np.load(os.path.join(res["path"], "vol_gt.npy"))
    for i in range(mine.shape[2]):
        assert np.array_equal(np.load(os.path.join(res["path"], "reconstruction", f"{i:05d}_pred.npy")), mine[..., i])
        assert np.array_equal(np.load(os.path.join(res["path"], "reconstruction", f"{i:05d}_gt.npy")), vg[..., i])
    _eval_against_trainer(model, res, n)
    _renders_are_render(model, res, evaltest.load_settings(model), n)
    print(f"plain: {res['seconds']}")
    # an earlier save
    early = evaltest.main(["-m", model, "--iteration", str(ITERS[0]), "--quiet"])
    assert early["path"] == os.path.join(model, "test", f"iter_{ITERS[0]}")
    _eval_against_trainer(model, early, ITERS[0])


@pytest.mark.parametrize("kind", ["pose", "detector"])
def test_the_driver_applies_the_learned_corrections(models, kind):
    from r2_gaussian_b200 import test as evaltest
    from r2_gaussian_b200.metrics import projection_metrics
    from r2_gaussian_b200.render_query import render
    model = str(models[kind])
    n = ITERS[-1]
    it_dir = os.path.join(model, "point_cloud", f"iteration_{n}")
    assert os.path.exists(os.path.join(it_dir, "train_poses.npz" if kind == "pose" else "detector_offset.yml"))
    res = evaltest.main(["-m", model, "--quiet"])
    _eval_against_trainer(model, res, n)
    scene, g, pipe = _renders_are_render(model, res, evaltest.load_settings(model), n)
    # without the corrections the train scores differ
    with torch.no_grad():
        cams = scene.getTrainCameras()
        preds = torch.cat([render(c, g, pipe)["render"] for c in cams], 0)
        gts = torch.cat([c.original_image for c in cams], 0)
        nominal = projection_metrics(gts, preds)
    corrected = _load(os.path.join(res["path"], "eval2d_render_train.yml"))
    print(f"{kind}: train psnr_2d corrected {corrected['psnr_2d']:.6f}, nominal {nominal['psnr_2d']:.6f}")
    assert nominal["psnr_2d"] != corrected["psnr_2d"] and nominal["psnr_2d_projs"] != corrected["psnr_2d_projs"]


def test_each_skip_flag_removes_exactly_its_files(models):
    from r2_gaussian_b200 import test as evaltest
    model = str(models["plain"])
    out = os.path.join(model, "test", f"iter_{ITERS[-1]}")
    shutil.rmtree(out, ignore_errors=True)
    evaltest.main(["-m", model, "--quiet"])
    full = set(_files(out))
    groups = {"--skip_render_train": lambda f: f.startswith("render_train") or f == "eval2d_render_train.yml",
              "--skip_render_test": lambda f: f.startswith("render_test") or f == "eval2d_render_test.yml",
              "--skip_recon": lambda f: f.startswith("reconstruction") or f.startswith("vol_") or f == "eval3d.yml"}
    assert len(full) == 2 * 24 + 1 + 2 * 6 + 1 + 2 * 48 + 1 + 4
    for flag, owned in groups.items():
        shutil.rmtree(out)
        evaltest.main(["-m", model, flag, "--quiet"])
        assert set(_files(out)) == {f for f in full if not owned(f)}, flag
