"""Training on B views per iteration, without a GPU: the new C entries reject bad arguments before any CUDA call, the
trainer refuses `--batch_size` values and combinations it cannot run before any CUDA work or process group, leaves
`cfg_args` as it was at B = 1, and draws the B = 1 camera sequence grouped by B."""
import ast
import ctypes
import json
import random

import numpy as np
import pytest
import torch

from r2_gaussian_b200 import _lib, trainer
from r2_gaussian_b200.dataset import write_blender

NEW = ["r2x_raster_forward_views_async_raw", "r2x_raster_backward_views_raw", "r2x_image_loss_views_scratch_bytes",
       "r2x_image_loss_views", "r2x_densify_stats_views"]
FAKE = ctypes.c_void_p(1 << 20)   # never dereferenced: every case fails its checks first


def test_abi_exports_the_batch_calls():
    lib = _lib.load()
    for name in NEW:
        assert hasattr(lib, name) and name in _lib.PROTOTYPES


def _act():
    a = _lib.ActivationDesc()
    a.scale_mode, a.scale_lo, a.scale_hi = 1, 0.001, 1.0
    return a


def _fwd(lib, P=10, N=2, W=64, H=64, ptr=FAKE, binning=FAKE, act=True):
    return lib.r2x_raster_forward_views_async_raw(None, P, N, W, H, ptr, ptr, ptr, 1.0, ptr, ptr, ptr, 1.0, 1.0, 1, ptr,
                                                  ptr, ptr, ptr, binning, 1 << 20, None,
                                                  ctypes.byref(_act()) if act else None)


def _bwd(lib, N=2, H=64, ptr=FAKE, views=FAKE, act=True):
    return lib.r2x_raster_backward_views_raw(None, 10, N, 100, 64, H, ptr, ptr, 1.0, ptr, views, ptr, 1.0, 1.0, ptr, ptr,
                                             ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr, ptr, 1,
                                             ctypes.byref(_act()) if act else None)


@pytest.mark.parametrize("kw,msg", [
    (dict(N=0), b"bad N"), (dict(N=-1), b"bad N"), (dict(N=4097, H=256), b"tile rows"), (dict(ptr=None), b"null"),
    (dict(binning=None), b"binning"), (dict(act=False), b"null activation"),
])
def test_raw_views_forward_rejects_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    assert _fwd(lib, **kw) != 0
    err = lib.r2x_last_error()
    assert b"r2x_raster_forward_views_async" in err and msg in err, err


@pytest.mark.parametrize("kw,msg", [
    (dict(N=0), b"bad N"), (dict(N=4097, H=256), b"tile rows"), (dict(views=None), b"null"), (dict(ptr=None), b"null"),
    (dict(act=False), b"null activation"),
])
def test_raw_views_backward_rejects_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    assert _bwd(lib, **kw) != 0
    err = lib.r2x_last_error()
    assert b"r2x_raster_backward_views" in err and msg in err, err


def _loss(lib, N=3, H=64, W=64, img=FAKE, scratch=FAKE, nbytes=None):
    nbytes = lib.r2x_image_loss_views_scratch_bytes(max(N, 1), H, W) if nbytes is None else nbytes
    return lib.r2x_image_loss_views(None, N, H, W, img, FAKE, 1.0, 0.25, FAKE, FAKE, scratch, nbytes)


@pytest.mark.parametrize("kw,msg", [
    (dict(N=0), b"bad N"), (dict(N=-2), b"bad N"), (dict(N=65536), b"bad N"), (dict(H=0), b"bad H/W"),
    (dict(img=None), b"null pointer"), (dict(scratch=None), b"null pointer"), (dict(nbytes=1024), b"scratch too small"),
])
def test_image_loss_views_rejects_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    assert _loss(lib, **kw) != 0
    err = lib.r2x_last_error()
    assert b"r2x_image_loss_views" in err and msg in err, err


def test_image_loss_views_scratch_is_one_slab_per_image():
    lib = _lib.load()
    one = lib.r2x_image_loss_views_scratch_bytes(1, 512, 512)
    assert one >= lib.r2x_image_loss_scratch_bytes(512, 512)
    assert lib.r2x_image_loss_views_scratch_bytes(4, 512, 512) - 256 == 4 * (one - 256)
    assert lib.r2x_image_loss_views_scratch_bytes(0, 512, 512) == 0


@pytest.mark.parametrize("kw,msg", [(dict(N=0), b"bad N"), (dict(P=-1), b"bad N/P"), (dict(radii=None), b"null")])
def test_densify_stats_views_rejects_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    a = dict(N=2, P=10, radii=FAKE)
    a.update(kw)
    assert lib.r2x_densify_stats_views(None, a["N"], a["P"], a["radii"], FAKE, FAKE, FAKE, FAKE, None, None) != 0
    err = lib.r2x_last_error()
    assert b"r2x_densify_stats_views" in err and msg in err, err


# ---- trainer -----------------------------------------------------------------------------------------------------------

def _scene(tmp_path, n_train=4):
    from r2_gaussian_b200 import scene
    rng = np.random.RandomState(0)
    sc = scene.cone_beam_scanner(16, 8)
    sc.update({"filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0, "noise": False})
    frames = [(0.4 * k, rng.rand(16, 16).astype(np.float32)) for k in range(n_train + 1)]
    src = str(tmp_path / "scene")
    write_blender(src, sc, frames[:n_train], frames[n_train:], rng.rand(8, 8, 8).astype(np.float32))
    return src


def _refused(capsys, argv, needle):
    with pytest.raises(SystemExit) as e:
        trainer.parse_args(argv)
    assert e.value.code != 0
    assert needle in capsys.readouterr().err


def test_batch_size_limits_are_refused(tmp_path, capsys):
    src = _scene(tmp_path)
    _refused(capsys, ["-s", src, "--batch_size", "0"], "at least 1")
    _refused(capsys, ["-s", src, "--batch_size", "5"], "exceeds the scene's 4 train views")
    a, *_ = trainer.parse_args(["-s", src, "--batch_size", "4"])
    assert a.batch_size == 4
    assert trainer.parse_args(["-s", "no-such-scene"])[0].batch_size == 1      # B = 1 never reads the scene


def test_batch_size_combinations_are_refused(tmp_path, capsys, monkeypatch):
    src = _scene(tmp_path)
    _refused(capsys, ["-s", src, "--batch_size", "2", "--pose_refine"], "--pose_refine")
    _refused(capsys, ["-s", src, "--batch_size", "2", "--compute_cov3D_python"], "compute_cov3D_python")
    monkeypatch.setenv("WORLD_SIZE", "2")
    _refused(capsys, ["-s", src, "--batch_size", "2"], "WORLD_SIZE > 1")


def test_batch_size_with_sharding_is_refused_before_any_process_group(tmp_path, monkeypatch, capsys):
    import torch.distributed as dist
    src = _scene(tmp_path)
    monkeypatch.setenv("WORLD_SIZE", "2")
    out = tmp_path / "out"
    with pytest.raises(SystemExit):
        trainer.main(["-s", src, "-m", str(out), "--batch_size", "2"])
    assert "WORLD_SIZE" in capsys.readouterr().err
    assert not dist.is_initialized() and not out.exists()


def test_training_refuses_before_the_scene_is_loaded():
    model = trainer.ModelParams(source_path="no-such-scene")
    for kw, msg in ((dict(batch_size=0), "at least 1"),
                    (dict(batch_size=2, pose_params=trainer.PoseParams(pose_refine=True)), "--pose_refine")):
        with pytest.raises(ValueError, match=msg):
            trainer.training(model, trainer.OptimizationParams(), trainer.PipelineParams(), **kw)
    with pytest.raises(ValueError, match="compute_cov3D_python"):
        trainer.training(model, trainer.OptimizationParams(), trainer.PipelineParams(compute_cov3D_python=True),
                         batch_size=2)


def _cfg_keys(tmp_path, argv):
    src = _scene(tmp_path)
    out = tmp_path / "out"
    seen = {}
    real = trainer.training
    try:
        trainer.training = lambda *a, **k: seen.update(k) or {"eval": {}, "iterations": 1, "seconds": 0.0,
                                                             "train_seconds": 0.0, "gaussians": 0}
        trainer.main(["-s", src, "-m", str(out), *argv])
    finally:
        trainer.training = real
    text = (out / "cfg_args").read_text()
    return {kw.arg: kw.value for kw in ast.parse(text).body[0].value.keywords}, json.loads((out / "cfg_args.json").read_text()), seen


def test_cfg_args_unchanged_at_batch_size_one(tmp_path, capsys):
    keys, doc, seen = _cfg_keys(tmp_path, [])
    a, model, pipe, opt, _ = trainer.parse_args(["-s", "x"])
    extra = {"test_iterations", "save_iterations", "checkpoint_iterations", "start_checkpoint", "quiet", "config",
             "detect_anomaly"}
    assert set(keys) == set(vars(model)) | set(vars(pipe)) | set(vars(opt)) | extra
    assert set(doc) == {"model", "pipe", "opt"} and seen["batch_size"] == 1
    printed = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
    assert "batch_size" not in printed
    keys4, _, seen4 = _cfg_keys(tmp_path / "b4", ["--batch_size", "4"])
    assert set(keys4) == set(keys) | {"batch_size"} and ast.literal_eval(keys4["batch_size"]) == 4 and seen4["batch_size"] == 4


def _draws(B, steps, n_train=6, seed=0):
    random.seed(seed)
    cams, stack, out = list(range(n_train)), None, []
    for _ in range(steps):
        views, stack = trainer.draw_train_views(stack, cams, B)
        out.append(views)
    return out


def test_camera_sequence_is_the_single_view_one_grouped_by_b():
    one, four = _draws(1, 20), _draws(4, 5)
    assert all(len(d) == 1 for d in one) and all(len(d) == 4 for d in four)
    flat = [u for d in one for u in d]
    assert [u for d in four for u in d] == flat
    assert sorted(flat[:6]) == list(range(6)) and sorted(flat[6:12]) == list(range(6))   # one pass, then a refill
