"""The horizontal detector offset, without a GPU: both device entries reject bad arguments before any CUDA call, the
trainer's `--detector_offset_refine` settings parse into their own dataclass, leave `cfg_args` as it was when off, and
are refused with --pose_refine and with Gaussian sharding before any CUDA work or process group."""
import ast
import ctypes
import json
from dataclasses import asdict

import pytest

from r2_gaussian_b200 import _lib, trainer

_P = lambda x: None if x is None else ctypes.c_void_p(0x1000 * x)   # never dereferenced: the checks come first


def _apply(lib, offset=1, W=64, n=3, full=1, out=2):
    return lib.r2x_detector_offset_apply(None, _P(offset), W, n, _P(full), _P(out))


def _grad(lib, P=100, n=2, W=64, g=1, out=1, scratch=1, nbytes=None):
    if nbytes is None:
        nbytes = lib.r2x_detector_offset_grad_scratch_bytes(max(P, 0), max(n, 1))
    return lib.r2x_detector_offset_grad(None, P, n, W, _P(g), _P(out), _P(scratch), nbytes)


@pytest.mark.parametrize("kw,msg", [
    (dict(offset=None), b"null pointer"), (dict(full=None), b"null pointer"), (dict(out=None), b"null pointer"),
    (dict(W=0), b"W must be positive"), (dict(W=-5), b"W must be positive"), (dict(n=0), b"n_views"),
    (dict(n=-1), b"n_views"), (dict(n=1 << 27), b"n_views"),
])
def test_detector_offset_apply_rejects_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    assert _apply(lib, **kw) == 1
    err = lib.r2x_last_error()
    assert b"r2x_detector_offset_apply" in err and msg in err, err


@pytest.mark.parametrize("kw,msg", [
    (dict(g=None), b"null pointer"), (dict(out=None), b"null pointer"), (dict(scratch=None), b"null pointer"),
    (dict(P=-1), b"P must be non-negative"), (dict(n=0), b"n_views"), (dict(W=0), b"W must be positive"),
    (dict(nbytes=0), b"scratch smaller"), (dict(P=10 ** 6, n=4, nbytes=8), b"scratch smaller"),
])
def test_detector_offset_grad_rejects_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    assert _grad(lib, **kw) == 1
    err = lib.r2x_last_error()
    assert b"r2x_detector_offset_grad" in err and msg in err, err


def test_detector_offset_grad_scratch_grows_with_the_rows_and_is_bounded():
    lib = _lib.load()
    sizes = [lib.r2x_detector_offset_grad_scratch_bytes(P, n) for P, n in ((0, 1), (1, 1), (5000, 1), (100_000, 1),
                                                                          (100_000, 4), (10 ** 8, 16))]
    assert sizes[0] == sizes[1] == 8
    assert sizes == sorted(sizes) and sizes[-1] == 1024 * 8
    assert lib.r2x_detector_offset_grad_scratch_bytes(-1, 1) == 0 and lib.r2x_detector_offset_grad_scratch_bytes(5, 0) == 0


def test_detector_offset_refine_parses_into_its_own_dataclass():
    a, model, pipe, opt, pose = trainer.parse_args(["-s", "scene"])
    assert a.detector_params == trainer.DetectorParams() and not a.detector_params.detector_offset_refine
    assert not any(k.startswith("detector") for k in asdict(opt))
    assert not any(k.startswith("detector") for k in asdict(pose))
    a2, _, _, opt2, pose2 = trainer.parse_args(["-s", "scene", "--detector_offset_refine", "--detector_offset_lr_init",
                                                "0.2", "--batch_size", "1"])
    d = a2.detector_params
    assert d.detector_offset_refine and d.detector_offset_lr_init == 0.2
    assert d.detector_offset_lr_final == trainer.DetectorParams.detector_offset_lr_final
    assert opt2 == opt and pose2 == pose


def test_detector_params_defaults_decay():
    d = trainer.DetectorParams()
    assert not d.detector_offset_refine
    assert 0 < d.detector_offset_lr_final < d.detector_offset_lr_init


def _cfg(tmp_path, det):
    a, model, pipe, opt, pose = trainer.parse_args(["-s", "scene"])
    extra = {"test_iterations": [1], "save_iterations": [], "checkpoint_iterations": [], "start_checkpoint": None,
             "quiet": False, "config": None, "detect_anomaly": False}
    trainer.write_cfg_args(str(tmp_path), model, pipe, opt, extra, pose, det)
    text = (tmp_path / "cfg_args").read_text()
    assert text.startswith("Namespace(")
    keys = {kw.arg for kw in ast.parse(text).body[0].value.keywords}
    doc = json.loads((tmp_path / "cfg_args.json").read_text())
    today = set(asdict(model)) | set(asdict(pipe)) | set(asdict(opt)) | set(extra)
    return keys, doc, today


@pytest.mark.parametrize("det", [None, trainer.DetectorParams()], ids=["no-detector-arg", "detector-off"])
def test_cfg_args_without_the_switch_has_todays_keys(tmp_path, det):
    keys, doc, today = _cfg(tmp_path, det)
    assert keys == today
    assert set(doc) == {"model", "pipe", "opt"}
    assert not any("detector" in k for k in keys)


def test_cfg_args_with_the_switch_records_the_detector_settings(tmp_path):
    keys, doc, today = _cfg(tmp_path, trainer.DetectorParams(detector_offset_refine=True))
    assert keys == today | set(asdict(trainer.DetectorParams()))
    assert doc["detector"] == asdict(trainer.DetectorParams(detector_offset_refine=True))


def test_refusal_rules():
    assert trainer.detector_refusal(False, True, 8) is None
    assert trainer.detector_refusal(True, False, 1) is None
    assert "--pose_refine" in trainer.detector_refusal(True, True, 1)
    assert "WORLD_SIZE" in trainer.detector_refusal(True, False, 2)


def _no_cuda_work(monkeypatch):
    """Any CUDA initialisation or library call from here on fails the test."""
    import torch

    def boom(*a, **k):
        raise AssertionError("CUDA work before the refusal")
    monkeypatch.setattr(torch.cuda, "init", boom)
    monkeypatch.setattr(torch.cuda, "synchronize", boom)
    monkeypatch.setattr(_lib, "load", boom)
    monkeypatch.setattr(trainer, "Scene", boom)


@pytest.mark.parametrize("args,env,needle", [
    (["--pose_refine"], "1", "--pose_refine"),
    ([], "2", "WORLD_SIZE"),
    (["--batch_size", "2"], "2", "WORLD_SIZE"),
], ids=["pose", "sharded", "sharded-batch"])
def test_refused_before_cuda_work_or_a_process_group(tmp_path, monkeypatch, capsys, args, env, needle):
    import torch.distributed as dist
    _no_cuda_work(monkeypatch)
    monkeypatch.setenv("WORLD_SIZE", env)
    out = tmp_path / "out"
    with pytest.raises(SystemExit) as e:
        trainer.main(["-s", str(tmp_path), "-m", str(out), "--detector_offset_refine", *args])
    assert e.value.code != 0
    err = capsys.readouterr().err
    assert needle in err, err
    assert not dist.is_initialized()
    assert not out.exists()


@pytest.mark.parametrize("pose,world,needle", [(True, 1, "--pose_refine"), (False, 2, "WORLD_SIZE")])
def test_training_refuses_before_cuda_work(tmp_path, monkeypatch, pose, world, needle):
    _no_cuda_work(monkeypatch)
    monkeypatch.setattr(trainer, "world_info", lambda: (0, world))
    with pytest.raises((ValueError, RuntimeError), match=needle):
        trainer.training(trainer.ModelParams(source_path=str(tmp_path)), trainer.OptimizationParams(iterations=1),
                         trainer.PipelineParams(), pose_params=trainer.PoseParams(pose_refine=pose),
                         detector_params=trainer.DetectorParams(detector_offset_refine=True))


def test_detector_offset_yml_names_the_horizontal_field_of_the_scanner_file(tmp_path):
    """Scanner files list offDetector as [u, v] (unlike nDetector / sDetector, [v, u]): the horizontal offset goes to
    offDetector[0], TIGRE's geo.offDetector[1], with the opposite sign of the learned offset."""
    import types

    import torch
    import yaml

    from r2_gaussian_b200.detector import SIGN_CONVENTION, DetectorOffset
    det = DetectorOffset("cpu")
    with torch.no_grad():
        det.offset.fill_(2.5)
    cfg = {"nDetector": [64, 128], "sDetector": [1.0, 2.0]}          # [v, u]
    sc = types.SimpleNamespace(model_path=str(tmp_path), scanner_cfg=cfg)
    (tmp_path / "point_cloud" / "iteration_7").mkdir(parents=True)
    trainer.save_detector_offset(sc, det, 7)
    doc = yaml.safe_load((tmp_path / "point_cloud" / "iteration_7" / "detector_offset.yml").read_text())
    assert doc["offset_px"] == 2.5
    assert doc["offset_scene"] == pytest.approx(2.5 * 2.0 / 128)     # pixels along u times dDetector[1] (u)
    assert doc["sign_convention"] == SIGN_CONVENTION
    assert "offDetector[0] (u; TIGRE geo.offDetector[1]) = -offset_scene" in SIGN_CONVENTION
    assert "offDetector[1] =" not in SIGN_CONVENTION
    assert "larger column index" in SIGN_CONVENTION


def _case(tmp_path, edge=0.0):
    import numpy as np

    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.dataset import write_blender
    rng = np.random.RandomState(0)
    sc = scene.cone_beam_scanner(16, 8)
    sc.update({"filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0, "noise": False})
    frames = []
    for k in range(3):
        a = np.zeros((16, 16), np.float32)
        a[:, 4:12] = rng.rand(16, 8) + 0.5
        a[0, -1] = edge
        frames.append((0.5 * k, a))
    path = str(tmp_path / "case")
    write_blender(path, sc, frames[:2], frames[2:], rng.rand(8, 8, 8).astype(np.float32))
    return path


def _projections(path):
    import numpy as np
    meta = json.load(open(f"{path}/meta_data.json"))
    return [np.load(f"{path}/{fr['file_path']}") for s in ("proj_train", "proj_test") for fr in meta[s]]


@pytest.mark.parametrize("k", [3, -2])
def test_shift_projections_moves_every_view_and_fills_zeros(tmp_path, k):
    import numpy as np

    from r2_gaussian_b200 import generate_data
    path = _case(tmp_path)
    before = _projections(path)
    generate_data.shift_projections(path, k)
    after = _projections(path)
    assert len(after) == 3
    for a, b in zip(before, after):
        assert np.array_equal(b, np.roll(a, k, axis=1))                  # content was clear of the lost columns
        assert not np.any(b[:, :k] if k > 0 else b[:, k:])


def test_shift_projections_refuses_content_that_would_fall_off_and_writes_nothing(tmp_path):
    import numpy as np

    from r2_gaussian_b200 import generate_data
    path = _case(tmp_path, edge=0.25)
    before = _projections(path)
    with pytest.raises(ValueError, match="not empty"):
        generate_data.shift_projections(path, 3)
    assert all(np.array_equal(a, b) for a, b in zip(before, _projections(path)))
    generate_data.shift_projections(path, -3)                           # the other edge is empty
