"""Pose refinement in training, without a GPU: the device pose entries reject bad arguments before any CUDA call, and
the trainer's `--pose_refine` settings parse into their own dataclass, leave `cfg_args` as it was when off, and are
refused together with Gaussian sharding before any process group exists."""
import ast
import ctypes
import json
from dataclasses import asdict

import pytest

from r2_gaussian_b200 import _lib, trainer

_P = lambda x: None if x is None else ctypes.c_void_p(0x1000 * x)   # never dereferenced: the checks come first


def _apply(lib, omega=1, nu=1, n=4, i=0, view=1, full=1, proj=1, out_view=1, out_full=1):
    return lib.r2x_pose_apply(None, _P(omega), _P(nu), n, i, _P(view), _P(full), _P(proj), _P(out_view), _P(out_full))


def _grad(lib, omega=1, nu=1, n=4, i=0, anchor=0, view=1, proj=1, gview=1, gproj=1, go=1, gn=1):
    return lib.r2x_pose_grad(None, _P(omega), _P(nu), n, i, anchor, _P(view), _P(proj), _P(gview), _P(gproj), _P(go),
                             _P(gn))


@pytest.mark.parametrize("kw,msg", [
    (dict(omega=None), b"null pointer"), (dict(nu=None), b"null pointer"), (dict(view=None), b"null pointer"),
    (dict(full=None), b"null pointer"), (dict(proj=None), b"null pointer"), (dict(out_view=None), b"null pointer"),
    (dict(out_full=None), b"null pointer"), (dict(n=0), b"n_views"), (dict(n=-2), b"n_views"),
    (dict(i=-1), b"view index"), (dict(i=4), b"view index"),
])
def test_pose_apply_rejects_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    assert _apply(lib, **kw) == 1
    err = lib.r2x_last_error()
    assert b"r2x_pose_apply" in err and msg in err, err


@pytest.mark.parametrize("kw,msg", [
    (dict(omega=None), b"null pointer"), (dict(nu=None), b"null pointer"), (dict(view=None), b"null pointer"),
    (dict(proj=None), b"null pointer"), (dict(gview=None), b"null pointer"), (dict(gproj=None), b"null pointer"),
    (dict(go=None), b"null pointer"), (dict(gn=None), b"null pointer"), (dict(n=0), b"n_views"),
    (dict(i=-1), b"view index"), (dict(i=4), b"view index"), (dict(anchor=-2), b"anchor"), (dict(anchor=4), b"anchor"),
])
def test_pose_grad_rejects_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    assert _grad(lib, **kw) == 1
    err = lib.r2x_last_error()
    assert b"r2x_pose_grad" in err and msg in err, err


def test_pose_refine_parses_into_its_own_dataclass():
    a, model, pipe, opt, pose = trainer.parse_args(["-s", "scene"])
    assert pose == trainer.PoseParams() and not pose.pose_refine
    assert not any(k.startswith("pose") for k in asdict(opt))
    _, _, _, opt2, pose = trainer.parse_args(["-s", "scene", "--pose_refine", "--pose_rotation_lr_init", "2e-3",
                                              "--pose_translation_lr_final", "1e-6"])
    assert pose.pose_refine and pose.pose_rotation_lr_init == 2e-3 and pose.pose_translation_lr_final == 1e-6
    assert pose.pose_rotation_lr_final == trainer.PoseParams.pose_rotation_lr_final
    assert opt2 == opt


def _cfg(tmp_path, pose):
    a, model, pipe, opt, _ = trainer.parse_args(["-s", "scene"])
    extra = {"test_iterations": [1], "save_iterations": [], "checkpoint_iterations": [], "start_checkpoint": None,
             "quiet": False, "config": None, "detect_anomaly": False}
    trainer.write_cfg_args(str(tmp_path), model, pipe, opt, extra, pose)
    text = (tmp_path / "cfg_args").read_text()
    assert text.startswith("Namespace(")
    keys = {kw.arg for kw in ast.parse(text).body[0].value.keywords}
    doc = json.loads((tmp_path / "cfg_args.json").read_text())
    today = set(asdict(model)) | set(asdict(pipe)) | set(asdict(opt)) | set(extra)
    return keys, doc, today


@pytest.mark.parametrize("pose", [None, trainer.PoseParams()], ids=["no-pose-arg", "pose-off"])
def test_cfg_args_without_pose_refine_has_todays_keys(tmp_path, pose):
    keys, doc, today = _cfg(tmp_path, pose)
    assert keys == today
    assert set(doc) == {"model", "pipe", "opt"}
    assert not any("pose" in k for k in keys)


def test_cfg_args_with_pose_refine_records_the_pose_settings(tmp_path):
    keys, doc, today = _cfg(tmp_path, trainer.PoseParams(pose_refine=True))
    assert keys == today | set(asdict(trainer.PoseParams()))
    assert doc["pose"] == asdict(trainer.PoseParams(pose_refine=True))


def test_pose_refine_with_sharding_is_refused_before_any_process_group(tmp_path, monkeypatch, capsys):
    import torch.distributed as dist
    monkeypatch.setenv("WORLD_SIZE", "2")
    out = tmp_path / "out"
    with pytest.raises(SystemExit) as e:
        trainer.main(["-s", str(tmp_path), "-m", str(out), "--pose_refine"])
    assert e.value.code != 0
    assert "--pose_refine" in capsys.readouterr().err
    assert not dist.is_initialized()
    assert not out.exists()
