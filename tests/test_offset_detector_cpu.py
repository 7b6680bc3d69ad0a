"""The scanner's detector offset (offDetector) without a GPU: the convention of `scene.detector_shift`, the offset
cameras of `scene.make_view` / `dataset.Camera` against the formula and bit for bit today's without the switch, the
float64 oracle's integer-shift identities, the half-fan weights, and every refusal of the Python surface and the command
lines before any CUDA work."""
import math

import numpy as np
import pytest
import yaml

import fdk_cases as fc
import offset_detector_oracle as oo
from oracle import projector_oracle as po
from r2_gaussian_b200 import scene
from r2_gaussian_b200.dataset import Camera, _camera_info


def _cone(det=(12, 16), vox=10):
    sc = fc.scanner("cone", 8, vox)
    sc["nDetector"], sc["sDetector"] = list(det), [3.0, 4.0]
    return sc


def _with_off(sc, u, v):
    return dict(sc, offDetector=[u, v])


def _du_dv(sc):
    return sc["sDetector"][1] / sc["nDetector"][1], sc["sDetector"][0] / sc["nDetector"][0]


# ---- convention ------------------------------------------------------------------------------------------------------

def test_detector_shift_is_the_offset_over_the_pixel_pitch():
    sc = _cone((12, 16))                                                  # [v, u]: 12 rows, 16 columns
    du, dv = _du_dv(sc)
    assert scene.detector_shift(sc) == (0.0, 0.0)
    assert scene.detector_shift({k: v for k, v in sc.items() if k != "offDetector"}) == (0.0, 0.0)
    t_u, t_v = scene.detector_shift(_with_off(sc, 2.4 * du, -1.7 * dv))   # offDetector is [u, v]
    assert t_u == pytest.approx(2.4, rel=1e-12) and t_v == pytest.approx(-1.7, rel=1e-12)


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_make_view_is_bit_identical_without_the_switch_or_the_offset(mode):
    sc = fc.scanner(mode, 16, 8)
    off = _with_off(sc, 0.3, -0.2)
    for a in (0.0, 0.7, 4.1):
        ref = scene.make_view(sc, a)
        for v in (scene.make_view(off, a), scene.make_view(sc, a, use_offDetector=True)):
            assert v.projmatrix.tobytes() == ref.projmatrix.tobytes()
            assert v.viewmatrix.tobytes() == ref.viewmatrix.tobytes()
            assert v.campos.tobytes() == ref.campos.tobytes()


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_make_view_carries_the_offset_in_the_projection_matrix(mode):
    sc = fc.scanner(mode, 8, 8)
    sc["nDetector"] = [12, 16]
    du, dv = _du_dv(sc)
    t_u, t_v = 2.4, -1.7
    off = _with_off(sc, t_u * du, t_v * dv)
    H, W = 12, 16
    P = scene.projection_matrix(*(scene.make_view(sc, 0.0).FoVx, scene.make_view(sc, 0.0).FoVy), 1 if mode == "cone" else 0)
    Q = scene.shifted_projection_matrix(P, t_u, t_v, W, H)
    col = 2 if mode == "cone" else 3                                      # the w row is (0,0,1,0) or (0,0,0,1)
    changed = np.argwhere(Q != P)
    assert sorted(map(tuple, changed)) == [(0, col), (1, col)]
    assert Q[0, col] == np.float32(P[0, col] - 2.0 * t_u / W)
    assert Q[1, col] == np.float32(P[1, col] + 2.0 * t_v / H)
    rng = np.random.RandomState(3)
    for a in (0.0, 1.1, 3.9):
        c, s = scene.make_view(sc, a), scene.make_view(off, a, use_offDetector=True)
        assert s.viewmatrix.tobytes() == c.viewmatrix.tobytes()
        assert s.projmatrix.tobytes() == (c.viewmatrix @ Q.T).astype(np.float32).tobytes()
        # a point's pixel moves by -t_u columns and +t_v rows: pixel (r, c) sees the centred (r - t_v, c + t_u)
        X = np.concatenate([rng.uniform(-0.8, 0.8, (20, 3)), np.ones((20, 1))], 1)
        def pix(m):
            h = X @ m.astype(np.float64)
            return ((h[:, 0] / h[:, 3] + 1.0) * W - 1.0) / 2.0, ((h[:, 1] / h[:, 3] + 1.0) * H - 1.0) / 2.0
        (cx, cy), (sx, sy) = pix(c.projmatrix), pix(s.projmatrix)
        np.testing.assert_allclose(sx, cx - t_u, atol=1e-4)
        np.testing.assert_allclose(sy, cy + t_v, atol=1e-4)


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_camera_matches_make_view_and_is_bit_identical_without_the_switch(mode):
    sc = fc.scanner(mode, 16, 8)
    du, dv = _du_dv(sc)
    off = _with_off(sc, 1.5 * du, 0.75 * dv)
    img = np.zeros((16, 16), np.float32)
    for a in (0.0, 2.3):
        ref = Camera(_camera_info(0, a, img, "x", None, sc), device="cpu")
        for cam in (Camera(_camera_info(0, a, img, "x", None, off), device="cpu"),
                    Camera(_camera_info(0, a, img, "x", None, sc), device="cpu", use_offDetector=True)):
            for k in ("projection_matrix", "full_proj_transform", "world_view_transform", "camera_center"):
                assert getattr(cam, k).numpy().tobytes() == getattr(ref, k).numpy().tobytes(), k
        cam = Camera(_camera_info(0, a, img, "x", None, off), device="cpu", use_offDetector=True)
        v = scene.make_view(off, a, use_offDetector=True)
        assert cam.full_proj_transform.numpy().tobytes() == v.projmatrix.tobytes()
        P = scene.projection_matrix(v.FoVx, v.FoVy, v.mode)
        want = scene.shifted_projection_matrix(P, 1.5, 0.75, 16, 16).T
        np.testing.assert_array_equal(cam.projection_matrix.numpy(), want)


# ---- the oracle's convention ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_oracle_integer_shifts_move_the_projection(mode):
    """offDetector = [k dDetector_u, 0] gives the centred projection moved k columns towards smaller index;
    [0, k dDetector_v] moves it k rows towards larger index."""
    sc = fc.scanner(mode, 8, 10)
    sc["nDetector"] = [12, 16]
    du, dv = _du_dv(sc)
    vol = np.random.RandomState(0).uniform(0.0, 1.0, (10, 10, 10))
    angles = [0.3, 2.0]
    base = po.project_scene(vol, angles, sc)
    assert np.abs(oo.project_scene(vol, angles, sc) - base).max() == 0.0
    k = 3
    got = oo.project_scene(vol, angles, _with_off(sc, k * du, 0.0))
    np.testing.assert_allclose(got[..., :-k], base[..., k:], rtol=0, atol=1e-9 * base.max())
    got = oo.project_scene(vol, angles, _with_off(sc, 0.0, k * dv))
    np.testing.assert_allclose(got[:, k:, :], base[:, :-k, :], rtol=0, atol=1e-9 * base.max())


def test_oracle_backprojection_is_the_transpose():
    sc = _with_off(_cone((9, 11), 7), 0.6, -0.3)
    rng = np.random.RandomState(1)
    x, y = rng.rand(7, 7, 7), rng.rand(2, 9, 11)
    ax, aty = oo.project_scene(x, [0.4, 2.5], sc), oo.backproject_scene(y, [0.4, 2.5], sc)
    assert float((ax * y).sum()) == pytest.approx(float((x * aty).sum()), rel=1e-12)


# ---- half-fan weights ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("t_u", [5.3, -5.3, 0.4, -31.0])
def test_half_fan_weights(t_u):
    from r2_gaussian_b200.fdk import half_fan_weight

    W, fan = 64, 0.4
    delta = (1.0 - 2.0 * abs(t_u) / W) * fan
    a = np.linspace(-delta, delta, 401)
    w = half_fan_weight(a, t_u, W, fan)
    np.testing.assert_allclose(w + half_fan_weight(-a, t_u, W, fan), 2.0, rtol=0, atol=1e-12)
    np.testing.assert_allclose(w, oo.half_fan_weight(a, t_u, W, fan), rtol=0, atol=1e-12)
    wide = math.copysign(1.0, t_u) * np.linspace(delta, fan * 1.6, 50)
    np.testing.assert_array_equal(half_fan_weight(wide, t_u, W, fan), 2.0)
    np.testing.assert_array_equal(oo.half_fan_weight(wide, t_u, W, fan), 2.0)
    s = math.copysign(1.0, t_u)
    for edge, val in ((s * delta, 2.0), (-s * delta, 0.0)):                 # continuous at +-delta
        for eps in (1e-9, -1e-9):
            assert float(oo.half_fan_weight(edge + eps, t_u, W, fan)) == pytest.approx(val, abs=1e-6)
    # every column of the offset detector lies in the overlap or on the wide side
    ndx = oo.ndc(8, W, t_u)[0] * fan
    assert (s * ndx > -delta).all()


def test_half_fan_refusals():
    import torch

    from r2_gaussian_b200.fdk import check_half_fan_shift, fdk, scan_arc

    for t_u in (0.0, 32.0, -32.0, 40.0):
        with pytest.raises(ValueError, match="half fan"):
            check_half_fan_shift(t_u, 64)
    assert scan_arc(fc.full_scan(36)) == pytest.approx(2 * math.pi)
    assert scan_arc(np.linspace(0.0, math.pi, 30)) < 1.1 * math.pi
    sc = fc.scanner("cone", 16, 8)
    du, dv = _du_dv(sc)
    off = _with_off(sc, 3 * du, 0.5 * dv)
    projs = torch.zeros(36, 16, 16)                                        # on the CPU: every refusal comes first
    full = fc.full_scan(36)
    cases = [(dict(half_fan=True), off, full, "use_offDetector"),
             (dict(half_fan=True, short_scan=True, use_offDetector=True), off, full, "cannot be combined"),
             (dict(half_fan=True, use_offDetector=True), sc, full, "centred"),
             (dict(half_fan=True, use_offDetector=True), _with_off(sc, 8 * du, 0.0), full, "strictly inside"),
             (dict(half_fan=True, use_offDetector=True), off, np.linspace(0.0, 1.5 * math.pi, 36), "full circle"),
             (dict(short_scan=True, use_offDetector=True), off, np.linspace(0.0, 1.5 * math.pi, 36), "vertical offset only")]
    for kw, cfg, angles, match in cases:
        with pytest.raises(ValueError, match=match):
            fdk(projs, angles, cfg, **kw)
    with pytest.warns(UserWarning, match="ignored"), pytest.raises(RuntimeError, match="CUDA"):
        fdk(projs, full, off)


# ---- Python surface and command lines --------------------------------------------------------------------------------

def test_projector_pair_refuses_the_offset_without_the_switch():
    import torch

    from r2_gaussian_b200.projector import backproject, project

    sc = _with_off(fc.scanner("cone", 8, 4), 0.1, 0.0)
    with pytest.raises(ValueError, match="use_offDetector"):
        project(torch.zeros(4, 4, 4), [0.0], sc)
    with pytest.raises(ValueError, match="use_offDetector"):
        backproject(torch.zeros(1, 8, 8), [0.0], sc)
    with pytest.raises(RuntimeError, match="CUDA"):                       # accepted with it; then it needs the GPU
        project(torch.zeros(4, 4, 4), [0.0], sc, use_offDetector=True)
    with pytest.raises(ValueError, match="finite"):
        project(torch.zeros(4, 4, 4), [0.0], _with_off(sc, float("nan"), 0.0), use_offDetector=True)


def test_recon_volume_refuses_half_fan_for_iterative_methods():
    import torch

    from r2_gaussian_b200.recon import recon_volume

    with pytest.raises(ValueError, match="half_fan applies to fdk only"):
        recon_volume(torch.zeros(2, 8, 8), [0.0, 1.0], fc.scanner("cone", 8, 4), "cgls", half_fan=True,
                     use_offDetector=True)


def _offset_scene(tmp_path):
    from r2_gaussian_b200.dataset import write_blender

    sc = fc.scanner("cone", 16, 8)
    sc.update({"filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0, "noise": False,
               "offDetector": [0.5, 0.0]})
    sc.pop("dDetector"), sc.pop("dVoxel")
    frames = [(a, np.ones((16, 16), np.float32)) for a in fc.full_scan(10)]
    path = str(tmp_path / "case")
    write_blender(path, sc, frames, frames[:2], np.zeros((8, 8, 8), np.float32))
    return path, sc


@pytest.mark.parametrize("argv,match", [
    (["--methods", "cgls", "--half_fan", "--use_offDetector"], "--half_fan applies to the fdk method"),
    (["--methods", "fdk", "--half_fan"], "--half_fan needs --use_offDetector"),
    (["--methods", "fdk", "--half_fan", "--use_offDetector", "--short_scan"], "cannot be combined"),
])
def test_recon_cli_refusals(tmp_path, argv, match):
    from r2_gaussian_b200 import recon

    path, _ = _offset_scene(tmp_path)
    with pytest.raises(SystemExit, match=match):
        recon.main(["-s", path, "-m", str(tmp_path / "out"), *argv])


@pytest.mark.parametrize("argv,match", [
    (["--recon_method", "cgls", "--half_fan", "--use_offDetector"], "--half_fan applies to --recon_method fdk only"),
    (["--recon_method", "fdk", "--half_fan"], "--half_fan needs --use_offDetector"),
    (["--recon_method", "fdk", "--half_fan", "--use_offDetector", "--short_scan"], "cannot be combined"),
    (["--recon_method", "random", "--use_offDetector"], "--use_offDetector applies to --recon_method fdk"),
    (["--recon_method", "volume", "--use_offDetector"], "--use_offDetector applies to --recon_method fdk"),
])
def test_initialize_pcd_cli_refusals(tmp_path, argv, match):
    import os

    from r2_gaussian_b200 import initialize_pcd

    path, _ = _offset_scene(tmp_path)
    out = str(tmp_path / "init.npy")
    with pytest.raises(SystemExit, match=match):
        initialize_pcd.main(["--data", path, "--output", out, *argv])
    assert not os.path.exists(out)


def test_generate_data_refuses_an_offset_scanner_without_the_switch(tmp_path):
    from r2_gaussian_b200 import generate_data

    _, sc = _offset_scene(tmp_path)
    yml = tmp_path / "off.yml"
    yml.write_text(yaml.safe_dump(sc))
    np.save(tmp_path / "vol.npy", np.zeros((8, 8, 8), np.float32))
    with pytest.raises(SystemExit, match="--use_offDetector"):
        generate_data.main(["--vol", str(tmp_path / "vol.npy"), "--scanner", str(yml), "--output", str(tmp_path / "o")])
    assert not (tmp_path / "o").exists()


def test_trainer_switch_and_the_total_offset_report(tmp_path):
    import types

    import torch

    from r2_gaussian_b200 import trainer
    from r2_gaussian_b200.detector import DetectorOffset

    a = trainer.parse_args(["-s", "x", "--use_offDetector", "--detector_offset_refine"])[0]
    assert a.use_offDetector and a.detector_params.detector_offset_refine
    assert not trainer.parse_args(["-s", "x"])[0].use_offDetector
    det = DetectorOffset("cpu")
    with torch.no_grad():
        det.offset.fill_(2.5)
    cfg = {"nDetector": [64, 128], "sDetector": [1.0, 2.0], "offDetector": [0.1, 0.05]}   # scaled by scene_scale 0.5
    for on in (False, True):
        sc = types.SimpleNamespace(model_path=str(tmp_path), scanner_cfg=cfg, scene_scale=0.5, use_offDetector=on)
        (tmp_path / "point_cloud" / "iteration_3").mkdir(parents=True, exist_ok=True)
        trainer.save_detector_offset(sc, det, 3)
        doc = yaml.safe_load((tmp_path / "point_cloud" / "iteration_3" / "detector_offset.yml").read_text())
        assert doc["offset_px"] == 2.5
        if on:   # file value - s dDetector_u, in the file's units
            assert doc["offDetector_u"] == pytest.approx((0.1 - 2.5 * 2.0 / 128) / 0.5)
        else:
            assert "offDetector_u" not in doc
