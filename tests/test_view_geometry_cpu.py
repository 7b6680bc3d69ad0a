"""Per-view scan geometry without a GPU: the frame keys' rescaling, the cameras of a per-view scene against those of a
scanner holding each view's values (bit for bit), today's cameras without the keys or the flag, the offOrigin
convention, the helical generator's ramp and test arc, and the refusals of the CLIs, the Python operators and the
C ABI before any CUDA work."""
import ctypes
import json
import math

import numpy as np
import pytest
import torch

import view_geometry_oracle as vgo
from r2_gaussian_b200 import dataset, scene

CAMERA_FIELDS = ("world_view_transform", "full_proj_transform", "camera_center", "projection_matrix")

OVERRIDES = [
    {},
    {"DSO": 9.5},
    {"DSD": 14.6, "offDetector": [0.35, -0.2]},
    {"offOrigin": [0.1, -0.2, 0.7]},
    {"DSO": 10.4, "DSD": 13.1, "offOrigin": [0.0, 0.0, -1.3], "offDetector": [-0.5, 0.0]},
]


def _scene(tmp_path, name="s", overrides=OVERRIDES, scanner=None):
    frames = list(zip(vgo.ANGLES, overrides))
    return vgo.write_scene(str(tmp_path / name), scanner or vgo.file_scanner(), frames)


def _same_camera(a, b):
    for f in CAMERA_FIELDS:
        ta, tb = getattr(a, f), getattr(b, f)
        assert ta.dtype == tb.dtype and torch.equal(ta.view(torch.int32), tb.view(torch.int32)), f
    assert a.FoVx == b.FoVx and a.FoVy == b.FoVy


def test_frame_keys_are_rescaled_like_the_scanner(tmp_path):
    info = dataset.read_blender(_scene(tmp_path), eval=False, use_view_geometry=True)
    scale = info.scene_scale
    assert scale == 0.5
    for cam, over in zip(info.train_cameras, OVERRIDES):
        assert set(cam.view_geometry) == set(over)
        for k, v in over.items():
            want = (np.asarray(v, np.float64) * scale).tolist()
            assert cam.view_geometry[k] == want, k
        # the camera's scanner is the rescaled scanner with the frame's rescaled values
        for k in ("DSO", "DSD", "offDetector"):
            assert cam.scanner_cfg[k] == cam.view_geometry.get(k, info.scanner_cfg[k])
    assert info.scanner_cfg["DSO"] == 5.0 and info.scanner_cfg["offOrigin"] == [0.0, 0.0, 0.0]


def test_each_camera_is_the_camera_of_a_scanner_holding_its_values(tmp_path):
    per_view = dataset.Scene(_scene(tmp_path), eval=False, shuffle=False, device="cpu", use_view_geometry=True)
    geometry = [c.view_geometry for c in dataset.read_blender(str(tmp_path / "s"), True, True).train_cameras]
    assert per_view.use_offDetector and per_view.use_view_geometry
    for i, (angle, over) in enumerate(zip(vgo.ANGLES, OVERRIDES)):
        if "offOrigin" in over:
            continue                       # a scanner file's offOrigin moves the grid: see the convention test
        sc = vgo.file_scanner()
        sc.update({k: v for k, v in over.items()})
        one = vgo.write_scene(str(tmp_path / f"one{i}"), sc, [(angle, {})])
        ref = dataset.Scene(one, eval=False, shuffle=False, device="cpu", use_offDetector=True)
        _same_camera(per_view.getTrainCameras()[i], ref.getTrainCameras()[0])
        # and the View of scene.make_view for the same scanner dict
        v = scene.make_view(scene.view_scanner(per_view.scanner_cfg, geometry[i]), angle, True)
        ref_v = scene.make_view(ref.scanner_cfg, angle, True)
        assert np.array_equal(v.viewmatrix.view(np.int32), ref_v.viewmatrix.view(np.int32))
        assert np.array_equal(v.projmatrix.view(np.int32), ref_v.projmatrix.view(np.int32))
        assert (v.tanfovx, v.tanfovy, v.FoVx, v.FoVy) == (ref_v.tanfovx, ref_v.tanfovy, ref_v.FoVx, ref_v.FoVy)


def test_without_keys_or_without_the_flag_the_cameras_are_todays(tmp_path):
    plain = _scene(tmp_path, "plain", [{}] * len(vgo.ANGLES))
    today = dataset.Scene(plain, eval=False, shuffle=False, device="cpu")
    flagged = dataset.Scene(plain, eval=False, shuffle=False, device="cpu", use_view_geometry=True)
    for a, b in zip(today.getTrainCameras(), flagged.getTrainCameras()):
        _same_camera(a, b)
    with pytest.warns(UserWarning, match="--use_view_geometry"):
        keyed = dataset.Scene(_scene(tmp_path), eval=False, shuffle=False, device="cpu")
    for a, b in zip(today.getTrainCameras(), keyed.getTrainCameras()):
        _same_camera(a, b)
    # the camera_pose translation of a zero offset changes no bit
    sc = scene.cone_beam_scanner(16, 8)
    same = scene.view_scanner(sc, {"offOrigin": list(sc["offOrigin"])})
    for a in vgo.ANGLES:
        v0, v1 = scene.make_view(sc, a), scene.make_view(same, a)
        assert np.array_equal(v0.viewmatrix, v1.viewmatrix) and np.array_equal(v0.projmatrix, v1.projmatrix)


def _pixel(view: scene.View, p) -> np.ndarray:
    """Pixel coordinates of world point p through the view's full projection (row-vector convention)."""
    h = np.append(np.asarray(p, np.float64), 1.0) @ view.projmatrix.astype(np.float64)
    ndc = h[:2] / h[3]
    return np.array([(ndc[0] + 1.0) * view.image_width / 2.0, (ndc[1] + 1.0) * view.image_height / 2.0])


def test_offorigin_is_where_the_volume_sits_during_the_view():
    sc = scene.cone_beam_scanner(64, 16)
    sc["offOrigin"] = [0.05, -0.1, 0.2]
    pos = [0.3, -0.25, 0.9]
    per_view = scene.view_scanner(sc, {"offOrigin": pos})
    rng = np.random.RandomState(0)
    for a in vgo.ANGLES:
        nominal, moved = scene.make_view(sc, a), scene.make_view(per_view, a)
        for r in rng.uniform(-0.6, 0.6, (6, 3)):
            # the grid point offOrigin + r, seen in view v, lands where the nominal view sees the volume's point at
            # offOrigin_v + r (where the object sits during view v)
            got = _pixel(moved, np.asarray(sc["offOrigin"]) + r)
            want = _pixel(nominal, np.asarray(pos) + r)
            assert np.allclose(got, want, atol=2e-3), (a, r, got, want)
        c = np.asarray(nominal.campos, np.float64) + np.asarray(sc["offOrigin"]) - np.asarray(pos)
        assert np.allclose(moved.campos, c, atol=1e-5)


def test_helical_generator_ramp_and_test_arc():
    from r2_gaussian_b200.generate_data import draw_arc_angles, helical_offsets, train_angles

    cfg = dict(vgo.file_scanner(), totalAngle=720.0, startAngle=30.0, offOrigin=[0.1, 0.2, -0.3])
    ang = train_angles(cfg, 16)
    rows = helical_offsets(cfg, ang, 2.0)
    z = np.array([r["offOrigin"][2] for r in rows])
    frac = np.arange(16) / 16.0 - 0.5
    assert np.allclose(z, -0.3 + 2.0 * frac, rtol=0, atol=1e-12)
    assert all(r["offOrigin"][:2] == [0.1, 0.2] for r in rows)
    test = draw_arc_angles(cfg, 200, np.random.RandomState(0))
    assert np.all(np.diff(test) >= 0)
    lo, hi = math.radians(30.0), math.radians(30.0 + 720.0)
    assert test.min() >= lo and test.max() < hi and test.max() > lo + 2.5 * math.pi   # beyond one turn
    tz = np.array([r["offOrigin"][2] for r in helical_offsets(cfg, test, 2.0)])
    assert tz.min() >= -0.3 - 1.0 and tz.max() < -0.3 + 1.0


def _generate(tmp_path, *extra):
    from r2_gaussian_b200 import generate_data

    import yaml
    np.save(tmp_path / "v.npy", np.zeros((4, 4, 4), np.float32))
    with open(tmp_path / "sc.yml", "w") as f:
        yaml.safe_dump(vgo.file_scanner(), f)
    return generate_data.main(["--vol", str(tmp_path / "v.npy"), "--scanner", str(tmp_path / "sc.yml"), "--output",
                               str(tmp_path / "out"), "--n_train", "3", "--n_test", "2", *extra])


def test_generate_data_refuses_bad_override_files(tmp_path):
    bad = [({"train": [{}] * 2, "test": [{}] * 2}, "train holds 2 entries, --n_train is 3"),
           ({"train": [{}] * 3, "test": [{}] * 3}, "test holds 3 entries, --n_test is 2"),
           ({"train": [{}, {"dso": 1.0}, {}], "test": [{}] * 2}, r"train\[1\] has unknown keys \['dso'\]"),
           ({"train": [{}] * 3}, "keys 'train' and 'test'"),
           ({"train": [{}, {}, {"offOrigin": [0, 1]}], "test": [{}] * 2}, "offOrigin must hold 3 numbers")]
    for table, msg in bad:
        with open(tmp_path / "g.json", "w") as f:
            json.dump(table, f)
        with pytest.raises(SystemExit, match=msg):
            _generate(tmp_path, "--view_geometry", str(tmp_path / "g.json"))
    with pytest.raises(SystemExit, match="cannot be combined"):
        _generate(tmp_path, "--view_geometry", str(tmp_path / "g.json"), "--helical_travel", "1")


def test_command_lines_refuse_fixed_circle_flags(tmp_path):
    from r2_gaussian_b200 import initialize_pcd, recon, trainer

    src = _scene(tmp_path)
    for flags, msg in ((["--estimate_offDetector"], "--estimate_offDetector cannot be combined"),
                       (["--half_fan", "--use_offDetector"], "--half_fan cannot be combined"),
                       (["--short_scan"], "--short_scan cannot be combined")):
        with pytest.raises(SystemExit, match=msg):
            recon.main(["-s", src, "-m", str(tmp_path / "o"), "--methods", "fdk", "--use_view_geometry", *flags])
        with pytest.raises(SystemExit, match=msg):
            initialize_pcd.main(["--data", src, "--recon_method", "fdk", "--use_view_geometry", *flags])
    with pytest.raises(SystemExit, match="--recon_method cgls"):
        initialize_pcd.main(["--data", src, "--recon_method", "fdk", "--use_view_geometry"])
    with pytest.raises(SystemExit):
        trainer.parse_args(["-s", src, "--use_view_geometry", "--estimate_offDetector"])
    with pytest.raises(SystemExit):
        trainer.parse_args(["-s", src, "--use_view_geometry", "--batch_size", "2"])   # the DSD differ
    assert "DSD varies" in trainer.view_geometry_refusal(True, False, 1, 2, src)
    assert trainer.view_geometry_refusal(True, False, 1, 2, _scene(tmp_path, "flat", [{"offOrigin": [0, 0, 1]}] * 5)) \
        is None
    assert "sharding" in trainer.view_geometry_refusal(True, False, 2, 1, src)
    for flag in ("--pose_refine", "--detector_offset_refine"):
        assert trainer.parse_args(["-s", src, "--use_view_geometry", flag])[0].use_view_geometry


def test_python_operators_refuse_before_any_cuda_work():
    from r2_gaussian_b200 import fdk, projector

    sc = scene.cone_beam_scanner(16, 8)
    angles = np.linspace(0, 2 * math.pi, 6)[:-1]
    geo = vgo.helix(5, sc, 1.0)
    with pytest.raises(ValueError, match="cgls, sart, fista_tv or cp_tv"):
        fdk.fdk(torch.zeros(5, 16, 16), angles, sc, view_geometry=geo)
    for kw in ({"short_scan": True}, {"half_fan": True, "use_offDetector": True}):
        with pytest.raises(ValueError, match="cannot be combined with view_geometry"):
            fdk.fdk(torch.zeros(5, 16, 16), angles, sc, view_geometry=[{}] * 5, **kw)
    with pytest.raises(ValueError, match="4 entries for 5 angles"):
        projector.view_table(angles, sc, [{}] * 4)
    with pytest.raises(ValueError, match="finite"):
        projector.view_table(angles, sc, [{}] * 4 + [{"DSO": float("nan")}])
    with pytest.raises(ValueError, match="DSO > 0"):
        projector.view_table(angles, sc, [{}] * 4 + [{"DSO": -1.0}])
    views, table = projector.view_table(angles, sc, vgo.jittered(5, sc))
    assert table.shape == (5, 5) and table.dtype == np.float64 and table.flags.c_contiguous
    for v, row, g in zip(views, table, vgo.jittered(5, sc)):
        c = scene.view_scanner(sc, g)
        assert tuple(row) == (v.tanfovx, v.tanfovy, *scene.detector_shift(c), c["DSO"])


def _table(rows):
    return np.ascontiguousarray(np.asarray(rows, np.float64).reshape(-1, 5))


def test_abi_refuses_bad_tables_before_any_cuda_call():
    from r2_gaussian_b200 import _lib

    lib = _lib.load()
    d = ctypes.c_void_p(16)
    good = [0.3, 0.3, 0.5, -0.25, 5.0]

    def project(t, dev=d, mode=1):
        return lib.r2x_volume_project_views(None, 4, 4, 4, d, 2.0, 2.0, 2.0, 0.0, 0.0, 0.0, len(t), 8, 8, d, mode, 0.01,
                                            dev, None if t is None else t.ctypes.data, d)

    def back(t, dev=d, mode=1):
        return lib.r2x_volume_backproject_views(None, len(t), 8, 8, d, d, d, mode, 4, 4, 4, 2.0, 2.0, 2.0, 0.0, 0.0, 0.0,
                                                0.01, dev, t.ctypes.data, d, None, d, 1 << 30)

    def fdk_(t, weighting=0, dev=d, mode=1):
        return lib.r2x_fdk_views(None, len(t), 8, 8, d, d, d, mode, weighting, 4, 4, 4, 2.0, 2.0, 2.0, 0.0, 0.0, 0.0,
                                 dev, t.ctypes.data, d, d, 1 << 30)

    ok = _table([good, good])
    for call, who in ((project, "r2x_volume_project_views"), (back, "r2x_volume_backproject_views"),
                      (fdk_, "r2x_fdk_views")):
        assert call(ok, dev=None) != 0
        assert lib.r2x_last_error().decode() == f"{who}: bad pointer (view_geometry NULL)"
        for col, val, why in ((0, float("nan"), "values must be finite"), (3, float("inf"), "values must be finite"),
                              (2, 1e300, "values must be finite"), (4, 0.0, "cone beam needs dso > 0"),
                              (4, -2.0, "cone beam needs dso > 0"), (1, 0.0, "tan_fov must be > 0"),
                              (0, 1e-60, "tan_fov must be > 0")):
            t = _table([good, good])
            t[1, col] = val
            assert call(t) != 0, (who, col, val)
            assert lib.r2x_last_error().decode() == f"{who}: bad view_geometry (view 1: {why})", (col, val)
    # parallel beam reads no DSO
    par = _table([[1.0, 1.0, 0.0, 0.0, 0.0]])
    assert project(par, dev=None, mode=0) != 0 and b"view_geometry NULL" in lib.r2x_last_error()
    for w in (1, 2, 0x101, 0x402):
        assert fdk_(ok, weighting=w) != 0
        assert b"r2x_fdk_views: bad weighting (Parker and half-fan" in lib.r2x_last_error(), hex(w)
    # a valid table reaches the scalar entries' own checks (here: too little scratch), still before any CUDA work
    assert lib.r2x_fdk_views(None, 2, 8, 8, d, d, d, 1, 0, 4, 4, 4, 2.0, 2.0, 2.0, 0.0, 0.0, 0.0, d, ok.ctypes.data, d,
                             d, 16) != 0
    assert lib.r2x_last_error().decode() == "r2x_fdk: bad scratch (too small)"
    assert lib.r2x_volume_project_views(None, 4, 4, 4, d, 2.0, 2.0, 2.0, 0.0, 0.0, 0.0, 2, 8, 8, d, 1, 0.0, d,
                                        ok.ctypes.data, d) != 0
    assert lib.r2x_last_error().decode() == "r2x_volume_project: bad step (must be finite and > 0)"
