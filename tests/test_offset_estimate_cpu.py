"""The detector-offset estimate without a GPU: the float64 oracle (tests/offset_estimate_oracle.py) against brute force
and the closed-form blob projections, the oracle's search on blob phantoms, the host pair table of
`detector.estimate_offset`, its refusals, and the `--estimate_offDetector` flags of initialize_pcd, recon and trainer."""
import argparse
import math
import types

import numpy as np
import pytest

import offset_estimate_oracle as oo
from r2_gaussian_b200 import detector, scene


def _scanner(mode, n=64):
    return scene.cone_beam_scanner(n, 32) if mode == "cone" else scene.parallel_beam_scanner(n, 32)


def _angles(kind, n=24):
    if kind == "uniform":
        return np.linspace(0, 2 * np.pi, n + 1)[:-1] + 0.3
    if kind == "uneven":
        return np.sort(np.random.RandomState(3).uniform(0, 2 * np.pi, n))
    # a short scan: 180 degrees plus the fan angle (2 atan(2 / 7)) plus 10 degrees, with both ends in
    return np.linspace(0, np.pi + 2 * math.atan(2 / 7) + math.radians(10), n)


# ---- the oracle ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["cone", "parallel"])
@pytest.mark.parametrize("kind", ["uniform", "uneven", "short"])
def test_pair_table_is_the_brute_force_enumeration(mode, kind):
    sc = _scanner(mode)
    ang = _angles(kind, 24 if kind != "uneven" else 31)
    tol = 1e-4 if kind != "uneven" else 0.05
    views, dbeta = detector.conjugate_pairs(ang, sc, 31.5 + 17, tol)
    brute = oo.pairs(ang, sc, 31.5 + 17, tol)
    assert [tuple(v) for v in views.tolist()] == [(i, j) for i, j, _ in brute]
    assert np.allclose(dbeta, [d for *_, d in brute], rtol=0, atol=1e-15)
    if mode == "cone":
        assert len(brute) > 0


def test_partner_rays_carry_the_same_line_integral():
    """P(beta, gamma) = P(beta + pi - 2 gamma, -gamma) in the mid-plane (cone) and P(beta, u, v) = P(beta + pi, -u, v)
    (parallel) on the closed-form blob projections, to 1e-9 relative."""
    bl = oo.blobs(9, seed=1, radius=0.5)
    rng = np.random.RandomState(0)
    DSD, DSO = 7.0, 5.0
    for _ in range(200):
        beta, gamma = rng.uniform(0, 2 * np.pi), rng.uniform(-0.27, 0.27)
        b2, g2 = oo.partner(beta, gamma)
        a = oo.line_integral(bl, beta, DSD * math.tan(gamma), 0.0, "cone", DSD, DSO)
        b = oo.line_integral(bl, b2, DSD * math.tan(g2), 0.0, "cone", DSD, DSO)
        assert abs(a - b) <= 1e-9 * max(abs(a), 1e-12), (beta, gamma, a, b)
        u, v = rng.uniform(-1, 1), rng.uniform(-1, 1)
        a = oo.line_integral(bl, beta, u, v, "parallel", DSD, DSO)
        b = oo.line_integral(bl, beta + np.pi, -u, v, "parallel", DSD, DSO)
        assert abs(a - b) <= 1e-9 * max(abs(a), 1e-12)
    # the identity's sign: with + 2 gamma the rays differ
    a = oo.line_integral(bl, 0.4, DSD * math.tan(0.2), 0.0, "cone", DSD, DSO)
    b = oo.line_integral(bl, 0.4 + np.pi + 0.4, DSD * math.tan(-0.2), 0.0, "cone", DSD, DSO)
    assert abs(a - b) > 1e-3 * abs(a)


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_oracle_geometry_is_make_view_s(mode):
    """The oracle's detector coordinate of a point is the column make_view's projection matrix puts it in."""
    sc = _scanner(mode)
    W = sc["nDetector"][1]
    du = sc["sDetector"][1] / W
    rng = np.random.RandomState(2)
    for beta in (0.0, 0.7, 2.9, 4.4):
        view = scene.make_view(sc, beta)
        for p in rng.uniform(-0.6, 0.6, (5, 3)):
            h = np.append(p, 1.0) @ view.projmatrix.astype(np.float64)      # row vector times the transposed matrix
            pix = ((h[0] / h[3] + 1.0) * W - 1.0) / 2.0
            u = oo.project_point(p, beta, mode, sc["DSD"], sc["DSO"])
            assert abs(u / du + (W - 1) / 2 - pix) < 1e-3, (beta, p)


SHIFTS = [-3.7, -0.4, 0.0, 1.25, 2.4]
# |oracle estimate - truth| in pixels on the 64^2 blob phantom below, measured on the CPU: largest 0.0141 px (cone, 24
# views, 1.25 px); every parallel-beam case within 0.0014 px.
ORACLE_TOL = 0.03


@pytest.mark.parametrize("n", [24, 50])
@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_oracle_recovers_sub_pixel_shifts_on_blob_phantoms(mode, n):
    """Measured errors (px) of the oracle estimate, shifts -3.7, -0.4, 0, 1.25, 2.4 and then the quarter-width half-fan
    scan (file offset t_u = -16 px, 1.25 px on top):
      cone 24:     +0.0112 -0.0054 +0.0000 +0.0141 +0.0055 -0.0010
      cone 50:     -0.0050 +0.0011 -0.0009 -0.0044 -0.0031 -0.0044
      parallel 24: +0.0010 -0.0006 -0.0000 +0.0011 +0.0006 +0.0014
      parallel 50: +0.0010 -0.0006 -0.0000 +0.0011 +0.0006 +0.0014
    The bar is ORACLE_TOL = 0.03 px, about twice the largest."""
    sc = _scanner(mode)
    bl = oo.blobs(9, seed=0, radius=0.5)
    ang = np.linspace(0, 2 * np.pi, n + 1)[:-1] + 0.3
    for s in SHIFTS:
        est, _ = oo.estimate(oo.project(bl, ang, sc, sigma=s), ang, sc)
        assert abs(est - s) <= ORACLE_TOL, (s, est)
    t_u, s = -16.0, 1.25
    est, _ = oo.estimate(oo.project(bl, ang, sc, sigma=s - t_u), ang, sc, t_u=t_u)
    assert abs(est - s) <= ORACLE_TOL, (s, est)


# ---- refusals --------------------------------------------------------------------------------------------------------

def _inputs(mode="cone", n=24, N=None, H=64, W=64, dtype=None):
    import torch
    sc = _scanner(mode, W)
    sc["nDetector"] = [H, W]
    ang = np.linspace(0, 2 * np.pi, n + 1)[:-1]
    return torch.zeros((N or n, H, W), dtype=dtype or torch.float32), ang, sc


def test_estimate_refuses_bad_dtypes_and_shapes():
    import torch
    p, ang, sc = _inputs(dtype=torch.float64)
    with pytest.raises(TypeError, match="float32"):
        detector.estimate_offset(p, ang, sc)
    with pytest.raises(TypeError, match="torch tensor"):
        detector.estimate_offset(np.zeros((24, 64, 64), np.float32), ang, sc)
    p, ang, sc = _inputs()
    with pytest.raises(ValueError, match=r"\[N, H, W\]"):
        detector.estimate_offset(p[0], ang, sc)
    with pytest.raises(ValueError, match="23 angles for 24"):
        detector.estimate_offset(p, ang[:-1], sc)
    with pytest.raises(ValueError, match="detector is 64x32"):
        detector.estimate_offset(p, ang, dict(sc, nDetector=[64, 32]))
    with pytest.raises(ValueError, match="parallel beam only"):
        detector.estimate_offset(p, ang, sc, rows=(0, 4))
    p, ang, sc = _inputs("parallel")
    with pytest.raises(ValueError, match="rows"):
        detector.estimate_offset(p, ang, sc, rows=(4, 4))
    with pytest.raises(ValueError, match="max_shift"):
        detector.estimate_offset(p, ang, sc, max_shift=0)
    with pytest.raises(ValueError, match="angle_tol"):
        detector.estimate_offset(p, ang, sc, angle_tol=-1)


def test_estimate_refuses_an_arc_without_conjugate_pairs():
    p, _, sc = _inputs()
    short = np.linspace(0, 0.7 * np.pi, 24)                          # less than 180 degrees minus the fan
    with pytest.raises(detector.OffsetEstimateError, match="no conjugate pairs"):
        detector.estimate_offset(p, short, sc, max_shift=1)
    p, _, sc = _inputs("parallel", n=23)
    odd = np.linspace(0, 2 * np.pi, 24)[:-1]                         # no two views pi apart
    with pytest.raises(detector.OffsetEstimateError, match="180 degrees apart"):
        detector.estimate_offset(p, odd, sc)


def test_estimate_refuses_a_cpu_tensor_once_the_pairs_exist():
    p, ang, sc = _inputs()
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        detector.estimate_offset(p, ang, sc)


def test_cost_entry_point_refuses_sizes_it_cannot_take():
    """Checked before any CUDA work, so no device is needed (dummy pointers are never dereferenced)."""
    from r2_gaussian_b200._lib import R2XError, check, load
    lib = load()
    d = 16
    base = dict(mode=1, N=4, H=8, W=8, projs=d, n_pairs=3, views=d, dbeta=d, DSD=7.0, du=0.1, t_v=0.0, row_lo=0,
                n_rows=1, K=5, sigma=d, num=d, den=d, count=d, scratch=d, nbytes=1 << 20)

    def call(**kw):
        a = dict(base, **kw)
        check(lib.r2x_detector_offset_cost(None, a["mode"], a["N"], a["H"], a["W"], a["projs"], a["n_pairs"],
                                           a["views"], a["dbeta"], a["DSD"], a["du"], a["t_v"], a["row_lo"],
                                           a["n_rows"], a["K"], a["sigma"], a["num"], a["den"], a["count"],
                                           a["scratch"], a["nbytes"]), "r2x_detector_offset_cost")
    for kw, msg in [({"K": 65536}, "K must be"), ({"K": 0}, "K must be"), ({"n_pairs": 0}, "no conjugate pairs"),
                    ({"n_rows": 2}, "one row"), ({"t_v": 4.0}, "mid-plane row"), ({"W": 0}, "positive"),
                    ({"mode": 2}, "mode"), ({"DSD": 0.0}, "DSD"), ({"projs": None}, "null pointer"),
                    ({"mode": 0, "row_lo": 1, "n_rows": 8}, "outside the image"), ({"nbytes": 8}, "scratch"),
                    ({"mode": 0, "N": 1, "H": 2**31 - 1, "W": 2**31 - 1, "n_rows": 2**31 - 1, "n_pairs": 2**31 - 1},
                     "too many samples")]:
        with pytest.raises(R2XError, match=msg):
            call(**kw)
    assert lib.r2x_detector_offset_cost_scratch_bytes(1, 8, 3, 1, 65536) == 0
    assert lib.r2x_detector_offset_cost_scratch_bytes(1, 8, 3, 1, 65535) > 0


# ---- the flags -------------------------------------------------------------------------------------------------------

def test_recon_and_initialize_pcd_parse_the_flag_and_half_fan_needs_an_offset(tmp_path, monkeypatch):
    import torch

    from r2_gaussian_b200 import initialize_pcd, recon
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(SystemExit, match="applies to --recon_method fdk, cgls or fista_tv"):
        initialize_pcd.main(["--data", str(tmp_path), "--recon_method", "random", "--estimate_offDetector"])
    for argv in (["--estimate_offDetector"], ["--estimate_offDetector", "--use_offDetector", "--half_fan"],
                 ["--estimate_offDetector", "--half_fan"]):
        with pytest.raises(SystemExit, match="needs a CUDA device"):           # parsed and accepted
            initialize_pcd.main(["--data", str(tmp_path), "--recon_method", "fdk", *argv])
        with pytest.raises(SystemExit, match="need a CUDA device"):
            recon.main(["-s", str(tmp_path), "-m", str(tmp_path / "o"), "--methods", "fdk", *argv])
    ns = lambda **kw: argparse.Namespace(**{"short_scan": False, "half_fan": False, "fdk_filter": None,
                                            "use_offDetector": False, "estimate_offDetector": False, **kw})
    with pytest.raises(SystemExit, match="--half_fan needs --use_offDetector"):
        recon.check_fdk_flags(ns(half_fan=True), True, "{flag}")
    recon.check_fdk_flags(ns(half_fan=True, estimate_offDetector=True), True, "{flag}")


def test_trainer_parses_the_flag_next_to_refinement_and_the_file_offset(tmp_path):
    from r2_gaussian_b200 import trainer
    a, *_ = trainer.parse_args(["-s", str(tmp_path), "--estimate_offDetector", "--detector_offset_refine",
                                "--use_offDetector"])
    assert a.estimate_offDetector and a.use_offDetector and a.detector_params.detector_offset_refine
    a, *_ = trainer.parse_args(["-s", str(tmp_path)])
    assert not a.estimate_offDetector


@pytest.mark.parametrize("refine", [False, True])
def test_detector_offset_yml_carries_the_estimate_and_the_total(tmp_path, refine):
    import torch
    import yaml

    from r2_gaussian_b200 import trainer
    det = None
    if refine:
        det = detector.DetectorOffset("cpu")
        with torch.no_grad():
            det.offset.fill_(0.5)
    du = 2.0 / 128
    cfg = {"nDetector": [64, 128], "sDetector": [1.0, 2.0], "offDetector": [-(3.0 - 0.25) * du, 0.0]}   # scene units
    sc = types.SimpleNamespace(model_path=str(tmp_path), scanner_cfg=cfg, use_offDetector=True, scene_scale=0.5,
                               offset_estimate={"offset_px": 3.0, "offset_scene": 3.0 * du})
    (tmp_path / "point_cloud" / "iteration_3").mkdir(parents=True)
    trainer.save_detector_offset(sc, det, 3)
    doc = yaml.safe_load((tmp_path / "point_cloud" / "iteration_3" / "detector_offset.yml").read_text())
    assert doc["estimate_px"] == 3.0 and doc["estimate_scene"] == pytest.approx(3.0 * du)
    assert ("offset_px" in doc) == refine
    learned = 0.5 if refine else 0.0
    assert doc["offDetector_u"] == pytest.approx(-(3.0 - 0.25 + learned) * du / 0.5)
    keys = list(doc)
    assert keys[-1] == "offDetector_u"


def test_scene_takes_an_offset_override_in_a_copy_of_the_scanner(tmp_path):
    import torch

    from r2_gaussian_b200 import dataset
    from r2_gaussian_b200.dataset import write_blender
    rng = np.random.RandomState(0)
    sc = scene.cone_beam_scanner(16, 8)
    sc.update({"filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0, "noise": False})
    frames = [(0.5 * k, rng.rand(16, 16).astype(np.float32)) for k in range(3)]
    path = str(tmp_path / "case")
    write_blender(path, sc, frames[:2], frames[2:], rng.rand(8, 8, 8).astype(np.float32))
    plain = dataset.Scene(path, shuffle=False, device="cpu", use_offDetector=True)
    moved = dataset.Scene(path, shuffle=False, device="cpu", use_offDetector=True, offDetector_u=0.25)
    same = dataset.Scene(path, shuffle=False, device="cpu")
    assert moved.scanner_cfg["offDetector"] == [0.25, 0.0] and plain.scanner_cfg["offDetector"] == [0.0, 0.0]
    for a, b in zip(plain.train_cameras, same.train_cameras):
        assert torch.equal(a.full_proj_transform, b.full_proj_transform)
    t_u = 0.25 / (sc["sDetector"][1] / 16)
    for a, b in zip(moved.train_cameras, plain.train_cameras):
        d = (a.projection_matrix - b.projection_matrix).double()
        assert float(d[2, 0]) == pytest.approx(-2 * t_u / 16, rel=1e-5)   # the x row gains -(2 t_u / W) w row
