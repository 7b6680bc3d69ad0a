"""The detector-offset estimate on the GPU: r2x_detector_offset_cost against the float64 oracle
(tests/offset_estimate_oracle.py) at odd shapes, pair counts around its CTA and chunk sizes and its launch limits;
bitwise reproducibility; `detector.estimate_offset` against the oracle's estimate on blob phantoms; recovery of the
projector's own sub-pixel detector offsets and of the 3-column recovery scene; and `--estimate_offDetector` end to end
through recon, initialize_pcd and the trainer."""
import json
import math

import numpy as np
import pytest

import offset_estimate_oracle as oo

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
REL = 1e-6


def _scanner(mode, n=64):
    from r2_gaussian_b200 import scene
    return scene.cone_beam_scanner(n, 32) if mode == "cone" else scene.parallel_beam_scanner(n, 32)


def _kernel(projs, table, sc, sigmas, t_v=0.0, rows=None):
    from r2_gaussian_b200 import detector
    p = torch.tensor(np.asarray(projs, np.float32), device=DEV)
    cone = sc["mode"] == "cone"
    H, W = int(p.shape[1]), int(p.shape[2])
    views = torch.tensor(np.array([(i, j) for i, j, _ in table], np.int32).reshape(-1, 2), device=DEV)
    dbeta = torch.tensor(np.array([d for *_, d in table], np.float64), device=DEV)
    row_lo, n_rows = (0, 1) if cone else ((0, H) if rows is None else (rows[0], rows[1] - rows[0]))
    geom = (float(sc["DSD"]) if cone else 0.0, sc["sDetector"][1] / W, float(t_v), row_lo, n_rows)
    return detector._offset_cost(p, 1 if cone else 0, (views, dbeta), geom, np.asarray(sigmas, np.float64))


def _compare(projs, table, sc, sigmas, t_v=0.0, rows=None):
    p32 = np.asarray(projs, np.float32)
    num, den, cnt = _kernel(p32, table, sc, sigmas, t_v, rows)
    onum, oden, ocnt = oo.cost_terms(p32.astype(np.float64), table, sc, sigmas, t_v, rows)
    assert np.array_equal(cnt, ocnt), (cnt, ocnt)
    scale = max(float(oden.max()), 1e-300)
    assert np.all(np.abs(num - onum) <= REL * np.maximum(np.abs(onum), 1e-12 * scale)), np.abs(num - onum).max()
    assert np.all(np.abs(den - oden) <= REL * np.maximum(np.abs(oden), 1e-12 * scale))
    return num, den, cnt


def _random_table(n_pairs, N, mode, seed=0):
    rng = np.random.RandomState(seed)
    i = rng.randint(0, N, n_pairs)
    j = (i + rng.randint(1, N, n_pairs)) % N
    d = np.pi + (rng.uniform(-0.5, 0.5, n_pairs) if mode == "cone" else 0.0)
    return [(int(a), int(b), float(c)) for a, b, c in zip(i, j, d)]


# ---- the cost kernel against the oracle ------------------------------------------------------------------------------

@pytest.mark.parametrize("W", [1, 2, 3, 255, 256, 257])
@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_cost_matches_the_oracle_at_odd_widths(mode, W):
    rng = np.random.RandomState(W)
    sc = _scanner(mode, W)
    H, N = 3, 6
    sc["nDetector"] = [H, W]
    projs = rng.rand(N, H, W)
    table = [(0, 3, np.pi), (1, 4, np.pi), (5, 2, np.pi)] if mode == "parallel" else _random_table(40, N, mode, W)
    sigmas = np.concatenate([[0.0, 0.5, -0.25], rng.uniform(-W / 2 - 1, W / 2 + 1, 8)])
    _, _, cnt = _compare(projs, table, sc, sigmas)
    if W == 1 and mode == "parallel":
        assert cnt[0] == 3 * H and cnt[1] == 0                      # one column: only sigma = 0 lands on it


@pytest.mark.parametrize("n_pairs", [1, 255, 256, 257, 4095, 4096, 4097, 256 * 4096 + 1])
def test_cost_matches_the_oracle_at_pair_counts_around_the_cta_and_chunk(n_pairs):
    """Cone beam, one sample per pair: 256 threads per CTA, 4096 samples per chunk, at most 256 chunks."""
    rng = np.random.RandomState(n_pairs % 1000)
    sc = _scanner("cone", 32)
    projs = rng.rand(16, 32, 32)
    _compare(projs, _random_table(n_pairs, 16, "cone", 1), sc, rng.uniform(-4, 4, 5))


@pytest.mark.parametrize("W", [15, 16, 17])
def test_parallel_cost_at_sample_counts_around_the_chunk(W):
    rng = np.random.RandomState(W)
    sc = _scanner("parallel", W)
    H = 4096 // W + 1
    sc["nDetector"] = [H, W]
    projs = rng.rand(4, H, W)
    _compare(projs, [(0, 2, np.pi), (1, 3, np.pi)], sc, rng.uniform(-3, 3, 5), rows=(1, H))


def test_cost_at_the_candidate_limit_and_refused_past_it():
    from r2_gaussian_b200._lib import R2XError
    rng = np.random.RandomState(0)
    sc = _scanner("cone", 16)
    projs = rng.rand(6, 16, 16).astype(np.float32)
    table = _random_table(7, 6, "cone")
    sig = np.linspace(-9, 9, 65535)
    num, den, cnt = _kernel(projs, table, sc, sig)
    pick = np.r_[0:65535:4099, 65534]
    onum, oden, ocnt = oo.cost_terms(projs.astype(np.float64), table, sc, sig[pick])
    assert np.array_equal(cnt[pick], ocnt)
    assert np.allclose(num[pick], onum, rtol=REL, atol=0) and np.allclose(den[pick], oden, rtol=REL, atol=0)
    with pytest.raises(R2XError, match="K must be"):
        _kernel(projs, table, sc, np.zeros(65536))


def test_cost_on_721_cone_views_of_512_squared_with_1024_candidates():
    rng = np.random.RandomState(1)
    sc = _scanner("cone", 512)
    ang = np.linspace(0, 2 * np.pi, 722)[:-1]
    table = oo.pairs(ang, sc, 255.5 + 20)
    projs = rng.rand(721, 512, 512).astype(np.float32)
    _compare(projs, table, sc, np.linspace(-19.5, 19.5, 1024))


def test_cost_on_720_parallel_views_of_512_squared():
    rng = np.random.RandomState(2)
    sc = _scanner("parallel", 512)
    ang = np.linspace(0, 2 * np.pi, 721)[:-1]
    table = oo.pairs(ang, sc, 0)
    assert len(table) == 360
    projs = rng.rand(720, 512, 512).astype(np.float32)
    _compare(projs, table, sc, [-1.3, 0.0, 2.7], rows=(240, 272))
    num, den, cnt = _kernel(projs, table, sc, [0.0, 0.5])           # every row: 360 x 512 x 512 samples
    assert cnt[0] == 360 * 512 * 512 and cnt[1] == 360 * 512 * 510      # m + 0.5 <= 511 and 511.5 - m <= 511


def test_two_calls_give_the_same_bits():
    from r2_gaussian_b200 import detector
    sc = _scanner("parallel")
    ang = np.linspace(0, 2 * np.pi, 25)[:-1]
    p = torch.tensor(oo.project(oo.blobs(9, radius=0.5), ang, sc, sigma=1.3), dtype=torch.float32, device=DEV)
    a = detector.estimate_offset(p, ang, sc)
    b = detector.estimate_offset(p, ang, sc)
    assert np.array_equal(np.array(a["fine"][1]), np.array(b["fine"][1])) and a["offset_px"] == b["offset_px"]
    table = oo.pairs(ang, sc, 0)
    x, y = _kernel(p.cpu().numpy(), table, sc, np.linspace(-3, 3, 77)), _kernel(p.cpu().numpy(), table, sc,
                                                                                 np.linspace(-3, 3, 77))
    assert all(np.array_equal(u.view(np.int64), v.view(np.int64)) for u, v in zip(x, y))


# ---- the estimate ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n", [24, 50])
@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_estimate_equals_the_oracle_estimate_on_blob_phantoms(mode, n):
    from r2_gaussian_b200 import detector
    sc = _scanner(mode)
    bl = oo.blobs(9, seed=0, radius=0.5)
    ang = np.linspace(0, 2 * np.pi, n + 1)[:-1] + 0.3
    du = sc["sDetector"][1] / 64
    for s, t_u in ((-3.7, 0.0), (-0.4, 0.0), (0.0, 0.0), (1.25, 0.0), (2.4, 0.0), (1.25, -16.0)):
        p = oo.project(bl, ang, sc, sigma=s - t_u).astype(np.float32)
        ref, _ = oo.estimate(p.astype(np.float64), ang, sc, t_u=t_u)
        cfg = dict(sc, offDetector=[t_u * du, 0.0])
        est = detector.estimate_offset(torch.tensor(p, device=DEV), ang, cfg, use_offDetector=t_u != 0.0)
        assert abs(est["offset_px"] - ref) <= 0.01, (s, t_u, est["offset_px"], ref)
        assert abs(est["offset_px"] - s) <= 0.03
        assert est["offDetector_u"] == pytest.approx((t_u - est["offset_px"]) * du)


def test_estimate_refuses_an_empty_mid_plane_and_a_minimum_on_the_edge():
    from r2_gaussian_b200 import detector
    sc = _scanner("cone")
    ang = np.linspace(0, 2 * np.pi, 25)[:-1]
    with pytest.raises(detector.OffsetEstimateError, match="no signal"):
        detector.estimate_offset(torch.zeros((24, 64, 64), device=DEV), ang, sc)
    p = oo.project(oo.blobs(9, radius=0.5), ang, sc, sigma=9.0).astype(np.float32)
    with pytest.raises(detector.OffsetEstimateError, match="edge of the search range"):
        detector.estimate_offset(torch.tensor(p, device=DEV), ang, sc, max_shift=4)


# ---- generate_data scenes --------------------------------------------------------------------------------------------

def _scene(tmp_path, name, off_px, noise):
    """The round-trip volume (48^3, 96^2 detector) projected by generate_data with the scanner's offDetector[0] =
    off_px pixels (24 train views), with the reference's Poisson + Gaussian noise when `noise`."""
    import projector_cases as pc
    from r2_gaussian_b200 import generate_data, scene
    from test_projector_gpu import _write_inputs
    tmp_path.mkdir(parents=True, exist_ok=True)
    _, vol_path, *_ = _write_inputs(tmp_path, noise=False)
    sc = scene.cone_beam_scanner(pc.ROUND_TRIP_DET, pc.ROUND_TRIP_VOX)
    phys = {k: (np.asarray(v, float) * 2.0).tolist() if k in ("DSD", "DSO", "sDetector", "sVoxel", "offOrigin")
            else v for k, v in sc.items()}
    phys["offDetector"] = [off_px * phys["sDetector"][1] / pc.ROUND_TRIP_DET, 0.0]
    phys.update({"filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 30.0, "noise": noise,
                 "possion_noise": 100000, "gaussian_noise": [0, 10]})
    yml = tmp_path / f"{name}.yml"
    yml.write_text("".join(f"{k}: {json.dumps(v)}\n" for k, v in phys.items()))
    return generate_data.main(["--vol", str(vol_path), "--scanner", str(yml), "--n_train", "24", "--n_test", "6",
                               "--output", str(tmp_path / name), "--use_offDetector"])


# |estimate - truth| (px) on the generate_data scenes below, from the nominal (centred) geometry, measured on an H100
# (the estimate equals the float64 oracle's to 1e-4 px on each): noise-free at most 0.0045 (t_u = -0.35), with the
# reference's Poisson + Gaussian noise at most 0.0084 (t_u = -2.6, +3.45); the 3-column recovery scenes 0.0000.
SCENE_TOL = 0.02
NOISY_TOL = 0.05


@pytest.mark.parametrize("noise", [False, True], ids=["clean", "noisy"])
def test_estimate_recovers_the_projector_s_sub_pixel_offsets(tmp_path, noise):
    from r2_gaussian_b200.dataset import read_scene
    from r2_gaussian_b200.estimate_offset import estimate_scene
    errs = []
    for k, t_u in enumerate((-2.6, -0.35, 0.0, 1.3, 3.45)):
        info = read_scene(_scene(tmp_path / f"s{k}", f"off{k}", t_u, noise), eval=False)
        est = estimate_scene(info)                                   # nominal geometry: s = -t_u
        p = np.stack([c.image for c in info.train_cameras]).astype(np.float32).astype(np.float64)
        ref, _ = oo.estimate(p, [c.angle for c in info.train_cameras], info.scanner_cfg)
        errs.append((t_u, est["offset_px"] + t_u, ref + t_u))
    print(f"noise={noise}: (t_u, estimate error, oracle error) px: " + ", ".join(f"({a:+.2f}, {b:+.4f}, {c:+.4f})"
                                                                         for a, b, c in errs))
    for t_u, e, r in errs:
        assert abs(e - r) <= 0.01                                    # the GPU estimate is the oracle's
        assert abs(e) <= (NOISY_TOL if noise else SCENE_TOL), (t_u, e)


@pytest.fixture(scope="module")
def shifted_scenes(tmp_path_factory):
    from detector_cases import recovery_scenes
    return recovery_scenes(tmp_path_factory.mktemp("estimate_scene"))


def test_estimate_on_the_recovery_scenes(shifted_scenes, tmp_path):
    from detector_cases import SHIFT
    from r2_gaussian_b200 import estimate_offset
    out = {}
    for name in ("plain", "shifted"):
        out[name] = estimate_offset.main(["-s", shifted_scenes[name][0], "--output", str(tmp_path / f"{name}.yml")])
    print(f"recovery scenes: plain {out['plain']['offset_px']:+.4f} px, shifted {out['shifted']['offset_px']:+.4f} px")
    assert abs(out["shifted"]["offset_px"] - SHIFT) <= SCENE_TOL
    assert abs(out["plain"]["offset_px"]) <= SCENE_TOL
    import yaml
    doc = yaml.safe_load((tmp_path / "shifted.yml").read_text())
    assert set(doc) >= {"offset_px", "offset_scene", "sign_convention", "offDetector_u"}
    assert doc["offDetector_u"] < 0                                   # content moved right: the file's u is negative


def test_estimate_offDetector_end_to_end(shifted_scenes, tmp_path):
    """recon's fdk on the shifted scene with the flag against fdk on the plain scene, initialize_pcd with the flag, and
    the trainer with the flag (no refinement) against the plain scene's 2000-iteration score."""
    from detector_cases import ITERATIONS as it, train
    from r2_gaussian_b200 import initialize_pcd, recon, trainer
    plain, shifted = shifted_scenes["plain"][0], shifted_scenes["shifted"][0]
    r_plain = recon.main(["-s", plain, "-m", str(tmp_path / "r_plain"), "--methods", "fdk"])["fdk"]
    r_est = recon.main(["-s", shifted, "-m", str(tmp_path / "r_est"), "--methods", "fdk", "--estimate_offDetector"])["fdk"]
    r_off = recon.main(["-s", shifted, "-m", str(tmp_path / "r_off"), "--methods", "fdk"])["fdk"]
    init = initialize_pcd.main(["--data", shifted, "--recon_method", "fdk", "--n_points", "2000",
                                "--output", str(tmp_path / "init_est.npy"), "--estimate_offDetector"])
    import random
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    model = trainer.ModelParams(source_path=shifted, model_path=str(tmp_path / "m_est"), ply_path=init)
    h = trainer.training(model, trainer.OptimizationParams(iterations=it), trainer.PipelineParams(), {it}, {it},
                         log=lambda *a: None, estimate_offDetector=True)
    h_plain = train(plain, shifted_scenes["plain"][1], tmp_path / "m_plain", trainer.DetectorParams())
    p_est, p_plain = h["eval"][it]["psnr_3d"], h_plain["eval"][it]["psnr_3d"]
    print(f"fdk psnr_3d: plain {r_plain['psnr_3d']:.2f}, shifted {r_off['psnr_3d']:.2f}, shifted + estimate "
          f"{r_est['psnr_3d']:.2f}; trainer psnr_3d: plain {p_plain:.2f}, shifted + estimate {p_est:.2f} "
          f"(estimate {h['detector_estimate_px']:+.4f} px)")
    assert r_est["psnr_3d"] >= r_plain["psnr_3d"] - 0.5
    assert r_est["estimated_offset_px"] == pytest.approx(h["detector_estimate_px"])
    assert p_est >= p_plain - 1.5
    import yaml
    doc = yaml.safe_load((tmp_path / "m_est" / "point_cloud" / f"iteration_{it}" / "detector_offset.yml").read_text())
    assert doc["estimate_px"] == pytest.approx(h["detector_estimate_px"]) and "offset_px" not in doc
