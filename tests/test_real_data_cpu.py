"""Real-scan scene builder without a GPU: the numpy restatement of the preparation chain against cv2's golden bytes,
config.txt parsing, angles and the train / test split against a restatement of the reference's lines, the refusals,
and r2x_projection_prepare's argument checks through the C ABI."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import real_data_oracle as oracle
import util
from r2_gaussian_b200 import _lib, generate_real_data as grd

GOLDEN = os.path.join(util.ROOT, "tests", "golden", "real_data", "cases.npz")
CASES = ("divisible", "not_divisible", "odd_crop", "diff_one", "no_subsample", "ratio_5", "half")


def golden(name):
    g = np.load(GOLDEN)
    s, rescale, obj = g[name + "_params"]
    return g[name + "_img"], int(s), float(rescale), float(obj), g[name + "_out"]


@pytest.mark.parametrize("name", CASES)
def test_oracle_equals_cv2_golden_bytes(name):
    img, s, rescale, obj, want = golden(name)
    got = oracle.prepare(img, s, rescale, obj)
    assert got.dtype == np.float32 and got.shape == want.shape
    assert got.tobytes() == want.tobytes()


def test_golden_shapes_cover_the_crop_rules():
    shapes = {name: golden(name)[4].shape for name in CASES}
    assert shapes["odd_crop"] == (20, 21)          # difference 7: the reference's off-by-one, non-square
    assert shapes["diff_one"] == (17, 16)          # difference 1: nothing cropped
    assert shapes["no_subsample"] == (32, 40)      # s = 1: no resize, no crop


def test_fma_f32_rounds_once():
    rng = np.random.default_rng(3)
    a, b, c = (rng.standard_normal(20000).astype(np.float32) for _ in range(3))
    got = oracle.fma_f32(a, b, c)
    exact = [float(np.float32(float(x) * float(y) + float(z))) for x, y, z in zip(a[:2000], b[:2000], c[:2000])]
    assert np.array_equal(got[:2000], np.array(exact, np.float32))
    # a float64 sum exactly half-way between two float32 values with a non-zero remainder
    a1, b1 = np.float32(1 + 2 ** -12), np.float32(1 + 2 ** -12)     # a b = 1 + 2^-11 + 2^-24
    c1 = np.float32(2 ** -60)
    assert oracle.fma_f32(a1, b1, c1) == np.float32(1 + 2 ** -11 + 2 ** -23)


def _reference_config(path, proj_subsample, object_scale):
    with open(path, "r") as f:
        for config_line in f.readlines():
            if "NumberImages" in config_line:
                n_proj = int(config_line.split("=")[-1])
            elif "AngleInterval" in config_line:
                angle_interval = float(config_line.split("=")[-1])
            elif "AngleFirst" in config_line:
                angle_start = float(config_line.split("=")[-1])
            elif "AngleLast" in config_line:
                angle_last = float(config_line.split("=")[-1])
            elif "DistanceSourceDetector" in config_line:
                DSD = float(config_line.split("=")[-1]) / 1000 * object_scale
            elif "DistanceSourceOrigin" in config_line:
                DSO = float(config_line.split("=")[-1]) / 1000 * object_scale
            elif "PixelSize" in config_line and "PixelSizeUnit" not in config_line:
                dDetector = float(config_line.split("=")[-1]) * proj_subsample / 1000 * object_scale
    angles = np.concatenate([np.arange(angle_start, angle_last, angle_interval), [angle_last]]) / 180.0 * np.pi
    return n_proj, angle_interval, angle_start, angle_last, DSD, DSO, dDetector, angles


def _reference_ids(n_proj, n_train, n_test):
    state = random.getstate()
    try:
        random.seed(0)
        train_ids = np.linspace(0, n_proj - 1, n_train).astype(int)
        test_ids = sorted(random.sample(np.setdiff1d(np.arange(n_proj), train_ids).tolist(), n_test))
    finally:
        random.setstate(state)
    return train_ids, test_ids


def _write_config(tmp_path, text):
    p = tmp_path / "config.txt"
    p.write_text(text)
    return str(p)


FIPS_CONFIG = oracle.CONFIG_TEMPLATE.format(n=721, interval=0.5, first=0, last=360, dsd=553.74, dso=410.66,
                                            pixel=0.05) + "PixelSizeUnitNote = 7\n"


@pytest.mark.parametrize("subsample,object_scale", [(4, 50), (1, 50), (3, 20)])
def test_config_and_angles_equal_the_reference(tmp_path, subsample, object_scale):
    path = _write_config(tmp_path, FIPS_CONFIG)
    cfg = grd.read_config(path, subsample, object_scale)
    n, interval, first, last, DSD, DSO, dDet, angles = _reference_config(path, subsample, object_scale)
    assert (cfg["n_proj"], cfg["angle_interval"], cfg["angle_first"], cfg["angle_last"]) == (n, interval, first, last)
    assert (cfg["DSD"], cfg["DSO"], cfg["dDetector"]) == (DSD, DSO, dDet)
    got = grd.scan_angles(cfg)
    assert len(got) == 721 and np.array_equal(got, angles)


@pytest.mark.parametrize("n_proj,n_train,n_test", [(721, 75, 100), (721, 50, 100), (721, 25, 100), (40, 7, 33),
                                                   (10, 1, 0), (100, 100, 0)])
def test_split_ids_equal_the_reference(n_proj, n_train, n_test):
    train, test = grd.split_ids(n_proj, n_train, n_test)
    rt, rs = _reference_ids(n_proj, n_train, n_test)
    assert np.array_equal(train, rt) and test == rs


def test_split_leaves_the_global_random_state_alone():
    random.seed(1234)
    state = random.getstate()
    grd.split_ids(721, 75, 100)
    assert random.getstate() == state


def test_missing_key_is_refused_by_name(tmp_path):
    text = FIPS_CONFIG.replace("DistanceSourceOrigin", "SourceOriginDistance")
    with pytest.raises(ValueError, match="DistanceSourceOrigin"):
        grd.read_config(_write_config(tmp_path, text), 4, 50)
    text = FIPS_CONFIG.replace("PixelSize =", "Pitch =")      # only PixelSizeUnit left: still missing
    with pytest.raises(ValueError, match="PixelSize"):
        grd.read_config(_write_config(tmp_path, text), 4, 50)


def _case(tmp_path, n=6, n_proj=None, shape=(24, 24)):
    imgs = [np.full(shape, float(i)) for i in range(n)]
    oracle.write_fips_case(str(tmp_path / "scan"), imgs, 0.0, 60.0, n_proj=n_proj)
    return str(tmp_path / "scan")


def test_count_mismatch_is_refused(tmp_path):
    d = _case(tmp_path, n=6)
    os.remove(os.path.join(d, "scan_0005.mat"))
    with pytest.raises(ValueError, match="5 .mat files"):
        grd.generate(d, str(tmp_path / "out"), n_train=2, n_test=1)
    d2 = _case(tmp_path / "b", n=6, n_proj=7)
    with pytest.raises(ValueError, match="NumberImages = 7"):
        grd.generate(d2, str(tmp_path / "out2"), n_train=2, n_test=1)


def test_too_many_views_are_refused(tmp_path):
    d = _case(tmp_path, n=6)
    with pytest.raises(ValueError, match="scan with 6"):
        grd.generate(d, str(tmp_path / "out"), n_train=4, n_test=3)


def test_no_cuda_is_refused(tmp_path, monkeypatch):
    import torch

    d = _case(tmp_path, n=6)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(RuntimeError, match="CUDA"):
        grd.generate(d, str(tmp_path / "out"), n_train=2, n_test=1)
    assert not os.path.exists(tmp_path / "out")


@pytest.mark.parametrize("H0,W0,s", [(64, 72, 4), (67, 81, 4), (61, 83, 3), (70, 64, 4), (32, 40, 1), (97, 131, 5),
                                     (2368, 2240, 4), (1536, 1944, 4), (5, 5, 5), (1, 9, 1)])
def test_prepared_shape_matches_the_oracle(H0, W0, s):
    assert grd.prepared_shape(H0, W0, s) == oracle.output_shape(H0, W0, s)[4:]


def test_c_abi_refuses_bad_arguments_without_a_gpu():
    lib = _lib.load()
    hw = (C.c_int * 2)()
    buf = C.c_void_p(16)    # never dereferenced: every call below fails its checks first
    cases = [
        (lambda: lib.r2x_projection_prepare_shape(0, 8, 1, hw), b"bad image size"),
        (lambda: lib.r2x_projection_prepare_shape(8, 8, 0, hw), b"bad subsample"),
        (lambda: lib.r2x_projection_prepare_shape(3, 8, 4, hw), b"bad subsample"),
        (lambda: lib.r2x_projection_prepare_shape(8, 8, 2, None), b"bad pointer"),
        (lambda: lib.r2x_projection_prepare_shape(65536, 65536, 1, hw), b"bad image size"),
        (lambda: lib.r2x_projection_prepare(None, 0, 8, 8, 1, buf, 400.0, 50.0, buf), b"bad n_views"),
        (lambda: lib.r2x_projection_prepare(None, 1, 8, -1, 1, buf, 400.0, 50.0, buf), b"bad image size"),
        (lambda: lib.r2x_projection_prepare(None, 1, 8, 8, -2, buf, 400.0, 50.0, buf), b"bad subsample"),
        (lambda: lib.r2x_projection_prepare(None, 1, 8, 8, 1, None, 400.0, 50.0, buf), b"bad pointer"),
        (lambda: lib.r2x_projection_prepare(None, 1, 8, 8, 1, buf, 400.0, 50.0, None), b"bad pointer"),
        (lambda: lib.r2x_projection_prepare(None, 1, 8, 8, 1, buf, 0.0, 50.0, buf), b"bad proj_rescale"),
        (lambda: lib.r2x_projection_prepare(None, 1, 8, 8, 1, buf, float("inf"), 50.0, buf), b"bad proj_rescale"),
        (lambda: lib.r2x_projection_prepare(None, 1, 8, 8, 1, buf, 400.0, float("nan"), buf), b"bad object_scale"),
    ]
    for call, msg in cases:
        assert call() == 1      # R2X_ERR_INVALID
        assert msg in lib.r2x_last_error(), (msg, lib.r2x_last_error())
    assert lib.r2x_projection_prepare_shape(70, 64, 4, hw) == 0 and tuple(hw) == (17, 16)
