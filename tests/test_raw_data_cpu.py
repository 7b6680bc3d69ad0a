"""Raw-volume processing without a GPU: the float64 restatement of scipy's cubic zoom against scipy, the chains of
`process_raw_data` run with a scipy stand-in for the GPU zoom against a restatement of the reference's chains (bit for
bit), the refusals, skip-if-exists, the CLI defaults and the C-ABI argument checks of the zoom entry points."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import scipy.ndimage as ndimage

import raw_data_oracle as oracle
from r2_gaussian_b200 import _lib, process_raw_data as prd, resample

# (shape, factors): dims 1, 2, 3, 24, 25, 31, 33; factors 0.1 to 7; a unit axis; a unit factor beside others
ZOOM_CASES = [
    ((1, 2, 3), (3.0, 2.5, 1.7)),
    ((2, 3, 1), (7.0, 0.5, 4.0)),
    ((24, 25, 31), (0.1, 0.37, 1.9)),
    ((33, 31, 25), (1.3, 0.8, 0.1)),
    ((25, 1, 33), (0.5, 6.0, 1.0)),
    ((31, 24, 2), (2.0, 1.5, 7.0)),
    ((3, 33, 24), (1.0, 1.0, 0.25)),
    ((1, 1, 1), (2.0, 3.0, 5.0)),
]


@pytest.mark.parametrize("shape,factors", ZOOM_CASES)
def test_oracle_zoom_matches_scipy(shape, factors):
    x = np.random.default_rng(sum(shape)).random(shape)
    want = ndimage.zoom(x, factors, order=3, mode="nearest")
    got = oracle.zoom(x, factors)
    assert got.shape == want.shape == resample.zoom_shape(shape, factors)
    assert np.abs(got - want).max() <= 1e-13


def test_unit_factors_are_a_copy_bit_for_bit():
    x = np.random.default_rng(1).random((5, 6, 7))
    want = ndimage.zoom(x, (1, 1, 1), order=3, mode="nearest")
    assert want.tobytes() == x.tobytes() and oracle.zoom(x, 1.0).tobytes() == x.tobytes()


def test_windowed_zoom_equals_the_full_one():
    x = np.random.default_rng(2).random((30, 26, 40))
    full = oracle.zoom(x, (0.7, 1.9, 0.4))
    box = [(3, 6), (10, 14), (0, 3)]
    win = oracle.zoom_box(lambda i, j, k: x[np.ix_(i, j, k)], x.shape, (0.7, 1.9, 0.4), box=box, margin=32)
    assert np.abs(win - full[3:6, 10:14, 0:3]).max() <= 1e-15


def test_zoom_factor_and_shape_rules():
    assert resample.zoom_factors(2) == (2.0, 2.0, 2.0)
    assert resample.zoom_shape((373, 512, 512), (466 / 373, 500 / 512, 1.0)) == (466, 500, 512)
    assert resample.zoom_shape((5, 5, 5), (0.5, 0.7, 0.9)) == (2, 4, 4)      # round(2.5) = 2, half to even
    for bad in [(0.0, 1.0, 1.0), (1.0, -2.0, 1.0), (1.0, float("nan"), 1.0), (1.0, 1.0), float("inf")]:
        with pytest.raises(ValueError, match="finite positive"):
            resample.zoom_factors(bad)
    with pytest.raises(ValueError, match="empty axis"):
        resample.zoom_shape((1, 8, 8), (0.4, 1.0, 1.0))


def test_zoom_refuses_cpu_tensors_and_other_dtypes():
    import torch

    for vol in (torch.zeros((4, 4, 4), dtype=torch.float64), torch.zeros((4, 4, 4)), np.zeros((4, 4, 4))):
        with pytest.raises(ValueError, match="CUDA float64"):
            resample.zoom(vol, 2.0)


def test_placement_expands_crops_and_normalises():
    src = np.arange(24, dtype=np.uint16).reshape(2, 3, 4) + 10
    v = oracle.place(src, prd.cube_place(src.shape, "expand"))
    assert v.shape == (4, 4, 4) and v[1:3, 0:3, 0:4].tolist() == src.astype(float).tolist() and v.sum() == src.sum()
    v = oracle.place(src, prd.cube_place(src.shape, "crop"))
    assert v.shape == (2, 2, 2) and v.tolist() == src[:, 0:2, 1:3].astype(float).tolist()
    p = prd.normalising_place(src, "c")
    assert (p.lo, p.hi) == (10.0, 33.0)
    assert oracle.place(src, p).tobytes() == ((src.astype(float) - 10.0) / 23.0).tobytes()


# ---- the chains against the reference's, bit for bit, with scipy as the zoom ------------------------------------

@pytest.fixture
def readers(monkeypatch):
    monkeypatch.setitem(sys.modules, "tifffile", oracle.fake_tifffile())
    monkeypatch.setitem(sys.modules, "pydicom", oracle.fake_pydicom())


def make_cases(root, rng):
    """Seeded raw / tif / dcm cases covering every reshape mode, transpose, z_invert and xy_invert."""
    os.makedirs(root, exist_ok=True)
    cases = []

    def raw(name, shape, dtype, **kw):
        path = os.path.join(root, name + ".raw")
        oracle.write_raw(path, oracle.blob_volume(shape, rng, dtype))
        cases.append(dict(raw_path=path, output_name=name, file_type="raw", dtype=np.dtype(dtype).name,
                          shape=list(shape), **kw))

    def tif(name, shape, dtype, **kw):
        path = os.path.join(root, name + ".tif")
        oracle.write_tif(path, oracle.blob_volume(shape, rng, dtype))
        cases.append(dict(raw_path=path, output_name=name, file_type="tif", **kw))

    # 10 * 1.25 = 12.5 and 14 * 1.25 = 17.5: numpy's half-to-even rounding picks 12 and 18
    raw("raw_expand", (14, 10, 12), np.uint8, spacing=[1.25, 1.25, 1.0], reshape="expand", transpose=[1, 0, 2],
        z_invert=False)
    raw("raw_crop", (18, 13, 11), np.uint16, spacing=[0.9766, 0.9766, 1.25], reshape="crop", transpose=[0, 2, 1],
        z_invert=True)
    raw("raw_none", (9, 12, 7), np.float32, spacing=[1.0, 1.0, 1.0], reshape=None, transpose=[2, 0, 1], z_invert=True)
    raw("raw_unit", (16, 16, 16), np.uint8, spacing=[1.0, 1.0, 1.0], reshape="expand", transpose=[0, 1, 2],
        z_invert=False)
    raw("raw_int16", (12, 8, 10), np.int16, spacing=[1.0, 1.5, 0.5], reshape="expand", transpose=[0, 1, 2],
        z_invert=True)
    tif("tif_crop", (13, 15, 17), np.uint16, spacing=[1.0, 1.0, 1.0], reshape="crop", transpose=[1, 2, 0],
        z_invert=True)
    tif("tif_expand", (11, 9, 14), np.float64, spacing=[1.2, 0.8, 1.0], reshape="expand", transpose=[0, 1, 2],
        z_invert=False)
    tif("tif_none", (10, 12, 14), np.uint8, spacing=[1.0, 1.0, 1.0], reshape=None, transpose=[1, 2, 0],
        z_invert=True)
    for name, inv, slope, icpt in (("dcm_chest", False, 1.0, -1024.0), ("dcm_pancreas", True, 2.5, -3000.0)):
        folder = os.path.join(root, name)
        slices = [rng.integers(0, 2600, (12, 14)).astype(np.int16) for _ in range(9)]
        oracle.write_dcm_series(folder, slices, slope, icpt)
        cases.append(dict(raw_path=folder, output_name=name, file_type="dcm", thickness=None, xy_invert=inv))
    return cases


def reference_case(case, target_size):
    if case["file_type"] == "raw":
        return oracle.reference_raw(case, target_size)
    if case["file_type"] == "tif":
        return oracle.reference_tif(case, target_size, oracle.fake_tifffile().imread)
    return oracle.reference_dcm(case, target_size, oracle.fake_pydicom().dcmread)


TARGET = 16


def test_chains_equal_the_reference_bit_for_bit(tmp_path, readers):
    cases = make_cases(str(tmp_path / "raw"), np.random.default_rng(7))
    meta = str(tmp_path / "meta.py")
    oracle.write_metadata(meta, cases)
    written = prd.run(meta, str(tmp_path / "out"), TARGET, zoom=oracle.scipy_zoom_placed)
    assert len(written) == len(cases)
    for case in cases:
        got = np.load(os.path.join(tmp_path, "out", case["output_name"] + ".npy"))
        want = reference_case(case, TARGET).astype(np.float32)
        assert got.dtype == np.float32 and got.shape == (TARGET,) * 3, case["output_name"]
        assert got.tobytes() == want.tobytes(), case["output_name"]
        # in float64 too, before the cast
        f64 = prd.PROCESS[case["file_type"]](case, TARGET, oracle.scipy_zoom_placed)
        assert np.ascontiguousarray(f64).tobytes() == np.ascontiguousarray(reference_case(case, TARGET)).tobytes()


def test_reshape_plan_rounds_half_to_even():
    factors, places = prd.reshape_plan((14, 10, 12), [1.25, 1.25, 1.0], 16, "expand")
    assert resample.zoom_shape((14, 10, 12), factors[0]) == (18, 12, 12)
    assert places[0] == resample.Place((18, 18, 18), (0, 3, 3)) and factors[1] == (16 / 18,) * 3
    factors, places = prd.reshape_plan((512, 512, 373), [0.9766, 0.9766, 1.25], 256, "expand")
    assert resample.zoom_shape((512, 512, 373), factors[0]) == (500, 500, 466)
    factors, places = prd.reshape_plan((1024, 1024, 795), [0.03174 * 20, 0.03174 * 20, 0.0688 * 20], 256, "expand")
    assert resample.zoom_shape((1024, 1024, 795), factors[0]) == (650, 650, 1094) and places[0].shape == (1094,) * 3
    assert prd.reshape_plan((10, 20, 30), [2.0, 1.0, 1.0], 16, None) == ([(1.6, 0.8, 16 / 30)], [])


# ---- refusals, skipping, CLI ------------------------------------------------------------------------------------

def _one(tmp_path, case):
    meta = str(tmp_path / "meta.py")
    oracle.write_metadata(meta, [case])
    return meta


def _raw_case(tmp_path, vol=None, **over):
    vol = oracle.blob_volume((6, 5, 4), np.random.default_rng(0)) if vol is None else vol
    path = str(tmp_path / "v.raw")
    oracle.write_raw(path, vol)
    case = dict(raw_path=path, output_name="vol", file_type="raw", dtype="uint8", shape=[6, 5, 4],
                spacing=[1.0, 1.0, 1.0], reshape="expand", transpose=[0, 1, 2], z_invert=False)
    case.update(over)
    return case


def test_missing_key_unknown_type_and_mode_are_refused_by_case(tmp_path):
    case = _raw_case(tmp_path)
    del case["spacing"]
    with pytest.raises(ValueError, match=r"case vol: metadata has no 'spacing'"):
        prd.run(_one(tmp_path, case), str(tmp_path / "out"), 8, zoom=oracle.scipy_zoom_placed)
    with pytest.raises(ValueError, match=r"case vol: unsupported file_type 'nii'"):
        prd.run(_one(tmp_path, _raw_case(tmp_path, file_type="nii")), str(tmp_path / "out"), 8,
                zoom=oracle.scipy_zoom_placed)
    with pytest.raises(ValueError, match=r"case vol: unsupported reshape 'pad'"):
        prd.run(_one(tmp_path, _raw_case(tmp_path, reshape="pad")), str(tmp_path / "out"), 8,
                zoom=oracle.scipy_zoom_placed)
    with pytest.raises(ValueError, match=r"case \?: metadata has no 'output_name'"):
        prd.check_case({"file_type": "raw"})
    # every case is checked before any is processed
    good, bad = _raw_case(tmp_path), _raw_case(tmp_path, output_name="bad", file_type="mhd")
    meta = str(tmp_path / "two.py")
    oracle.write_metadata(meta, [good, bad])
    with pytest.raises(ValueError, match="case bad"):
        prd.run(meta, str(tmp_path / "out2"), 8, zoom=oracle.scipy_zoom_placed)
    assert not os.path.exists(tmp_path / "out2" / "vol.npy")


def test_raw_size_mismatch_is_refused(tmp_path):
    with pytest.raises(ValueError, match=r"case vol: .* has 120 bytes, shape \[6, 5, 5\] of uint8 needs 150"):
        prd.run(_one(tmp_path, _raw_case(tmp_path, shape=[6, 5, 5])), str(tmp_path / "out"), 8,
                zoom=oracle.scipy_zoom_placed)
    with pytest.raises(ValueError, match="needs 240"):
        prd.run(_one(tmp_path, _raw_case(tmp_path, dtype="uint16")), str(tmp_path / "out"), 8,
                zoom=oracle.scipy_zoom_placed)


def test_constant_and_non_finite_volumes_are_refused(tmp_path):
    case = _raw_case(tmp_path, vol=np.full((6, 5, 4), 7, np.uint8))
    with pytest.raises(ValueError, match="case vol: the volume is constant"):
        prd.run(_one(tmp_path, case), str(tmp_path / "out"), 8, zoom=oracle.scipy_zoom_placed)
    vol = np.ones((6, 5, 4))
    vol[1, 2, 3] = np.nan
    case = _raw_case(tmp_path, vol=vol, dtype="float64")
    with pytest.raises(ValueError, match="case vol: the volume has non-finite values"):
        prd.run(_one(tmp_path, case), str(tmp_path / "out"), 8, zoom=oracle.scipy_zoom_placed)
    assert not os.path.exists(tmp_path / "out" / "vol.npy")


def test_missing_readers_are_named(tmp_path, monkeypatch):
    monkeypatch.setitem(sys.modules, "tifffile", None)      # import raises ImportError
    monkeypatch.setitem(sys.modules, "pydicom", None)
    tif = dict(raw_path=str(tmp_path / "x.tif"), output_name="pepper", file_type="tif", spacing=[1, 1, 1],
               reshape=None, transpose=[0, 1, 2], z_invert=False)
    with pytest.raises(RuntimeError, match="case pepper: reading it needs the 'tifffile' package"):
        prd.run(_one(tmp_path, tif), str(tmp_path / "out"), 8, zoom=oracle.scipy_zoom_placed)
    dcm = dict(raw_path=str(tmp_path), output_name="chest", file_type="dcm", thickness=None, xy_invert=False)
    with pytest.raises(RuntimeError, match="case chest: reading it needs the 'pydicom' package"):
        prd.run(_one(tmp_path, dcm), str(tmp_path / "out"), 8, zoom=oracle.scipy_zoom_placed)


def test_tif_of_an_unrestated_dtype_is_refused(tmp_path, readers):
    oracle.write_tif(str(tmp_path / "x.tif"), np.arange(64, dtype=np.int16).reshape(4, 4, 4))
    tif = dict(raw_path=str(tmp_path / "x.tif"), output_name="t", file_type="tif", spacing=[1, 1, 1],
               reshape=None, transpose=[0, 1, 2], z_invert=False)
    with pytest.raises(ValueError, match="case t: .* int16"):
        prd.run(_one(tmp_path, tif), str(tmp_path / "out"), 8, zoom=oracle.scipy_zoom_placed)


def test_existing_outputs_are_skipped_without_a_gpu(tmp_path, monkeypatch):
    import torch

    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    meta = _one(tmp_path, _raw_case(tmp_path))
    out = tmp_path / "out"
    with pytest.raises(RuntimeError, match="CUDA"):
        prd.run(meta, str(out), 8)
    out.mkdir(exist_ok=True)
    np.save(out / "vol.npy", np.zeros(3, np.float32))
    assert prd.run(meta, str(out), 8) == []
    assert np.load(out / "vol.npy").tolist() == [0.0, 0.0, 0.0]


def test_cli_defaults(monkeypatch):
    seen = {}
    monkeypatch.setattr(prd, "run", lambda *a: seen.setdefault("args", a))
    prd.main([])
    assert seen["args"] == ("data_generator/raw_metadata.py", "data_generator/volume_gt", 256)
    seen.clear()
    prd.main(["--metadata", "m.py", "--output", "o", "--target_size", "64"])
    assert seen["args"] == ("m.py", "o", 64)


# ---- C ABI ------------------------------------------------------------------------------------------------------

def _desc(**over):
    d = _lib.PlaceDesc()
    d.src, d.dtype = 16, 0          # never dereferenced: every call below fails its checks first
    for a in range(3):
        d.src_shape[a], d.src_strides[a], d.shape[a], d.offset[a] = 4, [16, 4, 1][a], 4, 0
    d.lo, d.hi = 0.0, 1.0
    for k, v in over.items():
        if isinstance(v, tuple):
            getattr(d, k)[v[0]] = v[1]
        else:
            setattr(d, k, v)
    return d


def test_c_abi_refuses_bad_arguments_without_a_gpu():
    lib = _lib.load()
    assert lib.r2x_zoom_workspace_bytes(4, 5, 6) == 28 * 29 * 30 * 8
    assert lib.r2x_zoom_workspace_bytes(1094, 1094, 1094) == 1118 ** 3 * 8
    assert lib.r2x_zoom_workspace_bytes(0, 5, 6) == 0 and lib.r2x_zoom_workspace_bytes(4, 32769, 6) == 0
    buf = C.c_void_p(16)
    ws = lib.r2x_zoom_workspace_bytes(4, 4, 4)
    bad_descs = [
        (_desc(src=None), b"bad pointer"),
        (_desc(dtype=3), b"bad dtype"),
        (_desc(src_shape=(1, 0)), b"bad source shape"),
        (_desc(src_strides=(2, -1)), b"bad source strides"),
        (_desc(shape=(0, 0)), b"bad placed shape"),
        (_desc(shape=(2, 40000)), b"bad placed shape"),
        (_desc(lo=1.0, hi=1.0), b"bad lo / hi"),
        (_desc(hi=float("inf")), b"bad lo / hi"),
    ]
    for d, msg in bad_descs:
        for fn, call in (("r2x_volume_place", lambda: lib.r2x_volume_place(None, C.byref(d), buf)),
                         ("r2x_zoom_cubic", lambda: lib.r2x_zoom_cubic(None, C.byref(d), 8, 8, 8, buf, ws, buf))):
            assert call() == 1, (fn, msg)
            err = lib.r2x_last_error()
            assert msg in err and fn.encode() in err, (msg, err)
    d = _desc()
    cases = [
        (lambda: lib.r2x_volume_place(None, None, buf), b"bad pointer"),
        (lambda: lib.r2x_volume_place(None, C.byref(d), None), b"bad pointer"),
        (lambda: lib.r2x_zoom_cubic(None, C.byref(d), 0, 8, 8, buf, ws, buf), b"bad output shape"),
        (lambda: lib.r2x_zoom_cubic(None, C.byref(d), 8, 8, 32769, buf, ws, buf), b"bad output shape"),
        (lambda: lib.r2x_zoom_cubic(None, C.byref(d), 8, 8, 8, None, ws, buf), b"bad pointer"),
        (lambda: lib.r2x_zoom_cubic(None, C.byref(d), 8, 8, 8, buf, ws, None), b"bad pointer"),
        (lambda: lib.r2x_zoom_cubic(None, C.byref(d), 8, 8, 8, buf, ws - 1, buf), b"bad workspace"),
    ]
    for call, msg in cases:
        assert call() == 1
        assert msg in lib.r2x_last_error(), (msg, lib.r2x_last_error())
