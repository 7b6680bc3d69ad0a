"""The limit cases of the scene rasterizer, the B-spline zoom, projection preparation and the detector-offset gradient
(tests/scene_data_limit_cases.py) without a GPU: each sits where it claims, with the limits read from the CUDA sources;
the scene tile kernel's record search, with its midpoint read from the source and run in 32-bit arithmetic, never
probes outside the record list, at the largest list the API accepts included; and the C ABI refuses one size past the
zoom's and the preparation's limits before any CUDA call."""
import bisect
import ctypes as C

import numpy as np
import pytest

import scene_data_limit_cases as sl
from r2_gaussian_b200 import _lib


def test_limits_are_read_from_the_sources():
    k = sl.K
    assert (k["R2X_SV_TILE"], k["R2X_SV_MAX_SIDE"]) == (16, 16384)
    assert (k["SV_TILE_CTAS"], k["SV_SCAN_THREADS"], k["SV_MAX_GRID"]) == (4096, 1024, 65535)
    assert (k["ZOOM_MAX_DIM"], k["ZOOM_PAD"]) == (32768, 12)
    assert (k["kThreads"], k["kMaxBlocks"], k["kPerBlock"]) == (256, 1024, 2048)


def test_every_case_claims_something_and_fits_one_h100():
    for case in sl.ALL_CASES.values():
        assert case.claims and case.boundary, case.name
        assert 0 < case.peak <= 60 * sl.GiB, (case.name, case.peak / sl.GiB)


@pytest.mark.parametrize("name", sorted(sl.ALL_CASES))
def test_case_lands_where_it_claims(name):
    case = sl.ALL_CASES[name]
    assert sl.claim_failures(case) == [], (case.boundary, sl.claim_failures(case))


# ---- the scene tile search in 32-bit arithmetic ----------------------------------------------------------------------

def test_int32_evaluator_wraps_like_the_gpu():
    assert sl.eval_int32("(lo + hi + 1) >> 1", {"lo": 2**30, "hi": 2**30}) == -(2**30) + 0
    assert sl.eval_int32("lo + hi", {"lo": 2**31 - 1, "hi": 1}) == -(2**31)
    assert sl.eval_int32("-7 / 2", {}) == -3 and sl.eval_int32("x >> 1", {"x": -3}) == -2
    with pytest.raises(ValueError):
        sl.eval_int32("(long long)lo", {"lo": 1})


def test_tile_search_midpoint_is_an_upper_middle_for_small_lists():
    """For every lo < hi below 200 the midpoint lies in (lo, hi] and halves the range as (lo + hi + 1) / 2 does, and
    the search finds bisect's record for every tile of lists with mixed tile counts."""
    mid = sl.tile_search_midpoint()
    for lo in range(200):
        for hi in range(lo + 1, 200):
            assert sl.eval_int32(mid, {"lo": lo, "hi": hi}) == (lo + hi + 1) // 2, (lo, hi)
    rng = np.random.default_rng(3)
    for n in (1, 2, 3, 17, 1000):
        counts = rng.integers(1, 40, n)
        base = np.concatenate([[0], np.cumsum(counts)[:-1]]).tolist()
        for t in range(int(counts.sum())):
            r, probes = sl.tile_search(n, t, base.__getitem__, mid)
            assert r == bisect.bisect_right(base, t) - 1, (n, t)
            assert all(0 <= p < n for p in probes)


def test_tile_search_stays_in_the_record_list_past_2_30_records():
    """The records case (two tiles per record, more than 2^30 records) and the largest list the API accepts
    (n_prims n_frames = 2^31 - 1): every probe of the searches for the tiles at the end of the list, where lo + hi
    passes INT_MAX, and at the first record where it does, stays in [0, nrec) and finds the right record."""
    mid = sl.tile_search_midpoint()
    n_case = sl.quantity(sl.SCENE_CASES["scene_records_past_2_30"], "n_records")
    for nrec in (n_case, sl.INT_MAX):
        tiles = 2 * nrec
        first_wrap = 2**31 - nrec          # the first record r with r + (nrec - 1) + 1 > INT_MAX
        for t in (0, 1, nrec, 2 * first_wrap - 1, 2 * first_wrap, 2 * first_wrap + 3, tiles - 3, tiles - 2,
                  tiles - 1):
            r, probes = sl.tile_search(nrec, t, lambda i: 2 * i, mid)
            assert r is not None, (nrec, t, [p for p in probes if not 0 <= p < nrec][:1])
            assert r == t // 2 and all(0 <= p < nrec for p in probes), (nrec, t)
        # the worst step: lo and hi on the last two records
        assert sl.eval_int32(mid, {"lo": nrec - 2, "hi": nrec - 1}) == nrec - 1


# ---- refusals before any CUDA work -----------------------------------------------------------------------------------

FAKE = C.c_void_p(1 << 20)    # never dereferenced: every call below is refused first


def _desc(src_shape, shape):
    d = _lib.PlaceDesc()
    d.src, d.dtype = FAKE.value, 2
    for a in range(3):
        d.src_shape[a], d.src_strides[a], d.shape[a], d.offset[a] = src_shape[a], 1, shape[a], 0
    d.lo, d.hi = 0.0, 1.0
    return d


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_zoom_refuses_one_past_zoom_max_dim(axis):
    lib = _lib.load()
    M = sl.K["ZOOM_MAX_DIM"]
    ok, over = [1, 2, 3], [1, 2, 3]
    ok[axis], over[axis] = M, M + 1
    assert lib.r2x_zoom_workspace_bytes(*ok) == 8 * np.prod([n + 2 * sl.K["ZOOM_PAD"] for n in ok])
    assert lib.r2x_zoom_workspace_bytes(*over) == 0
    rc = lib.r2x_zoom_cubic(None, C.byref(_desc(over, over)), 2, 2, 2, FAKE, C.c_size_t(2**40), FAKE)
    assert rc == 1 and b"bad placed shape" in lib.r2x_last_error(), lib.r2x_last_error()
    rc = lib.r2x_zoom_cubic(None, C.byref(_desc(ok, ok)), *over, FAKE, C.c_size_t(2**40), FAKE)
    assert rc == 1 and b"bad output shape" in lib.r2x_last_error(), lib.r2x_last_error()
    rc = lib.r2x_volume_place(None, C.byref(_desc(over, over)), FAKE)
    assert rc == 1 and b"bad placed shape" in lib.r2x_last_error(), lib.r2x_last_error()


def test_prepare_shape_accepts_just_under_2_31_pixels_and_refuses_2_31():
    lib = _lib.load()
    hw = (C.c_int * 2)()
    assert 46340 * 46341 < 2**31 <= 46341 * 46341
    assert lib.r2x_projection_prepare_shape(46340, 46341, 1, hw) == 0 and tuple(hw) == (46340, 46341)
    assert lib.r2x_projection_prepare_shape(46341, 46340, 1, hw) == 0 and tuple(hw) == (46341, 46340)
    assert lib.r2x_projection_prepare_shape(46341, 46341, 1, hw) == 1
    assert b"H * W must be < 2^31" in lib.r2x_last_error()
    rc = lib.r2x_projection_prepare(None, 1, 46341, 46341, 1, FAKE, C.c_double(400.0), C.c_double(50.0), FAKE)
    assert rc == 1 and b"H * W must be < 2^31" in lib.r2x_last_error()


def test_grad_sum_closed_form():
    for N in (0, 1, 4092, 4093, 4094, 3 * 4093 + 17, 100_000):
        assert sl.grad_sum_units(N) == sum(i % sl.GRAD_MOD for i in range(N)), N
