"""The inputs of tests/binning_limit_cases.py land where they claim (judged by the CPU oracle's forward for single views
and voxel grids, by the restated views_shape for batched views), and the entry points accept a grid at each size limit
and refuse one step past it, before any CUDA call."""
import ctypes

import pytest

import binning_limit_cases as blc
from r2_gaussian_b200 import _lib

K = blc.K
CASES = {c.name: c for c in blc.all_cases()}


def test_limits_are_read_from_the_sources():
    assert K["SORT_CHUNK"] == K["SORT_THREADS"] * K["SORT_ITEMS"] and K["SORT_MAX_BLOCKS"] > 1
    assert K["PLAN_THREADS"] * K["PLAN_RUN"] > K["DIRECT_MAX_TILES"]
    # the per-axis tile limits are CUDA's grid y / z limit (the render grids put tile rows there)
    assert K["VIEWS_GX_MAX"] == K["VIEWS_ROWS_MAX"] == blc.GRID_YZ_MAX
    assert K["RASTER_GX_MAX"] == K["RASTER_GY_MAX"] == blc.GRID_YZ_MAX
    assert K["VOXEL_G_MAX"] == (blc.GRID_YZ_MAX,) * 3 and K["VOXEL_T_MAX"] == K["VIEWS_T_MAX"] == 1 << 30
    assert blc.GRID_YZ_MAX <= blc.UINT16_MAX    # every end coordinate fits the uint16 cube
    assert K["VIEWS_PV_MAX"] == 2 ** 31 - 1


def test_restated_sort_passes_and_sweeps():
    B = 2 ** K["SORT_BITS"]
    assert [blc.sort_passes(T) for T in (2, B, B + 1, B * B, B * B + 1, B ** 3, B ** 3 + 1)] == [1, 1, 2, 2, 3, 3, 4]
    S = K["PLAN_THREADS"] * K["PLAN_RUN"]
    assert [blc.plan_sweeps(T) for T in (1, S, S + 1, 2 * S, 2 * S + 1)] == [1, 1, 2, 2, 3]
    assert blc.sort_chunks_per_cta(K["SORT_CHUNK"] - 1, 1 << 14) == 1
    assert blc.sort_chunks_per_cta(K["SORT_CHUNK"] * K["SORT_MAX_BLOCKS"] + 1, 1 << 22) == 2


def test_the_radix_path_never_takes_a_single_pass():
    """The radix path starts above DIRECT_MAX_TILES tiles, which needs more than SORT_BITS bits: the first-and-last
    scatter instantiation cannot run.  A DIRECT_MAX_TILES below 2^SORT_BITS would make it reachable, untested."""
    assert K["DIRECT_MAX_TILES"] >= 2 ** K["SORT_BITS"]
    assert blc.sort_passes(K["DIRECT_MAX_TILES"] + 1) >= 2


@pytest.mark.parametrize("name", list(CASES))
def test_case_lands_on_its_side(name):
    case = CASES[name]
    orc = None
    if case.kind == "raster":
        cloud, view = case.make()
        orc = blc.oracle(case, cloud, view)
    elif case.kind == "voxel":
        orc = blc.oracle(case, case.make())
    lines = blc.check_case(case, orc)
    print(f"\n{name}:\n  " + "\n  ".join(lines))


def test_every_boundary_has_a_case():
    """Three passes (single view, voxel, views), a grid at each per-axis limit, both sides of the direct / radix switch
    of the stacked views, and crowded tiles on a thread-run and a sweep boundary and at T - 1."""
    ex = {n: c.expect for n, c in CASES.items()}
    for kind in ("raster", "voxel", "views"):
        assert any(c.kind == kind and c.expect.get("passes") == 3 for c in CASES.values()), kind
    assert {"x1", "z1"} <= {a for e in ex.values() for a, v in e.get("cube_max", {}).items() if v == blc.UINT16_MAX}
    assert {("direct", K["DIRECT_MAX_TILES"]), ("radix", K["DIRECT_MAX_TILES"] + 1)} <= {
        (c.path, c.T) for c in CASES.values() if c.kind == "views"}
    kinds = {w for e in ex.values() for _, _, w in e.get("straddle", [])}
    assert kinds == set(blc.STRADDLE_UNIT)
    assert any(c.T - 1 in c.expect.get("crowded", {}) and c.path == "radix" for c in CASES.values())
    assert {c.expect.get("sort") for c in CASES.values()} >= {"one_cta", "multi_chunk"}
    for c in CASES.values():
        assert 0 < c.mem_gb <= 4.0, c.name


# ---- the entry points' limits, through the library on the CPU ----------------------------------------------------------
def _lib_handle():
    return _lib.load()


FAKE = ctypes.c_void_p(1 << 20)   # never dereferenced: every call below fails its checks first


def _views_fwd(lib, P, N, W, H):
    return lib.r2x_raster_forward_views_async(None, P, N, W, H, FAKE, FAKE, FAKE, 1.0, FAKE, FAKE, FAKE, 1.0, 1.0, 1, FAKE,
                                              FAKE, FAKE, FAKE, FAKE, 1 << 20, None)


def _views_limits():
    """(name, (P, N, W, H) at the limit, the same one step past it, what the refusal says)."""
    T = blc.TILE
    rows, gxm, pv, tm = K["VIEWS_ROWS_MAX"], K["VIEWS_GX_MAX"], K["VIEWS_PV_MAX"], K["VIEWS_T_MAX"]
    Pp = 1 << 16                                      # N * Pp reaches the Gaussian limit before the row limit
    n_pv = pv // Pp
    gx_t = tm // (1 << 15)                            # gx * N = 2^30 with N = 2^15 rows
    return [
        ("rows", (10, rows, T, T), (10, rows + 1, T, T), b"tile rows"),
        ("rows_gy2", (10, rows // 2, T, 2 * T), (10, rows // 2 + 1, T, 2 * T), b"tile rows"),
        ("gx", (10, 1, gxm * T, T), (10, 1, gxm * T + 1, T), b"tile rows"),
        ("gaussians", (Pp, n_pv, T, T), (Pp, n_pv + 1, T, T), b"views x Gaussians"),
        ("gaussians_P", (pv // rows // 256 * 256, rows, T, T), (pv // rows // 256 * 256 + 1, rows, T, T),
         b"views x Gaussians"),
        ("tiles", (10, 1 << 15, gx_t * T, T), (10, (1 << 15) + 1, gx_t * T, T), b"tiles"),
    ]


@pytest.mark.parametrize("name,at,past,msg", _views_limits(), ids=[x[0] for x in _views_limits()])
def test_views_shape_limits_exactly(name, at, past, msg):
    """r2x_raster_views_geom_bytes / _image_bytes are non-zero at each views_shape limit and 0 one step past it; the
    asynchronous forward refuses the step past by name."""
    lib = _lib_handle()
    assert blc.views_ok(*at) and not blc.views_ok(*past)
    P, N, W, H = at
    assert lib.r2x_raster_views_image_bytes(P, N, W, H) > 0 and lib.r2x_raster_views_geom_bytes(P, N) > 0, at
    P, N, W, H = past
    assert lib.r2x_raster_views_image_bytes(P, N, W, H) == 0, past
    if name in ("gaussians", "gaussians_P"):
        assert lib.r2x_raster_views_geom_bytes(P, N) == 0, past
    assert _views_fwd(lib, P, N, W, H) != 0
    err = lib.r2x_last_error()
    assert b"r2x_raster_forward_views_async" in err and msg in err, err


def test_single_view_and_voxel_refuse_one_tile_past_65535():
    lib = _lib_handle()
    T, V = blc.TILE, blc.VTILE
    gm = K["RASTER_GX_MAX"]
    for W, H in (((gm + 1) * T, T), (T, (gm + 1) * T), (gm * T + 1, T)):
        rc = lib.r2x_raster_forward_async(None, 10, W, H, FAKE, FAKE, FAKE, 1.0, FAKE, None, FAKE, FAKE, FAKE, 1.0, 1.0,
                                          0, 1, FAKE, FAKE, FAKE, FAKE, FAKE, 1 << 20, None)
        assert rc != 0 and b"detector too large" in lib.r2x_last_error(), (W, H)
    vm = K["VOXEL_G_MAX"][2]
    for n in ((V, V, (vm + 1) * V), (V, V, vm * V + 1), ((vm + 1) * V, V, V)):
        rc = lib.r2x_voxel_forward_async(None, 10, *n, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0, FAKE, FAKE, FAKE, 1.0, FAKE, None, 0,
                                         FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, 1 << 20, None)
        assert rc != 0 and b"grid too large" in lib.r2x_last_error(), n
    # 2^15 x 2^15 x 2 tiles: every axis within its limit, the tile count past 2^30
    n = (V << 15, V << 15, 2 * V)
    rc = lib.r2x_voxel_forward_async(None, 10, *n, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0, FAKE, FAKE, FAKE, 1.0, FAKE, None, 0,
                                     FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, 1 << 20, None)
    assert rc != 0 and b"too many tiles" in lib.r2x_last_error()
