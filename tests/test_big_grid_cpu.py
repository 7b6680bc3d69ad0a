"""The cases of tests/big_grid_cases.py land where they claim, on the CPU: their tile counts and sort passes (read from
the CUDA sources), the key buffer that ends up holding the sorted ids, the flat indices inside the judged windows, the
library's size queries, the clouds as the CPU oracle's preprocess places them, and a stated peak that covers every
buffer the GPU test allocates."""
import functools

import numpy as np
import pytest

import big_grid_cases as bg
import binning_limit_cases as blc
import regime_cases as rc
from r2_gaussian_b200 import _lib

K = bg.K
CASES = bg.CASES
GRIDS = [n for n, c in CASES.items() if c.kind != "tv"]


@pytest.mark.parametrize("name", list(CASES))
def test_case_lands_on_its_side(name):
    case = CASES[name]
    n, T = case.n, case.T
    assert n > 2 ** 31, name
    for label, f in case.sites.items():
        assert 0 <= f < n, (name, label)
        if label.startswith("2^"):
            assert f == 1 << int(label[2:]) and n > f
    if case.kind == "tv":
        assert case.shape == CASES["voxel_past_2_31"].shape
        for label, box in bg.tv_windows(case).items():
            lo, hi = case.flat_range(box)
            assert all(b - a >= 1 for a, b in box) and lo <= hi, (label, box)
        lo, hi = case.flat_range(bg.tv_windows(case)["2^31"])
        assert lo < 2 ** 31 <= hi
        return
    assert T == case.expect["T"], (name, T)
    passes = bg.sort_passes(T)
    assert passes == case.expect["passes"], (name, passes)
    # four passes: keys[0] -> [1] -> [0] -> [1] -> [0]; three: the sorted ids end in keys[1]
    assert bg.sorted_buffer(T) == passes % 2 == (0 if passes == 4 else 1)
    if passes == 4:
        assert T > bg.FOURTH_DIGIT and {bg.FOURTH_DIGIT - 1, bg.FOURTH_DIGIT} <= set(case.judged_tiles())
    # every site and the element before it lie in judged tiles, whose boxes hold them
    for label, f in case.sites.items():
        for g in (f, f - 1) if f > 0 else (f,):
            t = case.tile_of(g)
            assert t in case.judged_tiles(), (name, label)
            lo, hi = case.flat_range(case.tile_box(t))
            assert lo <= g <= hi, (name, label, lo, g, hi)
    assert case.tile_of(n - 1) == T - 1 and case.tile_of(0) == 0
    if case.kind == "voxel":
        assert rc.binning_path(case.shape) == "radix"
        assert all(v % 8 != 0 for v in case.shape), "every axis ends on a partial tile"
        assert max(case.grid) <= K["VOXEL_G_MAX"][0] and T <= K["VOXEL_T_MAX"]
    elif case.kind == "raster":
        H, W = case.shape
        assert W % blc.TILE and H % blc.TILE and case.grid[0] == K["RASTER_GX_MAX"]
    else:
        N, H, W = case.shape
        assert blc.views_ok(case.P, N, W, H) and blc.views_path(N, H, W) == "radix"
        per = H * W
        assert bg.judged_views(case) == sorted({0, 2 ** 31 // per, 2 ** 32 // per, N // 3, N - 1})
        # pixels 2^31 and 2^32 fall inside a view's image, not on a view boundary
        assert all(0 < (1 << p) % per for p in (31, 32)) and W % blc.TILE
    print(f"\n{name}: {n} elements, T={T}, {passes} sort passes (sorted ids in keys[{bg.sorted_buffer(T)}]), "
          f"{bg.plan_sweeps(T)} plan sweeps")


def test_size_queries_accept_every_shape():
    lib = _lib.load()
    for name, case in CASES.items():
        if case.kind == "voxel":
            b = lib.r2x_voxel_image_bytes(1000, *case.shape)
            assert b >= case.T * 8, name
            assert lib.r2x_voxel_geom_bytes(1000) > 0
        elif case.kind == "raster":
            H, W = case.shape
            assert lib.r2x_raster_image_bytes(1000, W, H) >= case.T * 8, name
        elif case.kind == "views":
            N, H, W = case.shape
            assert lib.r2x_raster_views_image_bytes(case.P, N, W, H) >= case.T * 8, name
            assert lib.r2x_raster_views_geom_bytes(case.P, N) > 0, name
        else:
            assert lib.r2x_tv3d_scratch_bytes(*case.shape) >= (case.n + 255) // 256 * 4, name


def _cloud_and_pre(case):
    if case.kind == "voxel":
        cloud = bg.voxel_cloud(case)
        return cloud, bg.oracle_voxel_preprocess(cloud, bg.voxel_grid(case))
    cloud, view = bg.raster_cloud(case)
    return cloud, bg.oracle_raster_preprocess(cloud, view)


@pytest.mark.parametrize("name", [n for n in GRIDS if CASES[n].kind != "views"])
def test_cloud_lands_in_its_tiles(name):
    """Every Gaussian touches exactly the tile it was placed in (the oracle's preprocess), the crowded tile holds
    several work-plan chunks, and the predicted ranges are those of the placements."""
    case = CASES[name]
    cloud, pre = _cloud_and_pre(case)
    assert np.all(pre["tiles_touched"] == 1), f"{name}: {int((pre['tiles_touched'] != 1).sum())} Gaussians off"
    tiles, gids = bg.predicted_keys(case, pre)
    assert len(tiles) == pre["R"] == cloud.P
    np.testing.assert_array_equal(np.sort(tiles), np.sort(case.placements()))
    counts = np.bincount(tiles, minlength=case.T)
    C = blc.chunk_of("voxel" if case.kind == "voxel" else "raster", pre["R"])
    assert counts[case.crowded_tile()] == bg.CROWD > 2 * C
    assert all(counts[t] >= 1 for t in case.judged_tiles())
    rg = bg.predicted_ranges(case.T, tiles)
    assert rg[-1, 1] == pre["R"] and rg[0, 0] == 0
    print(f"\n{name}: P={cloud.P}, crowded tile {case.crowded_tile()}: {bg.CROWD} instances = "
          f"{-(-bg.CROWD // C)} chunks of {C}; judged tiles {case.judged_tiles()}")


@functools.lru_cache(maxsize=None)
def _views_instances(name):
    case = CASES[name]
    cloud, views = bg.views_scene(case)
    R, per_view = 0, {}
    for v, view in enumerate(views):
        pre = bg.oracle_raster_preprocess(cloud, view)
        R += pre["R"]
        per_view[v] = pre["R"]
    return cloud, R, per_view


def test_views_case_renders_every_judged_view():
    case = CASES["views_four_passes"]
    cloud, R, per_view = _views_instances(case.name)
    assert cloud.P == case.P
    for v in bg.judged_views(case):
        assert per_view[v] > 0, v
    # the instances of the last views carry tile ids past 2^24: the fourth sort pass has a digit to sort
    N = case.shape[0]
    assert (N - 1) * case.T // N >= bg.FOURTH_DIGIT
    print(f"\nviews_four_passes: R={R} instances over {case.shape[0]} views")


@pytest.mark.parametrize("name", list(CASES))
def test_peak_covers_the_buffers(name):
    case = CASES[name]
    if case.kind == "tv":
        P = R = 0
    elif case.kind == "views":
        _, R, _ = _views_instances(case.name)
        P = case.P
    else:
        cloud, pre = _cloud_and_pre(case)
        P, R = cloud.P, pre["R"]
    buf = bg.device_buffers(case, P, R)
    total = sum(buf.values())
    print(f"\n{name}: buffers {total / bg.GiB:.2f} GiB of the stated {case.peak / bg.GiB:.2f} GiB: "
          + ", ".join(f"{k} {v / bg.GiB:.3f}" for k, v in buf.items()))
    assert total <= case.peak, name
    assert case.peak <= 48 * bg.GiB, "each case must fit an 80 GB card with room for others"


def test_dl_field_is_one_function_on_host_and_device():
    torch = pytest.importorskip("torch")
    start = 2 ** 33 - 1000
    t = torch.empty(5000, dtype=torch.float32)
    bg.dl_fill(t, seed=7, start=start)
    want = bg.dl_host(np.arange(start, start + 5000), 7)
    assert np.array_equal(t.numpy().view(np.uint32), want.view(np.uint32))
    assert want.min() >= -1.0 and want.max() < 1.0 and len(np.unique(want)) > 4000
    f = bg.FlatField((3, 2 ** 20, 2 ** 13 + 1), 7)
    got = f[slice(2, 3), slice(5, 9), slice(100, 103)]
    idx = (2 * 2 ** 20 + np.arange(5, 9)[:, None]) * (2 ** 13 + 1) + np.arange(100, 103)[None, :]
    assert np.array_equal(got[0], bg.dl_host(idx, 7).astype(np.float64))
