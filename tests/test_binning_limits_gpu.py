"""The binning front-end at its size limits (tests/binning_limit_cases.py; tests/test_binning_limits_cpu.py checks that
each case lands where it claims): three-pass sorts, multi-sweep work plans, tile coordinates of 65535 and the batched-view
grid at its limits.

Single views and voxel grids are compared against the CPU oracle at the bars of test_regimes_gpu.py: radii,
tiles_touched, the exported key multiset, ranges and point_list bit for bit, the image / volume within 1e-5 of its scale
(crowded tiles against a float64 sum), and the backward, which on the radix path reads inst_pos (written by the last
sort pass only).  The two-level voxel binning must give the radix path's volume and gradients bit for bit.  Batched
views are held to test_views_gpu.py's statement: each image, radii and per-view dL/dmean2D bit for bit the single-view
call's, the summed gradients the view-order float32 sum, and two runs bitwise equal."""
import time

import numpy as np
import pytest
import torch

import binning_limit_cases as blc
import test_regimes_gpu as trg
import test_views_gpu as tvg
import util
from r2_gaussian_b200 import _lib

pytestmark = pytest.mark.gpu

CASES = {c.name: c for c in blc.all_cases()}
RASTER = [n for n, c in CASES.items() if c.kind == "raster"]
VOXEL = [n for n, c in CASES.items() if c.kind == "voxel"]
VIEWS = [n for n, c in CASES.items() if c.kind == "views"]
# batched views checked forward only, on views_subset (every other one forward and backward, on every view)
FORWARD_SUBSET = {"views_65535x32x16"}


class _Report:
    """Wall time and torch's peak device memory of one case, printed, and the peak held to the case's estimate."""

    def __init__(self, case):
        self.case = case

    def __enter__(self):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        self.base = torch.cuda.memory_allocated()     # what earlier tests' cached workspaces still hold
        self.t0 = time.perf_counter()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - self.base
        print(f"\n{self.case.name}: {time.perf_counter() - self.t0:.1f} s, peak device memory {peak / 2 ** 30:.2f} GiB "
              f"above the {self.base / 2 ** 30:.2f} GiB held before it (estimate {self.case.mem_gb} GiB)")
        if exc[0] is None:
            assert peak <= self.case.mem_gb * 2 ** 30, f"{self.case.name}: {peak / 2 ** 30:.2f} GiB"
        return False


@pytest.mark.parametrize("name", RASTER)
def test_raster_case(name):
    case = CASES[name]
    with _Report(case):
        cloud, view = case.make()
        orc = trg._raster_both(cloud, view, crowded=tuple(case.expect.get("crowded", {})))
        print("  " + "\n  ".join(blc.check_case(case, orc)))


def _voxel_pair(case, cloud, monkeypatch, binning, seed=11):
    if binning:
        monkeypatch.setenv("R2X_VOXEL_BINNING", binning)
    else:
        monkeypatch.delenv("R2X_VOXEL_BINNING", raising=False)
    nV, sV, ctr = case.grid
    ours = util.ours_voxel_forward(cloud, nV, sV, ctr)
    dL = np.random.RandomState(seed).randn(*nV).astype(np.float32)
    return ours, dL, util.ours_voxel_backward(cloud, nV, sV, ctr, ours, dL)


@pytest.mark.parametrize("name", VOXEL)
def test_voxel_case(name, monkeypatch):
    case = CASES[name]
    with _Report(case):
        cloud = case.make()
        nV, sV, ctr = case.grid
        ours, dL, g = _voxel_pair(case, cloud, monkeypatch, case.binning)
        orc = util.oracle_voxel_forward(cloud, nV, sV, ctr)
        trg.assert_voxel_forward(ours, orc, nV, crowded=tuple(case.expect.get("crowded", {})))
        go = util.oracle_voxel_backward(cloud, nV, sV, orc, dL)
        util.assert_grads_close(g, go, trg.VOXEL_GRADS)
        print("  " + "\n  ".join(blc.check_case(case, orc)))


def test_two_level_equals_radix_bit_for_bit(monkeypatch):
    """The same grid of 35937 tiles through two-level binning and through the radix sort: the same tile lists, so the
    same volume and gradients, bit for bit."""
    two, radix = (CASES[n] for n in ("voxel_264cube", "voxel_264cube_radix"))
    assert two.path == "two_level" and radix.path == "radix" and two.shape == radix.shape
    cloud = two.make()
    a, dL, ga = _voxel_pair(two, cloud, monkeypatch, "")
    b, _, gb = _voxel_pair(radix, cloud, monkeypatch, "radix")
    assert a["R"] == b["R"] > 0
    np.testing.assert_array_equal(a["ranges"], b["ranges"])
    np.testing.assert_array_equal(a["point_list"], b["point_list"])
    np.testing.assert_array_equal(a["vol"].view(np.uint32), b["vol"].view(np.uint32))
    for k in trg.VOXEL_GRADS:
        np.testing.assert_array_equal(ga[k].view(np.uint32), gb[k].view(np.uint32), err_msg=k)


def _views_forward_subset(cloud, views, subset):
    t = tvg._inputs(cloud, views)
    b = tvg._batched(t, views)
    for v in subset:
        s = tvg._single(t, views[v], v)
        assert tvg._bit_equal(b["images"][v], s["image"]), f"view {v}: image differs from the single-view render"
        assert b["radii"][v].equal(s["radii"]), f"view {v}: radii differ"
    assert b["R"] > 0
    return t, b


@pytest.mark.parametrize("name", VIEWS)
def test_views_case(name):
    case = CASES[name]
    with _Report(case):
        cloud, views = case.make()
        N = len(views)
        assert N == case.shape[0]
        if name in FORWARD_SUBSET:
            subset = blc.views_subset(N, case.T // N)
            print(f"  views checked one by one: {subset}")
            t, b = _views_forward_subset(cloud, views, subset)
            # every view in the subset renders something, so the tile ids it checks are in use
            assert all(float(b["images"][v].abs().max()) > 0 for v in subset)
            again = tvg._batched(t, views)
            for k in ("images", "radii"):
                assert tvg._bit_equal(b[k], again[k]), k
        else:
            b = tvg._check_backward(cloud, views, seed=len(name))
            assert b["R"] > 0
            t = tvg._inputs(cloud, views)
            dL = tvg._dL(views, len(name))
            again = tvg._batched(t, views, dL)
            for k in ("images", "radii", "mean2D", "opacity", "mean3D", "cov3D", "scale", "rot"):
                assert tvg._bit_equal(b[k], again[k]), f"{k}: two runs differ"
        print("  " + "\n  ".join(blc.check_case(case)))


def test_refusals_before_any_launch():
    """One tile past each per-axis limit is refused by return code, with real device buffers, and leaves the device
    without an error."""
    lib = _lib.load()
    T, V = blc.TILE, blc.VTILE
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    torch.cuda.synchronize()
    W = (blc.K["RASTER_GX_MAX"] + 1) * T
    rc = lib.r2x_raster_forward_async(None, 10, W, T, p, p, p, 1.0, p, None, p, p, p, 1.0, 1.0, 0, 1, p, p, p, p, p,
                                      1 << 10, None)
    assert rc != 0 and b"detector too large" in lib.r2x_last_error()
    nz = (blc.K["VOXEL_G_MAX"][2] + 1) * V
    rc = lib.r2x_voxel_forward_async(None, 10, V, V, nz, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0, p, p, p, 1.0, p, None, 0, p, p, p,
                                     p, p, p, p, 1 << 10, None)
    assert rc != 0 and b"grid too large" in lib.r2x_last_error()
    N = blc.K["VIEWS_ROWS_MAX"] + 1
    rc = lib.r2x_raster_forward_views_async(None, 10, N, T, T, p, p, p, 1.0, p, p, p, 1.0, 1.0, 1, p, p, p, p, p, 1 << 10,
                                            None)
    assert rc != 0 and b"tile rows" in lib.r2x_last_error()
    torch.cuda.synchronize()
    assert int(buf.sum()) == 0, "a refused call wrote to its buffers"
