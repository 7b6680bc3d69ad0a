"""The voxelizer past 2^31 and 2^32 voxels, the four-pass radix sort past 2^24 tiles (voxel grid, batched views, one
wide view) and the TV loss past 2^31 voxels (tests/big_grid_cases.py; tests/test_big_grid_cpu.py checks that each case
lands where it claims).

Nothing of these sizes is copied to the host.  Per case:
  * the per-Gaussian stage outputs bit for bit the CPU oracle's preprocess (radii, tiles_touched, positions, depths);
  * the exported tile lists: every key's tile, in order, that of the instances the oracle's cubes / rectangles predict,
    the key multiset, the ranges (empty tiles empty) and point_list ascending in Gaussian id within each tile -- the
    direct check of which ping-pong buffer a sort of 3 or 4 passes leaves the ids in;
  * every element of every tile a Gaussian reaches against the float64 statement of forward_float64.py at the bars of
    test_forward_float64_gpu.py, and every other element exactly 0 (counted on the device, slab by slab);
  * the backward against grad_float64 at the bars of test_grad_float64_gpu.py, with dL a seeded function of the flat
    index written on the device (big_grid_cases.dl_fill) and read back only at the Gaussians' tiles; the four-pass
    voxel grid has room for one volume only, so dL overwrites the volume after its checks;
  * two runs bitwise equal, by a device-side digest.
Batched views are held to test_views_gpu.py's statement over all views; voxel_past_2_31 also runs through query() and
autograd, bit for bit the C entry points, and a forward of no Gaussian must zero its whole volume.  Before each case the free device memory is compared with the case's stated
peak, and a case that does not fit is skipped with both numbers; each case prints its peak and wall time."""
import contextlib
import gc
import time
import types

import numpy as np
import pytest

import big_grid_cases as bg
import forward_float64 as f64
import grad_float64 as g64
import train_edge_cases as te
import util

torch = pytest.importorskip("torch")

from r2_gaussian_b200 import _C, _lib  # noqa: E402
from r2_gaussian_b200.render_query import query  # noqa: E402
from test_grad_float64_cpu import voxel_judge  # noqa: E402
from test_grad_float64_gpu import _judge as raster_judge  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = bg.CASES
GiB = bg.GiB
VOXEL_GRADS = ("dL_dopacity", "dL_dmean3D", "dL_dcov3D", "dL_dscale", "dL_drot")
RASTER_GRADS = ("dL_dmean2D", "dL_dopacity", "dL_dmu", "dL_dmean3D", "dL_dcov3D", "dL_dscale", "dL_drot")


@contextlib.contextmanager
def _budget(case):
    """Skip unless the case's stated peak fits in the free device memory; report (and hold to it) the peak reached, and
    the wall time."""
    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < case.peak:
        pytest.skip(f"{case.name}: needs {case.peak / GiB:.1f} GiB, {free / GiB:.1f} GiB free")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    try:
        yield
    finally:
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        print(f"\n[big grid] {case.name}: peak {peak / GiB:.2f} GiB (stated {case.peak / GiB:.2f}), "
              f"wall {time.perf_counter() - t0:.1f} s")
    assert peak <= case.peak, f"{case.name}: peak {peak / GiB:.2f} GiB over the stated {case.peak / GiB:.2f}"


# ---- device-side helpers ------------------------------------------------------------------------------------------------
def _digest(t) -> tuple:
    """(sum, position-weighted sum) of the int32 bits of t, slab by slab on the device."""
    flat = t.reshape(-1).view(torch.int32)
    s0 = torch.zeros((), dtype=torch.int64, device=t.device)
    s1 = torch.zeros((), dtype=torch.int64, device=t.device)
    for k, c in enumerate(flat.split(bg.SLAB)):
        b = c.to(torch.int64)
        s0 += b.sum()
        s1 += (b * (torch.arange(c.numel(), device=c.device, dtype=torch.int64) % 65521 + 1 + k)).sum()
        del b
    return int(s0), int(s1)


def _count_nonzero(t) -> int:
    n = torch.zeros((), dtype=torch.int64, device=t.device)
    for c in t.reshape(-1).split(bg.SLAB):
        n += torch.count_nonzero(c)
    return int(n)


def _boxes(case, tiles) -> dict:
    """{tile: (box, flat indices [box shape])} of tile boxes, in the output's array layout."""
    out = {}
    for t in tiles:
        box = case.tile_box(int(t))
        axes = [np.arange(a, b) for a, b in box]
        idx = np.zeros([len(a) for a in axes], np.int64)
        for d, a in enumerate(axes):
            sh = [1] * len(axes)
            sh[d] = len(a)
            idx = idx * case.shape[d] + a.reshape(sh)
        out[int(t)] = (box, idx)
    return out


def _gather(t, boxes) -> dict:
    """The elements of each box, one device gather for all of them."""
    flat = np.concatenate([idx.reshape(-1) for _, idx in boxes.values()])
    vals = t.reshape(-1)[torch.from_numpy(flat).to(t.device)].cpu().numpy()
    out, o = {}, 0
    for k, (_, idx) in boxes.items():
        out[k] = vals[o:o + idx.size].reshape(idx.shape)
        o += idx.size
    return out


def _bits(a):
    return a.contiguous().view(torch.int32)


def _judge_tiles(label, case, blocks, statement):
    """Every element of every block within its float64 bar (forward_float64.ratio <= 1), an element no pair reaches
    exactly 0, and in every block at least one element reached; returns the number of judged elements."""
    worst, judged_n = 0.0, 0
    for t, block in blocks.items():
        st = statement(t)
        got = np.asarray(block, np.float64)
        judged = f64.judged(st)
        assert judged.any(), f"{label}: tile {t} holds Gaussians, yet no element reaches the alpha cut"
        assert np.all(got[~judged] == 0.0), f"{label}: tile {t}: an element no pair reaches is not 0"
        r = f64.ratio(got, st)[judged]
        assert np.isfinite(r).all() and r.max(initial=0.0) <= 1.0, f"{label}: tile {t}: worst {r.max():.3g} x bar"
        worst = max(worst, float(r.max(initial=0.0)))
        judged_n += int(judged.sum())
    print(f"  {label}: {len(blocks)} tiles, {judged_n} elements judged against float64, worst {worst:.3g} x bar")
    return judged_n


def _check_lists(case, ex, pre, R):
    """The exported keys, ranges and point_list against the instances the oracle's cubes / rectangles predict."""
    tiles, gids = bg.predicted_keys(case, pre)
    assert int(R) == len(tiles) == pre["R"], (int(R), len(tiles))
    keys = ex["keys"].astype(np.uint64)
    np.testing.assert_array_equal((keys >> np.uint64(32)).astype(np.int64), tiles, err_msg="key tiles in sorted order")
    want = (tiles.astype(np.uint64) << np.uint64(32)) | pre["depth"][gids].view(np.uint32).astype(np.uint64)
    assert util.key_multiset_equal(keys, want)
    np.testing.assert_array_equal(ex["ranges"], bg.predicted_ranges(case.T, tiles))
    # (tile, id) order: within each tile ascending in Gaussian id, as the stable sort promises
    np.testing.assert_array_equal(ex["point_list"].astype(np.int64), gids)
    return tiles


# ---- voxel grids ----------------------------------------------------------------------------------------------------------
def _voxel_forward(t, grid):
    nV, sV, ctr = grid
    return _C.voxelize_gaussians(t["means"], t["dens"], t["scales"], t["rots"], 1.0, torch.Tensor([]), *nV, *sV, *ctr,
                                 False, False)


def _voxel_backward(t, grid, fw, dL):
    nV, sV, ctr = grid
    R, _, rx, ry, rz, geom, binning, img = fw
    g = _C.voxelize_gaussians_backward(t["means"], rx, ry, rz, t["scales"], t["rots"], 1.0, torch.Tensor([]), dL, geom,
                                       R, binning, img, *nV, *sV, *ctr, False)
    return dict(zip(VOXEL_GRADS, g))


def _voxel_statement(ex, nV, case):
    """forward_float64.voxel_statement of one tile, on a one-tile grid: positions shifted by the tile's origin (exact in
    float64), so that no array of the whole grid is allocated."""
    def st(t):
        box = case.tile_box(t)
        a, b = (int(v) for v in ex["ranges"][t])
        xyz = ex["xyz_vol"].astype(np.float64) - np.array([lo for lo, _ in box], np.float64)
        return f64.voxel_statement(xyz, ex["conic_opacity"], np.array([[0, b - a]], np.uint32),
                                   ex["point_list"][a:b], tuple(hi - lo for lo, hi in box))
    return st


@pytest.mark.parametrize("name", [n for n, c in CASES.items() if c.kind == "voxel"])
def test_voxel_case(name):
    case = CASES[name]
    with _budget(case):
        cloud, grid = bg.voxel_cloud(case), bg.voxel_grid(case)
        nV = grid[0]
        pre = bg.oracle_voxel_preprocess(cloud, grid)
        t = util.to_torch(cloud, None)
        fw = _voxel_forward(t, grid)
        R, vol = fw[0], fw[1]
        ex = util.voxel_export(cloud.P, nV, R, *fw[5:])
        for k, r in zip(("radii_x", "radii_y", "radii_z"), fw[2:5]):
            ex[k] = r.cpu().numpy()
            np.testing.assert_array_equal(ex[k], pre[k], err_msg=k)
        np.testing.assert_array_equal(ex["tiles_touched"], pre["tiles_touched"])
        for k in ("xyz_vol", "depth"):
            np.testing.assert_array_equal(ex[k].view(np.uint32), pre[k].view(np.uint32), err_msg=k)
        np.testing.assert_allclose(ex["conic_opacity"], pre["conic_opacity"], rtol=2e-6, atol=0)
        tiles = _check_lists(case, ex, pre, R)
        occupied = np.unique(tiles)
        assert set(case.judged_tiles()) <= set(occupied.tolist())
        boxes = _boxes(case, occupied)
        blocks = _gather(vol, boxes)
        _judge_tiles(name, case, blocks, _voxel_statement(ex, nV, case))
        inside = sum(int(np.count_nonzero(b)) for b in blocks.values())
        assert _count_nonzero(vol) == inside, f"{name}: a voxel outside every Gaussian's tile is not 0"
        d0 = _digest(vol)
        print(f"  {name}: R={int(R)}, {len(occupied)} occupied tiles of {case.T}, {inside} non-zero voxels")

        seed = case.seed
        if case.one_buffer:                       # no room for a second volume: run again, then overwrite with dL
            del vol, fw, blocks
            gc.collect()
            fw = _voxel_forward(t, grid)
            assert int(fw[0]) == int(R) and _digest(fw[1]) == d0, f"{name}: two forwards differ"
            dL = fw[1]
        else:
            dL = torch.empty(tuple(nV), dtype=torch.float32, device="cuda")
        bg.dl_fill(dL, seed)
        g = _voxel_backward(t, grid, fw, dL)
        g2 = _voxel_backward(t, grid, fw, dL)
        for k in VOXEL_GRADS:
            assert torch.equal(_bits(g[k]), _bits(g2[k])), f"{name}: {k}: two backwards differ"
        got = {k: v.cpu().numpy() for k, v in g.items()}
        ratio, idx, ill, _ = voxel_judge(cloud, grid, ex, bg.FlatField(nV, seed), got)
        assert len(idx) >= 0.9 * cloud.P and np.isfinite(ratio).all()
        worst = {k: float(v.max()) for k, v in g64.voxel_split(ratio).items()}
        print(f"  {name} backward: {len(idx)} Gaussians against float64 ({ill} ill-conditioned), worst x bar: "
              + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
        assert max(worst.values()) <= 1.0, worst

        if not case.one_buffer:
            del fw, vol
            gc.collect()
            if case.python_path:
                _python_path(name, cloud, grid, dL, d0, g)
                _empty_forward(name, grid, dL)
            else:
                fw = _voxel_forward(t, grid)
                assert int(fw[0]) == int(R) and _digest(fw[1]) == d0, f"{name}: two forwards differ"


def _empty_forward(name, grid, out):
    """A forward of no Gaussian (forward_empty) into a volume that holds dL: every voxel must come back 0."""
    nV, sV, ctr = grid
    lib = _lib.load()
    assert _count_nonzero(out) > 0
    u8 = lambda n: torch.empty(max(int(n), 1024), dtype=torch.uint8, device=out.device)   # noqa: E731
    geom, img = u8(lib.r2x_voxel_geom_bytes(0)), u8(lib.r2x_voxel_image_bytes(0, *nV))
    rc = lib.r2x_voxel_forward_async(torch.cuda.current_stream().cuda_stream, 0, *nV, *sV, *ctr, None, None, None, 1.0,
                                     None, None, 0, out.data_ptr(), None, None, None, geom.data_ptr(), img.data_ptr(),
                                     None, 0, None)
    _lib.check(rc, "r2x_voxel_forward_async")
    assert _count_nonzero(out) == 0, f"{name}: the forward of no Gaussian left non-zero voxels"
    print(f"  {name}: the forward of no Gaussian zeroes all {out.numel()} voxels")


def _python_path(name, cloud, grid, dL, d0, g):
    """query() and autograd: the volume's digest and the gradients bit for bit those of the C entry points."""
    nV, sV, ctr = grid
    tg = util.to_torch(cloud, None, requires_grad=True)
    pc = types.SimpleNamespace(get_xyz=tg["means"], get_density=tg["dens"], get_scaling=tg["scales"],
                               get_rotation=tg["rots"])
    pipe = types.SimpleNamespace(debug=False, compute_cov3D_python=False)
    vol = query(pc, ctr, nV, sV, pipe)["vol"]
    assert tuple(vol.shape) == tuple(nV) and _digest(vol.detach()) == d0, f"{name}: query() differs from the C call"
    vol.backward(dL)
    for k, p in (("dL_dopacity", "dens"), ("dL_dmean3D", "means"), ("dL_dscale", "scales"), ("dL_drot", "rots")):
        assert torch.equal(_bits(tg[p].grad.reshape(g[k].shape)), _bits(g[k])), f"{name}: autograd {p}.grad"
    print(f"  {name}: query() + autograd bit for bit the C entry points")


# ---- one wide view ----------------------------------------------------------------------------------------------------------
def _raster_forward(t, view):
    return _C.rasterize_gaussians(t["means"], t["dens"], t["scales"], t["rots"], 1.0, torch.Tensor([]), t["view"],
                                  t["proj"], view.tanfovx, view.tanfovy, view.image_height, view.image_width, t["campos"],
                                  False, view.mode, False)


def _raster_statement(ex, case):
    def st(t):
        (y0, y1), (x0, x1) = case.tile_box(t)
        a, b = (int(v) for v in ex["ranges"][t])
        xy = ex["xy"].astype(np.float64) - np.array([x0, y0], np.float64)
        return f64.raster_statement(xy, ex["conic_opacity"], ex["mu"], np.array([[0, b - a]], np.uint32),
                                    ex["point_list"][a:b], x1 - x0, y1 - y0, "kernel")
    return st


def test_raster_four_passes():
    case = CASES["raster_four_passes"]
    H, W = case.shape
    with _budget(case):
        cloud, view = bg.raster_cloud(case)
        pre = bg.oracle_raster_preprocess(cloud, view)
        t = util.to_torch(cloud, view)
        fw = _raster_forward(t, view)
        R, image, radii = fw[0], fw[1][0], fw[2]
        ex = util.raster_export(cloud.P, W, H, R, *fw[3:])
        ex["radii"] = radii.cpu().numpy()
        np.testing.assert_array_equal(ex["radii"], pre["radii"])
        np.testing.assert_array_equal(ex["tiles_touched"], pre["tiles_touched"])
        vis = pre["radii"] > 0
        for k in ("depth", "xy", "conic_opacity", "mu"):
            np.testing.assert_array_equal(ex[k][vis].view(np.uint32), pre[k][vis].view(np.uint32), err_msg=k)
        tiles = _check_lists(case, ex, pre, R)
        occupied = np.unique(tiles)
        assert set(case.judged_tiles()) <= set(occupied.tolist())
        blocks = _gather(image, _boxes(case, occupied))
        _judge_tiles("raster_four_passes", case, blocks, _raster_statement(ex, case))
        inside = sum(int(np.count_nonzero(b)) for b in blocks.values())
        assert _count_nonzero(image) == inside, "a pixel outside every Gaussian's tile is not 0"
        d0 = _digest(image)
        print(f"  raster_four_passes: R={int(R)}, {len(occupied)} occupied tiles of {case.T}")

        dL = torch.empty((1, H, W), dtype=torch.float32, device="cuda")
        bg.dl_fill(dL, case.seed)
        args = (t["means"], radii, t["scales"], t["rots"], 1.0, torch.Tensor([]), t["view"], t["proj"], view.tanfovx,
                view.tanfovy, dL, t["campos"], fw[3], R, fw[4], fw[5], view.mode, False)
        g = dict(zip(RASTER_GRADS, _C.rasterize_gaussians_backward(*args)))
        g2 = dict(zip(RASTER_GRADS, _C.rasterize_gaussians_backward(*args)))
        for k in RASTER_GRADS:
            assert torch.equal(_bits(g[k]), _bits(g2[k])), f"{k}: two backwards differ"
        got = {k: v.cpu().numpy() for k, v in g.items()}
        raster_judge("raster_four_passes backward", got, ex, view, cloud, bg.FlatField((H, W), case.seed))

        del fw, image, radii
        gc.collect()
        fw = _raster_forward(t, view)
        assert int(fw[0]) == int(R) and _digest(fw[1]) == d0, "two forwards differ"


# ---- batched views ----------------------------------------------------------------------------------------------------
def test_views_four_passes():
    """Every view's image, radii and dL/dmean2D bit for bit its single-view call, the per-Gaussian gradients the
    view-order float32 sum of the single-view backwards (test_views_gpu.py), the judged views' radii bit for bit the
    oracle's preprocess, and two batched calls bitwise equal."""
    import test_views_gpu as tvg

    case = CASES["views_four_passes"]
    N, H, W = case.shape
    with _budget(case):
        cloud, views = bg.views_scene(case)
        t = tvg._inputs(cloud, views)
        dL = torch.empty((N, H, W), dtype=torch.float32, device="cuda")
        bg.dl_fill(dL, case.seed)
        b = tvg._batched(t, views, dL)
        judged = bg.judged_views(case)
        for v in judged:
            pre = bg.oracle_raster_preprocess(cloud, views[v])
            np.testing.assert_array_equal(b["radii"][v].cpu().numpy(), pre["radii"], err_msg=f"view {v}")
            assert int((pre["radii"] > 0).sum()) > 0 and float(b["images"][v].abs().max()) > 0, f"view {v}"
        mism = torch.zeros((), dtype=torch.int64, device="cuda")
        acc = None
        keys = ("opacity", "mean3D", "cov3D", "scale", "rot")
        for v, view in enumerate(views):
            s = tvg._single(t, view, v, dL)
            if v in judged:
                assert tvg._bit_equal(b["images"][v], s["image"]), f"view {v}: image"
                assert b["radii"][v].equal(s["radii"]), f"view {v}: radii"
                assert tvg._bit_equal(b["mean2D"][v], s["mean2D"]), f"view {v}: dL/dmean2D"
            mism += (_bits(b["images"][v]) != _bits(s["image"])).sum() + (b["radii"][v] != s["radii"]).sum()
            mism += (_bits(b["mean2D"][v]) != _bits(s["mean2D"])).sum()
            acc = {k: s[k].clone() for k in keys} if acc is None else {k: acc[k] + s[k] for k in keys}
        assert int(mism) == 0, f"{int(mism)} elements of the batched images / radii / dL/dmean2D differ from the views'"
        for k in keys:
            assert tvg._bit_equal(b[k], acc[k]), f"{k}: not the view-ordered float32 sum of the single-view gradients"
        d0 = _digest(b["images"])
        grads = {k: b[k] for k in keys + ("mean2D",)}
        R = b["R"]
        del b, acc
        gc.collect()
        again = tvg._batched(t, views, dL)
        assert again["R"] == R and _digest(again["images"]) == d0, "two batched forwards differ"
        for k, x in grads.items():
            assert tvg._bit_equal(again[k], x), f"{k}: two batched backwards differ"
        print(f"  views_four_passes: R={R}, views {judged} against the oracle, all {N} against single-view calls")


# ---- TV ---------------------------------------------------------------------------------------------------------------------
def _tv_volume(shape, seed):
    """tv_volume's distribution (exact plateaus at 0 and 0.5), generated on the device slab by slab."""
    vol = torch.empty(shape, dtype=torch.float32, device="cuda")
    flat = vol.view(-1)
    for k, c in enumerate(flat.split(bg.SLAB)):
        gen = torch.Generator("cuda").manual_seed(seed * 1000 + k)
        u = torch.rand(c.numel(), generator=gen, device="cuda")
        r = torch.rand(c.numel(), generator=gen, device="cuda")
        c.copy_(u * 1.3 - 0.3)
        c[r < 1 / 3] = 0.0
        c[(r >= 1 / 3) & (r < 0.5)] = 0.5
        del u, r
    return vol


def _tv_sum_f64(vol, planes=24) -> float:
    """sum of |differences| along the three axes in float64, x-slab by x-slab (each slab with the next plane)."""
    nx = vol.shape[0]
    s = torch.zeros((), dtype=torch.float64, device=vol.device)
    for a in range(0, nx, planes):
        b = min(nx, a + planes)
        blk = vol[a:min(nx, b + 1)].double()
        s += (blk[1:] - blk[:-1]).abs().sum()
        core = blk[: b - a]
        s += (core[:, 1:] - core[:, :-1]).abs().sum() + (core[:, :, 1:] - core[:, :, :-1]).abs().sum()
        del blk, core
    return float(s)


def test_tv3d_past_2_31():
    """r2x_tv3d_loss (mean): the loss within 1e-6 of a float64 sum (each CTA's float32 partial adds at most 16 levels
    of terms of one sign: 16.5 u < 1e-6), the gradient bit for bit the integer sign statement in windows around flat
    index 2^31, the plane and row boundaries nearest it and the first and last voxel, and two calls bitwise equal."""
    case = CASES["tv3d_past_2_31"]
    nx, ny, nz = case.shape
    L = _lib
    lib = L.load()
    with _budget(case):
        vol = _tv_volume(case.shape, case.seed)
        nb = lib.r2x_tv3d_scratch_bytes(nx, ny, nz)
        scratch = torch.empty(nb, dtype=torch.uint8, device="cuda")
        out = torch.full((2,), -1.0, device="cuda")
        g = torch.empty_like(vol)
        st = torch.cuda.current_stream().cuda_stream

        def run(o, grad):
            L.check(lib.r2x_tv3d_loss(st, nx, ny, nz, vol.data_ptr(), 1, o, grad, scratch.data_ptr(), nb),
                    "r2x_tv3d_loss")
        run(out.data_ptr(), g.data_ptr())
        tot = (nx - 1) * ny * nz + nx * (ny - 1) * nz + nx * ny * (nz - 1)
        want = _tv_sum_f64(vol) / tot
        got = float(out[0])
        print(f"  tv3d_past_2_31: loss {got:.9g}, float64 {want:.9g}, rel {abs(got - want) / want:.3g}")
        assert abs(got - want) <= 1e-6 * want
        scale = np.float32(1.0 / tot)
        for label, box in bg.tv_windows(case).items():
            hb = bg.halo(box, case.shape)
            blk = vol[tuple(slice(a, b) for a, b in hb)].cpu().numpy()
            exact = (te.tv_grad_exact(blk, False) * scale).astype(np.float32)
            inner = tuple(slice(a - h, b - h) for (a, b), (h, _) in zip(box, hb))
            gw = g[tuple(slice(a, b) for a, b in box)].cpu().numpy()
            assert np.array_equal(gw.view(np.uint32), exact[inner].view(np.uint32)), \
                f"window {label}: {int((gw != exact[inner]).sum())} voxels differ"
        d0 = _digest(g)
        run(out[1:].data_ptr(), g.data_ptr())
        assert _digest(g) == d0 and torch.equal(_bits(out[:1]), _bits(out[1:])), "two calls differ"
        run(out[1:].data_ptr(), None)
        assert torch.equal(_bits(out[:1]), _bits(out[1:])), "the loss without the gradient differs"
