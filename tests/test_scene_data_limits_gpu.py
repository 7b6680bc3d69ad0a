"""The scene rasterizer, the cubic B-spline zoom, projection preparation and the detector-offset gradient on the GPU at
their launch limits and past 2^31 elements (tests/scene_data_limit_cases.py) against the oracles.

Scene keys are compared bit for bit and colours within 1e-6 with tests/scene_view_oracle.py and
tests/gaussian_view_oracle.py, whole frames where they are small and windows where they are large.  Zooms are compared
within 1e-12 with raw_data_oracle.zoom_box, preparation bit for bit with real_data_oracle.prepare, and the gradient
bit for bit with its closed form.  Before each case the free device memory is compared with the case's peak; a case
that does not fit is skipped with both numbers.  Each case prints its peak memory and wall time."""
import contextlib
import gc
import time

import numpy as np
import pytest

import gaussian_view_oracle as gvo
import raw_data_oracle as zo
import real_data_oracle as ro
import scene_data_limit_cases as sl
import scene_view_oracle as so

pytestmark = pytest.mark.gpu

TOL = 1e-6             # scene colours, as tests/test_scene_view_gpu.py
ZOOM_TOL = 1e-12       # zoom, relative to max(1, max |want|), as tests/test_raw_data_gpu.py


def _torch():
    import torch

    return torch


@contextlib.contextmanager
def _budget(case):
    """Skip unless the case's peak fits in the free device memory; report the peak reached and the wall time."""
    torch = _torch()
    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < case.peak:
        pytest.skip(f"{case.name}: needs {case.peak / sl.GiB:.1f} GiB, {free / sl.GiB:.1f} GiB free")
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    try:
        yield
    finally:
        torch.cuda.synchronize()
        print(f"[limits] {case.name}: peak {torch.cuda.max_memory_allocated() / sl.GiB:.2f} GiB "
              f"(stated {case.peak / sl.GiB:.2f}), wall {time.perf_counter() - t0:.1f} s")


# ---- scene rasterizer ----------------------------------------------------------------------------------------------

def _render(sc: sl.Scene):
    from r2_gaussian_b200 import scene_view as sv

    torch = _torch()
    t = lambda x, dt: torch.as_tensor(np.ascontiguousarray(x), dtype=dt, device="cuda")
    prims = sv.Primitives(t(sc.pos, torch.float64), t(sc.meta, torch.int32), t(sc.attr, torch.float32),
                          t(sc.tex, torch.float32) if sc.textured else None)
    cams = [sc.cams[f % len(sc.cams)] for f in range(sc.frames)]
    return sv.render(prims, cams, background=sl.BG, lut=sl.LUT, near=sl.NEAR, return_keys=True)


def _oracle(sc: sl.Scene, cams, window=None):
    recs = np.stack([c.record() for c in cams])
    return gvo.raster(sc.pos, sc.meta, sc.attr, sc.tex, sl.LUT, recs, sc.H, sc.W, sc.parallel, sl.NEAR, sl.BG, window)


def _check_window(keys, rgb, okeys, orgb, window, what, local=False):
    """Keys bit for bit and colours within TOL on the window; `local`: keys and rgb hold only the window."""
    y0, y1, x0, x1 = window
    k, ok = (keys if local else keys[..., y0:y1, x0:x1]), okeys[..., y0:y1, x0:x1]
    g = rgb if local else rgb[..., y0:y1, x0:x1, :]
    assert np.array_equal(k, ok), (what, window, int((k != ok).sum()))
    err = float(np.abs(g - orgb[..., y0:y1, x0:x1, :]).max())
    assert err <= TOL, (what, window, err)
    return int((k != so.EMPTY).sum())


def test_scene_records_past_2_30_and_tiles_past_2_31():
    """65535 frames of 17000 full-row lines: 1.1e9 records of two tiles.  Every frame equals the oracle's frame of its
    camera; the tiles at the end of the list are found by the record search where lo + hi passes INT_MAX."""
    case = sl.SCENE_CASES["scene_records_past_2_30"]
    sc = case.extra["scene"]()
    with _budget(case):
        rgb, keys = _render(sc)
        k = keys.cpu().numpy().view(np.uint64)
        g = rgb.cpu().numpy()
        del rgb, keys
    okeys, orgb = _oracle(sc, sc.cams)
    which = np.arange(sc.frames) % len(sc.cams)
    bad = np.nonzero((k != okeys[which]).reshape(sc.frames, -1).any(1))[0]
    assert len(bad) == 0, (len(bad), bad[:10].tolist())
    assert float(np.abs(g - orgb[which]).max()) <= TOL
    winners = [len(set((okeys[c] & np.uint64(0xFFFFFFFF)).ravel().tolist())) for c in range(len(sc.cams))]
    assert (okeys != so.EMPTY).all() and min(winners) > sc.W // 2, winners
    assert len({okeys[c].tobytes() for c in range(len(sc.cams))}) == len(sc.cams)     # the frames differ
    print(f"records case: {sc.frames} frames, distinct winners per camera {winners}")


def test_scene_pixels_past_2_31_in_one_call():
    case = sl.SCENE_CASES["scene_pixels_past_2_31"]
    sc = case.extra["scene"]()
    torch = _torch()
    with _budget(case):
        rgb, keys = _render(sc)
        fr = list(case.extra["frames_checked"])
        k = keys[fr].cpu().numpy().view(np.uint64)
        g = rgb[fr].cpu().numpy()
        del rgb, keys
        gc.collect()
        torch.cuda.empty_cache()
    hits = 0
    for win in case.extra["windows"]:
        okeys, orgb = _oracle(sc, [sc.cams[f] for f in fr], win)
        hits += _check_window(k, g, okeys, orgb, win, "frames " + str(fr))
    assert hits > 0
    # the last frame starts at pixel 2^31: it equals the frame rendered alone
    alone_rgb, alone_keys = _render(sl.Scene(sc.pos, sc.meta, sc.attr, sc.tex, [sc.cams[fr[-1]]], 1, sc.textured))
    assert np.array_equal(alone_keys[0].cpu().numpy().view(np.uint64), k[-1])
    assert np.array_equal(alone_rgb[0].cpu().numpy(), g[-1])
    print(f"pixels case: frames {fr}, {hits} covered pixels checked in windows")


def test_scene_one_record_of_a_million_tiles():
    case = sl.SCENE_CASES["scene_one_record_1M_tiles"]
    sc = case.extra["scene"]()
    with _budget(case):
        rgb, keys = _render(sc)
        ids = set()
        for win in case.extra["windows"]:
            y0, y1, x0, x1 = win
            k = keys[:, y0:y1, x0:x1].cpu().numpy().view(np.uint64)
            g = rgb[:, y0:y1, x0:x1].cpu().numpy()
            okeys, orgb = _oracle(sc, sc.cams, win)
            assert _check_window(k, g, okeys, orgb, win, "16384^2", local=True) == (y1 - y0) * (x1 - x0)
            ids |= set((k & np.uint64(0xFFFFFFFF)).ravel().tolist())
            del okeys, orgb
    assert ids == {0, 1, 2, 3}, ids
    print(f"one-record case: winners in the windows {sorted(ids)}")


def test_scene_scan_of_many_passes():
    case = sl.SCENE_CASES["scene_scan_many_passes"]
    sc = case.extra["scene"]()
    with _budget(case):
        rgb, keys = _render(sc)
        k = keys.cpu().numpy().view(np.uint64)
        g = rgb.cpu().numpy()
    okeys, orgb = _oracle(sc, sc.cams)
    n = _check_window(k, g, okeys, orgb, (0, sc.H, 0, sc.W), "whole frame")
    winners = len(set((okeys & np.uint64(0xFFFFFFFF)).ravel().tolist()))
    print(f"scan case: {sl.quantity(case, 'n_records')} records, {n} covered pixels, {winners} winners")
    assert winners > 1000


# ---- cubic B-spline zoom -------------------------------------------------------------------------------------------

def _zoom_source(case):
    shape = case.extra["src_shape"]
    rng = np.random.default_rng(sum(map(ord, case.name)))
    if case.extra.get("lo") is None:
        return rng.random(shape)
    # uint8, laid out z-major: the view [x, y, z] has strides (ny, 1, nx ny)
    nx, ny, nz = shape
    base = np.frombuffer(bytearray(rng.bytes(nx * ny * nz)), np.uint8).reshape(nz, nx, ny)
    return base.transpose(1, 2, 0)


def _placed_get(case, src):
    """get(i0, i1, i2) of zoom_box: the placed, normalised source at placed indices."""
    ex = case.extra
    if ex.get("lo") is None:
        return lambda i0, i1, i2: src[np.ix_(i0, i1, i2)]
    off = ex["offset"]
    lo, hi = ex["lo"], ex["hi"]

    def get(*idx):
        q = [np.asarray(i) - o for i, o in zip(idx, off)]
        inside = [(v >= 0) & (v < n) for v, n in zip(q, src.shape)]
        out = np.zeros(tuple(len(v) for v in q))
        sub = [v[m] for v, m in zip(q, inside)]
        if all(len(s) for s in sub):
            out[np.ix_(*inside)] = (src[np.ix_(*sub)].astype(np.float64) - lo) / (hi - lo)
        return out

    return get


@pytest.mark.parametrize("name", sorted(sl.ZOOM_CASES))
def test_zoom_at_its_limits(name):
    from r2_gaussian_b200.resample import Place, zoom_placed

    torch = _torch()
    case = sl.ZOOM_CASES[name]
    ex = case.extra
    src = _zoom_source(case)
    placed = sl.quantity(case, "placed")
    place = Place(placed, ex.get("offset", (0, 0, 0)), ex.get("lo") or 0.0, ex.get("hi") or 1.0)
    get = _placed_get(case, src)
    with _budget(case):
        dev = src if ex.get("lo") is not None else torch.from_numpy(src).cuda()
        out = zoom_placed(dev, ex["factors"], place)
        assert tuple(out.shape) == sl.quantity(case, "out")
        worst = 0.0
        for label, box in ex["windows"] or (("whole", None),):
            sl_ = tuple(slice(lo, hi) for lo, hi in box) if box else ...
            got = out[sl_].cpu().numpy()
            want = zo.zoom_box(get, placed, ex["factors"], box=box, margin=32 if box else None)
            err = float(np.abs(got - want).max()) / max(1.0, float(np.abs(want).max()))
            worst = max(worst, err)
            assert err <= ZOOM_TOL, (name, label, err)
        del out
    print(f"{name}: out {sl.quantity(case, 'out')}, max err {worst:.3g}")


# ---- projection preparation ----------------------------------------------------------------------------------------

def test_prepare_past_2_31_pixels():
    from r2_gaussian_b200 import generate_real_data as grd

    torch = _torch()
    case = sl.PREPARE_CASES["prepare_past_2_31"]
    ex = case.extra
    n, H0, W0 = ex["n"], ex["H0"], ex["W0"]
    with _budget(case):
        img = torch.empty((n, H0, W0), dtype=torch.float64, device="cuda")
        gen = torch.Generator("cuda").manual_seed(8)
        for a in range(0, n, 60):
            img[a:a + 60].uniform_(-40.0, 400.0, generator=gen)
        out = grd.prepare(img, 1, ex["rescale"], ex["object_scale"])
        for v in ex["views"]:
            want = ro.prepare(img[v].cpu().numpy(), 1, ex["rescale"], ex["object_scale"])
            assert np.array_equal(out[v].cpu().numpy().view(np.uint32), want.view(np.uint32)), ("s1", v)
        del out
        out = grd.prepare(img, 4, ex["rescale"], ex["object_scale"])
        assert tuple(out.shape) == (n,) + sl.quantity(case, "sub4")
        for v in ex["views"]:
            want = ro.prepare(img[v].cpu().numpy(), 4, ex["rescale"], ex["object_scale"])
            assert np.array_equal(out[v].cpu().numpy().view(np.uint32), want.view(np.uint32)), ("s4", v)
    print(f"prepare: {n} x {H0} x {W0}, views {ex['views']} bit for bit at subsample 1 and 4")


# ---- detector-offset gradient --------------------------------------------------------------------------------------

def test_detector_offset_grad_past_2_31_rows():
    from r2_gaussian_b200 import _lib

    torch = _torch()
    case = sl.GRAD_CASES["grad_rows_past_2_31"]
    P, nv, W = case.extra["P"], case.extra["n_views"], case.extra["W"]
    N = P * nv
    with _budget(case):
        g = torch.full((N, 3), 1e30, dtype=torch.float32, device="cuda")
        step = 1 << 27
        for a in range(0, N, step):
            b = min(a + step, N)
            g[a:b, 0] = (torch.arange(a, b, dtype=torch.int64, device="cuda") % sl.GRAD_MOD).to(torch.float32) / 4096.0
        lib = _lib.load()
        nbytes = int(lib.r2x_detector_offset_grad_scratch_bytes(P, nv))
        assert nbytes == 8 * sl.quantity(case, "nb")
        scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        out = torch.empty(1, dtype=torch.float32, device="cuda")
        stream = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.r2x_detector_offset_grad(stream, P, nv, W, g.data_ptr(), out.data_ptr(), scratch.data_ptr(),
                                                nbytes), "r2x_detector_offset_grad")
        got = np.float32(out.item())
        S = sl.grad_sum_units(N) / 4096.0                         # exact: below 2^53 units of 2^-12
        want = np.float32(2.0 / W * S)
        assert got.view(np.uint32) == want.view(np.uint32), (got, want)
        # the float64 partials of the blocks, each the closed-form sum of its chunk
        nb, chunk = sl.quantity(case, "nb"), sl.quantity(case, "chunk")
        part = scratch.view(torch.float64).cpu().numpy()
        for b in (0, nb // 2, nb - 1):
            lo, hi = b * chunk, min((b + 1) * chunk, N)
            assert part[b] == (sl.grad_sum_units(hi) - sl.grad_sum_units(lo)) / 4096.0, b
    print(f"detector grad: N = {N}, {nb} blocks of {chunk}, {got!r}")
