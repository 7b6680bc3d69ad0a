"""The TV (prox, value, Chambolle-Pock step), volume-render and marching-cubes kernels on the GPU at their launch limits
and past 2^31 elements (tests/ct_limit_cases.py) against the float64 oracles.

Volumes too large for the host are compared in windows of whole TV tiles plus the stencil's halo (sound by
tests/test_ct_limits_cpu.py): the first tile, the last (holding the far faces) and the tiles around each flat index
whose 32-bit form would wrap.  Renders are compared frame by frame, or row by row, against separate single-camera calls
bit for bit and against the float64 oracle on chosen pixels.  Meshes are counted independently in torch and compared
slab by slab with mesh_oracle bit for bit.  Before each big case the free device memory is compared with the case's
peak; a case that does not fit is skipped with both numbers.  Each case prints its peak memory and wall time."""
import contextlib
import gc
import math
import time

import numpy as np
import pytest

import cp_tv_oracle as cpo
import ct_limit_cases as cl
import mesh_oracle as mo
import tv_oracle as tvo
import volume_render_oracle as vo

pytestmark = pytest.mark.gpu

STEP_BOUND = 1e-5      # CP step: max error over max |want|, as tests/test_cp_tv_gpu.py
PROX_BOUND = 1e-5      # TV prox: max error over max |want|, as tests/test_ct_edges_gpu.py
VALUE_BOUND = 1e-6     # TV value, relative, as tests/test_ct_edges_gpu.py
RENDER_TOL = 1e-4      # volume render: per channel, as _compare in tests/test_volume_render_gpu.py
WHOLE = 2**23          # grids up to this many voxels are compared whole


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
        pytest.skip(f"{case.name}: needs {case.peak / cl.GiB:.1f} GiB, {free / cl.GiB:.1f} GiB free")
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    try:
        yield
    finally:
        torch.cuda.synchronize()
        print(f"[limits] {case.name}: peak {torch.cuda.max_memory_allocated() / cl.GiB:.2f} GiB "
              f"(stated {case.peak / cl.GiB:.2f}), wall {time.perf_counter() - t0:.1f} s")


def _digest(t) -> tuple:
    """(sum, position-weighted sum) of the int32 bits of `t`, in chunks: two runs with equal digests are equal bit for
    bit but for a vanishing chance, without a second copy of an 8-30 GB output."""
    torch = _torch()
    flat = t.reshape(-1).view(torch.int32)
    s0 = s1 = 0
    for k, c in enumerate(flat.split(1 << 24)):
        b = c.to(torch.int64)
        w = torch.arange(c.numel(), device=c.device, dtype=torch.int64) % 65521 + 1 + k
        s0 += int(b.sum())
        s1 += int((b * w).sum())
    return s0, s1


def _bits_equal(a, b) -> bool:
    torch = _torch()
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _windows(case):
    """(label, box) of the case: the whole grid when small, else each site's tile window."""
    shape = case.shape
    if math.prod(shape) <= WHOLE:
        return [("whole", tuple((0, n) for n in shape))]
    return [(label, cl.tile_window(shape, cl.site_index(case, s))) for label, s in case.sites]


def _host(t, box, lead=False):
    sl = ((slice(None),) if lead else ()) + cl.slices(box)
    return t[sl].cpu().numpy()


def _rel_err(got, want) -> float:
    return float(np.abs(np.asarray(got, np.float64) - want).max() / max(np.abs(want).max(), 1e-30))


# ---- TV ---------------------------------------------------------------------------------------------------------------

def _volume(shape, seed, lo, hi):
    torch = _torch()
    gen = torch.Generator("cuda").manual_seed(seed)
    return torch.rand(shape, generator=gen, device="cuda").mul_(hi - lo).add_(lo)


def _cp_inputs(shape, seed):
    torch = _torch()
    nu = cl.CP_PARAMS[2]
    gen = torch.Generator("cuda").manual_seed(seed)
    x = torch.rand(shape, generator=gen, device="cuda").mul_(1.2).sub_(0.2)
    xbar = torch.rand(shape, generator=gen, device="cuda").mul_(0.6).sub_(0.3).add_(x)
    g = torch.randn(shape, generator=gen, device="cuda")
    p = torch.randn((3,) + tuple(shape), generator=gen, device="cuda").mul_(0.7 / nu)
    return x, xbar, p, g


def _check_cp(case, nonneg, seed=1):
    from r2_gaussian_b200.tv import tv_cp_step

    ins = _cp_inputs(case.shape, seed)
    out = tv_cp_step(*ins, *cl.CP_PARAMS, nonneg)
    worst = 0.0
    for label, box in _windows(case):
        outer = cl.grow(box, case.shape, cl.CP_HALO)
        keep = cl.inner(box, outer)
        host = [_host(t, outer, t.dim() == 4) for t in ins]
        want = cpo.cp_step(*host, *cl.CP_PARAMS, nonneg)
        for name, got, w in zip(("x", "xbar", "p"), out, want):
            w = w[((slice(None),) if name == "p" else ()) + keep]
            err = _rel_err(_host(got, box, name == "p"), w)
            worst = max(worst, err)
            assert err <= STEP_BOUND, (case.name, label, name, err)
        if nonneg:
            assert _host(out[0], box).min() >= 0.0
    first = [_digest(t) for t in out]
    del out, got
    again = tv_cp_step(*ins, *cl.CP_PARAMS, nonneg)
    assert [_digest(t) for t in again] == first                                    # bitwise reproducible
    print(f"{case.name} cp nonneg {nonneg}: max err / max = {worst:.3g}")


def _check_prox(case, nonneg, seed=2):
    from r2_gaussian_b200.tv import tv_denoise

    v = _volume(case.shape, seed, -0.3, 1.0)
    out = tv_denoise(v, cl.PROX_WEIGHT, case.niter, nonneg)
    worst = 0.0
    for label, box in _windows(case):
        outer = cl.grow(box, case.shape, cl.prox_halo(case.niter))
        want = tvo.fgp(_host(v, outer), cl.PROX_WEIGHT, case.niter, nonneg)[0][cl.inner(box, outer)]
        err = _rel_err(_host(out, box), want)
        worst = max(worst, err)
        assert err <= PROX_BOUND, (case.name, label, err)
    first = _digest(out)
    del out
    assert _digest(tv_denoise(v, cl.PROX_WEIGHT, case.niter, nonneg)) == first
    print(f"{case.name} prox nonneg {nonneg}: max err / max = {worst:.3g}")


def _tv_value64(x) -> float:
    """TV(x) with every difference and the sum in float64, slab by slab of x-planes in torch on the device."""
    torch = _torch()
    nx, ny, nz = x.shape
    total = torch.zeros((), dtype=torch.float64, device=x.device)
    S = 32
    for a in range(0, nx, S):
        b = min(a + S, nx)
        blk = x[a:min(b + 1, nx)].double()
        n, m = b - a, min(b - a, blk.shape[0] - 1)
        g = torch.zeros((3, n, ny, nz), dtype=torch.float64, device=x.device)
        g[0, :m] = blk[1:m + 1] - blk[:m]
        g[1, :, :-1] = blk[:n, 1:] - blk[:n, :-1]
        g[2, :, :, :-1] = blk[:n, :, 1:] - blk[:n, :, :-1]
        total += g.square_().sum(0).sqrt_().sum()
        del blk, g
    return float(total)


def _check_value(case, seed=3):
    from r2_gaussian_b200.tv import tv_value

    x = _volume(case.shape, seed, 0.0, 1.0)
    got = tv_value(x)
    assert got == tv_value(x)
    want = tvo.tv_value(x.cpu().numpy()) if math.prod(case.shape) <= WHOLE else _tv_value64(x)
    print(f"{case.name} value: {got!r} vs {want!r}")
    if want == 0.0:
        assert got == 0.0
    else:
        assert abs(got - want) <= VALUE_BOUND * want, (got, want)


@pytest.mark.parametrize("name", sorted(n for n, c in cl.TV_CASES.items() if c.kind == "tv"))
def test_tv_kernels_at_the_grid_limits(name):
    case = cl.TV_CASES[name]
    with _budget(case):
        for nonneg in (True, False):
            _check_prox(case, nonneg)
            _check_cp(case, nonneg)
        _check_value(case)


def test_cp_step_with_p_past_2_31():
    case = cl.TV_CASES["cp_p_plane_past_2_31"]
    with _budget(case):
        _check_cp(case, True)


def test_prox_with_scratch_past_2_31():
    case = cl.TV_CASES["prox_scratch_past_2_31"]
    with _budget(case):
        _check_prox(case, True)


def test_tv_value_past_2_31_voxels():
    case = cl.TV_CASES["value_past_2_31"]
    with _budget(case):
        _check_value(case)


# ---- volume rendering ---------------------------------------------------------------------------------------------------

def _render_pixels(case, frame_pixels, out, vol, cams, **kw):
    """Each (frame, flat pixels) of `out` against the float64 oracle on those pixels only."""
    okw = {"unit" if k == "opacity_unit" else k: v for k, v in kw.items()}
    worst = 0.0
    for f, px in frame_pixels:
        want = vo.render_frame(vol, cams[f].record(), case.H, case.W, cams[f].parallel, pixels=px, **okw)
        got = out[f].reshape(-1, 4)[_torch().as_tensor(px, device=out.device)].cpu().numpy().astype(np.float64)
        worst = max(worst, float(np.abs(got - want).max()))
    return worst


@pytest.mark.parametrize("name", ["vr_frames_max", "vr_output_past_2_31"])
def test_volume_render_orbits_at_the_frame_and_index_limits(name):
    from r2_gaussian_b200 import volume_render as vr

    torch = _torch()
    case = cl.VR_CASES[name]
    with _budget(case):
        vol = cl.vr_volume(case)
        vol_d = torch.from_numpy(vol).cuda()
        cams = vr.orbit(cl.vr_camera(case), case.frames)
        out = vr.render(vol_d, cams)
        assert out.shape == (case.frames, case.H, case.W, 4)
        T = cl.K["R2X_VR_TILE"]
        rows = sorted({0, T - 1, T, case.H // 2, case.H - 1} & set(range(case.H)))
        cols = sorted({0, T - 1, T, case.W // 2, case.W - 1} & set(range(case.W)))
        px = sorted({r * case.W + c for r in rows for c in range(case.W)} | {r * case.W + c for r in range(case.H)
                                                                             for c in cols})
        for f in case.sites:
            assert _bits_equal(vr.render(vol_d, cams[f])[0], out[f]), f                # the frame alone, same bits
        err = _render_pixels(case, [(f, px) for f in case.sites], out, vol, cams)
        print(f"{name}: frames {case.sites}, max err {err:.3g}")
        assert err <= RENDER_TOL, err
        first = _digest(out)
        del out
        assert _digest(vr.render(vol_d, cams)) == first


@pytest.mark.parametrize("name", ["vr_rows_max", "vr_cols_max"])
def test_volume_render_at_the_tile_grid_limit(name):
    from r2_gaussian_b200 import volume_render as vr

    torch = _torch()
    case = cl.VR_CASES[name]
    with _budget(case):
        vol = cl.vr_volume(case)
        vol_d = torch.from_numpy(vol).cuda()
        cam = cl.vr_camera(case)
        out = vr.render(vol_d, cam)
        assert _bits_equal(out, vr.render(vol_d, cam))
        if case.extra["axis"] == "rows":
            px = [r * case.W + c for r in case.sites for c in range(case.W)]
        else:
            px = [r * case.W + c for c in case.sites for r in range(case.H)]
        err = _render_pixels(case, [(0, px)], out, vol, [cam])
        alpha = out[..., 3]
        print(f"{name}: {case.extra['axis']} {case.sites}, max err {err:.3g}, alpha in [{float(alpha.min()):.3g}, "
              f"{float(alpha.max()):.3g}]")
        assert err <= RENDER_TOL, err
        assert float(alpha.max()) > 0.05                                           # the rays meet the volume


def test_volume_render_rays_of_1e5_samples():
    """The float32 compositing of n samples against float64.  Per sample: exp2f is within 2 ulp, so 1 - alpha, in
    [1/2, 1], is off by at most 2^-23 absolute (2^-22 relative); T *= (1 - alpha), T alpha, the colour product and
    C += each round once (2^-24).  Over n samples T drifts by n (2^-22 + 2^-24) relative and C by
    sum_k T_k |d alpha_k| + n 2^-24 + (1 - T) n (2^-22 + 2^-24) <= n (2^-23 + 2^-24 + 2^-22 + 2^-24) = 8 n 2^-24,
    with colours in [0, 1]."""
    from r2_gaussian_b200 import volume_render as vr

    torch = _torch()
    case = cl.VR_CASES["vr_long_rays"]
    n = cl._Quantities(case)["n_samples"]
    bar = 8.0 * n * 2.0 ** -24
    with _budget(case):
        vol = cl.vr_volume(case)
        cam = cl.vr_camera(case)
        kw = dict(step=case.extra["step"], opacity_unit=case.extra["unit"], background=(0.2, 0.4, 0.6))
        out = vr.render(torch.from_numpy(vol).cuda(), cam, **kw)
        px = list(range(0, case.H * case.W, 5))
        err = _render_pixels(case, [(0, px)], out, vol, [cam], **kw)
        alpha = out[..., 3].cpu().numpy()
        print(f"long rays: {n} samples, max err {err:.3g}, bar {bar:.3g}, alpha in [{alpha.min():.4f}, "
              f"{alpha.max():.4f}]")
        assert err <= bar, (err, bar)
        assert alpha.max() < 1.0 - 16 * cl.K["VR_T_STOP"] and alpha.min() > 0.5         # composited, never stopped


def test_volume_render_stops_on_the_known_sample():
    from r2_gaussian_b200 import volume_render as vr

    torch = _torch()
    case = cl.VR_CASES["vr_stop_known_sample"]
    with _budget(case):
        vol = cl.vr_volume(case)
        cam = cl.vr_camera(case)
        kw = dict(step=case.extra["step"], opacity_unit=case.extra["unit"], background=(0.3, 0.6, 0.9))
        out = vr.render(torch.from_numpy(vol).cuda(), cam, **kw)[0].cpu().numpy().astype(np.float64)
        want = vo.render_frame(vol, cam.record(), case.H, case.W, True, **{"unit" if k == "opacity_unit" else k: v
                                                                         for k, v in kw.items()})
        assert np.abs(out - want).max() <= RENDER_TOL
        e, ks = 1.0 - case.extra["t_stop"], case.extra["k_stop"]
        T = 1.0 - out[..., 3]
        # 1 - alpha in float32 resolves T to 2^-24 / 1.1e-5 = 0.5 %; the neighbouring stops are 1 / e apart (77 %)
        assert np.abs(T / e ** ks - 1.0).max() < 0.02, (T.min(), T.max(), e ** ks)


# ---- marching cubes ---------------------------------------------------------------------------------------------------

def _table():
    import ctypes as C

    from r2_gaussian_b200 import _lib

    ntri = np.zeros(256, np.int32)
    edges = np.zeros((256, 15), np.int8)
    _lib.check(_lib.load().r2x_marching_cubes_table(ntri.ctypes.data_as(C.c_void_p), edges.ctypes.data_as(C.c_void_p)),
               "r2x_marching_cubes_table")
    return ntri


def _near_max_volume(shape, seed=4):
    """A sphere and a tilted half-space (max of their signed distances, level 0) with uniform noise in [-1/2, 1/2) in
    the first and last 3 x-planes, built plane by plane on the device."""
    torch = _torch()
    nx, ny, nz = shape
    gen = torch.Generator("cuda").manual_seed(seed)
    vol = torch.empty(shape, dtype=torch.float32, device="cuda")
    j = torch.arange(ny, device="cuda", dtype=torch.float32)[:, None]
    k = torch.arange(nz, device="cuda", dtype=torch.float32)[None, :]
    c, R = (0.5 * nx + 0.3, 0.5 * ny - 0.7, 0.5 * nz + 0.2), 0.3 * nx
    yz = (j - c[1]) ** 2 + (k - c[2]) ** 2
    for i in range(nx):
        if i < 3 or i >= nx - 3:
            vol[i] = torch.rand((ny, nz), generator=gen, device="cuda") - 0.5
            continue
        sphere = R - torch.sqrt(yz + (i - c[0]) ** 2)
        plane = (0.31 * i + 0.52 * j + 0.79 * k - 1.45 * nx) * 0.5
        vol[i] = torch.maximum(sphere, plane)
    return vol


def _plane_counts(vol, level, ntri_d):
    """Per x-plane: cut edges along x, y, z owned by its samples, and triangles of its cubes (ntri[case] summed), in
    torch on the device, independently of the kernels."""
    torch = _torch()
    nx = vol.shape[0]
    cuts = torch.zeros((nx, 3), dtype=torch.int64, device=vol.device)
    tris = torch.zeros(nx, dtype=torch.int64, device=vol.device)
    cur = vol[0] > level
    for i in range(nx):
        cuts[i, 1] = (cur[1:] != cur[:-1]).sum()
        cuts[i, 2] = (cur[:, 1:] != cur[:, :-1]).sum()
        if i + 1 < nx:
            nxt = vol[i + 1] > level
            cuts[i, 0] = (nxt != cur).sum()
            pl = (cur.to(torch.int32), nxt.to(torch.int32))
            ny, nz = cur.shape
            case = torch.zeros((ny - 1, nz - 1), dtype=torch.int32, device=vol.device)
            for b, (dx, dy, dz) in enumerate(mo.CORNERS):
                case |= pl[dx][dy:ny - 1 + dy, dz:nz - 1 + dz] << b
            tris[i] = ntri_d[case.long()].sum()
            cur = nxt
    return cuts.cpu().numpy(), tris.cpu().numpy()


def test_marching_cubes_just_under_the_sample_limit():
    from r2_gaussian_b200 import mesh

    torch = _torch()
    case = cl.MC_CASES["mc_near_max"]
    level = 0.0
    with _budget(case):
        vol = _near_max_volume(case.shape)
        verts, faces = mesh.marching_cubes(vol, level)
        cuts, tris = _plane_counts(vol, level, torch.from_numpy(_table().astype(np.int64)).cuda())
        nv = cuts.sum(1)
        print(f"mc_near_max: {len(verts)} vertices ({cuts.sum(0).tolist()} per axis), {len(faces)} triangles")
        assert len(verts) == nv.sum() and len(faces) == tris.sum()
        assert cuts[-1, 0] == 0 and (cuts[:3].sum() > 0) and (cuts[-3:].sum() > 0)
        cv, ct = np.concatenate([[0], np.cumsum(nv)]), np.concatenate([[0], np.cumsum(tris)])
        for a, b in case.sites:
            sv, st = cl.slab_mesh(vol[a:b + 1].cpu().numpy(), level, a, b)
            gv = verts[cv[a]:cv[b]].cpu().numpy()
            gt = verts[faces[ct[a]:ct[b]].long()].cpu().numpy()
            assert len(sv) == cv[b] - cv[a] and len(st) == ct[b] - ct[a], (a, b)
            assert np.array_equal(gv.view(np.uint32), sv.view(np.uint32)), (a, b)
            assert np.array_equal(gt.view(np.uint32), st.view(np.uint32)), (a, b)
        again = mesh.marching_cubes(vol, level)
        assert _bits_equal(again[0], verts) and torch.equal(again[1], faces)


def _line_values(n: int) -> dict:
    """Sample -> value of the long lines (0 elsewhere, level 1/2): runs at the start, around 2^30, around
    2^31 - 2^20, in the last (31-sample) word and on the last sample."""
    w = 32 * (n // 32)
    runs = {0: (0.9, 0.7), 2**30 - 1: (0.8,), 2**31 - 2**20 - 1: (1.3, 0.6, 2.0), w - 1: (0.75,), w + 3: (3.0, 0.55),
            n - 1: (0.9,)}
    return {s + d: v for s, vals in runs.items() for d, v in enumerate(vals)}


@pytest.mark.parametrize("name", sorted(n for n in cl.MC_CASES if n.startswith("mc_line")))
def test_marching_cubes_on_lines_of_2_31_minus_1_samples(name):
    from r2_gaussian_b200 import mesh

    torch = _torch()
    case = cl.MC_CASES[name]
    n = math.prod(case.shape)
    axis = int(np.argmax(case.shape))
    vals = _line_values(n)
    with _budget(case):
        vol = torch.zeros(case.shape, dtype=torch.float32, device="cuda")
        idx = sorted(vals)
        vol.view(-1)[torch.tensor(idx, device="cuda")] = torch.tensor([vals[i] for i in idx], device="cuda")
        verts, faces = mesh.marching_cubes(vol, 0.5)
        # the closed form: a vertex on each edge (t, t + 1) with one end above 1/2, at float32(t) + f in float32
        lv = np.float32(0.5)
        want = []
        for t in sorted({i - 1 for i in idx if i > 0} | set(idx)):
            if t + 1 >= n:
                continue
            a, b = np.float32(vals.get(t, 0.0)), np.float32(vals.get(t + 1, 0.0))
            if (a > lv) != (b > lv):
                p = np.zeros(3, np.float32)
                p[axis] = np.float32(t) + (lv - a) / (b - a)
                want.append(p)
        want = np.asarray(want, np.float32)
        got = verts.cpu().numpy()
        print(f"{name}: {len(got)} vertices, {len(faces)} triangles")
        assert len(faces) == 0 and got.shape == want.shape
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
