"""The limit cases of the TV, volume-render and marching-cubes kernels (tests/ct_limit_cases.py) without a GPU: each
sits where it claims, with the limits read from the CUDA sources; the C ABI refuses every out-of-range size, sizes
within one tile of INT_MAX included, before any CUDA call; and every windowed comparison tests/test_ct_limits_gpu.py
makes is sound: the float64 oracles on a window plus its halo give the full grid's result on the window."""
import ctypes as C
import itertools

import numpy as np
import pytest

import cp_tv_oracle as cpo
import ct_limit_cases as cl
import mesh_oracle as mo
import tv_oracle as tvo
import volume_render_oracle as vo
from r2_gaussian_b200 import _lib


def test_limits_are_read_from_the_sources():
    k = cl.K
    assert (k["TV_TX"], k["TV_TY"], k["TV_TZ"], k["TVV_PER_BLOCK"], k["TVV_MAX_BLOCKS"]) == (4, 8, 32, 2048, 1024)
    assert (k["R2X_VR_TILE"], k["VR_MAX_GRID"], k["VR_MAX_LUT"], k["VR_T_STOP"]) == (16, 65535, 4096, 2.0 ** -16)
    assert (k["MC_THREADS"], k["MC_WORDS"], k["MC_CLASSIFY_WORDS"], k["MC_MAX_SAMPLES"]) == (256, 8, 4, 2**31 - 1)
    assert all(isinstance(k[n], int) for n in k if n != "VR_T_STOP")


def test_every_case_claims_something_and_fits_one_h100():
    for case in cl.ALL_CASES.values():
        assert case.claims and case.boundary, case.name
        if not case.kind.startswith("refuse"):
            assert 0 < case.peak <= 40 * cl.GiB, (case.name, case.peak / cl.GiB)


@pytest.mark.parametrize("name", sorted(cl.ALL_CASES))
def test_case_lands_where_it_claims(name):
    case = cl.ALL_CASES[name]
    assert cl.claim_failures(case) == [], (case.boundary, cl.claim_failures(case))


@pytest.mark.parametrize("name", sorted(n for n, c in cl.TV_CASES.items() if c.sites))
def test_tv_windows_hold_both_sides_of_each_site(name):
    """A site's window is whole TV tiles (or the grid's end) holding voxels site - 1 and site, small enough to copy."""
    case = cl.TV_CASES[name]
    nx, ny, nz = case.shape
    for label, site in case.sites:
        i = cl.site_index(case, site)
        box = cl.tile_window(case.shape, i)
        for f in (max(i - 1, 0), i):
            ijk = (f // (ny * nz), (f // nz) % ny, f % nz)
            assert all(lo <= c < hi for c, (lo, hi) in zip(ijk, box)), (label, ijk, box)
        for (lo, hi), n, t in zip(box, case.shape, (cl.K["TV_TX"], cl.K["TV_TY"], cl.K["TV_TZ"])):
            assert lo % t == 0 and (hi % t == 0 or hi == n)
        halo = cl.grow(box, case.shape, cl.prox_halo(case.niter))
        assert np.prod([hi - lo for lo, hi in halo]) <= 2**21, (label, halo)


# ---- refusals before any CUDA work ---------------------------------------------------------------------------------

FAKE = C.c_void_p(1 << 20)    # never dereferenced: every call below is refused first


@pytest.mark.parametrize("name", sorted(n for n, c in cl.REFUSALS.items() if c.kind == "refuse_tv"))
def test_tv_abi_refuses_out_of_range_grids(name):
    lib = _lib.load()
    nx, ny, nz = cl.REFUSALS[name].shape
    rc = lib.r2x_tv_prox(None, nx, ny, nz, FAKE, C.c_float(0.1), 3, 1, FAKE, FAKE, C.c_size_t(2**62))
    assert rc == 1 and lib.r2x_last_error().startswith(b"r2x_tv_prox: bad grid"), (rc, lib.r2x_last_error())
    f = [C.c_void_p((1 << 40) + (k << 38)) for k in range(7)]     # disjoint fake buffers
    rc = lib.r2x_tv_cp_step(None, nx, ny, nz, *f[:4], C.c_float(0.3), C.c_float(0.4), C.c_float(0.7), 1, *f[4:])
    assert rc == 1 and lib.r2x_last_error().startswith(b"r2x_tv_cp_step: bad grid"), (rc, lib.r2x_last_error())


@pytest.mark.parametrize("name", sorted(n for n, c in cl.REFUSALS.items() if c.kind == "refuse_vr"))
def test_volume_render_abi_refuses_out_of_range_images(name):
    lib = _lib.load()
    case = cl.REFUSALS[name]
    bg = (C.c_float * 3)(0, 0, 0)
    rc = lib.r2x_volume_render(None, 4, 4, 4, FAKE, case.frames, case.H, case.W, FAKE, 0, 0, C.c_float(0.0),
                               C.c_float(1.0), FAKE, 2, C.c_float(0.5), C.c_float(1.0), bg, FAKE)
    msg = lib.r2x_last_error()
    assert rc == 1 and msg.startswith(b"r2x_volume_render: bad image") and b"65535" in msg, (rc, msg)


@pytest.mark.parametrize("name", sorted(n for n, c in cl.REFUSALS.items() if c.kind == "refuse_mc"))
def test_marching_cubes_abi_refuses_one_sample_past_the_maximum(name):
    lib = _lib.load()
    shape = cl.REFUSALS[name].shape
    assert lib.r2x_marching_cubes_scratch_bytes(*shape) == 0
    rc = lib.r2x_marching_cubes_count(None, *shape, FAKE, C.c_float(0.5), FAKE, FAKE, C.c_size_t(2**40))
    assert rc == 1 and b"2^31 - 1" in lib.r2x_last_error()
    rc = lib.r2x_marching_cubes_emit(None, *shape, FAKE, C.c_float(0.5), 10, 10, FAKE, FAKE, FAKE, C.c_size_t(2**40))
    assert rc == 1 and b"2^31 - 1" in lib.r2x_last_error()
    for case in cl.MC_CASES.values():                                       # the largest grids are accepted
        assert lib.r2x_marching_cubes_scratch_bytes(*case.shape) > 0


# ---- the windowed comparisons are sound ----------------------------------------------------------------------------

SMALL = (13, 19, 70)          # 4 x 3 x 3 TV tiles, none of them whole along x, z


def _boxes(shape):
    """Windows of whole tiles: the first tile, the last (holding the far faces), interior ones, and boxes around flat
    indices that cross a y row and an x plane."""
    nx, ny, nz = shape
    nvox = nx * ny * nz
    flats = [0, nvox - 1, nvox // 2 + 7, ny * nz * 5, nz * 9, nz * 9 + 40, ny * nz * 3 + nz * 17 + 33]
    return [cl.tile_window(shape, f) for f in flats]


def _cp_inputs(shape, seed):
    rng = np.random.RandomState(seed)
    tau, sigma, nu = cl.CP_PARAMS
    x = rng.uniform(-0.2, 1.0, shape)
    xbar = x + rng.uniform(-0.3, 0.3, shape)
    g = rng.normal(0.0, 1.0, shape)
    p = rng.normal(0.0, 0.7, (3,) + shape) / nu
    return x, xbar, p, g


def _cp_window(ins, box, halo, nonneg):
    shape = ins[0].shape
    outer = cl.grow(box, shape, halo)
    sl = cl.slices(outer)
    x, xbar, p, g = (a[(slice(None),) + sl] if a.ndim == 4 else a[sl] for a in ins)
    got = cpo.cp_step(x, xbar, p, g, *cl.CP_PARAMS, nonneg)
    keep = cl.inner(box, outer)
    return got[0][keep], got[1][keep], got[2][(slice(None),) + keep]


@pytest.mark.parametrize("nonneg", [True, False])
def test_cp_step_on_a_window_plus_halo_is_the_full_step(nonneg):
    ins = _cp_inputs(SMALL, 3)
    full = cpo.cp_step(*ins, *cl.CP_PARAMS, nonneg)
    narrower = 0
    for box in _boxes(SMALL):
        want = (full[0][cl.slices(box)], full[1][cl.slices(box)], full[2][(slice(None),) + cl.slices(box)])
        for a, b in zip(_cp_window(ins, box, cl.CP_HALO, nonneg), want):
            assert np.array_equal(a, b), box
        # the halo is needed: without it a window that does not reach a grid face differs
        short = _cp_window(ins, box, cl.CP_HALO - 1, nonneg)
        narrower += any(not np.array_equal(a, b) for a, b in zip(short, want))
    assert narrower > 0


@pytest.mark.parametrize("niter", [2, 3])
def test_prox_on_a_window_plus_halo_is_the_full_prox(niter):
    v = np.random.RandomState(niter).uniform(-0.3, 1.0, SMALL)
    full = tvo.fgp(v, cl.PROX_WEIGHT, niter, True)[0]
    narrower = 0
    for box in _boxes(SMALL):
        for halo, must in ((cl.prox_halo(niter), True), (cl.prox_halo(niter) - 1, False)):
            outer = cl.grow(box, SMALL, halo)
            got = tvo.fgp(v[cl.slices(outer)], cl.PROX_WEIGHT, niter, True)[0][cl.inner(box, outer)]
            same = np.array_equal(got, full[cl.slices(box)])
            if must:
                assert same, (box, halo)
            else:
                narrower += not same
    assert narrower > 0


def test_marching_cubes_on_a_slab_is_the_full_grid():
    rng = np.random.RandomState(5)
    vol = rng.uniform(0.0, 1.0, (11, 7, 13)).astype(np.float32)
    vol[4:7] = (vol[4:7] > 0.5) * 0.9 + 0.05                                 # whole planes of one value, too
    verts, faces = mo.marching_cubes(vol, 0.5)
    nv, nt = cl.plane_counts(vol, 0.5)
    assert nv.sum() == len(verts) and nt.sum() == len(faces)
    cv, ct = np.concatenate([[0], np.cumsum(nv)]), np.concatenate([[0], np.cumsum(nt)])
    for a, b in [(0, 3), (2, 5), (5, 6), (8, 11), (0, 11), (10, 11)]:
        sv, st = cl.slab_mesh(vol[a:b + 1], 0.5, a, b)
        assert np.array_equal(sv.view(np.uint32), verts[cv[a]:cv[b]].view(np.uint32)), (a, b)
        assert np.array_equal(st.view(np.uint32), verts[faces[ct[a]:ct[b]]].view(np.uint32)), (a, b)
    # the origin matters: a slab's x coordinates are the full grid's, not the slab's
    sv = cl.slab_mesh(vol[2:6], 0.5, 2, 5)[0]
    assert not np.array_equal(mo.marching_cubes(vol[2:6], 0.5)[0][:len(sv)], sv)


# ---- the render cases' oracle ----------------------------------------------------------------------------------------

def test_render_oracle_pixel_subset_is_the_frame():
    from r2_gaussian_b200 import volume_render as vr

    vol = np.random.RandomState(0).uniform(0.0, 1.0, (9, 8, 10)).astype(np.float32)
    cam = vr.default_camera(vol.shape, 19, 17)
    full = vo.render_frame(vol, cam.record(), 17, 19, False, clim=(0.1, 0.9))
    px = np.array([0, 18, 19, 5 * 19 + 7, 17 * 19 - 1])
    sub = vo.render_frame(vol, cam.record(), 17, 19, False, clim=(0.1, 0.9), pixels=px)
    assert np.array_equal(sub, full.reshape(-1, 4)[px])


def test_stop_case_stops_on_its_sample_in_the_oracle():
    case = cl.VR_CASES["vr_stop_known_sample"]
    cam = cl.vr_camera(case)
    e = 1.0 - float(case.extra["t_stop"])
    ks = case.extra["k_stop"]
    out = vo.render_frame(cl.vr_volume(case), cam.record(), case.H, case.W, True, step=case.extra["step"],
                          unit=case.extra["unit"])
    T = 1.0 - out[..., 3]
    assert np.allclose(T, e ** ks, rtol=1e-9, atol=0.0), (T.min(), T.max(), e ** ks)


def test_long_ray_case_has_its_samples_and_never_stops():
    case = cl.VR_CASES["vr_long_rays"]
    q = cl._Quantities(case)
    assert q["n_samples"] == case.extra["samples"]
    vol = cl.vr_volume(case)
    assert case.extra["vmin"] <= vol.min() and vol.max() <= case.extra["vmax"]
    assert vol.max() - vol.min() > 0.5 * (case.extra["vmax"] - case.extra["vmin"])


def test_case_iteration_is_cheap():
    """Each windowed site's box and halo, each render check and each slab fit in host memory of a test runner."""
    for case in cl.MC_CASES.values():
        for a, b in case.sites:
            assert 0 <= a < b <= case.shape[0] and (b - a + 1) * case.shape[1] * case.shape[2] <= 2**23
    for case in cl.VR_CASES.values():
        lim = case.frames if case.frames > 1 else (case.H if case.extra.get("axis") == "rows" else case.W)
        assert all(0 <= s < lim for s in case.sites) or not case.sites
    assert len(list(itertools.chain(*(c.sites for c in cl.TV_CASES.values())))) >= 10
