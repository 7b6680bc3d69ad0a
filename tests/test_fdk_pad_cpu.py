"""FDK's truncation pad on the CPU: the float64 oracle tests/fdk_pad_oracle.py against the existing FDK oracles at pad 0
and against a direct sum of the model, the extension's constant-row, mirror and full-width (L = W) properties, the
fraction-to-pixels rounding, and every refusal before any CUDA call (fdk(), recon_volume, both command lines, the C
ABI)."""
import argparse
import ctypes
import math

import numpy as np
import pytest

import ct_edge_cases as ct
import fdk_cases as fc
import fdk_pad_oracle as fpo
import fdk_window_oracle as fwo


# ---- the oracle ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("short_scan", [False, True])
@pytest.mark.parametrize("mode", ["cone", "parallel"])
@pytest.mark.parametrize("name", fwo.FILTERS)
def test_pad_zero_is_the_existing_oracles(name, mode, short_scan):
    rng = np.random.RandomState(len(name))
    sc = fc.scanner(mode, 12, 6)
    angles = (np.linspace(0.0, math.radians(250.0), 9)[:-1] + 0.4) if short_scan else fc.full_scan(8) + 0.2
    projs = rng.uniform(0.0, 1.0, (8, 12, 12))
    want = fwo.fdk_scene(projs, angles, sc, name, short_scan=short_scan)
    got = fpo.fdk_scene(projs, angles, sc, name, 0, short_scan=short_scan)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()
    want_q = fwo.filter_projections(projs, name, 0.3, 0.2, 1, 5.0)
    got_q = fpo.filter_projections(projs, name, 0, 0.3, 0.2, 1, 5.0)
    assert np.abs(got_q - want_q).max() <= 1e-12 * np.abs(want_q).max()


@pytest.mark.parametrize("W,L", [(1, 1), (2, 1), (2, 2), (7, 3), (7, 7), (16, 5)])
@pytest.mark.parametrize("name", ["ram_lak", "hann"])
def test_filter_is_the_direct_sum_of_the_model(name, W, L):
    r = np.random.RandomState(W + 10 * L).uniform(-1.0, 1.0, (3, W))
    t = fpo.taper(L)
    e = {i: r[:, i] for i in range(W)}
    for k in range(1, L + 1):
        e[-k] = t[k - 1] * r[:, k - 1]
        e[W - 1 + k] = t[k - 1] * r[:, W - k]
    want = np.stack([sum(float(fwo.taps(name, j - i)) * e[i] for i in range(-L, W + L)) for j in range(W)], -1) / 0.7
    got = fpo.filter_rows(r, name, L, 0.7)
    assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


def test_constant_row_extends_to_the_taper():
    for W, L in ((5, 3), (8, 8), (1, 1)):
        e = fpo.extend(np.full((2, W), 2.5), L)
        k = np.arange(1, L + 1)
        t = 0.5 * (1.0 + np.cos(math.pi * k / (L + 1)))
        np.testing.assert_allclose(e[:, :L], np.broadcast_to(2.5 * t[::-1], (2, L)), rtol=0, atol=1e-15)
        np.testing.assert_allclose(e[:, L + W:], np.broadcast_to(2.5 * t, (2, L)), rtol=0, atol=1e-15)
        assert (e[:, L:L + W] == 2.5).all()
    # the roll-off falls from near 1 to near 0 and never reaches either
    t = fpo.taper(40)
    assert np.all(np.diff(t) < 0) and 0.99 < t[0] < 1.0 and 0.0 < t[-1] < 0.01


def test_extension_is_mirror_symmetric():
    r = np.random.RandomState(3).uniform(0.0, 1.0, (4, 11))
    for L in (1, 5, 11):
        np.testing.assert_array_equal(fpo.extend(r[:, ::-1], L), fpo.extend(r, L)[:, ::-1])
        e = fpo.extend(r, L)
        t = fpo.taper(L)
        for k in range(1, L + 1):                             # e[-k] and e[W-1+k] mirror r about each edge
            assert np.array_equal(e[:, L - k], t[k - 1] * r[:, k - 1])
            assert np.array_equal(e[:, L + 10 + k], t[k - 1] * r[:, 11 - k])


def test_full_width_pad_needs_no_clamping():
    for W in (1, 2, 5):
        r = np.arange(1.0, W + 1.0)[None, :]
        e = fpo.extend(r, W)
        assert e.shape == (1, 3 * W)
        t = fpo.taper(W)
        assert e[0, 0] == t[-1] * r[0, W - 1] and e[0, -1] == t[-1] * r[0, 0]
    with pytest.raises(ValueError):
        fpo.extend(np.ones((1, 4)), 5)


def test_pad_pixels_rounds_halves_up():
    from r2_gaussian_b200.fdk import pad_pixels

    assert [pad_pixels(f, 10) for f in (0.0, 0.04, 0.05, 0.25, 0.5, 1.0)] == [0, 0, 1, 3, 5, 10]
    assert pad_pixels(0.5, 6145) == 3073 and pad_pixels(1.0, 6145) == 6145


# ---- refusals ------------------------------------------------------------------------------------------------------

def _host_call(**kw):
    torch = pytest.importorskip("torch")
    from r2_gaussian_b200.fdk import fdk

    return fdk(torch.zeros(2, 8, 8), [0.0, 1.0], kw.pop("sc", fc.scanner("cone", 8, 4)), **kw)


def test_fdk_refuses_bad_pads_and_combinations():
    for bad in (-0.1, 1.01, float("nan"), float("inf"), "0.5", True, None):
        with pytest.raises(ValueError, match="pad must be a fraction of the detector width in"):
            _host_call(pad=bad)
    off = ct._offset(fc.scanner("cone", 8, 4), 1.5, 0.0)
    with pytest.raises(ValueError, match="pad cannot be combined with half_fan"):
        _host_call(sc=off, pad=0.5, use_offDetector=True, half_fan=True)
    with pytest.raises(ValueError, match="pad cannot be combined with helical"):
        _host_call(pad=0.5, helical=True, view_geometry=[{}, {}])
    with pytest.raises(ValueError, match="pad cannot be combined with view_geometry"):
        _host_call(pad=0.5, view_geometry=[{}, {}])
    for ok in (0, 0.0, 0.25, 1, 1.0):                            # valid pads reach the CUDA check
        with pytest.raises(RuntimeError, match="CUDA"):
            _host_call(pad=ok)
    with pytest.raises(RuntimeError, match="CUDA"):
        _host_call(pad=0.5, short_scan=True, sc=fc.scanner("parallel", 8, 4))


def test_recon_volume_refuses_fdk_pad_without_fdk():
    from r2_gaussian_b200 import recon

    with pytest.raises(ValueError, match="fdk_pad applies to fdk only"):
        recon.recon_volume(None, [0.0, 1.0], {}, "cgls", fdk_pad=0.5)


def _recon_argv(tmp_path, *flags, methods="fdk"):
    return ["-s", str(tmp_path / "none"), "-m", str(tmp_path / "out"), "--methods", methods, *flags]


def _init_argv(tmp_path, *flags, method="fdk"):
    return ["--data", str(tmp_path / "none"), "--recon_method", method, *flags]


def test_recon_refuses_fdk_pad(tmp_path):
    from r2_gaussian_b200 import recon

    with pytest.raises(SystemExit, match="--fdk_pad applies to the fdk method"):
        recon.main(_recon_argv(tmp_path, "--fdk_pad", "0.5", methods="sart,cgls"))
    for flags, msg in ((["--use_offDetector", "--half_fan"], "--fdk_pad cannot be combined with --half_fan"),
                       (["--use_view_geometry", "--helical"], "--fdk_pad cannot be combined with --helical"),
                       (["--use_view_geometry"], "--fdk_pad cannot be combined with --use_view_geometry")):
        for pad in ("0.5", "0"):
            with pytest.raises(SystemExit, match=msg):
                recon.main(_recon_argv(tmp_path, "--fdk_pad", pad, *flags))
    for bad in ("-0.5", "1.5", "nan"):
        with pytest.raises(SystemExit, match="--fdk_pad must be a fraction of the detector width"):
            recon.main(_recon_argv(tmp_path, "--fdk_pad", bad))


@pytest.mark.parametrize("method", ["random", "cgls", "fista_tv", "volume"])
def test_initialize_pcd_refuses_fdk_pad_without_fdk(method, tmp_path):
    from r2_gaussian_b200 import initialize_pcd

    with pytest.raises(SystemExit, match="--fdk_pad applies to --recon_method fdk only"):
        initialize_pcd.main(_init_argv(tmp_path, "--fdk_pad", "0.5", method=method))


def test_initialize_pcd_refuses_fdk_pad_combinations(tmp_path):
    from r2_gaussian_b200 import initialize_pcd

    for flags, msg in ((["--use_offDetector", "--half_fan"], "--fdk_pad cannot be combined with --half_fan"),
                       (["--use_view_geometry", "--helical"], "--fdk_pad cannot be combined with --helical"),
                       (["--use_view_geometry"], "--fdk_pad cannot be combined with --use_view_geometry")):
        with pytest.raises(SystemExit, match=msg):
            initialize_pcd.main(_init_argv(tmp_path, "--fdk_pad", "0.25", *flags))
    with pytest.raises(SystemExit, match="--fdk_pad must be a fraction of the detector width"):
        initialize_pcd.main(_init_argv(tmp_path, "--fdk_pad", "2"))


def test_check_fdk_flags_without_the_pad_attribute():
    """Callers whose parser has no --fdk_pad keep the shared check's behaviour."""
    from r2_gaussian_b200 import recon

    ns = argparse.Namespace(short_scan=False, half_fan=False, fdk_filter=None, use_offDetector=False)
    recon.check_fdk_flags(ns, False, "{flag}")


def _abi_call(lib, W=8, pad=0, weighting=0, su=0.0):
    dummy = ctypes.c_void_p(16)
    return lib.r2x_fdk_pad(None, 2, 8, W, dummy, dummy, dummy, 0.3, 0.3, 1, su, 0.0, weighting, None, 0.0, 5.0, 4, 4, 4,
                           2.0, 2.0, 2.0, 0.0, 0.0, 0.0, dummy, dummy, 1 << 24, pad)


def test_abi_refuses_bad_pads_before_any_cuda_call():
    from r2_gaussian_b200 import _lib

    lib = _lib.load()
    for W, pad in ((8, -1), (8, 9), (1, 2), (8, -(1 << 30))):
        assert _abi_call(lib, W, pad) != 0
        assert b"r2x_fdk_pad: bad pad (needs 0 <= pad <= W)" in lib.r2x_last_error(), (W, pad)
    for f in (0x000, 0x100, 0x400):
        for pad in (0, 1, 8):
            assert _abi_call(lib, pad=pad, weighting=f | 2, su=1.5) != 0
            assert b"r2x_fdk_pad: bad weighting (no pad with R2X_FDK_HALF_FAN" in lib.r2x_last_error()
    # a valid pad reaches r2x_fdk's own checks: Parker without weights, an unknown filter field
    assert _abi_call(lib, pad=4, weighting=1) != 0
    assert b"bad pointer (view_weights NULL)" in lib.r2x_last_error()
    assert _abi_call(lib, pad=4, weighting=0x500) != 0
    assert b"bad weighting" in lib.r2x_last_error()


def _pad_smem(window: int, W: int, L: int) -> int:
    """The padded stage's shared memory in bytes, as include/r2x.h states it."""
    return 4 * ((3 * W + 2 * L + (W + L + 1) // 2) if window == 0 else (2 * W + 3 * L))


def test_abi_refuses_pads_past_the_shared_memory_limit():
    from r2_gaussian_b200 import _lib

    lib = _lib.load()
    assert _pad_smem(0, 9685, 9685) <= ct.H100_SMEM_OPTIN < _pad_smem(0, 9686, 9686)
    assert _pad_smem(0x100, 11622, 11622) <= ct.H100_SMEM_OPTIN < _pad_smem(0x100, 11623, 11623)
    for window, W, L in ((0, 9686, 9686), (0x100, 11623, 11623), (0, 16384, 308), (0x400, 16384, 8449)):
        assert _pad_smem(window, W, L) > ct.H100_SMEM_OPTIN
        assert _abi_call(lib, W, L, window) != 0
        assert b"r2x_fdk_pad: bad pad (the padded row and its taps exceed 227 KB" in lib.r2x_last_error(), (W, L)
    # the largest stages that fit reach r2x_fdk's checks (here: Parker without weights)
    for window, W, L in ((0, 9685, 9685), (0, 16384, 307), (0x100, 16384, 8448)):
        assert _pad_smem(window, W, L) <= ct.H100_SMEM_OPTIN
        assert _abi_call(lib, W, L, window | 1) != 0
        assert b"bad pointer (view_weights NULL)" in lib.r2x_last_error(), (window, W, L)
