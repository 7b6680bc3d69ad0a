"""FDK's windowed ramp filters on the CPU: the closed-form taps of tests/fdk_window_oracle.py against quadrature of their
integral definition, Hann and Hamming as 3-tap combinations of Ram-Lak outputs, the oracle with "ram_lak" against the
plain, short-scan and offset oracles, the windowed kernel's shared-memory layout as r2x_fdk.cu states it, and every
refusal before any CUDA call (fdk(), recon_volume, both command lines, the C ABI)."""
import ctypes
import math

import numpy as np
import pytest
from scipy.integrate import quad

import ct_edge_cases as ct
import fdk_cases as fc
import fdk_short_scan_oracle as sso
import fdk_window_oracle as fwo
import offset_detector_oracle as oo
from oracle import fdk_oracle
from regime_cases import _find, _source

WINDOWED = ("shepp_logan", "cosine", "hamming", "hann")


def window_smem(W: int) -> int:
    """fdk_window_smem(W) in bytes, as r2x_fdk.cu states it."""
    expr = _find(r"fdk_window_smem\(int W\) \{ return \(size_t\)\((.+)\) \* sizeof\(float\); \}", _source("r2x_fdk.cu"),
                 "fdk_window_smem").group(1)
    return 4 * int(eval(expr.replace("/", "//"), {"__builtins__": {}}, {"W": int(W)}))


def first_window_opt_in_width() -> int:
    W = 1
    while window_smem(W) <= ct.K["FDK_SMEM_DEFAULT"]:
        W += 1
    return W


# QAWO reports roundoff at the tightest tolerances where the integral is ~1e-6; the 1e-12 bar below is the check
@pytest.mark.filterwarnings("ignore::scipy.integrate.IntegrationWarning")
@pytest.mark.parametrize("name", fwo.FILTERS)
def test_closed_form_taps_equal_the_integral(name):
    win = fwo.WINDOWS[name]
    ks = np.arange(0, 301)
    want = np.array([quad(lambda w: w * win(np.asarray(w)), 0.0, math.pi, weight="cos", wvar=float(k),
                          epsabs=1e-15, epsrel=1e-13, limit=400)[0] for k in ks]) / (2.0 * math.pi ** 2)
    got = fwo.taps(name, ks)
    assert np.abs(got - want).max() <= 1e-12, np.abs(got - want).max()
    np.testing.assert_allclose(fwo.taps(name, -ks), got, rtol=0, atol=0)


def test_tap_values_at_zero():
    got = [float(fwo.taps(n, 0)) for n in fwo.FILTERS]
    np.testing.assert_allclose(got, [0.25, 0.202642, 0.115668, 0.088392, 0.074339], rtol=0, atol=5e-7)


@pytest.mark.parametrize("name,c0,c1", [("hamming", 0.54, 0.23), ("hann", 0.5, 0.25)])
@pytest.mark.parametrize("W", [1, 2, 7, 32])
def test_hann_and_hamming_are_three_tap_combinations_of_ram_lak(name, c0, c1, W):
    """Q_win[j] = c0 Q_RL[j] + c1 (Q_RL[j-1] + Q_RL[j+1]), with Q_RL at -1 and W the out-of-row sums."""
    p = np.random.RandomState(W).uniform(-1.0, 1.0, (2, 3, W))
    padded = np.pad(p, ((0, 0), (0, 0), (1, 1)))
    # the same pitch D = 2 / W for both: parallel beam, and the padded row's pitch rescaled
    rl = fdk_oracle.filter_projections(padded, 1.0, 1.0, 0, 1.0) * (W / (W + 2))
    want = c0 * rl[..., 1:-1] + c1 * (rl[..., :-2] + rl[..., 2:])
    got = fwo.filter_projections(p, name, 1.0, 1.0, 0, 1.0)
    assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("name", fwo.FILTERS)
def test_single_impulse_row_gives_the_taps(name):
    W = 16
    D = 2.0 / W
    for j in (0, 5, W - 1):
        p = np.zeros((1, 1, W))
        p[0, 0, j] = 1.0
        q = fwo.filter_projections(p, name, 1.0, 1.0, 0, 1.0)[0, 0]
        np.testing.assert_allclose(q, fwo.taps(name, np.arange(W) - j) / D, rtol=1e-12, atol=1e-12)


def test_ram_lak_equals_the_existing_oracles():
    rng = np.random.RandomState(0)
    for mode in ("cone", "parallel"):
        sc = fc.scanner(mode, 12, 6)
        angles = fc.full_scan(8) + 0.2
        projs = rng.uniform(0.0, 1.0, (8, 12, 12))
        want = fdk_oracle.fdk_scene(projs, angles, sc)
        got = fwo.fdk_scene(projs, angles, sc, "ram_lak")
        assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()
        short = np.linspace(0.0, math.radians(250.0), 9)[:-1] + 0.4
        want = sso.fdk_short_scan_scene(projs, short, sc)
        got = fwo.fdk_scene(projs, short, sc, "ram_lak", short_scan=True)
        assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()
        off = ct._offset(sc, 2.3, -0.7)
        for half_fan in (False, True):
            want = oo.fdk_scene(projs, angles, off, half_fan=half_fan)
            got = fwo.fdk_scene(projs, angles, off, "ram_lak", use_offDetector=True, half_fan=half_fan)
            assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()


def test_windows_differ_from_ram_lak_and_damp_noise():
    """Each window passes less of a white-noise row than Ram-Lak (its gain is below 1 towards Nyquist)."""
    p = np.random.RandomState(1).randn(1, 64, 128)
    rl = np.linalg.norm(fwo.filter_projections(p, "ram_lak", 1.0, 1.0, 0, 1.0))
    for name in WINDOWED:
        assert np.linalg.norm(fwo.filter_projections(p, name, 1.0, 1.0, 0, 1.0)) < 0.9 * rl, name


def test_window_kernel_shared_memory_layout():
    """The windowed kernel stages 2 W floats: the widest row fits an H100's opt-in, and it opts in above 6144."""
    assert [window_smem(W) for W in (1, 2, 6144, 6145)] == [8, 16, 49152, 49160]
    assert first_window_opt_in_width() == 6145
    assert window_smem(ct.K["FDK_MAX_W"]) <= ct.H100_SMEM_OPTIN
    # the Ram-Lak kernel's constants are still the ones the edge-case tests read
    assert ct.filter_smem(3511) == 49156 and ct.K["FDK_FILTER_THREADS"] == 256


# ---- refusals ------------------------------------------------------------------------------------------------------

def _host_call(**kw):
    torch = pytest.importorskip("torch")
    from r2_gaussian_b200.fdk import fdk

    return fdk(torch.zeros(2, 8, 8), [0.0, 1.0], kw.pop("sc", fc.scanner("cone", 8, 4)), **kw)


@pytest.mark.parametrize("name", WINDOWED)
def test_scanner_window_needs_the_keyword(name):
    sc = dict(fc.scanner("cone", 8, 4), filter=name)
    with pytest.raises(ValueError, match=rf"filter={name!r}.*--fdk_filter {name}"):
        _host_call(sc=sc)
    with pytest.raises(RuntimeError, match="CUDA"):                # the keyword passes the check
        _host_call(sc=sc, filter=name)
    with pytest.raises(RuntimeError, match="CUDA"):                # and overrides the scanner's
        _host_call(sc=sc, filter="ram_lak")


def test_unknown_filters_are_refused():
    names = "ram_lak, shepp_logan, cosine, hamming, hann"
    for bad in ("hanning", "Hann", "ramp", ""):
        with pytest.raises(ValueError, match=f"unknown filter.*{names}"):
            _host_call(filter=bad)
    with pytest.raises(ValueError, match="filter 'parzen' is not supported"):
        _host_call(sc=dict(fc.scanner("cone", 8, 4), filter="parzen"))
    for ok in (None, "ram_lak"):
        with pytest.raises(RuntimeError, match="CUDA"):
            _host_call(sc=dict(fc.scanner("cone", 8, 4), filter=ok))


@pytest.mark.parametrize("method", ["random", "cgls", "fista_tv", "volume"])
def test_initialize_pcd_refuses_fdk_filter_without_fdk(method, tmp_path):
    from r2_gaussian_b200 import initialize_pcd

    with pytest.raises(SystemExit, match="--fdk_filter applies to --recon_method fdk only"):
        initialize_pcd.main(["--data", str(tmp_path / "none"), "--recon_method", method, "--fdk_filter", "hann"])


def test_recon_refuses_fdk_filter_without_fdk(tmp_path):
    from r2_gaussian_b200 import recon

    with pytest.raises(SystemExit, match="--fdk_filter applies to the fdk method"):
        recon.main(["-s", str(tmp_path / "none"), "-m", str(tmp_path / "out"), "--methods", "sart,cgls",
                    "--fdk_filter", "hann"])
    with pytest.raises(ValueError, match="fdk_filter applies to fdk only"):
        recon.recon_volume(None, [0.0, 1.0], {}, "cgls", fdk_filter="hann")


def test_command_lines_refuse_unknown_filter_names(tmp_path, capsys):
    from r2_gaussian_b200 import initialize_pcd, recon

    with pytest.raises(SystemExit):
        initialize_pcd.main(["--data", str(tmp_path / "none"), "--recon_method", "fdk", "--fdk_filter", "hanning"])
    assert "invalid choice: 'hanning'" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        recon.main(["-s", str(tmp_path / "none"), "-m", str(tmp_path / "out"), "--methods", "fdk", "--fdk_filter",
                    "ramp"])
    assert "invalid choice: 'ramp'" in capsys.readouterr().err


def test_abi_refuses_bad_filter_fields_before_any_cuda_call():
    from r2_gaussian_b200 import _lib

    lib = _lib.load()
    dummy = ctypes.c_void_p(16)

    def call(weighting, su=0.0):
        return lib.r2x_fdk(None, 2, 8, 8, dummy, dummy, dummy, 0.3, 0.3, 1, su, 0.0, weighting, None, 0.0, 5.0, 4, 4, 4,
                           2.0, 2.0, 2.0, 0.0, 0.0, 0.0, dummy, dummy, 1 << 20)

    for w in (3, -1, 0x500, 0x800, 0x1000, 1 << 30, -0x100, 0x103, 0x480, 0x40, 0x4ff, 0x100 | 0x10000):
        assert call(w) != 0, hex(w)
        assert b"bad weighting" in lib.r2x_last_error(), hex(w)
    # a valid filter field reaches the weighting's own checks: half fan with a centred axis, Parker without weights
    for f in (0x000, 0x100, 0x200, 0x300, 0x400):
        assert call(f | 2) != 0
        assert b"bad shift_u for half fan" in lib.r2x_last_error(), hex(f)
        assert call(f | 1) != 0
        assert b"bad pointer (view_weights NULL)" in lib.r2x_last_error(), hex(f)
