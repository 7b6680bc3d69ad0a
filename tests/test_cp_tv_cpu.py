"""cp_tv (Chambolle-Pock for min TV(x) s.t. |A x - b| <= epsilon, x >= 0) without a GPU: `recon.cp_tv_solve` over
the float64 oracle operators and the float64 step of tests/cp_tv_oracle.py against the iteration as recon.py states
it, the closed form epsilon >= |b| (x = 0 exactly), a long run reaching the constraint with less TV than a feasible
CGLS iterate, and the argument checks of the Python functions, the C ABI and the command line."""
import ctypes
import math

import numpy as np
import pytest

import backproject_oracle as bo
import cp_tv_oracle as cpo
import tv_oracle as tvo
from test_recon_cpu import TINY_ANGLES, _dense_matrix, _tiny

torch = pytest.importorskip("torch")


def _noisy(mode):
    sc = _tiny(mode)
    M = _dense_matrix(TINY_ANGLES, sc)
    truth = np.random.RandomState(4).uniform(0.0, 1.0, size=M.shape[1])
    noise = np.random.RandomState(5).normal(0.0, 0.05, size=M.shape[0])
    return sc, M, truth, M @ truth + noise, float(np.linalg.norm(noise))


def _bt(b):
    return torch.from_numpy(b.reshape(len(TINY_ANGLES), 8, 8))


def _dense_ops(M, vol_shape):
    """The oracle projector as a dense matrix and its exact transpose (fast enough for thousands of iterations)."""
    def A(x, views):
        assert views == slice(None)
        return torch.from_numpy((M @ x.numpy().reshape(-1)).reshape(len(TINY_ANGLES), 8, 8))

    def At(y, views, weights):
        assert views == slice(None) and not weights
        return torch.from_numpy((M.T @ y.numpy().reshape(-1)).reshape(vol_shape))

    return A, At


def _cp_loop(A, At, b, shape, niter, eps, L, nonneg):
    """The iteration as stated: u = q + sigma (A xbar - b), q = max(1 - sigma eps / |u|, 0) u, then the step."""
    tau = sigma = 0.99 / math.sqrt(2.0 * L)
    nu = math.sqrt(L / 12.0)
    x = np.zeros(shape)
    xbar, p, q = x.copy(), np.zeros((3,) + shape), np.zeros(b.shape)
    hist = []
    for _ in range(niter):
        u = q + sigma * (A(torch.from_numpy(xbar), slice(None)).numpy() - b)
        q = max(1.0 - sigma * eps / np.linalg.norm(u), 0.0) * u
        g = At(torch.from_numpy(q), slice(None), False).numpy()
        x_next, xbar, p = cpo.cp_step(x, xbar, p, g, tau, sigma, nu, nonneg)
        r = A(torch.from_numpy(x_next), slice(None)).numpy() - b
        hist.append((float(np.linalg.norm(r)), tvo.tv_value(x_next)))
        x = x_next
    return x, hist


@pytest.mark.parametrize("nonneg", [True, False])
@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_cp_tv_solve_matches_the_stated_iteration(mode, nonneg):
    from r2_gaussian_b200.recon import cp_tv_solve, schur_lipschitz

    sc, M, truth, b, noise = _noisy(mode)
    shape = tuple(sc["nVoxel"])
    A, At = bo.operators(TINY_ANGLES, sc)
    bt = _bt(b)
    eps, niter = 1.5 * noise, 6
    got, hist = cp_tv_solve(bt, A, At, shape, niter, eps, nonneg=nonneg, step=cpo.step, tv=tvo.tv)
    L = schur_lipschitz(bt, A, At, shape)
    want, want_hist = _cp_loop(A, At, bt.numpy(), shape, niter, eps, L, nonneg)
    assert np.abs(got.numpy() - want).max() <= 1e-12 * np.abs(want).max(), np.abs(got.numpy() - want).max()
    assert len(hist) == niter and list(hist[0]) == ["residual", "tv"]
    for h, (res, tv) in zip(hist, want_hist):
        assert abs(h["residual"] - res) <= 1e-12 * res and abs(h["tv"] - tv) <= 1e-12 * tv, (h, res, tv)


@pytest.mark.parametrize("nonneg", [True, False])
def test_epsilon_above_the_data_norm_gives_exactly_zero(nonneg):
    from r2_gaussian_b200.recon import _dot, cp_tv_solve

    sc, M, truth, b, noise = _noisy("cone")
    A, At = bo.operators(TINY_ANGLES, sc)
    bt = _bt(b)
    norm_b = _dot(bt, bt) ** 0.5
    for eps in (norm_b, 2.0 * norm_b):
        x, hist = cp_tv_solve(bt, A, At, sc["nVoxel"], 5, eps, nonneg=nonneg, step=cpo.step, tv=tvo.tv)
        assert x.dtype == torch.float64 and not x.numpy().any() and not np.signbit(x.numpy()).any()
        assert [h["tv"] for h in hist] == [0.0] * 5 and [h["residual"] for h in hist] == [norm_b] * 5


# residual after the long run, relative to epsilon
FEASIBLE = 1e-3


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_long_run_meets_the_constraint_with_less_tv_than_a_feasible_point(mode):
    """3000 iterations on the 27-voxel problem (the oracle projector as a dense matrix): the residual reaches epsilon
    within FEASIBLE and TV(x) lies below that of two feasible points, the truth and the first CGLS iterate whose
    residual is <= epsilon."""
    from r2_gaussian_b200.recon import cgls_solve, cp_tv_solve

    sc, M, truth, b, noise = _noisy(mode)
    shape = tuple(sc["nVoxel"])
    A, At = _dense_ops(M, shape)
    bt = _bt(b)
    eps = 1.5 * noise
    x, hist = cp_tv_solve(bt, A, At, shape, 3000, eps, step=cpo.step, tv=tvo.tv)
    _, l2 = cgls_solve(bt, A, At, 60)
    k = next(i for i, r in enumerate(l2) if r <= eps)
    x_cgls, _ = cgls_solve(bt, A, At, k + 1)
    tv_cgls, tv_truth = tvo.tv_value(x_cgls.numpy()), tvo.tv_value(truth.reshape(shape))
    res = float(np.linalg.norm(M @ x.numpy().reshape(-1) - b))
    print(f"{mode}: residual / eps {res / eps:.9f}, TV {hist[-1]['tv']:.6g}, CGLS ({k + 1} iterations) TV "
          f"{tv_cgls:.6g}, truth TV {tv_truth:.6g}")
    assert abs(hist[-1]["residual"] - res) <= 1e-12 * res
    assert res <= eps * (1.0 + FEASIBLE)
    assert float(x.min()) >= 0.0
    assert hist[-1]["tv"] < tv_cgls and hist[-1]["tv"] < tv_truth


def test_python_argument_checks():
    from r2_gaussian_b200 import recon
    from r2_gaussian_b200.tv import tv_cp_step

    sc = _tiny("cone")
    A, At = bo.operators(TINY_ANGLES, sc)
    b = torch.zeros(len(TINY_ANGLES), 8, 8, dtype=torch.float64)
    for kw, match in ((dict(niter=0), "niter"), (dict(niter=2.5), "niter"), (dict(epsilon=-1.0), "epsilon"),
                      (dict(epsilon=math.nan), "epsilon"), (dict(epsilon=math.inf), "epsilon"),
                      (dict(L=0.0), "L must"), (dict(L=-1.0), "L must"), (dict(L=math.nan), "L must"),
                      (dict(L=math.inf), "L must")):
        args = dict(dict(niter=2, epsilon=0.1, L=None), **kw)
        with pytest.raises(ValueError, match=match):
            recon.cp_tv_solve(b, A, At, sc["nVoxel"], args["niter"], args["epsilon"], args["L"], step=cpo.step,
                              tv=tvo.tv)
        with pytest.raises(ValueError, match=match):
            recon.cp_tv(b.float(), TINY_ANGLES, sc, **args)
    with pytest.raises(ValueError, match="epsilon must be given"):
        recon.cp_tv_solve(b, A, At, sc["nVoxel"], 2, None, step=cpo.step, tv=tvo.tv)
    for ratio in (-0.1, math.nan, math.inf):
        with pytest.raises(ValueError, match="epsilon_ratio"):
            recon.cp_tv(b.float(), TINY_ANGLES, sc, epsilon_ratio=ratio)
        with pytest.raises(ValueError, match="epsilon_ratio"):
            recon.cp_tv_epsilon(b.float(), TINY_ANGLES, sc, ratio)
    with pytest.raises(RuntimeError, match="CUDA"):
        recon.cp_tv(b.float(), TINY_ANGLES, sc, niter=2)
    vol = torch.zeros(3, 4, 5)
    with pytest.raises(RuntimeError, match="CUDA"):
        tv_cp_step(vol, vol, torch.zeros(3, 3, 4, 5), vol, 0.1, 0.1, 1.0)


def test_step_sizes_satisfy_the_convergence_condition():
    """tau sigma |K|^2 < 1 for K = [A; nu grad] whenever |A|^2 <= L, on the 27-voxel cone problem."""
    from r2_gaussian_b200.recon import cp_step_sizes

    sc = _tiny("cone")
    M = _dense_matrix(TINY_ANGLES, sc)
    shape = tuple(sc["nVoxel"])
    n = M.shape[1]
    G = np.stack([tvo.grad(e.reshape(shape)).reshape(-1) for e in np.eye(n)], axis=1)
    for L in (np.linalg.norm(M, 2) ** 2, float((M @ np.ones(n)).max() * (M.T @ np.ones(M.shape[0])).max())):
        tau, sigma, nu = cp_step_sizes(L)
        K = np.concatenate([M, nu * G])
        assert tau == sigma and tau * sigma * np.linalg.norm(K, 2) ** 2 <= 0.99 ** 2


def test_abi_rejects_bad_arguments_before_any_cuda_call():
    from r2_gaussian_b200 import _lib

    lib = _lib.load()
    nx, ny, nz = 4, 5, 6
    nvox = nx * ny * nz
    base_addr = 1 << 20
    span = 4 * nvox
    # disjoint fake device addresses: x, xbar, g, x_out, xbar_out (nvox floats), p, p_out (3 nvox floats)
    at = {k: ctypes.c_void_p(base_addr + i * 4 * span) for i, k in enumerate(("x", "xbar", "g", "xo", "xbo", "p", "po"))}
    base = dict(nx=nx, ny=ny, nz=nz, tau=0.1, sigma=0.1, nu=0.5, nonneg=1, **at)

    def step(**kw):
        a = dict(base, **kw)
        return lib.r2x_tv_cp_step(None, a["nx"], a["ny"], a["nz"], a["x"], a["xbar"], a["p"], a["g"], a["tau"],
                                  a["sigma"], a["nu"], a["nonneg"], a["xo"], a["xbo"], a["po"])

    def addr(k, off_floats=0):
        return ctypes.c_void_p(at[k].value + 4 * off_floats)

    bad = [dict(nx=0), dict(ny=0), dict(nz=-1), dict(nx=4 * 65535 + 1), dict(ny=8 * 65535 + 1)]
    bad += [{k: None} for k in at]
    for name in ("tau", "sigma", "nu"):
        bad += [{name: 0.0}, {name: -0.1}, {name: math.nan}, {name: math.inf}]
    bad += [dict(nu=1e-39), dict(nu=1e30, sigma=1e30), dict(nu=1e30, tau=1e30), dict(nonneg=2), dict(nonneg=-1)]
    # an output overlapping an input or another output
    bad += [dict(xo=at["x"]), dict(xbo=at["xbar"]), dict(po=at["p"]), dict(xo=addr("p", 3 * nvox - 1)),
            dict(po=addr("g", nvox - 1)), dict(xbo=addr("xo", nvox - 1)), dict(po=addr("xbo", 1)),
            dict(xo=addr("g", -nvox + 1))]
    for kw in bad:
        assert step(**kw) != 0, kw
        assert b"r2x_tv_cp_step: bad" in lib.r2x_last_error(), kw


def test_command_line_accepts_cp_tv(tmp_path, monkeypatch):
    from r2_gaussian_b200 import recon

    assert recon.METHODS[-1] == "cp_tv"
    assert recon._parse_methods("fdk,cp_tv") == ["fdk", "cp_tv"]
    for m in ("asd_pocs", "os_asd_pocs"):
        with pytest.raises(SystemExit, match=f"method {m} is not built .*fista_tv is its TV-regularised alternative"):
            recon._parse_methods(f"fdk,{m}")
    for flag in (["--short_scan"], ["--fdk_filter", "hann"]):
        with pytest.raises(SystemExit, match="applies to the fdk method"):
            recon.main(["-s", str(tmp_path), "-m", str(tmp_path / "out"), "--methods", "cp_tv", *flag])
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(SystemExit, match="CUDA device"):                   # parsed, then refused for want of a GPU
        recon.main(["-s", str(tmp_path), "-m", str(tmp_path / "out"), "--methods", "cp_tv", "--use_offDetector"])
