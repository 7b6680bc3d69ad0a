"""FISTA-TV without a GPU: the float64 TV operators of tests/tv_oracle.py (gradient / divergence adjointness, the FGP
prox reaching the constrained ROF optimum), `recon.fista_tv_solve` over the float64 oracle operators against a loop
restatement and against the least-squares solution, its history, the Schur Lipschitz bound, and the argument checks
of the Python functions, the C ABI and the command lines."""
import ctypes
import math

import numpy as np
import pytest

import backproject_oracle as bo
import tv_oracle as tvo
from test_recon_cpu import TINY_ANGLES, _dense_matrix, _tiny


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 5, 4), (2, 3, 7), (4, 1, 2), (6, 5, 7), (2, 2, 2)])
def test_gradient_and_divergence_are_adjoint(shape):
    rng = np.random.RandomState(sum(shape))
    x = rng.standard_normal(shape)
    p = rng.standard_normal((3,) + shape)
    g = tvo.grad(x)
    lhs = float((g * p).sum())
    rhs = -float((x * tvo.div(p)).sum())
    scale = float((np.abs(g) * np.abs(p)).sum()) + float((np.abs(x) * np.abs(tvo.div(p))).sum())
    assert abs(lhs - rhs) <= 1e-12 * max(scale, 1.0), (lhs, rhs)
    # the last index along each axis has no forward difference
    assert not g[0, -1].any() and not g[1, :, -1].any() and not g[2, :, :, -1].any()


# FGP after 3000 iterations on a 4x5x6 volume: primal-dual gap below this fraction of the primal objective
ROF_GAP = 1e-5


@pytest.mark.parametrize("nonneg", [True, False])
@pytest.mark.parametrize("w", [0.05, 0.3])
def test_fgp_reaches_the_rof_optimum(nonneg, w):
    v = np.random.RandomState(7).uniform(-0.5, 1.0, size=(4, 5, 6))
    x, p = tvo.fgp(v, w, 3000, nonneg)
    assert np.sqrt((p ** 2).sum(0)).max() <= 1.0 + 1e-12
    if nonneg:
        assert x.min() >= 0.0
    primal, gap = tvo.dual_gap(v, w, x, p, nonneg)
    print(f"w {w} nonneg {nonneg}: primal {primal:.6g} gap {gap:.3g}")
    assert -1e-12 * primal <= gap <= ROF_GAP * primal, (primal, gap)
    # and it is a real denoising: TV drops below that of v
    assert tvo.tv_value(x) < tvo.tv_value(v)


def test_fgp_weight_zero_is_the_projection():
    v = np.random.RandomState(8).uniform(-1.0, 1.0, size=(3, 4, 5))
    assert np.array_equal(tvo.fgp(v, 0.0, 5, True)[0], np.where(v < 0.0, 0.0, v))
    assert np.array_equal(tvo.fgp(v, 0.0, 5, False)[0], v)


def _dense_ops(M, det_shape, vol_shape):
    import torch

    def A(x, views):
        assert views == slice(None)
        return torch.from_numpy((M @ x.numpy().reshape(-1)).reshape(det_shape))

    def At(y, views, weights):
        assert views == slice(None) and not weights
        return torch.from_numpy((M.T @ y.numpy().reshape(-1)).reshape(vol_shape))

    return A, At


def _fista_loop(M, b, shape, niter, lmbda, tviter, L, nonneg):
    """FISTA-TV on a dense matrix, written out with the float64 FGP prox."""
    x_prev = np.zeros(M.shape[1])
    y = x_prev.copy()
    t = 1.0
    hist = []
    for _ in range(niter):
        v = y - (M.T @ (M @ y - b)) / L
        x = tvo.fgp(v.reshape(shape), lmbda / L, tviter, nonneg)[0].reshape(-1)
        t_next = (1.0 + math.sqrt(1.0 + 4.0 * t * t)) / 2.0
        y = x + ((t - 1.0) / t_next) * (x - x_prev)
        data = 0.5 * float(((M @ x - b) ** 2).sum())
        hist.append((data, tvo.tv_value(x.reshape(shape))))
        x_prev, t = x, t_next
    return x_prev, hist


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_fista_tv_solve_matches_a_loop_restatement(mode):
    torch = pytest.importorskip("torch")
    from r2_gaussian_b200.recon import fista_tv_solve

    sc = _tiny(mode)
    M = _dense_matrix(TINY_ANGLES, sc)
    shape = tuple(sc["nVoxel"])
    truth = np.random.RandomState(4).uniform(0.0, 1.0, size=M.shape[1])
    b = M @ truth + np.random.RandomState(5).normal(0.0, 0.05, size=M.shape[0])
    L = float((M @ np.ones(M.shape[1])).max() * (M.T @ np.ones(M.shape[0])).max())
    Aop, Atop = bo.operators(TINY_ANGLES, sc)
    lmbda, niter, tviter = 0.02, 4, 10
    got, hist = fista_tv_solve(torch.from_numpy(b.reshape(len(TINY_ANGLES), 8, 8)), Aop, Atop, shape, niter, lmbda,
                               tviter, prox=tvo.prox, tv=tvo.tv)
    want, want_hist = _fista_loop(M, b, shape, niter, lmbda, tviter, L, True)
    got = got.numpy().reshape(-1)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max(), np.abs(got - want).max()
    assert len(hist) == niter
    for h, (data, tv) in zip(hist, want_hist):
        assert abs(h["data"] - data) <= 1e-12 * data and abs(h["tv"] - tv) <= 1e-12 * tv, (h, data, tv)
        assert h["F"] == h["data"] + lmbda * h["tv"]
    # the iterate is a descent from x = 0 and TV is active
    assert hist[-1]["F"] < 0.5 * float((b ** 2).sum())
    assert got.min() >= 0.0


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_fista_without_tv_reaches_the_least_squares_solution(mode):
    """lmbda = 0, nonneg=False: FISTA on 1/2 |A x - b|^2.  Beck-Teboulle's bound F(x_k) - F* <= 2 L |x*|^2 / (k + 1)^2
    (from x_0 = 0) and, with F(x) - F* = 1/2 |A (x - x*)|^2 >= 1/2 s_min^2 |x - x*|^2, |x_k - x*| <= 2 sqrt(L) |x*| /
    (s_min (k + 1)) are the tolerances."""
    torch = pytest.importorskip("torch")
    from r2_gaussian_b200.recon import fista_tv_solve

    sc = _tiny(mode)
    M = _dense_matrix(TINY_ANGLES, sc)
    b = np.random.RandomState(1).uniform(0.0, 1.0, size=M.shape[0])       # the CGLS least-squares test's b
    want = np.linalg.lstsq(M, b, rcond=None)[0]
    f_star = 0.5 * float(((M @ want - b) ** 2).sum())
    s_min = np.linalg.svd(M, compute_uv=False).min()
    A, At = _dense_ops(M, (len(TINY_ANGLES), 8, 8), tuple(sc["nVoxel"]))
    niter = 500
    x, hist = fista_tv_solve(torch.from_numpy(b.reshape(len(TINY_ANGLES), 8, 8)), A, At, sc["nVoxel"], niter, 0.0,
                             nonneg=False, prox=tvo.prox, tv=tvo.tv)
    L = float((M @ np.ones(M.shape[1])).max() * (M.T @ np.ones(M.shape[0])).max())
    got = x.numpy().reshape(-1)
    err = np.linalg.norm(got - want)
    print(f"{mode}: |x - x*| / |x*| = {err / np.linalg.norm(want):.3g}, "
          f"bound {2 * math.sqrt(L) / (s_min * (niter + 1)):.3g}; F - F* = {hist[-1]['F'] - f_star:.3g}")
    assert hist[-1]["F"] - f_star <= 2.0 * L * float((want ** 2).sum()) / (niter + 1) ** 2
    assert err <= 2.0 * math.sqrt(L) * np.linalg.norm(want) / (s_min * (niter + 1))


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_schur_bound_is_above_the_operator_norm(mode):
    torch = pytest.importorskip("torch")
    from r2_gaussian_b200.recon import schur_lipschitz

    sc = _tiny(mode)
    Aop, Atop = bo.operators(TINY_ANGLES, sc)
    b = torch.zeros(len(TINY_ANGLES), 8, 8, dtype=torch.float64)
    L = schur_lipschitz(b, Aop, Atop, sc["nVoxel"])
    x = torch.from_numpy(np.random.RandomState(6).uniform(0.5, 1.0, size=sc["nVoxel"]))
    est = 0.0
    for _ in range(30):                                                    # power iteration on A^T A
        x = x / torch.linalg.vector_norm(x)
        x = Atop(Aop(x, slice(None)), slice(None), False)
        est = float(torch.linalg.vector_norm(x))
    exact = np.linalg.norm(_dense_matrix(TINY_ANGLES, sc), 2) ** 2
    print(f"{mode}: Schur L {L:.6g}, power iteration {est:.6g}, |A|^2 {exact:.6g}, ratio {L / exact:.3f}")
    assert est <= exact * (1 + 1e-9)
    assert L >= exact


def test_python_argument_checks():
    torch = pytest.importorskip("torch")
    from r2_gaussian_b200 import recon
    from r2_gaussian_b200.tv import tv_denoise, tv_value

    sc = _tiny("cone")
    A, At = bo.operators(TINY_ANGLES, sc)
    b = torch.zeros(len(TINY_ANGLES), 8, 8, dtype=torch.float64)
    for kw, match in ((dict(niter=0), "niter"), (dict(niter=1.5), "niter"), (dict(lmbda=-1.0), "lmbda"),
                      (dict(lmbda=math.nan), "lmbda"), (dict(tviter=0), "tviter"), (dict(L=0.0), "L must"),
                      (dict(L=-2.0), "L must"), (dict(L=math.inf), "L must")):
        args = dict(dict(niter=2, lmbda=0.1, tviter=5, L=None), **kw)
        with pytest.raises(ValueError, match=match):
            recon.fista_tv_solve(b, A, At, sc["nVoxel"], args["niter"], args["lmbda"], args["tviter"], args["L"],
                                 prox=tvo.prox, tv=tvo.tv)
        with pytest.raises(ValueError, match=match):
            recon.fista_tv(b.float(), TINY_ANGLES, sc, **args)
    with pytest.raises(RuntimeError, match="CUDA"):
        recon.fista_tv(b.float(), TINY_ANGLES, sc, niter=2)
    vol = torch.zeros(3, 4, 5)
    with pytest.raises(RuntimeError, match="CUDA"):
        tv_denoise(vol, 0.1)
    with pytest.raises(RuntimeError, match="CUDA"):
        tv_value(vol)
    with pytest.raises(ValueError, match="weight"):
        tv_denoise(vol, -0.1)
    with pytest.raises(ValueError, match="niter"):
        tv_denoise(vol, 0.1, niter=0)


def test_abi_rejects_bad_arguments_before_any_cuda_call():
    from r2_gaussian_b200 import _lib

    lib = _lib.load()
    dummy = ctypes.c_void_p(16)
    need = int(lib.r2x_tv_prox_scratch_bytes(4, 5, 6))
    assert need == 36 * 4 * 5 * 6
    base = dict(nx=4, ny=5, nz=6, v=dummy, w=0.1, niter=3, nonneg=1, out=dummy, scratch=dummy, nbytes=need)

    def prox(**kw):
        a = dict(base, **kw)
        return lib.r2x_tv_prox(None, a["nx"], a["ny"], a["nz"], a["v"], a["w"], a["niter"], a["nonneg"], a["out"],
                               a["scratch"], a["nbytes"])

    for kw in (dict(nx=0), dict(ny=0), dict(nz=-1), dict(nx=4 * 65535 + 1), dict(ny=8 * 65535 + 1), dict(v=None),
               dict(out=None), dict(scratch=None), dict(w=-0.1), dict(w=math.nan), dict(w=math.inf), dict(niter=0),
               dict(niter=-3), dict(nonneg=2), dict(nbytes=need - 1)):
        assert prox(**kw) != 0, kw
        assert b"r2x_tv_prox: bad" in lib.r2x_last_error(), kw
    vneed = int(lib.r2x_tv_value_scratch_bytes(4, 5, 6))
    assert vneed >= 8

    def value(nx=4, x=dummy, out=dummy, scratch=dummy, nbytes=vneed):
        return lib.r2x_tv_value(None, nx, 5, 6, x, out, scratch, nbytes)

    for kw in (dict(nx=0), dict(x=None), dict(out=None), dict(scratch=None), dict(nbytes=vneed - 1)):
        assert value(**kw) != 0, kw
        assert b"r2x_tv_value: bad" in lib.r2x_last_error(), kw


def test_command_lines_accept_fista_tv(tmp_path, monkeypatch):
    torch = pytest.importorskip("torch")
    from r2_gaussian_b200 import initialize_pcd, recon

    assert "fista_tv" in recon.METHODS
    assert recon._parse_methods("fdk,fista_tv") == ["fdk", "fista_tv"]
    with pytest.raises(SystemExit, match="fista_tv"):                      # the refusal names the alternative
        recon._parse_methods("asd_pocs")
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(SystemExit, match="CUDA device"):                   # parsed, then refused for want of a GPU
        recon.main(["-s", str(tmp_path), "-m", str(tmp_path / "out"), "--methods", "fista_tv"])
    with pytest.raises(SystemExit, match="fista_tv needs a CUDA device"):
        initialize_pcd.main(["--data", str(tmp_path), "--recon_method", "fista_tv"])
