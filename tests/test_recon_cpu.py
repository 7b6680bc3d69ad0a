"""The matched backprojector and the iterative reconstructions without a GPU: the float64 backprojection oracle is the
exact transpose of the projector oracle, the C ABI and backproject() reject bad arguments before any CUDA call, and the
CGLS / SART solvers of r2_gaussian_b200.recon, run over the oracle operators, match a dense least-squares solve and a
loop restatement of SART."""
import ctypes
import math

import numpy as np
import pytest

import backproject_oracle as bo
import fdk_cases as fc
from oracle import projector_oracle as po

HALF_PI = math.pi / 2


def _tiny(mode, n_det=8, n_vox=3):
    return fc.scanner(mode, n_det, n_vox)


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_oracle_backprojection_is_the_transpose(mode):
    sc = fc.scanner(mode, 12, 6)
    sc["nDetector"] = [11, 13]
    sc["nVoxel"], sc["sVoxel"], sc["offOrigin"] = [6, 5, 7], [1.6, 1.4, 1.8], [0.1, -0.15, 0.05]
    angles = [0.0, HALF_PI, 2.3]
    rng = np.random.RandomState(0)
    x = rng.uniform(0.0, 1.0, size=sc["nVoxel"])
    y = rng.uniform(0.0, 1.0, size=(len(angles), 11, 13))
    lhs = float((po.project_scene(x, angles, sc) * y).sum())
    rhs = float((x * bo.backproject_scene(y, angles, sc)).sum())
    assert lhs > 0.0
    assert abs(lhs - rhs) <= 1e-12 * abs(lhs), (lhs, rhs)


def test_abi_rejects_bad_arguments_before_any_cuda_call():
    from r2_gaussian_b200 import _lib

    lib = _lib.load()
    dummy = ctypes.c_void_p(16)
    need = int(lib.r2x_volume_backproject_scratch_bytes(2, 8, 8))
    assert need >= 2 * 8 * 8 * 32
    base = dict(N=2, H=8, W=8, projs=dummy, vm=dummy, pm=dummy, tan=0.3, mode=1, su=0.0, sv=0.0, n=4, nx=4, s=2.0,
                c=0.0, step=0.25, out=dummy, wgt=None, scratch=dummy, nbytes=need)

    def call(**kw):
        a = dict(base, **kw)
        return lib.r2x_volume_backproject(None, a["N"], a["H"], a["W"], a["projs"], a["vm"], a["pm"], a["tan"],
                                          a["tan"], a["mode"], a["su"], a["sv"], a["nx"], a["n"], a["n"], a["s"], a["s"],
                                          a["s"], a["c"], a["c"], a["c"], a["step"], a["out"], a["wgt"], a["scratch"],
                                          a["nbytes"])

    bad = (dict(n=0), dict(nx=0), dict(nx=65536), dict(n=4 * 65535 + 1), dict(N=0), dict(H=0), dict(W=0),
           dict(mode=2), dict(mode=-1), dict(s=0.0), dict(s=-1.0), dict(s=math.inf), dict(s=math.nan),
           dict(c=math.nan), dict(tan=0.0), dict(tan=math.inf), dict(step=0.0), dict(step=-0.1), dict(step=math.nan),
           dict(step=math.inf), dict(step=1e-8), dict(projs=None), dict(vm=None), dict(pm=None), dict(out=None),
           dict(scratch=None), dict(nbytes=need - 1), dict(su=math.nan), dict(su=math.inf), dict(sv=-math.inf),
           dict(sv=math.nan))
    for kw in bad:
        assert call(**kw) != 0, kw
        assert b"r2x_volume_backproject: bad" in lib.r2x_last_error(), kw


def test_backproject_argument_errors():
    torch = pytest.importorskip("torch")
    from r2_gaussian_b200.projector import backproject

    sc = fc.scanner("cone", 8, 4)
    y = torch.zeros(2, 8, 8)
    with pytest.raises(RuntimeError, match="CUDA"):
        backproject(y, [0.0, 1.0], sc)
    with pytest.raises(RuntimeError, match="CUDA"):
        backproject(y, [0.0, 1.0], dict(fc.scanner("parallel", 8, 4), accuracy=1.0), weights=True)
    for proj, angles, cfg, match in (
            (torch.zeros(8, 8), [0.0], sc, r"\[N, H, W\]"),
            (y, [0.0, 1.0, 2.0], sc, "angles"),
            (torch.zeros(2, 8, 9), [0.0, 1.0], sc, "nDetector"),
            (y, [0.0, 1.0], dict(sc, accuracy=0.0), "accuracy"),
            (y, [0.0, 1.0], dict(sc, accuracy=-0.5), "accuracy"),
            (y, [0.0, 1.0], dict(sc, offDetector=[0.1, 0.0]), "offDetector"),
            (y, [0.0, 1.0], dict(fc.scanner("parallel", 8, 4), sDetector=[2.0, 3.0]), "sDetector")):
        with pytest.raises(ValueError, match=match):
            backproject(proj, angles, cfg)


# ---- the solvers over the float64 oracle operators ------------------------------------------------------------------

TINY_ANGLES = (0.0, HALF_PI, 1.1, 2.5)


def _dense_matrix(angles, sc):
    """A as a dense [N*H*W, nx*ny*nz] float64 matrix (columns = projections of the unit volumes)."""
    n = int(np.prod(sc["nVoxel"]))
    cols = []
    for i in range(n):
        e = np.zeros(n)
        e[i] = 1.0
        cols.append(po.project_scene(e.reshape(sc["nVoxel"]), angles, sc).reshape(-1))
    return np.stack(cols, axis=1)


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_cgls_reaches_the_least_squares_solution(mode):
    torch = pytest.importorskip("torch")
    from r2_gaussian_b200.recon import cgls_solve

    sc = _tiny(mode)
    A = _dense_matrix(TINY_ANGLES, sc)
    ncols = A.shape[1]
    assert np.linalg.matrix_rank(A) == ncols
    b = np.random.RandomState(1).uniform(0.0, 1.0, size=(len(TINY_ANGLES), 8, 8))
    want = np.linalg.lstsq(A, b.reshape(-1), rcond=None)[0]
    Aop, Atop = bo.operators(TINY_ANGLES, sc)
    x, l2 = cgls_solve(torch.from_numpy(b), Aop, Atop, ncols)
    got = x.numpy().reshape(-1)
    assert np.linalg.norm(got - want) <= 1e-6 * np.linalg.norm(want), np.linalg.norm(got - want) / np.linalg.norm(want)
    assert len(l2) == ncols and all(b_ <= a_ * (1 + 1e-12) for a_, b_ in zip(l2, l2[1:]))   # |r| never grows
    np.testing.assert_allclose(l2[-1], np.linalg.norm(A @ got - b.reshape(-1)), rtol=1e-9)


def _sart_loop(A, b, niter, lmbda, lmbda_red, blocksize, nonneg, rows_per_view):
    """SART / OS-SART on a dense matrix, written out as loops over views and blocks."""
    n_views = b.size // rows_per_view
    x = np.zeros(A.shape[1])
    a1 = A @ np.ones(A.shape[1])
    W = np.zeros_like(a1)
    W[a1 > 0] = 1.0 / a1[a1 > 0]
    for _ in range(niter):
        v = 0
        while v < n_views:
            rows = slice(v * rows_per_view, min(v + blocksize, n_views) * rows_per_view)
            AB = A[rows]
            r = W[rows] * (b[rows] - AB @ x)
            num, den = AB.T @ r, AB.T @ np.ones(AB.shape[0])
            upd = np.zeros_like(x)
            upd[den > 0] = num[den > 0] / den[den > 0]
            x = x + lmbda * upd
            if nonneg:
                x = np.maximum(x, 0.0)
            v += blocksize
        lmbda *= lmbda_red
    return x


@pytest.mark.parametrize("blocksize", [1, 3])
@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_sart_matches_a_loop_restatement(mode, blocksize):
    torch = pytest.importorskip("torch")
    from r2_gaussian_b200.recon import sart_solve

    sc = _tiny(mode)
    A = _dense_matrix(TINY_ANGLES, sc)
    truth = np.random.RandomState(2).uniform(0.0, 1.0, size=A.shape[1])
    b = (A @ truth).reshape(len(TINY_ANGLES), 8, 8)
    Aop, Atop = bo.operators(TINY_ANGLES, sc)
    got = sart_solve(torch.from_numpy(b), Aop, Atop, sc["nVoxel"], 4, 0.9, 0.95, blocksize, True).numpy().reshape(-1)
    want = _sart_loop(A, b.reshape(-1), 4, 0.9, 0.95, blocksize, True, 64)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()
    # the iteration moves toward the truth
    assert np.linalg.norm(got - truth) < 0.9 * np.linalg.norm(truth)


def test_sart_nonneg():
    torch = pytest.importorskip("torch")
    from r2_gaussian_b200.recon import sart_solve

    sc = _tiny("cone")
    Aop, Atop = bo.operators(TINY_ANGLES, sc)
    rng = np.random.RandomState(3)
    b = torch.from_numpy(rng.uniform(-1.0, 1.0, size=(len(TINY_ANGLES), 8, 8)))   # inconsistent, partly negative
    free = sart_solve(b, Aop, Atop, sc["nVoxel"], 3, blocksize=2, nonneg=False)
    clamped = sart_solve(b, Aop, Atop, sc["nVoxel"], 3, blocksize=2, nonneg=True)
    assert float(free.min()) < 0.0
    assert float(clamped.min()) >= 0.0


def test_cli_rejects_methods_that_are_not_built(tmp_path):
    from r2_gaussian_b200 import recon

    for methods, match in (("asd_pocs", "not built"), ("fdk,os_asd_pocs", "not built"), ("fdk,bogus", "supported"),
                           ("", "supported")):
        with pytest.raises(SystemExit, match=match):
            recon.main(["-s", str(tmp_path), "-m", str(tmp_path / "out"), "--methods", methods])
    assert not (tmp_path / "out").exists()
    with pytest.raises(ValueError, match="supported"):
        recon.recon_volume(None, [0.0], _tiny("cone"), "asd_pocs")
