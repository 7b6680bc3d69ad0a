"""The CT operators on the GPU at their edge shapes and launch limits (tests/ct_edge_cases.py) against the float64
oracles: the projector pair (r2x_volume_project / r2x_volume_backproject), FDK (r2x_fdk and its two entry points
r2x_fdk_filter / r2x_fdk_backproject) and the TV prox and value (r2x_tv_prox / r2x_tv_value).  Besides the error
bars of the nominal tests, each case checks the exact properties: a ray that misses the box and a voxel no ray reaches
give exactly 0, the backprojector's weights are backproject(ones) bit for bit, two runs are bitwise equal, and the pair
passes the dot-product test."""
import math

import numpy as np
import pytest

import ct_edge_cases as ct
import tv_oracle as tvo
from oracle import fdk_oracle

pytestmark = pytest.mark.gpu

PAIR_BOUND = 1e-5      # project / backproject: max error over max |want|
DOT_BOUND = 1e-5       # <A x, y> against <x, A^T y>, relative
FDK_BOUND = 1e-4       # FDK and its filter: max error over max |want|
PROX_BOUND = 1e-5      # TV prox: max error over max |want|
VALUE_BOUND = 1e-6     # TV value, relative


def _sum_bound(bound: float, n_views: int) -> float:
    """`bound`, or 4 sqrt(N) 2^-24 when that is larger: the backprojector sums each voxel's N views in float32, whose
    rounding grows as sqrt(N) 2^-24 relative (1.2e-5 measured at N = 65 537).  Below 1000 views `bound` stands."""
    return max(bound, 4.0 * math.sqrt(n_views) * 2.0 ** -24)


def _torch():
    import torch

    return torch


def _bits(t):
    return t.contiguous().view(_torch().int32)


def _max_err(got, want) -> float:
    return float(np.abs(np.asarray(got, np.float64) - want).max())


def _operator(case):
    """CTOperator of the case; an axis-aligned case gets its exact-zero matrices in place of make_view's."""
    torch = _torch()
    from r2_gaussian_b200.projector import CTOperator

    op = CTOperator(case.angles, case.sc, "cuda", case.use_off)
    if case.axis_aligned:
        vs = ct.views(case)
        op.vm = torch.from_numpy(np.stack([v.viewmatrix.reshape(16) for v in vs])).cuda()
        op.pm = torch.from_numpy(np.stack([v.projmatrix.reshape(16) for v in vs])).cuda()
    return op


@pytest.mark.parametrize("name", sorted(ct.PAIR_CASES))
def test_projector_pair_matches_oracle(name):
    torch = _torch()
    case = ct.PAIR_CASES[name]
    x, y = ct.pair_inputs(case)
    vs, t = ct.views(case), ct.shift(case)
    op = _operator(case)
    xt, yt = torch.tensor(x, device="cuda"), torch.tensor(y, device="cuda")

    ax = op.A(xt)
    assert _bits(ax).equal(_bits(op.A(xt)))                                   # bitwise reproducible
    ax = ax.cpu().numpy()
    want = ct.project_views(x, vs, case.sc, *t)
    assert ax.shape == want.shape
    assert _max_err(ax, want) <= PAIR_BOUND * np.abs(want).max(), (_max_err(ax, want), np.abs(want).max())
    assert (ax[want == 0.0] == 0.0).all()                                      # a ray that misses gives exactly 0

    aty, wgt = op.At(yt, slice(None), True)
    assert _bits(aty).equal(_bits(op.At(yt)))                                  # with or without the weights
    assert _bits(wgt).equal(_bits(op.At(torch.ones_like(yt))))                 # weights = backproject(ones)
    again = op.At(yt, slice(None), True)
    assert _bits(aty).equal(_bits(again[0])) and _bits(wgt).equal(_bits(again[1]))
    aty, wgt = aty.cpu().numpy(), wgt.cpu().numpy()
    want_b = ct.backproject_views(y, vs, case.sc, *t)
    bar = _sum_bound(PAIR_BOUND, len(case.angles))
    assert _max_err(aty, want_b) <= bar * np.abs(want_b).max(), (_max_err(aty, want_b), np.abs(want_b).max())
    unreached = ct.backproject_views(np.ones_like(y), vs, case.sc, *t) == 0.0
    assert (aty[unreached] == 0.0).all() and (wgt[unreached] == 0.0).all()    # a voxel no ray reaches gets exactly 0

    lhs = float((ax.astype(np.float64) * y).sum())
    rhs = float((x.astype(np.float64) * aty).sum())
    print(f"{name}: project err {_max_err(ax, want):.3g}, backproject err {_max_err(aty, want_b):.3g}, "
          f"dot {lhs:.9g} vs {rhs:.9g}")
    if name.startswith("box_off_detector"):
        assert not ax.any() and not aty.any() and not wgt.any()
    else:
        assert abs(lhs - rhs) <= _sum_bound(DOT_BOUND, len(case.angles)) * lhs, (lhs, rhs)


def _fdk(case, projs_t):
    from r2_gaussian_b200.fdk import fdk

    return fdk(projs_t, case.angles, case.sc, short_scan=case.weighting == "parker", use_offDetector=case.use_off,
               half_fan=case.weighting == "half_fan")


@pytest.mark.parametrize("name", sorted(ct.FDK_CASES))
def test_fdk_matches_oracle(name):
    torch = _torch()
    case = ct.FDK_CASES[name]
    projs = ct.fdk_inputs(case)
    pt = torch.tensor(projs, device="cuda")
    got = _fdk(case, pt)
    assert _bits(got).equal(_bits(_fdk(case, pt)))                            # bitwise reproducible
    got = got.cpu().numpy()
    want = ct.fdk_want(case, projs)
    print(f"{name}: max err / max = {_max_err(got, want) / np.abs(want).max():.3g}")
    assert got.shape == want.shape
    assert _max_err(got, want) <= FDK_BOUND * np.abs(want).max(), (_max_err(got, want), np.abs(want).max())
    assert (got[want == 0.0] == 0.0).all()                                     # a voxel no ray reaches gets exactly 0


PLAIN_FDK = sorted(n for n, c in ct.FDK_CASES.items() if c.weighting == "plain" and not c.use_off)


@pytest.mark.parametrize("name", PLAIN_FDK)
def test_fdk_entry_points(name):
    """r2x_fdk_filter against the oracle's filter, and r2x_fdk_backproject(r2x_fdk_filter(p)) = r2x_fdk(p) bit for
    bit: the same two kernels with the same arguments (a centred detector's zero shifts add exact zeros)."""
    torch = _torch()
    from r2_gaussian_b200._lib import check, load

    case = ct.FDK_CASES[name]
    projs = ct.fdk_inputs(case, smooth=False)
    pt = torch.tensor(projs, device="cuda")
    vs = ct.views(case)
    v0, dso = vs[0], float(case.sc["DSO"])
    N, H, W = projs.shape
    lib = load()
    stream = torch.cuda.current_stream().cuda_stream
    q = torch.empty_like(pt)
    check(lib.r2x_fdk_filter(stream, N, H, W, pt.data_ptr(), v0.tanfovx, v0.tanfovy, v0.mode, dso, q.data_ptr()),
          "r2x_fdk_filter")
    want_q = fdk_oracle.filter_projections(projs, v0.tanfovx, v0.tanfovy, v0.mode, dso)
    got_q = q.cpu().numpy()
    assert _max_err(got_q, want_q) <= FDK_BOUND * np.abs(want_q).max(), (_max_err(got_q, want_q), np.abs(want_q).max())

    vm = torch.from_numpy(np.stack([v.viewmatrix.reshape(16) for v in vs])).cuda()
    pm = torch.from_numpy(np.stack([v.projmatrix.reshape(16) for v in vs])).cuda()
    nx, ny, nz = case.sc["nVoxel"]
    vol = torch.empty((nx, ny, nz), dtype=torch.float32, device="cuda")
    check(lib.r2x_fdk_backproject(stream, N, H, W, q.data_ptr(), vm.data_ptr(), pm.data_ptr(), v0.mode, dso, nx, ny, nz,
                                  *case.sc["sVoxel"], *case.sc["offOrigin"], vol.data_ptr()), "r2x_fdk_backproject")
    assert _bits(vol).equal(_bits(_fdk(case, pt)))


def test_fdk_refuses_rows_wider_than_the_limit():
    torch = _torch()
    from r2_gaussian_b200._lib import R2XError, load
    from r2_gaussian_b200.fdk import fdk

    W = ct.K["FDK_MAX_W"] + 1
    sc = ct._scanner("cone", (1, W), (4, 4, 4))
    pt = torch.zeros((2, 1, W), dtype=torch.float32, device="cuda")
    with pytest.raises(R2XError, match=rf"r2x_fdk: bad W \(detector rows wider than {W - 1} pixels\)"):
        fdk(pt, [0.0, 1.0], sc)
    lib = load()
    q = torch.empty_like(pt)
    assert lib.r2x_fdk_filter(torch.cuda.current_stream().cuda_stream, 2, 1, W, pt.data_ptr(), 0.3, 0.3, 1, 5.0,
                              q.data_ptr()) != 0
    assert lib.r2x_last_error().decode() == "r2x_fdk_filter: bad N/H/W"


@pytest.mark.parametrize("nonneg", [True, False])
@pytest.mark.parametrize("name", sorted(ct.TV_CASES))
def test_tv_prox_matches_float64_fgp(name, nonneg):
    torch = _torch()
    from r2_gaussian_b200.tv import tv_denoise

    case = ct.TV_CASES[name]
    v = ct.tv_inputs(case)
    vt = torch.tensor(v, device="cuda")
    got = tv_denoise(vt, 0.1, case.niter, nonneg)
    assert _bits(got).equal(_bits(tv_denoise(vt, 0.1, case.niter, nonneg)))   # bitwise reproducible
    got = got.cpu().numpy()
    want = tvo.fgp(v, 0.1, case.niter, nonneg)[0]
    scale = np.abs(want).max()
    print(f"{name} nonneg {nonneg}: max err / max = {_max_err(got, want) / max(scale, 1e-30):.3g}")
    assert _max_err(got, want) <= PROX_BOUND * scale, (_max_err(got, want), scale)
    if nonneg:
        assert got.min() >= 0.0


@pytest.mark.parametrize("name", sorted(ct.TV_CASES))
def test_tv_value_matches_float64(name):
    torch = _torch()
    from r2_gaussian_b200.tv import tv_value

    case = ct.TV_CASES[name]
    v = np.abs(ct.tv_inputs(case))
    vt = torch.tensor(v, device="cuda")
    got = tv_value(vt)
    assert got == tv_value(vt)
    want = tvo.tv_value(v)
    print(f"{name}: {got!r} vs {want!r}")
    if want == 0.0:                                                            # a single voxel has no differences
        assert got == 0.0
    else:
        assert abs(got - want) <= VALUE_BOUND * want, (got, want)
