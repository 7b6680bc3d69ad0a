"""The CT edge cases (tests/ct_edge_cases.py) without a GPU: each sits on the side of the limit it claims, with the limits
read from the CUDA sources; the float64 oracles are adjoint at every projector-pair case; the FDK oracle's filter is
the direct convolution; and the all-views-in-one-call oracle is the per-view one."""
import math
from dataclasses import replace

import numpy as np
import pytest

import backproject_oracle as bo
import ct_edge_cases as ct
import offset_detector_oracle as oo
from oracle import fdk_oracle
from oracle import projector_oracle as po
from r2_gaussian_b200 import scene


def test_limits_are_read_from_the_sources():
    k = ct.K
    for name in ("PRJ_BV", "PRJ_BU", "PRJ_MAX_VIEWS", "BP_BZ", "BP_BY", "BP_CHUNK", "FDK_MAX_W", "FDK_BX", "FDK_BY",
                 "FDK_ZR", "FDK_VCHUNK", "TV_TX", "TV_TY", "TV_TZ", "TVV_THREADS", "TVV_MAX_BLOCKS", "TVV_PER_BLOCK",
                 "FDK_FILTER_THREADS", "FDK_SMEM_DEFAULT"):
        assert isinstance(k[name], int) and k[name] > 1, name
    # the filter stages 3 W + ceil(W / 2) floats; its default limit is 48 KiB, so 3511 is the first width that opts in
    assert [ct.filter_smem(W) for W in (1, 2, 3510, 3511)] == [16, 28, 49140, 49156]
    assert k["FDK_SMEM_DEFAULT"] == 48 * 1024 and ct.first_opt_in_width() == 3511
    assert ct.filter_smem(k["FDK_MAX_W"]) <= ct.H100_SMEM_OPTIN
    assert ct.tv_value_blocks(1) == (1, 1) and ct.tv_value_blocks(163 * 127 * 129) == (1024, 2608)


def test_every_case_claims_something():
    for case in ct.ALL_CASES.values():
        assert case.claims and case.boundary, case.name


@pytest.mark.parametrize("name", sorted(ct.ALL_CASES))
def test_case_lands_where_it_claims(name):
    case = ct.ALL_CASES[name]
    assert ct.claim_failures(case) == [], (case.boundary, ct.claim_failures(case))


def test_off_detector_cases_reach_nothing():
    """The box off the detector: the oracle's projections of any volume and its backprojection of any y are exactly 0."""
    for mode in ("cone", "parallel"):
        case = ct.PAIR_CASES[f"box_off_detector_{mode}"]
        x, y = ct.pair_inputs(case)
        vs = ct.views(case)
        assert not ct.project_views(x, vs, case.sc).any()
        assert not ct.backproject_views(y, vs, case.sc).any()


@pytest.mark.parametrize("name", sorted(ct.PAIR_CASES))
def test_oracles_are_adjoint(name):
    case = ct.PAIR_CASES[name]
    x, y = ct.pair_inputs(case)
    vs = ct.views(case)
    ax = ct.project_views(x, vs, case.sc, *ct.shift(case))
    aty = ct.backproject_views(y, vs, case.sc, *ct.shift(case))
    lhs, rhs = float((ax * y).sum()), float((x * aty).sum())
    assert abs(lhs - rhs) <= 1e-12 * max(abs(lhs), abs(rhs)), (lhs, rhs)
    if not name.startswith("box_off_detector"):
        assert lhs > 0.0


def _direct_filter(projs, tan_fovx, tan_fovy, mode, dso):
    """fdk_oracle.filter_projections by the O(W^2) sum over every pair of pixels of a row."""
    p = np.asarray(projs, np.float64)
    N, H, W = p.shape
    if mode == 1:
        a = ((2.0 * np.arange(W) + 1.0) / W - 1.0) * tan_fovx
        b = ((2.0 * np.arange(H) + 1.0) / H - 1.0) * tan_fovy
        p = p / np.sqrt(1.0 + a[None, None, :] ** 2 + b[None, :, None] ** 2)
    D = fdk_oracle.ramp_pitch(W, tan_fovx, mode, dso)
    q = np.zeros_like(p)
    for j in range(W):
        for i in range(W):
            k = abs(j - i)
            h = 1.0 / (4.0 * D * D) if k == 0 else (-1.0 / (math.pi ** 2 * k * k * D * D) if k % 2 else 0.0)
            q[..., j] += h * p[..., i]
    return q * D


@pytest.mark.parametrize("mode", [1, 0])
@pytest.mark.parametrize("W", [1, 2, ct.K["FDK_FILTER_THREADS"] + 1])
def test_fdk_oracle_filter_is_the_direct_convolution(W, mode):
    p = np.random.RandomState(W).uniform(0.0, 1.0, (2, 3, W))
    want = _direct_filter(p, 0.4, 0.3, mode, 5.0)
    got = fdk_oracle.filter_projections(p, 0.4, 0.3, mode, 5.0)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()


@pytest.mark.parametrize("use_off", [False, True])
@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_all_views_in_one_call_is_the_per_view_oracle(mode, use_off):
    sc = ct._scanner(mode, (5, 7), (6, 5, 4), (1.4, 1.2, 1.0), (0.1, -0.1, 0.05))
    if use_off:
        sc = ct._offset(sc, 1.6, -0.7)
    angles = [0.0, 0.9, math.pi / 2, 2.6, 4.4]
    rng = np.random.RandomState(3)
    x = rng.uniform(0.0, 1.0, (6, 5, 4)).astype(np.float32)
    y = rng.uniform(0.0, 1.0, (5, 5, 7)).astype(np.float32)
    vs = [scene.make_view(sc, a, use_off) for a in angles]
    t = scene.detector_shift(sc) if use_off else (0.0, 0.0)
    got_p, got_b = ct.project_views(x, vs, sc, *t), ct.backproject_views(y, vs, sc, *t)
    if use_off:
        want_p, want_b = oo.project_scene(x, angles, sc), oo.backproject_scene(y, angles, sc)
    else:
        want_p, want_b = po.project_scene(x, angles, sc), bo.backproject_scene(y, angles, sc)
    assert got_p.shape == want_p.shape and got_b.shape == want_b.shape
    assert np.abs(want_p).min() < np.abs(want_p).max()
    assert np.abs(got_p - want_p).max() <= 1e-13 * np.abs(want_p).max()
    assert np.abs(got_b - want_b).max() <= 1e-13 * np.abs(want_b).max()


@pytest.mark.parametrize("weighting", ["plain", "parker", "half_fan"])
@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_fdk_case_oracle_is_the_existing_statement(mode, weighting):
    """fdk_want of a weighting case equals the oracle that states that weighting (fdk_oracle, the short-scan oracle,
    the offset oracle); for Parker, on the case without its vertical offset, which the short-scan oracle lacks."""
    import fdk_short_scan_oracle as so

    case = ct.FDK_CASES[f"fdk_{weighting}_{mode}_H1"]
    projs = ct.fdk_inputs(case)
    if weighting == "plain":
        want = fdk_oracle.fdk_scene(projs, case.angles, case.sc)
    elif weighting == "parker":
        case = replace(case, sc=dict(case.sc, offDetector=[0.0, 0.0]))
        want = so.fdk_short_scan_scene(projs, case.angles, case.sc)
    else:
        want = oo.fdk_scene(projs, case.angles, case.sc, half_fan=True)
    got = ct.fdk_want(case, projs)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()


def test_vertical_offset_moves_the_parker_case():
    """The Parker case's vertical offset is not a no-op in its oracle (H = 1: the cosine weight's row moves)."""
    case = ct.FDK_CASES["fdk_parker_cone_H1"]
    projs = ct.fdk_inputs(case)
    centred = replace(case, sc=dict(case.sc, offDetector=[0.0, 0.0]))
    a, b = ct.fdk_want(case, projs), ct.fdk_want(centred, projs)
    assert np.abs(a - b).max() > 1e-3 * np.abs(b).max()
