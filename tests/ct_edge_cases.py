"""Inputs of the CT operators that sit on their kernels' tilings, chunk sizes and launch limits, a float64 oracle of the
projector pair that runs all views in one call, and the claim each case makes about where it sits.

The projector (r2x_project.cu), its matched backprojector (r2x_backproject.cu), FDK (r2x_fdk.cu) and the TV kernels
(r2x_tv.cu) tile detectors, grids and view lists with fixed CTA shapes and chunk sizes, and switch launch paths on
sizes (views per launch, the filter's shared-memory opt-in, the TV value's per-block chunk).  Index arithmetic goes wrong
on either side of such a limit and at size 1, so each case here lands on a stated side of one.  Every limit is read from
the CUDA sources by regular expression, as `regime_cases.read_constants` does for the binning: a retuned constant moves
the cases with it, and a renamed one fails the suite.  Each case carries `claims`, expressions over those constants and
over quantities of the case (`quantities`), which tests/test_ct_edges_cpu.py evaluates without a GPU, so a case cannot
quietly stop sitting where its name says.  tests/test_ct_edges_gpu.py runs every case against the float64 oracles.

`project_views` / `backproject_views` stack the rays of all views and make one `project_rays` / `backproject_rays`
call: the per-view `project_scene` costs a few milliseconds per view, minutes for the 65 537-view case.
"""
from __future__ import annotations

import math
import re
from dataclasses import dataclass, replace

import numpy as np

import backproject_oracle as bo
import fdk_cases as fc
import offset_detector_oracle as oo
from fdk_short_scan_oracle import fan_angles, parker_weights
from oracle import fdk_oracle
from oracle import projector_oracle as po
from r2_gaussian_b200 import scene
from regime_cases import _find, _source

# shared memory one H100 CTA can opt in to (cudaDevAttrMaxSharedMemoryPerBlockOptin: 227 KB)
H100_SMEM_OPTIN = 227 * 1024


def _constexpr(name: str, text: str, env: dict) -> int:
    """The value of `constexpr <type> ... NAME = <expr>` (one of several declarators is fine), <expr> over `env`."""
    m = _find(rf"constexpr\s+(?:int|long long|unsigned)\s+[^;]*?\b{name}\s*=\s*([^,;]+)[,;]", text, name)
    return int(eval(m.group(1), {"__builtins__": {}}, dict(env)))


def read_constants() -> dict:
    """The tile shapes, chunk sizes and launch limits of the CT kernels, as the CUDA sources state them."""
    src = {f: _source(f) for f in ("r2x_project.cu", "r2x_backproject.cu", "r2x_fdk.cu", "r2x_tv.cu")}
    names = {"r2x_project.cu": ("PRJ_BV", "PRJ_BU", "PRJ_MAX_VIEWS"),
             "r2x_backproject.cu": ("BP_BZ", "BP_BY", "BP_CHUNK"),
             "r2x_fdk.cu": ("FDK_MAX_W", "FDK_BX", "FDK_BY", "FDK_ZR", "FDK_VCHUNK"),
             "r2x_tv.cu": ("TV_TX", "TV_TY", "TV_TZ", "TVV_THREADS", "TVV_MAX_BLOCKS", "TVV_PER_BLOCK")}
    k: dict = {}
    for f, ns in names.items():
        for name in ns:
            k[name] = _constexpr(name, src[f], k)
    fdk = src["r2x_fdk.cu"]
    k["FDK_FILTER_THREADS"] = int(_find(r"__launch_bounds__\(([0-9]+)\) fdk_filter_kernel", fdk,
                                        "fdk_filter_kernel's threads per row").group(1))
    # the filter's dynamic shared memory in floats, a C expression in W, and the size above which it opts in
    k["FDK_SMEM_FLOATS"] = _find(r"fdk_filter_smem\(int W\) \{ return \(size_t\)\((.+)\) \* sizeof\(float\); \}", fdk,
                                 "fdk_filter_smem").group(1)
    m = _find(r"if \(smem > ([0-9]+) \* ([0-9]+)\)", fdk, "the filter's opt-in size")
    k["FDK_SMEM_DEFAULT"] = int(m.group(1)) * int(m.group(2))
    return k


K = read_constants()


def filter_smem(W: int) -> int:
    """fdk_filter_smem(W) in bytes (C integer division of non-negative ints is floor division)."""
    return 4 * int(eval(re.sub(r"/", "//", K["FDK_SMEM_FLOATS"]), {"__builtins__": {}}, {"W": int(W)}))


def first_opt_in_width() -> int:
    """The narrowest detector row whose filter needs more than the default shared memory."""
    W = 1
    while filter_smem(W) <= K["FDK_SMEM_DEFAULT"]:
        W += 1
    return W


def tv_value_blocks(nvox: int) -> tuple[int, int]:
    """(blocks, chunk) of r2x_tv_value: ceil(nvox / per-block) blocks capped at TVV_MAX_BLOCKS, chunk = ceil(nvox / nb)."""
    nb = min(max(-(-nvox // K["TVV_PER_BLOCK"]), 1), K["TVV_MAX_BLOCKS"])
    return nb, -(-nvox // nb)


@dataclass
class Case:
    name: str
    kind: str                     # "pair" (project + backproject), "fdk" or "tv"
    boundary: str                 # the limit it lands on, in words
    claims: tuple                 # expressions over K and `quantities` that must hold
    sc: dict | None = None
    angles: np.ndarray | None = None
    seed: int = 0
    use_off: bool = False         # through the scanner's offDetector (use_offDetector=True)
    weighting: str = "plain"      # fdk: "plain", "parker" (short_scan) or "half_fan"
    axis_aligned: bool = False    # pair: views whose matrices have their rounding residues set to exact zeros
    shape: tuple | None = None    # tv
    niter: int = 7                # tv


def _scanner(mode, det_hw, vox, s_voxel=(1.2, 1.4, 1.0), off=(0.05, -0.1, 0.08), accuracy=0.5, **over) -> dict:
    sc = fc.scanner(mode, 8, 8)
    sc["nDetector"] = [int(det_hw[0]), int(det_hw[1])]
    if mode == "cone":
        sc["sDetector"] = [3.0, 4.0]
    sc["nVoxel"], sc["sVoxel"], sc["offOrigin"] = [int(v) for v in vox], list(s_voxel), list(off)
    sc["accuracy"] = accuracy
    sc.update(over)
    return sc


def _offset(sc: dict, t_u: float, t_v: float) -> dict:
    du, dv = sc["sDetector"][1] / sc["nDetector"][1], sc["sDetector"][0] / sc["nDetector"][0]
    return dict(sc, offDetector=[t_u * du, t_v * dv])


def _angles(seed: int, n: int) -> np.ndarray:
    return np.random.RandomState(1000 + seed).uniform(0.0, 2.0 * math.pi, n)


def _pair_cases() -> list[Case]:
    BV, BU, C, BZ, BY = K["PRJ_BV"], K["PRJ_BU"], K["BP_CHUNK"], K["BP_BZ"], K["BP_BY"]
    out = []
    seed = 0
    # the projector's 32 x 8 CTA: detector rows and columns on either side of it, and a single row or column
    for mode in ("cone", "parallel"):
        for H, hs in ((1, "1"), (BV - 1, "PRJ_BV - 1"), (BV, "PRJ_BV"), (BV + 1, "PRJ_BV + 1")):
            for W, ws in ((1, "1"), (BU - 1, "PRJ_BU - 1"), (BU, "PRJ_BU"), (BU + 1, "PRJ_BU + 1")):
                seed += 1
                out.append(Case(f"det_{mode}_{H}x{W}", "pair", f"projector CTA: H = {hs}, W = {ws}",
                                (f"H == {hs}", f"W == {ws}"), _scanner(mode, (H, W), (5, 6, 7)), _angles(seed, 2), seed))
    # a grid with one voxel along an axis
    for mode in ("cone", "parallel"):
        for a, vox, sv in ((0, (1, 6, 7), (0.3, 1.4, 1.0)), (1, (5, 1, 7), (1.2, 0.3, 1.0)),
                           (2, (5, 6, 1), (1.2, 1.4, 0.3))):
            seed += 1
            ax = "xyz"[a]
            out.append(Case(f"grid_{mode}_n{ax}1", "pair", f"a size-1 grid axis: n{ax} = 1", (f"n{ax} == 1",),
                            _scanner(mode, (9, 10), vox, sv), _angles(seed, 3), seed))
    # parallel beam along the grid axes: with the matrices' rounding residues zeroed, direction components are exactly
    # 0 (the slab test's st == 0 branch); through make_view they are ~1e-16 instead
    quarter = np.array([0.0, 0.5, 1.0, 1.5]) * math.pi
    out.append(Case("parallel_axis_aligned_exact", "pair", "parallel rays with direction components exactly 0",
                    ("st_zero > 0",), _scanner("parallel", (7, 9), (5, 6, 7)), quarter, 71, axis_aligned=True))
    out.append(Case("parallel_axis_aligned", "pair", "parallel rays at 0, pi/2, pi, 3 pi/2 through make_view",
                    ("N == 4",), _scanner("parallel", (7, 9), (5, 6, 7)), quarter, 72))
    # more views than one projector launch takes (grid.z): the chunk loop's second pass
    out.append(Case("views_max_plus_2", "pair", "projector view chunks: N = PRJ_MAX_VIEWS + 2",
                    ("N == PRJ_MAX_VIEWS + 2",),
                    _scanner("cone", (2, 3), (4, 4, 4), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0)),
                    _angles(73, K["PRJ_MAX_VIEWS"] + 2), 73))
    # the source inside the box: the cone-beam cut t > 0 of the projector, the backprojector's `behind` footprint
    out.append(Case("source_inside_box", "pair", "cone source inside the box (t > 0 cut, backprojector's behind)",
                    ("source_inside", "cut_margin > 1e-6", "behind_voxels > 0", "front_voxels > 0"),
                    _scanner("cone", (11, 13), (6, 5, 7), (3.0, 3.0, 3.0), (0.1, -0.05, 0.0), DSO=1.2, DSD=2.4,
                             sDetector=[4.0, 4.0]), _angles(74, 3), 74))
    # a box that lies entirely off the detector: every ray misses it, no ray reaches any voxel
    for mode in ("cone", "parallel"):
        out.append(Case(f"box_off_detector_{mode}", "pair", "box off the detector: all projections exactly 0",
                        ("oracle_max == 0",), _scanner(mode, (6, 7), (4, 5, 3), (1.0, 1.0, 1.0), (0.0, 0.0, 3.0)),
                        _angles(75, 3), 75))
    # the backprojector's view chunks (ray tables and matrix staging)
    for N, ns in ((1, "1"), (C - 1, "BP_CHUNK - 1"), (C, "BP_CHUNK"), (C + 1, "BP_CHUNK + 1"),
                  (2 * C + 1, "2 * BP_CHUNK + 1")):
        seed += 1
        out.append(Case(f"bp_views_{N}", "pair", f"backprojector view chunks: N = {ns}", (f"N == {ns}",),
                        _scanner("cone", (5, 6), (4, 5, 6)), _angles(seed, N), seed))
    # the backprojector's 32 (z) x 4 (y) gather CTA, nx = 1
    for nz, zs in ((1, "1"), (BZ - 1, "BP_BZ - 1"), (BZ, "BP_BZ"), (BZ + 1, "BP_BZ + 1")):
        for ny, ys in ((1, "1"), (BY - 1, "BP_BY - 1"), (BY, "BP_BY"), (BY + 1, "BP_BY + 1")):
            seed += 1
            out.append(Case(f"bp_grid_1x{ny}x{nz}", "pair", f"backprojector CTA: nz = {zs}, ny = {ys}, nx = 1",
                            (f"nz == {zs}", f"ny == {ys}", "nx == 1"),
                            _scanner("cone", (6, 7), (1, ny, nz), (0.4, 1.2, 1.6)), _angles(seed, 2), seed))
    # an offset detector with a single row
    for mode in ("cone", "parallel"):
        seed += 1
        out.append(Case(f"offset_{mode}_H1", "pair", "offset detector, H = 1", ("H == 1", "t_u != 0", "t_v != 0"),
                        _offset(_scanner(mode, (1, 12), (5, 6, 7)), 2.4, 0.3), _angles(seed, 3), seed, use_off=True))
    return out


def _fdk_cases() -> list[Case]:
    T, BX, BY, ZR, VC = K["FDK_FILTER_THREADS"], K["FDK_BX"], K["FDK_BY"], K["FDK_ZR"], K["FDK_VCHUNK"]
    full = lambda n: fc.full_scan(n) + 0.2                               # noqa: E731
    out = []
    # the filter's threads per detector row
    for W, ws in ((1, "1"), (2, "2"), (T - 1, "FDK_FILTER_THREADS - 1"), (T, "FDK_FILTER_THREADS"),
                  (T + 1, "FDK_FILTER_THREADS + 1")):
        out.append(Case(f"fdk_W{W}", "fdk", f"filter threads per row: W = {ws}", (f"W == {ws}",),
                        _scanner("cone", (3, W), (5, 6, 7)), full(4), W))
    # either side of the filter's shared-memory opt-in, and the widest row it takes
    Wo = first_opt_in_width()
    out.append(Case(f"fdk_W{Wo - 1}_H1", "fdk", "filter shared memory: the widest row without the opt-in",
                    ("H == 1", "filter_smem(W) <= FDK_SMEM_DEFAULT", "filter_smem(W + 1) > FDK_SMEM_DEFAULT"),
                    _scanner("cone", (1, Wo - 1), (5, 6, 7)), full(3), 11))
    out.append(Case(f"fdk_W{Wo}_H1", "fdk", "filter shared memory: the narrowest row with the opt-in",
                    ("H == 1", "filter_smem(W) > FDK_SMEM_DEFAULT", "filter_smem(W - 1) <= FDK_SMEM_DEFAULT"),
                    _scanner("cone", (1, Wo), (5, 6, 7)), full(3), 12))
    out.append(Case("fdk_W_max_H1", "fdk", "filter: W = FDK_MAX_W",
                    ("W == FDK_MAX_W", "H == 1", "N == 2", "filter_smem(W) <= H100_SMEM_OPTIN"),
                    _scanner("cone", (1, K["FDK_MAX_W"]), (5, 6, 7)), full(2), 13))
    # the backprojection's 32 (y) x 4 (x) CTA and its 8-voxel z run, and a 1^3 grid
    for d, ds in ((-1, " - 1"), (0, ""), (1, " + 1")):
        out.append(Case(f"fdk_grid_{BY + d}x{BX + d}x{ZR + d}", "fdk", f"FDK CTA: ny = FDK_BX{ds}, nx = FDK_BY{ds}, "
                        f"nz = FDK_ZR{ds}", (f"ny == FDK_BX{ds}", f"nx == FDK_BY{ds}", f"nz == FDK_ZR{ds}"),
                        _scanner("cone", (8, 10), (BY + d, BX + d, ZR + d), (1.0, 1.6, 1.2)), full(5), 20 + d))
    out.append(Case("fdk_grid_1x1x1", "fdk", "a 1^3 grid", ("nx == 1", "ny == 1", "nz == 1"),
                    _scanner("cone", (8, 10), (1, 1, 1), (0.4, 0.4, 0.4)), full(5), 22))
    # the backprojection's view staging
    for N, ns in ((VC, "FDK_VCHUNK"), (VC + 1, "FDK_VCHUNK + 1")):
        out.append(Case(f"fdk_views_{N}", "fdk", f"FDK view staging: N = {ns}", (f"N == {ns}",),
                        _scanner("cone", (6, 8), (4, 5, 6)), full(N), 30 + N))
    # each weighting in both beams on a single detector row
    for mode in ("cone", "parallel"):
        sc = _scanner(mode, (1, 24), (5, 6, 7))
        out.append(Case(f"fdk_plain_{mode}_H1", "fdk", "plain weights, H = 1", ("H == 1",), sc, full(12), 40))
        # a short scan: Parker weights, a vertical offset only
        arc = math.radians(240.0 if mode == "cone" else 200.0)
        out.append(Case(f"fdk_parker_{mode}_H1", "fdk", "Parker weights with a vertical offset, H = 1",
                        ("H == 1", "t_u == 0", "t_v != 0"), _offset(sc, 0.0, 0.3),
                        np.linspace(0.0, arc, 19)[:-1] + 0.3, 41, use_off=True, weighting="parker"))
        # half-fan weights with the rotation axis close to the detector's edge
        out.append(Case(f"fdk_half_fan_{mode}_H1", "fdk", "half-fan weights, |t_u| close to W / 2, H = 1",
                        ("H == 1", "abs(t_u) > 0.45 * W", "abs(t_u) < 0.5 * W"), _offset(sc, -11.3, 0.0), full(12),
                        42, use_off=True, weighting="half_fan"))
    # the source inside the box: voxels behind it (z_view <= 0) are skipped
    out.append(Case("fdk_source_inside_box", "fdk", "cone source inside the box (z_view <= 0 skip)",
                    ("source_inside", "zv_behind > 0", "zv_margin > 0.05"),
                    _scanner("cone", (11, 13), (6, 5, 7), (3.0, 3.0, 3.0), (0.1, -0.05, 0.0), DSO=1.2, DSD=2.4,
                             sDetector=[4.0, 4.0]), _angles(32, 6), 50))
    return out


def _tv_cases() -> list[Case]:
    TX, TY, TZ = K["TV_TX"], K["TV_TY"], K["TV_TZ"]
    out = [Case("tv_tile", "tv", "TV tile: one whole tile", ("nx == TV_TX", "ny == TV_TY", "nz == TV_TZ"),
                shape=(TX, TY, TZ), seed=1),
           Case("tv_tile_plus_1", "tv", "TV tile: one more voxel on each axis",
                ("nx == TV_TX + 1", "ny == TV_TY + 1", "nz == TV_TZ + 1"), shape=(TX + 1, TY + 1, TZ + 1), seed=2),
           Case("tv_tile_minus_1", "tv", "TV tile: one voxel short on each axis",
                ("nx == TV_TX - 1", "ny == TV_TY - 1", "nz == TV_TZ - 1"), shape=(TX - 1, TY - 1, TZ - 1), seed=3),
           Case("tv_1x1x2tz", "tv", "TV: a single line of two tiles along z", ("nx == 1", "ny == 1", "nz == 2 * TV_TZ"),
                shape=(1, 1, 2 * TZ), seed=4),
           Case("tv_2x1x1", "tv", "TV: two voxels along x", ("nx == 2", "ny == 1", "nz == 1"), shape=(2, 1, 1), seed=5),
           Case("tv_1x1x1", "tv", "TV: one voxel", ("nvox == 1",), shape=(1, 1, 1), seed=6),
           # above TVV_MAX_BLOCKS blocks of TVV_PER_BLOCK voxels each block's chunk grows; a count that is not a multiple
           # of the block count leaves the last block short, where a truncated chunk would drop voxels
           Case("tv_value_big", "tv", "TV value: chunk above TVV_PER_BLOCK, last block short",
                ("nvox > TVV_MAX_BLOCKS * TVV_PER_BLOCK", "TVV_PER_BLOCK == 8 * TVV_THREADS", "nb == TVV_MAX_BLOCKS",
                 "nvox % TVV_MAX_BLOCKS != 0", "chunk > TVV_PER_BLOCK", "nvox - (nb - 1) * chunk < chunk"),
                shape=(163, 127, 129), seed=7, niter=3)]
    return out


PAIR_CASES = {c.name: c for c in _pair_cases()}
FDK_CASES = {c.name: c for c in _fdk_cases()}
TV_CASES = {c.name: c for c in _tv_cases()}
ALL_CASES = {**PAIR_CASES, **FDK_CASES, **TV_CASES}
assert len(ALL_CASES) == len(PAIR_CASES) + len(FDK_CASES) + len(TV_CASES), "case names must be unique"


# ---- geometry and the float64 oracles ---------------------------------------------------------------------------------

def _snap(view: scene.View) -> scene.View:
    """The view with the rounding residues of its matrices (|m| < 1e-12, e.g. cos(pi / 2)) set to exact zeros."""
    vm, pm = view.viewmatrix.copy(), view.projmatrix.copy()
    vm[np.abs(vm) < 1e-12] = 0.0
    pm[np.abs(pm) < 1e-12] = 0.0
    return replace(view, viewmatrix=vm, projmatrix=pm)


def views(case: Case) -> list[scene.View]:
    """The views the GPU operators use for `case` (offset projmatrices when use_off)."""
    out = [scene.make_view(case.sc, float(a), case.use_off) for a in case.angles]
    return [_snap(v) for v in out] if case.axis_aligned else out


def shift(case: Case) -> tuple[float, float]:
    return scene.detector_shift(case.sc) if case.use_off else (0.0, 0.0)


def stacked_rays(vs, t_u: float = 0.0, t_v: float = 0.0):
    """Origins and unit directions [N, H, W, 3] of every pixel of every view (detector offset by (t_u, t_v) pixels)."""
    o, d = zip(*(oo.rays(v, t_u, t_v) for v in vs))
    return np.stack(o), np.stack(d)


def project_views(volume, vs, sc: dict, t_u: float = 0.0, t_v: float = 0.0) -> np.ndarray:
    """po.project_scene (or oo.project_scene with an offset) of `volume` for the views `vs`, in one project_rays call."""
    o, d = stacked_rays(vs, t_u, t_v)
    return po.project_rays(volume, o, d, vs[0].mode == 1, sc["sVoxel"], sc["offOrigin"], po.step_length(sc))


def backproject_views(y, vs, sc: dict, t_u: float = 0.0, t_v: float = 0.0) -> np.ndarray:
    """The exact transpose of `project_views`, in one backproject_rays call."""
    o, d = stacked_rays(vs, t_u, t_v)
    return bo.backproject_rays(y, o, d, vs[0].mode == 1, tuple(int(v) for v in sc["nVoxel"]), sc["sVoxel"],
                               sc["offOrigin"], po.step_length(sc))


def fdk_want(case: Case, projs) -> np.ndarray:
    """fdk(projs, case.angles, case.sc, short_scan=parker, use_offDetector=case.use_off, half_fan=half_fan) in
    float64: the offset oracle's filter (cosine and half-fan weights at the offset ndc), Parker weights before it for a
    short scan (scale 1 instead of pi / N), then the plain backprojection through the case's matrices."""
    from r2_gaussian_b200.fdk import short_scan_views

    vs = views(case)
    v0, dso = vs[0], float(case.sc["DSO"])
    p = np.asarray(projs, np.float64)
    scale = 1.0
    if case.weighting == "parker":
        vw, arc = short_scan_views(case.angles, v0.mode, v0.tanfovx)
        w = parker_weights(vw[:, :1], fan_angles(p.shape[2], v0.tanfovx, v0.mode)[None, :], arc)
        p = p * (w * vw[:, 1:])[:, None, :]
        scale = len(vs) / math.pi
    q = oo.filter_projections(p, v0.tanfovx, v0.tanfovy, v0.mode, dso, *shift(case), case.weighting == "half_fan")
    return scale * fdk_oracle.backproject(q, [v.viewmatrix for v in vs], [v.projmatrix for v in vs], v0.mode, dso,
                                          case.sc["nVoxel"], case.sc["sVoxel"], case.sc["offOrigin"])


def pair_inputs(case: Case):
    """(x [nx, ny, nz], y [N, H, W]) float32, positive, seeded by the case."""
    rng = np.random.RandomState(case.seed)
    x = rng.uniform(0.1, 1.0, tuple(case.sc["nVoxel"])).astype(np.float32)
    y = rng.uniform(0.1, 1.0, (len(case.angles), *case.sc["nDetector"])).astype(np.float32)
    return x, y


def fdk_inputs(case: Case, smooth: bool | None = None) -> np.ndarray:
    """Projections [N, H, W] float32 seeded by the case: uniform noise, or with `smooth` (by default for rows wider than
    SMOOTH_ABOVE pixels) a sinusoid of SMOOTH_CYCLES cycles per pixel under a sin^2 window along each row.  The
    backprojection samples the filtered rows at float32 pixel coordinates, whose rounding (ulp(W / 2): 1e-3 pixel at
    W = 16384) times the pixel-to-pixel jumps of filtered noise grows with W and passes the 1e-4 bar near W = 2000; the
    smooth row keeps that term near 3e-5 at W = 16384, and its filtered values, small differences of large sums, expose
    a filter that drops its small taps.  The filter alone is compared on noise at every width."""
    N, H, W = len(case.angles), *case.sc["nDetector"]
    rng = np.random.RandomState(case.seed)
    if not (W > SMOOTH_ABOVE if smooth is None else smooth):
        return rng.uniform(0.0, 1.0, (N, H, W)).astype(np.float32)
    u = (np.arange(W) + 0.5) / W
    amp, phase = rng.uniform(0.5, 1.0, (N, H, 1)), rng.uniform(0.0, 2.0 * math.pi, (N, H, 1))
    wave = np.sin(2.0 * math.pi * SMOOTH_CYCLES * np.arange(W) + phase)
    return (amp * np.sin(math.pi * u) ** 2 * (0.6 + 0.4 * wave)).astype(np.float32)


SMOOTH_ABOVE, SMOOTH_CYCLES = 64, 0.005


def tv_inputs(case: Case) -> np.ndarray:
    return np.random.RandomState(case.seed).uniform(-0.3, 1.0, case.shape).astype(np.float32)


# ---- what a case claims ------------------------------------------------------------------------------------------------

def _voxel_grid(sc: dict):
    return np.meshgrid(*fdk_oracle.voxel_centres(sc["nVoxel"], sc["sVoxel"], sc["offOrigin"]), indexing="ij")


def _z_view(v: scene.View, X, Y, Z):
    return fdk_oracle._row(np.asarray(v.viewmatrix, np.float64).reshape(16), 2, X, Y, Z)


class _Quantities(dict):
    """The quantities a claim may name, computed on first use."""

    def __init__(self, case: Case):
        super().__init__(K)
        self.case = case
        self.update(filter_smem=filter_smem, abs=abs, H100_SMEM_OPTIN=H100_SMEM_OPTIN)

    def __missing__(self, name):
        self[name] = value = getattr(self, "_" + name)()
        return value

    # sizes
    def _N(self): return len(self.case.angles)
    def _H(self): return int(self.case.sc["nDetector"][0])
    def _W(self): return int(self.case.sc["nDetector"][1])
    def _nx(self): return int((self.case.shape or self.case.sc["nVoxel"])[0])
    def _ny(self): return int((self.case.shape or self.case.sc["nVoxel"])[1])
    def _nz(self): return int((self.case.shape or self.case.sc["nVoxel"])[2])
    def _nvox(self): return self["nx"] * self["ny"] * self["nz"]
    def _nb(self): return tv_value_blocks(self["nvox"])[0]
    def _chunk(self): return tv_value_blocks(self["nvox"])[1]
    def _t_u(self): return shift(self.case)[0]
    def _t_v(self): return shift(self.case)[1]

    # geometry
    def _source_inside(self):
        """Every view's source strictly inside the box offOrigin +- sVoxel / 2."""
        c, h = np.asarray(self.case.sc["offOrigin"], float), 0.5 * np.asarray(self.case.sc["sVoxel"], float)
        return all(bool((np.abs(np.asarray(v.campos, float) - c) < h).all()) for v in views(self.case))

    def _cut_margin(self):
        """The least distance of -t_c / step from an integer over all rays: the t > 0 cut is not on a rounding edge."""
        o, d = stacked_rays(views(self.case), *shift(self.case))
        r = -((np.asarray(self.case.sc["offOrigin"], float) - o) * d).sum(-1) / po.step_length(self.case.sc)
        f = r - np.floor(r)
        return float(np.minimum(f, 1.0 - f).min())

    def _corner_z(self):
        """Per view and voxel, the least z_view over the corners of the voxel's support box (x - 1, x + 1)^3."""
        sc = self.case.sc
        X, Y, Z = _voxel_grid(sc)
        dv = np.asarray(sc["sVoxel"], float) / np.asarray(sc["nVoxel"], float)
        out = []
        for v in views(self.case):
            m = np.asarray(v.viewmatrix, np.float64).reshape(16)
            out.append(_z_view(v, X, Y, Z) - (abs(m[2]) * dv[0] + abs(m[6]) * dv[1] + abs(m[10]) * dv[2]))
        return np.stack(out)

    def _behind_voxels(self):
        """(view, voxel) pairs whose support box has a corner at z_view <= 0: the backprojector's whole-detector path."""
        return int((self["corner_z"] <= 0.0).sum())

    def _front_voxels(self):
        return int((self["corner_z"] > 0.0).sum())

    def _zv(self):
        X, Y, Z = _voxel_grid(self.case.sc)
        return np.stack([_z_view(v, X, Y, Z) for v in views(self.case)])

    def _zv_behind(self):
        """(view, voxel) pairs with z_view <= 0 at the voxel centre: FDK skips them."""
        return int((self["zv"] <= 0.0).sum())

    def _zv_margin(self):
        return float(np.abs(self["zv"]).min())

    def _st_zero(self):
        """Rays with a direction component exactly 0 in the kernel's float64 setup (a zero column entry of the
        viewmatrix's rotation times the camera-frame direction (0, 0, 1))."""
        vm = np.stack([np.asarray(v.viewmatrix, np.float64).reshape(16) for v in views(self.case)])
        return int((vm[:, [2, 6, 10]] == 0.0).sum())

    def _oracle_max(self):
        x = np.ones(tuple(self.case.sc["nVoxel"]), np.float32)
        return float(np.abs(project_views(x, views(self.case), self.case.sc, *shift(self.case))).max())


def claim_failures(case: Case) -> list[str]:
    """The claims of `case` that do not hold (empty when it sits where it says)."""
    q = _Quantities(case)
    return [c for c in case.claims if not eval(c, {"__builtins__": {}}, q)]
