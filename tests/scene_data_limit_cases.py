"""Inputs of the scene-view rasterizer (r2x_scene.cu), the cubic B-spline zoom (r2x_zoom.cu), projection preparation
(r2x_prepare.cu) and the detector-offset gradient (r2x_detector.cu) at their launch limits and past 2^31 elements, the
windows the GPU tests compare against the oracles, and the claim each case makes about where it sits.

Every limit is read from the CUDA sources by regular expression, so a retuned constant moves the cases with it and a
renamed one fails the suite.  Each case carries `claims`, expressions over those constants and over quantities of the
case, which tests/test_scene_data_limits_cpu.py evaluates without a GPU, and its peak device memory (`peak`, bytes),
which tests/test_scene_data_limits_gpu.py compares with the free memory before it runs.

The scene tile kernel finds a tile's record by a binary search over the records' first tiles; `tile_search_midpoint`
is its midpoint expression, read from the source, and `tile_search` runs that search in 32-bit two's-complement
arithmetic, so the CPU tests can show that no probe leaves the record list at the largest list the API accepts.
"""
from __future__ import annotations

import ast
import functools
import math
import os
import re
from dataclasses import dataclass, field

import numpy as np

import gaussian_view_oracle as gvo
import scene_view_oracle as so
from ct_limit_cases import _constexpr
from regime_cases import _find, _source

INT_MAX = 2**31 - 1
GiB = 2**30
HDR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "r2x.h")


def read_constants() -> dict:
    """The scene rasterizer's launch limits, the zoom's size limit and padding, the gradient's block plan."""
    hdr = open(HDR).read()
    k: dict = {n: int(_find(rf"#define {n} (\d+)", hdr, n).group(1)) for n in ("R2X_SV_TILE", "R2X_SV_MAX_SIDE")}
    names = {"r2x_scene.cu": ("SV_TILE_CTAS", "SV_SCAN_THREADS", "SV_MAX_GRID"),
             "r2x_zoom.cu": ("ZOOM_MAX_DIM", "ZOOM_PAD"),
             "r2x_detector.cu": ("kThreads", "kMaxBlocks", "kPerBlock")}
    for f, ns in names.items():
        src = _source(f)
        for name in ns:
            k[name] = _constexpr(name, src, k)
    return k


K = read_constants()


def tiles(n: int, t: int) -> int:
    return -(-n // t)


@dataclass
class Case:
    name: str
    kind: str                 # "scene", "zoom", "prepare" or "grad"
    boundary: str             # the limit it lands on, in words
    claims: tuple             # expressions over K and the case's quantities that must hold
    extra: dict = field(default_factory=dict)
    peak: int = 0             # device bytes the GPU test needs at once


# ---- the scene tile search ----------------------------------------------------------------------------------------

def tile_search_midpoint() -> str:
    """The right-hand side of `const int mid = ...;` in sv_tile_kernel's record search."""
    src = re.sub(r"//[^\n]*", "", _source("r2x_scene.cu"))
    body = re.search(r"__global__[^{]*sv_tile_kernel\(.*?\n}\n", src, re.S)
    if body is None:
        raise LookupError("sv_tile_kernel: not found in r2x_scene.cu")
    return _find(r"const\s+int\s+mid\s*=\s*([^;]+);", body.group(0), "sv_tile_kernel midpoint").group(1).strip()


def _wrap32(v: int) -> int:
    return (v + 2**31) % 2**32 - 2**31


def eval_int32(expr: str, env: dict) -> int:
    """A C integer expression over `env` (+, -, *, /, >>, <<, unary -, parentheses) in 32-bit int: every operation
    wraps to two's complement, >> is arithmetic and / truncates towards zero, as the GPU computes it."""
    ops = {ast.Add: lambda a, b: a + b, ast.Sub: lambda a, b: a - b, ast.Mult: lambda a, b: a * b,
           ast.RShift: lambda a, b: a >> b, ast.LShift: lambda a, b: a << b,
           ast.Div: lambda a, b: (abs(a) // abs(b)) * (1 if (a >= 0) == (b > 0) else -1)}

    def ev(n):
        if isinstance(n, ast.Expression):
            return ev(n.body)
        if isinstance(n, ast.Constant) and isinstance(n.value, int):
            return _wrap32(n.value)
        if isinstance(n, ast.Name):
            return _wrap32(int(env[n.id]))
        if isinstance(n, ast.UnaryOp) and isinstance(n.op, ast.USub):
            return _wrap32(-ev(n.operand))
        if isinstance(n, ast.BinOp) and type(n.op) in ops:
            return _wrap32(ops[type(n.op)](ev(n.left), ev(n.right)))
        raise ValueError(f"eval_int32: cannot evaluate {ast.dump(n)} of {expr!r}")

    try:
        tree = ast.parse(expr, mode="eval")
    except SyntaxError as e:
        raise ValueError(f"eval_int32: {expr!r} is not a plain integer expression") from e
    return ev(tree)


def tile_search(nrec: int, t: int, base, mid_expr: str):
    """(record, probes) of sv_tile_kernel's search for tile t: the last record r with base(r) <= t, with the midpoint
    `mid_expr` in int32.  Stops at the first probe outside [0, nrec) (record None): the kernel would read rec[mid]
    outside the list there."""
    lo, hi = 0, nrec - 1
    probes = []
    while lo < hi:
        mid = eval_int32(mid_expr, {"lo": lo, "hi": hi})
        probes.append(mid)
        if not 0 <= mid < nrec:
            return None, probes
        if base(mid) <= t:
            lo = mid
        else:
            hi = mid - 1
    return lo, probes


# ---- scene cases --------------------------------------------------------------------------------------------------

LUT = np.array([[0.1, 0.2, 0.3], [0.9, 0.5, 0.1], [0.4, 1.0, 0.6]], np.float32)
NEAR = 1e-3
BG = (1.0, 1.0, 1.0)


@dataclass
class Scene:
    pos: np.ndarray           # float64 [n, 3, 3]
    meta: np.ndarray          # int32 [n, 2]
    attr: np.ndarray          # float32 [n, 12]
    tex: np.ndarray           # float32 [n_tex, th, tw] (a 1 x 1 x 1 zero texture when nothing is textured)
    cams: list                # the distinct cameras (volume_render.Camera)
    frames: int               # frame f is seen by cams[f % len(cams)]
    textured: bool = False

    @property
    def H(self):
        return self.cams[0].height

    @property
    def W(self):
        return self.cams[0].width

    @property
    def parallel(self):
        return self.cams[0].parallel

    def records(self, cam_index: int = 0) -> np.ndarray:
        """Tile counts of the records camera `cam_index` makes: one per primitive whose clamped pixel box (the
        oracles' boxes) is non-empty and wider or taller than R2X_SV_TILE pixels."""
        T = K["R2X_SV_TILE"]
        k = so.Cam(self.cams[cam_index].record(), self.H, self.W, self.parallel)
        ell = self.meta[:, 0] == gvo.ELLIPSOID
        boxes = []
        for i in np.nonzero(~ell)[0]:
            g = so.geometry(k, NEAR, self.pos[i], int(self.meta[i, 0]), self.attr[i, 3])
            if g is not None:
                boxes.append((g["x0"], g["x1"], g["y0"], g["y1"]))
        if ell.any():
            boxes += [tuple(b) for b in gvo.boxes(k, NEAR, gvo.Ellipsoids(self.pos[ell], self.attr[ell])).tolist()]
        b = np.array(boxes, np.int64).reshape(-1, 4)
        live = (b[:, 0] <= b[:, 1]) & (b[:, 2] <= b[:, 3])
        big = live & ((b[:, 1] - b[:, 0] >= T) | (b[:, 3] - b[:, 2] >= T))
        b = b[big]
        return ((b[:, 1] - b[:, 0]) // T + 1) * ((b[:, 3] - b[:, 2]) // T + 1)


def _lines(a, b, colours, width):
    n = len(a)
    pos = np.zeros((n, 3, 3))
    pos[:, 0], pos[:, 1] = a, b
    meta = np.zeros((n, 2), np.int32)
    meta[:, 0] = so.LINE
    attr = np.zeros((n, 12), np.float32)
    attr[:, 0:3] = colours
    attr[:, 3] = width
    return pos, meta, attr


def _ellipsoids(c, s, q, colours):
    n = len(c)
    pos = np.zeros((n, 3, 3))
    pos[:, 0], pos[:, 1] = c, s
    meta = np.zeros((n, 2), np.int32)
    meta[:, 0] = gvo.ELLIPSOID
    attr = np.zeros((n, 12), np.float32)
    attr[:, 0:3] = colours
    attr[:, 3:7] = q
    return pos, meta, attr


def _cat(*parts):
    return tuple(np.concatenate([p[i] for p in parts]) for i in range(3))


REC_LINES, REC_CAMS, REC_W = 17000, 7, 29


@functools.lru_cache(maxsize=None)
def records_scene() -> Scene:
    """n_frames = SV_MAX_GRID frames of a 1 x REC_W row, REC_LINES lines each clipped to the whole row (two tiles per
    (line, frame) record).  Seven parallel cameras shifted along the row take turns.  Line i's depth along the row is
    the tangent at s_i of the concave parabola 300 - x^2 / 100, so the nearest line at x is the one whose s_i is closest
    to x (ties in float32 to the lower id): each pixel's winner depends on the frame."""
    rng = np.random.default_rng(41)
    s = rng.permutation(np.linspace(-20.0, 52.0, REC_LINES))
    R, C = 50.0, 300.0
    x = np.array([-200.0, 200.0])
    depth = C + s[:, None] ** 2 / (2 * R) - s[:, None] * x[None, :] / R       # [n, 2], from 92 to 530
    a = np.stack([np.full(REC_LINES, x[0]), np.zeros(REC_LINES), 10.0 - depth[:, 0]], 1)
    b = np.stack([np.full(REC_LINES, x[1]), np.zeros(REC_LINES), 10.0 - depth[:, 1]], 1)
    pos, meta, attr = _lines(a, b, rng.random((REC_LINES, 3)), 1.5)
    from r2_gaussian_b200.volume_render import look_at

    cams = [look_at((5.3 * k, 0.0, 10.0), (5.3 * k, 0.0, 0.0), (0, 1, 0), REC_W, 1, parallel_scale=0.5)
            for k in range(REC_CAMS)]
    return Scene(pos, meta, attr, np.zeros((1, 1, 1), np.float32), cams, K["SV_MAX_GRID"])


def _soup(rng, n_tri, n_line, n_ell, spread, size, tex_shape=(7, 5)):
    """Random triangles (flat, mesh, textured on two textures), lines of several widths and ellipsoids."""
    c = rng.uniform(-spread, spread, (n_tri + n_line, 1, 3))
    pos = c + rng.normal(0, 1, (n_tri + n_line, 3, 3)) * rng.uniform(0.05, 1, (n_tri + n_line, 1, 1)) * size
    meta = np.zeros((len(pos), 2), np.int32)
    meta[:n_tri, 0] = rng.integers(0, 3, n_tri)
    meta[n_tri:, 0] = so.LINE
    meta[:, 1] = rng.integers(0, 2, len(pos))
    attr = rng.random((len(pos), 12)).astype(np.float32)
    attr[:, 3:12] = np.where((meta[:, 0] == so.MESH)[:, None], rng.normal(0, 1, (len(pos), 9)), attr[:, 3:12])
    attr[n_tri:, 3] = rng.choice([0.5, 1.0, 1.5, 3.0, 7.0], n_line)
    e = _ellipsoids(rng.uniform(-spread, spread, (n_ell, 3)), rng.uniform(0.05, 1.0, (n_ell, 3)) * size,
                    rng.normal(0, 1, (n_ell, 4)), rng.random((n_ell, 3)))
    pos, meta, attr = _cat((pos, meta, attr), e)
    return pos, meta, attr, rng.random((2,) + tex_shape).astype(np.float32)


PIX_FRAMES, PIX_SIDE = 8193, 512


@functools.lru_cache(maxsize=None)
def pixels_scene() -> Scene:
    """An orbit of PIX_FRAMES frames of PIX_SIDE^2 pixels: more than 2^31 pixels in one call, the last frame starting
    at pixel 2^31, over a soup of triangles, textured triangles, lines and ellipsoids."""
    from r2_gaussian_b200.scene_view import scan_orbit
    from r2_gaussian_b200.volume_render import look_at

    pos, meta, attr, tex = _soup(np.random.default_rng(42), 300, 100, 60, 1.0, 0.4)
    cams = scan_orbit(look_at((3.0, 1.0, 2.0), (0, 0, 0), (0, 0, 1), PIX_SIDE, PIX_SIDE, 40.0), PIX_FRAMES)
    return Scene(pos, meta, attr, tex, cams, PIX_FRAMES, textured=True)


@functools.lru_cache(maxsize=None)
def one_record_scene() -> Scene:
    """One R2X_SV_MAX_SIDE^2 frame from inside an ellipsoid (a record of every tile), a tilted quad covering the whole
    frame that cuts the ellipsoid's far wall (two more), and a line across the whole width on the centre row."""
    from r2_gaussian_b200.volume_render import look_at

    S = K["R2X_SV_MAX_SIDE"]
    ell = _ellipsoids(np.array([[0.2, 0.1, -0.1]]), np.array([[3.0, 2.5, 2.0]]), np.array([[0.9, 0.2, -0.3, 0.1]]),
                      np.array([[0.8, 0.6, 0.4]]))
    plane = lambda y, z: (2.0 + 0.3 * y + 0.2 * z, y, z)          # in front of the camera for every ray of the frame
    q = np.array([plane(-10, -10), plane(10, -10), plane(10, 10), plane(-10, 10)])
    tri = (np.stack([q[[0, 1, 2]], q[[2, 3, 0]]]), np.array([[so.FLAT, 0], [so.FLAT, 0]], np.int32),
           np.zeros((2, 12), np.float32))
    tri[2][:, 0:3] = [[0.2, 0.7, 0.3], [0.1, 0.3, 0.9]]
    line = _lines(np.array([[1.0, -5.0, 0.0]]), np.array([[1.0, 5.0, 0.0]]), np.array([[1.0, 0.0, 0.0]]), 1.5)
    pos, meta, attr = _cat(ell, tri, line)
    cam = look_at((0.0, 0.0, 0.0), (1.0, 0.0, 0.0), (0, 0, 1), S, S, 60.0)
    return Scene(pos, meta, attr, np.zeros((1, 1, 1), np.float32), [cam], 1)


@functools.lru_cache(maxsize=None)
def scan_scene() -> Scene:
    """A 400 x 300 perspective frame of 3600 lines and 900 ellipsoids of sizes spread over a decade or more: several
    thousand records with tile counts from 2 to several hundred, so the single-CTA scan runs many passes."""
    from r2_gaussian_b200.volume_render import look_at

    rng = np.random.default_rng(44)
    n_line, n_ell = 3600, 900
    c = rng.uniform(-2.0, 2.0, (n_line, 3))
    d = rng.normal(0, 1, (n_line, 3))
    d *= (np.exp(rng.uniform(np.log(0.4), np.log(12.0), n_line)) / np.linalg.norm(d, axis=1))[:, None]
    lines = _lines(c - d / 2, c + d / 2, rng.random((n_line, 3)), rng.choice([0.7, 1.5, 3.0], n_line))
    s = np.exp(rng.uniform(np.log(0.02), np.log(0.9), (n_ell, 1))) * rng.uniform(0.5, 1.0, (n_ell, 3))
    ells = _ellipsoids(rng.uniform(-2.0, 2.0, (n_ell, 3)), s, rng.normal(0, 1, (n_ell, 4)), rng.random((n_ell, 3)))
    pos, meta, attr = _cat(lines, ells)
    cam = look_at((0.3, -7.0, 0.4), (0.0, 0.0, 0.0), (0, 0, 1), 400, 300, 50.0)
    return Scene(pos, meta, attr, np.zeros((1, 1, 1), np.float32), [cam], 1)


def _scene_peak(frames, H, W, n_prims) -> int:
    # keys (8 B) and colours (12 B) per pixel, one record (40 B) per (primitive, frame), the inputs, slack
    return 20 * frames * H * W + 40 * n_prims * frames + 64 + GiB


def _corner_windows(H, W, s):
    return ((0, s, 0, s), (0, s, W - s, W), (H - s, H, 0, s), (H - s, H, W - s, W),
            (H // 2 - s // 2, H // 2 + s // 2, W // 2 - s // 2, W // 2 + s // 2))


def _scene_cases() -> list[Case]:
    out = [Case("scene_records_past_2_30", "scene",
                "scene raster: more than 2^30 records and 2^31 tiles, n_frames == SV_MAX_GRID",
                ("frames == SV_MAX_GRID", "n_records > 2**30", "n_records <= INT_MAX", "tiles > 2**31",
                 "tiles == 2 * n_records", "R2X_SV_TILE < W <= 2 * R2X_SV_TILE", "H == 1",
                 "(n_records - 2) + (n_records - 1) + 1 > INT_MAX", "n_cams == 7"),
                extra={"scene": records_scene}, peak=_scene_peak(K["SV_MAX_GRID"], 1, REC_W, REC_LINES))]
    H = W = PIX_SIDE
    out.append(Case("scene_pixels_past_2_31", "scene", "scene raster: more than 2^31 pixels in one call",
                    ("frames * H * W > 2**31", "(frames - 1) * H * W == 2**31", "frames <= SV_MAX_GRID",
                     "n_kinds == 5"),
                    extra={"scene": pixels_scene, "frames_checked": (0, PIX_FRAMES // 2, PIX_FRAMES - 1),
                           "windows": _corner_windows(H, W, 24)},
                    peak=_scene_peak(PIX_FRAMES, H, W, 460)))
    S = K["R2X_SV_MAX_SIDE"]
    out.append(Case("scene_one_record_1M_tiles", "scene", "scene raster: one record of R2X_SV_MAX_SIDE^2 / 256 tiles",
                    ("H == R2X_SV_MAX_SIDE", "W == R2X_SV_MAX_SIDE", "max_tiles == (H // R2X_SV_TILE) ** 2",
                     "max_tiles >= 256 * SV_TILE_CTAS", "n_records == 4"),
                    extra={"scene": one_record_scene,
                           "windows": _corner_windows(S, S, 48) + ((S // 2 - 16, S // 2 + 16, 0, 48),
                                                                  (S // 2 - 16, S // 2 + 16, S - 48, S))},
                    peak=_scene_peak(1, S, S, 4)))
    out.append(Case("scene_scan_many_passes", "scene", "scene raster: a scan of more than 3 * SV_SCAN_THREADS records",
                    ("n_records > 3 * SV_SCAN_THREADS", "min_tiles == 2", "max_tiles >= 300",
                     "n_distinct_tiles >= 50"),
                    extra={"scene": scan_scene}, peak=_scene_peak(1, 300, 400, 4500)))
    return out


# ---- zoom cases ---------------------------------------------------------------------------------------------------

def _zoom_peak(placed, out, src_bytes) -> int:
    pad = 2 * K["ZOOM_PAD"]
    return 8 * math.prod(n + pad for n in placed) + 8 * math.prod(out) + src_bytes + GiB


def _zoom_cases() -> list[Case]:
    M, P = K["ZOOM_MAX_DIM"], K["ZOOM_PAD"]
    out = []
    n, o = 48, 1291
    f = o / n
    big = [(0, 4)] * 3
    wrap = np.unravel_index(2**31, (o, o, o))
    out.append(Case("zoom_output_past_2_31", "zoom", "zoom: an output of more than 2^31 voxels",
                    ("math.prod(out) > 2**31", "out == (1291, 1291, 1291)", "max(out) <= ZOOM_MAX_DIM"),
                    extra={"src_shape": (n, n, n), "factors": (f, f, f), "place": None,
                           "windows": (("origin", big), ("last row", [(o - 1, o), (o - 1, o), (0, o)]),
                                       ("last voxel", [(o - 3, o)] * 3),
                                       ("flat 2^31", [(max(int(w) - 2, 0), min(int(w) + 3, o)) for w in wrap]))},
                    peak=_zoom_peak((n,) * 3, (o,) * 3, 8 * n**3)))
    # a host uint8 view whose strides are not C order, expanded along z into a 1290^3 placed cube
    m, sz, off = 1290, 1100, 95
    po = m + 2 * P
    wi = np.unravel_index(2**31, (po, po, po))
    fo = 0.1
    near = [int(round((int(w) - P) * (round(m * fo) - 1) / (m - 1))) for w in wi]
    out.append(Case("zoom_workspace_past_2_31", "zoom",
                    "zoom: a padded workspace of more than 2^31 voxels from a strided, expanded uint8 source",
                    ("padded ** 3 > 2**31", "placed == (1290, 1290, 1290)", "src_z + 2 * off_z == 1290"),
                    extra={"src_shape": (m, m, sz), "factors": (fo, fo, fo), "offset": (0, 0, off), "lo": 3.0,
                           "hi": 250.0, "place": (m, m, m),
                           "windows": (("origin", [(0, 3)] * 3), ("last voxel", [(126, 129)] * 3),
                                       ("padded flat 2^31", [(max(c - 2, 0), min(c + 2, 129)) for c in near]),
                                       ("source edge", [(60, 62), (60, 62), (8, 11)]))},
                    peak=_zoom_peak((m,) * 3, (129,) * 3, m * m * sz)))
    for a in range(3):
        src = [1, 2]
        src.insert(a, M)
        fac = [3.0, 0.5]
        fac.insert(a, 1.0)
        out.append(Case(f"zoom_max_dim_axis{a}", "zoom", f"zoom: ZOOM_MAX_DIM placed and output along axis {a}",
                        (f"src[{a}] == ZOOM_MAX_DIM", f"out[{a}] == ZOOM_MAX_DIM", "sorted(out) == [1, 3, ZOOM_MAX_DIM]"),
                        extra={"src_shape": tuple(src), "factors": tuple(fac), "place": None, "windows": None},
                        peak=_zoom_peak(src, src, 8 * M * 2)))
        src = [1, 3]
        src.insert(a, 1)
        fac = [1.0, 2.0]
        fac.insert(a, float(M))
        out.append(Case(f"zoom_upsample_to_max_axis{a}", "zoom",
                        f"zoom: a source of 1 upsampled to ZOOM_MAX_DIM along axis {a}, an output of 1 at factor 1",
                        (f"src[{a}] == 1", f"out[{a}] == ZOOM_MAX_DIM", "sorted(out) == [1, 6, ZOOM_MAX_DIM]"),
                        extra={"src_shape": tuple(src), "factors": tuple(fac), "place": None, "windows": None},
                        peak=_zoom_peak(src, [M, 6, 1], 24)))
    return out


# ---- projection preparation ---------------------------------------------------------------------------------------

def _prepare_cases() -> list[Case]:
    n, H0, W0 = 720, 1536, 1944
    return [Case("prepare_past_2_31", "prepare",
                 "projection prepare: 720 full-resolution views, 2^31 output pixels, then subsample 4 of the same input",
                 ("n * H0 * W0 > 2**31", "(n - 1) * H0 * W0 < 2**31", "sub4 == (384, 384)"),
                 extra={"n": n, "H0": H0, "W0": W0, "views": (0, n // 2 - 1, n - 1), "rescale": 400.0,
                        "object_scale": 50.0},
                 peak=8 * n * H0 * W0 + 4 * n * H0 * W0 + GiB)]


# ---- the detector-offset gradient ---------------------------------------------------------------------------------

def grad_blocks(N: int) -> tuple[int, int]:
    """(blocks, chunk) of r2x_detector_offset_grad over N rows."""
    nb = min(max(tiles(N, K["kPerBlock"]), 1), K["kMaxBlocks"])
    return nb, tiles(N, nb)


GRAD_MOD = 4093           # x components (i mod 4093) / 4096: exact in float32, every partial sum exact in float64


def grad_sum_units(N: int) -> int:
    """4096 times the sum over rows i < N of (i mod GRAD_MOD) / 4096, in closed form."""
    q, r = divmod(N, GRAD_MOD)
    return q * (GRAD_MOD * (GRAD_MOD - 1) // 2) + r * (r - 1) // 2


def _grad_cases() -> list[Case]:
    P, n = 2**27, 17
    return [Case("grad_rows_past_2_31", "grad", "detector-offset gradient: N = P n_views rows past 2^31",
                 ("N > 2**31", "3 * N > 2**32", "nb == kMaxBlocks", "chunk > kPerBlock", "(nb - 1) * chunk < N",
                  "sum_units < 2**53"),
                 extra={"P": P, "n_views": n, "W": 800},
                 peak=12 * P * n + 3 * GiB)]


SCENE_CASES = {c.name: c for c in _scene_cases()}
ZOOM_CASES = {c.name: c for c in _zoom_cases()}
PREPARE_CASES = {c.name: c for c in _prepare_cases()}
GRAD_CASES = {c.name: c for c in _grad_cases()}
ALL_CASES = {**SCENE_CASES, **ZOOM_CASES, **PREPARE_CASES, **GRAD_CASES}
assert len(ALL_CASES) == len(SCENE_CASES) + len(ZOOM_CASES) + len(PREPARE_CASES) + len(GRAD_CASES)


# ---- what a case claims -------------------------------------------------------------------------------------------

class _Quantities(dict):
    """The quantities a claim may name, computed on first use."""

    def __init__(self, case: Case):
        super().__init__(K)
        self.case = case
        self.update(INT_MAX=INT_MAX, math=math, sorted=sorted, max=max, **case.extra)

    def __missing__(self, name):
        self[name] = value = getattr(self, "_" + name)()
        return value

    # scene
    def _sc(self): return self.case.extra["scene"]()
    def _frames(self): return self["sc"].frames
    def _H(self): return self["sc"].H
    def _W(self): return self["sc"].W
    def _n_cams(self): return len(self["sc"].cams)
    def _n_kinds(self): return len(set(self["sc"].meta[:, 0].tolist()))

    def _per_cam(self):
        sc = self["sc"]
        return [sc.records(c) for c in range(len(sc.cams))]

    def _frames_of(self):
        sc = self["sc"]
        return [len(range(c, sc.frames, len(sc.cams))) for c in range(len(sc.cams))]

    def _n_records(self): return sum(len(r) * f for r, f in zip(self["per_cam"], self["frames_of"]))
    def _tiles(self): return sum(int(r.sum()) * f for r, f in zip(self["per_cam"], self["frames_of"]))
    def _max_tiles(self): return max(int(r.max()) for r in self["per_cam"])
    def _min_tiles(self): return min(int(r.min()) for r in self["per_cam"])
    def _n_distinct_tiles(self): return len(set(np.concatenate(self["per_cam"]).tolist()))

    # zoom
    def _src(self): return tuple(self.case.extra["src_shape"])
    def _placed(self): return tuple(self.case.extra["place"] or self["src"])

    def _out(self):
        from r2_gaussian_b200.resample import zoom_shape

        return zoom_shape(self["placed"], self.case.extra["factors"])

    def _padded(self): return self["placed"][0] + 2 * K["ZOOM_PAD"]
    def _src_z(self): return self["src"][2]
    def _off_z(self): return self.case.extra["offset"][2]

    # prepare
    def _sub4(self):
        import real_data_oracle as ro

        return tuple(ro.output_shape(self["H0"], self["W0"], 4)[4:])

    # gradient
    def _N(self): return self["P"] * self["n_views"]
    def _nb(self): return grad_blocks(self["N"])[0]
    def _chunk(self): return grad_blocks(self["N"])[1]
    def _sum_units(self): return grad_sum_units(self["N"])


def claim_failures(case: Case) -> list[str]:
    """The claims of `case` that do not hold (empty when it sits where it says)."""
    q = _Quantities(case)
    return [c for c in case.claims if not eval(c, {"__builtins__": {}}, q)]


def quantity(case: Case, name: str):
    return _Quantities(case)[name]
