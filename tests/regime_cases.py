"""Inputs whose code paths in the rasterizer and the voxelizer are known, and a classifier that says which paths an input
takes.

The kernels switch between code paths on the tile count (direct / radix binning, two-level voxel binning), on the
instances of each direct_fill CTA (staged / unstaged stores), on the per-tile instance counts (work-plan chunks, voxel
segments) and, per Gaussian, on its conic and weight (fast / exact render path).  Random clouds land on whichever side
they happen to; the clouds here are built so that each lands on a stated side of a stated boundary, and
`tests/test_regimes_cpu.py` checks that they do, on the CPU oracle, so that the GPU tests that use them cannot quietly
stop exercising what they are named after.

Every threshold is read from the CUDA sources (`r2_gaussian_b200/csrc/`) by regular expression: a retuned constant moves
the cases with it, and a renamed or reworded one fails the suite instead of leaving a case on the wrong side.
"""
from __future__ import annotations

import math
import os
import re
from dataclasses import dataclass, field

import numpy as np

from r2_gaussian_b200 import scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "r2_gaussian_b200", "csrc")
RASTER_TILE, VOXEL_TILE = 16, 8
_NUM = r"([-+]?[0-9]*\.?[0-9]+(?:[eE][-+]?[0-9]+)?)f?"


def _source(name: str) -> str:
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def _find(pattern: str, text: str, what: str) -> re.Match:
    m = re.search(pattern, text)
    if m is None:
        raise LookupError(f"{what}: not found in the CUDA sources (pattern {pattern!r})")
    return m


def _constexpr(name: str, text: str, env: dict):
    m = _find(rf"constexpr\s+(?:int|float|unsigned)\s+{name}\s*=\s*([^;]+);", text, name)
    expr = re.sub(r"(?<=[0-9])[fu]\b", "", m.group(1))
    return eval(expr, {"__builtins__": {}}, dict(env))   # e.g. "4 * DIRECT_BLOCK"


def read_constants() -> dict:
    """The thresholds of the binning, work-plan and fast-path switches, as the CUDA sources state them."""
    cuh, cu, cu2 = _source("r2x_binning.cuh"), _source("r2x_binning.cu"), _source("r2x_binning2.cu")
    ras, vox = _source("r2x_raster.cu"), _source("r2x_voxel.cu")
    k: dict = {}
    for name, text in [("DIRECT_MAX_TILES", cuh), ("DIRECT_BLOCK", cuh), ("PLAN_CHUNK", cuh), ("VOX_CHUNK_CAP", cuh),
                       ("FILL_STAGE_TILES", cu), ("FILL_STAGE_CAP", cu), ("SUP", cu2), ("Q_CUT", ras),
                       ("VQ_CUT", vox)]:
        k[name] = _constexpr(name, text, k)
    # plan_chunk_for: the voxelizer's chunk is the instances per this many work items, rounded up to PLAN_CHUNK
    k["PLAN_ITEMS"] = int(_find(r"const uint32_t want = \(R / ([0-9]+)u", cuh, "plan_chunk_for's item target").group(1))
    # the per-Gaussian fast-path tests (raster preprocess, voxel preprocess)
    m = _find(rf"conx \* conz - cony \* cony > {_NUM} \* conx \* conz", ras, "raster det-ratio limit")
    k["RAS_DET_RATIO"] = float(m.group(1))
    m = _find(rf"const bool fast = !\(w > 0\.0f\) \|\| \(pd && A2 <= {_NUM} && lw <= {_NUM} && lw >= {_NUM}\);", ras,
              "raster fast-path limits")
    k["RAS_A2_MAX"], k["RAS_LW_MAX"], k["RAS_LW_MIN"] = (float(m.group(i)) for i in (1, 2, 3))
    m = _find(rf"m01 > {_NUM} \* inv\[0\] \* inv\[3\]\) &&\s*\(det3 > {_NUM} \* inv\[0\] \* inv\[3\] \* inv\[5\]\)", vox,
              "voxel det-ratio limits")
    k["VOX_M01_RATIO"], k["VOX_DET3_RATIO"] = float(m.group(1)), float(m.group(2))
    m = _find(rf"const bool fast = !\(rho > 0\.0f\) \|\| \(pd && F2 <= {_NUM} && lw <= {_NUM} && lw >= {_NUM}\);", vox,
              "voxel fast-path limits")
    k["VOX_F2_MAX"], k["VOX_LW_MAX"], k["VOX_LW_MIN"] = (float(m.group(i)) for i in (1, 2, 3))
    # raster_render_bwd2_kernel redoes a row with bwd_row_careful when a pixel's G lies in [gcut * lo, gcut * hi]
    m = _find(rf"bwd_row_careful\([^;]*gcut \* {_NUM}, gcut \* {_NUM}", ras, "bwd_row_careful band")
    k["CAREFUL_HI"], k["CAREFUL_LO"] = float(m.group(1)), float(m.group(2))
    return k


K = read_constants()
LOG2E = np.float32(1.4426950408889634)


# ---- the classifier --------------------------------------------------------------------------------------------------
def plan_chunk_for(R: int, chunk_cap: int) -> int:
    """Chunk size of a launch with R instances (automatic policy; restates r2x_binning.cuh's plan_chunk_for, which
    tests/host/plan_check.cu checks on the host)."""
    pc = K["PLAN_CHUNK"]
    cap = max(chunk_cap, pc)
    if cap <= pc:
        return pc
    want = (R // K["PLAN_ITEMS"] + pc - 1) // pc * pc
    return min(max(want, pc), cap)


def tile_grid(shape) -> tuple:
    if len(shape) == 2:   # raster (H, W)
        H, W = shape
        return (-(-W // RASTER_TILE), -(-H // RASTER_TILE))
    return tuple(-(-int(n) // VOXEL_TILE) for n in shape)


def binning_path(shape) -> str:
    g = tile_grid(shape)
    T = int(np.prod(g))
    if T <= K["DIRECT_MAX_TILES"]:
        return "direct"
    if len(shape) == 3 and int(np.prod([-(-n // K["SUP"]) for n in g])) <= K["DIRECT_MAX_TILES"]:
        return "two_level"
    return "radix"


def raster_fast(orc) -> np.ndarray:
    """Per Gaussian: True if it takes the fast render path (the raster preprocess's own float32 expression, from the
    oracle's exported conic, density and mu).  Culled Gaussians are reported as fast (they are never rendered)."""
    co = orc["conic_opacity"].astype(np.float32)
    conx, cony, conz, rho = co[:, 0], co[:, 1], co[:, 2], co[:, 3]
    with np.errstate(all="ignore"):
        w = (rho * orc["mu"].astype(np.float32)).astype(np.float32)
        A2 = (conx * np.float32(0.5 * LOG2E)).astype(np.float32)
        lw = np.where(w > 0, np.log2(w.astype(np.float64)), -np.inf).astype(np.float32)
        pd = (conx > 0) & (conz > 0) & (conx * conz - cony * cony > np.float32(K["RAS_DET_RATIO"]) * conx * conz)
    fast = ~(w > 0) | (pd & (A2 <= K["RAS_A2_MAX"]) & (lw <= K["RAS_LW_MAX"]) & (lw >= K["RAS_LW_MIN"]))
    return fast | (orc["radii"] <= 0)


def raster_margins(orc) -> dict:
    """Each fast-path quantity against its limit (float64), oriented so that < 1 is inside (fast) and > 1 outside:
    A2 / max, log2 w / max, log2 w / min (both limits' signs), det-ratio limit / det ratio."""
    co = orc["conic_opacity"].astype(np.float64)
    conx, cony, conz = co[:, 0], co[:, 1], co[:, 2]
    w = (orc["conic_opacity"][:, 3] * orc["mu"]).astype(np.float32).astype(np.float64)
    with np.errstate(all="ignore"):
        lw = np.log2(w)
        return dict(A2=conx * 0.5 * float(LOG2E) / K["RAS_A2_MAX"], lw_max=lw / K["RAS_LW_MAX"],
                    lw_min=lw / K["RAS_LW_MIN"], det=K["RAS_DET_RATIO"] / ((conx * conz - cony * cony) / (conx * conz)))


def voxel_fast(orc) -> np.ndarray:
    co = orc["conic_opacity"].astype(np.float32)
    inv, rho = [co[:, i] for i in range(6)], co[:, 6]
    with np.errstate(all="ignore"):
        lw = np.where(rho > 0, np.log2(rho.astype(np.float64)), -np.inf).astype(np.float32)
        F2 = (inv[5] * np.float32(0.5 * LOG2E)).astype(np.float32)
        m01 = inv[0] * inv[3] - inv[1] * inv[1]
        det3 = (inv[0] * (inv[3] * inv[5] - inv[4] * inv[4]) - inv[1] * (inv[1] * inv[5] - inv[4] * inv[2])
                + inv[2] * (inv[1] * inv[4] - inv[3] * inv[2]))
        pd = ((inv[0] > 0) & (inv[3] > 0) & (inv[5] > 0) & (m01 > np.float32(K["VOX_M01_RATIO"]) * inv[0] * inv[3])
              & (det3 > np.float32(K["VOX_DET3_RATIO"]) * inv[0] * inv[3] * inv[5]))
    fast = ~(rho > 0) | (pd & (F2 <= K["VOX_F2_MAX"]) & (lw <= K["VOX_LW_MAX"]) & (lw >= K["VOX_LW_MIN"]))
    return fast | (orc["tiles_touched"] == 0)


def voxel_margins(orc) -> dict:
    co = orc["conic_opacity"].astype(np.float64)
    i0, i1, i2, i3, i4, i5 = (co[:, i] for i in range(6))
    with np.errstate(all="ignore"):
        lw = np.log2(co[:, 6])
        m01 = (i0 * i3 - i1 * i1) / (i0 * i3)
        return dict(F2=i5 * 0.5 * float(LOG2E) / K["VOX_F2_MAX"], lw_max=lw / K["VOX_LW_MAX"],
                    lw_min=lw / K["VOX_LW_MIN"], det=K["VOX_M01_RATIO"] / m01)


def regime(orc, shape) -> dict:
    """Which code paths one forward takes, from the oracle's outputs alone.  `shape` is (H, W) for the rasterizer and
    (nx, ny, nz) for the voxelizer.

    path       'direct' | 'two_level' | 'radix'
    cta_total  direct binning: instances of each direct_fill CTA (sum of tiles_touched over DIRECT_BLOCK Gaussians)
    staged     direct binning: whether each CTA stages its stores in shared memory
    counts     instances per tile (from the oracle's ranges); chunk = the launch's chunk size
    chunks     work items per tile;  segments: per tile, the most PLAN_CHUNK-record segments one of its items is walked in
    fast       per Gaussian: the fast (True) or exact (False) render path;  margins: the fast-path quantities / limits
    """
    raster = len(shape) == 2
    g = tile_grid(shape)
    T = int(np.prod(g))
    path = binning_path(shape)
    tt = np.asarray(orc["tiles_touched"], dtype=np.int64)
    out = dict(kind="raster" if raster else "voxel", grid=g, T=T, path=path, R=int(orc["R"]))
    if not raster:
        out["T1"] = int(np.prod([-(-n // K["SUP"]) for n in g]))
    if path == "direct":
        nb = -(-len(tt) // K["DIRECT_BLOCK"])
        pad = np.zeros(nb * K["DIRECT_BLOCK"], np.int64)
        pad[:len(tt)] = tt
        out["cta_total"] = pad.reshape(nb, K["DIRECT_BLOCK"]).sum(axis=1)
        out["staged"] = (T <= K["FILL_STAGE_TILES"]) & (out["cta_total"] <= K["FILL_STAGE_CAP"])
    rg = np.asarray(orc["ranges"], dtype=np.int64)
    counts = rg[:, 1] - rg[:, 0]
    assert int(counts.sum()) == out["R"]
    chunk = plan_chunk_for(out["R"], K["PLAN_CHUNK"] if raster else K["VOX_CHUNK_CAP"])
    chunks = np.maximum(1, -(-counts // chunk))
    longest = -(-counts // chunks)                       # equal slices: the first ones hold ceil(n / chunks)
    out.update(counts=counts, chunk=chunk, chunks=chunks, segments=np.maximum(1, -(-longest // K["PLAN_CHUNK"])))
    out["fast"] = raster_fast(orc) if raster else voxel_fast(orc)
    out["margins"] = raster_margins(orc) if raster else voxel_margins(orc)
    return out


def careful_pairs(orc, W, H) -> int:
    """(Gaussian, pixel) pairs of the forward whose G = exp(power) lies inside the band around the alpha cut that
    raster_render_bwd2_kernel redoes with bwd_row_careful (float64, from the oracle's xy / conic / w)."""
    cut = 2.0 ** -K["Q_CUT"]
    n = 0
    co, xy = orc["conic_opacity"].astype(np.float64), orc["xy"].astype(np.float64)
    w = (orc["conic_opacity"][:, 3] * orc["mu"]).astype(np.float32).astype(np.float64)
    for i in np.nonzero((orc["radii"] > 0) & (w > 0))[0]:
        x0, y0, x1, y1 = (int(v) for v in orc["rect"][i])
        ys, xs = np.mgrid[y0 * RASTER_TILE:min(H, y1 * RASTER_TILE), x0 * RASTER_TILE:min(W, x1 * RASTER_TILE)]
        dx, dy = xy[i, 0] - xs, xy[i, 1] - ys
        G = np.exp(-0.5 * (co[i, 0] * dx * dx + co[i, 2] * dy * dy) - co[i, 1] * dx * dy)
        gcut = cut / w[i]
        n += int(np.count_nonzero((G >= gcut * K["CAREFUL_LO"]) & (G <= gcut * K["CAREFUL_HI"])))
    return n


# ---- building clouds --------------------------------------------------------------------------------------------------
def parallel_view(W: int, H: int):
    """Parallel beam at angle 0: view x = world y, view y = -world z, depth = 5 - world x; pixel pitch 2 / W by 2 / H."""
    sc = scene.parallel_beam_scanner(max(W, H))
    sc["nDetector"] = [H, W]
    return scene.make_view(sc, 0.0)


def cone_view(W: int, H: int, angle: float = 0.9):
    """Cone beam whose pixel pitch is that of a 512-pixel detector of 4 units, whatever the pixel counts."""
    sc = scene.cone_beam_scanner(max(W, H))
    sc["nDetector"] = [H, W]
    sc["sDetector"] = [4.0 * H / 512, 4.0 * W / 512]
    return scene.make_view(sc, angle)


def world_at_pixel(view, px, py, depth=5.0) -> np.ndarray:
    """World points that a parallel-beam view puts at pixel centres (px, py) (arrays) at the given view depth."""
    V = view.viewmatrix.astype(np.float64).T
    px, py = np.broadcast_arrays(np.asarray(px, np.float64), np.asarray(py, np.float64))
    xv = (2.0 * px + 1.0) / view.image_width - 1.0
    yv = (2.0 * py + 1.0) / view.image_height - 1.0
    h = np.stack([xv, yv, np.full_like(xv, depth), np.ones_like(xv)], axis=-1)
    return (h @ np.linalg.inv(V).T)[..., :3]


def view_axes(view) -> np.ndarray:
    """World axis index along view x, view y and view depth (the parallel view at angle 0 is axis-aligned)."""
    V = view.viewmatrix.astype(np.float64).T
    return np.array([int(np.argmax(np.abs(V[i, :3]))) for i in range(3)])


def make(means, scales, rots=None, dens=None) -> scene.Cloud:
    means = np.asarray(means, np.float32).reshape(-1, 3)
    P = len(means)
    scales = np.broadcast_to(np.asarray(scales, np.float32), (P, 3)).copy()
    if rots is None:
        rots = np.tile(np.float32([1, 0, 0, 0]), (P, 1))
    rots = np.broadcast_to(np.asarray(rots, np.float32), (P, 4)).copy()
    dens = np.broadcast_to(np.asarray(0.5 if dens is None else dens, np.float32).reshape(-1, 1), (P, 1)).copy()
    return scene.Cloud(means, scales, rots, dens)


def concat(*clouds) -> scene.Cloud:
    return scene.Cloud(*(np.concatenate([getattr(c, k) for c in clouds]).astype(np.float32)
                         for k in ("means", "scales", "rotations", "density")))


SMALL = 1e-4    # a world scale far below a pixel / voxel: the minimum footprint, one tile when centred in it


def raster_in_tiles(view, tiles, rng, scale=SMALL, jitter=2.0, dens=(0.3, 0.7)):
    """One Gaussian per entry of `tiles` ((tx, ty) pairs), near the centre of that tile, position and density
    jittered so that no two are identical (within +-jitter px: the footprint stays in the tile)."""
    tiles = np.asarray(tiles, np.float64).reshape(-1, 2)
    n = len(tiles)
    px = tiles[:, 0] * RASTER_TILE + 7.5 + rng.uniform(-jitter, jitter, n)
    py = tiles[:, 1] * RASTER_TILE + 7.5 + rng.uniform(-jitter, jitter, n)
    depth = 5.0 + rng.uniform(-0.5, 0.5, n)
    return make(world_at_pixel(view, px, py, depth), np.full((n, 3), scale), dens=rng.uniform(*dens, n))


def voxel_world(grid, pv):
    """World coordinates of voxel-space positions pv ([..., 3], voxel i spans [i, i + 1))."""
    nV, sV, ctr = grid
    dv = np.asarray(sV, np.float64) / np.asarray(nV, np.float64)
    return np.asarray(pv, np.float64) * dv - 0.5 * np.asarray(sV, np.float64) + np.asarray(ctr, np.float64)


def voxel_in_tiles(grid, tiles, rng, jitter=2.0, dens=(0.3, 0.7)):
    tiles = np.asarray(tiles, np.float64).reshape(-1, 3)
    n = len(tiles)
    pv = tiles * VOXEL_TILE + 4.0 + rng.uniform(-jitter, jitter, (n, 3))
    return make(voxel_world(grid, pv), np.full((n, 3), SMALL), dens=rng.uniform(*dens, n))


def _oracle_raster(cloud, view, render=False):
    import util
    return util.oracle_raster_forward(cloud, view, render=render)


def _oracle_voxel(cloud, grid, render=False):
    import util
    return util.oracle_voxel_forward(cloud, *grid, render=render)


def bisect(f, lo, hi, target, iters=60):
    """x in [lo, hi] with f(x) = target for a monotonic f (either direction), in float64."""
    flo = f(lo)
    for _ in range(iters):
        mid = 0.5 * (lo + hi)
        if (f(mid) < target) == (flo < target):
            lo = mid
        else:
            hi = mid
    return 0.5 * (lo + hi)


# ---- the cases --------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    """An input and the sides of the boundaries it is built to land on.

    expect keys: path; cta_total {cta: n}; staged {cta: bool}; counts {tile: n}; min_chunks (some tile has at least
    this many work items); chunk_gt (the launch's chunk size exceeds this); min_segments (some item spans at least this
    many segments); fast {gaussian index: bool}; margins [(name, indices, lo, hi)]: every margins[name][indices] in
    [lo, hi]; careful (pairs in the bwd_row_careful band > 0)."""
    name: str
    kind: str                  # 'raster' | 'voxel'
    cloud: scene.Cloud
    view: object = None        # raster
    grid: tuple = None         # voxel: (nVoxel, sVoxel, center)
    expect: dict = field(default_factory=dict)
    crowded: tuple = ()        # tiles whose image is compared against a float64 sum (see test_regimes_gpu.py)
    needles: tuple = ()        # Gaussians 1e-4 from a singular conic: gradients ill-conditioned in float32

    @property
    def shape(self):
        return (self.view.image_height, self.view.image_width) if self.kind == "raster" else tuple(self.grid[0])

    def oracle(self):
        return _oracle_raster(self.cloud, self.view, True) if self.kind == "raster" else _oracle_voxel(self.cloud, self.grid, True)


def check_case(case: Case, orc) -> list:
    """Asserts every side `case` claims, from the oracle's forward; returns one report line per boundary."""
    reg = regime(orc, case.shape)
    ex, lines = case.expect, []
    if "path" in ex:
        assert reg["path"] == ex["path"], (case.name, reg["path"])
        lines.append(f"binning T={reg['T']}" + (f" T1={reg['T1']}" if "T1" in reg else "") + f": {reg['path']}")
    for b, n in ex.get("cta_total", {}).items():
        assert int(reg["cta_total"][b]) == n, (case.name, b, int(reg["cta_total"][b]), n)
        lines.append(f"direct_fill CTA {b}: {n} instances (cap {K['FILL_STAGE_CAP']})")
    for b, s in ex.get("staged", {}).items():
        assert bool(reg["staged"][b]) == s, (case.name, b)
        lines.append(f"direct_fill CTA {b}: {'staged' if s else 'unstaged'} (T={reg['T']})")
    for t, n in ex.get("counts", {}).items():
        assert int(reg["counts"][t]) == n, (case.name, t, int(reg["counts"][t]), n)
        lines.append(f"tile {t}: {n} instances = {int(reg['chunks'][t])} chunk(s) of <= {reg['chunk']}"
                     + (f", {int(reg['segments'][t])} segment(s)" if case.kind == "voxel" else ""))
    if "min_chunks" in ex:
        assert int(reg["chunks"].max()) >= ex["min_chunks"], (case.name, int(reg["chunks"].max()))
        lines.append(f"most chunks of a tile: {int(reg['chunks'].max())} >= {ex['min_chunks']}")
    if "chunk_gt" in ex:
        assert reg["chunk"] > ex["chunk_gt"], (case.name, reg["chunk"])
        lines.append(f"chunk {reg['chunk']} > {ex['chunk_gt']} (R = {reg['R']})")
    if "min_segments" in ex:
        assert int(reg["segments"].max()) >= ex["min_segments"], (case.name, int(reg["segments"].max()))
        lines.append(f"an item spans {int(reg['segments'].max())} segments of {K['PLAN_CHUNK']}")
    if "fast" in ex:
        idx = np.asarray(list(ex["fast"].keys()))
        want = np.asarray(list(ex["fast"].values()))
        got = reg["fast"][idx]
        assert np.array_equal(got, want), (case.name, idx[got != want])
        lines.append(f"fast path: {int(want.sum())} Gaussians, exact path: {int((~want).sum())}")
    for name, idx, lo, hi in ex.get("margins", []):
        v = reg["margins"][name][idx]
        assert np.all((v >= lo) & (v <= hi)), (case.name, name, v.min(), v.max())
        lines.append(f"{name}: margin in [{v.min():.5f}, {v.max():.5f}], {'inside (fast)' if hi <= 1 else 'outside (exact)'}")
    if ex.get("careful"):
        n = careful_pairs(orc, case.view.image_width, case.view.image_height)
        assert n > 0, case.name
        lines.append(f"pairs in the bwd_row_careful band: {n}")
    return lines


def _exact_total(n_big: int, S: int, block: int):
    """(k big, singles, doubles) with k * n_big + singles + 2 * doubles == S and k + singles + doubles == block."""
    for k in range(block + 1):
        rest, m = S - k * n_big, block - k
        if m <= rest <= 2 * m:
            return k, m - (rest - m), rest - m
    raise ValueError(f"no mix of {n_big}-tile, 1-tile and 2-tile Gaussians gives {S}")


def cta_total_case() -> Case:
    """direct_fill at T = 1024 (a 512^2 detector): CTA 0 holds exactly FILL_STAGE_CAP instances (staged), CTA 1 one
    more (unstaged), CTA 2 (a partial CTA) far fewer (staged)."""
    rng = np.random.RandomState(11)
    view = parallel_view(512, 512)
    gx, gy = tile_grid((512, 512))
    B, S = K["DIRECT_BLOCK"], K["FILL_STAGE_CAP"]
    # a multi-tile Gaussian at a tile centre: its rectangle, as the oracle finds it
    big_scale = 40.0 / (0.5 * 512) / 3.0          # 3 sigma ~ 40 px: 7 x 7 tiles at a tile centre
    probe = raster_in_tiles(view, [(10, 10)], rng, scale=big_scale, jitter=0.0)
    n_big = int(_oracle_raster(probe, view)["tiles_touched"][0])

    def block(total, first_tile):
        k, singles, doubles = _exact_total(n_big, total, B)
        big_tiles = [((first_tile + 3 * i) % (gx - 8) + 4, (first_tile + 3 * i) // (gx - 8) % (gy - 8) + 4) for i in range(k)]
        big = raster_in_tiles(view, big_tiles, rng, scale=big_scale, jitter=0.25)
        one = raster_in_tiles(view, rng.randint(0, [gx, gy], (singles, 2)), rng)
        # two tiles: centred on a vertical tile border
        tiles2 = rng.randint([1, 0], [gx, gy], (doubles, 2))
        two = raster_in_tiles(view, tiles2, rng, jitter=0.0)
        pix = np.stack([tiles2[:, 0] * RASTER_TILE + rng.uniform(-0.3, 0.3, doubles),
                        tiles2[:, 1] * RASTER_TILE + 7.5 + rng.uniform(-2, 2, doubles)], 1)
        two.means[:] = world_at_pixel(view, pix[:, 0], pix[:, 1], 5.0 + rng.uniform(-0.5, 0.5, doubles))
        c = concat(big, one, two)
        perm = rng.permutation(B)
        return scene.Cloud(c.means[perm], c.scales[perm], c.rotations[perm], c.density[perm])

    tail = raster_in_tiles(view, rng.randint(0, [gx, gy], (100, 2)), rng, scale=big_scale)
    cloud = concat(block(S, 0), block(S + 1, 7), tail)
    return Case("cta_4608_4609", "raster", cloud, view=view,
                expect=dict(path="direct", cta_total={0: S, 1: S + 1}, staged={0: True, 1: False, 2: True}))


def _tile_counts(counts_per_tile: dict, grid_tiles, maker, rng):
    tiles = []
    for t, n in counts_per_tile.items():
        tiles += [grid_tiles[t]] * n
    tiles = np.asarray(tiles)
    c = maker(tiles, rng)
    perm = rng.permutation(c.P)
    return scene.Cloud(c.means[perm], c.scales[perm], c.rotations[perm], c.density[perm])


def raster_counts_case() -> Case:
    """Per-tile instance counts around the chunk of the work plan (PLAN_CHUNK) and one tile of >= 40 chunks, on a
    256^2 detector (T = 256).  Tile 0 stays empty."""
    rng = np.random.RandomState(12)
    view = parallel_view(256, 256)
    gx, gy = tile_grid((256, 256))
    C = K["PLAN_CHUNK"]
    want = {1: 0, 3: 1, 5: C - 1, 20: C, 37: C + 1, 54: 2 * C, 71: 2 * C + 1, 120: 40 * C + 1}
    tiles = {t: (t % gx, t // gx) for t in want}
    cloud = _tile_counts(want, tiles, lambda t, r: raster_in_tiles(view, t, r), rng)
    return Case("raster_tile_counts", "raster", cloud, view=view, crowded=(120,),
                expect=dict(path="direct", counts={0: 0, **want}, min_chunks=40))


def voxel_counts_case() -> Case:
    """The same per-tile counts for the voxelizer, whose chunk grows with R: filler Gaussians covering the upper half of
    a 64 x 64 x 128 grid (T = 1024) bring R above PLAN_ITEMS * (PLAN_CHUNK + 1), so the chunk is 2 PLAN_CHUNK and an
    item of more than PLAN_CHUNK records is walked in several segments.  The fillers' density puts every one of their
    alphas below the cut: they are binned, planned and walked, and add nothing to the volume."""
    rng = np.random.RandomState(13)
    grid = ((64, 64, 128), (1.0, 1.0, 2.0), (0.0, 0.0, 0.0))
    g = tile_grid(grid[0])
    C2 = 2 * K["PLAN_CHUNK"]
    want = {1: 0, 2: 1, 3: K["PLAN_CHUNK"] - 1, 4: K["PLAN_CHUNK"] + 1, 9: C2 - 1, 10: C2, 11: C2 + 1,
            12: 2 * C2 + 1, 27: 40 * C2 + 1}
    tiles = {t: (t % g[0], (t // g[0]) % g[1], t // (g[0] * g[1])) for t in want}
    cells = _tile_counts(want, tiles, lambda t, r: voxel_in_tiles(grid, t, r), rng)
    # fillers: centred on the upper half, radius 31 voxels -> tiles x, y 0..7, z 8..15 (512 each)
    dv = 1.0 / 64
    R_min = K["PLAN_ITEMS"] * (K["PLAN_CHUNK"] + 1)
    nfill = -(-(R_min - cells.P) // 512) + 8
    pv = np.array([32.0, 32.0, 96.0]) + rng.uniform(-0.4, 0.4, (nfill, 3))
    fill = make(voxel_world(grid, pv), np.full((nfill, 3), 30.5 * dv / 3), dens=rng.uniform(2e-7, 8e-7, nfill))
    cloud = concat(cells, fill)
    return Case("voxel_tile_counts", "voxel", cloud, grid=grid, crowded=(27,),
                expect=dict(path="direct", counts={0: 0, **want}, chunk_gt=K["PLAN_CHUNK"], min_segments=2,
                            min_chunks=40))


def _straddle(f, lo, hi, limit, inside_below=True, rel=0.005):
    """Parameters x_in, x_out with f(x) = limit * (1 -+ rel): just inside / just outside a limit (f monotonic)."""
    t_in = limit * (1 - rel) if inside_below else limit * (1 + rel)
    t_out = limit * (1 + rel) if inside_below else limit * (1 - rel)
    return bisect(f, lo, hi, t_in), bisect(f, lo, hi, t_out)


def _margins(name, n):
    """The first n Gaussians just inside the limit `name` (margin in [0.99, 1)), the next n just outside."""
    return [(name, np.arange(n), 0.99, 1.0), (name, np.arange(n, 2 * n), 1.0, 1.01)]


def raster_fastpath_cases() -> list:
    """Gaussians just inside and just outside each limit of the raster fast path (0.5 % either side), 16 of each, plus
    ordinary Gaussians; one cloud per limit, so that each image's bar is set by the Gaussians under test."""
    view = parallel_view(256, 256)
    ax = view_axes(view)
    fx = 0.5 * view.image_width
    n, depth_scale = 16, 0.01

    def scales(sx, sy, k=1):
        sc = np.full((k, 3), depth_scale)
        sc[:, ax[0]], sc[:, ax[1]] = sx, sy
        return sc

    def probe(sc, dens=0.5):
        return _oracle_raster(make(world_at_pixel(view, 128.3, 128.6), sc, dens=dens), view)

    # A2: a conic narrow along view x (the pixel-space variance along x shrinks towards the low-pass floor)
    a2 = lambda s: float(probe(scales(s, 2.0 / fx))["conic_opacity"][0, 0]) * 0.5 * float(LOG2E)
    s_in, s_out = _straddle(a2, 1e-6, 3.0 / fx, K["RAS_A2_MAX"])
    # log2 w at both ends: w = rho mu, mu proportional to the depth extent (parallel beam)
    mu = float(probe(scales(3.0 / fx, 3.0 / fx))["mu"][0])
    specs = {
        "a2": ((s_in, 2.0 / fx), (s_out, 2.0 / fx), None),
        "lw_max": ((3.0 / fx, 3.0 / fx),) * 2 + ((2.0 ** (K["RAS_LW_MAX"] * 0.995) / mu, 2.0 ** (K["RAS_LW_MAX"] * 1.005) / mu),),
        "lw_min": ((3.0 / fx, 3.0 / fx),) * 2 + ((2.0 ** (K["RAS_LW_MIN"] * 0.995) / mu, 2.0 ** (K["RAS_LW_MIN"] * 1.005) / mu),),
    }
    out = []
    for name, (p_in, p_out, rho) in specs.items():
        rng = np.random.RandomState(len(name))
        parts = []
        for side, (sx, sy) in enumerate((p_in, p_out)):
            sc = scales(sx, sy * rng.uniform(0.9, 1.1, n), n)     # the y extent does not move A2
            sc[:, ax[2]] *= rng.uniform(0.9, 1.1, n)              # the depth extent moves mu only ...
            d = rng.uniform(0.3, 0.7, n) if rho is None else rho[side] * depth_scale / sc[:, ax[2]]   # ... w stays
            pix = rng.uniform(20, 236, (n, 2))
            parts.append(make(world_at_pixel(view, pix[:, 0], pix[:, 1], 5.0 + rng.uniform(-0.3, 0.3, n)), sc, dens=d))
        ordinary = scene.make_cloud(200, kind="trained", seed=len(name))
        if name == "lw_max":   # of the same magnitude as the Gaussians under test
            ordinary.density *= np.float32(2.0 ** (K["RAS_LW_MAX"] * 0.98) / mu)
        fast = {i: i < n for i in range(2 * n)}
        out.append(Case(f"raster_fast_{name}", "raster", concat(*parts, ordinary), view=view,
                        expect=dict(fast=fast, margins=_margins(name if name != "a2" else "A2", n))))
    out.append(raster_det_case())
    return out


def _quat_about(axis_world: int, angle: float):
    q = np.zeros(4)
    q[0] = math.cos(angle / 2)
    q[1 + axis_world] = math.sin(angle / 2)
    return q


def raster_det_case() -> Case:
    """Needles at 45 degrees in the image plane whose conic's (conx conz - cony^2) / (conx conz) sits 0.5 % above and
    below the det-ratio limit."""
    view = parallel_view(256, 256)
    ax = view_axes(view)
    fx = 0.5 * view.image_width
    q = _quat_about(ax[2], math.pi / 4)

    def needle(s_long, n=1, rng=None, pix=((128.3, 128.6),)):
        sc = np.full((n, 3), 0.5 / fx)
        sc[:, ax[0]] = s_long
        sc[:, ax[2]] = 0.01
        pix = np.asarray(pix, np.float64)
        return make(world_at_pixel(view, pix[:, 0], pix[:, 1]), sc, rots=q, dens=0.5)

    ratio = lambda s: K["RAS_DET_RATIO"] / float(raster_margins(_oracle_raster(needle(s), view))["det"][0])
    s_in, s_out = _straddle(ratio, 2.0 / fx, 400.0 / fx, K["RAS_DET_RATIO"], inside_below=False)
    rng = np.random.RandomState(21)
    n = 12
    parts = []
    for s in (s_in, s_out):
        pix = rng.uniform(60, 196, (n, 2))
        c = needle(s * rng.uniform(0.9999, 1.0001, n), n, pix=pix)
        c.density[:, 0] = rng.uniform(0.3, 0.7, n)
        parts.append(c)
    cloud = concat(*parts, scene.make_cloud(100, kind="trained", seed=4))
    fast = {i: i < n for i in range(2 * n)}
    return Case("raster_fast_det", "raster", cloud, view=view, expect=dict(fast=fast, margins=_margins("det", n)),
                needles=tuple(range(2 * n)))


def voxel_fastpath_cases() -> list:
    """The voxelizer's fast-path limits: F2 (the z-z entry of the voxel-space conic), log2 rho at both ends and the
    2 x 2 minor ratio, 0.5 % either side; on a 48^3 grid (T = 216)."""
    grid = ((48, 48, 48), (1.5, 1.5, 1.5), (0.0, 0.0, 0.0))
    dv = 1.5 / 48
    out = []
    centre = voxel_world(grid, [24.2, 23.7, 24.4])

    def orc1(c):
        return _oracle_voxel(c, grid)

    f2 = lambda s: float(orc1(make(centre, [0.3 * dv, 0.3 * dv, s]))["conic_opacity"][0, 5]) * 0.5 * float(LOG2E)
    s_in, s_out = _straddle(f2, 0.2 * dv, 3.0 * dv, K["VOX_F2_MAX"])
    q = _quat_about(2, math.pi / 4)
    m01 = lambda s: K["VOX_M01_RATIO"] / float(voxel_margins(orc1(make(centre, [s, 0.4 * dv, 0.8 * dv], rots=q)))["det"][0])
    d_in, d_out = _straddle(m01, 0.5 * dv, 500 * dv, K["VOX_M01_RATIO"], inside_below=False)
    specs = {
        "F2": (lambda k: np.c_[np.full(k, 0.3 * dv), np.full(k, 0.3 * dv), np.full(k, s_in)],
               lambda k: np.c_[np.full(k, 0.3 * dv), np.full(k, 0.3 * dv), np.full(k, s_out)], None, None),
        "lw_max": (lambda k: np.full((k, 3), 1.5 * dv),) * 2 + (None, (2.0 ** (K["VOX_LW_MAX"] * 0.995), 2.0 ** (K["VOX_LW_MAX"] * 1.005))),
        "lw_min": (lambda k: np.full((k, 3), 1.5 * dv),) * 2 + (None, (2.0 ** (K["VOX_LW_MIN"] * 0.995), 2.0 ** (K["VOX_LW_MIN"] * 1.005))),
        "det": (lambda k: np.c_[np.full(k, d_in), np.full(k, 0.4 * dv), np.full(k, 0.8 * dv)],
                lambda k: np.c_[np.full(k, d_out), np.full(k, 0.4 * dv), np.full(k, 0.8 * dv)], q, None),
    }
    n = 16
    for name, (sc_in, sc_out, rot, rho) in specs.items():
        rng = np.random.RandomState(30 + len(name))
        parts = []
        for side, scf in enumerate((sc_in, sc_out)):
            pv = rng.uniform(10, 38, (n, 3))
            d = rng.uniform(0.3, 0.7, n) if rho is None else rho[side] * rng.uniform(0.9999, 1.0001, n)
            parts.append(make(voxel_world(grid, pv), scf(n), rots=rot, dens=d))
        ordinary = scene.make_cloud(150, kind="trained", seed=len(name), s_voxel=(1.5, 1.5, 1.5),
                                    scale_bound=(0.001, 0.08))
        if name == "lw_max":
            ordinary.density *= np.float32(2.0 ** (K["VOX_LW_MAX"] * 0.98))
        fast = {i: i < n for i in range(2 * n)}
        out.append(Case(f"voxel_fast_{name}", "voxel", concat(*parts, ordinary), grid=grid,
                        expect=dict(fast=fast, margins=_margins(name, n))))
    return out


def careful_case() -> Case:
    """A dense cone-beam cloud: some (Gaussian, pixel) pairs fall inside the bwd_row_careful band."""
    view = cone_view(192, 160, 1.3)
    cloud = scene.make_cloud(4000, kind="trained", seed=17)
    return Case("raster_careful_band", "raster", cloud, view=view, expect=dict(path="direct", careful=True))


def engineered_cases() -> list:
    return [cta_total_case(), raster_counts_case(), voxel_counts_case(), *raster_fastpath_cases(),
            *voxel_fastpath_cases(), careful_case()]
