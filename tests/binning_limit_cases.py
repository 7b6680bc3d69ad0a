"""Inputs at the size limits of the binning front-end: sort pass counts, work-plan sweeps, the batched-view grid's
limits and the largest tile coordinate a uint16 cube holds.

The radix sort takes SORT_BITS bits of tile id per pass, so its pass count (and with it which scatter instantiations
run and which ping-pong buffer ends up sorted) changes at 2^8, 2^16 and 2^24 tiles; the work plan is one CTA that walks
PLAN_THREADS * PLAN_RUN tiles per sweep and carries its running sum from one sweep to the next; the batched-view entry
points accept a stacked tile grid up to the limits `views_shape` (r2x_api.cu) checks, and the single-view and voxel
entry points up to 65535 tiles per axis.  Shapes that cross these limits are large, so the rest of the suite stays
below them; the cases here are built on stated sides of each, and `tests/test_binning_limits_cpu.py` checks on the CPU
oracle that they land there, so that `tests/test_binning_limits_gpu.py` cannot quietly stop exercising them.

Every limit is read from the CUDA sources by regular expression (regime_cases.K where it already has the constant): a
retuned constant moves the cases with it, and a reworded one fails the suite.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

import regime_cases as rc
from r2_gaussian_b200 import scene

TILE, VTILE = rc.RASTER_TILE, rc.VOXEL_TILE


def read_limits() -> dict:
    cuh, cu, api = rc._source("r2x_binning.cuh"), rc._source("r2x_binning.cu"), rc._source("r2x_api.cu")
    k = {n: rc.K[n] for n in ("DIRECT_MAX_TILES", "DIRECT_BLOCK", "PLAN_CHUNK", "VOX_CHUNK_CAP", "SUP")}
    for name in ("SORT_THREADS", "SORT_ITEMS", "SORT_CHUNK", "SORT_MAX_BLOCKS", "DSCAN_COLS"):
        k[name] = rc._constexpr(name, cuh, k)
    k["PLAN_RUN"] = rc._constexpr("PLAN_RUN", cu, k)
    # sort_passes: ceil(bits / SORT_BITS), written as (bits + SORT_BITS - 1) / SORT_BITS
    m = rc._find(r"static int sort_passes\(int num_tiles\) \{[^}]*?return \(bits \+ (\d+)\) / (\d+);", cu, "sort_passes")
    k["SORT_BITS"] = int(m.group(2))
    assert int(m.group(1)) == k["SORT_BITS"] - 1, "sort_passes no longer rounds up"
    # plan_kernel: one CTA of PLAN_THREADS threads, PLAN_THREADS * PLAN_RUN tiles per sweep
    bounds = int(rc._find(r"__launch_bounds__\((\d+)\) plan_kernel", cu, "plan_kernel's launch bounds").group(1))
    launch = int(rc._find(r"plan_kernel<<<1, (\d+), 0", cu, "plan_kernel's launch").group(1))
    sweep = int(rc._find(r"sweep \+= (\d+) \* PLAN_RUN", cu, "plan_kernel's sweep stride").group(1))
    assert bounds == launch == sweep, (bounds, launch, sweep)
    k["PLAN_THREADS"] = sweep
    # views_shape's four limits
    m = rc._find(r"if \(gx > (\d+) \|\| \(long long\)N \* gy > (\d+)\)", api, "views_shape's tile-row limits")
    k["VIEWS_GX_MAX"], k["VIEWS_ROWS_MAX"] = int(m.group(1)), int(m.group(2))
    m = rc._find(r"if \(Pp \* N > \(1ll << (\d+)\) - 1 \|\| gx \* gy \* N > \(1ll << (\d+)\)\)", api,
                 "views_shape's Gaussian and tile limits")
    k["VIEWS_PV_MAX"], k["VIEWS_T_MAX"] = (1 << int(m.group(1))) - 1, 1 << int(m.group(2))
    # the single-view and voxel entry points
    m = rc._find(r"if \(s\.geom\.gx > (\d+) \|\| s\.geom\.gy > (\d+)\)", api, "r2x_raster_forward's detector limit")
    k["RASTER_GX_MAX"], k["RASTER_GY_MAX"] = int(m.group(1)), int(m.group(2))
    m = rc._find(r"if \(vg\.gx > (\d+) \|\| vg\.gy > (\d+) \|\| vg\.gz > (\d+)\)", api, "r2x_voxel_forward's grid limit")
    k["VOXEL_G_MAX"] = tuple(int(m.group(i)) for i in (1, 2, 3))
    k["VOXEL_T_MAX"] = 1 << int(rc._find(r"if \(tiles_ll > \(1ll << (\d+)\)\)", api, "r2x_voxel_forward's tile limit").group(1))
    return k


K = read_limits()
UINT16_MAX = 65535          # the tile cube is uint16 (x0, y0, z0, x1, y1, z1): an end coordinate of 65535 is the largest
GRID_YZ_MAX = 65535         # CUDA's gridDim.y / gridDim.z limit, which the per-axis tile limits follow


# ---- the restatements ---------------------------------------------------------------------------------------------
def sort_passes(T: int) -> int:
    """r2x_binning.cu's sort_passes: SORT_BITS-bit passes over ceil(log2 T) bits (at least one bit)."""
    bits = 1
    while (1 << bits) < T:
        bits += 1
    return -(-bits // K["SORT_BITS"])


def sorted_buffer(T: int) -> int:
    """Which ping-pong key buffer holds the sorted tile ids after the sort (sorted_tile_ids): the pass count's parity."""
    return sort_passes(T) & 1


def plan_sweeps(T: int) -> int:
    """Sweeps of plan_kernel over T tiles."""
    return -(-T // (K["PLAN_THREADS"] * K["PLAN_RUN"]))


def sort_ctas(capacity: int) -> int:
    return min(-(-capacity // K["SORT_CHUNK"]), K["SORT_MAX_BLOCKS"])


def sort_chunks_per_cta(R: int, capacity: int) -> int:
    """SORT_CHUNK chunks each sort CTA walks (per_block_items / SORT_CHUNK)."""
    nb = sort_ctas(capacity)
    per = -(-R // nb)
    return -(-per // K["SORT_CHUNK"])


def views_ok(P: int, N: int, W: int, H: int) -> bool:
    """views_shape's acceptance test."""
    if N < 1 or W <= 0 or H <= 0 or P < 0:
        return False
    gx, gy = -(-W // TILE), -(-H // TILE)
    if gx > K["VIEWS_GX_MAX"] or N * gy > K["VIEWS_ROWS_MAX"]:
        return False
    Pp = -(-max(P, 1) // K["DIRECT_BLOCK"]) * K["DIRECT_BLOCK"]
    return Pp * N <= K["VIEWS_PV_MAX"] and gx * gy * N <= K["VIEWS_T_MAX"]


def views_path(N: int, H: int, W: int) -> str:
    return "direct" if N * (-(-W // TILE)) * (-(-H // TILE)) <= K["DIRECT_MAX_TILES"] else "radix"


def chunk_of(kind: str, R: int) -> int:
    return rc.plan_chunk_for(R, K["PLAN_CHUNK"] if kind == "raster" else K["VOX_CHUNK_CAP"])


# ---- the cases ----------------------------------------------------------------------------------------------------
@dataclass
class Case:
    """One input and what it claims.  kind 'raster' | 'voxel' | 'views'.

    expect: path, T, passes, sweeps, cube_max ({axis: largest end coordinate}), crowded ({tile: at least this many
    instances}), sort ('one_cta' | 'multi_chunk'), straddle ([(tile a, tile b, what the boundary between them is)]).
    mem_gb: the device memory the GPU test may use for the case (torch's peak, checked there)."""
    name: str
    kind: str
    make: object                   # () -> cloud (and views for 'views')
    shape: tuple                   # raster (H, W); voxel (nx, ny, nz); views (N, H, W)
    expect: dict = field(default_factory=dict)
    mem_gb: float = 4.0
    binning: str = ""              # R2X_VOXEL_BINNING
    P: int = 0                     # views: the cloud size (the batched geometry is N * ceil(P / DIRECT_BLOCK) CTAs)

    @property
    def T(self) -> int:
        if self.kind == "raster":
            H, W = self.shape
            return -(-W // TILE) * -(-H // TILE)
        if self.kind == "voxel":
            return int(np.prod([-(-n // VTILE) for n in self.shape]))
        N, H, W = self.shape
        return N * -(-W // TILE) * -(-H // TILE)

    @property
    def path(self) -> str:
        if self.kind == "views":
            return views_path(*self.shape)
        if self.kind == "voxel" and self.binning == "radix" and self.T > K["DIRECT_MAX_TILES"]:
            return "radix"
        return rc.binning_path(self.shape)

    @property
    def grid(self):
        """voxel: (nVoxel, sVoxel, center) with cubic voxels of VOXEL_PITCH."""
        n = self.shape
        return (tuple(n), tuple(float(v) * VOXEL_PITCH for v in n), (0.0, 0.0, 0.0))


VOXEL_PITCH = 1.0 / 128


def flat_view(W: int, H: int):
    """Parallel beam at angle 0, W x H pixels: a pixel is 2 / W by 2 / H world units (rc.parallel_view)."""
    return rc.parallel_view(W, H)


def raster_cloud(view, tiles, seed):
    """One tiny Gaussian per (tx, ty) entry of `tiles`, near that tile's centre: each touches that tile only.  The scale
    is 0.2 px along the detector's longer side."""
    scale = 0.2 * 2.0 / max(view.image_width, view.image_height)
    return rc.raster_in_tiles(view, tiles, np.random.RandomState(seed), scale=scale)


def _tiles_of(ids, gx):
    ids = np.asarray(ids, np.int64)
    return np.stack([ids % gx, ids // gx], 1)


def crowd(tile_ids, n):
    """Each tile id repeated n times."""
    return np.repeat(np.asarray(tile_ids, np.int64), n)


SWEEP = K["PLAN_THREADS"] * K["PLAN_RUN"]
RUN = K["PLAN_RUN"]
CROWD = 2 * K["PLAN_CHUNK"] + 1          # more than 2 C instances: three work items, two extra ones


def plan_crowded(T: int) -> list:
    """Crowded tiles of the work plan: both sides of the first thread-run boundary, of the first sweep boundary, and
    the last tile (which writes extra_off[T])."""
    return [RUN - 1, RUN, SWEEP - 1, SWEEP, T - 1]


def _raster_single(name, side_w, side_h, n_random, crowded, seed, expect, mem_gb, extra=None, few=()):
    W, H = TILE * side_w, TILE * side_h

    def make():
        view = flat_view(W, H)
        T = side_w * side_h
        rng = np.random.RandomState(seed)
        ids = np.concatenate([rng.randint(0, T, n_random), crowd(crowded, CROWD), crowd(few, 4)])
        parts = [raster_cloud(view, _tiles_of(ids, side_w), seed + 1)]
        if extra is not None:
            parts.append(extra(view, rng))
        c = rc.concat(*parts)
        perm = rng.permutation(c.P)
        return scene.Cloud(c.means[perm], c.scales[perm], c.rotations[perm], c.density[perm]), view
    return Case(name, "raster", make, (H, W), expect, mem_gb)


def _big_gaussians(n, px_sigma):
    """n Gaussians of ~px_sigma pixels spread over the detector: each touches about (6 px_sigma / 16)^2 tiles."""
    def extra(view, rng):
        W, H = view.image_width, view.image_height
        m = 4 * px_sigma
        px, py = rng.uniform(m, W - m, n), rng.uniform(m, H - m, n)
        means = rc.world_at_pixel(view, px, py, 5.0 + rng.uniform(-0.5, 0.5, n))
        scale = px_sigma * 2.0 / W * rng.uniform(0.8, 1.2, n)
        # dense enough that the image's scale is several times the alpha cut: a pair within float32 of the cut may be
        # kept by one side and dropped by the other, and the image bar (1e-5 of the scale) must cover one such term
        return rc.make(means, np.repeat(scale[:, None], 3, 1), dens=rng.uniform(3.0, 15.0, n))
    return extra


def raster_cases() -> list:
    B = 2 ** K["SORT_BITS"]
    T2, T3 = B * B, (B + 1) * (B + 1)      # 65536: the last two-pass tile count; 66049: three passes
    wide = K["RASTER_GX_MAX"]              # a tile row 65535 tiles long
    out = [
        # T = 2^16: the largest two-pass grid; exactly two full sweeps, crowded tiles on the sweep boundary
        _raster_single("raster_4096sq", B, B, 3000, [SWEEP - 1, SWEEP, T2 - 1], 1,
                       dict(T=T2, path="radix", passes=2, sweeps=2, cube_max={"x1": B, "y1": B},
                            crowded={SWEEP - 1: CROWD, SWEEP: CROWD, T2 - 1: CROWD},
                            straddle=[(SWEEP - 1, SWEEP, "sweep")]), 1.5),
        # T = (2^8 + 1)^2: three passes (the middle-pass scatter runs, the sorted ids end in keys[1]), three sweeps;
        # R < SORT_CHUNK: one sort CTA holds every instance
        _raster_single("raster_4112sq_few", B + 1, B + 1, 800, plan_crowded(T3), 2,
                       dict(T=T3, path="radix", passes=3, sweeps=3, sort="one_cta",
                            crowded={t: CROWD for t in plan_crowded(T3)},
                            straddle=[(RUN - 1, RUN, "thread run"), (SWEEP - 1, SWEEP, "sweep"),
                                      (T2 - 1, T2, "third sort digit")]), 1.5, few=[T2 - 1, T2]),
        # the same grid with R > SORT_CHUNK * SORT_MAX_BLOCKS: every sort CTA walks several chunks
        _raster_single("raster_4112sq_many", B + 1, B + 1, 2000, [T2 - 1, T2, T3 - 1], 3,
                       dict(T=T3, path="radix", passes=3, sweeps=3, sort="multi_chunk",
                            crowded={T2 - 1: CROWD, T2: CROWD, T3 - 1: CROWD}), 2.0,
                       extra=_big_gaussians(5000, 40.0)),
        # two tile rows of 65535 tiles: the largest x1 a cube holds, three passes, four sweeps
        _raster_single("raster_wide_2x65535", wide, 2, 4000, [wide - 1, 2 * wide - 1, SWEEP, T2], 4,
                       dict(T=2 * wide, path="radix", passes=3, sweeps=plan_sweeps(2 * wide),
                            cube_max={"x1": UINT16_MAX}, crowded={2 * wide - 1: CROWD, SWEEP: CROWD}), 1.5),
    ]
    return out


def _voxel_case(name, n, n_random, crowded, seed, expect, mem_gb, binning=""):
    def make():
        grid = ((n[0], n[1], n[2]), tuple(float(v) * VOXEL_PITCH for v in n), (0.0, 0.0, 0.0))
        g = [-(-v // VTILE) for v in n]
        T = int(np.prod(g))
        rng = np.random.RandomState(seed)
        ids = np.concatenate([rng.randint(0, T, n_random), crowd(crowded, CROWD)])
        tiles = np.stack([ids % g[0], (ids // g[0]) % g[1], ids // (g[0] * g[1])], 1)
        c = rc.voxel_in_tiles(grid, tiles, rng)
        c.scales[:] = np.float32(0.02 * VOXEL_PITCH)      # well inside one voxel: one tile each
        perm = rng.permutation(c.P)
        return scene.Cloud(c.means[perm], c.scales[perm], c.rotations[perm], c.density[perm])
    return Case(name, "voxel", make, tuple(n), expect, mem_gb, binning)


def voxel_cases() -> list:
    S, V = K["SUP"], VTILE
    # 33^3 tiles: more than one sweep, supertiles 9^3 <= DIRECT_MAX_TILES (two-level)
    side = next(s for s in range(1, SWEEP) if s ** 3 > SWEEP)   # 33: the smallest cube of tiles past one sweep
    n264 = (V * side,) * 3
    T264 = side ** 3
    crowd264 = [SWEEP - 1, SWEEP, T264 - 1]
    common = dict(T=T264, sweeps=2, crowded={t: CROWD for t in crowd264}, straddle=[(SWEEP - 1, SWEEP, "sweep")])
    gz = K["VOXEL_G_MAX"][2]
    tall = (V, 2 * V, gz * V)                                  # 1 x 2 x 65535 tiles: supertiles 1 x 1 x 16384
    Tt = 2 * gz
    return [
        _voxel_case(f"voxel_{n264[0]}cube", n264, 3000, crowd264, 5, dict(path="two_level", **common), 1.0),
        _voxel_case(f"voxel_{n264[0]}cube_radix", n264, 3000, crowd264, 5,
                    dict(path="radix", passes=2, **common), 1.0, binning="radix"),
        _voxel_case("voxel_tall_1x2x65535", tall, 4000, [SWEEP - 1, SWEEP, Tt - 1], 6,
                    dict(T=Tt, path="radix", passes=3, sweeps=plan_sweeps(Tt), cube_max={"z1": UINT16_MAX},
                         T1_gt=K["DIRECT_MAX_TILES"], crowded={SWEEP: CROWD, Tt - 1: CROWD}), 2.0),
    ]


def _views(N, H, W, P, seed, kind="trained"):
    """A cone-beam detector of H x W pixels whose longer side spans 4 units (the 512-pixel scanner's), N views evenly
    around the circle, and a cloud of P Gaussians."""
    def make():
        sc = scene.cone_beam_scanner(max(H, W), 64)
        sc["nDetector"] = [H, W]
        sc["sDetector"] = [4.0 * H / max(H, W), 4.0 * W / max(H, W)]
        angles = np.linspace(0.0, 2.0 * math.pi, N + 1)[:-1] + 0.1
        return scene.make_cloud(P, kind=kind, seed=seed), [scene.make_view(sc, float(a)) for a in angles]
    return make


def views_cases() -> list:
    D = K["DIRECT_MAX_TILES"]
    rows = K["VIEWS_ROWS_MAX"]
    B = 2 ** K["SORT_BITS"]
    out = [
        # one-tile bands: every direct_scan CTA's DSCAN_COLS columns are DSCAN_COLS different views
        Case("views_4096x16sq", "views", _views(D, TILE, TILE, 300, 21), (D, TILE, TILE),
             dict(T=D, path="direct", band_tiles=1), 2.0, P=300),
        Case("views_4097x16sq", "views", _views(D + 1, TILE, TILE, 300, 22), (D + 1, TILE, TILE),
             dict(T=D + 1, path="radix", passes=2, sweeps=1), 2.0, P=300),
        # N * gy = 65535 stacked tile rows, two tiles per band: 131070 tiles, three passes
        Case("views_65535x32x16", "views", _views(rows, TILE, 2 * TILE, 24, 23), (rows, TILE, 2 * TILE),
             dict(T=2 * rows, path="radix", passes=3, sweeps=plan_sweeps(2 * rows), cube_max={"z1": UINT16_MAX}), 3.5,
             P=24),
        # a training batch of 17 views of 1024^2: 69632 tiles, three passes, three sweeps
        Case("views_17x1024sq", "views", _views(17, 1024, 1024, 25_000, 24, kind="init"), (17, 1024, 1024),
             dict(T=17 * 64 * 64, path="radix", passes=3, sweeps=3), 4.0, P=25_000),
    ]
    for P in (1, B - 1, B, B + 1):
        out.append(Case(f"views_P{P}_N3", "views", _views(3, 64, 64, P, 30 + P), (3, 64, 64),
                        dict(T=3 * 16, path="direct", band_ctas=-(-P // K["DIRECT_BLOCK"])), 0.5, P=P))
    return out


def views_subset(N: int, tiles_per_view: int) -> list:
    """Views checked one by one for the largest batch: the first, the last, and the views on either side of tile ids
    2^8 and 2^16 (where the second and third sort digits first change)."""
    out = {0, N - 1}
    for b in (K["SORT_BITS"], 2 * K["SORT_BITS"]):
        t = 1 << b
        out |= {(t - 1) // tiles_per_view, t // tiles_per_view}
    return sorted(v for v in out if 0 <= v < N)


def all_cases() -> list:
    return raster_cases() + voxel_cases() + views_cases()


STRADDLE_UNIT = {"thread run": RUN, "sweep": SWEEP, "third sort digit": 1 << (2 * K["SORT_BITS"])}


def check_case(case: Case, orc=None, R=None) -> list:
    """Asserts the case's claims; raster and voxel cases from the oracle's forward (ranges, cubes, R).  Returns one
    report line per claim."""
    ex, T, lines = case.expect, case.T, []
    assert T == ex["T"], (case.name, T, ex["T"])
    assert case.path == ex["path"], (case.name, case.path)
    line = f"T={T} path={case.path}"
    if case.path == "radix":
        assert sort_passes(T) == ex["passes"], (case.name, sort_passes(T))
        line += f" passes={sort_passes(T)} (sorted ids in keys[{sorted_buffer(T)}])"
    if "sweeps" in ex:
        assert plan_sweeps(T) == ex["sweeps"], (case.name, plan_sweeps(T))
        line += f" sweeps={plan_sweeps(T)}"
    lines.append(line)
    if case.kind == "views":
        N, H, W = case.shape
        assert views_ok(case.P, N, W, H), case.name
        if "band_tiles" in ex:
            assert -(-W // TILE) * -(-H // TILE) == ex["band_tiles"], case.name
            lines.append(f"band of {ex['band_tiles']} tile(s): a direct_scan CTA spans {K['DSCAN_COLS']} views")
        if "band_ctas" in ex:
            lines.append(f"P={case.P}: {ex['band_ctas']} padded CTA(s) per view")
        for axis, v in ex.get("cube_max", {}).items():
            assert axis == "z1" and N == v, case.name   # the view is the stacked grid's z: the last view ends at N
            lines.append(f"largest cube z1 = N = {N}")
        return lines
    rg = np.asarray(orc["ranges"], np.int64)
    counts = rg[:, 1] - rg[:, 0]
    R = int(orc["R"])
    assert int(counts.sum()) == R and len(counts) == T
    C = chunk_of(case.kind, R)
    for t, n in ex.get("crowded", {}).items():
        assert counts[t] >= n and counts[t] > 2 * C, (case.name, t, int(counts[t]), C)
        lines.append(f"tile {t}: {int(counts[t])} instances > 2 C = {2 * C}: {-(-int(counts[t]) // C)} work items")
    for a, b, what in ex.get("straddle", []):
        unit = STRADDLE_UNIT[what]
        need = 1 if what == "third sort digit" else 2 * C + 1     # plan boundaries need crowded tiles
        assert b == a + 1 and b % unit == 0 and counts[a] >= need and counts[b] >= need, (case.name, a, b, what)
        lines.append(f"tiles {a} | {b} ({int(counts[a])} | {int(counts[b])} instances) straddle a {what} boundary "
                     f"({unit} tiles)")
    if ex.get("sort") == "one_cta":
        assert 0 < R < K["SORT_CHUNK"], (case.name, R)
        lines.append(f"R={R} < SORT_CHUNK={K['SORT_CHUNK']}: one sort CTA holds every instance")
    if ex.get("sort") == "multi_chunk":
        assert R > K["SORT_CHUNK"] * K["SORT_MAX_BLOCKS"], (case.name, R)
        lines.append(f"R={R} > SORT_CHUNK * SORT_MAX_BLOCKS: each of {K['SORT_MAX_BLOCKS']} sort CTAs walks "
                     f"{sort_chunks_per_cta(R, R)} chunks")
    if case.kind == "raster":
        box = np.asarray(orc["rect"])[np.asarray(orc["radii"]) > 0]
        cols = {"x1": box[:, 2], "y1": box[:, 3]}
    else:
        box = np.asarray(orc["cube"])[np.asarray(orc["tiles_touched"]) > 0]
        cols = {"x1": box[:, 3], "y1": box[:, 4], "z1": box[:, 5]}
    for axis, v in ex.get("cube_max", {}).items():
        assert int(cols[axis].max()) == v, (case.name, axis, int(cols[axis].max()), v)
        lines.append(f"largest cube {axis} = {v}")
    if "T1_gt" in ex:
        T1 = int(np.prod([-(-(-(-n // VTILE)) // K["SUP"]) for n in case.shape]))
        assert T1 > ex["T1_gt"], (case.name, T1)
        lines.append(f"supertiles T1={T1} > {ex['T1_gt']}: radix by default")
    return lines


def oracle(case: Case, cloud, view=None):
    import util
    if case.kind == "raster":
        return util.oracle_raster_forward(cloud, view)
    return util.oracle_voxel_forward(cloud, *case.grid)
