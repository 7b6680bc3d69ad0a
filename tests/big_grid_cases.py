"""Grids past 2^31 and 2^32 elements, and tile grids past 2^24 tiles, for the voxelizer, the rasterizer, batched views
and the TV loss.

Two families of code paths run only at these sizes.  The voxelizer's stores, its backward's dL_dvol gather, the zero
fill of an empty forward and the TV loss index a flat volume with 64-bit offsets; a 32-bit product anywhere wraps once
the grid passes 2^31 (signed) or 2^32 (unsigned) elements.  The radix sort of the binning takes SORT_BITS bits of tile
id per pass and needs a fourth pass past 2^24 tiles: the middle <false, false> scatter then runs twice in a row, the
sorted ids end back in keys[0] (sort_passes() even) and the backward reads inst_pos, which only the last pass writes.
None of the other case tables reaches either.

Each case is a grid whose every element is held in device memory, and a small cloud: each Gaussian sits inside one
tile.  The clouds fill the first tile, the tiles holding the flat indices each case is named after, the last tile, one
crowded tile of several work-plan chunks (and, with four passes, both sides of tile id 2^24) plus some random tiles;
the rest of the grid stays empty, so a run is dominated by memory traffic, not by render work.  `peak` is the device
memory the GPU test may use for the case; `tests/test_big_grid_cpu.py` checks it against the buffers that test
allocates, and that every case lands where it claims (tile count, sort passes, the windows' flat indices), on the CPU.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

import binning_limit_cases as blc
import regime_cases as rc
from r2_gaussian_b200 import scene
from binning_limit_cases import K, plan_sweeps, sort_passes, sorted_buffer  # noqa: F401  (re-exported for the tests)

TILE, VTILE = blc.TILE, blc.VTILE
GiB = 1 << 30
SLAB = 1 << 25                      # elements per device slab: dL generation, zero counts and digests
FOURTH_DIGIT = 1 << (3 * K["SORT_BITS"])
CROWD = blc.CROWD
VOXEL_PITCH = blc.VOXEL_PITCH
VOXEL_SCALE = 0.3                   # Gaussian sigma in voxels: radius ceil(3 sigma) = 1 voxel
RASTER_SCALE = 0.3                  # Gaussian sigma in detector pixels (the kernel adds 0.3 to the 2-D covariance)
RASTER_DEPTH = 0.1                  # world sigma along the view's depth: the line integral mu, so alpha, is of order 0.1


@dataclass
class Case:
    """kind 'voxel' | 'raster' | 'views' | 'tv'.  shape: voxel / tv (nx, ny, nz); raster (H, W); views (N, H, W).
    sites: {label: flat element index} the case must hold in a judged window.  expect: T, passes (and for the tv case
    nothing).  one_buffer: the forward's volume is overwritten with dL for the backward (no room for both)."""
    name: str
    kind: str
    shape: tuple
    sites: dict
    expect: dict = field(default_factory=dict)
    peak: int = 0
    n_random: int = 600
    seed: int = 0
    P: int = 0                       # views: the cloud size
    one_buffer: bool = False
    python_path: bool = False        # also run through query() + autograd and compare bit for bit

    @property
    def n(self) -> int:
        return math.prod(self.shape)

    @property
    def grid(self) -> tuple:
        """Tiles per axis: voxel (gx, gy, gz), raster (gx, gy), views (gx, gy) of one view."""
        if self.kind in ("voxel", "tv"):
            return tuple(-(-v // VTILE) for v in self.shape)
        H, W = self.shape[-2:]
        return (-(-W // TILE), -(-H // TILE))

    @property
    def T(self) -> int:
        t = math.prod(self.grid)
        return t * self.shape[0] if self.kind == "views" else t

    def tile_of(self, flat: int) -> int:
        """The tile holding flat element `flat` (voxel: x-major volume, x-fastest tile ids; raster / views: row-major
        image(s), x-fastest tiles, the view as the stacked grid's slowest axis)."""
        if self.kind in ("voxel", "tv"):
            nx, ny, nz = self.shape
            x, y, z = flat // (ny * nz), (flat // nz) % ny, flat % nz
            gx, gy, _ = self.grid
            return x // VTILE + gx * (y // VTILE + gy * (z // VTILE))
        H, W = self.shape[-2:]
        gx, gy = self.grid
        v, r = divmod(flat, H * W)
        y, x = divmod(r, W)
        return v * gx * gy + x // TILE + gx * (y // TILE)

    def tile_box(self, t: int) -> tuple:
        """((lo, hi) per array axis) of tile t's elements: voxel (x, y, z); raster (y, x); views (v, y, x)."""
        if self.kind in ("voxel", "tv"):
            gx, gy, _ = self.grid
            o = (t % gx, (t // gx) % gy, t // (gx * gy))
            return tuple((VTILE * k, min(n, VTILE * k + VTILE)) for k, n in zip(o, self.shape))
        H, W = self.shape[-2:]
        gx, gy = self.grid
        v, r = divmod(t, gx * gy)
        ty, tx = divmod(r, gx)
        box = ((TILE * ty, min(H, TILE * ty + TILE)), (TILE * tx, min(W, TILE * tx + TILE)))
        return ((v, v + 1),) + box if self.kind == "views" else box

    def flat_range(self, box) -> tuple:
        """(smallest, largest) flat index of the elements of a box."""
        lo = [a for a, _ in box]
        hi = [b - 1 for _, b in box]
        return flat_index(self.shape, lo), flat_index(self.shape, hi)

    def crowded_tile(self) -> int:
        return self.T // 2 + 1

    def placements(self) -> np.ndarray:
        """Tile ids of the cloud's Gaussians: the judged tiles, the crowded one CROWD times, random tiles."""
        rng = np.random.RandomState(self.seed)
        return np.concatenate([np.asarray(self.judged_tiles(), np.int64), blc.crowd([self.crowded_tile()], CROWD - 1),
                               rng.randint(0, self.T, self.n_random)])

    def judged_tiles(self) -> list:
        """First and last tile, the tiles holding each site and the element before it, the crowded tile and (four passes)
        both sides of tile id 2^24."""
        t = {0, self.T - 1, self.crowded_tile()} | {self.tile_of(f) for f in self.sites.values()}
        t |= {self.tile_of(f - 1) for f in self.sites.values() if f > 0}
        if self.T > FOURTH_DIGIT:
            t |= {FOURTH_DIGIT - 1, FOURTH_DIGIT}
        return sorted(t)


def flat_index(shape, idx) -> int:
    f = 0
    for i, n in zip(idx, shape):
        f = f * n + int(i)
    return f


def unflat(shape, f) -> tuple:
    out = []
    for n in reversed(shape):
        f, r = divmod(int(f), n)
        out.append(r)
    return tuple(reversed(out))


# ---- clouds ---------------------------------------------------------------------------------------------------------
def _inside(tiles, edge, end, margin):
    """Per axis, the range of centres inside tile `tiles` whose cube / rectangle of radius `margin` stays in that tile,
    cut at `end` (a partial last tile: the centre stays within reach of its elements)."""
    lo = tiles * edge + margin + 0.05
    hi = np.minimum(tiles * edge + edge - margin - 0.05, end)
    return lo, np.maximum(hi, lo + 0.1)


def voxel_cloud(case: Case):
    """One Gaussian per placement, sigma VOXEL_SCALE voxels (cube radius 1 voxel), inside its tile."""
    rng = np.random.RandomState(case.seed + 1)
    ids = case.placements()
    gx, gy, _ = case.grid
    tiles = np.stack([ids % gx, (ids // gx) % gy, ids // (gx * gy)], 1)
    pv = np.empty((len(ids), 3))
    for a in range(3):
        lo, hi = _inside(tiles[:, a], VTILE, float(case.shape[a]), 1.0)
        pv[:, a] = rng.uniform(lo, hi)
    grid = voxel_grid(case)
    c = rc.make(rc.voxel_world(grid, pv), np.full((len(ids), 3), VOXEL_SCALE * VOXEL_PITCH),
                dens=rng.uniform(0.3, 0.7, len(ids)))
    perm = rng.permutation(c.P)
    return scene.Cloud(c.means[perm], c.scales[perm], c.rotations[perm], c.density[perm])


def voxel_grid(case: Case) -> tuple:
    n = case.shape
    return (tuple(n), tuple(float(v) * VOXEL_PITCH for v in n), (0.0, 0.0, 0.0))


def raster_view(case: Case):
    H, W = case.shape
    return rc.parallel_view(W, H)


def raster_cloud(case: Case):
    """One Gaussian per placement, sigma RASTER_SCALE pixels along both detector axes (the 2-D footprint's radius is 2
    pixels) and RASTER_DEPTH along the view's depth, inside its tile."""
    view = raster_view(case)
    H, W = case.shape
    rng = np.random.RandomState(case.seed + 1)
    ids = case.placements()
    gx, _ = case.grid
    px_lo, px_hi = _inside(ids % gx, TILE, W - 0.5, 2.5)
    py_lo, py_hi = _inside(ids // gx, TILE, H - 0.5, 2.5)
    px, py = rng.uniform(px_lo, px_hi), rng.uniform(py_lo, py_hi)
    means = rc.world_at_pixel(view, px, py, 5.0 + rng.uniform(-0.5, 0.5, len(ids)))
    scales = np.zeros((len(ids), 3))
    ax = rc.view_axes(view)                       # world axis along view x, view y and view depth
    scales[:, ax[0]], scales[:, ax[1]], scales[:, ax[2]] = RASTER_SCALE * 2.0 / W, RASTER_SCALE * 2.0 / H, RASTER_DEPTH
    c = rc.make(means, scales, dens=rng.uniform(0.3, 0.7, len(ids)))
    perm = rng.permutation(c.P)
    return scene.Cloud(c.means[perm], c.scales[perm], c.rotations[perm], c.density[perm]), view


VIEWS_SCALES = (0.001, 0.004)      # world scale bounds of the views case's cloud: a few tiles per Gaussian and view


def views_scene(case: Case):
    """A cone-beam detector of H x W pixels whose longer side spans 4 units, N views around the circle (the scanner of
    binning_limit_cases._views), and a trained cloud of small Gaussians squeezed into the slab of the volume the
    detector's rows see."""
    N, H, W = case.shape
    _, views = blc._views(N, H, W, 1, case.seed)()
    cloud = scene.make_cloud(case.P, kind="trained", seed=case.seed, s_voxel=(2.0, 2.0, 0.2), scale_bound=VIEWS_SCALES)
    return cloud, views


# ---- the oracle's per-Gaussian stage ----------------------------------------------------------------------------------
def oracle_voxel_preprocess(cloud, grid) -> dict:
    """The CPU oracle's voxel preprocess alone (no volume is allocated): radii, xyz_vol, depth, cov3D, conic_opacity,
    tiles_touched, cube."""
    import ctypes as C

    from oracle import r2_oracle as orc

    (nx, ny, nz), sV, ctr = grid
    P = cloud.P
    f = np.float32
    out = dict(radii_x=np.zeros(P, np.int32), radii_y=np.zeros(P, np.int32), radii_z=np.zeros(P, np.int32),
               xyz_vol=np.zeros((P, 3), f), depth=np.zeros(P, f), cov3D=np.zeros((P, 6), f),
               conic_opacity=np.zeros((P, 7), f), tiles_touched=np.zeros(P, np.uint32), cube=np.zeros((P, 6), np.int32))
    m, s, r, o = (orc._c(a, f) for a in (cloud.means, cloud.scales, cloud.rotations, cloud.density.reshape(-1)))
    R = orc.lib().orc_voxel_preprocess(
        C.c_int(P), orc._p(m, orc._fp), orc._p(s, orc._fp), C.c_float(1.0), orc._p(r, orc._fp), orc._p(o, orc._fp),
        None, C.c_int(nx), C.c_int(ny), C.c_int(nz), *(C.c_float(v) for v in sV), *(C.c_float(v) for v in ctr),
        orc._p(out["radii_x"], orc._ip), orc._p(out["radii_y"], orc._ip), orc._p(out["radii_z"], orc._ip),
        orc._p(out["xyz_vol"], orc._fp), orc._p(out["depth"], orc._fp), orc._p(out["cov3D"], orc._fp),
        orc._p(out["conic_opacity"], orc._fp), orc._p(out["tiles_touched"], orc._up), orc._p(out["cube"], orc._ip))
    out["R"] = int(R)
    return out


def oracle_raster_preprocess(cloud, view) -> dict:
    """The CPU oracle's raster preprocess alone (no image is allocated)."""
    import ctypes as C

    from oracle import r2_oracle as orc

    P, W, H = cloud.P, view.image_width, view.image_height
    f = np.float32
    out = dict(radii=np.zeros(P, np.int32), xy=np.zeros((P, 2), f), depth=np.zeros(P, f), cov3D=np.zeros((P, 6), f),
               conic_opacity=np.zeros((P, 4), f), mu=np.zeros(P, f), tiles_touched=np.zeros(P, np.uint32),
               rect=np.zeros((P, 4), np.int32))
    m, s, r, o = (orc._c(a, f) for a in (cloud.means, cloud.scales, cloud.rotations, cloud.density.reshape(-1)))
    vm, pm = orc._c(view.viewmatrix, f).reshape(16), orc._c(view.projmatrix, f).reshape(16)
    R = orc.lib().orc_raster_preprocess(
        C.c_int(P), orc._p(m, orc._fp), orc._p(s, orc._fp), C.c_float(1.0), orc._p(r, orc._fp), orc._p(o, orc._fp),
        None, orc._p(vm, orc._fp), orc._p(pm, orc._fp), C.c_int(W), C.c_int(H), C.c_float(view.tanfovx),
        C.c_float(view.tanfovy), C.c_int(view.mode), orc._p(out["radii"], orc._ip), orc._p(out["xy"], orc._fp),
        orc._p(out["depth"], orc._fp), orc._p(out["cov3D"], orc._fp), orc._p(out["conic_opacity"], orc._fp),
        orc._p(out["mu"], orc._fp), orc._p(out["tiles_touched"], orc._up), orc._p(out["rect"], orc._ip))
    out["R"] = int(R)
    return out


def predicted_keys(case: Case, pre: dict) -> tuple:
    """(tile id, Gaussian id) of every instance the oracle's cubes / rectangles predict, sorted by (tile, id): the
    order the stable sort must leave point_list in, each Gaussian being emitted in id order."""
    tiles, gids = [], []
    if case.kind == "voxel":
        gx, gy, _ = case.grid
        for g in np.nonzero(pre["tiles_touched"] > 0)[0]:
            x0, y0, z0, x1, y1, z1 = (int(v) for v in pre["cube"][g])
            zz, yy, xx = np.meshgrid(np.arange(z0, z1), np.arange(y0, y1), np.arange(x0, x1), indexing="ij")
            t = (xx + gx * (yy + gy * zz)).reshape(-1)
            tiles.append(t)
            gids.append(np.full(len(t), g))
    else:
        gx, _ = case.grid
        for g in np.nonzero(pre["radii"] > 0)[0]:
            x0, y0, x1, y1 = (int(v) for v in pre["rect"][g])
            yy, xx = np.meshgrid(np.arange(y0, y1), np.arange(x0, x1), indexing="ij")
            t = (xx + gx * yy).reshape(-1)
            tiles.append(t)
            gids.append(np.full(len(t), g))
    t = np.concatenate(tiles).astype(np.int64)
    g = np.concatenate(gids).astype(np.int64)
    order = np.lexsort((g, t))
    return t[order], g[order]


def predicted_ranges(T: int, tiles: np.ndarray) -> np.ndarray:
    """[T, 2] ranges in the reference's convention (an empty tile reads (0, 0)) of a tile-sorted instance list."""
    cnt = np.bincount(tiles, minlength=T).astype(np.int64)
    end = np.cumsum(cnt)
    out = np.stack([end - cnt, end], 1)
    out[cnt == 0] = 0
    return out.astype(np.uint32)


# ---- dL: a seeded function of the flat index -------------------------------------------------------------------------
def _hash(idx, seed, xp):
    """24 bits of a hash of int64 flat indices (numpy or torch: the same integer arithmetic, no overflow below 2^36)."""
    h = idx * 40503 + (seed * 7919 + 12345)
    h = h ^ (h >> 13)
    h = (h * 1103) & 0xFFFFFF
    return h ^ ((h >> 7) & 0xFFF)


def dl_host(idx: np.ndarray, seed: int) -> np.ndarray:
    """dL at flat indices idx (int64 array of any shape), float32 in [-1, 1): an integer over 2^23, exact in float32."""
    h = _hash(np.asarray(idx, np.int64), seed, np)
    return ((h - (1 << 23)).astype(np.float32) * np.float32(2.0 ** -23)).astype(np.float32)


def dl_fill(t, seed: int, start: int = 0):
    """Write dl_host's values into the contiguous float32 tensor t (flat index = start + position), slab by slab."""
    import torch

    flat = t.view(-1)
    for lo in range(0, flat.numel(), SLAB):
        hi = min(flat.numel(), lo + SLAB)
        idx = torch.arange(start + lo, start + hi, device=t.device, dtype=torch.int64)
        h = _hash(idx, seed, torch)
        flat[lo:hi] = (h - (1 << 23)).to(torch.float32) * (2.0 ** -23)
        del idx, h


class FlatField:
    """dl_host over a whole grid of `shape`, read by slicing like the array it stands for: the float64 statements
    (grad_float64.voxel_moments / raster_moments) slice dL at each Gaussian's cube or rectangle only."""

    def __init__(self, shape, seed):
        self.shape, self.seed = tuple(shape), seed

    def astype(self, dtype):
        return self

    def __getitem__(self, key):
        axes = [np.arange(n)[k] for k, n in zip(key, self.shape)]
        idx = np.zeros([len(a) for a in axes], np.int64)
        for d, a in enumerate(axes):
            sh = [1] * len(axes)
            sh[d] = len(a)
            idx = idx * self.shape[d] + a.reshape(sh)
        return dl_host(idx, self.seed).astype(np.float64)


# ---- the cases ------------------------------------------------------------------------------------------------------
def _sites(shape, *powers) -> dict:
    n = math.prod(shape)
    out = {f"2^{p}": 1 << p for p in powers}
    out["last"] = n - 1
    return out


def cases() -> list:
    v31, v32, v4 = (1297, 1291, 1283), (1625, 1630, 1627), (2053, 2051, 2049)
    W, H = (blc.K["RASTER_GX_MAX"] - 1) * TILE + 7, (2 ** K["SORT_BITS"]) * TILE + 9    # 65535 x 257 tiles, both partial
    # batched views: N * ceil(H / 16) tile rows <= 65535 (views_shape), so 4095 views of 16 tile rows, 257 tiles wide
    N, Hv, Wv = blc.GRID_YZ_MAX // 16, 16 * TILE, (2 ** K["SORT_BITS"]) * TILE + 9
    B = lambda *vols: int(sum(vols) * 4)                                                # noqa: E731
    return [
        Case("voxel_past_2_31", "voxel", v31, _sites(v31, 31), dict(T=163 * 162 * 161, passes=3),
             peak=B(*[math.prod(v31)] * 3) + 4 * GiB, seed=31, python_path=True),
        Case("voxel_past_2_32", "voxel", v32, _sites(v32, 31, 32), dict(T=204 * 204 * 204, passes=3),
             peak=B(*[math.prod(v32)] * 2) + 4 * GiB, seed=32),
        Case("voxel_four_passes", "voxel", v4, _sites(v4, 31, 32, 33), dict(T=257 ** 3, passes=4),
             peak=B(math.prod(v4)) + 4 * GiB, seed=33, one_buffer=True),
        Case("views_four_passes", "views", (N, Hv, Wv), dict(view0=0, view_mid=N // 3 * Hv * Wv, **_sites((N, Hv, Wv), 31, 32)),
             dict(T=N * 16 * 257, passes=4), peak=B(*[N * Hv * Wv] * 2) + 8 * GiB, seed=34, P=500),
        Case("raster_four_passes", "raster", (H, W), _sites((H, W), 31, 32), dict(T=65535 * 257, passes=4),
             peak=B(*[W * H] * 2) + 4 * GiB, seed=35),
        Case("tv3d_past_2_31", "tv", v31, _sites(v31, 31), peak=B(*[math.prod(v31)] * 2) + 4 * GiB, seed=36),
    ]


def judged_views(case: Case) -> list:
    """The views of the batch judged one by one: those holding the case's sites (the first, a middle one, the one that
    holds pixel 2^31, the one that holds 2^32 and the last)."""
    H, W = case.shape[1:]
    return sorted({f // (H * W) for f in case.sites.values()})


CASES = {c.name: c for c in cases()}


def tv_windows(case: Case) -> dict:
    """TV gradient windows {label: box}: 8 voxels along each axis around flat index 2^31, the plane boundary (x) and row
    boundary (y) nearest it, the first and the last voxel."""
    nx, ny, nz = case.shape
    x, y, z = unflat(case.shape, 1 << 31)
    centres = {"2^31": (x, y, z), "x_plane": (x, 0, 0), "y_row": (x, y, 0), "first": (0, 0, 0),
               "last": (nx - 1, ny - 1, nz - 1)}
    return {k: tuple((max(0, c - 4), min(n, c + 4)) for c, n in zip(cen, case.shape)) for k, cen in centres.items()}


def halo(box, shape) -> tuple:
    return tuple((max(0, a - 1), min(n, b + 1)) for (a, b), n in zip(box, shape))


# ---- device memory -------------------------------------------------------------------------------------------------
def device_buffers(case: Case, P: int, R: int) -> dict:
    """Bytes of every device buffer the GPU test holds at the case's peak, for a cloud of P Gaussians (views: per view)
    and R instances."""
    from r2_gaussian_b200 import _C, _lib

    lib = _lib.load()
    n4 = case.n * 4
    slab = 6 * SLAB * 8                                   # dl_fill / digest / zero-count temporaries (int64)
    if case.kind == "tv":
        return dict(vol=n4, grad=n4, scratch=lib.r2x_tv3d_scratch_bytes(*case.shape), slab=slab)
    kind = _C.RASTER if case.kind in ("raster", "views") else _C.VOXEL
    Pb = P * case.shape[0] if case.kind == "views" else P
    cap = max(_C._Workspace.first(Pb, kind.seed), _C._Workspace.grown(R))
    out = dict(out=n4, binning=lib.r2x_binning_bytes(cap), export=case.T * 8 + cap * 12 + 64 * P, slab=slab)
    if case.kind == "voxel":
        out.update(geom=lib.r2x_voxel_geom_bytes(P), image=lib.r2x_voxel_image_bytes(P, *case.shape),
                   scratch=lib.r2x_voxel_bwd_scratch_bytes(cap))
        if not case.one_buffer:
            out["dL"] = n4
        if case.python_path:
            out["python_out"] = n4
    elif case.kind == "raster":
        H, W = case.shape
        out.update(geom=lib.r2x_raster_geom_bytes(P), image=lib.r2x_raster_image_bytes(P, W, H),
                   scratch=lib.r2x_raster_bwd_scratch_bytes(cap), dL=n4)
    else:
        N, H, W = case.shape
        out.update(geom=lib.r2x_raster_views_geom_bytes(P, N), image=lib.r2x_raster_views_image_bytes(P, N, W, H),
                   scratch=lib.r2x_raster_bwd_scratch_bytes(cap), dL=n4, mean2D=N * P * 12,
                   single=lib.r2x_raster_geom_bytes(P) + lib.r2x_raster_image_bytes(P, W, H) + 4 * H * W * 2
                   + lib.r2x_binning_bytes(_C._Workspace.first(P, kind.seed)) + 64 * P)
    return out
