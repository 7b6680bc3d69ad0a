"""Inputs of the TV (prox, value, Chambolle-Pock step), volume-render and marching-cubes kernels at their launch limits
and past 2^31 elements, the windows the GPU tests compare against the float64 oracles, and the claim each case makes
about where it sits.

tests/ct_edge_cases.py covers these kernels' tile edges; the cases here sit on their grid limits (gridDim.y / .z =
65535, gridDim.x far past it), on flat indices whose 32-bit form would wrap, and on MC_MAX_SAMPLES = 2^31 - 1.  Every
limit is read from the CUDA sources by regular expression, so a retuned constant moves the cases with it and a renamed
one fails the suite.  Each case carries `claims`, expressions over those constants and over quantities of the case,
which tests/test_ct_limits_cpu.py evaluates without a GPU: a case cannot quietly stop sitting where its name says.
Each big case also states its peak device memory (`peak`, bytes), which tests/test_ct_limits_gpu.py compares with the
free memory before it runs.

A volume too large to copy to the host is compared in windows: a box of TV tiles, grown by the stencil's reach
(`halo`), goes through the float64 oracle, whose result on the box equals the full grid's (proved on small grids by
tests/test_ct_limits_cpu.py).
"""
from __future__ import annotations

import math
import os
import re
from dataclasses import dataclass, field

import numpy as np

import mesh_oracle as mo
from regime_cases import _find, _source

INT_MAX = 2**31 - 1
GiB = 2**30
HDR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "r2x.h")


def _constexpr(name: str, text: str, env: dict):
    """The value of `constexpr <type> ... NAME = <expr>`, <expr> over `env` with C literal suffixes dropped."""
    m = _find(rf"constexpr\s+(int|long long|unsigned|float)\s+[^;]*?\b{name}\s*=\s*([^,;]+)[,;]", text, name)
    expr = re.sub(r"(?<=[0-9.])(?:LL|f)\b", "", m.group(2))
    if m.group(1) != "float":
        return int(eval(expr.replace("/", "//"), {"__builtins__": {}}, dict(env)))
    return float(eval(expr, {"__builtins__": {}}, dict(env)))


def read_constants() -> dict:
    """The tiles, chunk sizes and launch limits of the TV, volume-render and marching-cubes kernels."""
    k: dict = {"R2X_VR_TILE": int(_find(r"#define R2X_VR_TILE (\d+)", open(HDR).read(), "R2X_VR_TILE").group(1))}
    names = {"r2x_tv.cu": ("TV_TX", "TV_TY", "TV_TZ", "TVV_THREADS", "TVV_MAX_BLOCKS", "TVV_PER_BLOCK"),
             "r2x_volrender.cu": ("VR_MAX_LUT", "VR_MAX_GRID", "VR_T_STOP"),
             "r2x_mesh.cu": ("MC_THREADS", "MC_WORDS", "MC_CLASSIFY_WORDS", "MC_MAX_SAMPLES")}
    for f, ns in names.items():
        src = _source(f)
        for name in ns:
            k[name] = _constexpr(name, src, k)
    return k


K = read_constants()


def tiles(n: int, t: int) -> int:
    return -(-n // t)


def tv_value_blocks(nvox: int) -> tuple[int, int]:
    """(blocks, chunk) of r2x_tv_value."""
    nb = min(max(tiles(nvox, K["TVV_PER_BLOCK"]), 1), K["TVV_MAX_BLOCKS"])
    return nb, tiles(nvox, nb)


@dataclass
class Case:
    name: str
    kind: str                 # "tv" (prox, value, CP step), "prox", "cp", "value", "vr", "mc", or "refuse_*"
    boundary: str             # the limit it lands on, in words
    claims: tuple             # expressions over K and the case's quantities that must hold
    shape: tuple = ()         # volume [nx, ny, nz]
    frames: int = 0           # vr: n_frames, H, W
    H: int = 0
    W: int = 0
    sites: tuple = ()         # tv: (label, flat voxel index) windows; vr: frames, rows or columns checked; mc: slabs
    extra: dict = field(default_factory=dict)
    peak: int = 0             # device bytes the GPU test needs at once
    niter: int = 3            # prox iterations


# ---- TV -----------------------------------------------------------------------------------------------------------

CP_PARAMS = (0.3, 0.4, 0.7)   # (tau, sigma, nu), as tests/test_cp_tv_gpu.py; p ~ N(0, 0.7) / nu around the bound 1 / nu
PROX_WEIGHT = 0.1


def _tv_peak(kind: str, nvox: int) -> int:
    # cp: x, xbar, g, p (3), x+, xbar+, p+ (3); prox: v, out, scratch (9); value: x and float64 slabs of the check
    floats = {"cp": 11, "prox": 11, "tv": 11, "value": 1}[kind]
    return 4 * floats * nvox + (2 * GiB if kind == "value" else GiB // 2)


def _tv_cases() -> list[Case]:
    TX, TY, TZ = K["TV_TX"], K["TV_TY"], K["TV_TZ"]
    out = []

    def add(name, kind, boundary, claims, shape, sites=(), niter=3):
        n = math.prod(shape)
        out.append(Case(name, kind, boundary, claims, shape, sites=sites, peak=_tv_peak(kind, n), niter=niter))

    # grid limits: gridDim.z = tiles along x, gridDim.y = tiles along y, both at 65535; gridDim.x far past it
    add("tv_nx_max", "tv", "TV grid: nx = TV_TX * 65535, gridDim.z == 65535",
        ("nx == TV_TX * 65535", "grid_z == 65535", "ny == 1", "nz == 1"), (TX * 65535, 1, 1))
    add("tv_ny_max", "tv", "TV grid: ny = TV_TY * 65535, gridDim.y == 65535",
        ("ny == TV_TY * 65535", "grid_y == 65535", "nx == 1", "nz == 1"), (1, TY * 65535, 1))
    add("tv_nz_long_line", "tv", "TV grid: one z line, gridDim.x three times 65535",
        ("grid_x > 3 * 65535", "nz % TV_TZ != 0", "nx == 1", "ny == 1"), (1, 1, 3 * 65535 * TZ + 7))
    add("tv_nz_long_box", "tv", "TV grid: gridDim.x past 65535 with partial tiles along x and y",
        ("grid_x > 65535", "nx % TV_TX != 0", "ny % TV_TY != 0", "nz % TV_TZ != 0", "grid_z == 2", "grid_y == 2"),
        (TX + 1, TY + 1, 65536 * TZ + 5),
        sites=(("first", 0), ("mid", 45 * (32 * 32768)), ("last", -1)))
    # the 1-line shapes of ct_edge_cases' prox cases, through the CP step as well
    for shape, cl in (((1, 1, 2 * TZ), ("nx == 1", "ny == 1", "nz == 2 * TV_TZ")),
                      ((2, 1, 1), ("nx == 2", "ny == 1", "nz == 1")),
                      ((1, 1, 1), ("nvox == 1",)),
                      ((1, 2 * TY + 1, 1), ("nx == 1", "ny == 2 * TV_TY + 1", "nz == 1"))):
        add("tv_line_" + "x".join(map(str, shape)), "tv", "TV: a single line or voxel", cl, shape)
    # index limits.  CP step: p's third plane (2 nvox + i) crosses 2^31 inside the grid, and the byte offset 4 i of
    # a volume passes 2^31 at i = 2^29
    add("cp_p_plane_past_2_31", "cp", "CP step: p+'s third plane 2 nvox + i crosses 2^31",
        ("2 * nvox < 2**31 < 3 * nvox", "0 < wrap_p2 < nvox", "2 * nvox + wrap_p2 == 2**31", "4 * 2**29 == 2**31",
         "2**29 < nvox", "nx % TV_TX != 0", "ny % TV_TY != 0", "nz % TV_TZ != 0"),
        (897, 801, 1001),
        sites=(("first", 0), ("bytes 4 i = 2^31", 2**29), ("2 nvox + i = 2^31", "wrap_p2"), ("last", -1)))
    # prox: its scratch holds three dual fields of 3 nvox floats; the third starts past 2^31, and plane 5 (the second
    # field's third component) crosses it
    add("prox_scratch_past_2_31", "prox", "TV prox: the third scratch field starts past 2^31",
        ("6 * nvox > 2**31", "5 * nvox < 2**31", "0 < wrap_s5 < nvox", "5 * nvox + wrap_s5 == 2**31",
         "9 * nvox < 2**32", "nx % TV_TX != 0", "ny % TV_TY != 0", "nz % TV_TZ != 0"),
        (711, 701, 723),
        sites=(("first", 0), ("5 nvox + i = 2^31", "wrap_s5"), ("last", -1)))
    # the value: more voxels than int32 holds, on 64-bit i, i / sx, i % nz
    add("value_past_2_31", "value", "TV value: nvox > 2^31",
        ("nvox > 2**31", "nb == TVV_MAX_BLOCKS", "nb * chunk >= nvox", "(nb - 1) * chunk < nvox",
         "chunk > 2**21"), (1291, 1291, 1291))
    return out


def _tv_refusals() -> list[Case]:
    TX, TY = K["TV_TX"], K["TV_TY"]
    out = [Case("refuse_tv_nx", "refuse_tv", "TV grid: one x tile too many", ("grid_z == 65536",), (TX * 65535 + 1, 1, 1)),
           Case("refuse_tv_ny", "refuse_tv", "TV grid: one y tile too many", ("grid_y == 65536",), (1, TY * 65535 + 1, 1))]
    for k in range(TX - 1):
        out.append(Case(f"refuse_tv_nx_int_max_{k}", "refuse_tv", "TV grid: nx within a tile of INT_MAX",
                        ("nx + TV_TX - 1 > INT_MAX", "grid_z > 65535"), (INT_MAX - k, 1, 1)))
    for k in range(TY - 1):
        out.append(Case(f"refuse_tv_ny_int_max_{k}", "refuse_tv", "TV grid: ny within a tile of INT_MAX",
                        ("ny + TV_TY - 1 > INT_MAX", "grid_y > 65535"), (1, INT_MAX - k, 1)))
    return out


# ---- volume rendering ---------------------------------------------------------------------------------------------

def _vr_peak(frames, H, W, shape) -> int:
    # the frames, one more frame for the single-camera calls, the volume
    return 16 * (frames + 1) * H * W + 4 * math.prod(shape) + GiB // 2


def stop_opacity(k_stop: int) -> float:
    """The float32 opacity t whose per-sample transmittance 1 - t (step = unit) drops T below 2^-16 half-way between
    samples k_stop - 1 and k_stop: (1 - t)^(k_stop - 1/2) = VR_T_STOP."""
    return float(np.float32(1.0 - K["VR_T_STOP"] ** (1.0 / (k_stop - 0.5))))


def _vr_cases() -> list[Case]:
    T, G = K["R2X_VR_TILE"], K["VR_MAX_GRID"]
    out = []
    n = G
    out.append(Case("vr_frames_max", "vr", "volume render: n_frames == VR_MAX_GRID (gridDim.z), tiny image",
                    ("frames == VR_MAX_GRID", "H % R2X_VR_TILE != 0", "W % R2X_VR_TILE != 0"), (9, 10, 11), n, 5, 7,
                    sites=(0, 1, n // 2, n - 2, n - 1), peak=_vr_peak(n, 5, 7, (9, 10, 11))))
    H = T * G
    rows = (0, T - 1, T, H // 2, H - T - 1, H - T, H - 1)
    out.append(Case("vr_rows_max", "vr", "volume render: H = R2X_VR_TILE * VR_MAX_GRID, gridDim.y == VR_MAX_GRID",
                    ("tiles_y == VR_MAX_GRID", "W < R2X_VR_TILE"), (12, 11, 10), 1, H, 3, sites=rows,
                    extra={"axis": "rows"}, peak=_vr_peak(1, H, 3, (12, 11, 10))))
    out.append(Case("vr_cols_max", "vr", "volume render: W = R2X_VR_TILE * VR_MAX_GRID, gridDim.x == VR_MAX_GRID",
                    ("tiles_x == VR_MAX_GRID", "H < R2X_VR_TILE"), (12, 11, 10), 1, 3, H, sites=rows,
                    extra={"axis": "cols"}, peak=_vr_peak(1, 3, H, (12, 11, 10))))
    n, hw = 2100, 512
    fb, ff = 2**31 // (16 * hw * hw), 2**31 // (4 * hw * hw)
    out.append(Case("vr_output_past_2_31", "vr", "volume render: an orbit whose output passes 2^31 floats",
                    ("4 * frames * H * W > 2**31", "frames <= VR_MAX_GRID", "16 * H * W * f_bytes == 2**31",
                     "4 * H * W * f_floats == 2**31", "f_floats < frames - 1"), (16, 16, 16), n, hw, hw,
                    sites=(0, fb - 1, fb, ff - 1, ff, n - 1), extra={"f_bytes": fb, "f_floats": ff},
                    peak=16 * n * hw * hw + 64 * hw * hw + GiB // 2))
    # long rays: parallel along x through voxel centres, (nx - 1) / step = 10^5 - 1/2 (clear of the floor's edges in
    # float32): 10^5 samples, low opacity
    nx, samples = 65, 10**5
    step = float(np.float32((nx - 1) / (samples - 0.5)))
    out.append(Case("vr_long_rays", "vr", "volume render: composite rays of 10^5 samples that never stop",
                    ("n_samples == 10**5", "(1 - vmax) ** (n_samples * expo) > 16 * VR_T_STOP"), (nx, 6, 7), 1, 6, 7,
                    extra={"step": step, "unit": 1.0, "vmin": 0.02, "vmax": 0.06,
                           "samples": samples}, peak=GiB // 2))
    # a stop on a known sample: a constant volume, step = unit = 1, (1 - t)^k crosses 2^-16 half-way to k_stop
    ks = 20
    out.append(Case("vr_stop_known_sample", "vr", "volume render: T < 2^-16 first after sample k_stop",
                    ("(1 - t_stop) ** (k_stop - 1) >= 1.3 * VR_T_STOP", "(1 - t_stop) ** k_stop < VR_T_STOP / 1.3",
                     "k_stop + 10 < n_samples"), (41, 4, 5), 1, 4, 5,
                    extra={"k_stop": ks, "t_stop": stop_opacity(ks), "step": 1.0, "unit": 1.0, "samples": 41},
                    peak=GiB // 2))
    return out


def _vr_refusals() -> list[Case]:
    T, G = K["R2X_VR_TILE"], K["VR_MAX_GRID"]
    out = [Case("refuse_vr_frames", "refuse_vr", "one frame too many", ("frames == VR_MAX_GRID + 1",), frames=G + 1,
                H=1, W=1),
           Case("refuse_vr_rows", "refuse_vr", "one row tile too many", ("tiles_y == VR_MAX_GRID + 1",), frames=1,
                H=T * G + 1, W=1),
           Case("refuse_vr_cols", "refuse_vr", "one column tile too many", ("tiles_x == VR_MAX_GRID + 1",), frames=1,
                H=1, W=T * G + 1)]
    for k in (0, 1, T - 2):
        out.append(Case(f"refuse_vr_rows_int_max_{k}", "refuse_vr", "H within a tile of INT_MAX",
                        ("H + R2X_VR_TILE - 1 > INT_MAX",), frames=1, H=INT_MAX - k, W=1))
        out.append(Case(f"refuse_vr_cols_int_max_{k}", "refuse_vr", "W within a tile of INT_MAX",
                        ("W + R2X_VR_TILE - 1 > INT_MAX",), frames=1, H=1, W=INT_MAX - k))
    return out


# ---- marching cubes -----------------------------------------------------------------------------------------------

def _mc_peak(n: int) -> int:
    # the volume, the scratch (5 words per 32 samples and the scan state), the mesh and the counting temporaries
    return 4 * n + 5 * 4 * tiles(n, 32) + 3 * GiB


def _mc_cases() -> list[Case]:
    M = K["MC_MAX_SAMPLES"]
    out = []
    s = 1290
    plane = s * s
    p30, p31 = 2**30 // plane, (2**31 - 2**20) // plane
    out.append(Case("mc_near_max", "mc", "marching cubes: 1290^3 samples, just under MC_MAX_SAMPLES, 8 in the last word",
                    ("n <= MC_MAX_SAMPLES", "(nx + 1) * ny * nz > MC_MAX_SAMPLES", "n % 32 == 8", "n > 2**30",
                     "p30 * ny * nz <= 2**30 < (p30 + 1) * ny * nz",
                     "p31 * ny * nz <= 2**31 - 2**20 < (p31 + 1) * ny * nz"),
                    (s, s, s), sites=((0, 3), (p30 - 1, p30 + 2), (p31 - 1, p31 + 1), (s - 3, s)),
                    extra={"p30": p30, "p31": p31}, peak=_mc_peak(s ** 3)))
    for a in range(3):
        shape = tuple(M if b == a else 1 for b in range(3))
        out.append(Case(f"mc_line_{'xyz'[a]}", "mc", "marching cubes: exactly MC_MAX_SAMPLES samples on one axis",
                        ("n == MC_MAX_SAMPLES", "32 * words == 2**31", "n % 32 == 31"), shape, peak=_mc_peak(M)))
    return out


def _mc_refusals() -> list[Case]:
    return [Case(f"refuse_mc_{'_'.join(map(str, s))}", "refuse_mc", "marching cubes: one sample past the maximum",
                 ("n == MC_MAX_SAMPLES + 1",), s)
            for s in ((65536, 32768, 1), (1, 65536, 32768), (32768, 1, 65536))]


TV_CASES = {c.name: c for c in _tv_cases()}
VR_CASES = {c.name: c for c in _vr_cases()}
MC_CASES = {c.name: c for c in _mc_cases()}
REFUSALS = {c.name: c for c in _tv_refusals() + _vr_refusals() + _mc_refusals()}
ALL_CASES = {**TV_CASES, **VR_CASES, **MC_CASES, **REFUSALS}
assert len(ALL_CASES) == len(TV_CASES) + len(VR_CASES) + len(MC_CASES) + len(REFUSALS), "case names must be unique"


# ---- what a case claims -------------------------------------------------------------------------------------------

class _Quantities(dict):
    """The quantities a claim may name, computed on first use."""

    def __init__(self, case: Case):
        super().__init__(K)
        self.case = case
        self.update(INT_MAX=INT_MAX, **case.extra)

    def __missing__(self, name):
        self[name] = value = getattr(self, "_" + name)()
        return value

    def _nx(self): return int(self.case.shape[0])
    def _ny(self): return int(self.case.shape[1])
    def _nz(self): return int(self.case.shape[2])
    def _nvox(self): return self["nx"] * self["ny"] * self["nz"]
    def _n(self): return self["nvox"]
    def _words(self): return tiles(self["n"], 32)
    def _grid_x(self): return tiles(self["nz"], K["TV_TZ"])
    def _grid_y(self): return tiles(self["ny"], K["TV_TY"])
    def _grid_z(self): return tiles(self["nx"], K["TV_TX"])
    def _nb(self): return tv_value_blocks(self["nvox"])[0]
    def _chunk(self): return tv_value_blocks(self["nvox"])[1]
    def _wrap_p2(self): return 2**31 - 2 * self["nvox"]
    def _wrap_s5(self): return 2**31 - 5 * self["nvox"]
    def _frames(self): return self.case.frames
    def _H(self): return self.case.H
    def _W(self): return self.case.W
    def _tiles_x(self): return tiles(self["W"], K["R2X_VR_TILE"])
    def _tiles_y(self): return tiles(self["H"], K["R2X_VR_TILE"])
    def _expo(self): return float(self.case.extra["step"]) / float(self.case.extra["unit"])

    def _n_samples(self):
        """The oracle's sample count of the case's rays (all equal: parallel rays along x through voxel centres)."""
        import volume_render_oracle as vo

        cam = vr_camera(self.case)
        o, d, s0, s1, meets = vo.ray_setup(cam.record(), self["H"], self["W"], True, self.case.shape)
        n = vo.sample_counts(s0, s1, meets, self.case.extra["step"])
        assert meets.all() and (n == n[0]).all(), np.unique(n)
        return int(n[0])


def claim_failures(case: Case) -> list[str]:
    """The claims of `case` that do not hold (empty when it sits where it says)."""
    q = _Quantities(case)
    return [c for c in case.claims if not eval(c, {"__builtins__": {}, "abs": abs}, q)]


# ---- TV windows ---------------------------------------------------------------------------------------------------

def site_index(case: Case, site) -> int:
    """A site's flat voxel index: a number (negative from the end) or the name of a quantity."""
    q = _Quantities(case)
    i = q[site] if isinstance(site, str) else int(site)
    return i + q["nvox"] if i < 0 else i


def tile_window(shape, flat: int) -> tuple:
    """((x0, x1), (y0, y1), (z0, z1)): the box of whole TV tiles (clipped to the grid) holding voxels flat - 1 and
    flat, so that a window around a 32-bit wrap holds voxels on both sides of it."""
    nx, ny, nz = shape
    pts = [max(flat - 1, 0), flat]
    ijk = [(f // (ny * nz), (f // nz) % ny, f % nz) for f in pts]
    box = []
    for a, (n, t) in enumerate(zip(shape, (K["TV_TX"], K["TV_TY"], K["TV_TZ"]))):
        lo, hi = min(p[a] for p in ijk), max(p[a] for p in ijk)
        box.append((lo // t * t, min((hi // t + 1) * t, n)))
    return tuple(box)


def grow(box, shape, halo: int) -> tuple:
    return tuple((max(lo - halo, 0), min(hi + halo, n)) for (lo, hi), n in zip(box, shape))


def inner(box, outer) -> tuple:
    """Slices of `box` inside the array of the box `outer`."""
    return tuple(slice(lo - olo, hi - olo) for (lo, hi), (olo, _) in zip(box, outer))


def slices(box) -> tuple:
    return tuple(slice(lo, hi) for lo, hi in box)


# the stencil's reach per axis: one CP step reads xbar at i +- 1 (p+ at i - 1 needs xbar at i - 1 and i); niter prox
# iterations reach niter voxels (the first, from p = 0, reads v at i and i + e_a only).  tests/test_ct_limits_cpu.py
# shows both are enough and one voxel less is not
CP_HALO = 1


def prox_halo(niter: int) -> int:
    return niter


# ---- volume-render cameras ----------------------------------------------------------------------------------------

def vr_camera(case: Case):
    """The case's base camera: a parallel view along +x through voxel centres for the long-ray and stop cases, the
    default perspective view otherwise."""
    from r2_gaussian_b200 import volume_render as vr

    import volume_render_oracle as vo

    if "step" in case.extra:
        cam, lat, _ = vo.axis_view(case.shape, 0, 1)
        assert (lat >= 0).all()
        return cam
    return vr.default_camera(case.shape, case.W, case.H, view_angle=40.0)


def vr_volume(case: Case):
    """float32 volume of a render case: smooth and positive, in [vmin, vmax] for the long rays, t_stop everywhere for
    the stop case."""
    n = case.shape
    if "t_stop" in case.extra:
        return np.full(n, case.extra["t_stop"], np.float32)
    g = [np.linspace(-1.0, 1.0, m) for m in n]
    X, Y, Z = np.meshgrid(*g, indexing="ij")
    s = 0.5 + 0.5 * np.sin(3.0 * X + 1.0) * np.cos(2.0 * Y - 0.5) * np.cos(1.5 * Z)
    lo, hi = case.extra.get("vmin", 0.0), case.extra.get("vmax", 0.9)
    return (lo + (hi - lo) * s).astype(np.float32)


# ---- marching-cubes slabs ----------------------------------------------------------------------------------------

def plane_counts(vol, level):
    """(vertices owned by each x-plane, triangles of the cubes whose lower corner is in each x-plane), numpy."""
    ins = np.asarray(vol) > np.float32(level)
    ntri = mo.table()[0]
    nv = np.zeros(ins.shape[0], np.int64)
    nv[:-1] += (ins[1:] != ins[:-1]).sum((1, 2))
    nv += (ins[:, 1:] != ins[:, :-1]).sum((1, 2)) + (ins[:, :, 1:] != ins[:, :, :-1]).sum((1, 2))
    nt = np.zeros(ins.shape[0], np.int64)
    if min(ins.shape) > 1:
        case = sum(ins[dx:ins.shape[0] - 1 + dx, dy:ins.shape[1] - 1 + dy, dz:ins.shape[2] - 1 + dz].astype(np.int64)
                   << b for b, (dx, dy, dz) in enumerate(mo.CORNERS))
        nt[:-1] = ntri[case].sum((1, 2))
    return nv, nt


def slab_mesh(slab, level, a, b):
    """(vertices owned by x-planes [a, b), triangles of the cubes with lower corner in them as [T, 3, 3] coordinates)
    from mesh_oracle on `slab` alone: planes [a, b] of the grid, or [a, b) when b is its last."""
    verts, faces = mo.marching_cubes(slab, level, x_offset=a)
    nv, _ = plane_counts(slab, level)
    return verts[:int(nv[:b - a].sum())], verts[faces]
