"""Inputs of the training-step kernels that sit on their tilings and launch limits, the float64 (or exact float32)
statement each is judged against, and the claim each case makes about where it sits.

The kernels are those of every training iteration (r2x_train.cu: the L1 + D-SSIM image loss and its gradient, single
and batched, the 3-D TV loss, fused Adam, the densification statistics), of each densification step (r2x_compact.cu:
r2x_mask_select, r2x_gather_rows) and of each scene's initialisation (r2x_knn.cu: the 3-NN mean distance).  They tile
images, volumes and parameter tensors with fixed CTA shapes, reduce per-CTA partials with one fixed-size block, cap
their grids at a multiple of the SM count and run grid-stride loops past it, and split parameter lists into fixed-size
launches.  Index arithmetic goes wrong on either side of such a limit and at size 1, so each case lands on a stated side
of one.  Every limit is read from the CUDA sources by regular expression, as ct_edge_cases.read_constants does: a
retuned constant moves the cases with it and a renamed one fails the suite.  Each case carries `claims`, expressions
over those constants and the case's quantities, evaluated by tests/test_train_edges_cpu.py for an H100 SXM (132 SMs)
and re-evaluated by tests/test_train_edges_gpu.py with the SM count of the device it runs on.

The statements:
* image loss: the reference's SSIM (loss_utils.py:75-104) in float64 with the kernel's own float32 taps, its gradient
  by autograd, and per pixel an error bound of the kernel's float32 operation sequence (`ssim_f64`);
* TV: the float64 value, and the gradient exactly: float32(sign sum) * float32(1 / count) (`tv_grad_exact`);
* Adam: one step of torch.optim.Adam in float64 from the same float32 state, with per-element bounds derived from the
  kernel's operation sequence (`adam_f64`);
* densification statistics: the numpy float32 statement, bit for bit (`densify_f32`);
* compaction and kNN: torch indexing and the brute-force oracle, bit for bit.
"""
from __future__ import annotations

import math
import os
import re
from dataclasses import dataclass, field

import numpy as np

from ct_edge_cases import _constexpr
from regime_cases import _find, _source

INCLUDE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "r2x.h")
H100_SMS = 132          # SMs of an H100 SXM: the device the SM-dependent claims are stated for
U = 2.0 ** -24          # float32 unit roundoff
TINY = 2.0 ** -149      # float32's least subnormal: the absolute rounding of a result in the subnormal range


def _launch_bounds(kernel: str, text: str) -> int:
    return int(_find(rf"__launch_bounds__\(([0-9]+)\) {kernel}\(", text, f"{kernel}'s threads").group(1))


def _grid_cap(text: str, what: str) -> int:
    """The `k` of `if (nb > sms * k) nb = sms * k;`."""
    m = _find(r"if \(nb > sms \* ([0-9]+)\) nb = sms \* ([0-9]+);", text, what)
    assert m.group(1) == m.group(2), what
    return int(m.group(1))


def read_constants() -> dict:
    """The tile shapes, reduction blocks, grid caps and launch splits of the training-step kernels, as the sources state
    them."""
    tr, co, bi, kn = (_source(f) for f in ("r2x_train.cu", "r2x_compact.cu", "r2x_binning.cu", "r2x_knn.cu"))
    with open(INCLUDE) as f:
        hdr = f.read()
    k: dict = {}
    for name in ("LT", "LH", "LE", "IMAGE_LOSS_MAX_H"):
        k[name] = _constexpr(name, tr, k)
    k["SSIM_REDUCE_THREADS"] = _launch_bounds("ssim_reduce_kernel", tr)
    k["TV_REDUCE_THREADS"] = _launch_bounds("tv3d_reduce_kernel", tr)
    k["TV_THREADS"] = _launch_bounds("tv3d_kernel", tr)
    k["ADAM_THREADS"] = _launch_bounds("adam_kernel", tr)
    k["DENSIFY_THREADS"] = _launch_bounds("densify_stats_kernel", tr)
    # both reductions stride their partials by their block size
    strides = re.findall(r"i < nblk; i \+= ([0-9]+)\)", tr)
    assert len(strides) == 2 and {int(s) for s in strides} == {k["SSIM_REDUCE_THREADS"]} == {k["TV_REDUCE_THREADS"]}
    k["ADAM_GRID_PER_SM"] = _grid_cap(tr[tr.index("int launch_adam("):], "launch_adam's grid cap")
    k["VIEWS_MAX_N"] = int(_find(r"N > ([0-9]+)\) return fail_msg\(R2X_ERR_INVALID, \"r2x_image_loss_views: bad N",
                                 tr, "r2x_image_loss_views' bound on N").group(1))
    k["GATHER_THREADS"] = _launch_bounds("gather_rows_kernel", co)
    k["GATHER_GRID_PER_SM"] = _grid_cap(co, "launch_gather_rows' grid cap")
    k["SCAN_THREADS"] = _constexpr("SCAN_THREADS", bi, k)
    k["SCAN_ITEMS"] = _constexpr("SCAN_ITEMS", bi, k)
    k["SCAN_TILE"] = k["SCAN_THREADS"] * k["SCAN_ITEMS"]
    for name in ("R2X_ADAM_MAX_GROUPS", "R2X_GATHER_MAX_TENSORS"):
        k[name] = int(_find(rf"#define {name} ([0-9]+)", hdr, name).group(1))
    k["KNN_MAX_G"] = _constexpr("KNN_MAX_G", kn, k)
    _find(r"while \(\(long long\)g \* g \* g \* 2 < \(long long\)P && g < KNN_MAX_G\) \+\+g;", kn,
          "knn_grid's rule: the least g with 2 g^3 >= P, at most KNN_MAX_G")
    return k


K = read_constants()


def ssim_taps() -> np.ndarray:
    """The 11 float32 taps of make_window() in r2x_train.cu (hex float literals)."""
    body = _find(r"static const float g\[11\] = \{([^}]*)\}", _source("r2x_train.cu"), "the SSIM taps").group(1)
    lits = re.findall(r"(0x[0-9a-fA-F.]+p-?[0-9]+)f", body)
    assert len(lits) == 11, lits
    return np.array([float.fromhex(t) for t in lits], np.float32)


def knn_grid(P: int) -> int:
    """Cells per axis of r2x_knn3_mean_dist2: the least g >= 1 with 2 g^3 >= P, at most KNN_MAX_G."""
    g = 1
    while g * g * g * 2 < P and g < K["KNN_MAX_G"]:
        g += 1
    return g


def cdiv(a: int, b: int) -> int:
    return -(-a // b)


# ---- the cases ---------------------------------------------------------------------------------------------------------

@dataclass
class Case:
    name: str
    kind: str            # image, image_views, tv, adam, fused_adam, densify, mask, gather, knn
    boundary: str        # the limit it lands on, in words
    claims: tuple        # expressions over K and the case's quantities that must hold
    q: dict = field(default_factory=dict)   # the case's own quantities (shapes, sizes)
    content: str = "random"
    seed: int = 0


IMAGE_SIDES = (1, 2, 5, 6, 11, 15, 16, 17, 26, 27, 31, 32, 33)   # below the window, at the halo LE and at the tile


def _image_cases() -> list[Case]:
    LT, LE, R = K["LT"], K["LE"], K["SSIM_REDUCE_THREADS"]
    assert IMAGE_SIDES == (1, 2, 5, 6, 11, 15, 16, 17, LE, LE + 1, 2 * LT - 1, 2 * LT, 2 * LT + 1)
    out = []
    n = len(IMAGE_SIDES)
    for i, H in enumerate(IMAGE_SIDES):
        for W in sorted({H, IMAGE_SIDES[(i + 4) % n]}):
            out.append(Case(f"img_{H}x{W}", "image", "11-tap window, halo LE and tile LT edges",
                            (f"H == {H}", f"W == {W}", "ctas <= SSIM_REDUCE_THREADS"), dict(H=H, W=W), seed=H * 100 + W))
    # grids of exactly SSIM_REDUCE_THREADS CTAs and one more, flat and tall, with a ragged last tile
    for ctas, (a, b), rag in ((R, (2, R // 2), 5), (R + 1, (5, (R + 1) // 5), 7)):
        for layout, (ty, tx) in (("flat", (a, b)), ("tall", (b, a))):
            H, W = ty * LT - (rag if layout == "tall" else 0), tx * LT - (rag if layout == "flat" else 0)
            claim = "ctas == SSIM_REDUCE_THREADS" + ("" if ctas == R else " + 1")
            out.append(Case(f"img_{layout}_{ctas}ctas", "image", f"{ctas} CTAs ({layout}): the reduction's "
                            f"{'single' if ctas == R else 'second'} pass", (claim, "H % LT or W % LT"),
                            dict(H=H, W=W), seed=ctas + len(layout)))
    out.append(Case("img_560x560", "image", "the real-scan detector: 35^2 CTAs, past one reduction pass",
                    ("ctas > SSIM_REDUCE_THREADS", "ctas == 35 ** 2"), dict(H=560, W=560), content="proj", seed=560))
    out.append(Case("img_2048x2048", "image", "16 384 CTAs: 16 reduction passes",
                    ("ctas == 16 * SSIM_REDUCE_THREADS",), dict(H=2048, W=2048), content="proj", seed=2048))
    out.append(Case("img_max_H", "image", "H = IMAGE_LOSS_MAX_H: grid.y = 65535, the launch limit",
                    ("H == IMAGE_LOSS_MAX_H", "tiles_y == 65535"), dict(H=K["IMAGE_LOSS_MAX_H"], W=1), seed=7))
    # contents: the exact and the cancelling cases
    for content, shapes in (("identical", ((1, 1), (17, 33), (560, 560))), ("constant", ((6, 5), (33, 17))),
                            ("zeros", ((1, 2), (27, 26))), ("scaled50", ((31, 32), (560, 560)))):
        for H, W in shapes:
            out.append(Case(f"img_{content}_{H}x{W}", "image", f"{content} images", (f"H == {H}", f"W == {W}"),
                            dict(H=H, W=W), content=content, seed=H + W + len(content)))
    return out


def _image_views_cases() -> list[Case]:
    out = [Case(f"views_{N}_{H}x{W}", "image_views", "N ragged images, each against float64 on its own",
                (f"N == {N}", "N <= VIEWS_MAX_N"), dict(N=N, H=H, W=W), seed=N)
           for N, H, W in ((1, 17, 33), (2, 31, 26), (7, 27, 15), (7, 560, 35))]
    out.append(Case("views_max_4x4", "image_views", "N = VIEWS_MAX_N views of 4 x 4 (grid.z at its limit)",
                    ("N == VIEWS_MAX_N", "N == 65535"), dict(N=K["VIEWS_MAX_N"], H=4, W=4), seed=65535))
    return out


def _tv_cases() -> list[Case]:
    T, R = K["TV_THREADS"], K["TV_REDUCE_THREADS"]
    shapes = [((1, 5, 6), "nx == 1"), ((5, 1, 6), "ny == 1"), ((5, 6, 1), "nz == 1"), ((1, 1, 9), "nx == ny == 1"),
              ((1, 1, 1), "n == 1"), ((3, 5, 17), "n == TV_THREADS - 1"), ((4, 8, 8), "n == TV_THREADS"),
              ((1, 1, 257), "n == TV_THREADS + 1"), ((64, 64, 64), "nblk == TV_REDUCE_THREADS"),
              ((65, 64, 64), "nblk > TV_REDUCE_THREADS"), ((256, 256, 256), "nblk == 64 * TV_REDUCE_THREADS")]
    assert T == 256 and R == 1024, (T, R)
    return [Case("tv_{}x{}x{}".format(*s), "tv", c, (c,), dict(shape=s), seed=i) for i, (s, c) in enumerate(shapes)]


ADAM_GRADS = ("normal", "zeros", "subnormal", "huge")
ADAM_STEPS = (1, 2, 10, 10000)


def _adam_cases() -> list[Case]:
    cap = K["ADAM_THREADS"] * K["ADAM_GRID_PER_SM"] * H100_SMS
    out = []
    for grad in ADAM_GRADS:
        for step in ADAM_STEPS:
            out.append(Case(f"adam_mixed_{grad}_s{step}", "adam", "numel 0, 1, 255, 256, 257 in one launch",
                            ("numels == (0, 1, ADAM_THREADS - 1, ADAM_THREADS, ADAM_THREADS + 1)",),
                            dict(numels=(0, 1, 255, 256, 257), step=step), content=grad, seed=step))
    out.append(Case("adam_past_cap", "adam", "one group of ADAM_THREADS * ADAM_GRID_PER_SM * SMs + 1: the grid-stride "
                    "loop's second pass", ("maxn > ADAM_THREADS * grid", "grid == SMS * ADAM_GRID_PER_SM"),
                    dict(numels=(cap + 1,), step=3), content="huge", seed=11))
    out.append(Case("adam_4M", "adam", "4M elements, past the grid cap",
                    ("maxn > 7 * ADAM_THREADS * grid", "grid == SMS * ADAM_GRID_PER_SM"),
                    dict(numels=(4 << 20,), step=7), content="normal", seed=12))
    out.append(Case("adam_8_groups", "adam", "R2X_ADAM_MAX_GROUPS groups in one call",
                    ("len(numels) == R2X_ADAM_MAX_GROUPS",), dict(numels=(1, 3, 300, 4000, 77, 256, 1025, 9), step=5),
                    content="normal", seed=13))
    for n in (8, 9, 17):
        out.append(Case(f"fused_adam_{n}", "fused_adam", f"{n} parameters through FusedAdam",
                        (f"launches == {cdiv(n, 8)}", "nparams == len(numels)"),
                        dict(numels=tuple(37 * (i + 1) + i % 3 for i in range(n))), seed=20 + n))
    return out


def _densify_cases() -> list[Case]:
    T = K["DENSIFY_THREADS"]
    return [Case(f"densify_P{P}_N{N}", "densify", f"P = {Ps}, N = {N}", (f"P == {Ps}",), dict(P=P, N=N), seed=P + N)
            for P, Ps in ((T - 1, "DENSIFY_THREADS - 1"), (T, "DENSIFY_THREADS"), (T + 1, "DENSIFY_THREADS + 1"),
                          (1 << 20, "1 << 20"))
            for N in (1, 3, 16)]


MASKS = ("all", "none", "last", "alternating", "bytes")


def _mask_cases() -> list[Case]:
    T = K["SCAN_TILE"]
    sizes = ((1, "1"), (T - 1, "SCAN_TILE - 1"), (T, "SCAN_TILE"), (T + 1, "SCAN_TILE + 1"), (4 * T + 1, "4 * SCAN_TILE + 1"),
             ((1 << 20) + 1, "(1 << 20) + 1"), ((1 << 24) + 1, "(1 << 24) + 1"))
    return [Case(f"mask_{n}_{m}", "mask", f"n = {ns} ({m})", (f"n == {ns}",), dict(n=n), content=m, seed=n % 1000)
            for n, ns in sizes for m in MASKS]


def _gather_cases() -> list[Case]:
    M = K["R2X_GATHER_MAX_TENSORS"]
    widths = tuple((1, 3, 4, 7)[i % 4] for i in range(M))
    return [Case("gather_16", "gather", "R2X_GATHER_MAX_TENSORS tensors, n0 = 0 and NULL src1 among them",
                 ("ntensors == R2X_GATHER_MAX_TENSORS", "nb < cap"), dict(widths=widths, nsel=1000), seed=1),
            Case("gather_identity", "gather", "a NULL select (the identity)", ("ntensors == R2X_GATHER_MAX_TENSORS",),
                 dict(widths=widths, nsel=None), seed=2),
            Case("gather_past_cap", "gather", "nsel * width past SMS * GATHER_GRID_PER_SM * GATHER_THREADS",
                 ("nb > 2 * cap",), dict(widths=widths, nsel=200003), seed=3),
            Case("gather_17", "gather", "17 tensors through compact.gather_rows: two launches",
                 ("launches == 2",), dict(widths=widths + (5,), nsel=777), seed=4)]


def _knn_cases() -> list[Case]:
    G = K["KNN_MAX_G"]
    out = []
    for g in (1, 2, 3, 4):
        out.append(Case(f"knn_{2 * g ** 3}", "knn", f"P = 2 g^3 with g = {g}", (f"G == {g}",), dict(P=2 * g ** 3),
                        seed=g))
        out.append(Case(f"knn_{2 * g ** 3 + 1}", "knn", f"P = 2 g^3 + 1 with g = {g}: the grid grows",
                        (f"G == {g + 1}",), dict(P=2 * g ** 3 + 1), seed=10 + g))
    out.append(Case("knn_elongated", "knn", "a 4 x 1 x 0.25 box: three different cell counts",
                    ("len({nx, ny, nz}) == 3", "nx == G"), dict(P=20000), content="elongated", seed=21))
    out.append(Case("knn_lattice", "knn", "a 9^3 lattice of spacing h: every point on cell faces, many ties",
                    ("G == 8", "P == 9 ** 3"), dict(P=729), content="lattice", seed=22))
    out.append(Case("knn_at_cap", "knn", "P = 2 KNN_MAX_G^3: the last grid the rule picks",
                    ("G == KNN_MAX_G", "P == 2 * KNN_MAX_G ** 3"), dict(P=2 * G ** 3), content="faces", seed=23))
    out.append(Case("knn_past_cap", "knn", "P = 2 KNN_MAX_G^3 + 1: the grid stops growing",
                    ("G == KNN_MAX_G", "P > 2 * KNN_MAX_G ** 3"), dict(P=2 * G ** 3 + 1), content="faces", seed=24))
    out.append(Case("knn_5M", "knn", "5M points at the cell cap", ("G == KNN_MAX_G", "P > 2 * KNN_MAX_G ** 3"),
                    dict(P=5_000_000), content="faces", seed=25))
    return out


IMAGE_CASES = {c.name: c for c in _image_cases()}
VIEWS_CASES = {c.name: c for c in _image_views_cases()}
TV_CASES = {c.name: c for c in _tv_cases()}
ADAM_CASES = {c.name: c for c in _adam_cases()}
DENSIFY_CASES = {c.name: c for c in _densify_cases()}
MASK_CASES = {c.name: c for c in _mask_cases()}
GATHER_CASES = {c.name: c for c in _gather_cases()}
KNN_CASES = {c.name: c for c in _knn_cases()}
_TABLES = (IMAGE_CASES, VIEWS_CASES, TV_CASES, ADAM_CASES, DENSIFY_CASES, MASK_CASES, GATHER_CASES, KNN_CASES)
ALL_CASES = {n: c for t in _TABLES for n, c in t.items()}
assert len(ALL_CASES) == sum(len(t) for t in _TABLES), "case names must be unique"
KNN_BRUTE_MAX = 50_000    # clouds up to this size are checked against the whole brute-force oracle
KNN_QUERIES = 4096        # above it, the points checked with orc_knn3_mean_dist2_at


# ---- what a case claims ------------------------------------------------------------------------------------------------

class _Quantities(dict):
    """The quantities a claim may name: the constants, SMS, the case's own sizes and what follows from them."""

    def __init__(self, case: Case, sms: int):
        super().__init__(K)
        self.update(case.q, SMS=sms, len=len)
        self.case = case

    def __missing__(self, name):
        self[name] = value = getattr(self, "_" + name)()
        return value

    def _tiles_x(self): return cdiv(self["W"], K["LT"])
    def _tiles_y(self): return cdiv(self["H"], K["LT"])
    def _ctas(self): return self["tiles_x"] * self["tiles_y"]
    def _nx(self): return self["shape"][0] if "shape" in self else knn_cells(self.case)[0]
    def _ny(self): return self["shape"][1] if "shape" in self else knn_cells(self.case)[1]
    def _nz(self): return self["shape"][2] if "shape" in self else knn_cells(self.case)[2]
    def _n(self): return self["nx"] * self["ny"] * self["nz"]
    def _nblk(self): return cdiv(self["n"], K["TV_THREADS"])
    def _maxn(self): return max(self["numels"])
    def _grid(self): return min(cdiv(self["maxn"], K["ADAM_THREADS"]), self["SMS"] * K["ADAM_GRID_PER_SM"])
    def _nparams(self): return len(self["numels"])
    def _launches(self):
        if self.case.kind == "fused_adam":
            return cdiv(self["nparams"], K["R2X_ADAM_MAX_GROUPS"])
        return cdiv(self["ntensors"], K["R2X_GATHER_MAX_TENSORS"])
    def _ntensors(self): return len(self["widths"])
    def _nb(self):
        rows = self["nsel"] if self["nsel"] is not None else gather_rows_n0(self.case)[1]
        return cdiv(rows * max(self["widths"]), K["GATHER_THREADS"])
    def _cap(self): return self["SMS"] * K["GATHER_GRID_PER_SM"]
    def _G(self): return knn_grid(self["P"])


def claim_failures(case: Case, sms: int = H100_SMS) -> list[str]:
    """The claims of `case` that do not hold on a device of `sms` SMs (empty when it sits where it says)."""
    q = _Quantities(case, sms)
    return [c for c in case.claims if not eval(c, {"__builtins__": {}}, q)]


# ---- inputs ------------------------------------------------------------------------------------------------------------

def image_pair(H: int, W: int, content: str, seed: int, n: int | None = None):
    """(x, y) float32 [H, W] (or [n, H, W]): a smooth blob plus noise against a dimmer one ("random"), a projection-
    like pair ("proj"), the same image twice ("identical"), two constants ("constant": sigma = 0), zeros, or
    projections scaled to ~50 ("scaled50": E[x^2] - mu^2 cancels)."""
    rng = np.random.RandomState(seed)
    shape = (H, W) if n is None else (n, H, W)
    yy, xx = np.meshgrid(np.linspace(-1, 1, H), np.linspace(-1, 1, W), indexing="ij")
    base = np.exp(-(xx ** 2 + yy ** 2) * 3) * 2.0
    if content == "constant":
        return np.full(shape, 0.7, np.float32), np.full(shape, 0.3, np.float32)
    if content == "zeros":
        return np.zeros(shape, np.float32), np.zeros(shape, np.float32)
    scale = {"random": 1.0, "proj": 1.0, "identical": 1.0, "scaled50": 25.0}[content]
    a = scale * (base + (0.15 if content != "proj" else 0.05) * rng.uniform(0, 1, shape))
    b = scale * (base * 0.9 + 0.1 * rng.uniform(0, 1, shape))
    a, b = a.astype(np.float32), b.astype(np.float32)
    return (a, a.copy()) if content == "identical" else (a, b)


def tv_volume(case: Case) -> np.ndarray:
    """Uniform values with exact plateaus: a third of the voxels are 0 and a sixth are 0.5, so many differences are
    exactly 0 (sign(0) = 0)."""
    rng = np.random.RandomState(case.seed)
    v = rng.uniform(-0.3, 1.0, case.q["shape"]).astype(np.float32)
    r = rng.uniform(0, 1, case.q["shape"])
    v[r < 1 / 3] = 0.0
    v[(r >= 1 / 3) & (r < 0.5)] = 0.5
    return v


def adam_state(numel: int, grad: str, rng: np.random.RandomState, step: int):
    """(p, m, v, g) float32 for one group: a state as `step - 1` steps leave it (zeros at step 1) and a gradient of the
    given kind: normal with exact zeros, all zeros, |g| ~ 1e-20 (g^2 and (1 - beta2) g^2 subnormal) or |g| ~ 1e18."""
    p = rng.normal(0, 1, numel).astype(np.float32)
    if step == 1:
        m = np.zeros(numel, np.float32)
        v = np.zeros(numel, np.float32)
    else:
        m = (rng.normal(0, 0.1, numel)).astype(np.float32)
        v = (rng.uniform(0, 0.02, numel) ** 2).astype(np.float32)
    sign = np.where(rng.uniform(0, 1, numel) < 0.5, -1.0, 1.0)
    g = {"normal": rng.normal(0, 1, numel), "zeros": np.zeros(numel),
         "subnormal": sign * 1e-20 * rng.uniform(0.5, 2.0, numel),
         "huge": sign * 1e18 * rng.uniform(0.5, 2.0, numel)}[grad].astype(np.float32)
    if grad == "normal":
        g[::7] = 0.0
    if grad in ("subnormal", "huge") and step > 1:    # moments of the same magnitude as the gradient
        m = (m * np.float32(1e-19 if grad == "subnormal" else 1e19)).astype(np.float32)
        v = (g.astype(np.float64) ** 2 * rng.uniform(0, 1, numel)).astype(np.float32)
    return p, m, v, g


def densify_inputs(case: Case):
    """radii [N, P] int32 (negative, zero and positive; Gaussian 3k visible in no view, 3k + 1 in every view, the rest
    in some), grad2d [N, P, 3] float32, and the statistics [P] float32 ×3 they accumulate into."""
    P, N = case.q["P"], case.q["N"]
    rng = np.random.RandomState(case.seed)
    radii = rng.randint(-3, 6, (N, P)).astype(np.int32)
    g = np.arange(P)
    radii[:, g % 3 == 0] = rng.randint(-3, 1, (N, int((g % 3 == 0).sum())))
    radii[:, g % 3 == 1] = rng.randint(1, 9, (N, int((g % 3 == 1).sum())))
    grad2d = rng.normal(0, 1e-3, (N, P, 3)).astype(np.float32)
    grad2d[:, ::5, 0] = 0.0
    stats = (rng.randint(0, 5, P).astype(np.float32), rng.uniform(0, 1e-2, P).astype(np.float32),
             rng.randint(0, 40, P).astype(np.float32))
    return radii, grad2d, stats


def mask_bytes(case: Case) -> np.ndarray:
    n, m = case.q["n"], case.content
    if m == "all":
        return np.ones(n, np.uint8)
    if m == "none":
        return np.zeros(n, np.uint8)
    if m == "last":
        out = np.zeros(n, np.uint8)
        out[-1] = 1
        return out
    if m == "alternating":
        return (np.arange(n) % 2 == 0).astype(np.uint8)
    rng = np.random.RandomState(case.seed)        # any byte 0..255, 0 a third of the time: nonzero counts as selected
    out = rng.randint(0, 256, n).astype(np.uint8)
    out[rng.uniform(0, 1, n) < 1 / 3] = 0
    return out


def gather_rows_n0(case: Case):
    """Per tensor (n0, n1, has_src1): rows of src0 and of src1; tensor 2 has n0 = 0 (a NULL src0), tensors 3 and 5 a
    NULL src1 (their n1 rows past n0 are zeros); and the rows every tensor has, which a selection may name."""
    out = [(0 if t == 2 else 9 * t + 5, 200 - t, t not in (3, 5)) for t in range(len(case.q["widths"]))]
    return out, min(n0 + n1 for n0, n1, _ in out)


def knn_points(case: Case) -> np.ndarray:
    P, rng = case.q["P"], np.random.RandomState(case.seed)
    if case.content == "elongated":
        return (rng.uniform(0, 1, (P, 3)) * np.array([4.0, 1.0, 0.25])).astype(np.float32)
    if case.content == "lattice":      # spacing 0.25 (exact), extent 2 = 8 cells of 0.25: every coordinate on a face
        return (np.stack(np.meshgrid(*[np.arange(9)] * 3, indexing="ij"), -1).reshape(-1, 3) * 0.25).astype(np.float32)
    pts = rng.uniform(0, 1, (P, 3)).astype(np.float32)
    if case.content == "faces":        # box exactly [0, 1]^3, cell edge 1 / KNN_MAX_G: a quarter snapped onto faces
        pts[0], pts[1] = 0.0, 1.0
        snap = rng.uniform(0, 1, P) < 0.25
        G = K["KNN_MAX_G"]
        pts[snap] = (np.round(pts[snap] * G) / G).astype(np.float32)
    return pts


def knn_cells(case: Case):
    """The kernel's cells per axis (knn_make_grid) for the case's cloud, in float32."""
    pts = knn_points(case)
    lo, hi = pts.min(0), pts.max(0)
    ext = (hi - lo).astype(np.float32)
    e = np.float32(ext.max()) if ext.max() > 0 else np.float32(1.0)
    G = knn_grid(len(pts))
    inv_h = np.float32(np.float32(G) / e)
    return tuple(min(G, int(np.float32(x * inv_h)) + 1) for x in ext)


def knn_queries(pts: np.ndarray, n: int, seed: int) -> np.ndarray:
    """`n` query indices: the bounding-box extremes of each axis, points on cell faces (a coordinate a multiple of
    1 / KNN_MAX_G when the box is [0, 1]^3), and random ones."""
    G = K["KNN_MAX_G"]
    ext = np.concatenate([pts.argmin(0), pts.argmax(0)])
    on_face = np.flatnonzero((np.round(pts * G) == pts * G).any(1))[: n // 2]
    rng = np.random.RandomState(seed)
    rest = rng.choice(len(pts), min(n, len(pts)), replace=False)
    idx = np.unique(np.concatenate([ext, on_face, rest]))
    return idx[:n] if len(idx) > n else idx


# ---- the statements ----------------------------------------------------------------------------------------------------

def ssim_f64(x, y, w_l1: float, w_dssim: float):
    """loss = w_l1 mean|x - y| + w_dssim (1 - mean SSIM(x, y)) in float64 for float32 torch images x, y [H, W] (any
    device), with the kernel's taps: returns (l1, ssim, total, grad, bound), `grad` by autograd and `bound` per pixel
    a first-order bound of the error of the kernel's float32 operation sequence, in units of u = 2^-24.

    The bound follows the kernel step by step, each rounding worth u times its result, and each window sum (two 11-tap
    fma passes) 22 u times the window sum of the magnitudes:
      mu = W*x: 22 W*|x|;  E[x^2] = W*(x x): 23 W*x^2;  E[xy]: 23 W*|xy|
      s11 = E[x^2] - mu1^2, s12 = E[xy] - mu1 mu2, A1 = 2 mu1 mu2 + C1, A2 = 2 s12 + C2, B1 = mu1^2 + mu2^2 + C1,
      B2 = s11 + s22 + C2: the errors of their operands plus u times each result (3 C for the float32 constants);
      inv = 1 / (B1 B2), S = A1 A2 inv, the maps M3 = 2 A1 inv, M2 = -S / B2 and M1 = 2 mu2 A2 inv - 2 mu1 S / B1
      - 2 mu1 M2 - mu2 M3: first-order propagation (relative errors of products and quotients add), plus u per
      rounding of each term and 3 u of the sum of the four terms' magnitudes;
      grad = inv_n (w_l1 sign(x - y) - w_dssim (W*M1 + 2 x W*M2 + y W*M3)): W*(dM) + 22 W*|M| per map, 2 u of the
      bracket's magnitudes, 2 u of |grad| (inv_n's rounding and the product).
    The sign of a difference of two float32 values is exact, so the L1 term adds only the roundings of the bracket.
    Cancellation enters through the condition numbers it implies, e.g. dB2 / B2 = (E[x^2] + E[y^2] + mu1^2 + mu2^2) /
    B2 and dB1 / B1 = (mu1^2 + mu2^2) / B1 in units of u."""
    import torch
    import torch.nn.functional as F

    dev = x.device
    g = torch.tensor(ssim_taps(), dtype=torch.float64, device=dev)
    w2 = torch.outer(g, g)[None, None]
    LH = K["LH"]

    def conv(t):
        return F.conv2d(t[None, None], w2, padding=LH)[0, 0]

    xd = x.double().clone().requires_grad_(True)
    yd = y.double()
    H, W = x.shape
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    mu1, mu2 = conv(xd), conv(yd)
    e11, e22, e12 = conv(xd * xd), conv(yd * yd), conv(xd * yd)
    s11, s22, s12 = e11 - mu1 * mu1, e22 - mu2 * mu2, e12 - mu1 * mu2
    A1, A2, B1, B2 = 2 * mu1 * mu2 + C1, 2 * s12 + C2, mu1 * mu1 + mu2 * mu2 + C1, s11 + s22 + C2
    smap = A1 * A2 / (B1 * B2)
    l1 = (xd - yd).abs().mean()
    ssim = smap.mean()
    total = w_l1 * l1 + w_dssim * (1.0 - ssim)
    (grad,) = torch.autograd.grad(total, xd)
    with torch.no_grad():
        mu1, mu2, e11, e22, e12 = (t.detach() for t in (mu1, mu2, e11, e22, e12))
        s11, s22, s12, A1, A2, B1, B2 = (t.detach() for t in (s11, s22, s12, A1, A2, B1, B2))
        xa, ya = x.double().abs(), y.double().abs()
        dmu1, dmu2 = 22 * conv(xa), 22 * conv(ya)
        de11, de22, de12 = 23 * e11, 23 * e22, 23 * conv(xa * ya)
        m1s, m2s, m12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
        dm1s, dm2s = 2 * mu1.abs() * dmu1 + m1s, 2 * mu2.abs() * dmu2 + m2s
        dm12 = mu2.abs() * dmu1 + mu1.abs() * dmu2 + m12.abs()
        ds11, ds22 = de11 + dm1s + s11.abs(), de22 + dm2s + s22.abs()
        ds12 = de12 + dm12 + s12.abs()
        dA1 = 2 * dm12 + A1.abs() + 3 * C1
        dA2 = 2 * ds12 + A2.abs() + 3 * C2
        dB1 = dm1s + dm2s + 2 * B1 + 3 * C1
        dB2 = ds11 + ds22 + 2 * B2.abs() + 3 * C2
        inv = 1.0 / (B1 * B2)
        rinv = dB1 / B1 + dB2 / B2 + 2                    # relative error of inv
        S = A1 * A2 * inv
        dS = (dA1 * A2.abs() + A1.abs() * dA2) * inv.abs() + S.abs() * (rinv + 2)
        M2 = -S / B2
        dM2 = dS / B2 + M2.abs() * (dB2 / B2 + 1)
        M3 = 2 * A1 * inv
        dM3 = 2 * dA1 * inv.abs() + M3.abs() * (rinv + 1)
        t1, t2, t3, t4 = 2 * mu2 * A2 * inv, 2 * mu1 * S / B1, 2 * mu1 * M2, mu2 * M3
        dt1 = 2 * (dmu2 * (A2 * inv).abs() + mu2.abs() * dA2 * inv.abs() + (mu2 * A2 * inv).abs() * rinv) + 2 * t1.abs()
        dt2 = 2 * (dmu1 * S.abs() / B1 + mu1.abs() * dS / B1 + t2.abs() / 2 * dB1 / B1) + 2 * t2.abs()
        dt3 = 2 * (dmu1 * M2.abs() + mu1.abs() * dM2) + t3.abs()
        dt4 = dmu2 * M3.abs() + mu2.abs() * dM3 + t4.abs()
        M1 = t1 - t2 - t3 - t4
        dM1 = dt1 + dt2 + dt3 + dt4 + 3 * (t1.abs() + t2.abs() + t3.abs() + t4.abs())
        c1, c2, c3 = conv(M1), conv(M2), conv(M3)
        dc1 = conv(dM1) + 22 * conv(M1.abs())
        dc2 = conv(dM2) + 22 * conv(M2.abs())
        dc3 = conv(dM3) + 22 * conv(M3.abs())
        dssim = c1 + 2 * x.double() * c2 + y.double() * c3
        ddssim = dc1 + 2 * xa * dc2 + ya * dc3 + 2 * (c1.abs() + 2 * (xa * c2).abs() + (ya * c3).abs())
        inv_n = 1.0 / (H * W)
        bound = inv_n * (w_dssim * ddssim + (w_l1 + w_dssim * dssim.abs())) + 2 * grad.abs()
    return l1.item(), ssim.item(), total.item(), grad.detach(), bound


SSIM_K = 2.0     # per-pixel gradient bar: |g - g64| <= SSIM_K u bound (bound is first order; 2 absorbs the rest)


def tv_value_f64(vol: np.ndarray, mean: bool) -> float:
    v = vol.astype(np.float64)
    s = sum(np.abs(np.diff(v, axis=a)).sum() for a in range(3))
    nx, ny, nz = vol.shape
    tot = (nx - 1) * ny * nz + nx * (ny - 1) * nz + nx * ny * (nz - 1)
    if not mean:
        return float(s)
    return float(s / tot) if tot else float("nan")


def tv_grad_exact(vol: np.ndarray, mean: bool) -> np.ndarray:
    """float32(sum of the signs of the six incident differences) * float32(1 / count): the kernel's gradient exactly
    (the sign of a float32 difference is exact); a volume without differences has gradient 0."""
    g = np.zeros(vol.shape, np.float64)
    for a in range(3):
        s = np.sign(np.diff(vol, axis=a)).astype(np.float64)    # float32 differences, exact signs
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[a], hi[a] = slice(0, -1), slice(1, None)
        g[tuple(lo)] -= s
        g[tuple(hi)] += s
    g32 = g.astype(np.float32)
    if not mean:
        return g32
    nx, ny, nz = vol.shape
    tot = (nx - 1) * ny * nz + nx * (ny - 1) * nz + nx * ny * (nz - 1)
    return g32 * np.float32(1.0 / tot) if tot else np.zeros_like(g32)


def _rel32(v: float) -> float:
    """|float32(v) - v| / |v|: the relative rounding of a double constant the kernel receives as float."""
    return abs(float(np.float32(v)) - v) / abs(v)


def adam_f64(p, m, v, g, lr, b1, b2, eps, step, g2=None):
    """One torch.optim.Adam step in float64 from the float32 state (p, m, v) with gradient g (+ g2) and the float32
    learning rate lr; returns (p1, m1, v1) and per-element bounds (dp, dm, dv) of the kernel's float32 sequence

        g = g1 + g2;  m = fma(f(1 - b1), g - m, m);  v = fma(f(1 - b2), g g, f(b2) v);
        den = sqrtf(v) f(1 / sqrt(bc2)) + f(eps);  p = p - (lr f(1 / bc1)) (m / den)

    where f() is the float32 rounding of a double the host computes.  Each rounding is worth u times its result plus
    TINY/2 where the result may be subnormal; the constants' own roundings are exact (_rel32).  sqrt turns an error dv
    into min(dv / (2 sqrt v), sqrt dv)."""
    d = lambda a: np.asarray(a, np.float64)                                  # noqa: E731
    p, m, v, g = d(p), d(m), d(v), d(g)
    gs = g + d(g2) if g2 is not None else g
    bc1, bc2 = 1.0 - b1 ** step, 1.0 - b2 ** step
    m1 = m + (1.0 - b1) * (gs - m)
    v1 = b2 * v + (1.0 - b2) * gs * gs
    isb = 1.0 / math.sqrt(bc2)
    sv = np.sqrt(v1)
    den = sv * isb + eps
    ss = lr / bc1
    q = m1 / den
    p1 = p - ss * q
    t = TINY / 2
    dg = (U * np.abs(gs) + t) if g2 is not None else np.zeros_like(gs)
    ddiff = dg + U * np.abs(gs - m) + t
    dm = (1.0 - b1) * (ddiff + _rel32(1.0 - b1) * np.abs(gs - m)) + U * np.abs(m1) + t
    dgg = 2 * np.abs(gs) * dg + U * gs * gs + t
    dv = (1.0 - b2) * (dgg + _rel32(1.0 - b2) * gs * gs) + b2 * v * (_rel32(b2) + U) + t + U * v1 + t
    with np.errstate(divide="ignore", invalid="ignore"):
        dsv = np.minimum(np.where(sv > 0, dv / (2 * sv), np.inf), np.sqrt(dv)) + U * sv + t
    dden = isb * dsv + sv * isb * (_rel32(isb) + U) + eps * _rel32(eps) + U * den + t
    dq = dm / den + np.abs(q) * (dden / den + U)
    dss = ss * (_rel32(1.0 / bc1) + U)
    dp = ss * dq + np.abs(q) * dss + U * np.abs(ss * q) + U * np.abs(p1) + t
    slack = 1.0 + 2.0 ** -10          # the second-order terms
    return (p1, m1, v1), (slack * dp, slack * dm, slack * dv)


def densify_f32(radii, grad2d, max_radii, accum, denom):
    """The statistics after views 0 .. N-1 in order, in numpy float32 (correctly rounded, as __fmul_rn / __fadd_rn /
    sqrtf): for a view where radii > 0, max_radii = max(max_radii, radii), accum += sqrt(gx^2 + gy^2), denom += 1."""
    mr, acc, den = max_radii.copy(), accum.copy(), denom.copy()
    for r, g in zip(radii, grad2d):
        vis = r > 0
        gx, gy = g[:, 0], g[:, 1]
        norm = np.sqrt((gx * gx) + (gy * gy))
        mr = np.where(vis, np.maximum(mr, r.astype(np.float32)), mr)
        acc = np.where(vis, acc + norm, acc)
        den = np.where(vis, den + np.float32(1.0), den)
    return mr.astype(np.float32), acc.astype(np.float32), den.astype(np.float32)
