"""numpy restatement of the per-view chain that turns a processed FIPS projection into the detector image a real-scan
scene stores (the reference's `data_generator/real_dataset/generate_data.py`, lines 91-109), with the float32
INTER_LINEAR resize that `cv2.resize` runs written out step by step.  r2x_projection_prepare (csrc/r2x_prepare.cu)
is checked against it bit for bit, and it against cv2's own bytes (tests/golden/real_data/).

    out = prepare(img, subsample, proj_rescale, object_scale)     # img float64 [H0, W0] -> float32 [H, W]

The resize is the one the x86-64 OpenCV wheels run (their Intel IPP path, on by default): per axis the source position
x = (d + 0.5) (src / dst) - 0.5 in float64, i = floor(x), t = float32(x - i), neighbours i and min(i + 1, src - 1);
one value is a + t (b - a) as a single fused multiply-add, fma(t, b - a, a), in float32; a horizontal pass into float32
rows, then the same along the columns.  OpenCV built without IPP (or with it switched off) computes a (1 - t) + b t
with float32 weights instead and differs in the last bits; `reference_chain` says which one the installed cv2 runs.
"""
from __future__ import annotations

import numpy as np

SHIFT_ROWS = 5     # the FIPS data description: the image sits 5 rows low

f32 = np.float32


def fma_f32(a, b, c) -> np.ndarray:
    """float32 fma(a, b, c) rounded once, for float32 arrays: the product is exact in float64; the sum's float64
    rounding error e is recovered (two-sum) and decides the float32 rounding when the float64 sum sits exactly
    half-way between two float32 values (the only case where rounding twice differs from rounding once)."""
    a, b, c = (np.asarray(v, f32).astype(np.float64) for v in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    with np.errstate(over="ignore", invalid="ignore"):
        r = s.astype(f32)
        other = np.nextafter(r, np.where(s >= r.astype(np.float64), f32(np.inf), f32(-np.inf)).astype(f32))
        tie = (s == (r.astype(np.float64) + other.astype(np.float64)) * 0.5) & (e != 0)
        lo, hi = np.minimum(r, other), np.maximum(r, other)
    return np.where(tie, np.where(e > 0, hi, lo), r).astype(f32)


def scale_clamp(img, proj_rescale: float, object_scale: float) -> np.ndarray:
    """float32(img / proj_rescale * object_scale), each operation in float64 and one rounding to float32, negatives
    (not -0, not NaN) set to 0."""
    p = (np.asarray(img, np.float64) / float(proj_rescale) * float(object_scale)).astype(f32)
    p[p < 0] = 0
    return p


def shift_up(p: np.ndarray) -> np.ndarray:
    out = np.zeros_like(p)
    out[:-SHIFT_ROWS] = p[SHIFT_ROWS:]
    return out


def linear_taps(n_src: int, n_dst: int):
    """(i0, i1, t) per destination index: x = (d + 0.5) (n_src / n_dst) - 0.5 in float64 (0 when negative),
    i0 = floor(x), i1 = min(i0 + 1, n_src - 1), t = float32(x - i0)."""
    d = np.arange(n_dst, dtype=np.float64)
    x = np.maximum((d + 0.5) * (float(n_src) / float(n_dst)) - 0.5, 0.0)
    i0 = np.floor(x).astype(np.int64)
    return i0, np.minimum(i0 + 1, n_src - 1), (x - i0).astype(f32)


def resize_linear(p: np.ndarray, H: int, W: int) -> np.ndarray:
    """cv2.resize(p, (W, H)) of a float32 image (INTER_LINEAR, the IPP path): columns first, then rows."""
    p = np.asarray(p, f32)
    j0, j1, tx = linear_taps(p.shape[1], W)
    rows = fma_f32(tx[None, :], p[:, j1] - p[:, j0], p[:, j0])
    i0, i1, ty = linear_taps(p.shape[0], H)
    return fma_f32(ty[:, None], rows[i1] - rows[i0], rows[i0])


def output_shape(H0: int, W0: int, subsample: int):
    """(resized H, resized W, first row, first column, H, W) of the prepared image: int(H0 / s) x int(W0 / s), then
    the longer axis centre-cropped by int(diff / 2) on each side (a difference of 1 crops nothing).  s = 1: no
    resize, no crop."""
    if subsample == 1:
        return H0, W0, 0, 0, H0, W0
    Hr, Wr = int(H0 / subsample), int(W0 / subsample)
    off = int(abs(Hr - Wr) / 2)
    if Hr > Wr:
        return Hr, Wr, off, 0, Hr - 2 * off, Wr
    return Hr, Wr, 0, off, Hr, Wr - 2 * off


def prepare(img, subsample: int, proj_rescale: float, object_scale: float) -> np.ndarray:
    p = shift_up(scale_clamp(img, proj_rescale, object_scale))
    if subsample == 1:
        return p
    Hr, Wr, r0, c0, H, W = output_shape(*p.shape, subsample)
    return np.ascontiguousarray(resize_linear(p, Hr, Wr)[r0:r0 + H, c0:c0 + W])


def reference_chain(img, subsample: int, proj_rescale: float, object_scale: float):
    """The reference's own lines, run with cv2 (None when cv2 is not importable).  Its crop keeps the `off:-off`
    slice, so a difference of 1 gives an empty array here."""
    try:
        import cv2
    except ImportError:
        return None
    proj = np.asarray(img, np.float64) / proj_rescale * object_scale
    proj = proj.astype(np.float32)
    proj[proj < 0] = 0
    proj_new = np.zeros_like(proj)
    proj_new[:-5] = proj[5:]
    proj = proj_new
    if subsample != 1.0:
        h_ori, w_ori = proj.shape
        h_new, w_new = int(h_ori / subsample), int(w_ori / subsample)
        proj = cv2.resize(proj, [w_new, h_new])
        dim_x, dim_y = proj.shape
        if dim_x > dim_y:
            dim_offset = int((dim_x - dim_y) / 2)
            proj = proj[dim_offset:-dim_offset, :]
        elif dim_x < dim_y:
            dim_offset = int((dim_y - dim_x) / 2)
            proj = proj[:, dim_offset:-dim_offset]
    return proj


CONFIG_TEMPLATE = """[Geometry]
NumberImages = {n}
AngleInterval = {interval}
AngleFirst = {first}
AngleLast = {last}
DistanceSourceDetector = {dsd}
DistanceSourceOrigin = {dso}
PixelSize = {pixel}
PixelSizeUnit = mm
"""


def write_fips_case(path: str, imgs, first: float, interval: float, dsd: float = 553.74, dso: float = 410.66,
                    pixel: float = 0.05, n_proj=None) -> None:
    """A processed-scan directory: config.txt (lengths in millimetres) and one <name>_NNNN.mat per view with `img`."""
    import os

    import scipy.io

    os.makedirs(path, exist_ok=True)
    n = len(imgs)
    with open(os.path.join(path, "config.txt"), "w") as f:
        f.write(CONFIG_TEMPLATE.format(n=n if n_proj is None else n_proj, interval=interval, first=first,
                                       last=first + interval * (n - 1), dsd=dsd, dso=dso, pixel=pixel))
    for i, img in enumerate(imgs):
        scipy.io.savemat(os.path.join(path, f"scan_{i:04d}.mat"), {"img": np.asarray(img, np.float64)})
