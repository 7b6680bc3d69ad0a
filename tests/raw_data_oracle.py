"""Test oracles for `resample` and `process_raw_data`.

* `zoom` restates scipy.ndimage.zoom(x, zoom, order=3, mode="nearest") in float64 numpy: pad by 12 edge voxels,
  prefilter each axis (gain 6, pole sqrt(3) - 2, mirror start value over 30 terms), sample with the cubic B-spline
  weights at x = o (n - 1) / (out - 1) + 12.  `zoom_box` evaluates the same zoom on a box of output voxels from a window
  of the input (`margin` voxels beyond the taps; the prefilter's reach decays as 0.268^k, so 32 voxels leave 5e-19).
* `place` is the placement `resample.zoom_placed` folds into its fill pass, and `scipy_zoom_placed` the stand-in with
  the GPU zoom's signature that runs `process_raw_data`'s chains on the CPU.
* `reference_raw` / `reference_tif` / `reference_dcm` restate the reference's per-type chains line by line with scipy,
  and `fake_tifffile` / `fake_pydicom` stand in for the readers, which are not dependencies of this project.
"""
from __future__ import annotations

import glob
import os
import types

import numpy as np

PAD = 12
POLE = np.sqrt(3.0) - 2.0
CAUSAL_TERMS = 30


def _mirror(k, n):
    r = k % (2 * n - 2)
    return r if r < n else 2 * n - 2 - r


def prefilter_axis(c: np.ndarray, axis: int) -> None:
    """The cubic B-spline prefilter along `axis`, in place."""
    v = np.moveaxis(c, axis, 0)
    n = v.shape[0]
    v *= 6.0
    acc, zk = np.zeros(v.shape[1:]), 1.0
    for k in range(CAUSAL_TERMS):
        acc = acc + zk * v[_mirror(k, n)]
        zk *= POLE
    v[0] = acc
    for i in range(1, n):
        v[i] = v[i] + POLE * v[i - 1]
    v[n - 1] = POLE / (POLE * POLE - 1.0) * (v[n - 1] + POLE * v[n - 2])
    for i in range(n - 2, -1, -1):
        v[i] = POLE * (v[i + 1] - v[i])


def zoom_shape(shape, factors):
    return tuple(int(round(int(n) * float(f))) for n, f in zip(shape, factors))


def _taps(n, out, lo, hi):
    f = (n - 1) / (out - 1) if out > 1 else 1.0
    x = np.arange(lo, hi) * f + PAD
    fl = np.floor(x)
    t = x - fl
    s = 1.0 - t
    w = np.stack([s * s * s / 6.0, (t * t * (t - 2.0) * 3.0 + 4.0) / 6.0, (s * s * (s - 2.0) * 3.0 + 4.0) / 6.0,
                  t * t * t / 6.0], axis=1)
    return fl.astype(np.int64) - 1, w


def zoom_box(get, shape, factors, box=None, margin=None):
    """Zoom of the volume `get(i0, i1, i2)` returns (a float64 sub-array at index vectors i0, i1, i2) on the output box
    [(lo, hi)] * 3 (default: all of it).  margin None uses the whole padded input."""
    factors = [float(f) for f in factors]
    out = zoom_shape(shape, factors)
    box = box or [(0, o) for o in out]
    taps, idx = [], []
    for a in range(3):
        first, w = _taps(shape[a], out[a], *box[a])
        npad = shape[a] + 2 * PAD
        w0, w1 = (0, npad) if margin is None else (max(int(first.min()) - margin, 0),
                                                     min(int(first.max()) + 4 + margin, npad))
        taps.append((first - w0, w))
        idx.append(np.clip(np.arange(w0, w1) - PAD, 0, shape[a] - 1))
    c = np.array(get(*idx), dtype=np.float64)
    for a in range(3):
        prefilter_axis(c, a)
    for a in range(3):
        first, w = taps[a]
        bshape = [1, 1, 1]
        bshape[a] = -1
        c = sum(w[:, j].reshape(bshape) * np.take(c, first + j, axis=a) for j in range(4))
    return c


def zoom(x, factors):
    """scipy.ndimage.zoom(x, factors, order=3, mode="nearest"), restated."""
    x = np.asarray(x, dtype=np.float64)
    factors = [float(f) for f in (factors if np.ndim(factors) else [factors] * 3)]
    if all(f == 1.0 for f in factors):
        return x.copy()
    return zoom_box(lambda i0, i1, i2: x[np.ix_(i0, i1, i2)], x.shape, factors)


def place(src, place_):
    """The placed volume: src set at place_.offset in a volume of place_.shape, normalised, zero elsewhere."""
    src = np.asarray(src)
    out = np.zeros(tuple(place_.shape), dtype=np.float64)
    dst, cut = [], []
    for a in range(3):
        o = int(place_.offset[a])
        lo, hi = max(o, 0), min(o + src.shape[a], int(place_.shape[a]))
        dst.append(slice(lo, hi))
        cut.append(slice(lo - o, hi - o))
    sub = src[tuple(cut)].astype(np.float64)
    out[tuple(dst)] = (sub - float(place_.lo)) / (float(place_.hi) - float(place_.lo))
    return out


def scipy_zoom_placed(source, factors, place_):
    """`resample.zoom_placed` on the CPU with scipy: the stand-in the CPU tests run the chains with."""
    import scipy.ndimage as ndimage

    v = place(source, place_)
    return ndimage.zoom(v, np.asarray(factors, dtype=np.float64), order=3, mode="nearest")


# ---- the reference's chains (data_generator/synthetic_dataset/process_raw_data.py), restated with scipy ----------

def _ref_resample(image, spacing):
    import scipy.ndimage as ndimage

    spacing = np.array(list(spacing))
    resize_factor = spacing / np.array([1, 1, 1])
    new_shape = np.round(image.shape * resize_factor)
    return ndimage.zoom(image, new_shape / image.shape, mode="nearest")


def _ref_expand(a):
    m = max(a.shape)
    pad = [(m - s) // 2 for s in a.shape]
    return np.pad(a, [(p, m - s - p) for p, s in zip(pad, a.shape)], mode="constant", constant_values=0)


def _ref_crop(a):
    m = min(a.shape)
    st = [(s - m) // 2 for s in a.shape]
    return a[st[0]:st[0] + m, st[1]:st[1] + m, st[2]:st[2] + m]


def _ref_resize(scan, target_size):
    import scipy.ndimage as ndimage

    zx, zy, zz = (target_size / s for s in scan.shape)
    if zx != 1.0 or zy != 1.0 or zz != 1.0:
        scan = ndimage.zoom(scan, (zx, zy, zz), mode="nearest")
    return scan


def reference_reshape_vol(image, spacing, target_size, mode):
    if mode is not None:
        image = _ref_resample(image, spacing)
        image = _ref_crop(image) if mode == "crop" else _ref_expand(image)
    return _ref_resize(image, target_size)


def reference_raw(case, target_size):
    data = np.fromfile(case["raw_path"], dtype=case["dtype"]).reshape(case["shape"][::-1]).astype(float)
    data = data.transpose([2, 1, 0])
    data = (data - data.min()) / (data.max() - data.min())
    data = data.clip(0.0, 1.0)
    data = reference_reshape_vol(data, case["spacing"], target_size, case["reshape"]).clip(0.0, 1.0)
    data = data.transpose(case["transpose"])
    return data[:, :, ::-1] if case["z_invert"] else data


def reference_tif(case, target_size, imread):
    data = imread(case["raw_path"])
    data = (data - data.min()) / (data.max() - data.min())
    data = reference_reshape_vol(data, case["spacing"], target_size, case["reshape"]).clip(0.0, 1.0)
    data = data.transpose(case["transpose"])
    return data[:, :, ::-1] if case["z_invert"] else data


def reference_dcm(case, target_size, dcmread):
    slices = []
    for p in sorted(glob.glob(os.path.join(case["raw_path"], "*.dcm"))):
        ds = dcmread(p)
        slices.append(np.array(ds.pixel_array).astype(float) * float(ds.RescaleSlope) + float(ds.RescaleIntercept))
    vol = np.stack(slices, axis=-1)[:, :, ::-1].clip(-1000, 2000)
    vol = (vol - vol.min()) / (vol.max() - vol.min())
    vol = reference_reshape_vol(vol, None, target_size, None).clip(0.0, 1.0)
    return vol[::-1, ::-1, :] if case["xy_invert"] else vol


# ---- fake readers and seeded cases -------------------------------------------------------------------------------

def fake_tifffile():
    """A `tifffile` whose imread loads the .npy file saved under the .tif path."""
    def imread(path):
        with open(path, "rb") as f:
            return np.load(f)

    return types.SimpleNamespace(imread=imread)


def fake_pydicom():
    """A `pydicom` whose dcmread loads a .npz holding pixel_array, RescaleSlope and RescaleIntercept."""
    def dcmread(path):
        with open(path, "rb") as f:
            z = np.load(f)
            return types.SimpleNamespace(pixel_array=z["pixel_array"], RescaleSlope=str(z["slope"]),
                                         RescaleIntercept=str(z["intercept"]), SliceThickness=2.5,
                                         PixelSpacing=[0.7, 0.7])

    return types.SimpleNamespace(dcmread=dcmread)


def blob_volume(shape, rng, dtype=np.uint8):
    """A seeded volume of a few smooth blobs over noise, scaled to the range of `dtype`."""
    g = [np.linspace(-1, 1, n) for n in shape]
    x, y, z = np.meshgrid(*g, indexing="ij")
    v = rng.uniform(0, 0.05, shape)
    for _ in range(4):
        c, r = rng.uniform(-0.5, 0.5, 3), rng.uniform(0.2, 0.6, 3)
        v += rng.uniform(0.3, 0.8) * np.exp(-(((x - c[0]) / r[0]) ** 2 + ((y - c[1]) / r[1]) ** 2
                                              + ((z - c[2]) / r[2]) ** 2))
    v /= v.max()
    if np.dtype(dtype).kind == "f":
        return v.astype(dtype)
    return np.round(v * np.iinfo(dtype).max).astype(dtype)


def write_raw(path, vol):
    """Write vol[x, y, z] as the reference reads it: fromfile(...).reshape(shape[::-1]).transpose(2, 1, 0)."""
    np.ascontiguousarray(vol.transpose(2, 1, 0)).tofile(path)


def write_tif(path, vol):
    with open(path, "wb") as f:
        np.save(f, vol)


def write_dcm_series(folder, slices, slope, intercept):
    os.makedirs(folder, exist_ok=True)
    for i, s in enumerate(slices):
        with open(os.path.join(folder, f"{i:04d}.dcm"), "wb") as f:
            np.savez(f, pixel_array=s, slope=np.float64(slope), intercept=np.float64(intercept))


def write_metadata(path, raw_info):
    with open(path, "w") as f:
        f.write(f"raw_info = {raw_info!r}\n")
