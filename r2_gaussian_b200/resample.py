"""Cubic B-spline zoom of a 3-D volume on the GPU: `scipy.ndimage.zoom(x, zoom, order=3, mode="nearest")`.

    from r2_gaussian_b200.resample import zoom
    out = zoom(volume, (0.5, 2.0, 1.0))      # CUDA float64 [nx, ny, nz] -> CUDA float64

The output has int(round(n * zoom)) voxels per axis (Python's round, as scipy); all factors exactly 1 return a copy,
as scipy does.  Otherwise the volume is padded by 12 edge voxels, prefiltered along each axis and sampled with the
cubic B-spline weights (r2x_zoom_cubic, include/r2x.h).  Against scipy the results agree within 1e-12 on [0, 1]
data (tests/test_raw_data_gpu.py), not bit for bit: the prefilter's start values at the ends of a line and the
summation order differ in the last bits.  There is no CPU fallback.

`zoom_placed(source, zoom, place)` is the same zoom of a *placed* volume (`Place`): a source of uint8, uint16 or
float64 voxels (a host numpy array, uploaded in its own dtype, or a CUDA float64 tensor) set at an offset in a volume of
`place.shape`, zero where it does not reach, and normalised as (source - lo) / (hi - lo).  That is how
`process_raw_data` normalises, converts, expands or crops a raw volume inside the zoom's own fill pass, without ever
holding the normalised or cubed volume in memory.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import NamedTuple

import numpy as np

_DTYPES = {np.dtype(np.uint8): 0, np.dtype(np.uint16): 1, np.dtype(np.float64): 2}   # R2X_PLACE_U8 / U16 / F64


class Place(NamedTuple):
    """Where a source volume sits and how it is scaled: V[p] = (source[p - offset] - lo) / (hi - lo) where p - offset
    lies inside the source, else 0.  A positive offset pads with zeros, a negative one crops."""
    shape: tuple
    offset: tuple = (0, 0, 0)
    lo: float = 0.0
    hi: float = 1.0

    @staticmethod
    def of(source_shape) -> "Place":
        """The source as it is: same shape, no offset, values unchanged."""
        return Place(tuple(int(n) for n in source_shape))


def zoom_factors(zoom) -> tuple:
    """Three finite, positive float factors from a number or a sequence of three."""
    z = [zoom] * 3 if np.ndim(zoom) == 0 else list(np.asarray(zoom, dtype=np.float64).reshape(-1))
    if len(z) != 3 or not all(math.isfinite(float(f)) and float(f) > 0.0 for f in z):
        raise ValueError(f"zoom: factors must be one or three finite positive numbers, got {zoom!r}")
    return tuple(float(f) for f in z)


def zoom_shape(shape, zoom) -> tuple:
    """int(round(n * zoom)) per axis, refused when an axis would vanish."""
    out = tuple(int(round(int(n) * f)) for n, f in zip(shape, zoom_factors(zoom)))
    if min(out) < 1:
        raise ValueError(f"zoom: {tuple(shape)} zoomed by {zoom_factors(zoom)} leaves an empty axis {out}")
    return out


def workspace_bytes(shape) -> int:
    """Device bytes r2x_zoom_cubic pads a placed volume of `shape` into (no GPU needed)."""
    from ._lib import load

    n = int(load().r2x_zoom_workspace_bytes(*(int(s) for s in shape)))
    if n == 0:
        raise ValueError(f"zoom: volume shape {tuple(shape)} is out of range (each size in [1, 32768])")
    return n


def device_source(source):
    """(tensor that owns the device bytes, R2X_PLACE_* code, shape, element strides) of a host array, uploaded in its
    own dtype, or of a CUDA float64 tensor."""
    import torch

    if isinstance(source, torch.Tensor):
        if source.device.type != "cuda" or source.dtype != torch.float64 or source.dim() != 3:
            raise ValueError("zoom: the volume must be a CUDA float64 [nx, ny, nz] tensor (there is no CPU fallback)")
        return source, 2, tuple(source.shape), tuple(source.stride())
    arr = np.asarray(source)
    if arr.ndim != 3 or arr.dtype not in _DTYPES:
        raise ValueError(f"zoom: a host source must be a 3-D uint8, uint16 or float64 array, got {arr.dtype} {arr.shape}")
    # keep a transposed view's strides: upload the contiguous array behind it, not a transposed copy
    order = np.argsort([-s for s in arr.strides], kind="stable")
    if min(arr.strides) < 0 or not arr.transpose(order).flags.c_contiguous:
        arr = np.ascontiguousarray(arr)
        order = np.arange(3)
    flat = np.ascontiguousarray(arr.transpose(order)).reshape(-1).view(np.uint8)
    dev = torch.from_numpy(flat).cuda()
    return dev, _DTYPES[arr.dtype], arr.shape, tuple(s // arr.itemsize for s in arr.strides)


def _desc(dev, code, shape, strides, place: Place):
    from ._lib import PlaceDesc

    d = PlaceDesc()
    d.src, d.dtype = dev.data_ptr(), code
    for a in range(3):
        d.src_shape[a], d.src_strides[a] = int(shape[a]), int(strides[a])
        d.shape[a], d.offset[a] = int(place.shape[a]), int(place.offset[a])
    d.lo, d.hi = float(place.lo), float(place.hi)
    return d


def zoom_placed(source, zoom, place: Place):
    """scipy.ndimage.zoom(V, zoom, order=3, mode="nearest") of the placed volume V (`Place`) of `source` (a host numpy
    uint8 / uint16 / float64 array or a CUDA float64 tensor): a CUDA float64 tensor, on the current stream."""
    import torch

    _plan(zoom, place)                              # refuse bad arguments before uploading anything
    if not torch.cuda.is_available():
        raise RuntimeError("zoom needs a CUDA device: the cubic spline zoom runs on the GPU, with no CPU fallback")
    return zoom_device(*device_source(source), zoom, place)


def _plan(zoom, place: Place):
    """(copy?, output shape, workspace bytes) of a zoom of a placed volume; scipy returns a copy for all factors 1."""
    if len(place.shape) != 3 or len(place.offset) != 3:
        raise ValueError(f"zoom: a placement needs a 3-D shape and offset, got {place}")
    factors = zoom_factors(zoom)
    copy = all(f == 1.0 for f in factors)
    out_shape = tuple(int(n) for n in place.shape) if copy else zoom_shape(place.shape, factors)
    return copy, out_shape, workspace_bytes(place.shape)


def zoom_device(dev, code: int, shape, strides, zoom, place: Place):
    """`zoom_placed` of a source already on the device: `dev` owns its bytes, `code` is its R2X_PLACE_* element type,
    `shape` and `strides` (in elements) say where its voxels are."""
    import torch

    from ._lib import check, load

    copy, out_shape, ws = _plan(zoom, place)
    desc = _desc(dev, code, shape, strides, place)
    with torch.cuda.device(dev.device):
        stream = torch.cuda.current_stream(dev.device).cuda_stream
        out = torch.empty(out_shape, dtype=torch.float64, device=dev.device)
        if copy:
            check(load().r2x_volume_place(stream, C.byref(desc), out.data_ptr()), "r2x_volume_place")
        else:
            work = torch.empty(ws, dtype=torch.uint8, device=dev.device)
            check(load().r2x_zoom_cubic(stream, C.byref(desc), *out_shape, work.data_ptr(), ws, out.data_ptr()),
                  "r2x_zoom_cubic")
    return out


def zoom(volume, zoom):
    """scipy.ndimage.zoom(volume, zoom, order=3, mode="nearest") of a CUDA float64 [nx, ny, nz] tensor, as a new CUDA
    float64 tensor.  `zoom` is one positive factor or three.  Other dtypes and CPU tensors are refused."""
    import torch

    if not isinstance(volume, torch.Tensor) or volume.device.type != "cuda" or volume.dtype != torch.float64 \
            or volume.dim() != 3:
        raise ValueError("zoom: the volume must be a CUDA float64 [nx, ny, nz] tensor (there is no CPU fallback)")
    return zoom_placed(volume, zoom, Place.of(volume.shape))
