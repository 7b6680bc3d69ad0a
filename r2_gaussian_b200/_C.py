"""Python face of the native library with the reference extension's five entry points.

The reference registers `rasterize_gaussians`, `rasterize_gaussians_backward`, `voxelize_gaussians`,
`voxelize_gaussians_backward`, `mark_visible` in its pybind module `_C` (SUB/ext.cpp:17-23; argument
lists SUB/rasterize_points.h:18-61, SUB/voxelize_points.cu:29-167).  This module offers the same five
callables with the same positional arguments and return tuples, implemented over the C ABI of
libr2xray.so (include/r2x.h) with raw device pointers.  torch is used for device memory and the current
stream only.  There is no CPU path: non-CUDA inputs raise.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

import torch

from ._lib import ALLOC_FN, check, load

__all__ = [
    "rasterize_gaussians",
    "rasterize_gaussians_backward",
    "voxelize_gaussians",
    "voxelize_gaussians_backward",
    "mark_visible",
]


def _f32(t: torch.Tensor, dev) -> torch.Tensor:
    """float32, contiguous, on `dev` (empty tensors stay empty)."""
    if t.numel() == 0:
        return t
    if t.device != dev:
        if t.device.type != "cuda":
            t = t.to(dev)  # small host-side settings tensors (e.g. campos) only
        else:
            raise ValueError(f"tensor on {t.device}, expected {dev}")
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


def _ptr(t) -> int | None:
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


def _require_cuda(t: torch.Tensor, name: str):
    if not isinstance(t, torch.Tensor) or t.device.type != "cuda":
        raise RuntimeError(
            f"{name} must be a CUDA tensor: the GPU rasterizer/voxelizer has no CPU fallback "
            f"(got {getattr(t, 'device', type(t))})"
        )


class _Workspace:
    """Per-(device, kind, size) instance-capacity hints so that the binning buffer can be provisioned
    BEFORE the forward runs: the whole pipeline is then enqueued without a host round trip in the middle,
    and the one synchronisation the reference API needs anyway (num_rendered is a Python int) happens at
    the end.  If a call needs more instances than provisioned it is simply re-run with a larger buffer.
    Capacities are rounded to a coarse grid so that torch's caching allocator sees repeating sizes."""

    hints: dict = {}
    _pinned: list = []

    @classmethod
    def pinned_status(cls):
        return cls._pinned.pop() if cls._pinned else torch.zeros(2, dtype=torch.int32).pin_memory()

    @classmethod
    def release(cls, t):
        if len(cls._pinned) < 16:
            cls._pinned.append(t)

    @staticmethod
    def _round(n: int) -> int:
        step = 1 << max(12, int(n).bit_length() - 3)   # ~12.5 % granularity
        return (int(n) + step - 1) // step * step

    @classmethod
    def capacity(cls, key, P: int, per_gaussian: int) -> int:
        return cls.hints.get(key) or cls._round(max(per_gaussian * P, 1 << 14))

    @classmethod
    def update(cls, key, R: int):
        want = cls._round(int(R * 1.2) + 1024)
        cur = cls.hints.get(key, 0)
        # grow immediately, shrink slowly (keeps sizes stable while the cloud changes during training)
        cls.hints[key] = want if want > cur or want < cur // 2 else cur


class CapacityOverflow(RuntimeError):
    """A speculative forward (see `speculative`) needed more (Gaussian, tile) instances than its binning buffer was
    provisioned for; its image / volume is all zeros.  Raised by the matching backward (or by `NumRendered.resolve()`);
    the capacity hint has been raised, so simply repeating the iteration succeeds."""


class NumRendered(int):
    """`num_rendered` as the reference returns it (a Python int) that also remembers the instance capacity the
    binning buffer was carved for: the backward must carve the buffer with the same number.  The autograd
    bridges keep this object in `ctx` and hand it back unchanged, exactly like the reference's plain int.

    After a speculative forward the integer value is the provisioned capacity (an upper bound) and `pending` holds
    the pinned status word + event; `resolve()` waits for that event (long past by the time the backward runs),
    returns the exact count and raises CapacityOverflow if the forward had overflowed."""

    capacity: int
    pending = None

    def __new__(cls, value: int, capacity: int | None = None, pending=None):
        obj = super().__new__(cls, int(value))
        obj.capacity = int(value if capacity is None else capacity)
        obj.pending = pending
        return obj

    def resolve(self) -> int:
        if self.pending is None:
            return int(self)
        host, event, key = self.pending
        event.synchronize()
        R, overflow = int(host[0]), int(host[1])
        self.pending = None
        _Workspace.update(key, R)
        _Workspace.release(host)
        if overflow:
            raise CapacityOverflow(f"forward needed {R} instances, binning buffer provisioned for {self.capacity}; "
                                   "the capacity hint has been raised -- repeat the iteration")
        return R


class speculative:
    """Context manager used by the autograd bridges in training mode: inside it the forward entry points do NOT
    synchronise with the host (the one sync of the reference API, `num_rendered` being a Python int, is what
    serialises host and device twice per training iteration).  The binning buffer is provisioned from the instance
    count of the previous call with the same shape (+20 %), the status word travels to pinned host memory behind an
    event, and the check happens in the backward.  Disabled by R2X_SPECULATIVE=0, by debug=True, under no_grad, and
    for the first call of a shape (no hint yet)."""

    _tls = threading.local()

    def __init__(self, on: bool = True):
        self.on = bool(on) and os.environ.get("R2X_SPECULATIVE", "1") != "0"

    def __enter__(self):
        self.prev = getattr(self._tls, "on", False)
        self._tls.on = self.on
        return self

    def __exit__(self, *exc):
        self._tls.on = self.prev
        return False

    @classmethod
    def active(cls) -> bool:
        return bool(getattr(cls._tls, "on", False))


def _carved_capacity(binning: torch.Tensor, R) -> int:
    """Instance count the binning buffer was carved for (what the backward must carve with)."""
    return int(getattr(R, "capacity", R))


def _pending(status, cap, key, dev) -> NumRendered:
    """Ship the device status word {R, overflow} to pinned host memory behind an event (no host wait)."""
    host = _Workspace.pinned_status()
    host.copy_(status, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream(dev))
    return NumRendered(cap, cap, (host, ev, key))


def _status_pair(dev):
    st = torch.empty(2, dtype=torch.int32, device=dev)
    return st


def rasterize_gaussians(means3D, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                        projmatrix, tan_fovx, tan_fovy, image_height, image_width, campos, prefiltered, mode,
                        debug):
    """-> (num_rendered, out_color[1,H,W], radii[P] int32, geomBuffer, binningBuffer, imgBuffer).

    The binning buffer is provisioned for a capacity >= num_rendered (see _Workspace); num_rendered is a
    `NumRendered` int that carries that capacity to the backward."""
    _require_cuda(means3D, "means3D")
    if means3D.ndim != 2 or means3D.shape[1] != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    lib = load()
    dev = means3D.device
    P, H, W = int(means3D.shape[0]), int(image_height), int(image_width)
    with torch.cuda.device(dev):
        means3D = _f32(means3D, dev); opacity = _f32(opacity, dev)
        scales = _f32(scales, dev); rotations = _f32(rotations, dev); cov3D_precomp = _f32(cov3D_precomp, dev)
        viewmatrix = _f32(viewmatrix, dev); projmatrix = _f32(projmatrix, dev); campos = _f32(campos, dev)
        u8 = dict(dtype=torch.uint8, device=dev)
        out_color = torch.empty((1, H, W), dtype=torch.float32, device=dev)
        radii = torch.empty((P,), dtype=torch.int32, device=dev)
        geom = torch.empty(lib.r2x_raster_geom_bytes(P), **u8)
        img = torch.empty(lib.r2x_raster_image_bytes(P, W, H), **u8)
        status = _status_pair(dev)
        key = ("raster", dev.index, P, W, H)
        stream = torch.cuda.current_stream(dev).cuda_stream
        if debug or P == 0:
            alloc = _BinningAlloc(dev)
            nr = C.c_int(0)
            rc = lib.r2x_raster_forward(
                stream, P, W, H, _ptr(means3D), _ptr(opacity), _ptr(scales), float(scale_modifier), _ptr(rotations),
                _ptr(cov3D_precomp), _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos), float(tan_fovx), float(tan_fovy),
                int(bool(prefiltered)), int(mode), out_color.data_ptr(), _ptr(radii), geom.data_ptr(), img.data_ptr(),
                alloc.cb, None, int(bool(debug)), C.byref(nr))
            check(rc, "r2x_raster_forward")
            return NumRendered(nr.value), out_color, radii, geom, alloc.tensor, img
        cap = _Workspace.capacity(key, P, 12)
        spec = speculative.active() and key in _Workspace.hints
        if spec:    # generous: an overflow needs the instance count to double between two calls of this shape
            cap = _Workspace._round(max(2 * cap, 12 * P))
        while True:
            binning = torch.empty(lib.r2x_binning_bytes(cap), **u8)
            rc = lib.r2x_raster_forward_async(
                stream, P, W, H, _ptr(means3D), _ptr(opacity), _ptr(scales), float(scale_modifier), _ptr(rotations),
                _ptr(cov3D_precomp), _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos), float(tan_fovx), float(tan_fovy),
                int(bool(prefiltered)), int(mode), out_color.data_ptr(), _ptr(radii), geom.data_ptr(), img.data_ptr(),
                binning.data_ptr(), cap, status.data_ptr())
            check(rc, "r2x_raster_forward_async")
            if spec:
                return (_pending(status, cap, key, dev), out_color, radii, geom, binning, img)
            R, overflow = status.tolist()      # the one host synchronisation of the call
            _Workspace.update(key, R)
            if not overflow:
                break
            cap = _Workspace.capacity(key, P, 12)
    return NumRendered(R, cap), out_color, radii, geom, binning, img


class _BinningAlloc:
    """Allocator handed to the synchronous C entry point for the R-dependent binning buffer."""

    def __init__(self, device):
        self.device = device
        self.tensor = torch.empty(0, dtype=torch.uint8, device=device)
        self.cb = ALLOC_FN(self._alloc)

    def _alloc(self, nbytes, _user):
        self.tensor = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
        return self.tensor.data_ptr()


def rasterize_gaussians_backward(means3D, radii, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                                 projmatrix, tan_fovx, tan_fovy, dL_dout_color, campos, geomBuffer, R,
                                 binningBuffer, imageBuffer, mode, debug):
    """-> (dL_dmeans2D[P,3], dL_dopacity[P,1], dL_dmu[P,1], dL_dmeans3D[P,3], dL_dcov3D[P,6],
    dL_dscales[P,3], dL_drotations[P,4])."""
    _require_cuda(means3D, "means3D")
    lib = load()
    dev = means3D.device
    P = int(means3D.shape[0])
    H, W = int(dL_dout_color.shape[-2]), int(dL_dout_color.shape[-1])
    with torch.cuda.device(dev):
        means3D = _f32(means3D, dev); scales = _f32(scales, dev); rotations = _f32(rotations, dev)
        cov3D_precomp = _f32(cov3D_precomp, dev); viewmatrix = _f32(viewmatrix, dev)
        projmatrix = _f32(projmatrix, dev); campos = _f32(campos, dev); dL = _f32(dL_dout_color, dev)
        opts = dict(dtype=torch.float32, device=dev)
        g_mean2D = torch.empty((P, 3), **opts); g_op = torch.empty((P, 1), **opts); g_mu = torch.empty((P, 1), **opts)
        g_mean3D = torch.empty((P, 3), **opts); g_cov = torch.empty((P, 6), **opts)
        g_scale = torch.empty((P, 3), **opts); g_rot = torch.empty((P, 4), **opts)
        if getattr(R, "pending", None) is not None:
            R.resolve()                         # raises CapacityOverflow if the speculative forward did not fit
        R = _carved_capacity(binningBuffer, R)
        scratch = torch.empty(lib.r2x_raster_bwd_scratch_bytes(int(R)), dtype=torch.uint8, device=dev)
        rc = lib.r2x_raster_backward(
            torch.cuda.current_stream(dev).cuda_stream, P, int(R), W, H, _ptr(means3D), _ptr(scales),
            float(scale_modifier), _ptr(rotations), _ptr(cov3D_precomp), _ptr(viewmatrix), _ptr(projmatrix),
            _ptr(campos), float(tan_fovx), float(tan_fovy), _ptr(radii), _ptr(geomBuffer), _ptr(binningBuffer),
            _ptr(imageBuffer), scratch.data_ptr(), _ptr(dL), _ptr(g_mean2D), _ptr(g_op), _ptr(g_mu),
            _ptr(g_mean3D), _ptr(g_cov), _ptr(g_scale), _ptr(g_rot), int(mode), int(bool(debug)))
        check(rc, "r2x_raster_backward")
    return g_mean2D, g_op, g_mu, g_mean3D, g_cov, g_scale, g_rot


def mark_visible(means3D, viewmatrix, projmatrix):
    """-> bool[P]: view-space z > 0.2 (RAS/auxiliary.h:143-168)."""
    _require_cuda(means3D, "means3D")
    lib = load()
    dev = means3D.device
    P = int(means3D.shape[0])
    with torch.cuda.device(dev):
        means3D = _f32(means3D, dev); viewmatrix = _f32(viewmatrix, dev); projmatrix = _f32(projmatrix, dev)
        present = torch.zeros((P,), dtype=torch.bool, device=dev)
        rc = lib.r2x_mark_visible(torch.cuda.current_stream(dev).cuda_stream, P, _ptr(means3D), _ptr(viewmatrix),
                                  _ptr(projmatrix), _ptr(present))
        check(rc, "r2x_mark_visible")
    return present


def voxelize_gaussians(means3D, opacity, scales, rotations, scale_modifier, cov3D_precomp, nVoxel_x, nVoxel_y,
                       nVoxel_z, sVoxel_x, sVoxel_y, sVoxel_z, center_x, center_y, center_z, prefiltered, debug):
    """-> (num_rendered, out_volume[nx,ny,nz], radii_x, radii_y, radii_z, geomBuffer, binningBuffer, imgBuffer)."""
    _require_cuda(means3D, "means3D")
    if means3D.ndim != 2 or means3D.shape[1] != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")
    lib = load()
    dev = means3D.device
    P = int(means3D.shape[0])
    nx, ny, nz = int(nVoxel_x), int(nVoxel_y), int(nVoxel_z)
    with torch.cuda.device(dev):
        means3D = _f32(means3D, dev); opacity = _f32(opacity, dev)
        scales = _f32(scales, dev); rotations = _f32(rotations, dev); cov3D_precomp = _f32(cov3D_precomp, dev)
        u8 = dict(dtype=torch.uint8, device=dev)
        vol = torch.empty((nx, ny, nz), dtype=torch.float32, device=dev)
        rx = torch.empty((P,), dtype=torch.int32, device=dev)
        ry = torch.empty_like(rx); rz = torch.empty_like(rx)
        geom = torch.empty(lib.r2x_voxel_geom_bytes(P), **u8)
        img = torch.empty(lib.r2x_voxel_image_bytes(P, nx, ny, nz), **u8)
        stream = torch.cuda.current_stream(dev).cuda_stream
        grid_args = (nx, ny, nz, float(sVoxel_x), float(sVoxel_y), float(sVoxel_z), float(center_x), float(center_y),
                     float(center_z))
        in_args = (_ptr(means3D), _ptr(opacity), _ptr(scales), float(scale_modifier), _ptr(rotations),
                   _ptr(cov3D_precomp), int(bool(prefiltered)))
        if debug or P == 0:
            alloc = _BinningAlloc(dev)
            nr = C.c_int(0)
            rc = lib.r2x_voxel_forward(stream, P, *grid_args, *in_args, vol.data_ptr(), _ptr(rx), _ptr(ry), _ptr(rz),
                                       geom.data_ptr(), img.data_ptr(), alloc.cb, None, int(bool(debug)), C.byref(nr))
            check(rc, "r2x_voxel_forward")
            return NumRendered(nr.value), vol, rx, ry, rz, geom, alloc.tensor, img
        # the instance count depends strongly on the voxel pitch: key the hint on the grid as well
        key = ("voxel", dev.index, P, nx, ny, nz, round(float(sVoxel_x) / nx, 6))
        status = _status_pair(dev)
        cap = _Workspace.capacity(key, P, 8)
        spec = speculative.active() and key in _Workspace.hints
        if spec:    # (random TV crops see very different instance counts: keep at least 8 per Gaussian)
            cap = _Workspace._round(max(2 * cap, 8 * P))
        while True:
            binning = torch.empty(lib.r2x_binning_bytes(cap), **u8)
            rc = lib.r2x_voxel_forward_async(stream, P, *grid_args, *in_args, vol.data_ptr(), _ptr(rx), _ptr(ry),
                                             _ptr(rz), geom.data_ptr(), img.data_ptr(), binning.data_ptr(), cap,
                                             status.data_ptr())
            check(rc, "r2x_voxel_forward_async")
            if spec:
                return (_pending(status, cap, key, dev), vol, rx, ry, rz, geom, binning, img)
            R, overflow = status.tolist()
            _Workspace.update(key, R)
            if not overflow:
                break
            cap = _Workspace.capacity(key, P, 8)
    return NumRendered(R, cap), vol, rx, ry, rz, geom, binning, img


def voxelize_gaussians_backward(means3D, radii_x, radii_y, radii_z, scales, rotations, scale_modifier,
                                cov3D_precomp, dL_dout, geomBuffer, R, binningBuffer, imageBuffer, nVoxel_x,
                                nVoxel_y, nVoxel_z, sVoxel_x, sVoxel_y, sVoxel_z, center_x, center_y, center_z,
                                debug):
    """-> (dL_dopacity[P,1], dL_dmeans3D[P,3], dL_dcov3D[P,6], dL_dscales[P,3], dL_drotations[P,4])."""
    _require_cuda(means3D, "means3D")
    lib = load()
    dev = means3D.device
    P = int(means3D.shape[0])
    with torch.cuda.device(dev):
        means3D = _f32(means3D, dev); scales = _f32(scales, dev); rotations = _f32(rotations, dev)
        cov3D_precomp = _f32(cov3D_precomp, dev); dL = _f32(dL_dout, dev)
        opts = dict(dtype=torch.float32, device=dev)
        g_op = torch.empty((P, 1), **opts); g_mean = torch.empty((P, 3), **opts); g_cov = torch.empty((P, 6), **opts)
        g_scale = torch.empty((P, 3), **opts); g_rot = torch.empty((P, 4), **opts)
        if getattr(R, "pending", None) is not None:
            R.resolve()
        R = _carved_capacity(binningBuffer, R)
        scratch = torch.empty(lib.r2x_voxel_bwd_scratch_bytes(int(R)), dtype=torch.uint8, device=dev)
        rc = lib.r2x_voxel_backward(
            torch.cuda.current_stream(dev).cuda_stream, P, int(R), int(nVoxel_x), int(nVoxel_y), int(nVoxel_z),
            float(sVoxel_x), float(sVoxel_y), float(sVoxel_z), float(center_x), float(center_y), float(center_z),
            _ptr(means3D), _ptr(scales), float(scale_modifier), _ptr(rotations), _ptr(cov3D_precomp), _ptr(radii_x),
            _ptr(radii_y), _ptr(radii_z), _ptr(geomBuffer), _ptr(binningBuffer), _ptr(imageBuffer),
            scratch.data_ptr(), _ptr(dL), _ptr(g_op), _ptr(g_mean), _ptr(g_cov), _ptr(g_scale), _ptr(g_rot),
            int(bool(debug)))
        check(rc, "r2x_voxel_backward")
    return g_op, g_mean, g_cov, g_scale, g_rot
