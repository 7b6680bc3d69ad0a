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


def _u8(nbytes: int, dev) -> torch.Tensor:
    return torch.empty(int(nbytes), dtype=torch.uint8, device=dev)


class _Kind:
    """What the rasterizer's and the voxelizer's forward state differ in: the library's size functions, and `seed`,
    the instances per Gaussian provisioned for a shape that has no capacity hint yet."""

    def __init__(self, name: str, seed: int):
        self.name, self.seed = name, seed

    def state(self, P: int, grid, dev) -> tuple[torch.Tensor, torch.Tensor]:
        """(geom, image) buffers of one forward over `grid`: (W, H) for raster, (nx, ny, nz) for voxel."""
        lib = load()
        return (_u8(getattr(lib, f"r2x_{self.name}_geom_bytes")(P), dev),
                _u8(getattr(lib, f"r2x_{self.name}_image_bytes")(P, *grid), dev))

    def bwd_scratch(self, capacity: int, dev) -> torch.Tensor:
        """Scratch of a backward over a binning buffer carved for `capacity` instances."""
        return _u8(getattr(load(), f"r2x_{self.name}_bwd_scratch_bytes")(capacity), dev)


RASTER, VOXEL = _Kind("raster", 12), _Kind("voxel", 8)


def binning_buffer(capacity: int, dev) -> torch.Tensor:
    """Binning buffer for `capacity` (Gaussian, tile) instances (the same layout for both kinds)."""
    return _u8(load().r2x_binning_bytes(capacity), dev)


def raster_key(dev: torch.device, P: int, W: int, H: int) -> tuple:
    """Capacity-hint key of a raster shape (`dev` with its index, as a CUDA tensor's device has)."""
    return ("raster", dev.index, int(P), int(W), int(H))


def voxel_key(dev: torch.device, P: int, nx: int, ny: int, nz: int, sVoxel_x: float) -> tuple:
    """Capacity-hint key of a voxel shape: the instance count depends strongly on the voxel pitch, so it is part of it."""
    return ("voxel", dev.index, int(P), int(nx), int(ny), int(nz), round(float(sVoxel_x) / int(nx), 6))


class _Workspace:
    """The instance capacity of the binning buffer, decided here for every caller in the package.

    Per-shape hints (keys from `raster_key` / `voxel_key`) let the binning buffer be provisioned BEFORE the forward
    runs: the whole pipeline is then enqueued without a host round trip in the middle, and the one synchronisation the
    reference API needs anyway (num_rendered is a Python int) happens at the end.  If a call needs more instances than
    provisioned it is simply re-run with a larger buffer.  Capacities are rounded to a coarse grid so that torch's
    caching allocator sees repeating sizes."""

    hints: dict = {}
    _pinned: list = []

    @staticmethod
    def _round(n: int) -> int:
        step = 1 << max(12, int(n).bit_length() - 3)   # ~12.5 % granularity
        return (int(n) + step - 1) // step * step

    @classmethod
    def first(cls, P: int, seed: int) -> int:
        """Capacity for a shape without a hint: `seed` instances per Gaussian, at least 16384."""
        return cls._round(max(seed * P, 1 << 14))

    @classmethod
    def grown(cls, R: int) -> int:
        """Capacity for a forward that needed R instances: 20 % headroom plus 1024."""
        return cls._round(int(R * 1.2) + 1024)

    @classmethod
    def provision(cls, key, P: int, seed: int, speculative: bool = False) -> int:
        cap = cls.hints.get(key) or cls.first(P, seed)
        if speculative:     # generous: an overflow needs the instance count to double between two calls of this shape
            cap = cls._round(max(2 * cap, seed * P))
        return cap

    @classmethod
    def update(cls, key, R: int):
        want = cls.grown(R)
        cur = cls.hints.get(key, 0)
        # grow immediately, shrink slowly (keeps sizes stable while the cloud changes during training)
        cls.hints[key] = want if want > cur or want < cur // 2 else cur

    @classmethod
    def to_host(cls, status: torch.Tensor) -> torch.Tensor:
        """Start copying the device status word {R, overflow} to pinned host memory (no host wait).  Record an event
        after this call and `read` the returned tensor once the event has completed."""
        host = cls._pinned.pop() if cls._pinned else torch.zeros(2, dtype=torch.int32).pin_memory()
        host.copy_(status, non_blocking=True)
        return host

    @classmethod
    def read(cls, host: torch.Tensor, key) -> tuple[int, int]:
        """-> (R, overflow) of a status word from `to_host`; updates the hint of `key` and returns `host` to the pool."""
        R, overflow = int(host[0]), int(host[1])
        cls.update(key, R)
        if len(cls._pinned) < 16:
            cls._pinned.append(host)
        return R, overflow


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
        self.pending = None
        R, overflow = _Workspace.read(host, key)
        if overflow:
            raise CapacityOverflow(f"forward needed {R} instances, binning buffer provisioned for {self.capacity}; "
                                   "the capacity hint has been raised -- repeat the iteration")
        return R


class speculative:
    """Context manager used by the autograd bridges in training mode: inside it the forward entry points do NOT
    synchronise with the host (the one sync of the reference API, `num_rendered` being a Python int, is what
    serialises host and device twice per training iteration).  `_forward` provisions the binning buffer from the
    instance count of the previous call with the same shape (`_Workspace.provision`), the status word travels to pinned
    host memory behind an event, and the check happens in the backward.  Disabled by R2X_SPECULATIVE=0 (read by
    `active()` only), by debug=True, under no_grad, and for the first call of a shape (no hint yet)."""

    _tls = threading.local()

    def __init__(self, on: bool = True):
        self.on = bool(on)

    def __enter__(self):
        self.prev = getattr(self._tls, "on", False)
        self._tls.on = self.on
        return self

    def __exit__(self, *exc):
        self._tls.on = self.prev
        return False

    @classmethod
    def active(cls) -> bool:
        return bool(getattr(cls._tls, "on", False)) and os.environ.get("R2X_SPECULATIVE", "1") != "0"


def _forward(launch, key, P: int, seed: int, dev) -> tuple[NumRendered, torch.Tensor]:
    """Run one asynchronous forward; `launch(binning, capacity, status)` enqueues it.  -> (NumRendered, binning).

    Inside `speculative`, once the shape has a hint, the call returns at once: the status word travels to pinned host
    memory behind an event and `NumRendered.resolve()` reads it.  Otherwise the status is read here (the one host
    synchronisation of the call) and the forward is re-run with the raised hint until it fits."""
    spec = speculative.active() and key in _Workspace.hints
    cap = _Workspace.provision(key, P, seed, spec)
    status = torch.empty(2, dtype=torch.int32, device=dev)
    while True:
        binning = binning_buffer(cap, dev)
        launch(binning, cap, status)
        if spec:
            host = _Workspace.to_host(status)
            event = torch.cuda.Event()
            event.record(torch.cuda.current_stream(dev))
            return NumRendered(cap, cap, (host, event, key)), binning
        R, overflow = status.tolist()
        _Workspace.update(key, R)
        if not overflow:
            return NumRendered(R, cap), binning
        cap = _Workspace.provision(key, P, seed)


def _carved_capacity(binning: torch.Tensor, R) -> int:
    """Backward prologue: resolve a pending `num_rendered` (raises CapacityOverflow if its speculative forward did not
    fit), then return the instance count `binning` was carved for, which the backward must carve with.  The count
    travels with R (`NumRendered.capacity`); the buffer itself is not read."""
    if getattr(R, "pending", None) is not None:
        R.resolve()
    return int(getattr(R, "capacity", R))


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
        out_color = torch.empty((1, H, W), dtype=torch.float32, device=dev)
        radii = torch.empty((P,), dtype=torch.int32, device=dev)
        geom, img = RASTER.state(P, (W, H), dev)
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

        def launch(binning, cap, status):
            rc = lib.r2x_raster_forward_async(
                stream, P, W, H, _ptr(means3D), _ptr(opacity), _ptr(scales), float(scale_modifier), _ptr(rotations),
                _ptr(cov3D_precomp), _ptr(viewmatrix), _ptr(projmatrix), _ptr(campos), float(tan_fovx), float(tan_fovy),
                int(bool(prefiltered)), int(mode), out_color.data_ptr(), _ptr(radii), geom.data_ptr(), img.data_ptr(),
                binning.data_ptr(), cap, status.data_ptr())
            check(rc, "r2x_raster_forward_async")

        R, binning = _forward(launch, raster_key(dev, P, W, H), P, RASTER.seed, dev)
    return R, out_color, radii, geom, binning, img


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
        R = _carved_capacity(binningBuffer, R)
        scratch = RASTER.bwd_scratch(R, dev)
        rc = lib.r2x_raster_backward(
            torch.cuda.current_stream(dev).cuda_stream, P, R, W, H, _ptr(means3D), _ptr(scales),
            float(scale_modifier), _ptr(rotations), _ptr(cov3D_precomp), _ptr(viewmatrix), _ptr(projmatrix),
            _ptr(campos), float(tan_fovx), float(tan_fovy), _ptr(radii), _ptr(geomBuffer), _ptr(binningBuffer),
            _ptr(imageBuffer), scratch.data_ptr(), _ptr(dL), _ptr(g_mean2D), _ptr(g_op), _ptr(g_mu),
            _ptr(g_mean3D), _ptr(g_cov), _ptr(g_scale), _ptr(g_rot), int(mode), int(bool(debug)))
        check(rc, "r2x_raster_backward")
    return g_mean2D, g_op, g_mu, g_mean3D, g_cov, g_scale, g_rot


def rasterize_gaussians_backward_matrices(means3D, radii, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix,
                                          projmatrix, tan_fovx, tan_fovy, dL_dout_color, campos, geomBuffer, R,
                                          binningBuffer, imageBuffer, mode, debug, act=None):
    """`rasterize_gaussians_backward` that also returns the gradients with respect to the two matrices ->
    (dL_dmeans2D, dL_dopacity, dL_dmu, dL_dmeans3D, dL_dcov3D, dL_dscales, dL_drotations, dL_dviewmatrix[4,4],
    dL_dprojmatrix[4,4]).  With `act` (an `ActivationDesc`) scales / rotations are the raw parameters and dL_dopacity
    is the raw density gradient (dL_dmu is then None), as `fused` passes them.  The matrix gradients are laid out like
    the matrices (element [i, j] is dL / d matrix[i, j])."""
    _require_cuda(means3D, "means3D")
    lib = load()
    dev = means3D.device
    P = int(means3D.shape[0])
    H, W = int(dL_dout_color.shape[-2]), int(dL_dout_color.shape[-1])
    with torch.cuda.device(dev):
        means3D = _f32(means3D, dev); scales = _f32(scales, dev); rotations = _f32(rotations, dev)
        cov3D_precomp = None if cov3D_precomp is None else _f32(cov3D_precomp, dev)
        viewmatrix = _f32(viewmatrix, dev); projmatrix = _f32(projmatrix, dev); campos = _f32(campos, dev)
        dL = _f32(dL_dout_color, dev)
        opts = dict(dtype=torch.float32, device=dev)
        g_mean2D = torch.empty((P, 3), **opts); g_op = torch.empty((P, 1), **opts)
        g_mu = torch.empty((P, 1), **opts) if act is None else None
        g_mean3D = torch.empty((P, 3), **opts); g_cov = torch.empty((P, 6), **opts)
        g_scale = torch.empty((P, 3), **opts); g_rot = torch.empty((P, 4), **opts)
        g_view = torch.empty((4, 4), **opts); g_proj = torch.empty((4, 4), **opts)
        R = _carved_capacity(binningBuffer, R)
        scratch = RASTER.bwd_scratch(R, dev)
        pose_bytes = lib.r2x_raster_backward_pose_scratch_bytes(P)
        pose_scratch = _u8(pose_bytes, dev)
        rc = lib.r2x_raster_backward_pose(
            torch.cuda.current_stream(dev).cuda_stream, P, R, W, H, _ptr(means3D), _ptr(scales),
            float(scale_modifier), _ptr(rotations), _ptr(cov3D_precomp), _ptr(viewmatrix), _ptr(projmatrix),
            _ptr(campos), float(tan_fovx), float(tan_fovy), _ptr(radii), _ptr(geomBuffer), _ptr(binningBuffer),
            _ptr(imageBuffer), scratch.data_ptr(), _ptr(dL), _ptr(g_mean2D), _ptr(g_op), _ptr(g_mu),
            _ptr(g_mean3D), _ptr(g_cov), _ptr(g_scale), _ptr(g_rot), int(mode), int(bool(debug)),
            None if act is None else C.byref(act), g_view.data_ptr(), g_proj.data_ptr(), pose_scratch.data_ptr(),
            pose_bytes)
        check(rc, "r2x_raster_backward_pose")
    return g_mean2D, g_op, g_mu, g_mean3D, g_cov, g_scale, g_rot, g_view, g_proj


def views_key(dev: torch.device, P: int, N: int, W: int, H: int) -> tuple:
    """Capacity-hint key of a batched-views shape (its instance count is the sum over the N views)."""
    return ("raster_views", dev.index, int(P), int(N), int(W), int(H))


def views_state(P: int, N: int, W: int, H: int, dev) -> tuple[torch.Tensor, torch.Tensor]:
    """(geom, image) buffers of one batched forward of N views."""
    lib = load()
    return _u8(lib.r2x_raster_views_geom_bytes(P, N), dev), _u8(lib.r2x_raster_views_image_bytes(P, N, W, H), dev)


def check_views_args(means3D, viewmatrices, projmatrices) -> int:
    """Shape checks of a batched-views call (no CUDA call) -> N."""
    if means3D.ndim != 2 or means3D.shape[1] != 3:
        raise ValueError("means3D must have dimensions (num_points, 3)")
    if viewmatrices.ndim != 3 or tuple(viewmatrices.shape[1:]) != (4, 4) or viewmatrices.shape[0] < 1:
        raise ValueError(f"viewmatrices must have dimensions (N >= 1, 4, 4), got {tuple(viewmatrices.shape)}")
    if tuple(projmatrices.shape) != tuple(viewmatrices.shape):
        raise ValueError(f"projmatrices {tuple(projmatrices.shape)} must match viewmatrices {tuple(viewmatrices.shape)}")
    return int(viewmatrices.shape[0])


def rasterize_views(means3D, opacity, scales, rotations, scale_modifier, viewmatrices, projmatrices, tan_fovx, tan_fovy,
                    image_height, image_width, mode, act=None):
    """N views of one cloud in one call -> (num_rendered, images[N,H,W], radii[N,P] int32, geom, binning, img).

    Image v and radii[v] are bit for bit what `rasterize_gaussians` computes for view v alone.  num_rendered (summed
    over the views) is a `NumRendered` carrying the binning buffer's capacity, with the same overflow handling as the
    single-view call.  With `act` (an `ActivationDesc`) opacity / scales / rotations are the RAW parameters
    (`rasterize_views_raw`)."""
    N = check_views_args(means3D, viewmatrices, projmatrices)
    for t, name in ((means3D, "means3D"), (viewmatrices, "viewmatrices"), (projmatrices, "projmatrices")):
        _require_cuda(t, name)
    lib = load()
    dev = means3D.device
    P, H, W = int(means3D.shape[0]), int(image_height), int(image_width)
    with torch.cuda.device(dev):
        means3D = _f32(means3D, dev); opacity = _f32(opacity, dev)
        scales = _f32(scales, dev); rotations = _f32(rotations, dev)
        viewmatrices = _f32(viewmatrices, dev); projmatrices = _f32(projmatrices, dev)
        images = torch.empty((N, H, W), dtype=torch.float32, device=dev)
        radii = torch.empty((N, P), dtype=torch.int32, device=dev)
        geom, img = views_state(P, N, W, H, dev)
        stream = torch.cuda.current_stream(dev).cuda_stream

        def launch(binning, cap, status):
            args = (stream, P, N, W, H, _ptr(means3D), _ptr(opacity), _ptr(scales), float(scale_modifier),
                    _ptr(rotations), _ptr(viewmatrices), _ptr(projmatrices), float(tan_fovx), float(tan_fovy), int(mode),
                    images.data_ptr(), _ptr(radii), geom.data_ptr(), img.data_ptr(), binning.data_ptr(), cap,
                    status.data_ptr())
            if act is None:
                check(lib.r2x_raster_forward_views_async(*args), "r2x_raster_forward_views_async")
            else:
                check(lib.r2x_raster_forward_views_async_raw(*args, C.byref(act)), "r2x_raster_forward_views_async_raw")

        R, binning = _forward(launch, views_key(dev, P, N, W, H), P * N, RASTER.seed, dev)
    return R, images, radii, geom, binning, img


def rasterize_views_backward(means3D, radii, scales, rotations, scale_modifier, viewmatrices, projmatrices, tan_fovx,
                             tan_fovy, dL_dimages, geomBuffer, R, binningBuffer, imageBuffer, mode, debug=False, act=None):
    """-> (dL_dmeans2D[N,P,3] per view, dL_dopacity[P,1], dL_dmeans3D[P,3], dL_dcov3D[P,6], dL_dscales[P,3],
    dL_drotations[P,4]); the per-Gaussian gradients are summed over the views in view order (float32).  With `act`
    scales / rotations are the raw parameters and the gradients are those of the raw density / scales / rotations
    (`rasterize_views_raw_backward`)."""
    N = check_views_args(means3D, viewmatrices, projmatrices)
    _require_cuda(means3D, "means3D")
    lib = load()
    dev = means3D.device
    P = int(means3D.shape[0])
    H, W = int(dL_dimages.shape[-2]), int(dL_dimages.shape[-1])
    with torch.cuda.device(dev):
        means3D = _f32(means3D, dev); scales = _f32(scales, dev); rotations = _f32(rotations, dev)
        viewmatrices = _f32(viewmatrices, dev); projmatrices = _f32(projmatrices, dev); dL = _f32(dL_dimages, dev)
        opts = dict(dtype=torch.float32, device=dev)
        g_mean2D = torch.empty((N, P, 3), **opts); g_op = torch.empty((P, 1), **opts)
        g_mean3D = torch.empty((P, 3), **opts); g_cov = torch.empty((P, 6), **opts)
        g_scale = torch.empty((P, 3), **opts); g_rot = torch.empty((P, 4), **opts)
        R = _carved_capacity(binningBuffer, R)
        scratch = RASTER.bwd_scratch(R, dev)
        args = (torch.cuda.current_stream(dev).cuda_stream, P, N, R, W, H, _ptr(means3D), _ptr(scales),
                float(scale_modifier), _ptr(rotations), _ptr(viewmatrices), _ptr(projmatrices), float(tan_fovx),
                float(tan_fovy), _ptr(radii), _ptr(geomBuffer), _ptr(binningBuffer), _ptr(imageBuffer),
                scratch.data_ptr(), _ptr(dL), _ptr(g_mean2D), _ptr(g_op), _ptr(g_mean3D), _ptr(g_cov), _ptr(g_scale),
                _ptr(g_rot), int(mode))
        if act is None:
            check(lib.r2x_raster_backward_views(*args, int(bool(debug))), "r2x_raster_backward_views")
        else:
            check(lib.r2x_raster_backward_views_raw(*args, C.byref(act)), "r2x_raster_backward_views_raw")
    return g_mean2D, g_op, g_mean3D, g_cov, g_scale, g_rot


def rasterize_views_raw(means3D, raw_density, raw_scales, raw_rotations, scale_modifier, viewmatrices, projmatrices,
                        tan_fovx, tan_fovy, image_height, image_width, mode, act):
    """`rasterize_views` on the RAW parameters (the activations of `act`, an `ActivationDesc`, run in the kernels):
    image v and radii[v] are bit for bit the single-view raw render (`fused.rasterize_raw`) of view v."""
    return rasterize_views(means3D, raw_density, raw_scales, raw_rotations, scale_modifier, viewmatrices, projmatrices,
                           tan_fovx, tan_fovy, image_height, image_width, mode, act=act)


def rasterize_views_raw_backward(means3D, radii, raw_scales, raw_rotations, scale_modifier, viewmatrices, projmatrices,
                                 tan_fovx, tan_fovy, dL_dimages, geomBuffer, R, binningBuffer, imageBuffer, mode, act):
    """-> (dL_dmeans2D[N,P,3] per view, dL_draw_density[P,1], dL_dmeans3D[P,3], dL_dcov3D[P,6], dL_draw_scales[P,3],
    dL_draw_rotations[P,4]): each gradient is the view-order float32 sum of the single-view raw backward's."""
    return rasterize_views_backward(means3D, radii, raw_scales, raw_rotations, scale_modifier, viewmatrices,
                                    projmatrices, tan_fovx, tan_fovy, dL_dimages, geomBuffer, R, binningBuffer,
                                    imageBuffer, mode, act=act)


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
        vol = torch.empty((nx, ny, nz), dtype=torch.float32, device=dev)
        rx = torch.empty((P,), dtype=torch.int32, device=dev)
        ry = torch.empty_like(rx); rz = torch.empty_like(rx)
        geom, img = VOXEL.state(P, (nx, ny, nz), dev)
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

        def launch(binning, cap, status):
            rc = lib.r2x_voxel_forward_async(stream, P, *grid_args, *in_args, vol.data_ptr(), _ptr(rx), _ptr(ry),
                                             _ptr(rz), geom.data_ptr(), img.data_ptr(), binning.data_ptr(), cap,
                                             status.data_ptr())
            check(rc, "r2x_voxel_forward_async")

        R, binning = _forward(launch, voxel_key(dev, P, nx, ny, nz, sVoxel_x), P, VOXEL.seed, dev)
    return R, vol, rx, ry, rz, geom, binning, img


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
        R = _carved_capacity(binningBuffer, R)
        scratch = VOXEL.bwd_scratch(R, dev)
        rc = lib.r2x_voxel_backward(
            torch.cuda.current_stream(dev).cuda_stream, P, R, int(nVoxel_x), int(nVoxel_y), int(nVoxel_z),
            float(sVoxel_x), float(sVoxel_y), float(sVoxel_z), float(center_x), float(center_y), float(center_z),
            _ptr(means3D), _ptr(scales), float(scale_modifier), _ptr(rotations), _ptr(cov3D_precomp), _ptr(radii_x),
            _ptr(radii_y), _ptr(radii_z), _ptr(geomBuffer), _ptr(binningBuffer), _ptr(imageBuffer),
            scratch.data_ptr(), _ptr(dL), _ptr(g_op), _ptr(g_mean), _ptr(g_cov), _ptr(g_scale), _ptr(g_rot),
            int(bool(debug)))
        check(rc, "r2x_voxel_backward")
    return g_op, g_mean, g_cov, g_scale, g_rot
