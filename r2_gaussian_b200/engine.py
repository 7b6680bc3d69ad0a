"""Persistent-workspace projector / voxelizer over the asynchronous C ABI.

`render()` / `query()` through the autograd wrappers follow the reference call for call (one host
round trip to size the binning buffer, fresh state buffers every call).  Throughput paths -- bench.py,
evaluation sweeps over many views, the Gaussian-sharded multi-GPU projector -- use these engines instead:
all state lives in buffers allocated once, the forward never synchronises with the host, and the
instance capacity is checked after the fact (`check()`), growing the workspace and re-running if a scene
ever needs more instances than provisioned.
"""
from __future__ import annotations

import torch

from . import _C
from ._lib import check, load


def _ptr(t):
    return None if t is None or t.numel() == 0 else t.data_ptr()


class _Engine:
    """State kept across calls and the capacity check shared by both engines; capacities follow `_C._Workspace`."""

    def __init__(self, kind, P: int, grid, device, capacity: int | None):
        self.lib = load()
        self.P = int(P)
        self.device = torch.device(device)
        with torch.cuda.device(self.device):
            self.geom, self.img = kind.state(self.P, grid, self.device)
            self.status = torch.zeros(2, dtype=torch.int32, device=self.device)
            self._reserve(capacity if capacity is not None else _C._Workspace.first(self.P, kind.seed))

    def _reserve(self, capacity: int):
        self.capacity = int(capacity)
        self.binning = _C.binning_buffer(self.capacity, self.device)

    def grow(self, R: int):
        """Re-provision the binning buffer for a forward that needed R instances."""
        self._reserve(_C._Workspace.grown(R))

    def num_rendered(self) -> int:
        """Synchronises; instance count of the last forward."""
        return int(self.status.cpu()[0].item())

    def check(self) -> bool:
        """Synchronises; True if the last forward fitted the capacity, else grows it (caller re-runs)."""
        R, ov = (int(v) for v in self.status.cpu().tolist())
        if ov:
            self.grow(R)
            return False
        return True

    def fit(self, *fwd_args, **fwd_kw):
        """Run forward until it fits.  Returns R."""
        while True:
            self.forward(*fwd_args, **fwd_kw)
            if self.check():
                break
        return self.num_rendered()


class RasterEngine(_Engine):
    """Forward X-ray projector for a fixed (P, W, H) with preallocated state."""

    def __init__(self, P: int, W: int, H: int, device="cuda", capacity: int | None = None):
        self.W, self.H = int(W), int(H)
        super().__init__(_C.RASTER, P, (self.W, self.H), device, capacity)
        self.radii = torch.empty(self.P, dtype=torch.int32, device=self.device)
        self.out = torch.empty((1, self.H, self.W), dtype=torch.float32, device=self.device)
        self._views = {}   # N -> (geom, image, radii[N,P], images[N,H,W]) of forward_views

    def forward(self, means, dens, scales, rots, viewmatrix, projmatrix, campos, tanfovx, tanfovy, mode,
                scale_modifier: float = 1.0, cov3D_precomp=None, out=None):
        """Enqueue one projection on the current stream; returns the [1,H,W] output tensor."""
        out = self.out if out is None else out
        rc = self.lib.r2x_raster_forward_async(
            torch.cuda.current_stream(self.device).cuda_stream, self.P, self.W, self.H, _ptr(means), _ptr(dens),
            _ptr(scales), float(scale_modifier), _ptr(rots), _ptr(cov3D_precomp), _ptr(viewmatrix), _ptr(projmatrix),
            _ptr(campos), float(tanfovx), float(tanfovy), 0, int(mode), out.data_ptr(), self.radii.data_ptr(),
            self.geom.data_ptr(), self.img.data_ptr(), self.binning.data_ptr(), self.capacity, self.status.data_ptr())
        check(rc, "r2x_raster_forward_async")
        return out

    def forward_views(self, means, dens, scales, rots, viewmatrices, projmatrices, tanfovx, tanfovy, mode,
                      scale_modifier: float = 1.0, out=None):
        """Enqueue the projections of N = len(viewmatrices) views in one batched call on the current stream; returns
        the [N,H,W] output (image v is bit for bit `forward` of view v).  The views' state buffers are kept per N; the
        binning buffer, its capacity and the status word are the engine's (`check()` / `grow()` as for `forward`)."""
        N = int(viewmatrices.shape[0])
        if N not in self._views:
            with torch.cuda.device(self.device):
                geom, img = _C.views_state(self.P, N, self.W, self.H, self.device)
                radii = torch.empty((N, self.P), dtype=torch.int32, device=self.device)
                images = torch.empty((N, self.H, self.W), dtype=torch.float32, device=self.device)
            self._views[N] = (geom, img, radii, images)
        geom, img, radii, images = self._views[N]
        out = images if out is None else out
        rc = self.lib.r2x_raster_forward_views_async(
            torch.cuda.current_stream(self.device).cuda_stream, self.P, N, self.W, self.H, _ptr(means), _ptr(dens),
            _ptr(scales), float(scale_modifier), _ptr(rots), _ptr(viewmatrices), _ptr(projmatrices), float(tanfovx),
            float(tanfovy), int(mode), out.data_ptr(), radii.data_ptr(), geom.data_ptr(), img.data_ptr(),
            self.binning.data_ptr(), self.capacity, self.status.data_ptr())
        check(rc, "r2x_raster_forward_views_async")
        return out

    def views_radii(self, N: int) -> torch.Tensor:
        """radii[N,P] of the last `forward_views` of N views."""
        return self._views[int(N)][2]

    def render_only(self, out=None):
        """Re-run only the per-tile accumulation kernel on the state of the last forward (profiling)."""
        out = self.out if out is None else out
        rc = self.lib.r2x_raster_render_only(torch.cuda.current_stream(self.device).cuda_stream, self.P, self.W, self.H,
                                             self.capacity, self.geom.data_ptr(), self.binning.data_ptr(),
                                             self.img.data_ptr(), out.data_ptr())
        check(rc, "r2x_raster_render_only")
        return out


class VoxelEngine(_Engine):
    """Forward density-volume query for a fixed (P, grid) with preallocated state."""

    def __init__(self, P: int, nVoxel, device="cuda", capacity: int | None = None):
        self.nx, self.ny, self.nz = (int(v) for v in nVoxel)
        super().__init__(_C.VOXEL, P, (self.nx, self.ny, self.nz), device, capacity)
        self.radii = torch.empty((3, self.P), dtype=torch.int32, device=self.device)
        self.out = torch.empty((self.nx, self.ny, self.nz), dtype=torch.float32, device=self.device)

    def forward(self, means, dens, scales, rots, sVoxel, center, scale_modifier: float = 1.0, cov3D_precomp=None,
                out=None):
        out = self.out if out is None else out
        rc = self.lib.r2x_voxel_forward_async(
            torch.cuda.current_stream(self.device).cuda_stream, self.P, self.nx, self.ny, self.nz, float(sVoxel[0]),
            float(sVoxel[1]), float(sVoxel[2]), float(center[0]), float(center[1]), float(center[2]), _ptr(means),
            _ptr(dens), _ptr(scales), float(scale_modifier), _ptr(rots), _ptr(cov3D_precomp), 0, out.data_ptr(),
            self.radii[0].data_ptr(), self.radii[1].data_ptr(), self.radii[2].data_ptr(), self.geom.data_ptr(),
            self.img.data_ptr(), self.binning.data_ptr(), self.capacity, self.status.data_ptr())
        check(rc, "r2x_voxel_forward_async")
        return out

    def render_only(self, out=None):
        out = self.out if out is None else out
        rc = self.lib.r2x_voxel_render_only(torch.cuda.current_stream(self.device).cuda_stream, self.P, self.nx, self.ny,
                                            self.nz, self.capacity, self.geom.data_ptr(), self.binning.data_ptr(),
                                            self.img.data_ptr(), out.data_ptr())
        check(rc, "r2x_voxel_render_only")
        return out


class HostProjector:
    """Projection service over HOST buffers: pinned host parameters in, pinned host image out.

    `project()` is the strict call (upload -> 4 kernels -> download -> wait).  `submit()` / `wait()` pipeline
    consecutive projections: the upload of request i+1 and the download of image i-1 run on their own streams
    while request i computes (device inputs / outputs are ring-buffered `depth` deep; one RasterEngine, so the
    kernels themselves stay in order).  The instance-capacity status of every request travels back with its
    image; `wait()` re-runs a request synchronously with a larger workspace if it had overflowed.
    """

    def __init__(self, P: int, W: int, H: int, device="cuda", depth: int = 3, capacity: int | None = None):
        self.engine = RasterEngine(P, W, H, device, capacity)
        self.device = self.engine.device
        self.depth = int(depth)
        dev, f32 = self.device, torch.float32
        with torch.cuda.device(dev):
            mk = lambda *s: [torch.empty(s, dtype=f32, device=dev) for _ in range(self.depth)]
            self.d_means, self.d_dens, self.d_scales, self.d_rots = mk(P, 3), mk(P, 1), mk(P, 3), mk(P, 4)
            self.d_view, self.d_proj, self.d_campos = mk(4, 4), mk(4, 4), mk(3)
            self.d_out = mk(1, H, W)
            self.d_status = [torch.zeros(2, dtype=torch.int32, device=dev) for _ in range(self.depth)]
            self.h_status = [torch.zeros(2, dtype=torch.int32).pin_memory() for _ in range(self.depth)]
            self.s_in, self.s_out = torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev)
            self.s_compute = torch.cuda.Stream(device=dev)
            ev = lambda: [torch.cuda.Event() for _ in range(self.depth)]
            self.e_in, self.e_comp, self.e_out = ev(), ev(), ev()
        self._n = 0
        self._pending = {}

    def submit(self, h_means, h_dens, h_scales, h_rots, h_view, h_proj, h_campos, tanfovx, tanfovy, mode, h_out):
        """Enqueue one projection; returns a ticket for wait().  All host tensors should be pinned."""
        k = self._n % self.depth
        ticket = self._n
        self._n += 1
        if ticket - self.depth in self._pending:      # the ring slot is still owned by an unfinished request
            self.wait(ticket - self.depth)
        with torch.cuda.stream(self.s_in):
            if ticket >= self.depth:
                self.s_in.wait_event(self.e_comp[k])      # slot inputs free once the previous user computed
            for d, h in ((self.d_means, h_means), (self.d_dens, h_dens), (self.d_scales, h_scales), (self.d_rots, h_rots),
                         (self.d_view, h_view), (self.d_proj, h_proj), (self.d_campos, h_campos)):
                d[k].copy_(h.view_as(d[k]), non_blocking=True)
            self.e_in[k].record(self.s_in)
        with torch.cuda.stream(self.s_compute):
            self.s_compute.wait_event(self.e_in[k])
            if ticket >= self.depth:
                self.s_compute.wait_event(self.e_out[k])  # slot output free once its previous image went home
            self.engine.forward(self.d_means[k], self.d_dens[k], self.d_scales[k], self.d_rots[k], self.d_view[k],
                                self.d_proj[k], self.d_campos[k], tanfovx, tanfovy, mode, out=self.d_out[k])
            self.d_status[k].copy_(self.engine.status, non_blocking=True)
            self.e_comp[k].record(self.s_compute)
        with torch.cuda.stream(self.s_out):
            self.s_out.wait_event(self.e_comp[k])
            h_out.copy_(self.d_out[k].view_as(h_out), non_blocking=True)
            self.h_status[k].copy_(self.d_status[k], non_blocking=True)
            self.e_out[k].record(self.s_out)
        self._pending[ticket] = (k, (h_means, h_dens, h_scales, h_rots, h_view, h_proj, h_campos, tanfovx, tanfovy, mode,
                                     h_out))
        return ticket

    def wait(self, ticket):
        k, req = self._pending.pop(ticket)
        self.e_out[k].synchronize()
        if int(self.h_status[k][1]) != 0:              # capacity overflow: grow and redo this request, in order
            torch.cuda.synchronize(self.device)
            self.engine.grow(int(self.h_status[k][0]))
            t = self.submit(*req)
            return self.wait(t)
        return req[-1]

    def project(self, *request):
        return self.wait(self.submit(*request))

    def drain(self):
        for t in sorted(self._pending):
            self.wait(t)
