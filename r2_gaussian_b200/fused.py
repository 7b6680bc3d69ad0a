"""render() / query() on RAW parameters: the activations (softplus, bounded sigmoid / exp, normalize) run inside the
preprocess kernels and the per-Gaussian backward kernels return gradients with respect to the raw parameters
(libr2xray: r2x_*_raw, SURVEY 8(f) rank 2).  The reference applies them as six small torch kernels per iteration and
differentiates through them with autograd (`r2_gaussian/gaussian/gaussian_model.py:112-126`).

Used by `render_query.render/query` when the model offers `raw_parameters()` (this repository's GaussianModel) and
`R2X_FUSED_ACTIVATIONS` is not 0; models that only expose `get_density / get_scaling / get_rotation` (e.g. the
reference's own class) keep the plain path.  Training mode only has the speculative forward (no host synchronisation;
`_C.speculative`), evaluation synchronises like the plain path.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

from . import _C
from ._lib import ActivationDesc, check, load


def enabled() -> bool:
    return os.environ.get("R2X_FUSED_ACTIVATIONS", "1") != "0"


def _act(params) -> ActivationDesc:
    a = ActivationDesc()
    bound = params.get("scale_bound")
    if bound is None:
        a.scale_mode, a.scale_lo, a.scale_hi = 0, 0.0, 0.0
    else:
        a.scale_mode, a.scale_lo, a.scale_hi = 1, float(bound[0]), float(bound[1])
    return a


class _RasterizeRaw(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, raw_density, raw_scales, raw_rotations, settings, act):
        lib = load()
        s = settings
        dev = means3D.device
        P, H, W = int(means3D.shape[0]), int(s.image_height), int(s.image_width)
        f = lambda t: _C._f32(t, dev)
        means3D, raw_density, raw_scales, raw_rotations = f(means3D), f(raw_density), f(raw_scales), f(raw_rotations)
        view, proj, campos = f(s.viewmatrix), f(s.projmatrix), f(s.campos)
        with torch.cuda.device(dev), _C.speculative(any(ctx.needs_input_grad)):
            color = torch.empty((1, H, W), dtype=torch.float32, device=dev)
            radii = torch.empty((P,), dtype=torch.int32, device=dev)
            geom, img = _C.RASTER.state(P, (W, H), dev)
            stream = torch.cuda.current_stream(dev).cuda_stream

            def run(binning, cap, status):
                rc = lib.r2x_raster_forward_async_raw(
                    stream, P, W, H, _C._ptr(means3D), _C._ptr(raw_density), _C._ptr(raw_scales), float(s.scale_modifier),
                    _C._ptr(raw_rotations), _C._ptr(view), _C._ptr(proj), _C._ptr(campos), float(s.tanfovx), float(s.tanfovy),
                    int(s.mode), color.data_ptr(), _C._ptr(radii), geom.data_ptr(), img.data_ptr(), binning.data_ptr(), cap,
                    status.data_ptr(), C.byref(act))
                check(rc, "r2x_raster_forward_async_raw")

            R, binning = _C._forward(run, _C.raster_key(dev, P, W, H), P, _C.RASTER.seed, dev)
        ctx.settings, ctx.act, ctx.num_rendered = s, act, R
        ctx.save_for_backward(means3D, raw_scales, raw_rotations, radii, geom, binning, img, view, proj, campos)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, grad_color, _grad_radii):
        lib = load()
        s, act, R = ctx.settings, ctx.act, ctx.num_rendered
        means3D, raw_scales, raw_rotations, radii, geom, binning, img, view, proj, campos = ctx.saved_tensors
        cap = _C._carved_capacity(binning, R)
        dev = means3D.device
        P, H, W = int(means3D.shape[0]), int(s.image_height), int(s.image_width)
        with torch.cuda.device(dev):
            opts = dict(dtype=torch.float32, device=dev)
            g2 = torch.empty((P, 3), **opts); gd = torch.empty((P, 1), **opts); g3 = torch.empty((P, 3), **opts)
            gcov = torch.empty((P, 6), **opts); gs = torch.empty((P, 3), **opts); gr = torch.empty((P, 4), **opts)
            scratch = _C.RASTER.bwd_scratch(cap, dev)
            dL = _C._f32(grad_color, dev)
            rc = lib.r2x_raster_backward_raw(
                torch.cuda.current_stream(dev).cuda_stream, P, cap, W, H, _C._ptr(means3D), _C._ptr(raw_scales),
                float(s.scale_modifier), _C._ptr(raw_rotations), _C._ptr(view), _C._ptr(proj), _C._ptr(campos),
                float(s.tanfovx), float(s.tanfovy), _C._ptr(radii), _C._ptr(geom), _C._ptr(binning), _C._ptr(img),
                scratch.data_ptr(), _C._ptr(dL), _C._ptr(g2), _C._ptr(gd), _C._ptr(g3), _C._ptr(gcov), _C._ptr(gs), _C._ptr(gr),
                int(s.mode), C.byref(act))
            check(rc, "r2x_raster_backward_raw")
        return g3, g2, gd, gs, gr, None, None


class _RasterizeRawMatrices(torch.autograd.Function):
    """`_RasterizeRaw` with the view and projection matrices as differentiable inputs (the settings' own are ignored)."""

    @staticmethod
    def forward(ctx, means3D, means2D, raw_density, raw_scales, raw_rotations, viewmatrix, projmatrix, settings, act):
        s = settings._replace(viewmatrix=viewmatrix.detach(), projmatrix=projmatrix.detach())
        ctx.matrix_dtypes = (viewmatrix.dtype, projmatrix.dtype)
        return _RasterizeRaw.forward(ctx, means3D, means2D, raw_density, raw_scales, raw_rotations, s, act)

    @staticmethod
    def backward(ctx, grad_color, _grad_radii):
        s, act, R = ctx.settings, ctx.act, ctx.num_rendered
        means3D, raw_scales, raw_rotations, radii, geom, binning, img, view, proj, campos = ctx.saved_tensors
        g2, gd, _, g3, _gcov, gs, gr, gv, gp = _C.rasterize_gaussians_backward_matrices(
            means3D, radii, raw_scales, raw_rotations, s.scale_modifier, None, view, proj, s.tanfovx, s.tanfovy,
            grad_color, campos, geom, R, binning, img, s.mode, False, act=act)
        gv = gv.view(s.viewmatrix.shape).to(ctx.matrix_dtypes[0])
        gp = gp.view(s.projmatrix.shape).to(ctx.matrix_dtypes[1])
        return g3, g2, gd, gs, gr, gv, gp, None, None


class _RasterizeViewsRaw(torch.autograd.Function):
    """`_RasterizeRaw` for N views of one cloud in one native call: forward inputs (means3D, means2D[N,P,3], raw_density,
    raw_scales, raw_rotations, viewmatrices[N,4,4], projmatrices[N,4,4], settings, act) -> (images[N,H,W], radii[N,P]);
    the settings' own matrices are ignored.  The backward sums the raw gradients over the views in view order and hands
    means2D the per-view screen-space gradients."""

    @staticmethod
    def forward(ctx, means3D, means2D, raw_density, raw_scales, raw_rotations, viewmatrices, projmatrices, settings, act):
        s = settings
        with _C.speculative(any(ctx.needs_input_grad)):
            R, images, radii, geom, binning, img = _C.rasterize_views_raw(
                means3D, raw_density, raw_scales, raw_rotations, s.scale_modifier, viewmatrices, projmatrices, s.tanfovx,
                s.tanfovy, s.image_height, s.image_width, s.mode, act)
        ctx.settings, ctx.act, ctx.num_rendered = s, act, R
        ctx.save_for_backward(means3D, raw_scales, raw_rotations, viewmatrices, projmatrices, radii, geom, binning, img)
        ctx.mark_non_differentiable(radii)
        return images, radii

    @staticmethod
    def backward(ctx, grad_images, _grad_radii):
        s, act = ctx.settings, ctx.act
        means3D, raw_scales, raw_rotations, viewmatrices, projmatrices, radii, geom, binning, img = ctx.saved_tensors
        g2, gd, g3, _gcov, gs, gr = _C.rasterize_views_raw_backward(
            means3D, radii, raw_scales, raw_rotations, s.scale_modifier, viewmatrices, projmatrices, s.tanfovx,
            s.tanfovy, grad_images, geom, ctx.num_rendered, binning, img, s.mode, act)
        return g3, g2, gd, gs, gr, None, None, None, None


class _VoxelizeRaw(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, raw_density, raw_scales, raw_rotations, settings, act):
        lib = load()
        s = settings
        dev = means3D.device
        P = int(means3D.shape[0])
        nx, ny, nz = int(s.nVoxel_x), int(s.nVoxel_y), int(s.nVoxel_z)
        f = lambda t: _C._f32(t, dev)
        means3D, raw_density, raw_scales, raw_rotations = f(means3D), f(raw_density), f(raw_scales), f(raw_rotations)
        grid = (nx, ny, nz, float(s.sVoxel_x), float(s.sVoxel_y), float(s.sVoxel_z), float(s.center_x), float(s.center_y),
                float(s.center_z))
        with torch.cuda.device(dev), _C.speculative(any(ctx.needs_input_grad)):
            vol = torch.empty((nx, ny, nz), dtype=torch.float32, device=dev)
            rx = torch.empty((P,), dtype=torch.int32, device=dev); ry = torch.empty_like(rx); rz = torch.empty_like(rx)
            geom, img = _C.VOXEL.state(P, (nx, ny, nz), dev)
            stream = torch.cuda.current_stream(dev).cuda_stream

            def run(binning, cap, status):
                rc = lib.r2x_voxel_forward_async_raw(
                    stream, P, *grid, _C._ptr(means3D), _C._ptr(raw_density), _C._ptr(raw_scales), float(s.scale_modifier),
                    _C._ptr(raw_rotations), vol.data_ptr(), _C._ptr(rx), _C._ptr(ry), _C._ptr(rz), geom.data_ptr(),
                    img.data_ptr(), binning.data_ptr(), cap, status.data_ptr(), C.byref(act))
                check(rc, "r2x_voxel_forward_async_raw")

            R, binning = _C._forward(run, _C.voxel_key(dev, P, nx, ny, nz, s.sVoxel_x), P, _C.VOXEL.seed, dev)
        ctx.settings, ctx.act, ctx.num_rendered, ctx.grid = s, act, R, grid
        ctx.save_for_backward(means3D, raw_scales, raw_rotations, rx, ry, rz, geom, binning, img)
        return vol, (rx, ry, rz)

    @staticmethod
    def backward(ctx, grad_vol, _grad_radii):
        lib = load()
        s, act, R, grid = ctx.settings, ctx.act, ctx.num_rendered, ctx.grid
        means3D, raw_scales, raw_rotations, rx, ry, rz, geom, binning, img = ctx.saved_tensors
        cap = _C._carved_capacity(binning, R)
        dev = means3D.device
        P = int(means3D.shape[0])
        with torch.cuda.device(dev):
            opts = dict(dtype=torch.float32, device=dev)
            gd = torch.empty((P, 1), **opts); g3 = torch.empty((P, 3), **opts); gcov = torch.empty((P, 6), **opts)
            gs = torch.empty((P, 3), **opts); gr = torch.empty((P, 4), **opts)
            scratch = _C.VOXEL.bwd_scratch(cap, dev)
            dL = _C._f32(grad_vol, dev)
            rc = lib.r2x_voxel_backward_raw(
                torch.cuda.current_stream(dev).cuda_stream, P, cap, *grid, _C._ptr(means3D), _C._ptr(raw_scales),
                float(s.scale_modifier), _C._ptr(raw_rotations), _C._ptr(rx), _C._ptr(ry), _C._ptr(rz), _C._ptr(geom),
                _C._ptr(binning), _C._ptr(img), scratch.data_ptr(), _C._ptr(dL), _C._ptr(gd), _C._ptr(g3), _C._ptr(gcov),
                _C._ptr(gs), _C._ptr(gr), C.byref(act))
            check(rc, "r2x_voxel_backward_raw")
        return g3, gd, gs, gr, None, None


def rasterize_raw(means3D, means2D, raw, settings):
    """raw = model.raw_parameters(): {"density", "scaling", "rotation", "scale_bound"} -> (image [1,H,W], radii)."""
    return _RasterizeRaw.apply(means3D, means2D, raw["density"], raw["scaling"], raw["rotation"], settings, _act(raw))


def rasterize_raw_matrices(means3D, means2D, raw, viewmatrix, projmatrix, settings):
    """`rasterize_raw` whose image is also differentiable with respect to `viewmatrix` / `projmatrix`."""
    return _RasterizeRawMatrices.apply(means3D, means2D, raw["density"], raw["scaling"], raw["rotation"], viewmatrix,
                                       projmatrix, settings, _act(raw))


def rasterize_views_raw(means3D, means2D, raw, viewmatrices, projmatrices, settings):
    """`rasterize_raw` for N views in one call -> (images [N,H,W], radii [N,P]).  viewmatrices / projmatrices [N,4,4]
    (not differentiated); `means2D` [N,P,3] receives the per-view screen-space gradients.  Image v and radii[v] are bit
    for bit `rasterize_raw` of view v; each raw gradient is the single-view ones summed in view order (float32)."""
    N = _C.check_views_args(means3D, viewmatrices, projmatrices)
    if tuple(means2D.shape) != (N, means3D.shape[0], 3):
        raise ValueError(f"means2D must have dimensions ({N}, {means3D.shape[0]}, 3), got {tuple(means2D.shape)}")
    return _RasterizeViewsRaw.apply(means3D, means2D, raw["density"], raw["scaling"], raw["rotation"],
                                    viewmatrices.detach(), projmatrices.detach(), settings, _act(raw))


def voxelize_raw(means3D, raw, settings):
    return _VoxelizeRaw.apply(means3D, raw["density"], raw["scaling"], raw["rotation"], settings, _act(raw))
