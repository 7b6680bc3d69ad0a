"""X-ray projection front-end with the reference's Python surface.

Mirrors PYX/rasterization.py of the reference (PYX = r2_gaussian/submodules/
xray-gaussian-rasterization-voxelization/xray_gaussian_rasterization_voxelization):
`GaussianRasterizationSettings` (:200-211), `GaussianRasterizer` (:214-264) and the autograd bridge
`_RasterizeGaussians` (:46-196) -- same names, argument order, return values, gradient order and error
behaviour -- over the H100-native library (r2_gaussian_b200._C).
"""
from __future__ import annotations

from typing import NamedTuple

import torch
from torch import nn

from . import _C
from ._snapshot import call_with_snapshot


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    campos: torch.Tensor
    prefiltered: bool
    mode: int  # 0 = parallel beam, 1 = cone beam
    debug: bool


class _RasterizeGaussians(torch.autograd.Function):
    """forward inputs:  (means3D, means2D, opacities, scales, rotations, cov3Ds_precomp, settings)
    backward outputs: (d means3D, d means2D, d opacities, d scales, d rotations, d cov3Ds_precomp, None)."""

    @staticmethod
    def forward(ctx, means3D, means2D, opacities, scales, rotations, cov3Ds_precomp, raster_settings):
        s = raster_settings
        native_args = (means3D, opacities, scales, rotations, s.scale_modifier, cov3Ds_precomp, s.viewmatrix,
                       s.projmatrix, s.tanfovx, s.tanfovy, s.image_height, s.image_width, s.campos, s.prefiltered,
                       s.mode, s.debug)
        # training mode (some input needs a gradient): no host synchronisation in the forward, the instance-capacity
        # check is deferred to the backward (_C.speculative)
        with _C.speculative(any(ctx.needs_input_grad) and not s.debug):
            num_rendered, color, radii, geom, binning, img = call_with_snapshot(
                _C.rasterize_gaussians, native_args, s.debug, "snapshot_fw.dump", "forward")
        ctx.raster_settings = s
        ctx.num_rendered = num_rendered
        ctx.save_for_backward(means3D, scales, rotations, cov3Ds_precomp, radii, geom, binning, img)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, grad_color, _grad_radii):
        s = ctx.raster_settings
        means3D, scales, rotations, cov3Ds_precomp, radii, geom, binning, img = ctx.saved_tensors
        native_args = (means3D, radii, scales, rotations, s.scale_modifier, cov3Ds_precomp, s.viewmatrix,
                       s.projmatrix, s.tanfovx, s.tanfovy, grad_color, s.campos, geom, ctx.num_rendered, binning, img,
                       s.mode, s.debug)
        g_means2D, g_opac, _g_mu, g_means3D, g_cov, g_scales, g_rots = call_with_snapshot(
            _C.rasterize_gaussians_backward, native_args, s.debug, "snapshot_bw.dump", "backward")
        return g_means3D, g_means2D, g_opac, g_scales, g_rots, g_cov, None


def rasterize_gaussians(means3D, means2D, opacities, scales, rotations, cov3Ds_precomp, raster_settings):
    return _RasterizeGaussians.apply(means3D, means2D, opacities, scales, rotations, cov3Ds_precomp, raster_settings)


class _RasterizeGaussiansMatrices(torch.autograd.Function):
    """`_RasterizeGaussians` with the view and projection matrices as differentiable inputs (not part of the
    reference's surface: `GaussianRasterizer` keeps returning no gradient for the settings' matrices).
    forward inputs:  (means3D, means2D, opacities, scales, rotations, cov3Ds_precomp, viewmatrix, projmatrix, settings)
    The settings' own matrices are ignored."""

    @staticmethod
    def forward(ctx, means3D, means2D, opacities, scales, rotations, cov3Ds_precomp, viewmatrix, projmatrix,
                raster_settings):
        s = raster_settings._replace(viewmatrix=viewmatrix.detach(), projmatrix=projmatrix.detach())
        ctx.matrix_dtypes = (viewmatrix.dtype, projmatrix.dtype)
        return _RasterizeGaussians.forward(ctx, means3D, means2D, opacities, scales, rotations, cov3Ds_precomp, s)

    @staticmethod
    def backward(ctx, grad_color, _grad_radii):
        s = ctx.raster_settings
        means3D, scales, rotations, cov3Ds_precomp, radii, geom, binning, img = ctx.saved_tensors
        native_args = (means3D, radii, scales, rotations, s.scale_modifier, cov3Ds_precomp, s.viewmatrix,
                       s.projmatrix, s.tanfovx, s.tanfovy, grad_color, s.campos, geom, ctx.num_rendered, binning, img,
                       s.mode, s.debug)
        g_means2D, g_opac, _g_mu, g_means3D, g_cov, g_scales, g_rots, g_view, g_proj = call_with_snapshot(
            _C.rasterize_gaussians_backward_matrices, native_args, s.debug, "snapshot_bw.dump", "backward")
        g_view = g_view.view(s.viewmatrix.shape).to(ctx.matrix_dtypes[0])
        g_proj = g_proj.view(s.projmatrix.shape).to(ctx.matrix_dtypes[1])
        return g_means3D, g_means2D, g_opac, g_scales, g_rots, g_cov, g_view, g_proj, None


def rasterize_gaussians_matrices(means3D, means2D, opacities, scales, rotations, cov3Ds_precomp, viewmatrix, projmatrix,
                                 raster_settings):
    """-> (image [1,H,W], radii); the image is differentiable with respect to `viewmatrix` / `projmatrix` too."""
    _exactly_one_covariance_source(scales, rotations, cov3Ds_precomp)
    empty = torch.Tensor([])
    return _RasterizeGaussiansMatrices.apply(
        means3D, means2D, opacities, empty if scales is None else scales, empty if rotations is None else rotations,
        empty if cov3Ds_precomp is None else cov3Ds_precomp, viewmatrix, projmatrix, raster_settings)


class _RasterizeViews(torch.autograd.Function):
    """N views of one cloud in one native call (not part of the reference's surface).
    forward inputs:  (means3D, means2D[N,P,3], opacities, scales, rotations, viewmatrices[N,4,4], projmatrices[N,4,4],
    settings) -> (images[N,H,W], radii[N,P]); the settings' own matrices are ignored.  The backward sums the Gaussian
    gradients over the views and hands means2D the per-view screen-space gradients."""

    @staticmethod
    def forward(ctx, means3D, means2D, opacities, scales, rotations, viewmatrices, projmatrices, raster_settings):
        s = raster_settings
        with _C.speculative(any(ctx.needs_input_grad) and not s.debug):
            num_rendered, images, radii, geom, binning, img = _C.rasterize_views(
                means3D, opacities, scales, rotations, s.scale_modifier, viewmatrices, projmatrices, s.tanfovx,
                s.tanfovy, s.image_height, s.image_width, s.mode)
        ctx.raster_settings = s
        ctx.num_rendered = num_rendered
        ctx.save_for_backward(means3D, scales, rotations, viewmatrices, projmatrices, radii, geom, binning, img)
        ctx.mark_non_differentiable(radii)
        return images, radii

    @staticmethod
    def backward(ctx, grad_images, _grad_radii):
        s = ctx.raster_settings
        means3D, scales, rotations, viewmatrices, projmatrices, radii, geom, binning, img = ctx.saved_tensors
        g_means2D, g_opac, g_means3D, _g_cov, g_scales, g_rots = _C.rasterize_views_backward(
            means3D, radii, scales, rotations, s.scale_modifier, viewmatrices, projmatrices, s.tanfovx, s.tanfovy,
            grad_images, geom, ctx.num_rendered, binning, img, s.mode, s.debug)
        return g_means3D, g_means2D, g_opac, g_scales, g_rots, None, None, None


def rasterize_views(means3D, opacities, scales, rotations, viewmatrices, projmatrices, raster_settings, means2D=None):
    """Project one cloud into N views at once -> (images[N,H,W], radii[N,P] int32).

    All views share the settings' image size, tanfovx / tanfovy, scale_modifier and mode; view v has its own
    viewmatrices[v] / projmatrices[v] (the settings' viewmatrix / projmatrix / campos are not used).  Image v is bit
    for bit the single-view render of view v.  Gradients flow to means3D, opacities, scales and rotations (summed over
    the views); `means2D` (a [N,P,3] tensor, e.g. zeros with requires_grad) receives the per-view screen-space
    gradients, as `viewspace_points` does in `render()`.  Scales and rotations are required (no precomputed 3-D
    covariance); the camera matrices get no gradient."""
    N = _C.check_views_args(means3D, viewmatrices, projmatrices)
    if scales is None or rotations is None:
        raise ValueError("rasterize_views needs scales and rotations (cov3D_precomp is not supported)")
    if means2D is None:
        means2D = torch.zeros((N, means3D.shape[0], 3), dtype=means3D.dtype, device=means3D.device)
    elif tuple(means2D.shape) != (N, means3D.shape[0], 3):
        raise ValueError(f"means2D must have dimensions ({N}, {means3D.shape[0]}, 3), got {tuple(means2D.shape)}")
    return _RasterizeViews.apply(means3D, means2D, opacities, scales, rotations, viewmatrices.detach(),
                                 projmatrices.detach(), raster_settings)


def _exactly_one_covariance_source(scales, rotations, cov3D_precomp):
    have_sr = scales is not None or rotations is not None
    full_sr = scales is not None and rotations is not None
    if (not full_sr and cov3D_precomp is None) or (have_sr and cov3D_precomp is not None):
        raise Exception("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings: GaussianRasterizationSettings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        """bool[P]: which points pass the near-plane test of the current view."""
        with torch.no_grad():
            return _C.mark_visible(positions, self.raster_settings.viewmatrix, self.raster_settings.projmatrix)

    def forward(self, means3D, means2D, opacities, scales=None, rotations=None, cov3D_precomp=None):
        _exactly_one_covariance_source(scales, rotations, cov3D_precomp)
        empty = torch.Tensor([])
        return rasterize_gaussians(
            means3D, means2D, opacities,
            empty if scales is None else scales,
            empty if rotations is None else rotations,
            empty if cov3D_precomp is None else cov3D_precomp,
            self.raster_settings)
