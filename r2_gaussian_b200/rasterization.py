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
