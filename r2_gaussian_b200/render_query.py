"""render() / query(): the two calls the reference's training and test drivers make.

Same contract as r2_gaussian/gaussian/render_query.py of the reference (query :27-77, render :80-160):
`pc` is any object exposing get_xyz / get_density / get_scaling / get_rotation (and get_covariance when
pipe.compute_cov3D_python), `viewpoint_camera` exposes image_height/width, FoVx/FoVy, mode,
world_view_transform, full_proj_transform, camera_center; `pipe` exposes debug and compute_cov3D_python.
After `sharded.enable(group)` (Gaussian-sharded runs: the trainer, bench.py) each rank holds a shard of the
Gaussians and the image / volume is summed over ranks; the per-Gaussian outputs describe the local shard.
Without that opt-in an initialised process group changes nothing (data-parallel / multi-scene jobs).
When the camera's world_view_transform or full_proj_transform requires grad (e.g. `pose.PoseCorrection`), the
backward also fills their .grad (not with Gaussian sharding); otherwise render() runs exactly as the reference's.
"""
from __future__ import annotations

import math

import torch

from . import fused, sharded
from .rasterization import (GaussianRasterizationSettings, GaussianRasterizer, rasterize_gaussians_matrices,
                            rasterize_views)
from .sharded import sharded_sum
from .voxelization import GaussianVoxelizationSettings, GaussianVoxelizer


def _raw_parameters(pc, pipe):
    """The model's raw parameters when the activations can be folded into the kernels (fused.py): this repository's
    GaussianModel, covariance not precomputed in Python, debug off."""
    if not fused.enabled() or getattr(pipe, "compute_cov3D_python", False) or getattr(pipe, "debug", False):
        return None
    get = getattr(pc, "raw_parameters", None)
    return get() if callable(get) else None


def _covariance_inputs(pc, pipe, scaling_modifier):
    if getattr(pipe, "compute_cov3D_python", False):
        return None, None, pc.get_covariance(scaling_modifier)
    return pc.get_scaling, pc.get_rotation, None


def query(pc, center, nVoxel, sVoxel, pipe, scaling_modifier=1.0):
    """Density volume of the model on a regular grid -> {"vol": [nx,ny,nz], "radii": (rx, ry, rz)}."""
    settings = GaussianVoxelizationSettings(
        scale_modifier=scaling_modifier,
        nVoxel_x=int(nVoxel[0]), nVoxel_y=int(nVoxel[1]), nVoxel_z=int(nVoxel[2]),
        sVoxel_x=float(sVoxel[0]), sVoxel_y=float(sVoxel[1]), sVoxel_z=float(sVoxel[2]),
        center_x=float(center[0]), center_y=float(center[1]), center_z=float(center[2]),
        prefiltered=False, debug=bool(getattr(pipe, "debug", False)))
    raw = _raw_parameters(pc, pipe)
    if raw is not None:
        vol, radii = fused.voxelize_raw(pc.get_xyz, raw, settings)
        return {"vol": sharded_sum(vol), "radii": radii}
    scales, rotations, cov3D = _covariance_inputs(pc, pipe, scaling_modifier)
    vol, radii = GaussianVoxelizer(voxel_settings=settings)(
        means3D=pc.get_xyz, opacities=pc.get_density, scales=scales, rotations=rotations, cov3D_precomp=cov3D)
    return {"vol": sharded_sum(vol), "radii": radii}


def _tan_fov(camera) -> tuple[float, float]:
    mode = int(camera.mode)
    if mode == 0:
        return 1.0, 1.0
    if mode == 1:
        return math.tan(camera.FoVx * 0.5), math.tan(camera.FoVy * 0.5)
    raise ValueError("Unsupported mode!")


def render_views(cameras, pc, pipe, scaling_modifier=1.0):
    """X-ray projections of the model for N cameras in one batched call -> the `render()` dict with a leading view
    axis: {"render": [N,1,H,W], "viewspace_points": [N,P,3] (receives the per-view dL/dmean2D), "visibility_filter":
    bool[N,P], "radii": int[N,P]}.  render["render"][v] is bit for bit render(cameras[v], ...)["render"] (activated
    parameters).  The cameras must share image size, field of view and mode; they are not differentiated, the
    covariance is never precomputed in Python, and Gaussian sharding is not supported."""
    cameras = list(cameras)
    if not cameras:
        raise ValueError("render_views(): no camera")
    c0 = cameras[0]
    shape = lambda c: (int(c.image_height), int(c.image_width), int(c.mode), _tan_fov(c))
    if any(shape(c) != shape(c0) for c in cameras[1:]):
        raise ValueError("render_views(): all cameras must share image size, field of view and mode")
    if getattr(pipe, "compute_cov3D_python", False):
        raise ValueError("render_views(): compute_cov3D_python is not supported (needs scales and rotations)")
    if sharded.enabled():
        raise RuntimeError("render_views(): Gaussian sharding is not supported")
    tanfovx, tanfovy = _tan_fov(c0)
    views = torch.stack([c.world_view_transform.detach() for c in cameras])
    projs = torch.stack([c.full_proj_transform.detach() for c in cameras])
    xyz = pc.get_xyz
    screenspace_points = torch.zeros((len(cameras),) + tuple(xyz.shape), dtype=xyz.dtype, device=xyz.device,
                                     requires_grad=True) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    settings = GaussianRasterizationSettings(
        image_height=int(c0.image_height), image_width=int(c0.image_width), tanfovx=tanfovx, tanfovy=tanfovy,
        scale_modifier=scaling_modifier, viewmatrix=views[0], projmatrix=projs[0], campos=c0.camera_center,
        prefiltered=False, mode=int(c0.mode), debug=bool(getattr(pipe, "debug", False)))
    images, radii = rasterize_views(xyz, pc.get_density, pc.get_scaling, pc.get_rotation, views, projs, settings,
                                    means2D=screenspace_points)
    return {"render": images.unsqueeze(1), "viewspace_points": screenspace_points, "visibility_filter": radii > 0,
            "radii": radii}


def render(viewpoint_camera, pc, pipe, scaling_modifier=1.0):
    """X-ray projection of the model for one camera ->
    {"render": [1,H,W], "viewspace_points": [P,3] (receives dL/dmean2D), "visibility_filter": bool[P], "radii": int[P]}."""
    xyz = pc.get_xyz
    # zero tensor whose .grad receives the screen-space mean gradients (densification statistics)
    screenspace_points = torch.zeros_like(xyz, dtype=xyz.dtype, requires_grad=True, device=xyz.device) + 0
    try:
        screenspace_points.retain_grad()
    except Exception:
        pass
    mode = int(viewpoint_camera.mode)
    if mode == 0:
        tanfovx = tanfovy = 1.0
    elif mode == 1:
        tanfovx = math.tan(viewpoint_camera.FoVx * 0.5)
        tanfovy = math.tan(viewpoint_camera.FoVy * 0.5)
    else:
        raise ValueError("Unsupported mode!")
    settings = GaussianRasterizationSettings(
        image_height=int(viewpoint_camera.image_height), image_width=int(viewpoint_camera.image_width),
        tanfovx=tanfovx, tanfovy=tanfovy, scale_modifier=scaling_modifier,
        viewmatrix=viewpoint_camera.world_view_transform, projmatrix=viewpoint_camera.full_proj_transform,
        campos=viewpoint_camera.camera_center, prefiltered=False, mode=mode,
        debug=bool(getattr(pipe, "debug", False)))
    raw = _raw_parameters(pc, pipe)
    view, proj = viewpoint_camera.world_view_transform, viewpoint_camera.full_proj_transform
    matrices = torch.is_grad_enabled() and (view.requires_grad or proj.requires_grad)
    if matrices and sharded.enabled():
        raise RuntimeError("render(): gradients with respect to the camera matrices are not supported with Gaussian "
                           "sharding (each rank would hold a partial sum over its shard)")
    if raw is not None:
        if matrices:
            image, radii = fused.rasterize_raw_matrices(xyz, screenspace_points, raw, view, proj, settings)
        else:
            image, radii = fused.rasterize_raw(xyz, screenspace_points, raw, settings)
        return {"render": sharded_sum(image), "viewspace_points": screenspace_points,
                "visibility_filter": radii > 0, "radii": radii}
    scales, rotations, cov3D = _covariance_inputs(pc, pipe, scaling_modifier)
    if matrices:
        image, radii = rasterize_gaussians_matrices(xyz, screenspace_points, pc.get_density, scales, rotations, cov3D,
                                                    view, proj, settings)
    else:
        image, radii = GaussianRasterizer(raster_settings=settings)(
            means3D=xyz, means2D=screenspace_points, opacities=pc.get_density, scales=scales, rotations=rotations,
            cov3D_precomp=cov3D)
    return {"render": sharded_sum(image), "viewspace_points": screenspace_points,
            "visibility_filter": radii > 0, "radii": radii}
