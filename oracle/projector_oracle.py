"""Float64 NumPy statement of the volume forward projection that `r2_gaussian_b200.projector` runs on the GPU.

TEST INFRASTRUCTURE ONLY: imported by tests/, never by the product package.

All lengths are in the scene-scaled units of `dataset.read_scene`.  volume[nx,ny,nz] is the voxelizer's layout (z
fastest) with size sVoxel centred at offOrigin; each view is `scene.make_view(scanner_cfg, angle)`, so the projections
agree with render() by construction.

1. Rays.  Detector pixel (row i = v, column j = u) has ndc = ((2j+1)/W - 1, (2i+1)/H - 1), the inverse of the
   rasterizer's ndc2Pix.  Cone beam: the ray starts at the camera centre with camera-frame direction
   (ndc_x tan_fovx, ndc_y tan_fovy, 1); parallel beam: it starts at camera-frame (ndc_x, ndc_y, 0) with direction
   (0, 0, 1).  Both go to world space through the inverse of the viewmatrix.  Directions are unit vectors, so the ray
   parameter t is a length.
2. Field.  f is the trilinear interpolation of the volume between the voxel centres offOrigin - sVoxel/2 + (i + 1/2)
   dVoxel; every lattice point outside [0,n) has value 0.  So f is continuous and nonzero only inside the box
   offOrigin +- (sVoxel/2 + dVoxel/2).
3. Integral.  P = step * sum_k f(o + (t_c + k step) d) over the integers k whose sample lies inside that box (cone beam
   also t > 0), with step = accuracy * min(dVoxel) and t_c = (offOrigin - o).d, the ray's closest approach to the
   volume centre.  The sample positions do not depend on where the ray enters or leaves the box.  A ray that misses the
   box gives exactly 0.
"""
from __future__ import annotations

import math

import numpy as np


def step_length(scanner_cfg: dict) -> float:
    """accuracy * min(dVoxel); `accuracy` defaults to 0.5, the value of the reference's scanner files."""
    d = np.asarray(scanner_cfg["sVoxel"], np.float64) / np.asarray(scanner_cfg["nVoxel"], np.float64)
    return float(scanner_cfg.get("accuracy", 0.5)) * float(d.min())


def rays(view):
    """World-space origins and unit directions [H, W, 3] of the pixel centres of a `scene.View`."""
    H, W = view.image_height, view.image_width
    ndx = (2.0 * np.arange(W) + 1.0) / W - 1.0
    ndy = (2.0 * np.arange(H) + 1.0) / H - 1.0
    c2w = np.linalg.inv(view.viewmatrix.astype(np.float64).T)            # viewmatrix is stored transposed
    if view.mode == 1:
        d = np.stack(np.broadcast_arrays(ndx[None, :] * view.tanfovx, ndy[:, None] * view.tanfovy, 1.0), -1)
        o = np.broadcast_to(c2w[:3, 3], d.shape)
    else:
        d = np.broadcast_to(np.array([0.0, 0.0, 1.0]), (H, W, 3))
        o = np.stack(np.broadcast_arrays(ndx[None, :], ndy[:, None], 0.0), -1) @ c2w[:3, :3].T + c2w[:3, 3]
    d = d @ c2w[:3, :3].T
    return np.ascontiguousarray(o), d / np.linalg.norm(d, axis=-1, keepdims=True)


def field(padded, g):
    """Trilinear interpolation at index-space points g[..., 3] (lattice point i at g = i) of a volume padded by one
    layer of zeros (lattice points -1 and n)."""
    n = np.asarray(padded.shape) - 2
    g = np.clip(g, -1.0, n - 1e-9) + 1.0                                # beyond the padding f is 0 anyway
    i0 = np.floor(g).astype(np.int64)
    w = g - i0
    out = 0.0
    for cx in (0, 1):
        for cy in (0, 1):
            for cz in (0, 1):
                wt = ((w[..., 0] if cx else 1 - w[..., 0]) * (w[..., 1] if cy else 1 - w[..., 1]) *
                      (w[..., 2] if cz else 1 - w[..., 2]))
                out = out + wt * padded[i0[..., 0] + cx, i0[..., 1] + cy, i0[..., 2] + cz].astype(np.float64)
    return out


def project_rays(volume, o, d, cone: bool, sVoxel, offOrigin, step: float) -> np.ndarray:
    """The integral along rays with origins o[..., 3] and unit directions d[..., 3]."""
    padded = np.pad(np.asarray(volume), 1)                              # lattice points -1 and n are zeros
    n = np.asarray(volume.shape, np.float64)
    s = np.asarray(sVoxel, np.float64)
    c = np.asarray(offOrigin, np.float64)
    dv = s / n
    lo_box = c - s / 2.0 - dv / 2.0                                     # g = -1
    tc = ((c - o) * d).sum(-1)
    K = int(math.ceil(np.linalg.norm(s / 2.0 + dv / 2.0) / step)) + 1   # |t - t_c| <= half-diagonal inside the box
    acc = np.zeros(o.shape[:-1])
    for k in range(-K, K + 1):
        t = tc + k * step
        g = (o + t[..., None] * d - lo_box) / dv - 1.0
        inside = np.all((g > -1.0) & (g < n), axis=-1)
        if cone:
            inside &= t > 0
        acc += np.where(inside, field(padded, g), 0.0)
    return acc * step


def project_view(volume, view, sVoxel, offOrigin, step: float) -> np.ndarray:
    o, d = rays(view)
    return project_rays(volume, o, d, view.mode == 1, sVoxel, offOrigin, step)


def project_scene(volume, angles, scanner_cfg: dict, step: float | None = None) -> np.ndarray:
    """The oracle on a scanner dict (as `read_scene` returns it) and one angle per view: [N, H, W] float64."""
    from r2_gaussian_b200.scene import make_view

    step = step_length(scanner_cfg) if step is None else step
    return np.stack([project_view(volume, make_view(scanner_cfg, float(a)), scanner_cfg["sVoxel"],
                                  scanner_cfg["offOrigin"], step) for a in angles])
