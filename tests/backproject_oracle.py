"""Float64 NumPy statement of the matched backprojection that `r2_gaussian_b200.projector.backproject` runs on the GPU:
the exact transpose of oracle/projector_oracle.py's `project_scene`.

For every view, ray and sample k that `project_rays` sums, y[v,i,j] * step * w_corner is added (np.add.at) to each of
the 8 lattice points whose trilinear weight w_corner `field` uses at that sample; lattice points -1 and n (the zero
padding) are dropped.  So <project_scene(x), y> = <x, backproject_scene(y)> up to float64 rounding.
"""
from __future__ import annotations

import math

import numpy as np

from oracle import projector_oracle as po


def backproject_rays(y, o, d, cone: bool, shape, sVoxel, offOrigin, step: float) -> np.ndarray:
    """The transpose of `po.project_rays` for rays o[..., 3], d[..., 3] and values y[...]: a volume of `shape`."""
    n = np.asarray(shape, np.float64)
    s = np.asarray(sVoxel, np.float64)
    c = np.asarray(offOrigin, np.float64)
    dv = s / n
    lo_box = c - s / 2.0 - dv / 2.0
    tc = ((c - o) * d).sum(-1)
    K = int(math.ceil(np.linalg.norm(s / 2.0 + dv / 2.0) / step)) + 1
    padded = np.zeros(np.asarray(shape) + 2)
    y = np.asarray(y, np.float64) * step
    for k in range(-K, K + 1):
        t = tc + k * step
        g = (o + t[..., None] * d - lo_box) / dv - 1.0
        inside = np.all((g > -1.0) & (g < n), axis=-1)
        if cone:
            inside &= t > 0
        if not inside.any():
            continue
        gi = np.clip(g[inside], -1.0, n - 1e-9) + 1.0                   # as po.field
        yi = y[inside]
        i0 = np.floor(gi).astype(np.int64)
        w = gi - i0
        for cx in (0, 1):
            for cy in (0, 1):
                for cz in (0, 1):
                    wt = ((w[:, 0] if cx else 1 - w[:, 0]) * (w[:, 1] if cy else 1 - w[:, 1]) *
                          (w[:, 2] if cz else 1 - w[:, 2]))
                    np.add.at(padded, (i0[:, 0] + cx, i0[:, 1] + cy, i0[:, 2] + cz), wt * yi)
    return padded[1:-1, 1:-1, 1:-1]


def backproject_scene(projs, angles, scanner_cfg: dict, step: float | None = None) -> np.ndarray:
    """A^T projs for the oracle's A = `po.project_scene(., angles, scanner_cfg)`: [nx, ny, nz] float64."""
    from r2_gaussian_b200.scene import make_view

    step = po.step_length(scanner_cfg) if step is None else step
    shape = tuple(int(v) for v in scanner_cfg["nVoxel"])
    out = np.zeros(shape)
    for v, a in enumerate(angles):
        view = make_view(scanner_cfg, float(a))
        o, d = po.rays(view)
        out += backproject_rays(projs[v], o, d, view.mode == 1, shape, scanner_cfg["sVoxel"], scanner_cfg["offOrigin"],
                                step)
    return out


def operators(angles, scanner_cfg: dict):
    """The oracle pair as the callables `recon.cgls_solve` / `recon.sart_solve` take (float64 CPU torch tensors)."""
    import torch

    angles = list(angles)

    def A(x, views):
        return torch.from_numpy(po.project_scene(x.numpy(), angles[views], scanner_cfg))

    def At(y, views, weights):
        vol = torch.from_numpy(backproject_scene(y.numpy(), angles[views], scanner_cfg))
        if not weights:
            return vol
        return vol, torch.from_numpy(backproject_scene(np.ones(tuple(y.shape)), angles[views], scanner_cfg))

    return A, At
