"""Forward projection of a voxel volume on the GPU over the C ABI (r2x_volume_project) -- what the reference obtains from
TIGRE's `Ax` to synthesise its datasets (`data_generator/synthetic_dataset/generate_data.py`).

    projs = project(volume, angles, scanner_cfg)        # [N, H, W], rows = v, columns = u

`volume` is a CUDA float32 [nx, ny, nz] tensor in the voxelizer's layout; `scanner_cfg` is the scaled dict of
`dataset.read_scene` / `Scene.scanner_cfg`, and the result is in the same scene-scaled units (what the readers hand to
training).  The per-view geometry is the rasterizer's (`scene.make_view`), so the projections agree with render() by
construction.  Each pixel is the line integral of the volume's trilinear field, sampled every
`accuracy * min(dVoxel)` along the ray (`accuracy` defaults to 0.5, as in the reference's scanner files); the exact
definition is in include/r2x.h.  Runs on the current stream; no CPU fallback.
"""
from __future__ import annotations

import numpy as np
import torch

from ._lib import check, load
from .scene import make_view

DEFAULT_ACCURACY = 0.5


def project(volume: torch.Tensor, angles, scanner_cfg: dict) -> torch.Tensor:
    nvox = tuple(int(v) for v in scanner_cfg["nVoxel"])
    if tuple(getattr(volume, "shape", ())) != nvox:
        raise ValueError(f"project: volume shape {tuple(getattr(volume, 'shape', ()))} is not the scanner's nVoxel "
                         f"{list(nvox)}")
    accuracy = float(scanner_cfg.get("accuracy", DEFAULT_ACCURACY))
    if not accuracy > 0.0:
        raise ValueError(f"project: accuracy must be > 0, got {accuracy}")
    if np.any(np.asarray(scanner_cfg.get("offDetector", [0.0, 0.0]), np.float64) != 0.0):
        raise ValueError("project: offDetector must be [0, 0]: render() has no detector offset, so such projections "
                         "would not match training")
    if scanner_cfg["mode"] != "cone" and not np.allclose(np.asarray(scanner_cfg["sDetector"], np.float64), 2.0,
                                                         rtol=1e-6, atol=0.0):
        raise ValueError(f"project: a parallel-beam detector must span the scene's [-1, 1] (scaled sDetector [2, 2]), "
                         f"got {list(scanner_cfg['sDetector'])}: render() could not reproduce that geometry")
    if not isinstance(volume, torch.Tensor) or volume.device.type != "cuda":
        raise RuntimeError("project: volume must be a CUDA tensor (this build has no CPU fallback; "
                           f"got {getattr(volume, 'device', type(volume))})")
    angles =np.asarray(angles, dtype=np.float64).reshape(-1)
    if len(angles) == 0:
        raise ValueError("project: no angles")
    views = [make_view(scanner_cfg, float(a)) for a in angles]
    N, H, W = len(views), views[0].image_height, views[0].image_width
    sx, sy, sz = (float(v) for v in scanner_cfg["sVoxel"])
    cx, cy, cz = (float(v) for v in scanner_cfg["offOrigin"])
    step = accuracy * min(sx / nvox[0], sy / nvox[1], sz / nvox[2])
    dev = volume.device
    lib = load()
    with torch.cuda.device(dev):
        vol = volume.detach().to(torch.float32).contiguous()
        vm = torch.from_numpy(np.stack([v.viewmatrix.reshape(16) for v in views])).to(dev)
        out = torch.empty((N, H, W), dtype=torch.float32, device=dev)
        rc = lib.r2x_volume_project(torch.cuda.current_stream(dev).cuda_stream, *nvox, vol.data_ptr(), sx, sy, sz,
                                    cx, cy, cz, N, H, W, vm.data_ptr(), float(views[0].tanfovx),
                                    float(views[0].tanfovy), int(views[0].mode), step, out.data_ptr())
    check(rc, "r2x_volume_project")
    return out
