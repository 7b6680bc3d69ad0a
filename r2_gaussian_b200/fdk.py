"""FDK reconstruction on the GPU over the C ABI (r2x_fdk) -- what the reference obtains from TIGRE's `algs.fdk`
(`r2_gaussian/utils/ct_utils.py::recon_volume`) to initialise its point cloud.

    vol = fdk(projections, angles, scanner_cfg)        # [nx, ny, nz], the voxelizer's layout

`projections` is a CUDA float32 [N, H, W] tensor in the dataset layout (rows = v, columns = u, already multiplied by
scene_scale); `scanner_cfg` is the scaled dict of `dataset.read_scene` / `Scene.scanner_cfg`.  The per-view geometry is
the rasterizer's (`scene.make_view`), so the reconstruction agrees with render() on detector orientation, axis order and
angle convention by construction.  Band-limited Ram-Lak filter only (`filter: null` or "ram_lak"), no Parker weights
(a cone-beam short scan is reconstructed as a full scan, as TIGRE's default fdk does).  Runs on the current stream;
no CPU fallback.
"""
from __future__ import annotations

import numpy as np
import torch

from ._lib import check, load
from .scene import make_view

SUPPORTED_FILTERS = (None, "ram_lak")


def fdk(projections: torch.Tensor, angles, scanner_cfg: dict) -> torch.Tensor:
    if not isinstance(projections, torch.Tensor) or projections.device.type != "cuda":
        raise RuntimeError("fdk: projections must be a CUDA tensor (this build has no CPU fallback; "
                           f"got {getattr(projections, 'device', type(projections))})")
    if projections.dim() != 3:
        raise ValueError(f"fdk: expected projections of shape [N, H, W], got {tuple(projections.shape)}")
    filt = scanner_cfg.get("filter")
    if filt not in SUPPORTED_FILTERS:
        raise ValueError(f"fdk: filter {filt!r} is not supported (only the Ram-Lak filter: null or 'ram_lak')")
    angles = np.asarray(angles, dtype=np.float64).reshape(-1)
    N, H, W = (int(s) for s in projections.shape)
    if len(angles) != N:
        raise ValueError(f"fdk: {N} projections but {len(angles)} angles")
    if (H, W) != (int(scanner_cfg["nDetector"][0]), int(scanner_cfg["nDetector"][1])):
        raise ValueError(f"fdk: projections are {H}x{W}, scanner nDetector is {list(scanner_cfg['nDetector'])}")
    if N == 0:
        raise ValueError("fdk: no projections")
    views = [make_view(scanner_cfg, float(a)) for a in angles]
    mode = views[0].mode
    nx, ny, nz = (int(v) for v in scanner_cfg["nVoxel"])
    sx, sy, sz = (float(v) for v in scanner_cfg["sVoxel"])
    cx, cy, cz = (float(v) for v in scanner_cfg["offOrigin"])
    dev = projections.device
    lib = load()
    with torch.cuda.device(dev):
        projs = projections.detach().to(torch.float32).contiguous()
        vm = torch.from_numpy(np.stack([v.viewmatrix.reshape(16) for v in views])).to(dev, non_blocking=False)
        pm = torch.from_numpy(np.stack([v.projmatrix.reshape(16) for v in views])).to(dev, non_blocking=False)
        vol = torch.empty((nx, ny, nz), dtype=torch.float32, device=dev)
        nbytes = int(lib.r2x_fdk_scratch_bytes(N, H, W))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        rc = lib.r2x_fdk(torch.cuda.current_stream(dev).cuda_stream, N, H, W, projs.data_ptr(), vm.data_ptr(),
                         pm.data_ptr(), float(views[0].tanfovx), float(views[0].tanfovy), int(mode),
                         float(scanner_cfg["DSO"]), nx, ny, nz, sx, sy, sz, cx, cy, cz, vol.data_ptr(),
                         scratch.data_ptr(), nbytes)
    check(rc, "r2x_fdk")
    return vol
