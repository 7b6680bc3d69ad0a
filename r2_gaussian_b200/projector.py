"""Forward projection of a voxel volume on the GPU over the C ABI (r2x_volume_project) -- what the reference obtains from
TIGRE's `Ax` to synthesise its datasets (`data_generator/synthetic_dataset/generate_data.py`) -- and its exact
transpose (r2x_volume_backproject), TIGRE's `Atb` inside the iterative reconstructions of `r2_gaussian_b200.recon`.

    projs = project(volume, angles, scanner_cfg)                 # [N, H, W], rows = v, columns = u
    vol = backproject(projs, angles, scanner_cfg)                # [nx, ny, nz] = A^T projs
    projs = project(volume, angles, scanner_cfg, use_offDetector=True)   # through the scanner's offDetector
    vol, weight = backproject(projs, angles, scanner_cfg, weights=True)   # weight = A^T 1, from the same launch

`volume` is a CUDA float32 [nx, ny, nz] tensor in the voxelizer's layout; `scanner_cfg` is the scaled dict of
`dataset.read_scene` / `Scene.scanner_cfg`, and the result is in the same scene-scaled units (what the readers hand to
training).  The per-view geometry is the rasterizer's (`scene.make_view`), so the projections agree with render() by
construction.  Each pixel is the line integral of the volume's trilinear field, sampled every
`accuracy * min(dVoxel)` along the ray (`accuracy` defaults to 0.5, as in the reference's scanner files); the exact
definition is in include/r2x.h.  A scanner whose `offDetector` is not zero is refused unless `use_offDetector=True`,
which projects through the offset detector (the shift_u / shift_v of r2x_volume_project / r2x_volume_backproject,
TIGRE's `geo.offDetector`; the convention is `scene.detector_shift`'s) and matches a render() whose cameras carry the
same offset (`dataset.Scene(use_offDetector=True)`, `scene.make_view(..., use_offDetector=True)`).
`view_geometry=` (one dict per angle: a projection frame's overrides in scene units, `CameraInfo.view_geometry`, or a
`scene.view_scanner` dict) gives every view its own DSO, DSD, offOrigin and offDetector, as a helical scan or a
calibrated bench measures them; it implies `use_offDetector` and runs the `_views` entry points with the per-view table
of `view_table`.  Without it the scalar entry points run as before.
`backproject` sums every (ray, sample, voxel) triple `project` uses, with the same
weight, so <project(x), y> = <x, backproject(y)> up to float32 rounding.  Both run on the current stream; no CPU
fallback.  `CTOperator` binds the pair to one set of angles for repeated use (the iterative solvers).
"""
from __future__ import annotations

import numpy as np
import torch

from ._lib import check, load
from .scene import detector_shift, make_view, view_scanner

DEFAULT_ACCURACY = 0.5


def _check_geometry(what: str, scanner_cfg: dict, use_offDetector: bool = False) -> float:
    """The scanner settings the projector pair supports; returns `accuracy`."""
    accuracy = float(scanner_cfg.get("accuracy", DEFAULT_ACCURACY))
    if not accuracy > 0.0:
        raise ValueError(f"{what}: accuracy must be > 0, got {accuracy}")
    off = np.asarray(scanner_cfg.get("offDetector", [0.0, 0.0]), np.float64)
    if use_offDetector:
        if not np.all(np.isfinite(off)):
            raise ValueError(f"{what}: offDetector must be finite, got {off.tolist()}")
    elif np.any(off != 0.0):
        raise ValueError(f"{what}: offDetector must be [0, 0] without use_offDetector=True: the centred projector would "
                         "not match the scan, nor a render() of cameras without the offset")
    if scanner_cfg["mode"] != "cone" and not np.allclose(np.asarray(scanner_cfg["sDetector"], np.float64), 2.0,
                                                         rtol=1e-6, atol=0.0):
        raise ValueError(f"{what}: a parallel-beam detector must span the scene's [-1, 1] (scaled sDetector [2, 2]), "
                         f"got {list(scanner_cfg['sDetector'])}: render() could not reproduce that geometry")
    return accuracy


def view_table(angles, scanner_cfg: dict, view_geometry) -> tuple[list, np.ndarray]:
    """(views, table) of a per-view geometry: each angle's `scene.make_view` of `scene.view_scanner(scanner_cfg, g)`
    with its detector offset, and the float64 [N, 5] table of the `_views` entry points (include/r2x.h): tan_fovx,
    tan_fovy, shift_u, shift_v (`scene.detector_shift` of the view) and DSO.  Refuses a length mismatch and values the
    entry points would refuse."""
    angles = np.asarray(angles, dtype=np.float64).reshape(-1)
    view_geometry = list(view_geometry)
    if len(view_geometry) != len(angles):
        raise ValueError(f"view_geometry: {len(view_geometry)} entries for {len(angles)} angles")
    cfgs = [view_scanner(scanner_cfg, g or {}) for g in view_geometry]
    views = [make_view(c, float(a), True) for c, a in zip(cfgs, angles)]
    table = np.array([[v.tanfovx, v.tanfovy, *detector_shift(c), float(c["DSO"])] for v, c in zip(views, cfgs)],
                     dtype=np.float64).reshape(-1, 5)
    for c in cfgs:
        off, pos = c.get("offDetector", [0.0, 0.0]), c.get("offOrigin_view", c["offOrigin"])
        if not np.all(np.isfinite(np.asarray([c["DSO"], c["DSD"], *off, *pos], np.float64))):
            raise ValueError(f"view_geometry: values must be finite, got DSO {c['DSO']}, DSD {c['DSD']}, offDetector "
                             f"{off}, offOrigin {pos}")
        if c["mode"] == "cone" and not (float(c["DSO"]) > 0.0 and float(c["DSD"]) > 0.0):
            raise ValueError(f"view_geometry: cone beam needs DSO > 0 and DSD > 0, got {c['DSO']} and {c['DSD']}")
    return views, np.ascontiguousarray(table)


def project(volume: torch.Tensor, angles, scanner_cfg: dict, use_offDetector: bool = False,
            view_geometry=None) -> torch.Tensor:
    nvox = tuple(int(v) for v in scanner_cfg["nVoxel"])
    if tuple(getattr(volume, "shape", ())) != nvox:
        raise ValueError(f"project: volume shape {tuple(getattr(volume, 'shape', ()))} is not the scanner's nVoxel "
                         f"{list(nvox)}")
    _check_geometry("project", scanner_cfg, use_offDetector or view_geometry is not None)
    if not isinstance(volume, torch.Tensor) or volume.device.type != "cuda":
        raise RuntimeError("project: volume must be a CUDA tensor (this build has no CPU fallback; "
                           f"got {getattr(volume, 'device', type(volume))})")
    if np.asarray(angles, dtype=np.float64).size == 0:
        raise ValueError("project: no angles")
    return CTOperator(angles, scanner_cfg, volume.device, use_offDetector, view_geometry).A(volume)


class CTOperator:
    """A = r2x_volume_project and A^T = r2x_volume_backproject for fixed angles and scanner on one CUDA device, with the
    per-view matrices uploaded once.  `A(x, views)` projects a [nx, ny, nz] volume into the views `views` (a slice of
    the angle list) and `At(y, views, weights)` backprojects their [n, H, W] projections, returning (A_views^T y,
    A_views^T 1) when `weights` is true.  Inputs are used as float32 contiguous tensors on the operator's device.
    `use_offDetector` binds the offset-detector pair (both directions, and the offset projmatrices the backprojector's
    footprints need).  `view_geometry` binds the per-view pair (`view_table`; implies `use_offDetector`)."""

    def __init__(self, angles, scanner_cfg: dict, device, use_offDetector: bool = False, view_geometry=None):
        use_offDetector = use_offDetector or view_geometry is not None
        accuracy = _check_geometry("backproject", scanner_cfg, use_offDetector)
        angles = np.asarray(angles, dtype=np.float64).reshape(-1)
        if len(angles) == 0:
            raise ValueError("backproject: no angles")
        self.table = None
        if view_geometry is not None:
            views, self.table = view_table(angles, scanner_cfg, view_geometry)
        else:
            views = [make_view(scanner_cfg, float(a), use_offDetector) for a in angles]
        self.shift = detector_shift(scanner_cfg) if use_offDetector else (0.0, 0.0)
        self.device = torch.device(device)
        self.nvox = tuple(int(v) for v in scanner_cfg["nVoxel"])
        self.N, self.H, self.W = len(views), views[0].image_height, views[0].image_width
        self.size = tuple(float(v) for v in scanner_cfg["sVoxel"])
        self.centre = tuple(float(v) for v in scanner_cfg["offOrigin"])
        self.step = accuracy * min(s / n for s, n in zip(self.size, self.nvox))
        self.mode, self.tanx, self.tany = int(views[0].mode), float(views[0].tanfovx), float(views[0].tanfovy)
        self.vm = torch.from_numpy(np.stack([v.viewmatrix.reshape(16) for v in views])).to(self.device)
        self.pm = torch.from_numpy(np.stack([v.projmatrix.reshape(16) for v in views])).to(self.device)
        if self.table is not None:
            self.table_dev = torch.from_numpy(self.table).to(self.device)
        self.lib = load()

    def _table(self, v0: int):
        """(device, host) pointers of the per-view table from view v0."""
        return self.table_dev[v0].data_ptr(), self.table.ctypes.data + v0 * self.table.strides[0]

    def _views(self, views: slice) -> tuple[int, int]:
        v0, v1, stride = views.indices(self.N)
        if stride != 1 or v1 <= v0:
            raise ValueError(f"CTOperator: views must be a non-empty contiguous slice, got {views}")
        return v0, v1 - v0

    def A(self, x: torch.Tensor, views: slice = slice(None)) -> torch.Tensor:
        v0, n = self._views(views)
        with torch.cuda.device(self.device):
            vol = x.detach().to(self.device, torch.float32).contiguous()
            if tuple(vol.shape) != self.nvox:
                raise ValueError(f"project: volume shape {tuple(vol.shape)} is not the scanner's nVoxel {list(self.nvox)}")
            out = torch.empty((n, self.H, self.W), dtype=torch.float32, device=self.device)
            stream = torch.cuda.current_stream(self.device).cuda_stream
            if self.table is not None:
                rc = self.lib.r2x_volume_project_views(stream, *self.nvox, vol.data_ptr(), *self.size, *self.centre, n,
                                                       self.H, self.W, self.vm[v0].data_ptr(), self.mode, self.step,
                                                       *self._table(v0), out.data_ptr())
            else:
                rc = self.lib.r2x_volume_project(stream, *self.nvox, vol.data_ptr(), *self.size, *self.centre, n,
                                                 self.H, self.W, self.vm[v0].data_ptr(), self.tanx, self.tany,
                                                 self.mode, *self.shift, self.step, out.data_ptr())
        check(rc, "r2x_volume_project")
        return out

    def At(self, y: torch.Tensor, views: slice = slice(None), weights: bool = False):
        v0, n = self._views(views)
        with torch.cuda.device(self.device):
            projs = y.detach().to(self.device, torch.float32).contiguous()
            if tuple(projs.shape) != (n, self.H, self.W):
                raise ValueError(f"backproject: expected projections of shape {[n, self.H, self.W]}, "
                                 f"got {list(projs.shape)}")
            vol = torch.empty(self.nvox, dtype=torch.float32, device=self.device)
            wgt = torch.empty(self.nvox, dtype=torch.float32, device=self.device) if weights else None
            nbytes = int(self.lib.r2x_volume_backproject_scratch_bytes(n, self.H, self.W))
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
            stream = torch.cuda.current_stream(self.device).cuda_stream
            if self.table is not None:
                rc = self.lib.r2x_volume_backproject_views(stream, n, self.H, self.W, projs.data_ptr(),
                                                           self.vm[v0].data_ptr(), self.pm[v0].data_ptr(), self.mode,
                                                           *self.nvox, *self.size, *self.centre, self.step,
                                                           *self._table(v0), vol.data_ptr(),
                                                           wgt.data_ptr() if weights else None, scratch.data_ptr(),
                                                           nbytes)
            else:
                rc = self.lib.r2x_volume_backproject(stream, n, self.H, self.W, projs.data_ptr(),
                                                     self.vm[v0].data_ptr(), self.pm[v0].data_ptr(), self.tanx,
                                                     self.tany, self.mode, *self.shift, *self.nvox, *self.size,
                                                     *self.centre, self.step, vol.data_ptr(),
                                                     wgt.data_ptr() if weights else None, scratch.data_ptr(), nbytes)
        check(rc, "r2x_volume_backproject")
        return (vol, wgt) if weights else vol


def backproject(projections: torch.Tensor, angles, scanner_cfg: dict, weights: bool = False,
                use_offDetector: bool = False, view_geometry=None):
    """A^T projections for the projector of `project(., angles, scanner_cfg, use_offDetector, view_geometry)`:
    [nx, ny, nz], or (volume, A^T 1) when `weights` is true."""
    shape = tuple(getattr(projections, "shape", ()))
    if len(shape) != 3:
        raise ValueError(f"backproject: expected projections of shape [N, H, W], got {shape}")
    n_angles = np.asarray(angles, dtype=np.float64).reshape(-1).size
    if shape[0] != n_angles:
        raise ValueError(f"backproject: {shape[0]} projections but {n_angles} angles")
    det = (int(scanner_cfg["nDetector"][0]), int(scanner_cfg["nDetector"][1]))
    if shape[1:] != det:
        raise ValueError(f"backproject: projections are {shape[1]}x{shape[2]}, scanner nDetector is {list(det)}")
    _check_geometry("backproject", scanner_cfg, use_offDetector or view_geometry is not None)
    if not isinstance(projections, torch.Tensor) or projections.device.type != "cuda":
        raise RuntimeError("backproject: projections must be a CUDA tensor (this build has no CPU fallback; "
                           f"got {getattr(projections, 'device', type(projections))})")
    return CTOperator(angles, scanner_cfg, projections.device, use_offDetector, view_geometry).At(projections,
                                                                                                 slice(None), weights)
