"""FDK reconstruction on the GPU over the C ABI (r2x_fdk) -- what the reference obtains from TIGRE's `algs.fdk`
(`r2_gaussian/utils/ct_utils.py::recon_volume`) to initialise its point cloud.

    vol = fdk(projections, angles, scanner_cfg)                    # [nx, ny, nz], the voxelizer's layout
    vol = fdk(projections, angles, scanner_cfg, short_scan=True)   # Parker-weighted, for an arc short of 360 degrees
    vol = fdk(projections, angles, scanner_cfg, use_offDetector=True, half_fan=True)   # offset detector, 360 degrees
    vol = fdk(projections, angles, scanner_cfg, filter="hann")     # Hann-windowed ramp filter

`projections` is a CUDA float32 [N, H, W] tensor in the dataset layout (rows = v, columns = u, already multiplied by
scene_scale); `scanner_cfg` is the scaled dict of `dataset.read_scene` / `Scene.scanner_cfg`.  The per-view geometry is
the rasterizer's (`scene.make_view`), so the reconstruction agrees with render() on detector orientation, axis order and
angle convention by construction.  Runs on the current stream; no CPU fallback.

The ramp filter is the band-limited Ram-Lak filter unless `filter=` names one of TIGRE's windowed filters
(`FILTERS`: "ram_lak", "shepp_logan", "cosine", "hamming", "hann", the names of TIGRE's `geo.filter`).  A window damps
the ramp towards Nyquist, which passes less detector noise into the volume at some cost in resolution; it changes the
filter taps only (r2x_fdk's filter field), so it combines with every weighting below and any offset.  The keyword
overrides the scanner's `filter`.  Without it the scanner's `filter` must be null or "ram_lak", and a window named
there is refused rather than silently replaced by Ram-Lak: reconstructing with it is opt-in, as for `use_offDetector`.
The definition is stated in float64 in tests/fdk_window_oracle.py.

The plain path weights every view by pi / N, which assumes each ray is measured twice: right for a full 360-degree scan
and a 180-degree parallel scan, not for a cone-beam short scan (180 degrees plus the fan angle), which it reconstructs
as a full one with low-frequency shading, as TIGRE's default fdk does.  `short_scan=True` runs r2x_fdk with
R2X_FDK_PARKER instead: Parker redundancy weights (Parker 1982, in Silver 2000's overscan form) and each view's own
angular interval, from `short_scan_views`.  It refuses fewer than 2 views, an arc shorter than 180 degrees plus the fan
angle and a full circle.  The definition is stated in float64 in tests/fdk_short_scan_oracle.py (the plain FDK's in
oracle/fdk_oracle.py).

Without `use_offDetector` the scanner's `offDetector` is ignored (with a warning when it is not zero): the volume is
reconstructed as if the detector were centred.  `use_offDetector=True` reconstructs through the offset detector
(r2x_fdk's shift_u / shift_v, TIGRE's `geo.offDetector`; the convention is `scene.detector_shift`'s):
the cosine weight is taken at each pixel's offset position and the backprojection goes through the offset matrices.
A short scan allows a vertical offset only.  `half_fan=True` (with `use_offDetector`) is for a full-circle scan whose
detector is shifted sideways to widen the field of view: rays near the axis are measured twice and the outer rays once,
and Wang's (2002) redundancy weights (`half_fan_weight`) give each its share, where the plain FDK would reconstruct the
outer part at about half its density.  It refuses a centred axis, an axis not strictly inside the detector, views that
do not cover a full circle and a short scan.  The float64 statement is tests/offset_detector_oracle.py.
"""
from __future__ import annotations

import math
import warnings

import numpy as np
import torch

from ._lib import check, load
from .scene import MODE_CONE, detector_shift, make_view

# the scanner filters fdk reconstructs without its `filter` keyword
SUPPORTED_FILTERS = (None, "ram_lak")
# the filters of the `filter` keyword (TIGRE's names); r2x_fdk's filter field is the index << 8 (include/r2x.h)
FILTERS = ("ram_lak", "shepp_logan", "cosine", "hamming", "hann")
R2X_FDK_PLAIN, R2X_FDK_PARKER, R2X_FDK_HALF_FAN = 0, 1, 2   # r2x_fdk's weighting (include/r2x.h)
# slack on the arc refusals: a scan sampled at linspace(0, pi, n + 1)[:-1] covers pi only up to rounding
ARC_TOLERANCE = 1e-9


def _arc_positions(angles):
    """(beta, arc): each view's position (radians) from the start of the scan, which the largest circular gap between
    the angles marks, and the arc beta_max + D the views cover with the mean step D = beta_max / (N - 1).  N >= 2."""
    theta = np.mod(np.asarray(angles, np.float64).reshape(-1), 2.0 * math.pi)
    N = len(theta)
    s = np.sort(theta)
    gaps = np.append(np.diff(s), s[0] + 2.0 * math.pi - s[-1])
    start = s[(int(np.argmax(gaps)) + 1) % N]
    beta = np.mod(theta - start, 2.0 * math.pi)
    return beta, beta.max() + beta.max() / (N - 1)


def scan_arc(angles) -> float:
    """The arc (radians) that views at `angles` cover: the circle less its largest gap between the angles, plus the
    mean step between the views (the arc of `short_scan_views`; linspace(0, R, n + 1)[:-1] gives R)."""
    if np.asarray(angles).size < 2:
        return 0.0
    return float(_arc_positions(angles)[1])


def half_fan_weight(a, t_u: float, W: int, fan: float):
    """Wang's (2002) redundancy weight of the ray at fan coordinate `a` (tan of its fan angle for cone beam, ndc for
    parallel beam) on a full circle whose detector is offset by t_u pixels: delta = (1 - 2 |t_u| / W) fan is the
    half-width of the part of the detector symmetric about the axis, sigma = sign(t_u), and
    w(a) = 2 sin^2(pi/4 (1 + sigma a / delta)) for |a| <= delta, 2 beyond delta on the wide side (0 beyond it on the
    narrow side, where no pixel lies).  w(a) + w(-a) = 2, so a ray measured twice keeps the plain FDK's weight."""
    check_half_fan_shift(t_u, W)
    delta = (1.0 - 2.0 * abs(t_u) / W) * fan
    x = np.clip(math.copysign(1.0, t_u) * np.asarray(a, np.float64) / delta, -1.0, 1.0)
    return 2.0 * np.sin(0.25 * math.pi * (1.0 + x)) ** 2


def check_half_fan_shift(t_u: float, W: int):
    if t_u == 0.0:
        raise ValueError("fdk half fan: the detector is centred (offDetector[0] = 0): every ray is measured twice, so "
                         "use fdk without half_fan")
    if not abs(t_u) < 0.5 * W:
        raise ValueError(f"fdk half fan: the rotation axis is not strictly inside the detector (offset of {t_u:g} "
                         f"pixels on a detector {W} pixels wide needs |offset| < {0.5 * W:g})")


def short_scan_views(angles, mode: int, tan_fovx: float):
    """(view_weights [N, 2] float64 of (beta'_v, dbeta_v), arc B) of a short scan with the views at `angles` (radians,
    any order), after the refusals.  The largest circular gap between the angles marks the start of the scan; view v
    sits at beta_v = (theta_v - theta_start) mod 2 pi and stands for an interval of the mean step D = beta_max / (N - 1)
    around it, so beta'_v = beta_v + D / 2 and B = beta_max + D (`linspace(0, R, n + 1)[:-1]` gives B = R).  dbeta_v
    runs between the midpoints of the sorted beta' (0 and B at the ends); views at the same angle share theirs."""
    N = np.asarray(angles).size
    if N < 2:
        raise ValueError(f"fdk short scan: needs at least 2 views, got {N}")
    beta, arc = _arc_positions(angles)
    bp = beta + 0.5 * (beta.max() / (N - 1))
    gamma_max = math.atan(tan_fovx) if mode == MODE_CONE else 0.0
    need = math.pi + 2.0 * gamma_max
    if arc < need - ARC_TOLERANCE:
        raise ValueError(f"fdk short scan: the views cover an arc of {math.degrees(arc):.2f} degrees, a short scan needs "
                         f"at least {math.degrees(need):.2f} (180 plus the fan angle {math.degrees(2 * gamma_max):.2f})")
    if arc >= 2.0 * math.pi - ARC_TOLERANCE:
        raise ValueError(f"fdk short scan: the views cover an arc of {math.degrees(arc):.2f} degrees, a full circle, "
                         "which needs no redundancy weights: use fdk without short_scan")
    u, inv, count = np.unique(bp, return_inverse=True, return_counts=True)
    edges = np.concatenate([[0.0], 0.5 * (u[1:] + u[:-1]), [arc]])
    dbeta = (np.diff(edges) / count)[inv]
    return np.stack([bp, dbeta], 1), arc


def check_filter(filter, scanner_cfg: dict) -> str:
    """The filter fdk reconstructs with: `filter` (one of FILTERS) when given, else the scanner's, which must then be
    null or "ram_lak"."""
    if filter is not None:
        if filter not in FILTERS:
            raise ValueError(f"fdk: unknown filter {filter!r} (supported: {', '.join(FILTERS)})")
        return filter
    filt = scanner_cfg.get("filter")
    if filt in SUPPORTED_FILTERS:
        return "ram_lak"
    if filt in FILTERS:
        raise ValueError(f"fdk: the scanner's filter {filt!r} is used only on request: pass filter={filt!r} "
                         f"(--fdk_filter {filt} on the command lines); without it fdk reconstructs with the Ram-Lak "
                         "filter only (null or 'ram_lak')")
    raise ValueError(f"fdk: the scanner's filter {filt!r} is not supported (supported: null, {', '.join(FILTERS)})")


def fdk(projections: torch.Tensor, angles, scanner_cfg: dict, short_scan: bool = False, use_offDetector: bool = False,
        half_fan: bool = False, filter: str | None = None) -> torch.Tensor:
    filt = check_filter(filter, scanner_cfg)
    if half_fan and not use_offDetector:
        raise ValueError("fdk: half_fan needs use_offDetector=True (the half-fan weights follow the detector offset)")
    if half_fan and short_scan:
        raise ValueError("fdk: half_fan and short_scan cannot be combined (half-fan weights need a full circle, a short "
                         "scan's Parker weights a centred detector)")
    t_u, t_v = detector_shift(scanner_cfg) if use_offDetector else (0.0, 0.0)
    if not use_offDetector and np.any(np.asarray(scanner_cfg.get("offDetector", [0.0, 0.0]), np.float64) != 0.0):
        warnings.warn("fdk: the scanner's offDetector is not zero and is ignored (the volume is reconstructed as if the "
                      "detector were centred); pass use_offDetector=True to use it", stacklevel=2)
    if not (math.isfinite(t_u) and math.isfinite(t_v)):
        raise ValueError(f"fdk: offDetector must be finite, got {scanner_cfg.get('offDetector')}")
    if short_scan and t_u != 0.0:
        raise ValueError(f"fdk short scan: the detector has a horizontal offset of {t_u:g} pixels; Parker weights assume "
                         "that each ray's conjugate is on the detector, so a short scan allows a vertical offset only")
    if half_fan:
        check_half_fan_shift(t_u, int(scanner_cfg["nDetector"][1]))
        arc = scan_arc(angles)
        if arc < 2.0 * math.pi - ARC_TOLERANCE:
            raise ValueError(f"fdk half fan: the views cover an arc of {math.degrees(arc):.2f} degrees; half-fan "
                             "weights need a full circle")
    if not isinstance(projections, torch.Tensor) or projections.device.type != "cuda":
        raise RuntimeError("fdk: projections must be a CUDA tensor (this build has no CPU fallback; "
                           f"got {getattr(projections, 'device', type(projections))})")
    if projections.dim() != 3:
        raise ValueError(f"fdk: expected projections of shape [N, H, W], got {tuple(projections.shape)}")
    angles = np.asarray(angles, dtype=np.float64).reshape(-1)
    N, H, W = (int(s) for s in projections.shape)
    if len(angles) != N:
        raise ValueError(f"fdk: {N} projections but {len(angles)} angles")
    if (H, W) != (int(scanner_cfg["nDetector"][0]), int(scanner_cfg["nDetector"][1])):
        raise ValueError(f"fdk: projections are {H}x{W}, scanner nDetector is {list(scanner_cfg['nDetector'])}")
    if N == 0:
        raise ValueError("fdk: no projections")
    views = [make_view(scanner_cfg, float(a), use_offDetector) for a in angles]
    mode = views[0].mode
    weighting, view_weights, arc = (R2X_FDK_HALF_FAN if half_fan else R2X_FDK_PLAIN), None, 0.0
    if short_scan:
        weighting = R2X_FDK_PARKER
        view_weights, arc = short_scan_views(angles, mode, float(views[0].tanfovx))
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
        stream = torch.cuda.current_stream(dev).cuda_stream
        vw = None if view_weights is None else torch.from_numpy(view_weights.astype(np.float32)).to(dev)
        rc = lib.r2x_fdk(stream, N, H, W, projs.data_ptr(), vm.data_ptr(), pm.data_ptr(), float(views[0].tanfovx),
                         float(views[0].tanfovy), int(mode), t_u, t_v, weighting | (FILTERS.index(filt) << 8),
                         None if vw is None else vw.data_ptr(), float(arc), float(scanner_cfg["DSO"]), nx, ny, nz, sx,
                         sy, sz, cx, cy, cz, vol.data_ptr(), scratch.data_ptr(), nbytes)
    check(rc, "r2x_fdk")
    return vol
