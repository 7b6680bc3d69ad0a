"""FDK reconstruction on the GPU over the C ABI (r2x_fdk) -- what the reference obtains from TIGRE's `algs.fdk`
(`r2_gaussian/utils/ct_utils.py::recon_volume`) to initialise its point cloud.

    vol = fdk(projections, angles, scanner_cfg)                    # [nx, ny, nz], the voxelizer's layout
    vol = fdk(projections, angles, scanner_cfg, short_scan=True)   # Parker-weighted, for an arc short of 360 degrees
    vol = fdk(projections, angles, scanner_cfg, use_offDetector=True, half_fan=True)   # offset detector, 360 degrees
    vol = fdk(projections, angles, scanner_cfg, filter="hann")     # Hann-windowed ramp filter
    vol = fdk(projections, angles, scanner_cfg, pad=0.5)           # object wider than the field of view

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

`view_geometry=` (one dict per view, as for `projector.project`) reconstructs a calibrated circle whose DSO, DSD and
offDetector are measured per view (r2x_fdk_views: each view's cosine weight, isocentre pitch and (DSO / z)^2 weight
from its own row of the table).  It implies `use_offDetector`.  Plain FDK has no helical weighting, so a table whose
offOrigin varies between views (a helical scan) is refused, as are `short_scan` and `half_fan`: cgls, sart, fista_tv
and cp_tv (`recon`) are exact for any geometry, and `helical=True` is FDK's approximate answer.

`helical=True` (with `view_geometry`) reconstructs a helical scan with Tang et al.'s (2006) three-dimensional weighted
FDK (r2x_fdk_helical; model in include/r2x.h, float64 statement in tests/fdk_helical_oracle.py).  The filter is the
plain FDK's (any `filter=`); the backprojection weights each view of a voxel by W_Q of its detector row over the sum of
W_Q over every measurement of the same in-plane line (its other turns and its conjugate rays), where W_Q is 1 within
`helical_q` of the detector's centre (as a fraction of its half-height) and falls as cos^2 to 0 at its edge.
`helix_views` fits the helix z_s = z0 + h beta to the views; it needs one DSO and DSD, a centred detector, one
offOrigin x / y, an arc of at least 360 degrees and cone beam.  The views are reconstructed in beta order.  Pitch 0 (a
circle of 360 degrees or more) is allowed.  `helical` is refused with `short_scan` and `half_fan`.

`pad=F` (0 <= F <= 1) reconstructs a laterally truncated scan, one whose object is wider than the detector's field of
view (r2x_fdk_pad; model in include/r2x.h, float64 statement in tests/fdk_pad_oracle.py).  Each weighted row is
extended by L = round(F W) pixels on each side, a mirror of the row about its edge rolled off to zero by
(1 + cos(pi k / (L + 1))) / 2, before the ramp filter; only the W measured pixels are backprojected.  Without it the
filter sees a step at each edge of a truncated row, which shows as a bright rim at the edge of the field of view and
cupping inside it.  It combines with any filter and with `short_scan`; it is refused with `half_fan` (the offset
detector's truncation is deliberate and its weights handle it), `helical` and `view_geometry`.  pad=0 (the default)
runs the unpadded FDK.
"""
from __future__ import annotations

import math
import warnings

import numpy as np
import torch

from ._lib import check, load
from .scene import MODE_CONE, detector_shift, make_view, view_scanner

# the scanner filters fdk reconstructs without its `filter` keyword
SUPPORTED_FILTERS = (None, "ram_lak")
# the filters of the `filter` keyword (TIGRE's names); r2x_fdk's filter field is the index << 8 (include/r2x.h)
FILTERS = ("ram_lak", "shepp_logan", "cosine", "hamming", "hann")
R2X_FDK_PLAIN, R2X_FDK_PARKER, R2X_FDK_HALF_FAN = 0, 1, 2   # r2x_fdk's weighting (include/r2x.h)
# helical FDK: W_Q's default Q (DESIGN §8 measures psnr_3d against Q), and the largest residual of the helix fit, in
# voxels along z
HELICAL_Q = 0.75
HELIX_FIT_TOLERANCE = 1e-3
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


def helical(scanner_cfg: dict, view_geometry) -> bool:
    """Whether the volume's position offOrigin varies between the views of a per-view geometry."""
    pos = np.array([view_scanner(scanner_cfg, g or {}).get("offOrigin_view", scanner_cfg["offOrigin"])
                    for g in view_geometry], np.float64).reshape(-1, 3)
    return bool(len(pos) and np.any(pos != pos[0]))


def check_view_geometry(scanner_cfg: dict, view_geometry, short_scan: bool = False, half_fan: bool = False,
                        helical_fdk: bool = False):
    """The refusals of fdk's per-view geometry: Parker or half-fan weights, and an offOrigin that varies between
    views without `helical_fdk` (the plain FDK has no helical weighting)."""
    for flag, on in (("short_scan", short_scan), ("half_fan", half_fan)):
        if on:
            raise ValueError(f"fdk: {flag} cannot be combined with view_geometry (its redundancy weights assume one fixed "
                             "circle)")
    if not helical_fdk and helical(scanner_cfg, view_geometry):
        raise ValueError("fdk: the views' offOrigin varies (a helical scan) and FDK has no helical weighting: "
                         "reconstruct with cgls, sart, fista_tv or cp_tv, which are exact for any geometry, or pass "
                         "helical=True for FDK's approximate helical weighting")


class Helix:
    """The helix of `helix_views`: `order` sorts the views into beta order; `beta` (float64, strictly increasing) and
    `dbeta` are the sorted views' unwrapped angles and quadrature intervals; the source height is z0 + h beta over the
    arc [beta_lo, beta_hi); (c_x, c_y) is the rotation centre in the grid frame."""

    def __init__(self, order, beta, dbeta, z0, h, beta_lo, beta_hi, c_x, c_y):
        self.order, self.beta, self.dbeta = order, beta, dbeta
        self.z0, self.h, self.beta_lo, self.beta_hi, self.c_x, self.c_y = z0, h, beta_lo, beta_hi, c_x, c_y


def helix_views(angles, scanner_cfg: dict, view_geometry) -> Helix:
    """Fit a helix to a per-view geometry.  View v's source sits at (DSO cos a_v, DSO sin a_v) + (c_x, c_y) and at
    height z_v = offOrigin_z - offOrigin_v,z (`scene.camera_pose`).  The views are sorted by z_v (then by angle mod
    2 pi), their angles unwrapped in that order (reversed if they then decrease), and z = z0 + h beta is fitted by least
    squares.  The arc runs half a mean step beyond the first and last view; dbeta_v runs between the midpoints of its
    neighbours.  Refuses fewer than 2 views, parallel beam, DSO, DSD or offDetector that vary, a non-zero offDetector,
    an x / y offOrigin that varies, angles that do not advance monotonically along z, a fit residual above
    HELIX_FIT_TOLERANCE voxels and an arc shorter than 360 degrees."""
    angles = np.asarray(angles, np.float64).reshape(-1)
    view_geometry = list(view_geometry)
    N = len(angles)
    if len(view_geometry) != N:
        raise ValueError(f"fdk helical: {len(view_geometry)} view_geometry entries for {N} angles")
    if N < 2:
        raise ValueError(f"fdk helical: needs at least 2 views, got {N}")
    if scanner_cfg["mode"] != "cone":
        raise ValueError("fdk helical: cone beam only (parallel-beam helices are not supported)")
    cfgs = [view_scanner(scanner_cfg, g or {}) for g in view_geometry]
    for key in ("DSO", "DSD"):
        vals = np.array([float(c[key]) for c in cfgs])
        if np.any(vals != vals[0]):
            raise ValueError(f"fdk helical: the views' {key} varies ({vals.min():g} .. {vals.max():g}); the helical "
                             "weights need one circle radius and one detector distance")
    off = np.array([[float(v) for v in c.get("offDetector", [0.0, 0.0])] for c in cfgs]).reshape(-1, 2)
    if np.any(off != off[0]):
        raise ValueError("fdk helical: the views' offDetector varies; the helical weights need a centred detector")
    if np.any(off != 0.0):
        raise ValueError(f"fdk helical: the detector is offset (offDetector {off[0].tolist()}); the helical weights "
                         "need a centred detector")
    grid = np.asarray(scanner_cfg["offOrigin"], np.float64)
    pos = np.array([c.get("offOrigin_view", scanner_cfg["offOrigin"]) for c in cfgs], np.float64).reshape(-1, 3)
    if not np.all(np.isfinite(pos)) or not np.all(np.isfinite(angles)):
        raise ValueError("fdk helical: angles and offOrigin must be finite")
    if np.any(pos[:, :2] != pos[0, :2]):
        raise ValueError("fdk helical: the views' offOrigin x / y varies; a helix moves the volume along the rotation "
                         "axis only")
    z = grid[2] - pos[:, 2]
    order = np.lexsort((np.mod(angles, 2.0 * math.pi), z))
    beta = np.unwrap(angles[order])
    if beta[-1] < beta[0]:
        order, beta = order[::-1], beta[::-1]
    if not np.all(np.diff(beta) > 0.0):
        raise ValueError("fdk helical: the views' angles do not advance monotonically along the helix (sorted by the "
                         "volume's z, the unwrapped angles must strictly increase or decrease)")
    zs = z[order]
    dz = float(scanner_cfg["sVoxel"][2]) / float(scanner_cfg["nVoxel"][2])
    if np.max(np.abs(zs - zs.mean())) <= HELIX_FIT_TOLERANCE * dz:
        h, z0 = 0.0, float(zs.mean())
    else:
        A = np.stack([np.ones(N), beta], 1)
        (z0, h), *_ = np.linalg.lstsq(A, zs, rcond=None)
        z0, h = float(z0), float(h)
    resid = float(np.max(np.abs(zs - (z0 + h * beta))))
    if resid > HELIX_FIT_TOLERANCE * dz:
        raise ValueError(f"fdk helical: the volume's z is not affine in the view angle (a residual of {resid / dz:.3g} "
                         f"voxels after fitting z = z0 + h beta; at most {HELIX_FIT_TOLERANCE:g})")
    step = (beta[-1] - beta[0]) / (N - 1)
    beta_lo, beta_hi = beta[0] - 0.5 * step, beta[-1] + 0.5 * step
    if beta_hi - beta_lo < 2.0 * math.pi - ARC_TOLERANCE:
        raise ValueError(f"fdk helical: the views cover an arc of {math.degrees(beta_hi - beta_lo):.2f} degrees; the "
                         "helical weights need at least 360 (a circular short scan takes short_scan=True)")
    edges = np.concatenate([[beta_lo], 0.5 * (beta[1:] + beta[:-1]), [beta_hi]])
    c = grid[:2] - pos[0, :2]
    return Helix(order, beta, np.diff(edges), z0, h, float(beta_lo), float(beta_hi), float(c[0]), float(c[1]))


def check_pad(pad, half_fan: bool = False, helical: bool = False, view_geometry=None) -> float:
    """The refusals of fdk's `pad`: a number outside [0, 1], and a non-zero pad with half_fan, helical or
    view_geometry (r2x_fdk_views and r2x_fdk_helical take no pad)."""
    if isinstance(pad, bool) or not isinstance(pad, (int, float)) or not 0.0 <= float(pad) <= 1.0:
        raise ValueError(f"fdk: pad must be a fraction of the detector width in [0, 1], got {pad!r}")
    pad = float(pad)
    if pad > 0.0:
        for flag, on, why in (("half_fan", half_fan, "an offset detector's truncation is deliberate and its weights "
                               "already handle it"),
                              ("helical", helical, "the helical FDK has no truncation pad"),
                              ("view_geometry", view_geometry is not None, "the per-view FDK has no truncation pad")):
            if on:
                raise ValueError(f"fdk: pad cannot be combined with {flag} ({why})")
    return pad


def pad_pixels(pad: float, W: int) -> int:
    """L = round(pad W), halves rounded up: the pixels fdk(pad=...) adds on each side of a row of W."""
    return int(math.floor(float(pad) * W + 0.5))


def fdk(projections: torch.Tensor, angles, scanner_cfg: dict, short_scan: bool = False, use_offDetector: bool = False,
        half_fan: bool = False, filter: str | None = None, view_geometry=None, helical: bool = False,
        helical_q: float = HELICAL_Q, pad: float = 0.0) -> torch.Tensor:
    filt = check_filter(filter, scanner_cfg)
    pad = check_pad(pad, half_fan, helical, view_geometry)
    if helical:
        for flag, on in (("short_scan", short_scan), ("half_fan", half_fan)):
            if on:
                raise ValueError(f"fdk: helical cannot be combined with {flag} (its redundancy weights assume one fixed "
                                 "circle)")
        if view_geometry is None:
            raise ValueError("fdk: helical needs view_geometry (the helix is read from the views' offOrigin)")
        if not (isinstance(helical_q, (int, float)) and 0.0 <= float(helical_q) <= 1.0):
            raise ValueError(f"fdk: helical_q must be in [0, 1], got {helical_q!r}")
    if view_geometry is not None:
        check_view_geometry(scanner_cfg, view_geometry, short_scan, half_fan, helical)
        use_offDetector = True
    if helical:
        return _fdk_helical(projections, angles, scanner_cfg, filt, list(view_geometry), float(helical_q))
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
    table = None
    if view_geometry is not None:
        from .projector import view_table
        views, table = view_table(angles, scanner_cfg, view_geometry)
    else:
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
        if table is not None:
            table_dev = torch.from_numpy(table).to(dev)
            rc = lib.r2x_fdk_views(stream, N, H, W, projs.data_ptr(), vm.data_ptr(), pm.data_ptr(), int(mode),
                                   weighting | (FILTERS.index(filt) << 8), nx, ny, nz, sx, sy, sz, cx, cy, cz,
                                   table_dev.data_ptr(), table.ctypes.data, vol.data_ptr(), scratch.data_ptr(), nbytes)
        else:
            L = pad_pixels(pad, W)
            args = (stream, N, H, W, projs.data_ptr(), vm.data_ptr(), pm.data_ptr(), float(views[0].tanfovx),
                    float(views[0].tanfovy), int(mode), t_u, t_v, weighting | (FILTERS.index(filt) << 8),
                    None if vw is None else vw.data_ptr(), float(arc), float(scanner_cfg["DSO"]), nx, ny, nz, sx, sy,
                    sz, cx, cy, cz, vol.data_ptr(), scratch.data_ptr(), nbytes)
            rc = lib.r2x_fdk_pad(*args, L) if L > 0 else lib.r2x_fdk(*args)
    check(rc, "r2x_fdk")
    return vol


def _fdk_helical(projections, angles, scanner_cfg: dict, filt: str, view_geometry, q: float) -> torch.Tensor:
    """fdk(helical=True) after the keyword refusals: the helix fit, the views in beta order, r2x_fdk_helical."""
    hx = helix_views(angles, scanner_cfg, view_geometry)
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
    from .projector import view_table
    views, table = view_table(angles[hx.order], scanner_cfg, [view_geometry[i] for i in hx.order])
    nx, ny, nz = (int(v) for v in scanner_cfg["nVoxel"])
    sx, sy, sz = (float(v) for v in scanner_cfg["sVoxel"])
    cx, cy, cz = (float(v) for v in scanner_cfg["offOrigin"])
    dev = projections.device
    lib = load()
    with torch.cuda.device(dev):
        order = torch.from_numpy(np.ascontiguousarray(hx.order)).to(dev)
        projs = projections.detach().to(torch.float32).index_select(0, order).contiguous()
        vm = torch.from_numpy(np.stack([v.viewmatrix.reshape(16) for v in views])).to(dev)
        pm = torch.from_numpy(np.stack([v.projmatrix.reshape(16) for v in views])).to(dev)
        beta_host = np.ascontiguousarray(hx.beta, np.float64)
        beta = torch.from_numpy(beta_host).to(dev)
        dbeta = torch.from_numpy(np.ascontiguousarray(hx.dbeta, np.float64)).to(dev)
        vol = torch.empty((nx, ny, nz), dtype=torch.float32, device=dev)
        nbytes = int(lib.r2x_fdk_scratch_bytes(N, H, W))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        stream = torch.cuda.current_stream(dev).cuda_stream
        rc = lib.r2x_fdk_helical(stream, N, H, W, projs.data_ptr(), vm.data_ptr(), pm.data_ptr(),
                                 float(table[0, 0]), float(table[0, 1]), int(views[0].mode), FILTERS.index(filt) << 8,
                                 float(table[0, 4]), beta.data_ptr(), dbeta.data_ptr(), beta_host.ctypes.data, hx.z0,
                                 hx.h, hx.beta_lo, hx.beta_hi, hx.c_x, hx.c_y, q, nx, ny, nz, sx, sy, sz, cx, cy, cz,
                                 vol.data_ptr(), scratch.data_ptr(), nbytes)
    check(rc, "r2x_fdk_helical")
    return vol
