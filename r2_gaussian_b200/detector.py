"""The horizontal detector offset of a scan (centre-of-rotation offset), learned with the scene.

The most common geometry error of a real cone-beam scan is one constant shift of the detector across the rotation
axis, the same in every view.  Unlike a per-view pose error it is well posed in a full rotation: a scene translation
moves the projections sinusoidally with the angle, so no static scene fakes a shift that is constant over all views.

`DetectorOffset(device)` holds `offset`, a leaf tensor [1] (zero at start): s, the shift in detector pixels.

Convention.  s > 0 when the measured images show their content s columns towards LARGER column index than the
nominal geometry predicts.  In scene units at the detector that is s * sDetector[1] / nDetector[1] (`scene_units`).
Scanner files store nDetector / sDetector / dDetector as [v, u] but offDetector as [u, v] (the reference's
scanner yml comments index 0 "u direction"; its ct_utils hands TIGRE geo.offDetector = [cfg[1], cfg[0]], TIGRE's own
[v, u] order).  TIGRE places detector column j at u = dDetector_u * (j - nDetector_u / 2 + 0.5) + offDetector_u, and
image columns run along u (the reference flips only v), so a detector mounted with a horizontal offset d shows its
content d / dDetector_u columns towards SMALLER index: the learned offset corresponds to the scanner file's
offDetector[0] (u; TIGRE's geo.offDetector[1]) = -s * dDetector[1] = -s * sDetector[1] / nDetector[1]
(`scene.detector_shift`'s t_u = -s).  The learned offset is reported, not written back into the scene: put it into the
scanner file and run the projector, FDK and training with `use_offDetector` (`--use_offDetector`).  With
`trainer --use_offDetector` the learned s acts on top of the file's offset.

The map.  The shift moves the detector, not the source: every ray, conic and mu stays the same, and only each
Gaussian's 2-D mean moves by s pixels along u.  Since the rasterizer maps ndc to pixels by ((x / w + 1) W - 1) / 2,
the shifted full projection is the camera's with its x row plus (2 s / W) times its w row (`r2x_detector_offset_apply`,
float64, rounded once; s = 0 gives the camera's matrix bit for bit).  With cull, radii and tile rectangles held fixed
(the convention of every per-Gaussian gradient),

    dL/ds = sum over views and Gaussians of dL/dpix_x = (2 / W) sum dL_dmean2D.x

(`r2x_detector_offset_grad`: a fixed-order float64 sum, bitwise reproducible).  dL_dmean2D is what every raster
backward already writes -- `viewspace_points.grad` of `render()`, the [B, P, 3] one of a batched render -- so no
matrix gradient is needed and batches of views work.

In a custom loop:

    det = DetectorOffset("cuda")
    det_opt = FusedAdam([det.offset], lr=2e-2, eps=1e-15)
    pkg = render(det.camera(cam), gaussians, pipe)
    loss(pkg["render"], gt).backward()
    det.grad_from(pkg["viewspace_points"].grad, cam.image_width)     # writes det.offset.grad
    det_opt.step(); det_opt.zero_grad()

`NativeTrainStep(detector=(det, det_opt))` and `trainer --detector_offset_refine` do the same on the device.  Not
supported together with pose refinement or Gaussian sharding (each rank would see only its shard's part of the sum).
"""
from __future__ import annotations

import copy

import torch

from ._lib import check, load

SIGN_CONVENTION = ("offset_px > 0: the measured projections show their content offset_px columns towards larger column "
                   "index than the nominal geometry predicts; offset_scene = offset_px * sDetector[1] / nDetector[1] "
                   "(scene units at the detector); a scanner file would carry offDetector[0] (u; TIGRE geo.offDetector[1]) = "
                   "-offset_scene")


class DetectorOffset:
    """One horizontal detector offset in pixels, `offset` (leaf float32 tensor [1] on `device`, zero at start)."""

    def __init__(self, device=None):
        self.offset = torch.nn.Parameter(torch.zeros(1, dtype=torch.float32, device=device))

    def _check(self):
        p = self.offset
        if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous() or p.shape != (1,):
            raise RuntimeError("DetectorOffset: offset must be a contiguous float32 CUDA tensor of shape [1]")
        return p.device

    def apply(self, full: torch.Tensor, W: int) -> torch.Tensor:
        """Full projections [..., 4, 4] (n matrices) with the offset applied, in one launch; not differentiable (the
        gradient comes from `grad_from`)."""
        dev = self._check()
        full = full.detach()
        if full.dtype != torch.float32 or full.device != dev or not full.is_contiguous():
            full = full.to(device=dev, dtype=torch.float32).contiguous()
        if full.numel() == 0 or full.numel() % 16 != 0 or full.shape[-2:] != (4, 4):
            raise ValueError("DetectorOffset: full projections must have shape [..., 4, 4]")
        out = torch.empty_like(full)
        with torch.cuda.device(dev):
            check(load().r2x_detector_offset_apply(torch.cuda.current_stream(dev).cuda_stream, self.offset.data_ptr(),
                                                   int(W), full.numel() // 16, full.data_ptr(), out.data_ptr()),
                  "r2x_detector_offset_apply")
        return out

    def camera(self, cam):
        """A copy of `cam` whose full_proj_transform carries the offset (bit for bit the camera's at zero)."""
        return self.cameras([cam])[0]

    def cameras(self, cams):
        """Copies of `cams` (one image width) with the offset applied, in one launch."""
        cams = list(cams)
        if not cams:
            return []
        W = int(cams[0].image_width)
        if any(int(c.image_width) != W for c in cams):
            raise ValueError("DetectorOffset.cameras: the cameras must share one image width")
        full = self.apply(torch.stack([c.full_proj_transform.detach().reshape(4, 4) for c in cams]), W)
        out = []
        for c, f in zip(cams, full):
            o = copy.copy(c)
            o.full_proj_transform = f
            out.append(o)
        return out

    def grad_from(self, dL_dmean2D: torch.Tensor, W: int) -> torch.Tensor:
        """Write offset.grad = (2 / W) sum of dL_dmean2D[..., 0] over [P, 3] (one view) or [B, P, 3] (B views) and
        return it.  `dL_dmean2D` is `viewspace_points.grad` of the render made with `camera()` / `cameras()`."""
        dev = self._check()
        g = dL_dmean2D
        if g is None:
            raise ValueError("DetectorOffset.grad_from: no screen-space gradient (was backward() called?)")
        if g.dim() == 2:
            g = g.unsqueeze(0)
        if g.dim() != 3 or g.shape[2] != 3:
            raise ValueError("DetectorOffset.grad_from: dL_dmean2D must have shape [P, 3] or [B, P, 3]")
        if g.dtype != torch.float32 or g.device != dev or not g.is_contiguous():
            g = g.to(device=dev, dtype=torch.float32).contiguous()
        n, P = int(g.shape[0]), int(g.shape[1])
        lib = load()
        with torch.cuda.device(dev):
            nbytes = int(lib.r2x_detector_offset_grad_scratch_bytes(P, n))
            scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            grad = torch.empty(1, dtype=torch.float32, device=dev)
            check(lib.r2x_detector_offset_grad(torch.cuda.current_stream(dev).cuda_stream, P, n, int(W),
                                               g.data_ptr() if P else None, grad.data_ptr(), scratch.data_ptr(),
                                               nbytes), "r2x_detector_offset_grad")
        self.offset.grad = grad
        return grad

    def scene_units(self, scanner_cfg: dict) -> float:
        """The offset in scene units at the detector: s * sDetector[1] / nDetector[1] (host read)."""
        return float(self.offset.detach()[0]) * float(scanner_cfg["sDetector"][1]) / float(scanner_cfg["nDetector"][1])


# ---- the offset measured from the projections ------------------------------------------------------------------------

ANGLE_TOL = 1e-4          # parallel beam: |beta_j - beta_i - pi| up to this (radians) makes a pair
FINE_STEPS = 64           # the fine grid's points per pixel (and per coarse step)
MAX_CANDIDATES = 65535    # r2x_detector_offset_cost's K


def _wrap(a):
    """Angles reduced to [0, 2 pi)."""
    import numpy as np
    return np.mod(np.asarray(a, np.float64), 2.0 * np.pi)


def conjugate_pairs(angles, scanner_cfg: dict, reach: float, angle_tol: float = ANGLE_TOL):
    """The pair table of `estimate_offset` (host, numpy): (views int32 [n, 2] with i < j, dbeta float64 [n] =
    beta_j - beta_i in [0, 2 pi)).  Parallel beam: every pair with |dbeta - pi| <= angle_tol.  Cone beam: every pair
    whose shared mid-plane ray t = DSD tan((pi - dbeta) / 2) / du lies within `reach` pixels of the detector's centre
    column ((W - 1) / 2 plus the largest shift searched), so that it can land on both images."""
    import numpy as np
    beta = np.asarray(angles, np.float64).reshape(-1)
    n = beta.shape[0]
    i, j = np.triu_indices(n, k=1)
    d = _wrap(beta[j] - beta[i])
    if scanner_cfg["mode"] == "parallel":
        keep = np.abs(d - np.pi) <= float(angle_tol)
    else:
        du = float(scanner_cfg["sDetector"][1]) / float(scanner_cfg["nDetector"][1])
        half = 0.5 * (np.pi - d)
        keep = (d > 0.0) & (np.abs(half) < 0.5 * np.pi)
        t = np.full(d.shape, np.inf)
        t[keep] = float(scanner_cfg["DSD"]) * np.tan(half[keep]) / du
        keep &= np.abs(t) <= float(reach)
    views = np.stack([i[keep], j[keep]], axis=1).astype(np.int32)
    return np.ascontiguousarray(views), np.ascontiguousarray(d[keep])


class OffsetEstimateError(ValueError):
    """`estimate_offset` cannot measure the offset from these projections; the message says why."""


def _check_estimate_inputs(projs, angles, scanner_cfg, rows):
    if not isinstance(projs, torch.Tensor):
        raise TypeError(f"estimate_offset: projections must be a torch tensor, got {type(projs)}")
    if projs.dtype != torch.float32:
        raise TypeError(f"estimate_offset: projections must be float32, got {projs.dtype}")
    if projs.dim() != 3 or min(projs.shape) <= 0:
        raise ValueError(f"estimate_offset: projections must have shape [N, H, W], got {list(projs.shape)}")
    N, H, W = (int(x) for x in projs.shape)
    if len(angles) != N:
        raise ValueError(f"estimate_offset: {len(angles)} angles for {N} projections")
    if (H, W) != (int(scanner_cfg["nDetector"][0]), int(scanner_cfg["nDetector"][1])):
        raise ValueError(f"estimate_offset: projections of {H}x{W} pixels, the scanner's detector is "
                         f"{scanner_cfg['nDetector'][0]}x{scanner_cfg['nDetector'][1]}")
    if scanner_cfg["mode"] not in ("cone", "parallel"):
        raise ValueError(f"estimate_offset: unknown scanner mode {scanner_cfg['mode']!r}")
    if rows is not None:
        if scanner_cfg["mode"] == "cone":
            raise ValueError("estimate_offset: rows applies to parallel beam only (in cone beam only the mid-plane row "
                             "holds conjugate rays)")
        lo, hi = (int(r) for r in rows)
        if not 0 <= lo < hi <= H:
            raise ValueError(f"estimate_offset: rows ({lo}, {hi}) must satisfy 0 <= start < stop <= {H}")
    return N, H, W


def _offset_cost(projs, mode, pairs, geom, shifts):
    """(num, den, count) float64 / float64 / int64 host arrays of r2x_detector_offset_cost at `shifts` (one launch,
    one host read)."""
    import numpy as np
    views_d, dbeta_d, DSD, du, t_v, row_lo, n_rows = pairs + geom
    dev = projs.device
    N, H, W = (int(x) for x in projs.shape)
    K = len(shifts)
    lib = load()
    with torch.cuda.device(dev):
        sig = torch.tensor(np.asarray(shifts, np.float64), device=dev)
        out = torch.empty((3, K), dtype=torch.float64, device=dev)       # num, den and the count's int64 bits
        nbytes = int(lib.r2x_detector_offset_cost_scratch_bytes(mode, W, int(views_d.shape[0]), n_rows, K))
        scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        check(lib.r2x_detector_offset_cost(torch.cuda.current_stream(dev).cuda_stream, mode, N, H, W, projs.data_ptr(),
                                           int(views_d.shape[0]), views_d.data_ptr(), dbeta_d.data_ptr(), DSD, du,
                                           t_v, row_lo, n_rows, K, sig.data_ptr(), out[0].data_ptr(),
                                           out[1].data_ptr(), out[2].data_ptr(), scratch.data_ptr(), nbytes),
              "r2x_detector_offset_cost")
        host = out.cpu().numpy()
    return host[0], host[1], host[2].view(np.int64)


def _costs(num, den):
    import numpy as np
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(den > 0.0, num / np.where(den > 0.0, den, 1.0), np.inf)


def estimate_offset(projs: torch.Tensor, angles, scanner_cfg: dict, use_offDetector: bool = False, max_shift=None,
                    angle_tol: float = ANGLE_TOL, rows=None) -> dict:
    """The horizontal detector offset measured from the projections themselves, by the mismatch of conjugate rays
    (the model is r2x_detector_offset_cost's in include/r2x.h).

    `projs` float32 CUDA [N, H, W] at `angles` (radians) on `scanner_cfg`'s circle.  The cost of a candidate s is
    sum (a - b)^2 / sum (a^2 + b^2) over the conjugate samples that land on both images; it is searched on a coarse
    grid of whole pixels over +-max_shift (default W / 4) in one launch, then on a grid of 1/64 px over +-1 px around
    the coarse minimum in a second launch, and a parabola through the fine minimum and its neighbours gives the
    estimate.  Parallel beam uses the views pi apart (to `angle_tol` radians), every column and the rows `rows` (a
    (start, stop) range; default every row); cone beam uses each pair of views whose shared mid-plane ray falls on the
    detector, in the mid-plane row only.

    Returns {"offset_px": s (the DetectorOffset convention, relative to the geometry passed: on top of the scanner's
    offDetector when `use_offDetector`), "offset_scene": s du, "offDetector_u": the scanner's total offDetector[0] in
    `scanner_cfg`'s units, "n_pairs", "n_samples" (at the fine minimum), "cost_min", "coarse": (shifts, costs),
    "fine": (shifts, costs)}.  Raises OffsetEstimateError when the views hold no conjugate pairs (an arc shorter than
    180 degrees plus the fan angle), when the sampled rows carry no signal, or when the minimum lies on the edge of the
    search range."""
    import math

    import numpy as np

    from .scene import detector_shift
    N, H, W = _check_estimate_inputs(projs, angles, scanner_cfg, rows)
    cone = scanner_cfg["mode"] == "cone"
    M = W / 4.0 if max_shift is None else float(max_shift)
    if not (M > 0.0 and math.isfinite(M)):
        raise ValueError(f"estimate_offset: max_shift must be finite and positive, got {max_shift}")
    M = int(math.ceil(M))
    if 2 * M + 1 > MAX_CANDIDATES:
        raise ValueError(f"estimate_offset: max_shift {max_shift} needs more than {MAX_CANDIDATES} candidates")
    if not (float(angle_tol) >= 0.0 and math.isfinite(float(angle_tol))):
        raise ValueError(f"estimate_offset: angle_tol must be finite and >= 0, got {angle_tol}")
    t_u, t_v = detector_shift(scanner_cfg) if use_offDetector else (0.0, 0.0)
    du = float(scanner_cfg["sDetector"][1]) / float(scanner_cfg["nDetector"][1])
    views, dbeta = conjugate_pairs(angles, scanner_cfg, 0.5 * (W - 1) + M + 1 + abs(t_u), angle_tol)
    if views.shape[0] == 0:
        need = "two views 180 degrees apart" if not cone else "an arc of at least 180 degrees plus the fan angle"
        raise OffsetEstimateError(f"estimate_offset: the {N} views hold no conjugate pairs (this needs {need})")
    if projs.device.type != "cuda":
        raise RuntimeError("estimate_offset: projections must be a CUDA tensor (the cost runs on the GPU and has no CPU "
                           f"fallback; got {projs.device})")
    row_lo, n_rows = (0, H) if rows is None else (int(rows[0]), int(rows[1]) - int(rows[0]))
    if cone:
        row_lo, n_rows = 0, 1
    dev = projs.device
    pairs = (torch.from_numpy(views).to(dev), torch.from_numpy(dbeta).to(dev))
    geom = (float(scanner_cfg["DSD"]) if cone else 0.0, du, float(t_v), row_lo, n_rows)
    mode = 1 if cone else 0
    p = projs.contiguous()
    # the kernel's sigma is the shift of the rotation axis from the detector centre: s minus the file's t_u
    coarse = np.arange(-M, M + 1, dtype=np.float64)
    num, den, _ = _offset_cost(p, mode, pairs, geom, coarse - t_u)
    if not np.any(den > 0.0):
        raise OffsetEstimateError("estimate_offset: the conjugate samples carry no signal (an empty mid-plane?)")
    c_cost = _costs(num, den)
    k = int(np.argmin(c_cost))
    if k == 0 or k == len(coarse) - 1:
        raise OffsetEstimateError(f"estimate_offset: the cost is least on the edge of the search range (s = "
                                  f"{coarse[k]:+g} px of +-{M}); widen max_shift or check the geometry")
    fine = coarse[k] + np.arange(-FINE_STEPS, FINE_STEPS + 1, dtype=np.float64) / FINE_STEPS
    num, den, cnt = _offset_cost(p, mode, pairs, geom, fine - t_u)
    f_cost = _costs(num, den)
    j = int(np.argmin(f_cost))
    if j == 0 or j == len(fine) - 1:
        raise OffsetEstimateError("estimate_offset: the fine cost is least on the edge of its grid")
    y0, y1, y2 = f_cost[j - 1], f_cost[j], f_cost[j + 1]
    curv = y0 - 2.0 * y1 + y2
    delta = 0.5 * (y0 - y2) / curv / FINE_STEPS if curv > 0.0 else 0.0
    s = float(fine[j] + delta)
    return {"offset_px": s, "offset_scene": s * du, "offDetector_u": (t_u - s) * du,
            "n_pairs": int(views.shape[0]), "n_samples": int(cnt[j]), "cost_min": float(y1),
            "coarse": (coarse.tolist(), c_cost.tolist()), "fine": (fine.tolist(), f_cost.tolist())}


def with_offDetector_u(scanner_cfg: dict, offDetector_u: float) -> dict:
    """A deep copy of `scanner_cfg` whose offDetector[0] (u) is `offDetector_u` (offDetector[1] kept, 0 when absent)."""
    cfg = copy.deepcopy(scanner_cfg)
    off = list(cfg.get("offDetector", [0.0, 0.0]))
    cfg["offDetector"] = [float(offDetector_u), float(off[1])]
    return cfg

