"""Metal artifact reduction in the projections: linear-interpolation MAR (LI-MAR, Kalender et al. 1987) and normalised
MAR (NMAR, Meyer et al., Med. Phys. 37, 2010), with the metal-trace inpainting on the GPU, r2x_mar_inpaint.

Metal lets few or no photons through and hardens the beam, so every ray through it carries a wrong line integral, and
FDK and every iterative method spread those errors into streaks across the volume.  `reduce_metal`:
    1. segments the metal in an FDK of the projections (`FDK > threshold`, or a given mask);
    2. projects the mask: the metal trace is every detector pixel whose chord through metal exceeds
       TRACE_TAU * min(dVoxel), dilated by TRACE_DILATE columns;
    3. LI: replaces the trace by linear interpolation along each detector row from the nearest pixels outside it;
       NMAR: builds a tissue-class prior from the LI volume, divides the row by the prior's projection, interpolates and
       multiplies back, so the inpainted values keep the structure the prior predicts;
    4. returns the corrected projections; `reinsert` puts the metal of the uncorrected FDK back into a reconstruction.
MAR removes the metal from the data by design: a reconstruction of the corrected projections has no metal until it is
reinserted.  It helps when metal artifacts dominate and can cost a little where they are weak; the segmentation, a
fixed threshold, is the fragile step (DESIGN §8).  include/r2x.h states the inpainting model; tests/mar_oracle.py is
its numpy restatement.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

# the metal trace: chord length through metal above TRACE_TAU voxels, dilated by TRACE_DILATE detector columns; the
# best pair of the sweep of DESIGN §8 (every tau from 0.1 to 1 voxel with d = 0 or 1 was within 0.15 dB of it)
TRACE_TAU = 0.25
TRACE_DILATE = 0
# the NMAR prior's classes (Meyer et al.'s air / tissue / bone split), relative to the soft-tissue level s: the lower
# median of the non-metal voxels above PRIOR_FLOOR times their maximum.  Stated, not measured.
PRIOR_AIR = 0.5
PRIOR_BONE = 1.5
PRIOR_FLOOR = 0.1
EPS = 1e-3                  # the prior projection's floor in NMAR's division, scene units
MAX_W = 16384               # R2X_MAR_MAX_W
_MAX_ROWS = (1 << 31) - 1   # n H per kernel call (the grid); larger stacks run in windows of views
METHODS = ("nmar", "li")
FDK_KWARGS = ("use_offDetector", "short_scan", "half_fan", "fdk_filter", "fdk_pad")


def _check_stack(name, x, shape=None, dtype=None, device=None):
    import torch

    dtype = torch.float32 if dtype is None else dtype
    if not isinstance(x, torch.Tensor) or x.device.type != "cuda" or x.dtype != dtype or x.dim() != 3 \
            or not x.is_contiguous():
        raise ValueError(f"inpaint: {name} must be a contiguous CUDA {str(dtype).replace('torch.', '')} [N, H, W] "
                         "tensor")
    if shape is not None and (tuple(x.shape) != shape or x.device != device):
        raise ValueError(f"inpaint: {name} must have shape {list(shape)} on {device}, got {list(x.shape)} on "
                         f"{x.device}")


def inpaint(projs, mask_proj, tau: float, dilate: int, prior=None, eps: float = EPS, out=None, trace=None):
    """Metal-trace inpainting of a contiguous CUDA float32 [N, H, W] stack (views, detector rows, detector columns) on
    the current stream: `mask_proj` the projection of the metal mask, `tau` its trace threshold, `dilate` the trace's
    dilation in columns, `prior` the NMAR prior's projection or None for LI.  `out` is a float32 [N, H, W] tensor
    (`projs` itself for in place) or None for a new one; `trace` an optional uint8 [N, H, W] tensor for the trace.
    Returns `out`."""
    import torch

    from ._lib import check, load

    _check_stack("projs", projs)
    n, H, W = (int(s) for s in projs.shape)
    _check_stack("mask_proj", mask_proj, (n, H, W), device=projs.device)
    if prior is not None:
        _check_stack("prior", prior, (n, H, W), device=projs.device)
    if W > MAX_W:
        raise ValueError(f"inpaint: detector width {W} exceeds the kernel's {MAX_W}")
    if not math.isfinite(float(tau)):
        raise ValueError(f"inpaint: tau must be finite, got {tau}")
    if isinstance(dilate, bool) or int(dilate) != dilate or dilate < 0:
        raise ValueError(f"inpaint: dilate must be an integer >= 0, got {dilate}")
    if not (math.isfinite(float(eps)) and float(eps) > 0.0):
        raise ValueError(f"inpaint: eps must be finite and > 0, got {eps}")
    if out is None:
        out = torch.empty_like(projs)
    _check_stack("out", out, (n, H, W), device=projs.device)
    if trace is not None:
        _check_stack("trace", trace, (n, H, W), torch.uint8, projs.device)
    step = max(1, _MAX_ROWS // H)
    lib = load()
    with torch.cuda.device(projs.device):
        stream = torch.cuda.current_stream(projs.device).cuda_stream
        for v0 in range(0, n, step):
            k = min(step, n - v0)
            rc = lib.r2x_mar_inpaint(stream, k, H, W, projs[v0].data_ptr(), mask_proj[v0].data_ptr(), float(tau),
                                     min(int(dilate), W), None if prior is None else prior[v0].data_ptr(), float(eps),
                                     out[v0].data_ptr(), None if trace is None else trace[v0].data_ptr())
            check(rc, "r2x_mar_inpaint")
    return out


def segment(fdk_vol, threshold: float):
    """The metal mask FDK > threshold (scene-scaled units), or ValueError when it is empty."""
    mask = fdk_vol > float(threshold)
    if not bool(mask.any()):
        raise ValueError(f"reduce_metal: no voxel of the FDK exceeds the metal threshold {threshold:g} (its maximum is "
                         f"{float(fdk_vol.max()):g}); lower the threshold or pass a mask")
    return mask


def nmar_prior(x, mask):
    """The NMAR prior of an LI-MAR reconstruction `x` and the metal mask: voxels below PRIOR_AIR s become 0, voxels in
    [PRIOR_AIR s, PRIOR_BONE s) and every metal voxel the mean of that tissue class, voxels at or above PRIOR_BONE s
    keep their value; s is the lower median of the non-metal voxels above PRIOR_FLOOR times their maximum.  The class
    statistics are float64."""
    import torch

    x64 = x.double()
    keep = ~mask
    top = float(x64[keep].max())
    sel = x64[keep & (x64 > PRIOR_FLOOR * top)]
    if sel.numel() == 0:
        raise ValueError("reduce_metal: the LI-MAR volume has no non-metal voxel to build the NMAR prior from")
    s = float(sel.sort().values[(sel.numel() - 1) // 2])
    tissue = keep & (x64 >= PRIOR_AIR * s) & (x64 < PRIOR_BONE * s)
    mean = float(x64[tissue].mean())
    prior = torch.where(x64 < PRIOR_AIR * s, torch.zeros_like(x64), x64)
    prior = torch.where(tissue | mask, torch.full_like(x64, mean), prior)
    return prior.to(torch.float32).contiguous()


def reinsert(volume, fdk_with_metal, mask):
    """`volume` with its metal voxels (`mask`) taken from the uncorrected FDK `fdk_with_metal`."""
    import torch

    return torch.where(mask, fdk_with_metal, volume)


@dataclass
class MarResult:
    projs: object                   # the corrected [N, H, W] stack
    mask: object                    # bool [nx, ny, nz]
    fdk: object                     # the FDK of the uncorrected projections
    trace_fraction: float           # of the train stack's pixels
    all_trace_rows: int             # detector rows that are trace from edge to edge (train stack)
    trace: object = None            # uint8 [N, H, W]
    extra: list = field(default_factory=list)    # per `extra` set: (corrected stack, trace, trace fraction, rows)


def _trace_stats(trace):
    return float(trace.float().mean()), int(trace.bool().all(dim=2).sum())


def reduce_metal(projs, angles, scanner_cfg: dict, method: str = "nmar", threshold=None, mask=None, extra=(),
                 trace_tau: float = TRACE_TAU, trace_dilate: int = TRACE_DILATE, **fdk_kwargs) -> MarResult:
    """LI-MAR (method "li") or NMAR ("nmar") of a CUDA float32 [N, H, W] stack in scene units at `angles` (one fixed
    circle).  The metal is `FDK(projs) > threshold` or the bool [nx, ny, nz] `mask`; `extra` is a sequence of further
    (projections, angles) sets corrected with the same mask and prior (the test views).  `fdk_kwargs` (use_offDetector,
    short_scan, half_fan, fdk_filter, fdk_pad) go to both FDKs; use_offDetector also to the projector."""
    import torch

    from .fdk import fdk
    from .projector import CTOperator

    if method not in METHODS:
        raise ValueError(f"reduce_metal: method must be one of {', '.join(METHODS)}, got {method!r}")
    for k in ("view_geometry", "helical"):
        if fdk_kwargs.get(k):
            raise ValueError(f"reduce_metal: {k} scans are not supported (the trace and the prior would need the "
                             "per-view FDK)")
        fdk_kwargs.pop(k, None)
    unknown = sorted(set(fdk_kwargs) - set(FDK_KWARGS))
    if unknown:
        raise TypeError(f"reduce_metal: unexpected keyword arguments {unknown}; the FDK flags are {list(FDK_KWARGS)}")
    if (threshold is None) == (mask is None):
        raise ValueError("reduce_metal: give exactly one of a metal threshold and a metal mask")
    if threshold is not None and not math.isfinite(float(threshold)):
        raise ValueError(f"reduce_metal: the metal threshold must be finite, got {threshold}")
    nvox = tuple(int(v) for v in scanner_cfg["nVoxel"])
    if mask is not None and tuple(mask.shape) != nvox:
        raise ValueError(f"reduce_metal: the metal mask has shape {list(mask.shape)}, the volume {list(nvox)}")
    if not isinstance(projs, torch.Tensor) or projs.device.type != "cuda":
        raise RuntimeError("reduce_metal: projections must be a CUDA tensor (no CPU fallback)")
    dev = projs.device
    b = projs.detach().to(torch.float32).contiguous()
    fk = {"use_offDetector": fdk_kwargs.get("use_offDetector", False), "short_scan": fdk_kwargs.get("short_scan", False),
          "half_fan": fdk_kwargs.get("half_fan", False), "filter": fdk_kwargs.get("fdk_filter"),
          "pad": fdk_kwargs.get("fdk_pad") or 0.0}
    vol0 = fdk(b, angles, scanner_cfg, **fk)
    if mask is None:
        mask = segment(vol0, threshold)
    else:
        mask = torch.as_tensor(np.asarray(mask.cpu() if isinstance(mask, torch.Tensor) else mask), device=dev).bool()
        if not bool(mask.any()):
            raise ValueError("reduce_metal: the metal mask is empty")
    tau = float(trace_tau) * min(float(v) for v in scanner_cfg["dVoxel"])
    maskf = mask.to(torch.float32).contiguous()

    def correct(p, op, m, prior):
        P = None if prior is None else op.A(prior).contiguous()
        tr = torch.empty(p.shape, dtype=torch.uint8, device=dev)
        return inpaint(p, m, tau, trace_dilate, prior=P, trace=tr), tr

    op = CTOperator(angles, scanner_cfg, dev, fk["use_offDetector"])
    m = op.A(maskf).contiguous()
    out, trace = correct(b, op, m, None)
    prior = None
    if method == "nmar":
        prior = nmar_prior(fdk(out, angles, scanner_cfg, **fk), mask)
        out, trace = correct(b, op, m, prior)
    frac, rows = _trace_stats(trace)
    res = MarResult(out, mask, vol0, frac, rows, trace)
    for p_e, ang_e in extra:
        p_e = p_e.detach().to(torch.float32).contiguous()
        op_e = CTOperator(ang_e, scanner_cfg, dev, fk["use_offDetector"])
        o, t = correct(p_e, op_e, op_e.A(maskf).contiguous(), prior)
        res.extra.append((o, t, *_trace_stats(t)))
    return res


def psnr_outside_metal(vol_gt, pred, mask, k: int = 2) -> float:
    """PSNR of `pred` against `vol_gt` over the voxels outside `mask` dilated by k voxels (the (2k + 1)^3 cube), with
    the peak the maximum of vol_gt over those voxels; float64."""
    import torch

    m = torch.as_tensor(mask).to(torch.float32)[None, None]
    dil = torch.nn.functional.max_pool3d(m, 2 * k + 1, stride=1, padding=k)[0, 0] > 0
    out = ~dil
    g = torch.as_tensor(vol_gt).to(dil.device, torch.float64)[out]
    x = torch.as_tensor(pred).to(dil.device, torch.float64)[out]
    mse = float(((g - x) ** 2).mean())
    return 10.0 * math.log10(float(g.max()) ** 2 / mse)
