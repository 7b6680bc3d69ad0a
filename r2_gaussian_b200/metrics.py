"""Evaluation metrics with the reference's definitions (`r2_gaussian/utils/image_utils.py:19-183`): `mse`, `rmse`,
`psnr` on [b,c,h,w] batches, `metric_vol` (3-D PSNR; slice-wise SSIM averaged over the three axes) and
`metric_proj` (per-projection, each slice normalised by its own maximum).  SSIM here is the plain torch formulation
(any device), windows as in `loss_utils.py:45-104`.

`volume_metrics` / `projection_metrics` compute what `metric_vol` / `metric_proj` define for CUDA float32 tensors on
the device: every slice's SSIM in the fused image-loss kernel (`r2x_image_loss_views`, same window bits and
constants), maxima, MSE and PSNR as torch reductions, and one device-to-host read per call, after which the per-slice
values are summed on the host in the order the torch functions sum them.  No CPU fallback."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F


def _window(channel: int, like: torch.Tensor) -> torch.Tensor:
    g = torch.tensor([math.exp(-((x - 5) ** 2) / float(2 * 1.5 ** 2)) for x in range(11)])
    g = (g / g.sum()).unsqueeze(1)
    w = g.mm(g.t()).float().unsqueeze(0).unsqueeze(0)
    return w.expand(channel, 1, 11, 11).contiguous().to(device=like.device, dtype=like.dtype)


def ssim(img1: torch.Tensor, img2: torch.Tensor) -> torch.Tensor:
    """Mean SSIM of [b,c,h,w] (or [c,h,w]) images, 11x11 Gaussian window, zero padding."""
    c = img1.size(-3)
    w = _window(c, img1)
    mu1, mu2 = F.conv2d(img1, w, padding=5, groups=c), F.conv2d(img2, w, padding=5, groups=c)
    s11 = F.conv2d(img1 * img1, w, padding=5, groups=c) - mu1 * mu1
    s22 = F.conv2d(img2 * img2, w, padding=5, groups=c) - mu2 * mu2
    s12 = F.conv2d(img1 * img2, w, padding=5, groups=c) - mu1 * mu2
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    return (((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s11 + s22 + C2))).mean()


def mse(img1, img2, mask=None):
    if mask is None:
        return ((img1 - img2) ** 2).reshape(img1.shape[0], -1).mean(1, keepdim=True)
    n_channel = img1.shape[1]
    a, b = img1.flatten(1), img2.flatten(1)
    m = mask.flatten(1).repeat(1, n_channel) != 0
    return torch.stack([((a[i, m[i]] - b[i, m[i]]) ** 2).mean(0, keepdim=True) for i in range(a.shape[0])], dim=0)


def rmse(img1, img2, mask=None):
    return mse(img1, img2, mask) ** 0.5


@torch.no_grad()
def psnr(img1, img2, mask=None, pixel_max=1.0):
    out = 10 * torch.log10(pixel_max ** 2 / mse(img1, img2, mask).float())
    if mask is not None and torch.isinf(out).any():
        out = out[~torch.isinf(out)]
    return out


def _slices(vol, axis):
    for i in range(vol.shape[axis]):
        yield vol.select(axis, i)


def _as_tensor(a):
    return torch.from_numpy(np.array(a, copy=True)) if isinstance(a, np.ndarray) else a


@torch.no_grad()
def metric_vol(img1, img2, metric="psnr", pixel_max=1.0):
    """img1 = ground truth.  -> (value, per-axis list or None)."""
    assert metric in ("psnr", "ssim")
    img1, img2 = _as_tensor(img1), _as_tensor(img2)
    if metric == "psnr":
        if pixel_max is None:
            pixel_max = img1.max()
        return (10 * torch.log10(pixel_max ** 2 / torch.mean((img1 - img2) ** 2).float())).item(), None
    per_axis = []
    for axis in (0, 1, 2):
        vals, count = [], 0
        for s1, s2 in zip(_slices(img1, axis), _slices(img2, axis)):
            if s1.max() > 0:
                vals.append(float(ssim(s1[None, None], s2[None, None])))
                count += 1
            else:
                vals.append(0.0)
        per_axis.append(sum(vals) / count)
    return float(np.mean(per_axis)), per_axis


@torch.no_grad()
def metric_proj(img1, img2, metric="psnr", axis=2, pixel_max=1.0):
    """Stack of projections along `axis`; every non-empty slice is normalised by its own maximum first."""
    assert axis in (0, 1, 2, None) and metric in ("psnr", "ssim")
    img1, img2 = _as_tensor(img1), _as_tensor(img2)
    vals, count = [], 0
    for s1, s2 in zip(_slices(img1, axis), _slices(img2, axis)):
        if s1.max() > 0:
            a, b = (s1 / s1.max())[None, None], (s2 / s2.max())[None, None]
            vals.append(float(psnr(a, b, pixel_max=pixel_max)) if metric == "psnr" else float(ssim(a, b)))
            count += 1
        else:
            vals.append(0.0)
    return sum(vals) / count, vals


# ---- device-side evaluation ------------------------------------------------------------------------------------------

VIEWS_MAX_N = 65535               # r2x_image_loss_views: images per call
IMAGE_MAX_H = 65535 * 16          # r2x_image_loss_views: rows per image (grid.y of 16-row tiles)
SSIM_SCRATCH_BYTES = 1 << 30      # kernel scratch per call; a stack needing more runs in several calls


def _require_device_float32(name: str, *tensors):
    """Refuse anything but float32 CUDA tensors of one shape on one device, before any CUDA call."""
    for t in tensors:
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{name}: expected torch tensors, got {type(t).__name__}")
        if not t.is_cuda:
            raise RuntimeError(f"{name}: expected CUDA tensors, got a {t.device.type} tensor (the device metrics have "
                               "no CPU fallback; metric_vol / metric_proj take CPU data)")
        if t.dtype != torch.float32:
            raise TypeError(f"{name}: expected float32 tensors, got {t.dtype}")
    a, b = tensors
    if a.shape != b.shape:
        raise ValueError(f"{name}: shapes differ: {tuple(a.shape)} vs {tuple(b.shape)}")
    if a.device != b.device:
        raise ValueError(f"{name}: tensors on different devices: {a.device} vs {b.device}")
    if a.dim() != 3 or min(a.shape[1:]) == 0:
        raise ValueError(f"{name}: expected a 3-D tensor with non-empty slices, got shape {tuple(a.shape)}")


def ssim_rows(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """Mean SSIM of each image pair of two contiguous float32 CUDA stacks [N, H, W] -> [N] float32 on the device:
    column 1 of `r2x_image_loss_views` (no gradient), which is `ssim(x[i][None, None], y[i][None, None])` computed in
    the fused kernel.  Stacks of more than 65535 images, or whose kernel scratch would pass SSIM_SCRATCH_BYTES, run in
    several calls; images taller than the kernel's row limit are transposed first (the window is symmetric and
    separable, so the SSIM is the same up to rounding)."""
    from ._lib import check, load
    N, H, W = (int(s) for s in x.shape)
    if H > IMAGE_MAX_H:
        if W > IMAGE_MAX_H:
            raise ValueError(f"ssim_rows: images of {H} x {W} exceed the kernel's {IMAGE_MAX_H} rows either way")
        x, y, H, W = x.transpose(1, 2), y.transpose(1, 2), W, H
    x, y = x.contiguous(), y.contiguous()
    lib = load()
    dev = x.device
    scratch_bytes = lib.r2x_image_loss_views_scratch_bytes
    per_image = int(scratch_bytes(2, H, W)) - int(scratch_bytes(1, H, W))
    chunk = max(1, min(N, VIEWS_MAX_N, SSIM_SCRATCH_BYTES // per_image))
    with torch.cuda.device(dev):
        nbytes = int(scratch_bytes(chunk, H, W))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        out = torch.empty((N, 3), dtype=torch.float32, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        for s in range(0, N, chunk):
            n = min(chunk, N - s)
            check(lib.r2x_image_loss_views(st, n, H, W, x[s].data_ptr(), y[s].data_ptr(), 0.0, 1.0, out[s].data_ptr(),
                                           None, scratch.data_ptr(), nbytes), "r2x_image_loss_views")
    return out[:, 1]


def _counted_mean(vals, counted) -> float:
    """`sum(vals) / count` of metric_vol / metric_proj: uncounted slices add 0.0; no counted slice raises
    ZeroDivisionError."""
    vals = [float(v) if c else 0.0 for v, c in zip(vals, counted)]
    return sum(vals) / int(sum(bool(c) for c in counted))


def volume_slice_scores(vol_gt: torch.Tensor, vol_pred: torch.Tensor) -> list:
    """The device tensors `volume_metrics` reads, float64: [psnr_3d] and, for axes 0, 1, 2, the SSIM of every slice
    along the axis and whether it counts (1.0: its gt maximum is > 0)."""
    psnr = 10 * torch.log10(1.0 ** 2 / torch.mean((vol_gt - vol_pred) ** 2).float())
    parts = [psnr.reshape(1).double()]
    for axis in (0, 1, 2):
        g = vol_gt.movedim(axis, 0).contiguous()     # slice i along `axis` is g[i], in metric_vol's orientation
        p = vol_pred.movedim(axis, 0).contiguous()
        parts += [ssim_rows(g, p).double(), (g.amax(dim=(1, 2)) > 0).double()]
        del g, p
    return parts


@torch.no_grad()
def volume_metrics(vol_gt: torch.Tensor, vol_pred: torch.Tensor) -> dict:
    """`metric_vol`'s psnr and ssim of two CUDA float32 volumes [nx, ny, nz] (vol_gt first) with one device-to-host
    read -> {"psnr_3d", "ssim_3d", "ssim_3d_x", "ssim_3d_y", "ssim_3d_z"}.  psnr_3d is metric_vol's torch expression
    (pixel_max 1); the SSIM of every slice along each axis comes from `ssim_rows`, a slice counts when its gt maximum
    is > 0, and an axis without a counted slice raises ZeroDivisionError, as in metric_vol."""
    _require_device_float32("volume_metrics", vol_gt, vol_pred)
    if vol_gt.shape[0] == 0:
        raise ZeroDivisionError("volume_metrics: the volume has no slice along axis 0")
    host = torch.cat(volume_slice_scores(vol_gt, vol_pred)).cpu().numpy()
    out = {"psnr_3d": float(host[0])}
    per_axis, at = [], 1
    for n in vol_gt.shape:
        per_axis.append(_counted_mean(host[at:at + n], host[at + n:at + 2 * n]))
        at += 2 * n
    out["ssim_3d"] = float(np.mean(per_axis))
    out["ssim_3d_x"], out["ssim_3d_y"], out["ssim_3d_z"] = per_axis
    return out


def projection_view_scores(gt: torch.Tensor, pred: torch.Tensor) -> list:
    """The device tensors `projection_metrics` reads, float64 [N] each: every view's PSNR, its SSIM, and whether it
    counts (1.0: its gt maximum is > 0)."""
    N = int(gt.shape[0])
    gmax = gt.amax(dim=(1, 2), keepdim=True)
    a, b = gt / gmax, pred / pred.amax(dim=(1, 2), keepdim=True)
    mse = ((a - b) ** 2).reshape(N, -1).mean(1)
    psnr = 10 * torch.log10(1.0 ** 2 / mse)
    return [psnr.double(), ssim_rows(a, b).double(), (gmax.reshape(N) > 0).double()]


@torch.no_grad()
def projection_metrics(gt: torch.Tensor, pred: torch.Tensor) -> dict:
    """`metric_proj`'s psnr and ssim of two CUDA float32 stacks [N, H, W] (one view per image, gt first) with one
    device-to-host read -> {"psnr_2d", "ssim_2d", "psnr_2d_projs" (list of N), "ssim_2d_projs" (list of N)}.  Each gt
    view is divided by its own maximum and each prediction by its own; a view counts when its gt maximum is > 0
    (others score 0.0), PSNR is 10 log10(1 / mse) per view, and a prediction whose maximum is <= 0 gives the inf / NaN
    metric_proj gives.  No counted view raises ZeroDivisionError."""
    _require_device_float32("projection_metrics", gt, pred)
    N = int(gt.shape[0])
    if N == 0:
        raise ZeroDivisionError("projection_metrics: the stack has no view")
    host = torch.cat(projection_view_scores(gt, pred)).cpu().numpy()
    psnr_v, ssim_v, counted = host[:N], host[N:2 * N], host[2 * N:]
    psnr_l = [float(v) if c else 0.0 for v, c in zip(psnr_v, counted)]
    ssim_l = [float(v) if c else 0.0 for v, c in zip(ssim_v, counted)]
    return {"psnr_2d": _counted_mean(psnr_v, counted), "ssim_2d": _counted_mean(ssim_v, counted),
            "psnr_2d_projs": psnr_l, "ssim_2d_projs": ssim_l}
