"""Isotropic total variation of a volume on the GPU over the C ABI (r2x_tv_prox / r2x_tv_value / r2x_tv_cp_step,
csrc/r2x_tv.cu).

    x = tv_denoise(volume, weight, niter=20, nonneg=True)   # argmin_{x >= 0} 1/2 |x - volume|^2 + weight TV(x)
    t = tv_value(volume)                                    # TV(volume) as a Python float (float64 sum)
    x, xbar, p = tv_cp_step(x, xbar, p, g, tau, sigma, nu, nonneg=True)   # one Chambolle-Pock step of cp_tv

TV(x) = sum over voxels of sqrt(dx^2 + dy^2 + dz^2), forward differences, 0 across the last index.  This is not the
training loss `r2x_tv3d_loss` (the anisotropic mean of absolute differences of the reference's `loss_utils`).
`tv_denoise` is the proximal operator FISTA-TV (`recon.fista_tv`) applies each iteration, usable on its own, e.g. on
an FDK volume: `niter` iterations of Beck-Teboulle's fast gradient projection from a zero dual field.  `volume` is a
CUDA float32 [nx, ny, nz] tensor; both run on the current stream and are bitwise reproducible.  No CPU fallback.
`tv_cp_step` is the volume part of one iteration of `recon.cp_tv` (Chambolle-Pock for data-constrained TV), given
g = A^T q: p+ = P_{1/nu}(p + sigma nu grad xbar), x+ = P_C(x - tau g + tau nu div p+), xbar+ = 2 x+ - x, into new
tensors (the kernel reads p and xbar across tile edges, so it never writes in place).
"""
from __future__ import annotations

import torch

from ._lib import check, load


def _volume(what: str, volume) -> torch.Tensor:
    if not isinstance(volume, torch.Tensor) or volume.device.type != "cuda":
        raise RuntimeError(f"{what}: volume must be a CUDA tensor (this build has no CPU fallback; "
                           f"got {getattr(volume, 'device', type(volume))})")
    if volume.dim() != 3:
        raise ValueError(f"{what}: expected a [nx, ny, nz] volume, got shape {tuple(volume.shape)}")
    return volume.detach().to(torch.float32).contiguous()


def tv_denoise(volume: torch.Tensor, weight: float, niter: int = 20, nonneg: bool = True) -> torch.Tensor:
    """prox of weight * TV (+ the indicator of x >= 0 when nonneg) at `volume`, by `niter` FGP iterations."""
    weight = float(weight)
    if not weight >= 0.0:
        raise ValueError(f"tv_denoise: weight must be >= 0, got {weight}")
    if int(niter) != niter or niter < 1:
        raise ValueError(f"tv_denoise: niter must be an integer >= 1, got {niter}")
    v = _volume("tv_denoise", volume)
    nx, ny, nz = (int(s) for s in v.shape)
    lib = load()
    with torch.cuda.device(v.device):
        out = torch.empty_like(v)
        nbytes = int(lib.r2x_tv_prox_scratch_bytes(nx, ny, nz))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=v.device)
        rc = lib.r2x_tv_prox(torch.cuda.current_stream(v.device).cuda_stream, nx, ny, nz, v.data_ptr(), weight,
                             int(niter), int(bool(nonneg)), out.data_ptr(), scratch.data_ptr(), nbytes)
    check(rc, "r2x_tv_prox")
    return out


def tv_value(volume: torch.Tensor) -> float:
    """TV(volume), each term and the sum in float64 (fixed order)."""
    x = _volume("tv_value", volume)
    nx, ny, nz = (int(s) for s in x.shape)
    lib = load()
    with torch.cuda.device(x.device):
        out = torch.empty(1, dtype=torch.float64, device=x.device)
        nbytes = int(lib.r2x_tv_value_scratch_bytes(nx, ny, nz))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
        rc = lib.r2x_tv_value(torch.cuda.current_stream(x.device).cuda_stream, nx, ny, nz, x.data_ptr(),
                              out.data_ptr(), scratch.data_ptr(), nbytes)
    check(rc, "r2x_tv_value")
    return float(out)


def tv_cp_step(x: torch.Tensor, xbar: torch.Tensor, p: torch.Tensor, g: torch.Tensor, tau: float, sigma: float,
               nu: float, nonneg: bool = True):
    """(x+, xbar+, p+) of one Chambolle-Pock step (r2x_tv_cp_step): x, xbar, g [nx, ny, nz], p [3, nx, ny, nz]."""
    xs = _volume("tv_cp_step", x)
    shape = tuple(xs.shape)
    parts = {"xbar": xbar, "g": g, "p": p}
    for name, t in parts.items():
        want = (3,) + shape if name == "p" else shape
        if not isinstance(t, torch.Tensor) or t.device != xs.device:
            raise RuntimeError(f"tv_cp_step: {name} must be a tensor on {xs.device}, got {getattr(t, 'device', type(t))}")
        if tuple(t.shape) != want:
            raise ValueError(f"tv_cp_step: {name} must have shape {want}, got {tuple(t.shape)}")
    xb, gs, ps = (parts[k].detach().to(torch.float32).contiguous() for k in ("xbar", "g", "p"))
    nx, ny, nz = shape
    lib = load()
    with torch.cuda.device(xs.device):
        x_out, xbar_out, p_out = torch.empty_like(xs), torch.empty_like(xs), torch.empty_like(ps)
        rc = lib.r2x_tv_cp_step(torch.cuda.current_stream(xs.device).cuda_stream, nx, ny, nz, xs.data_ptr(),
                                xb.data_ptr(), ps.data_ptr(), gs.data_ptr(), float(tau), float(sigma), float(nu),
                                int(bool(nonneg)), x_out.data_ptr(), xbar_out.data_ptr(), p_out.data_ptr())
    check(rc, "r2x_tv_cp_step")
    return x_out, xbar_out, p_out
