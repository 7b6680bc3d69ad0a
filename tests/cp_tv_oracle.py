"""Float64 NumPy statement of one Chambolle-Pock step of r2x_tv_cp_step (csrc/r2x_tv.cu), with the grad / div of
tests/tv_oracle.py:

    p+ = P_{1/nu}(p + sigma nu grad xbar)        per voxel: u scaled by (1/nu) / |u| where |u| > 1/nu
    x+ = P_C(x - tau g + tau nu div p+)          C = {x >= 0} when nonneg, else everything
    xbar+ = 2 x+ - x

`step` wraps it as the callable `recon.cp_tv_solve` takes (float64 CPU torch tensors).
"""
from __future__ import annotations

import numpy as np

import tv_oracle as tvo


def cp_step(x, xbar, p, g, tau: float, sigma: float, nu: float, nonneg: bool):
    """(x+, xbar+, p+) in float64."""
    x, xbar, p, g = (np.asarray(a, np.float64) for a in (x, xbar, p, g))
    u = p + (sigma * nu) * tvo.grad(xbar)
    norm = np.sqrt((u ** 2).sum(0))
    p_next = u / np.maximum(1.0, norm * nu)
    x_next = tvo.proj_c(x - tau * g + (tau * nu) * tvo.div(p_next), nonneg)
    return x_next, 2.0 * x_next - x, p_next


def step(x, xbar, p, g, tau, sigma, nu, nonneg):
    import torch

    return tuple(torch.from_numpy(a) for a in cp_step(x.numpy(), xbar.numpy(), p.numpy(), g.numpy(), float(tau),
                                                      float(sigma), float(nu), bool(nonneg)))
