"""Float64 NumPy statement of the isotropic TV operators of csrc/r2x_tv.cu (r2x_tv_prox / r2x_tv_value).

grad x = forward differences along each axis, 0 across the last index; div p = -grad^T p; TV(x) = sum |grad x|.
`fgp` is Beck-Teboulle's fast gradient projection for prox_{w TV + indicator(C)}(v) with the recurrence the kernel
runs (r_1 = 0, p_k = P_1(r_k - grad P_C(v - w div r_k) / (12 w)), t_{k+1} = (1 + sqrt(1 + 4 t_k^2)) / 2,
r_{k+1} = p_k + ((t_k - 1) / t_{k+1}) (p_k - p_{k-1}), x = P_C(v - w div p)), and `dual_gap` the primal-dual gap
of the constrained ROF problem that certifies a (x, p) pair.  `prox` / `tv` wrap them as the callables
`recon.fista_tv_solve` takes (float64 CPU torch tensors).
"""
from __future__ import annotations

import math

import numpy as np


def grad(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x, np.float64)
    g = np.zeros((3,) + x.shape)
    g[0, :-1] = x[1:] - x[:-1]
    g[1, :, :-1] = x[:, 1:] - x[:, :-1]
    g[2, :, :, :-1] = x[:, :, 1:] - x[:, :, :-1]
    return g


def div(p: np.ndarray) -> np.ndarray:
    """-grad^T p: sum over axes of p_a[i] (i_a < n_a - 1) - p_a[i - e_a] (i_a > 0)."""
    p = np.asarray(p, np.float64)
    d = np.zeros(p.shape[1:])
    d[:-1] += p[0, :-1]
    d[1:] -= p[0, :-1]
    d[:, :-1] += p[1, :, :-1]
    d[:, 1:] -= p[1, :, :-1]
    d[:, :, :-1] += p[2, :, :, :-1]
    d[:, :, 1:] -= p[2, :, :, :-1]
    return d


def tv_value(x: np.ndarray) -> float:
    return float(np.sqrt((grad(x) ** 2).sum(0)).sum())


def proj_c(u: np.ndarray, nonneg: bool) -> np.ndarray:
    return np.where(u < 0.0, 0.0, u) if nonneg else u


def fgp(v: np.ndarray, w: float, niter: int, nonneg: bool):
    """(x, p): `niter` FGP iterations for prox_{w TV + indicator(C)}(v) from p = 0; w = 0 gives (P_C(v), 0)."""
    v = np.asarray(v, np.float64)
    p_prev = np.zeros((3,) + v.shape)
    if w == 0.0:
        return proj_c(v, nonneg), p_prev
    r = p_prev.copy()
    t = 1.0
    for _ in range(niter):
        q = r - grad(proj_c(v - w * div(r), nonneg)) / (12.0 * w)
        p = q / np.maximum(1.0, np.sqrt((q ** 2).sum(0)))
        t_next = 0.5 * (1.0 + math.sqrt(1.0 + 4.0 * t * t))
        r = p + ((t - 1.0) / t_next) * (p - p_prev)
        p_prev, t = p, t_next
    return proj_c(v - w * div(p_prev), nonneg), p_prev


def dual_gap(v: np.ndarray, w: float, x: np.ndarray, p: np.ndarray, nonneg: bool) -> tuple[float, float]:
    """(primal, primal - dual) for x in C and |p| <= 1: primal = 1/2 |x - v|^2 + w TV(x); dual(p) = min over C of
    1/2 |x - v|^2 + w <x, div p> = 1/2 |P_C(u) - u|^2 + 1/2 |v|^2 - 1/2 |u|^2 with u = v - w div p."""
    v = np.asarray(v, np.float64)
    primal = 0.5 * float(((x - v) ** 2).sum()) + w * tv_value(x)
    u = v - w * div(p)
    dual = 0.5 * float(((proj_c(u, nonneg) - u) ** 2).sum()) + 0.5 * float((v ** 2).sum()) - 0.5 * float((u ** 2).sum())
    return primal, primal - dual


def prox(v, weight, niter, nonneg):
    import torch

    return torch.from_numpy(fgp(v.numpy(), float(weight), int(niter), bool(nonneg))[0])


def tv(x) -> float:
    return tv_value(x.numpy())
