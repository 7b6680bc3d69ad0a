"""Traditional CT reconstructions on the GPU -- FDK, SART / OS-SART and CGLS, what the reference obtains from TIGRE's
`algs` (`r2_gaussian/utils/ct_utils.py::recon_volume` / `run_ct_recon_algs`, `scripts/run_traditional_methods.py`),
the TV-regularised FISTA-TV and the data-constrained TV reconstruction cp_tv.

    x, l2 = cgls(projs, angles, scanner_cfg, niter=60)
    x = sart(projs, angles, scanner_cfg, niter=20, lmbda=1.0, lmbda_red=0.999, blocksize=1, nonneg=True)
    x, history = fista_tv(projs, angles, scanner_cfg, niter=FISTA_NITER, lmbda=FISTA_LAMBDA, tviter=20, nonneg=True)
    x, history = cp_tv(projs, angles, scanner_cfg, niter=CP_NITER, epsilon=None, epsilon_ratio=0.15, nonneg=True)
    x = recon_volume(projs, angles, scanner_cfg, method)           # fdk | cgls | sart | ossart | fista_tv | cp_tv

`projs` is a CUDA [N, H, W] tensor in the dataset layout (scene units, as the readers return it) and `scanner_cfg` the
scaled dict of `dataset.read_scene`; volumes are [nx, ny, nz] in the voxelizer's layout.  A is `projector.project`
(r2x_volume_project) and A^T its exact transpose `projector.backproject` (r2x_volume_backproject), so CGLS runs on a
matched pair.  The solvers (`cgls_solve`, `sart_solve`) are written over two callables, A(x, views) and
At(y, views, weights), with `views` a contiguous slice of the view list.  Norms and dot products are float64
reductions without atomics, so every solve is bitwise reproducible.

CGLS (TIGRE's recurrence), from x = 0:
    r = b - A x,  p = A^T r,  gamma = |p|^2;
    per iteration:  q = A p,  alpha = gamma / |q|^2,  x += alpha p,  r -= alpha q,  s = A^T r,  beta = |s|^2 / gamma,
                    gamma = |s|^2,  p = s + beta p.
    l2[i] = |r| after iteration i (TIGRE's computel2 evaluates |b - A x| with one more projection; it is the same
    quantity in exact arithmetic).

SART (blocksize 1) / OS-SART (blocksize > 1), from x = 0:
    W = 1 / (A 1) where A 1 > 0, else 0, computed once;
    each sweep takes the views in index order, in consecutive blocks B of `blocksize`:
        r = W * (b_B - A_B x);  (num, den) = (A_B^T r, A_B^T 1) from one fused backprojection;
        x += lmbda * num / den where den > 0;  x = max(x, 0) if nonneg;
    after each sweep lmbda *= lmbda_red.

FISTA-TV solves the TV-regularised least-squares problem
    minimise  F(x) = 1/2 |A x - b|^2 + lmbda TV(x)   subject to x >= 0   (nonneg=False drops the constraint)
    TV(x) = sum over voxels of sqrt(dx^2 + dy^2 + dz^2)   (isotropic; forward differences, 0 across the last index)
in the scene-scaled units of `dataset.read_scene`.  This TV is not the training loss `r2x_tv3d_loss`, which is the
anisotropic sum of absolute differences of the reference's `loss_utils`.  FISTA (Beck-Teboulle), from x_0 = y_1 = 0,
t_1 = 1; per iteration k:
    v = y_k - (1/L) A^T (A y_k - b)                             (one A and one A^T over all views)
    x_k = prox_{(lmbda/L) TV + indicator(x >= 0)}(v)            (`tviter` FGP iterations, `tv.tv_denoise`)
    t_{k+1} = (1 + sqrt(1 + 4 t_k^2)) / 2,   y_{k+1} = x_k + ((t_k - 1) / t_{k+1}) (x_k - x_{k-1}).
The prox is Beck-Teboulle's fast gradient projection for constrained TV denoising (csrc/r2x_tv.cu): the dual field
p[3, nx, ny, nz] cold-started at 0, step 1 / (12 lmbda / L), projection onto |p_voxel| <= 1 and onto x >= 0.  L >= |A|^2
defaults to the Schur bound max(A 1) max(A^T 1) (A is non-negative; two operator calls), or is passed as `L=`.
history[k] = {"data": 1/2 |A x_k - b|^2, "tv": TV(x_k), "F": data + lmbda tv} (one more A per iteration).  It is a
recognised convex baseline (TIGRE's algorithm collection has a FISTA with a TV proximal step); ASD-POCS, whose adaptive
step and stop rules are defined by TIGRE's implementation, is not what it computes.

cp_tv solves the data-constrained TV problem that the reference's ASD-POCS baseline targets,
    minimise  TV(x)   subject to   |A x - b| <= epsilon,   x >= 0   (nonneg=False drops the constraint)
with the same isotropic TV, by Chambolle-Pock (primal-dual hybrid gradient, as Sidky, Jorgensen and Pan 2012 use it
for CT) on K = [A; nu grad] (grad / div = -grad^T of csrc/r2x_tv.cu).  Step sizes: L >= |A|^2 (the Schur bound, as for
FISTA-TV, or `L=`), nu = sqrt(L / 12) so that |K|^2 <= L + 12 nu^2 = 2 L, tau = sigma = 0.99 / sqrt(2 L), so
tau sigma |K|^2 <= 0.98 < 1.  From x_0 = xbar_0 = 0, q_0 = 0 ([N, H, W]) and p_0 = 0 ([3, nx, ny, nz]); per iteration:
    1. u = q + sigma (A xbar - b),  q = max(1 - sigma epsilon / |u|, 0) u     (prox of sigma F*, F the indicator of the
       epsilon-ball around b; |u| a float64 reduction in a fixed order, as `_dot`)
    2. p = P_{1/nu}(p + sigma nu grad xbar)                                    (per voxel onto |p_i| <= 1/nu)
    3. x+ = P_C(x - tau A^T q + tau nu div p)                                  (C = {x >= 0} or everything)
    4. xbar = 2 x+ - x,  x = x+
Step 1 runs in projection space in torch, in the scaled form v = q / sigma + (A xbar - b), q / sigma =
max(1 - epsilon / |v|, 0) v (the same q), so that epsilon >= |b| gives q = 0 exactly and x stays exactly 0; steps 2-4
are one launch of `tv.tv_cp_step` (r2x_tv_cp_step) given A^T q.  history[k] = {"residual": |A x_k - b|, "tv": TV(x_k)};
A xbar is then 2 A x_k - A x_{k-1} from the history's projections (A is linear), so an iteration costs one A and one
A^T.  `cp_tv` takes epsilon = epsilon_ratio |A FDK(b) - b| by default (the reference's asd_pocs rule, 0.15, with this
project's FDK and projector); the ratio has no units.  Convergence with these steps is slow: on the noisy 256^3 scene
of DESIGN §8 the residual is still 4.7 epsilon after CP_NITER = 300 iterations (4.6 after 600), although 3D PSNR is
within 1.1 dB of FISTA-TV's there; the Schur L is 1.67 |A|^2 on that geometry, and tau = sigma is not tuned to the
scale of b.  So at the default iteration count the volume is a TV-regularised iterate on its way to the constrained
optimum, not that optimum; `history` shows how far the residual is from epsilon.

Parity with TIGRE's binaries is not pinned (as for FDK and the projector).  ASD-POCS / OS-ASD-POCS are not built:
their adaptive step and stop rules are defined by TIGRE's implementation.  `cp_tv` solves their convex problem and
`fista_tv` the TV-regularised least-squares one.

    python -m r2_gaussian_b200.recon -s <scene> -m <output> [--methods fdk,sart,cgls] [--short_scan]
        [--use_offDetector] [--estimate_offDetector] [--half_fan] [--fdk_filter ram_lak|shepp_logan|cosine|hamming|hann]
        [--use_view_geometry [--helical [--helical_q Q]]] [--fdk_pad F]

mirrors `scripts/run_traditional_methods.py`: it reconstructs the scene's train views with each method, scores the
volume against `vol_gt` with `metrics.metric_vol` and writes, per method, `<output>/<method>/ct_gt.npy`, `ct_pred.npy`,
`eval_3d.yml` (method, psnr_3d, ssim_3d, ssim_3d_x/y/z, duration (sec), duration (min); fdk under `--short_scan`
also `short_scan: true`, and `filter: <name>` under a `--fdk_filter` other than ram_lak; cp_tv ends with `epsilon` and
`residual`, the final |A x - b|) and the test views
`projs/{i:05d}_render.npy` (projections of the reconstruction) and `projs/{i:05d}_gt.npy`, plus `<output>/eval_3d.yml`
keyed by method.  PNG slices and projections are not written (matplotlib is not a dependency of this project).
`--short_scan` reconstructs fdk with Parker redundancy weights (`fdk.fdk(short_scan=True)`), for scenes whose train
views cover less than a full circle; it is refused when --methods has no fdk.  `--use_offDetector` reconstructs and
reprojects every method through the scanner's offDetector (without it a non-zero offset is refused by the projector
pair and ignored by fdk); `--half_fan` (with it, fdk only, not with --short_scan) adds half-fan redundancy weights for
a full circle whose detector is shifted sideways.  The reports add `half_fan: true` / `use_offDetector: true` only when
those flags are on.  `--estimate_offDetector` measures the horizontal detector offset from the train views
(`detector.estimate_offset`, on top of the file's offset under `--use_offDetector`) and runs every method, and the
test-view projections, with a copy of the scanner whose offDetector[0] is that total; `--half_fan` then needs no
`--use_offDetector`, and the reports add `estimated_offset_px` and `offDetector_u` (the file's units).  `--fdk_filter NAME` reconstructs fdk with one of TIGRE's windowed ramp filters
(`fdk.fdk(filter=NAME)`, overriding the scanner's `filter`); it is refused when --methods has no fdk.  Without it fdk
refuses a scanner whose `filter` names a window.  `--use_view_geometry` reconstructs and reprojects every method
through each view's own DSO, DSD, offOrigin and offDetector (the frames' keys, `scene.view_scanner`; reports add
`use_view_geometry: true`); fdk then refuses a helical scan (an offOrigin that varies), and the flag is refused with
--estimate_offDetector, --half_fan and --short_scan, which assume one fixed circle.  `--helical` (with it) reconstructs
fdk with helical redundancy weights instead (`fdk.fdk(helical=True, helical_q=Q)`; the report adds `helical: true` and
`helical_q`); it is refused without --use_view_geometry, when --methods has no fdk, and with --short_scan, --half_fan
and --estimate_offDetector.  cp_tv's tolerance keeps the CGLS volume in the plain FDK's place on a helical scan.
`--fdk_pad F` reconstructs fdk of a laterally truncated scan with each detector row extended by F of its width before
the ramp filter (`fdk.fdk(pad=F)`, 0 <= F <= 1; the report adds `pad: F` when F is not 0); it is refused when --methods
has no fdk, and with --half_fan, --helical and --use_view_geometry.
`--mar li|nmar` with `--metal_threshold T` or `--metal_mask M.npy` reduces metal artifacts first (`mar.reduce_metal`:
the metal is FDK > T of the train views, or the bool mask M): every method reconstructs the corrected train views, and
its metal voxels are then reinserted from the uncorrected FDK (`mar.reinsert`); the test renders are projections of
that volume.  The reports add `mar`, `metal_voxels`, `trace_fraction` (of the train views' pixels) and
`psnr_3d_outside_metal`, the PSNR over the voxels outside the metal mask dilated by 2 voxels with the peak taken as
vol_gt's maximum there.  `--mar` is refused with --use_view_geometry and --helical, the metal flags without `--mar`.
"""
from __future__ import annotations

import argparse
import math
import os
import sys
import time

import numpy as np
import torch

METHODS = ("fdk", "sart", "ossart", "cgls", "fista_tv", "cp_tv")
NOT_BUILT = ("asd_pocs", "os_asd_pocs")
# iteration counts and parameters of ct_utils.recon_volume / run_ct_recon_algs
CGLS_NITER = 60
SART_NITER = 20
OSSART_BLOCKSIZE = 10
# FISTA-TV defaults, chosen on one noisy fixture (DESIGN §8)
FISTA_NITER = 50
FISTA_LAMBDA = 1e-3
FISTA_TVITER = 20
# cp_tv defaults: the reference's asd_pocs epsilon ratio; CP_NITER from the convergence curve of DESIGN §8
CP_NITER = 300
CP_EPSILON_RATIO = 0.15


def _dot(a: torch.Tensor, b: torch.Tensor) -> float:
    return float((a * b).sum(dtype=torch.float64))


def cgls_solve(b: torch.Tensor, A, At, niter: int):
    """CGLS from x = 0 over the callables A(x, views) / At(y, views, weights); returns (x, l2 per iteration)."""
    everything = slice(None)
    r = b.clone()                                         # b - A 0
    p = At(r, everything, False)
    x = torch.zeros_like(p)
    gamma = _dot(p, p)
    l2 = []
    for _ in range(niter):
        if gamma == 0.0:                                  # A^T r = 0: x is a least-squares solution
            break
        q = A(p, everything)
        alpha = gamma / _dot(q, q)
        x.add_(p, alpha=alpha)
        r.sub_(q, alpha=alpha)
        l2.append(_dot(r, r) ** 0.5)
        s = At(r, everything, False)
        gamma_new = _dot(s, s)
        p = s.add_(p, alpha=gamma_new / gamma)
        gamma = gamma_new
    return x, l2


def sart_solve(b: torch.Tensor, A, At, shape, niter: int, lmbda: float = 1.0, lmbda_red: float = 0.999,
               blocksize: int = 1, nonneg: bool = True) -> torch.Tensor:
    """SART / OS-SART from x = 0 over the callables A(x, views) / At(y, views, weights); `shape` is the volume's."""
    if blocksize < 1:
        raise ValueError(f"sart: blocksize must be >= 1, got {blocksize}")
    n = int(b.shape[0])
    x = torch.zeros(tuple(shape), dtype=b.dtype, device=b.device)
    w = A(torch.ones_like(x), slice(None))
    w = torch.where(w > 0, 1.0 / w, torch.zeros_like(w))
    blocks = [slice(v, min(v + blocksize, n)) for v in range(0, n, blocksize)]
    for _ in range(niter):
        for views in blocks:
            r = w[views] * (b[views] - A(x, views))
            num, den = At(r, views, True)
            x.add_(torch.where(den > 0, num / den, torch.zeros_like(num)), alpha=lmbda)
            if nonneg:
                x.clamp_(min=0.0)
        lmbda *= lmbda_red
    return x


def _check_fista(niter, lmbda, tviter, L):
    if int(niter) != niter or niter < 1:
        raise ValueError(f"fista_tv: niter must be an integer >= 1, got {niter}")
    if not (float(lmbda) >= 0.0 and math.isfinite(float(lmbda))):
        raise ValueError(f"fista_tv: lmbda must be finite and >= 0, got {lmbda}")
    if int(tviter) != tviter or tviter < 1:
        raise ValueError(f"fista_tv: tviter must be an integer >= 1, got {tviter}")
    if L is not None and not (float(L) > 0.0 and math.isfinite(float(L))):
        raise ValueError(f"fista_tv: L must be finite and > 0, got {L}")


def schur_lipschitz(b: torch.Tensor, A, At, shape) -> float:
    """max(A 1) max(A^T 1), an upper bound of |A|^2 for a non-negative A (|A|_2^2 <= |A|_1 |A|_inf)."""
    everything = slice(None)
    a1 = A(torch.ones(tuple(shape), dtype=b.dtype, device=b.device), everything)
    at1 = At(torch.ones_like(b), everything, False)
    return float(a1.max()) * float(at1.max())


def fista_tv_solve(b: torch.Tensor, A, At, shape, niter: int, lmbda: float, tviter: int = FISTA_TVITER, L=None,
                   nonneg: bool = True, prox=None, tv=None):
    """FISTA-TV from x = 0 over the callables A(x, views) / At(y, views, weights); `shape` is the volume's.  `prox(v,
    weight, tviter, nonneg)` and `tv(x)` default to the GPU `tv.tv_denoise` / `tv.tv_value`.  Returns (x, history)."""
    _check_fista(niter, lmbda, tviter, L)
    if prox is None:
        from .tv import tv_denoise as prox
    if tv is None:
        from .tv import tv_value as tv
    everything = slice(None)
    if L is None:
        L = schur_lipschitz(b, A, At, shape)
        if not L > 0.0:
            raise ValueError("fista_tv: A 1 or A^T 1 is zero: no ray meets the volume")
    L = float(L)
    x_prev = torch.zeros(tuple(shape), dtype=b.dtype, device=b.device)
    y = x_prev
    t = 1.0
    history = []
    for _ in range(niter):
        grad = At(A(y, everything).sub_(b), everything, False)
        x = prox(y.sub(grad, alpha=1.0 / L), float(lmbda) / L, tviter, nonneg)
        t_next = 0.5 * (1.0 + math.sqrt(1.0 + 4.0 * t * t))
        y = x.add(x - x_prev, alpha=(t - 1.0) / t_next)
        r = A(x, everything).sub_(b)
        data, tvx = 0.5 * _dot(r, r), float(tv(x))
        history.append({"data": data, "tv": tvx, "F": data + float(lmbda) * tvx})
        x_prev, t = x, t_next
    return x_prev, history


def _check_cp(niter, epsilon, L):
    if int(niter) != niter or niter < 1:
        raise ValueError(f"cp_tv: niter must be an integer >= 1, got {niter}")
    if epsilon is not None and not (float(epsilon) >= 0.0 and math.isfinite(float(epsilon))):
        raise ValueError(f"cp_tv: epsilon must be finite and >= 0, got {epsilon}")
    if L is not None and not (float(L) > 0.0 and math.isfinite(float(L))):
        raise ValueError(f"cp_tv: L must be finite and > 0, got {L}")


def cp_step_sizes(L: float) -> tuple[float, float, float]:
    """(tau, sigma, nu) of cp_tv for L >= |A|^2: nu = sqrt(L / 12), tau = sigma = 0.99 / sqrt(2 L)."""
    tau = 0.99 / math.sqrt(2.0 * L)
    return tau, tau, math.sqrt(L / 12.0)


def cp_tv_solve(b: torch.Tensor, A, At, shape, niter: int, epsilon: float, L=None, nonneg: bool = True, step=None,
                tv=None):
    """Chambolle-Pock for min TV(x) s.t. |A x - b| <= epsilon (and x >= 0 when nonneg) from x = 0, over the callables
    A(x, views) / At(y, views, weights); `shape` is the volume's.  `step(x, xbar, p, g, tau, sigma, nu, nonneg)` and
    `tv(x)` default to the GPU `tv.tv_cp_step` / `tv.tv_value`.  Returns (x, history)."""
    _check_cp(niter, epsilon, L)
    if epsilon is None:
        raise ValueError("cp_tv: epsilon must be given")
    if step is None:
        from .tv import tv_cp_step as step
    if tv is None:
        from .tv import tv_value as tv
    everything = slice(None)
    if L is None:
        L = schur_lipschitz(b, A, At, shape)
        if not L > 0.0:
            raise ValueError("cp_tv: A 1 or A^T 1 is zero: no ray meets the volume")
    tau, sigma, nu = cp_step_sizes(float(L))
    epsilon = float(epsilon)
    x = torch.zeros(tuple(shape), dtype=b.dtype, device=b.device)
    xbar = x
    p = torch.zeros((3,) + tuple(shape), dtype=b.dtype, device=b.device)
    y = torch.zeros_like(b)                               # q / sigma
    ax = torch.zeros_like(b)                              # A x_k (A 0 = 0)
    ax_bar = ax                                           # A xbar_k
    history = []
    for _ in range(niter):
        v = ax_bar.sub(b).add_(y)
        norm = _dot(v, v) ** 0.5
        y = torch.zeros_like(v) if norm <= epsilon else v.mul_(1.0 - epsilon / norm)
        g = At(y.mul(sigma), everything, False)
        x_next, xbar, p = step(x, xbar, p, g, tau, sigma, nu, nonneg)
        ax_next = A(x_next, everything)
        r = ax_next.sub(b)
        history.append({"residual": _dot(r, r) ** 0.5, "tv": float(tv(x_next))})
        ax_bar = ax_next.mul(2.0).sub_(ax)
        x, ax = x_next, ax_next
    return x, history


def _operator(projs, angles, scanner_cfg, use_offDetector: bool = False, view_geometry=None):
    from .projector import CTOperator

    if not isinstance(projs, torch.Tensor) or projs.device.type != "cuda":
        raise RuntimeError("recon: projections must be a CUDA tensor (this build has no CPU fallback; "
                           f"got {getattr(projs, 'device', type(projs))})")
    op = CTOperator(angles, scanner_cfg, projs.device, use_offDetector, view_geometry)
    b = projs.detach().to(torch.float32).contiguous()
    if tuple(b.shape) != (op.N, op.H, op.W):
        raise ValueError(f"recon: projections {list(b.shape)} do not match {op.N} angles of {op.H}x{op.W} pixels")
    return op, b


def cgls(projs: torch.Tensor, angles, scanner_cfg: dict, niter: int = CGLS_NITER, use_offDetector: bool = False,
         view_geometry=None):
    """CGLS on the GPU projector pair; returns (volume, l2 per iteration)."""
    op, b = _operator(projs, angles, scanner_cfg, use_offDetector, view_geometry)
    return cgls_solve(b, op.A, op.At, niter)


def sart(projs: torch.Tensor, angles, scanner_cfg: dict, niter: int = SART_NITER, lmbda: float = 1.0,
         lmbda_red: float = 0.999, blocksize: int = 1, nonneg: bool = True,
         use_offDetector: bool = False, view_geometry=None) -> torch.Tensor:
    """SART (blocksize 1) or OS-SART on the GPU projector pair."""
    op, b = _operator(projs, angles, scanner_cfg, use_offDetector, view_geometry)
    return sart_solve(b, op.A, op.At, op.nvox, niter, lmbda, lmbda_red, blocksize, nonneg)


def fista_tv(projs: torch.Tensor, angles, scanner_cfg: dict, niter: int = FISTA_NITER, lmbda: float = FISTA_LAMBDA,
             tviter: int = FISTA_TVITER, nonneg: bool = True, L=None, use_offDetector: bool = False,
             view_geometry=None):
    """FISTA-TV on the GPU projector pair and the GPU TV prox; returns (volume, history)."""
    _check_fista(niter, lmbda, tviter, L)
    op, b = _operator(projs, angles, scanner_cfg, use_offDetector, view_geometry)
    return fista_tv_solve(b, op.A, op.At, op.nvox, niter, lmbda, tviter, L, nonneg)


def _check_ratio(epsilon_ratio):
    if not (float(epsilon_ratio) >= 0.0 and math.isfinite(float(epsilon_ratio))):
        raise ValueError(f"cp_tv: epsilon_ratio must be finite and >= 0, got {epsilon_ratio}")


def cp_tv_epsilon(projs: torch.Tensor, angles, scanner_cfg: dict, epsilon_ratio: float = CP_EPSILON_RATIO,
                  use_offDetector: bool = False, view_geometry=None) -> float:
    """epsilon_ratio |A FDK(b) - b|, the reference's asd_pocs tolerance, with this project's FDK and projector.  FDK
    has no helical weighting, so a per-view geometry whose offOrigin varies takes the CGLS volume in FDK's place."""
    from .fdk import fdk, helical

    _check_ratio(epsilon_ratio)
    op, b = _operator(projs, angles, scanner_cfg, use_offDetector, view_geometry)
    if view_geometry is not None and helical(scanner_cfg, view_geometry):
        x0 = cgls_solve(b, op.A, op.At, CGLS_NITER)[0]
    else:
        x0 = fdk(b, angles, scanner_cfg, use_offDetector=use_offDetector, view_geometry=view_geometry)
    r = op.A(x0).sub_(b)
    return float(epsilon_ratio) * _dot(r, r) ** 0.5


def cp_tv(projs: torch.Tensor, angles, scanner_cfg: dict, niter: int = CP_NITER, epsilon=None,
          epsilon_ratio: float = CP_EPSILON_RATIO, L=None, nonneg: bool = True, use_offDetector: bool = False,
          view_geometry=None):
    """Data-constrained TV (Chambolle-Pock) on the GPU projector pair and the GPU step kernel; epsilon=None takes
    `cp_tv_epsilon(..., epsilon_ratio)`.  Returns (volume, history)."""
    _check_cp(niter, epsilon, L)
    _check_ratio(epsilon_ratio)
    op, b = _operator(projs, angles, scanner_cfg, use_offDetector, view_geometry)
    if epsilon is None:
        epsilon = cp_tv_epsilon(b, angles, scanner_cfg, epsilon_ratio, use_offDetector, view_geometry)
    return cp_tv_solve(b, op.A, op.At, op.nvox, niter, epsilon, L, nonneg)


def recon_volume(projs: torch.Tensor, angles, scanner_cfg: dict, method: str, short_scan: bool = False,
                 use_offDetector: bool = False, half_fan: bool = False, fdk_filter: str | None = None,
                 view_geometry=None, helical: bool = False, helical_q: float | None = None,
                 fdk_pad: float = 0.0) -> torch.Tensor:
    """The reconstructions of ct_utils.recon_volume / run_ct_recon_algs with their iteration counts.  `short_scan`
    selects the Parker-weighted FDK, `half_fan` the half-fan-weighted one, `helical` (with `helical_q`, None for
    fdk.HELICAL_Q) the helical one, `fdk_filter` FDK's ramp filter (`fdk.fdk(filter=...)`) and `fdk_pad` its truncation
    pad (`fdk.fdk(pad=...)`); all five apply to method fdk only.  `use_offDetector` reconstructs through the scanner's offDetector (every method), `view_geometry`
    through each view's own geometry (every method; `projector.project`)."""
    for flag, on in (("short_scan", short_scan), ("half_fan", half_fan), ("helical", helical)):
        if on and method != "fdk":
            raise ValueError(f"recon_volume: {flag} applies to fdk only, not {method!r} (the iterative methods need no "
                             "redundancy weights)")
    if fdk_filter is not None and method != "fdk":
        raise ValueError(f"recon_volume: fdk_filter applies to fdk only, not {method!r} (the iterative methods have no "
                         "ramp filter)")
    if fdk_pad and method != "fdk":
        raise ValueError(f"recon_volume: fdk_pad applies to fdk only, not {method!r} (the iterative methods have no "
                         "ramp filter)")
    off = use_offDetector
    if method == "fdk":
        from .fdk import HELICAL_Q, fdk

        return fdk(projs, angles, scanner_cfg, short_scan=short_scan, use_offDetector=off, half_fan=half_fan,
                   filter=fdk_filter, view_geometry=view_geometry, helical=helical,
                   helical_q=HELICAL_Q if helical_q is None else helical_q, pad=fdk_pad)
    vg = view_geometry
    if method == "cgls":
        return cgls(projs, angles, scanner_cfg, CGLS_NITER, use_offDetector=off, view_geometry=vg)[0]
    if method == "sart":
        return sart(projs, angles, scanner_cfg, SART_NITER, use_offDetector=off, view_geometry=vg)
    if method == "ossart":
        return sart(projs, angles, scanner_cfg, SART_NITER, blocksize=OSSART_BLOCKSIZE, use_offDetector=off,
                    view_geometry=vg)
    if method == "fista_tv":
        return fista_tv(projs, angles, scanner_cfg, use_offDetector=off, view_geometry=vg)[0]
    if method == "cp_tv":
        return cp_tv(projs, angles, scanner_cfg, use_offDetector=off, view_geometry=vg)[0]
    raise ValueError(f"recon_volume: unknown method {method!r} (supported: {', '.join(METHODS)})")


def check_fdk_flags(args, fdk_selected: bool, not_fdk: str):
    """The refusals of the FDK flags (--short_scan, --half_fan, --fdk_filter, --fdk_pad) that the recon and
    initialize_pcd CLIs share; `not_fdk` is the CLI's message for a flag given without the fdk method, with `{flag}`
    standing for the flag."""
    pad = getattr(args, "fdk_pad", None)
    for flag, on in (("--short_scan", args.short_scan), ("--half_fan", args.half_fan),
                     ("--fdk_filter", args.fdk_filter is not None), ("--fdk_pad", pad is not None)):
        if on and not fdk_selected:
            raise SystemExit(not_fdk.format(flag=flag))
    if pad is not None:
        if not 0.0 <= pad <= 1.0:
            raise SystemExit(f"--fdk_pad must be a fraction of the detector width in [0, 1], got {pad}")
        for flag, why in (("--half_fan", "an offset detector's truncation is deliberate and its weights already "
                                         "handle it"),
                          ("--helical", "the helical FDK has no truncation pad"),
                          ("--use_view_geometry", "the per-view FDK has no truncation pad")):
            if getattr(args, flag[2:], False):
                raise SystemExit(f"--fdk_pad cannot be combined with {flag} ({why})")
    if args.half_fan and not (args.use_offDetector or getattr(args, "estimate_offDetector", False)):
        raise SystemExit("--half_fan needs --use_offDetector (or --estimate_offDetector): the half-fan weights follow "
                         "the detector offset")
    if args.half_fan and args.short_scan:
        raise SystemExit("--half_fan and --short_scan cannot be combined (half-fan weights need a full circle)")


def add_fdk_filter_flag(ap, help_text: str):
    """--fdk_filter NAME (one of fdk.FILTERS) on a CLI's parser."""
    from .fdk import FILTERS

    ap.add_argument("--fdk_filter", default=None, choices=FILTERS, metavar="NAME",
                    help=f"{help_text}: {', '.join(FILTERS)} (TIGRE's names; default: the scanner's filter, which must "
                         "then be null or ram_lak)")


def add_fdk_pad_flag(ap, help_text: str):
    """--fdk_pad F on a CLI's parser."""
    ap.add_argument("--fdk_pad", default=None, type=float, metavar="F",
                    help=f"{help_text}: extend each detector row by F of its width (0 <= F <= 1) with its rolled-off "
                         "mirror before the ramp filter, for a scan whose object is wider than the detector's field of "
                         "view (fdk.fdk(pad=F))")


def add_helical_flags(ap):
    """--helical and --helical_q Q on a CLI's parser."""
    from .fdk import HELICAL_Q

    ap.add_argument("--helical", default=False, action="store_true",
                    help="with --use_view_geometry: reconstruct fdk with helical redundancy weights (fdk.fdk(helical="
                         "True); a helical scan, or a circle of 360 degrees or more)")
    ap.add_argument("--helical_q", default=None, type=float, metavar="Q",
                    help=f"with --helical: the fraction of the detector's half-height weighted fully before the "
                         f"weights fall to 0 at its edge, in [0, 1] (default {HELICAL_Q})")


def check_helical_flags(args, fdk_selected: bool, not_fdk: str):
    """The refusals of --helical and --helical_q that the recon and initialize_pcd CLIs share, before any CUDA work;
    `not_fdk` as for check_fdk_flags."""
    if args.helical_q is not None and not args.helical:
        raise SystemExit("--helical_q applies with --helical only")
    if not args.helical:
        return
    if not fdk_selected:
        raise SystemExit(not_fdk.format(flag="--helical"))
    if not args.use_view_geometry:
        raise SystemExit("--helical needs --use_view_geometry: the helix is read from the views' offOrigin")
    for flag in ("--short_scan", "--half_fan", "--estimate_offDetector"):
        if getattr(args, flag[2:], False):
            raise SystemExit(f"--helical cannot be combined with {flag} (its weights or its estimate assume one fixed "
                             "circle)")
    if args.helical_q is not None and not 0.0 <= args.helical_q <= 1.0:
        raise SystemExit(f"--helical_q must be in [0, 1], got {args.helical_q}")


def add_estimate_flag(ap, what: str):
    """--estimate_offDetector on a CLI's parser."""
    ap.add_argument("--estimate_offDetector", default=False, action="store_true",
                    help=f"estimate the horizontal detector offset from the train views (detector.estimate_offset; "
                         f"relative to the scanner's offDetector under --use_offDetector) and {what} through it")


def add_view_geometry_flag(ap, what: str):
    """--use_view_geometry on a CLI's parser."""
    ap.add_argument("--use_view_geometry", default=False, action="store_true",
                    help=f"{what} through each view's own DSO, DSD, offOrigin and offDetector (the projection frames' "
                         "keys; helical scans, calibrated benches); implies --use_offDetector")


def check_view_geometry_flags(args):
    """The refusals of --use_view_geometry that every CLI shares; checked before any CUDA work."""
    if not getattr(args, "use_view_geometry", False):
        return
    for flag, on in (("--estimate_offDetector", getattr(args, "estimate_offDetector", False)),
                     ("--half_fan", getattr(args, "half_fan", False)),
                     ("--short_scan", getattr(args, "short_scan", False))):
        if on:
            why = ("the conjugate-ray estimate assumes one fixed circle" if flag == "--estimate_offDetector" else
                   "its redundancy weights assume one fixed circle")
            raise SystemExit(f"{flag} cannot be combined with --use_view_geometry: {why}")


def view_geometry_of(cameras, on: bool):
    """The per-view geometry (`CameraInfo.view_geometry`) of `cameras` under --use_view_geometry, else None."""
    return [c.view_geometry for c in cameras] if on else None


def add_mar_flags(ap):
    """--mar li|nmar, --metal_threshold T and --metal_mask M.npy on a CLI's parser."""
    from .mar import METHODS as MAR_METHODS

    ap.add_argument("--mar", default=None, choices=MAR_METHODS,
                    help="reduce metal artifacts in the train views first (mar.reduce_metal) and reinsert the metal of "
                         "the uncorrected FDK into every reconstruction")
    ap.add_argument("--metal_threshold", default=None, type=float, metavar="T",
                    help="with --mar: metal = FDK of the train views > T (scene-scaled units)")
    ap.add_argument("--metal_mask", default=None, metavar="M.npy", help="with --mar: a bool nVoxel-shaped metal mask")


def check_mar_flags(args):
    """The refusals of --mar, --metal_threshold and --metal_mask, before any CUDA work."""
    given = [f for f in ("--metal_threshold", "--metal_mask") if getattr(args, f[2:]) is not None]
    if args.mar is None:
        if given:
            raise SystemExit(f"{given[0]} applies with --mar only")
        return
    for flag in ("--use_view_geometry", "--helical"):
        if getattr(args, flag[2:], False):
            raise SystemExit(f"--mar cannot be combined with {flag}: the metal trace and the NMAR prior would need the "
                             "per-view FDK")
    if len(given) != 1:
        raise SystemExit("--mar needs exactly one of --metal_threshold T and --metal_mask M.npy")
    if args.metal_threshold is not None and not math.isfinite(args.metal_threshold):
        raise SystemExit(f"--metal_threshold must be finite, got {args.metal_threshold}")


def _parse_methods(text: str) -> list[str]:
    methods = [m.strip() for m in text.split(",") if m.strip()]
    for m in methods:
        if m in NOT_BUILT:
            raise SystemExit(f"method {m} is not built (ASD-POCS is not part of this project; fista_tv is its "
                             f"TV-regularised alternative); supported: {', '.join(METHODS)}")
        if m not in METHODS:
            raise SystemExit(f"unknown method {m!r}; supported: {', '.join(METHODS)}")
    if not methods:
        raise SystemExit(f"no methods given; supported: {', '.join(METHODS)}")
    return methods


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description="Traditional CT reconstructions (FDK, SART, OS-SART, CGLS, FISTA-TV, "
                                             "CP-TV) of a scene")
    ap.add_argument("-s", "--source_path", required=True, help="scene directory or NAF pickle")
    ap.add_argument("-m", "--model_path", required=True, help="output directory")
    ap.add_argument("--methods", default="fdk,sart,cgls", help=f"comma-separated subset of {','.join(METHODS)}")
    ap.add_argument("--short_scan", default=False, action="store_true",
                    help="reconstruct fdk with Parker redundancy weights (a scan over less than 360 degrees)")
    ap.add_argument("--use_offDetector", default=False, action="store_true",
                    help="reconstruct and reproject through the scanner's offDetector (every method)")
    ap.add_argument("--half_fan", default=False, action="store_true",
                    help="with --use_offDetector: reconstruct fdk with half-fan redundancy weights (a full circle with "
                         "the detector shifted sideways)")
    add_fdk_filter_flag(ap, "reconstruct fdk with this ramp filter")
    add_fdk_pad_flag(ap, "reconstruct fdk of a laterally truncated scan")
    add_estimate_flag(ap, "reconstruct and reproject every method")
    add_view_geometry_flag(ap, "reconstruct and reproject every method")
    add_helical_flags(ap)
    add_mar_flags(ap)
    a = ap.parse_args(argv)
    methods = _parse_methods(a.methods)
    check_mar_flags(a)
    check_fdk_flags(a, "fdk" in methods, "{flag} applies to the fdk method, which --methods does not include (the "
                    "iterative methods need no redundancy weights)")
    check_helical_flags(a, "fdk" in methods, "{flag} applies to the fdk method, which --methods does not include (the "
                        "iterative methods need no redundancy weights)")
    check_view_geometry_flags(a)
    if not torch.cuda.is_available():
        raise SystemExit("the reconstructions need a CUDA device: they run on the GPU and have no CPU fallback")
    import yaml

    from .dataset import read_scene
    from .metrics import metric_vol
    from .projector import project

    source = os.path.abspath(a.source_path)
    info = read_scene(source, eval=True, use_view_geometry=a.use_view_geometry)
    cfg = info.scanner_cfg
    vg_train = view_geometry_of(info.train_cameras, a.use_view_geometry)
    vg_test = view_geometry_of(info.test_cameras, a.use_view_geometry)
    if a.helical:
        from .fdk import helix_views
        try:
            helix_views([c.angle for c in info.train_cameras], cfg, vg_train)
        except ValueError as e:
            raise SystemExit(f"--helical: {e}") from e
    projs_train = torch.from_numpy(np.stack([np.asarray(c.image, np.float32) for c in info.train_cameras])).cuda()
    train_angles = [c.angle for c in info.train_cameras]
    test_angles = [c.angle for c in info.test_cameras]
    vol_gt = np.asarray(info.vol, np.float32)
    use_off, estimate = a.use_offDetector or a.use_view_geometry, None
    if a.estimate_offDetector:
        from .estimate_offset import estimated_scanner
        cfg, estimate = estimated_scanner(info, a.use_offDetector)
        use_off = True
    metal = None
    if a.mar:
        from .mar import reduce_metal
        from .reduce_metal import load_mask

        mask = None
        if a.metal_mask is not None:
            mask = load_mask(a.metal_mask)
        metal = reduce_metal(projs_train, train_angles, cfg, method=a.mar, threshold=a.metal_threshold, mask=mask,
                             use_offDetector=use_off, short_scan=a.short_scan, half_fan=a.half_fan,
                             fdk_filter=a.fdk_filter, fdk_pad=a.fdk_pad or 0.0)
        projs_train = metal.projs
    out = {}
    print(f"Run traditional algorithms on {os.path.basename(source)}")
    for method in methods:
        print(f"Run {method}...")
        save = os.path.join(a.model_path, method)
        os.makedirs(os.path.join(save, "projs"), exist_ok=True)
        torch.cuda.synchronize()
        t0 = time.time()
        short_scan = a.short_scan and method == "fdk"
        half_fan = a.half_fan and method == "fdk"
        helical_fdk = a.helical and method == "fdk"
        fdk_filter = a.fdk_filter if method == "fdk" else None
        fdk_pad = (a.fdk_pad or 0.0) if method == "fdk" else 0.0
        extra = {}
        if method == "cp_tv":
            eps = cp_tv_epsilon(projs_train, train_angles, cfg, use_offDetector=use_off, view_geometry=vg_train)
            pred, hist = cp_tv(projs_train, train_angles, cfg, epsilon=eps, use_offDetector=use_off,
                               view_geometry=vg_train)
            extra = {"epsilon": eps, "residual": hist[-1]["residual"]}
        else:
            pred = recon_volume(projs_train, train_angles, cfg, method, short_scan=short_scan,
                                use_offDetector=use_off, half_fan=half_fan, fdk_filter=fdk_filter,
                                view_geometry=vg_train, helical=helical_fdk, helical_q=a.helical_q,
                                fdk_pad=fdk_pad)
        if metal is not None:
            from .mar import reinsert
            pred = reinsert(pred, metal.fdk, metal.mask)
        torch.cuda.synchronize()
        duration = time.time() - t0
        ct_pred = pred.cpu().numpy()
        psnr_3d, _ = metric_vol(vol_gt, ct_pred, "psnr")
        ssim_3d, ssim_axis = metric_vol(vol_gt, ct_pred, "ssim")
        np.save(os.path.join(save, "ct_gt.npy"), vol_gt)
        np.save(os.path.join(save, "ct_pred.npy"), ct_pred)
        report = {"method": method, "psnr_3d": float(psnr_3d), "ssim_3d": float(ssim_3d),
                  "ssim_3d_x": float(ssim_axis[0]), "ssim_3d_y": float(ssim_axis[1]), "ssim_3d_z": float(ssim_axis[2]),
                  "duration (sec)": duration, "duration (min)": duration / 60}
        if short_scan:
            report["short_scan"] = True
        if half_fan:
            report["half_fan"] = True
        if helical_fdk:
            from .fdk import HELICAL_Q
            report["helical"] = True
            report["helical_q"] = float(HELICAL_Q if a.helical_q is None else a.helical_q)
        if fdk_filter not in (None, "ram_lak"):
            report["filter"] = fdk_filter
        if fdk_pad:
            report["pad"] = float(fdk_pad)
        if a.use_offDetector:
            report["use_offDetector"] = True
        if a.use_view_geometry:
            report["use_view_geometry"] = True
        if estimate is not None:
            report["estimated_offset_px"] = estimate["offset_px"]
            report["offDetector_u"] = estimate["offDetector_u"] / info.scene_scale
        if metal is not None:
            from .mar import psnr_outside_metal
            report.update({"mar": a.mar, "metal_voxels": int(metal.mask.sum()),
                           "trace_fraction": metal.trace_fraction,
                           "psnr_3d_outside_metal": psnr_outside_metal(vol_gt, ct_pred, metal.mask.cpu())})
        report.update(extra)
        with open(os.path.join(save, "eval_3d.yml"), "w") as f:
            yaml.dump(report, f, default_flow_style=False, sort_keys=False)
        if test_angles:
            render = project(pred, test_angles, cfg, use_offDetector=use_off, view_geometry=vg_test).cpu().numpy()
            for i, cam in enumerate(info.test_cameras):
                np.save(os.path.join(save, "projs", f"{i:05d}_render.npy"), render[i])
                np.save(os.path.join(save, "projs", f"{i:05d}_gt.npy"), np.asarray(cam.image, np.float32))
        out[method] = report
        print(f"[{method}] psnr_3d: {psnr_3d}, ssim_3d: {ssim_3d}")
    with open(os.path.join(a.model_path, "eval_3d.yml"), "w") as f:
        yaml.dump(out, f, default_flow_style=False, sort_keys=False)
    print(f"Run traditional algorithms on {os.path.basename(source)} complete")
    return out


if __name__ == "__main__":
    main(sys.argv[1:])
