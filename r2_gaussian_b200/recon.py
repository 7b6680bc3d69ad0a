"""Traditional CT reconstructions on the GPU -- FDK, SART / OS-SART and CGLS, what the reference obtains from TIGRE's
`algs` (`r2_gaussian/utils/ct_utils.py::recon_volume` / `run_ct_recon_algs`, `scripts/run_traditional_methods.py`),
and the TV-regularised FISTA-TV.

    x, l2 = cgls(projs, angles, scanner_cfg, niter=60)
    x = sart(projs, angles, scanner_cfg, niter=20, lmbda=1.0, lmbda_red=0.999, blocksize=1, nonneg=True)
    x, history = fista_tv(projs, angles, scanner_cfg, niter=FISTA_NITER, lmbda=FISTA_LAMBDA, tviter=20, nonneg=True)
    x = recon_volume(projs, angles, scanner_cfg, method)           # fdk | cgls | sart | ossart | fista_tv

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

Parity with TIGRE's binaries is not pinned (as for FDK and the projector).  ASD-POCS / OS-ASD-POCS are not built;
`fista_tv` is the TV-regularised method this project offers.

    python -m r2_gaussian_b200.recon -s <scene> -m <output> [--methods fdk,sart,cgls] [--short_scan]
        [--use_offDetector [--half_fan]] [--fdk_filter ram_lak|shepp_logan|cosine|hamming|hann]

mirrors `scripts/run_traditional_methods.py`: it reconstructs the scene's train views with each method, scores the
volume against `vol_gt` with `metrics.metric_vol` and writes, per method, `<output>/<method>/ct_gt.npy`, `ct_pred.npy`,
`eval_3d.yml` (method, psnr_3d, ssim_3d, ssim_3d_x/y/z, duration (sec), duration (min); fdk under `--short_scan`
also `short_scan: true`, and `filter: <name>` under a `--fdk_filter` other than ram_lak) and the test views
`projs/{i:05d}_render.npy` (projections of the reconstruction) and `projs/{i:05d}_gt.npy`, plus `<output>/eval_3d.yml`
keyed by method.  PNG slices and projections are not written (matplotlib is not a dependency of this project).
`--short_scan` reconstructs fdk with Parker redundancy weights (`fdk.fdk(short_scan=True)`), for scenes whose train
views cover less than a full circle; it is refused when --methods has no fdk.  `--use_offDetector` reconstructs and
reprojects every method through the scanner's offDetector (without it a non-zero offset is refused by the projector
pair and ignored by fdk); `--half_fan` (with it, fdk only, not with --short_scan) adds half-fan redundancy weights for
a full circle whose detector is shifted sideways.  The reports add `half_fan: true` / `use_offDetector: true` only when
those flags are on.  `--fdk_filter NAME` reconstructs fdk with one of TIGRE's windowed ramp filters
(`fdk.fdk(filter=NAME)`, overriding the scanner's `filter`); it is refused when --methods has no fdk.  Without it fdk
refuses a scanner whose `filter` names a window.
"""
from __future__ import annotations

import argparse
import math
import os
import sys
import time

import numpy as np
import torch

METHODS = ("fdk", "sart", "ossart", "cgls", "fista_tv")
NOT_BUILT = ("asd_pocs", "os_asd_pocs")
# iteration counts and parameters of ct_utils.recon_volume / run_ct_recon_algs
CGLS_NITER = 60
SART_NITER = 20
OSSART_BLOCKSIZE = 10
# FISTA-TV defaults, chosen on one noisy fixture (DESIGN §8)
FISTA_NITER = 50
FISTA_LAMBDA = 1e-3
FISTA_TVITER = 20


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


def _operator(projs, angles, scanner_cfg, use_offDetector: bool = False):
    from .projector import CTOperator

    if not isinstance(projs, torch.Tensor) or projs.device.type != "cuda":
        raise RuntimeError("recon: projections must be a CUDA tensor (this build has no CPU fallback; "
                           f"got {getattr(projs, 'device', type(projs))})")
    op = CTOperator(angles, scanner_cfg, projs.device, use_offDetector)
    b = projs.detach().to(torch.float32).contiguous()
    if tuple(b.shape) != (op.N, op.H, op.W):
        raise ValueError(f"recon: projections {list(b.shape)} do not match {op.N} angles of {op.H}x{op.W} pixels")
    return op, b


def cgls(projs: torch.Tensor, angles, scanner_cfg: dict, niter: int = CGLS_NITER, use_offDetector: bool = False):
    """CGLS on the GPU projector pair; returns (volume, l2 per iteration)."""
    op, b = _operator(projs, angles, scanner_cfg, use_offDetector)
    return cgls_solve(b, op.A, op.At, niter)


def sart(projs: torch.Tensor, angles, scanner_cfg: dict, niter: int = SART_NITER, lmbda: float = 1.0,
         lmbda_red: float = 0.999, blocksize: int = 1, nonneg: bool = True,
         use_offDetector: bool = False) -> torch.Tensor:
    """SART (blocksize 1) or OS-SART on the GPU projector pair."""
    op, b = _operator(projs, angles, scanner_cfg, use_offDetector)
    return sart_solve(b, op.A, op.At, op.nvox, niter, lmbda, lmbda_red, blocksize, nonneg)


def fista_tv(projs: torch.Tensor, angles, scanner_cfg: dict, niter: int = FISTA_NITER, lmbda: float = FISTA_LAMBDA,
             tviter: int = FISTA_TVITER, nonneg: bool = True, L=None, use_offDetector: bool = False):
    """FISTA-TV on the GPU projector pair and the GPU TV prox; returns (volume, history)."""
    _check_fista(niter, lmbda, tviter, L)
    op, b = _operator(projs, angles, scanner_cfg, use_offDetector)
    return fista_tv_solve(b, op.A, op.At, op.nvox, niter, lmbda, tviter, L, nonneg)


def recon_volume(projs: torch.Tensor, angles, scanner_cfg: dict, method: str, short_scan: bool = False,
                 use_offDetector: bool = False, half_fan: bool = False, fdk_filter: str | None = None) -> torch.Tensor:
    """The reconstructions of ct_utils.recon_volume / run_ct_recon_algs with their iteration counts.  `short_scan`
    selects the Parker-weighted FDK, `half_fan` the half-fan-weighted one and `fdk_filter` FDK's ramp filter
    (`fdk.fdk(filter=...)`); all three apply to method fdk only.  `use_offDetector` reconstructs through the scanner's
    offDetector (every method)."""
    for flag, on in (("short_scan", short_scan), ("half_fan", half_fan)):
        if on and method != "fdk":
            raise ValueError(f"recon_volume: {flag} applies to fdk only, not {method!r} (the iterative methods need no "
                             "redundancy weights)")
    if fdk_filter is not None and method != "fdk":
        raise ValueError(f"recon_volume: fdk_filter applies to fdk only, not {method!r} (the iterative methods have no "
                         "ramp filter)")
    off = use_offDetector
    if method == "fdk":
        from .fdk import fdk

        return fdk(projs, angles, scanner_cfg, short_scan=short_scan, use_offDetector=off, half_fan=half_fan,
                   filter=fdk_filter)
    if method == "cgls":
        return cgls(projs, angles, scanner_cfg, CGLS_NITER, use_offDetector=off)[0]
    if method == "sart":
        return sart(projs, angles, scanner_cfg, SART_NITER, use_offDetector=off)
    if method == "ossart":
        return sart(projs, angles, scanner_cfg, SART_NITER, blocksize=OSSART_BLOCKSIZE, use_offDetector=off)
    if method == "fista_tv":
        return fista_tv(projs, angles, scanner_cfg, use_offDetector=off)[0]
    raise ValueError(f"recon_volume: unknown method {method!r} (supported: {', '.join(METHODS)})")


def check_fdk_flags(args, fdk_selected: bool, not_fdk: str):
    """The refusals of the FDK flags (--short_scan, --half_fan, --fdk_filter) that the recon and initialize_pcd CLIs
    share; `not_fdk` is the CLI's message for a flag given without the fdk method, with `{flag}` standing for the flag."""
    for flag, on in (("--short_scan", args.short_scan), ("--half_fan", args.half_fan),
                     ("--fdk_filter", args.fdk_filter is not None)):
        if on and not fdk_selected:
            raise SystemExit(not_fdk.format(flag=flag))
    if args.half_fan and not args.use_offDetector:
        raise SystemExit("--half_fan needs --use_offDetector: the half-fan weights follow the detector offset")
    if args.half_fan and args.short_scan:
        raise SystemExit("--half_fan and --short_scan cannot be combined (half-fan weights need a full circle)")


def add_fdk_filter_flag(ap, help_text: str):
    """--fdk_filter NAME (one of fdk.FILTERS) on a CLI's parser."""
    from .fdk import FILTERS

    ap.add_argument("--fdk_filter", default=None, choices=FILTERS, metavar="NAME",
                    help=f"{help_text}: {', '.join(FILTERS)} (TIGRE's names; default: the scanner's filter, which must "
                         "then be null or ram_lak)")


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
    ap = argparse.ArgumentParser(description="Traditional CT reconstructions (FDK, SART, OS-SART, CGLS, FISTA-TV) of a scene")
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
    a = ap.parse_args(argv)
    methods = _parse_methods(a.methods)
    check_fdk_flags(a, "fdk" in methods, "{flag} applies to the fdk method, which --methods does not include (the "
                    "iterative methods need no redundancy weights)")
    if not torch.cuda.is_available():
        raise SystemExit("the reconstructions need a CUDA device: they run on the GPU and have no CPU fallback")
    import yaml

    from .dataset import read_scene
    from .metrics import metric_vol
    from .projector import project

    source = os.path.abspath(a.source_path)
    info = read_scene(source, eval=True)
    cfg = info.scanner_cfg
    projs_train = torch.from_numpy(np.stack([np.asarray(c.image, np.float32) for c in info.train_cameras])).cuda()
    train_angles = [c.angle for c in info.train_cameras]
    test_angles = [c.angle for c in info.test_cameras]
    vol_gt = np.asarray(info.vol, np.float32)
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
        fdk_filter = a.fdk_filter if method == "fdk" else None
        pred = recon_volume(projs_train, train_angles, cfg, method, short_scan=short_scan,
                            use_offDetector=a.use_offDetector, half_fan=half_fan, fdk_filter=fdk_filter)
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
        if fdk_filter not in (None, "ram_lak"):
            report["filter"] = fdk_filter
        if a.use_offDetector:
            report["use_offDetector"] = True
        with open(os.path.join(save, "eval_3d.yml"), "w") as f:
            yaml.dump(report, f, default_flow_style=False, sort_keys=False)
        if test_angles:
            render = project(pred, test_angles, cfg, use_offDetector=a.use_offDetector).cpu().numpy()
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
