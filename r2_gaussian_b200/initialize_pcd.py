"""Initial point cloud for a scene -- the reference's `initialize_pcd.py:26-172`.

    python -m r2_gaussian_b200.initialize_pcd --data <scene dir | NAF pickle> [--output init.npy]
        [--recon_method random|fdk|cgls|fista_tv|volume] [--recon recon.npy] [--n_points 50000] [--density_thresh 0.05]
        [--density_rescale 0.15] [--random_density_max 1.0] [--evaluate] [--short_scan] [--use_offDetector [--half_fan]]
        [--fdk_filter ram_lak|shepp_logan|cosine|hamming|hann]

`random` draws positions uniformly in the volume and densities in [0, random_density_max) with numpy's global
generator seeded with 0, exactly like the reference.  `fdk` reconstructs the volume from the train views with the
GPU FDK of `r2_gaussian_b200.fdk` (the reference calls TIGRE's `algs.fdk`), then samples `n_points` voxels above
`density_thresh` and scales their densities by `density_rescale`, the reference's way; it needs a CUDA device and at
least MIN_FDK_VIEWS train views.  `--short_scan` makes that FDK Parker-weighted (`fdk.fdk(short_scan=True)`), for a
scan over less than 360 degrees: the plain FDK shades such a volume, which moves the `density_thresh` cut across it;
the flag is refused with any other method.  `--use_offDetector` reconstructs through the scanner's offDetector
(fdk, cgls and fista_tv; without it the projector pair refuses a non-zero offset and fdk ignores it), and `--half_fan`
adds half-fan redundancy weights to that FDK for a full circle whose detector is shifted sideways (`fdk.fdk(...,
half_fan=True)`; fdk only, not with --short_scan).  `--fdk_filter NAME` gives that FDK one of TIGRE's windowed ramp
filters (`fdk.fdk(filter=NAME)`): the reference's FDK takes its window from the scanner's `filter`, this one only on
request, and without the flag a scanner whose `filter` names a window is refused (fdk only).  `cgls` does the same with 60 CGLS iterations over the GPU projector pair
(`r2_gaussian_b200.recon`, the reference's `algs.cgls`); it also needs a CUDA device.  `fista_tv` does the same with
the TV-regularised FISTA-TV of `r2_gaussian_b200.recon` at its default settings (CUDA as well).  `volume` samples a reconstruction made elsewhere (`--recon`, an .npy in the scene's
voxel grid) the same way.  Writes [n_points, 4] = (x, y, z, density) in the scene's normalised [-1,1]^3 coordinates to
`<scene>/init_<name>.npy` unless `--output` is given.  `--evaluate` builds the Gaussians from the written cloud, queries
them on the scene grid and prints their 3D PSNR against the ground-truth volume (`initialize_pcd.py:135-156`).

The default `--recon_method` is `random` (the reference defaults to `fdk`).
"""
from __future__ import annotations

import argparse
import os

import numpy as np

from .dataset import init_point_cloud, read_scene
from .recon import add_fdk_filter_flag, check_fdk_flags
from .trainer import default_init_path

# A filtered backprojection from a handful of views is dominated by streaks, and thresholding it gives no useful
# initialisation (the reference's sparse-view setups use 25 to 75 views).
MIN_FDK_VIEWS = 8


def _require_cuda_for(method: str):
    import torch

    if not torch.cuda.is_available():
        raise SystemExit(f"--recon_method {method} needs a CUDA device: the reconstruction runs on the GPU and has no "
                         "CPU fallback (use --recon_method random, or --recon_method volume --recon <vol.npy>)")


def recon_train_views(info, method: str, short_scan: bool = False, use_offDetector: bool = False,
                      half_fan: bool = False, fdk_filter: str | None = None) -> np.ndarray:
    """`recon.recon_volume(..., method, short_scan, use_offDetector, half_fan, fdk_filter)` of the train views of a
    `read_scene` result, as a host float32 [nx, ny, nz] array."""
    import torch

    from .recon import recon_volume

    projs = torch.from_numpy(np.stack([np.asarray(c.image, np.float32) for c in info.train_cameras])).cuda()
    vol = recon_volume(projs, [c.angle for c in info.train_cameras], info.scanner_cfg, method, short_scan=short_scan,
                       use_offDetector=use_offDetector, half_fan=half_fan, fdk_filter=fdk_filter)
    return vol.cpu().numpy()


def evaluate_init(data: str, init_path: str) -> float:
    """3D PSNR of the Gaussians created from `init_path` against the scene's ground-truth volume."""
    import torch

    from .dataset import Scene
    from .gaussian_model import GaussianModel
    from .metrics import metric_vol
    from .render_query import query
    from .trainer import ModelParams, PipelineParams

    model, pipe = ModelParams(), PipelineParams()
    with torch.no_grad():
        scene = Scene(data, eval=False, shuffle=False, device="cuda")
        cfg = scene.scanner_cfg
        scale_bound = None
        if model.scale_min and model.scale_max:
            scale_bound = np.array([model.scale_min, model.scale_max]) * max(cfg["sVoxel"])
        gaussians = GaussianModel(scale_bound)
        pts = np.load(init_path)
        gaussians.create_from_pcd(pts[:, :3], pts[:, 3:4], 1.0)
        vol_pred = query(gaussians, cfg["offOrigin"], cfg["nVoxel"], cfg["sVoxel"], pipe)["vol"]
        psnr_3d, _ = metric_vol(scene.vol_gt, vol_pred, "psnr")
    print(f"3D PSNR for initial Gaussians: {psnr_3d}")
    return float(psnr_3d)


def main(argv=None) -> str:
    ap = argparse.ArgumentParser(description="Generate initialization parameters")
    ap.add_argument("--data", required=True, help="Path to data.")
    ap.add_argument("--output", default=None, help="Path to output.")
    ap.add_argument("--recon_method", default="random", choices=["random", "volume", "fdk", "cgls", "fista_tv"])
    ap.add_argument("--recon", default=None, help="reconstruction volume (.npy) for --recon_method volume")
    ap.add_argument("--n_points", type=int, default=50000)
    ap.add_argument("--density_thresh", type=float, default=0.05)
    ap.add_argument("--density_rescale", type=float, default=0.15)
    ap.add_argument("--random_density_max", type=float, default=1.0)
    ap.add_argument("--evaluate", default=False, action="store_true",
                    help="Add this flag to evaluate quality (given GT volume, for debug only)")
    ap.add_argument("--short_scan", default=False, action="store_true",
                    help="with --recon_method fdk: Parker redundancy weights for a scan over less than 360 degrees")
    ap.add_argument("--use_offDetector", default=False, action="store_true",
                    help="with --recon_method fdk, cgls or fista_tv: reconstruct through the scanner's offDetector")
    ap.add_argument("--half_fan", default=False, action="store_true",
                    help="with --recon_method fdk and --use_offDetector: half-fan redundancy weights for a full circle "
                         "with the detector shifted sideways")
    add_fdk_filter_flag(ap, "with --recon_method fdk: the ramp filter")
    a = ap.parse_args(argv)
    check_fdk_flags(a, a.recon_method == "fdk", f"{{flag}} applies to --recon_method fdk only, not {a.recon_method}: "
                    "the iterative methods need no redundancy weights")
    if a.use_offDetector and a.recon_method not in ("fdk", "cgls", "fista_tv"):
        raise SystemExit(f"--use_offDetector applies to --recon_method fdk, cgls or fista_tv, not {a.recon_method}: "
                         "no projections are reconstructed")
    if a.recon_method in ("fdk", "cgls", "fista_tv"):
        _require_cuda_for(a.recon_method)
    np.random.seed(0)                                    # initialize_pcd.py:23
    info = read_scene(os.path.abspath(a.data), eval=False)
    recon = None
    if a.recon_method == "volume":
        if not a.recon:
            raise SystemExit("--recon_method volume needs --recon <vol.npy>")
        recon = np.load(a.recon)
    if a.recon_method == "fdk" and len(info.train_cameras) < MIN_FDK_VIEWS:
        raise SystemExit(f"--recon_method fdk needs at least {MIN_FDK_VIEWS} train views, the scene has "
                         f"{len(info.train_cameras)}: use --recon_method random")
    out = a.output or default_init_path(os.path.abspath(a.data))
    if os.path.exists(out):
        raise SystemExit(f"Initialization file {out} exists! Delete it first.")
    os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
    if a.recon_method in ("fdk", "cgls", "fista_tv"):
        # no draws from numpy's generator before np.random.choice
        recon = recon_train_views(info, a.recon_method, a.short_scan, a.use_offDetector, a.half_fan, a.fdk_filter)
    pts = init_point_cloud(info.scanner_cfg, a.n_points, recon=recon, density_thresh=a.density_thresh,
                           density_rescale=a.density_rescale, random_density_max=a.random_density_max)
    np.save(out, pts)
    print(f"Initialization saved in {out}.")
    if a.evaluate:
        evaluate_init(os.path.abspath(a.data), out)
    return out


if __name__ == "__main__":
    main()
