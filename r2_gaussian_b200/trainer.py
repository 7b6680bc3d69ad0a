"""Training / evaluation driver with the flow and defaults of the reference's `train.py:36-240` and
`arguments/__init__.py:21-71`, built from this repository's pieces: `dataset.Scene`, `GaussianModel`,
`render()` / `query()`, the fused loss kernels and `FusedAdam`.

    python -m r2_gaussian_b200.trainer -s <scene dir or NAF pickle> -m <output dir> [--iterations N] [...]

Same order of random draws as the reference (camera: `random.randint` on a stack refilled when empty,
`train.py:103-106`; TV crop centre: CPU `torch.rand(3)`, `train.py:130-132`), same densification schedule and
thresholds (expressed relative to the volume size), same checkpoint tuple and `point_cloud.pickle` export.  Not
carried over: TensorBoard / matplotlib logging (absent from this image).  GPU only.

Under `torchrun --nproc-per-node N` the same command trains Gaussian-sharded: every rank owns an index slice of the
cloud with its own Adam state and densification (budget `max_num_gaussians / N`), `render()` / `query()` sum the
partial images / volumes over the ranks (NCCL, or the peer-memory kernel with `--peer_exchange`), the host RNG
streams stay in lock-step (same seed, same draws), rank 0 writes one merged `point_cloud.pickle`.

`--pose_refine` (single GPU only) also learns one rigid correction per train view (`pose.PoseCorrection`, row =
`cam.uid`, train view 0 held at zero) with its own FusedAdam (`PoseParams` learning rates, log-linear over
`--iterations`), on both training paths; the poses step wherever the Gaussians would and at densification iterations.
Train views are then evaluated with their corrected cameras, each save writes `train_poses.npz` and checkpoints carry
the poses.  Without the switch nothing changes: same launches, settings files, checkpoints and printed keys.

`--batch_size B` (default 1, at most the number of train views) takes B train views per optimizer step, rendered in one
batched call (`fused.rasterize_views_raw`; `NativeTrainStep` with a list of cameras).  The views are popped from the
camera stack with the draws B single-view iterations would make, so a run sees the B = 1 sequence of views grouped by
B.  The objective is the SUM of the B views' image losses plus B lambda_tv TV of one crop (B times the batch mean; Adam
is invariant to that scale up to its eps of 1e-15); the densification statistics count every view; the logged loss is
the batch mean plus lambda_tv TV.  Iteration counts and the learning-rate and densification schedules stay in optimizer
steps, so a run sees B times as many views.  B > 1 is refused with --pose_refine, Gaussian sharding and
compute_cov3D_python.  With B = 1 nothing changes.

`--detector_offset_refine` also learns the scan's horizontal detector offset (`detector.DetectorOffset`, one value in
pixels; `DetectorParams` learning rates, log-linear over `--iterations`) with its own FusedAdam, on both training paths
and at any --batch_size; it steps wherever the poses would.  Train and test views are evaluated with the offset (it is a
property of the scanner), each save writes `detector_offset.yml` and checkpoints carry the offset and its Adam state.
It is refused with --pose_refine and with Gaussian sharding.  Without the switch nothing changes.

`--use_offDetector` trains through the scanner's offDetector: every train and test camera carries it in its
projection_matrix (`dataset.Scene(use_offDetector=True)`, `scene.detector_shift`), so pose corrections, batched views
and the native step see it too.  With `--detector_offset_refine` the learned offset acts on top of the file's, and
`detector_offset.yml` also reports the total `offDetector_u` = offDetector[0] - offset_px * dDetector_u in the scanner
file's units.  The rasterizer clamps each Gaussian's EWA Jacobian at 1.3 tan_fov about the axis, as the reference does,
so with an offset of more than 0.15 W a Gaussian whose centre projects beyond that clamp gets a clamped footprint.
Without the switch the offset is ignored (the reference's render() has none) and nothing changes.

`--estimate_offDetector` measures the horizontal detector offset from the train views before training
(`detector.estimate_offset`, relative to the file's offset under `--use_offDetector`, else to a centred detector) and
trains as `--use_offDetector` would on a copy of the scanner whose offDetector[0] is the estimated total
(`dataset.Scene(offDetector_u=...)`).  With `--detector_offset_refine` the learned offset acts on top of the estimate.
Each save then writes `detector_offset.yml` with `estimate_px` / `estimate_scene` next to the learned offset (if any)
and the total `offDetector_u`; the printed result adds `detector_estimate_px`.

`--use_view_geometry` trains through each view's own DSO, DSD, offOrigin and offDetector, read from the projection
frames (`dataset.Scene(use_view_geometry=True)`, `scene.view_scanner`): a helical scan or a calibrated bench.  It implies
`--use_offDetector` and is recorded in `cfg_args`.  `--pose_refine` and `--detector_offset_refine` act on top of it.
It is refused with `--estimate_offDetector` (the estimate assumes one fixed circle), with Gaussian sharding, and with
`--batch_size` > 1 when the train views' DSD differ (a batch shares one field of view).
"""
from __future__ import annotations

import argparse
import json
import os
import random
import time
from dataclasses import asdict, dataclass

import numpy as np
import torch

from . import losses
from ._C import CapacityOverflow
from .dataset import Scene, train_view_count
from .gaussian_model import GaussianModel
from .gaussian_utils import get_expon_lr_func
from .metrics import metric_proj, metric_vol
from .optim import FusedAdam
from .detector import SIGN_CONVENTION, DetectorOffset
from .pose import PoseCorrection
from .rasterization import GaussianRasterizationSettings
from .render_query import _tan_fov, query, render
from . import fused, sharded, train_step
from .sharded import gather_point_cloud, shard_init_points, world_info


@dataclass
class ModelParams:
    source_path: str = ""
    model_path: str = ""
    data_device: str = "cuda"
    ply_path: str = ""           # initial cloud (.npy [N,4]); default: <source>/init_<name>.npy
    scale_min: float = 0.0005    # fraction of the volume size
    scale_max: float = 0.5
    eval: bool = True


@dataclass
class PipelineParams:
    compute_cov3D_python: bool = False
    debug: bool = False


@dataclass
class OptimizationParams:
    iterations: int = 30_000
    position_lr_init: float = 0.0002
    position_lr_final: float = 0.00002
    position_lr_max_steps: int = 30_000
    density_lr_init: float = 0.01
    density_lr_final: float = 0.001
    density_lr_max_steps: int = 30_000
    scaling_lr_init: float = 0.005
    scaling_lr_final: float = 0.0005
    scaling_lr_max_steps: int = 30_000
    rotation_lr_init: float = 0.001
    rotation_lr_final: float = 0.0001
    rotation_lr_max_steps: int = 30_000
    lambda_dssim: float = 0.25
    lambda_tv: float = 0.05
    tv_vol_size: int = 32
    density_min_threshold: float = 0.00001
    densification_interval: int = 100
    densify_from_iter: int = 500
    densify_until_iter: int = 15000
    densify_grad_threshold: float = 5.0e-5
    densify_scale_threshold: float | None = 0.1     # fraction of the volume size
    max_screen_size: float | None = None
    max_scale: float | None = None                  # fraction of the volume size
    max_num_gaussians: int | None = 500_000


@dataclass
class PoseParams:
    """`--pose_refine`: learn one rigid correction per train view together with the scene (`pose.PoseCorrection`; train
    view 0 anchors the frame).  Learning rates decay log-linearly from init to final over `--iterations`.  The defaults
    are a starting point (rotation in rad, translation in scene units), not tuned on real scans."""
    pose_refine: bool = False
    pose_rotation_lr_init: float = 1e-3
    pose_rotation_lr_final: float = 1e-5
    pose_translation_lr_init: float = 5e-3
    pose_translation_lr_final: float = 5e-5


POSE_ANCHOR = 0     # the train view whose correction stays exactly zero


@dataclass
class DetectorParams:
    """`--detector_offset_refine`: learn the horizontal detector offset (pixels, `detector.DetectorOffset`) together
    with the scene.  The learning rate decays log-linearly from init to final over `--iterations`; the defaults were
    chosen on a 48^3 generate_data scene (24 views of 96^2, cone beam) shifted by 3 columns, among 1e-1, 5e-2 and 2e-2
    (final = init / 100; DESIGN section 8)."""
    detector_offset_refine: bool = False
    detector_offset_lr_init: float = 2e-2
    detector_offset_lr_final: float = 2e-4


def detector_refusal(detector_offset_refine: bool, pose_refine: bool, world: int) -> str | None:
    """Why `--detector_offset_refine` cannot be used with these settings (None: it can).  Checked before any CUDA
    work."""
    if not detector_offset_refine:
        return None
    if pose_refine:
        return "--detector_offset_refine is not supported with --pose_refine (composing the two maps is not implemented)"
    if world > 1:
        return ("--detector_offset_refine is not supported with Gaussian sharding (WORLD_SIZE > 1): every rank would "
                "see only its shard's part of the offset gradient")
    return None


def default_init_path(source_path: str) -> str:
    """`<scene>/init_<scene>.npy` for directories, `<dir>/init_<stem>.npy` for NAF pickles (`initialize.py:29-41`)."""
    if os.path.exists(os.path.join(source_path, "meta_data.json")):
        return os.path.join(source_path, "init_" + os.path.basename(source_path.rstrip("/")) + ".npy")
    if source_path.split(".")[-1] in ("pickle", "pkl"):
        return os.path.join(os.path.dirname(source_path), "init_" + os.path.basename(source_path).split(".")[0] + ".npy")
    raise ValueError("Could not recognize scene type!")


def derived_settings(scanner_cfg: dict, model: ModelParams, opt: OptimizationParams) -> dict:
    """Volume-relative thresholds in world units (`train.py:50-62`, `:87-90`)."""
    to_world = max(scanner_cfg["sVoxel"])
    scale_bound = None
    if model.scale_min > 0 and model.scale_max > 0:
        scale_bound = np.array([model.scale_min, model.scale_max]) * to_world
    n = int(opt.tv_vol_size)
    return {"volume_to_world": to_world,
            "max_scale": opt.max_scale * to_world if opt.max_scale else None,
            "densify_scale_threshold": opt.densify_scale_threshold * to_world if opt.densify_scale_threshold else None,
            "scale_bound": scale_bound,
            "tv_vol_nVoxel": [n, n, n],
            "tv_vol_sVoxel": [float(d) * n for d in scanner_cfg["dVoxel"]]}


def evaluation_cameras(scene: Scene, pose=None, detector=None) -> list:
    """[("train", cams), ("test", cams)]: the cameras `evaluate` renders.  `pose` (a PoseCorrection over the train
    views, row = cam.uid): train views carry their corrections, test views keep their nominal poses.  `detector` (a
    DetectorOffset): both splits carry the offset."""
    out = []
    for name, cams in (("train", scene.getTrainCameras()), ("test", scene.getTestCameras())):
        if cams and name == "train" and pose is not None:
            cams = [pose.device_camera(c, c.uid, POSE_ANCHOR) for c in cams]
        if cams and detector is not None:
            cams = detector.cameras(cams)
        out.append((name, cams))
    return out


@torch.no_grad()
def evaluate(scene: Scene, gaussians: GaussianModel, pipe, with_ssim: bool = True, pose=None, detector=None) -> dict:
    """3-D PSNR / SSIM of the queried volume and 2-D PSNR / SSIM of the rendered train and test views, with the
    reference's metric definitions (`train.py:262-330`, `utils/image_utils.py:90-183`).  `pose` (a PoseCorrection over
    the train views): train views are rendered with their corrected cameras; test views keep their nominal poses.
    `detector` (a DetectorOffset): train and test views are rendered with the offset applied."""
    cfg = scene.scanner_cfg
    vol = query(gaussians, cfg["offOrigin"], cfg["nVoxel"], cfg["sVoxel"], pipe)["vol"]
    out = {"psnr_3d": metric_vol(scene.vol_gt, vol, "psnr")[0]}
    if with_ssim:
        out["ssim_3d"] = metric_vol(scene.vol_gt, vol, "ssim")[0]
    for name, cams in evaluation_cameras(scene, pose, detector):
        if not cams:
            continue
        imgs = torch.concat([render(c, gaussians, pipe)["render"] for c in cams], 0).permute(1, 2, 0)
        gts = torch.concat([c.original_image.to(imgs.device) for c in cams], 0).permute(1, 2, 0)
        out[f"psnr_2d_{name}"] = metric_proj(gts, imgs, "psnr")[0]
        if with_ssim:
            out[f"ssim_2d_{name}"] = metric_proj(gts, imgs, "ssim")[0]
    return out


def view_geometry_refusal(use_view_geometry: bool, estimate_offDetector: bool, world: int, batch_size: int,
                          source_path: str) -> str | None:
    """Why `--use_view_geometry` cannot be used with these settings (None: it can).  Checked before any CUDA work."""
    if not use_view_geometry:
        return None
    if estimate_offDetector:
        return ("--estimate_offDetector cannot be combined with --use_view_geometry: the conjugate-ray estimate assumes "
                "one fixed circle")
    if world > 1:
        return "--use_view_geometry is not supported with Gaussian sharding (WORLD_SIZE > 1): train on one GPU"
    if batch_size > 1:
        from .dataset import train_view_dsd
        dsd = train_view_dsd(source_path)
        if len(set(dsd)) > 1:
            return (f"--batch_size {batch_size} needs one field of view for every train view, but under "
                    f"--use_view_geometry their DSD varies ({min(dsd):g} to {max(dsd):g}): use --batch_size 1")
    return None


def batch_refusal(batch_size: int, pose_refine: bool, world: int, compute_cov3D_python: bool) -> str | None:
    """Why `--batch_size` cannot be used with these settings (None: it can).  Checked before any CUDA work."""
    if batch_size < 1:
        return f"--batch_size must be at least 1, got {batch_size}"
    if batch_size == 1:
        return None
    if pose_refine:
        return "--batch_size > 1 is not supported with --pose_refine (the batched rasterizer returns no matrix gradients)"
    if world > 1:
        return "--batch_size > 1 is not supported with Gaussian sharding (WORLD_SIZE > 1)"
    if compute_cov3D_python:
        return "--batch_size > 1 is not supported with compute_cov3D_python (the batched path folds the activations)"
    return None


def draw_train_views(stack, cameras, B: int):
    """Pop B train views off the camera stack -> (views, stack): the draws of B single-view iterations, each a
    `random.randint` on the stack, which is refilled from `cameras` when empty (`train.py:103-106`)."""
    views = []
    for _ in range(B):
        if not stack:
            stack = cameras.copy()
        views.append(stack.pop(random.randint(0, len(stack) - 1)))
    return views, stack


def render_batch(cams, gaussians: GaussianModel) -> dict:
    """The training render of B views of `gaussians` in one call on its raw parameters (`fused.rasterize_views_raw`) ->
    {"render": [B,H,W], "viewspace_points": [B,P,3] (its .grad receives the per-view dL/dmean2D), "radii": [B,P]}.
    Image v is bit for bit the single-view raw render of cams[v]."""
    c0 = cams[0]
    tanfovx, tanfovy = _tan_fov(c0)
    views = torch.stack([c.world_view_transform for c in cams])
    projs = torch.stack([c.full_proj_transform for c in cams])
    xyz = gaussians.get_xyz
    means2D = torch.zeros((len(cams),) + tuple(xyz.shape), dtype=xyz.dtype, device=xyz.device, requires_grad=True) + 0
    means2D.retain_grad()
    settings = GaussianRasterizationSettings(
        image_height=int(c0.image_height), image_width=int(c0.image_width), tanfovx=tanfovx, tanfovy=tanfovy,
        scale_modifier=1.0, viewmatrix=views[0], projmatrix=projs[0], campos=c0.camera_center, prefiltered=False,
        mode=int(c0.mode), debug=False)
    images, radii = fused.rasterize_views_raw(xyz, means2D, gaussians.raw_parameters(), views, projs, settings)
    return {"render": images, "viewspace_points": means2D, "radii": radii}


def training(model: ModelParams, opt: OptimizationParams, pipe: PipelineParams, testing_iterations=(),
             saving_iterations=(), checkpoint_iterations=(), checkpoint: str | None = None, init_points=None,
             log=print, pose_params: PoseParams | None = None, batch_size: int = 1,
             detector_params: DetectorParams | None = None, use_offDetector: bool = False,
             estimate_offDetector: bool = False, use_view_geometry: bool = False) -> dict:
    first_iter = 0
    why = view_geometry_refusal(use_view_geometry, estimate_offDetector, world_info()[1], int(batch_size),
                                model.source_path)
    if why is not None:
        raise ValueError(why)
    refine = pose_params is not None and pose_params.pose_refine
    if refine and world_info()[1] > 1:
        raise RuntimeError("--pose_refine is not supported with Gaussian sharding (WORLD_SIZE > 1): every rank would "
                           "hold only its shard's part of the camera-matrix gradients")
    refine_det = detector_params is not None and detector_params.detector_offset_refine
    why = detector_refusal(refine_det, refine, world_info()[1])
    if why is not None:
        raise ValueError(why)
    B = int(batch_size)
    why = batch_refusal(B, refine, world_info()[1], bool(getattr(pipe, "compute_cov3D_python", False)))
    if why is not None:
        raise ValueError(why)
    estimate = off_u = None
    if estimate_offDetector:
        # the offset measured from the train views, on top of the file's under use_offDetector, becomes the scene's
        from .dataset import read_scene
        from .estimate_offset import estimate_scene
        info = read_scene(model.source_path, eval=False)
        estimate = estimate_scene(info, use_offDetector)
        off_u, use_offDetector = estimate["offDetector_u"], True
        log(f"estimated detector offset: {estimate['offset_px']:+.4f} px, offDetector_u = "
            f"{off_u / info.scene_scale:.6g} ({estimate['n_pairs']} conjugate pairs)")
    scene = Scene(model.source_path, model.model_path, eval=model.eval, shuffle=False, device="cuda",
                  data_device=model.data_device, use_offDetector=use_offDetector, offDetector_u=off_u,
                  use_view_geometry=use_view_geometry)
    scene.offset_estimate = estimate
    cfg = scene.scanner_cfg
    if B > len(scene.getTrainCameras()):
        raise ValueError(f"--batch_size {B} exceeds the scene's {len(scene.getTrainCameras())} train views")
    bbox_cpu = scene.bbox.float()
    bbox = bbox_cpu.cuda()
    ds = derived_settings(cfg, model, opt)
    queryfunc = lambda g: query(g, cfg["offOrigin"], cfg["nVoxel"], cfg["sVoxel"], pipe)

    gaussians = GaussianModel(ds["scale_bound"])
    if init_points is None:
        path = model.ply_path or default_init_path(model.source_path)
        assert os.path.exists(path), f"Cannot find {path} for initialization."
        init_points = np.load(path)
    rank, world = world_info()
    dist2 = None
    if world > 1:
        sharded.enable()
        # Gaussian-sharded run (one process per GPU, torchrun): every rank owns an index slice of the cloud, its
        # Adam state and its densification; render() / query() sum the partial images / volumes over the ranks, so
        # loss and gradients are what a single GPU would compute.  3-NN distances come from the FULL cloud.
        from .simple_knn import distCUDA2
        full = torch.as_tensor(np.asarray(init_points[:, :3])).float().cuda()
        init_points, dist2 = shard_init_points(init_points, distCUDA2(full).cpu().numpy(), rank, world)
        if opt.max_num_gaussians:
            opt.max_num_gaussians = max(1, opt.max_num_gaussians // world)
    gaussians.create_from_pcd(init_points[:, :3], init_points[:, 3:4], 1.0, dist2=dist2)
    scene.gaussians = gaussians
    gaussians.training_setup(opt)
    corr = pose_opt = pose_lr = None
    if refine:
        # one correction per train camera, row = cam.uid (its position in getTrainCameras())
        corr = PoseCorrection(len(scene.getTrainCameras()), device="cuda")
        pose_opt = FusedAdam([{"params": [corr.omega], "lr": 0.0, "name": "omega"},
                              {"params": [corr.nu], "lr": 0.0, "name": "nu"}], lr=0.0, eps=1e-15)
        pose_lr = (get_expon_lr_func(pose_params.pose_rotation_lr_init, pose_params.pose_rotation_lr_final,
                                     max_steps=opt.iterations),
                   get_expon_lr_func(pose_params.pose_translation_lr_init, pose_params.pose_translation_lr_final,
                                     max_steps=opt.iterations))
    det = det_opt = det_lr = None
    if refine_det:
        det = DetectorOffset("cuda")
        det_opt = FusedAdam([{"params": [det.offset], "lr": 0.0, "name": "detector_offset"}], lr=0.0, eps=1e-15)
        det_lr = get_expon_lr_func(detector_params.detector_offset_lr_init, detector_params.detector_offset_lr_final,
                                   max_steps=opt.iterations)
    if checkpoint is not None:
        path = rank_checkpoint_path(checkpoint, rank, world)
        payload = torch.load(path, weights_only=False)
        model_state, first_iter = payload[0], payload[1]
        tag = payload[2] if len(payload) > 2 else {"rank": 0, "world": 1}
        if (tag["rank"], tag["world"]) != (rank, world):
            raise RuntimeError(f"checkpoint {path} was written by rank {tag['rank']} of {tag['world']}; this process is "
                               f"rank {rank} of {world} (a Gaussian-sharded run resumes with the same number of ranks)")
        pose_state = payload[3] if len(payload) > 3 else None
        if refine != (pose_state is not None):
            raise RuntimeError(f"checkpoint {path} was written {'with' if pose_state is not None else 'without'} "
                               f"--pose_refine; resume it with the same setting")
        gaussians.restore(model_state, opt)
        if refine:
            if tuple(pose_state["omega"].shape) != tuple(corr.omega.shape):
                raise RuntimeError(f"checkpoint {path} holds poses of {pose_state['omega'].shape[0]} train views, the "
                                   f"scene has {corr.omega.shape[0]}")
            with torch.no_grad():
                corr.omega.copy_(pose_state["omega"])
                corr.nu.copy_(pose_state["nu"])
            pose_opt.load_state_dict(pose_state["optimizer"])
        det_state = payload[4] if len(payload) > 4 else None
        if refine_det != (det_state is not None):
            raise RuntimeError(f"checkpoint {path} was written {'with' if det_state is not None else 'without'} "
                               f"--detector_offset_refine; resume it with the same setting")
        if refine_det:
            with torch.no_grad():
                det.offset.copy_(det_state["offset"])
            det_opt.load_state_dict(det_state["optimizer"])
        log(f"Load checkpoint {os.path.basename(path)}.")

    use_tv = opt.lambda_tv > 0
    tv_n = ds["tv_vol_nVoxel"]
    tv_s = torch.tensor(ds["tv_vol_sVoxel"])
    ckpt_dir = os.path.join(scene.model_path, "ckpt")
    if scene.model_path:
        os.makedirs(ckpt_dir, exist_ok=True)
    history = {"eval": {}, "loss": []}
    stack = None
    native = None
    if train_step.enabled() and not getattr(pipe, "debug", False) and not getattr(pipe, "compute_cov3D_python", False):
        native = train_step.NativeTrainStep(gaussians, opt.lambda_dssim, opt.lambda_tv if use_tv else 0.0, tv_n,
                                            [float(v) for v in tv_s],
                                            **({} if corr is None else dict(pose=(corr, pose_opt), pose_anchor=POSE_ANCHOR)),
                                            **({} if det is None else dict(detector=(det, det_opt))))
    if world > 1:
        # one exchange of each shape before the clock starts: the NCCL communicator / the peer-memory reducers are
        # created on first use (seconds at 8 ranks), which is set-up, not a training step
        cam0 = scene.getTrainCameras()[0]
        sharded.sharded_sum_(torch.zeros(int(cam0.image_height) * int(cam0.image_width) + 4, device="cuda"))
        sharded.sharded_sum_(torch.zeros((int(cam0.image_height), int(cam0.image_width)), device="cuda").unsqueeze(0))
        if use_tv:
            nvox = int(tv_n[0]) * int(tv_n[1]) * int(tv_n[2])
            sharded.sharded_sum_(torch.zeros(nvox + 4, device="cuda"))
            sharded.sharded_sum_(torch.zeros(tuple(int(v) for v in tv_n), device="cuda"))
        torch.cuda.synchronize()
        torch.distributed.barrier()
    torch.cuda.synchronize()
    t_start = time.perf_counter()
    t_aside = 0.0     # seconds spent saving / checkpointing / evaluating (reported apart from the training steps)
    t_mark = None     # (time, aside so far, iteration) after the first iterations: allocator / capacity hints warmed up

    class _aside:     # times a block that is not a training step; synchronises on both sides so it owns its GPU time
        def __enter__(self):
            torch.cuda.synchronize()
            self.t0 = time.perf_counter()

        def __exit__(self, *exc):
            nonlocal t_aside
            torch.cuda.synchronize()
            t_aside += time.perf_counter() - self.t0
            return False

    for iteration in range(first_iter + 1, opt.iterations + 1):
        if t_mark is None and iteration - first_iter == 51:
            torch.cuda.synchronize()
            t_mark = (time.perf_counter(), t_aside, iteration - 1)
        gaussians.update_learning_rate(iteration)
        if corr is not None:
            for group, schedule in zip(pose_opt.param_groups, pose_lr):
                group["lr"] = schedule(iteration)
        if det is not None:
            det_opt.param_groups[0]["lr"] = det_lr(iteration)
        cams, stack = draw_train_views(stack, scene.getTrainCameras(), B)
        cam = cams[0]

        densify_due = iteration < opt.densify_until_iter and iteration > opt.densify_from_iter \
            and iteration % opt.densification_interval == 0
        centre = None
        if use_tv:
            centre = (bbox_cpu[0] + tv_s / 2) + (bbox_cpu[1] - tv_s - bbox_cpu[0]) * torch.rand(3)
        logged = None
        if B > 1 and native is not None and gaussians.get_xyz.shape[0] > 0:
            # B views in one fixed launch sequence; at a densification iteration no Adam step, as below
            native(cams, torch.stack([c.original_image for c in cams]).cuda(), centre,
                   apply_update=(iteration < opt.iterations) and not densify_due,
                   **({} if det is None else dict(detector_update=iteration < opt.iterations)))
            total = None
            with torch.no_grad():
                if densify_due:
                    native.flush()
                    gaussians.densify_and_prune(opt.densify_grad_threshold, opt.density_min_threshold, opt.max_screen_size,
                                                ds["max_scale"], opt.max_num_gaussians, ds["densify_scale_threshold"], bbox)
        elif B > 1:
            gts = [c.original_image.cuda() for c in cams]

            def batch_objective():
                """sum over the views of the image loss + B lambda_tv TV, and the logged batch mean + lambda_tv TV"""
                pkg = render_batch(cams if det is None else det.cameras(cams), gaussians)
                image_sum = sum(losses.image_loss(pkg["render"][v], gts[v], lambda_dssim=opt.lambda_dssim)["total"]
                                for v in range(B))
                total, shown = image_sum, image_sum.detach() / B
                if use_tv:
                    tv = losses.tv_3d_loss(query(gaussians, centre, tv_n, tv_s, pipe)["vol"], reduction="mean")
                    total = total + (B * opt.lambda_tv) * tv
                    shown = shown + opt.lambda_tv * tv.detach()
                return pkg, total, shown

            pkg, total, logged = batch_objective()
            try:
                total.backward()
            except CapacityOverflow:      # as below: the same views again with the raised capacity hint
                gaussians.optimizer.zero_grad(set_to_none=True)
                pkg, total, logged = batch_objective()
                total.backward()
            with torch.no_grad():
                grads = pkg["viewspace_points"].grad
                if det is not None:
                    det.grad_from(grads, int(cam.image_width))
                for v in range(B):        # the statistics of each view, in view order
                    seen = pkg["radii"][v] > 0
                    gaussians.update_max_radii(pkg["radii"][v], seen)
                    gaussians.add_densification_stats(_ViewGrad(grads[v]), seen)
                if densify_due:
                    gaussians.densify_and_prune(opt.densify_grad_threshold, opt.density_min_threshold, opt.max_screen_size,
                                                ds["max_scale"], opt.max_num_gaussians, ds["densify_scale_threshold"], bbox)
        elif native is not None and (gaussians.get_xyz.shape[0] > 0 or world > 1):
            # fixed launch sequence, no autograd (train_step.py).  At a densification iteration the reference's
            # optimizer.step() comes AFTER the tensors were replaced and therefore applies nothing (their .grad is None,
            # train.py:158-176): the same here.
            # The pose gradient is valid at a densification iteration too, so the poses step there (both paths).
            gt = cam.original_image.cuda()
            pose_kw = {} if corr is None else dict(view=cam.uid, pose_update=iteration < opt.iterations)
            if det is not None:
                pose_kw = dict(detector_update=iteration < opt.iterations)
            native(cam, gt, centre, apply_update=(iteration < opt.iterations) and not densify_due, **pose_kw)
            total = None
            with torch.no_grad():
                if densify_due:
                    native.flush()
                    gaussians.densify_and_prune(opt.densify_grad_threshold, opt.density_min_threshold, opt.max_screen_size,
                                                ds["max_scale"], opt.max_num_gaussians, ds["densify_scale_threshold"], bbox)
        else:
            view_cam = (lambda: cam) if corr is None else (lambda: corr.device_camera(cam, cam.uid, POSE_ANCHOR))
            if det is not None:
                view_cam = lambda: det.camera(cam)
            pkg = render(view_cam(), gaussians, pipe)
            gt = cam.original_image.cuda()
            loss = losses.image_loss(pkg["render"], gt, lambda_dssim=opt.lambda_dssim)
            total = loss["total"]
            if use_tv:
                vol = query(gaussians, centre, tv_n, tv_s, pipe)["vol"]
                total = total + opt.lambda_tv * losses.tv_3d_loss(vol, reduction="mean")
            try:
                total.backward()
            except CapacityOverflow:
                # a speculative forward (no host sync) ran out of instance capacity: its image was all zeros and this
                # step's gradients are void.  The capacity hint has been raised; redo the step with the same camera.
                gaussians.optimizer.zero_grad(set_to_none=True)
                if pose_opt is not None:
                    pose_opt.zero_grad(set_to_none=True)
                pkg = render(view_cam(), gaussians, pipe)
                total = losses.image_loss(pkg["render"], gt, lambda_dssim=opt.lambda_dssim)["total"]
                if use_tv:
                    total = total + opt.lambda_tv * losses.tv_3d_loss(query(gaussians, centre, tv_n, tv_s, pipe)["vol"],
                                                                      reduction="mean")
                total.backward()
            with torch.no_grad():
                if det is not None:
                    det.grad_from(pkg["viewspace_points"].grad, int(cam.image_width))
                gaussians.update_max_radii(pkg["radii"], pkg["visibility_filter"])
                gaussians.add_densification_stats(pkg["viewspace_points"], pkg["visibility_filter"])
                if densify_due:
                    gaussians.densify_and_prune(opt.densify_grad_threshold, opt.density_min_threshold, opt.max_screen_size,
                                                ds["max_scale"], opt.max_num_gaussians, ds["densify_scale_threshold"], bbox)

        with torch.no_grad():
            # sharded: an EMPTY SHARD is fine and keeps going through the P == 0 path; the run stops -- on every rank at
            # once, so nobody is left waiting in a collective -- only when the whole cloud is gone (the count can only
            # change at a densification step, which is where the all-reduce is paid)
            if (world == 1 and gaussians.get_density.shape[0] == 0) or \
                    (world > 1 and iteration % opt.densification_interval == 0 and total_gaussians(gaussians, world) == 0):
                raise ValueError("No Gaussian left. Change adaptive control hyperparameters!")
            if total is not None and iteration < opt.iterations:
                gaussians.optimizer.step()
                gaussians.optimizer.zero_grad(set_to_none=True)
                if pose_opt is not None:
                    pose_opt.step()
                    pose_opt.zero_grad(set_to_none=True)
                if det_opt is not None:
                    det_opt.step()
                    det_opt.zero_grad(set_to_none=True)
            if native is not None and (iteration in saving_iterations or iteration in checkpoint_iterations or
                                       iteration in testing_iterations or iteration == opt.iterations):
                native.flush()       # the last enqueued iteration is checked (and repeated if it had overflowed)
            if scene.model_path and (iteration in saving_iterations or iteration == opt.iterations):
                log(f"[ITER {iteration}] Saving Gaussians")
                with _aside():
                    if world == 1:
                        scene.save(iteration, queryfunc)
                        if corr is not None:
                            save_train_poses(scene, corr, iteration)
                        if det is not None or estimate is not None:
                            save_detector_offset(scene, det, iteration)
                    else:
                        save_sharded(scene, gaussians, iteration, queryfunc, rank)
            if scene.model_path and iteration in checkpoint_iterations:
                log(f"[ITER {iteration}] Saving Checkpoint")
                with _aside():
                    name = os.path.basename(rank_checkpoint_path(f"chkpnt{iteration}.pth", rank, world))
                    payload = (gaussians.capture(), iteration) if world == 1 else \
                        (gaussians.capture(), iteration, {"rank": rank, "world": world})
                    if corr is not None:    # (model, iteration, tag, poses): written only with --pose_refine
                        payload = (payload[0], iteration, {"rank": rank, "world": world},
                                   {"omega": corr.omega.detach().cpu(), "nu": corr.nu.detach().cpu(),
                                    "optimizer": pose_opt.state_dict()})
                    if det is not None:     # (model, iteration, tag, poses or None, offset): only with the switch
                        payload = (payload[0], iteration, {"rank": rank, "world": world},
                                   payload[3] if len(payload) > 3 else None,
                                   {"offset": det.offset.detach().cpu(), "optimizer": det_opt.state_dict()})
                    torch.save(payload, os.path.join(ckpt_dir, name))
                    if world > 1:
                        torch.distributed.barrier()  # no rank runs ahead into the next exchange while others write
            if iteration % 100 == 0:
                shown = logged if logged is not None else total
                history["loss"].append((iteration, float(shown) if shown is not None else native.total_loss()))
                if world > 1:
                    sharded.check_peer_exchange()    # the loss read-out above synchronised anyway
            if iteration in testing_iterations:
                with _aside():
                    history["eval"][iteration] = evaluate(scene, gaussians, pipe, pose=corr, detector=det)
                log(f"[ITER {iteration}] {history['eval'][iteration]}  points {gaussians.get_xyz.shape[0]}")
                if world > 1:
                    sharded.check_peer_exchange()
                if scene.model_path and rank == 0:
                    write_eval_yaml(scene.model_path, iteration, history["eval"][iteration])
    if native is not None:
        native.flush()
        history["repeated_iterations"] = native.repeats
    torch.cuda.synchronize()
    history["seconds"] = time.perf_counter() - t_start
    history["train_seconds"] = history["seconds"] - t_aside   # the training steps alone
    if t_mark is not None and opt.iterations > t_mark[2]:
        history["steady_ms_per_iteration"] = ((time.perf_counter() - t_mark[0]) - (t_aside - t_mark[1])) / \
            (opt.iterations - t_mark[2]) * 1e3                # after the first 50 iterations (warm allocator / hints)
    history["iterations"] = opt.iterations - first_iter
    history["gaussians"] = int(gaussians.get_xyz.shape[0])
    history["scene"], history["model"] = scene, gaussians
    if corr is not None:
        history["pose"] = corr
    if det is not None:
        history["detector"] = det
        history["detector_offset_px"] = float(det.offset.detach()[0])
    if estimate is not None:
        history["detector_estimate_px"] = estimate["offset_px"]
    return history


@torch.no_grad()
def save_train_poses(scene: Scene, corr, iteration: int):
    """`point_cloud/iteration_<N>/train_poses.npz`: omega / nu [n,3], the corrected world_view_transform [n,4,4] of every
    train view (row = cam.uid, stored transposed like the camera's) and the nominal angles [n] of the dataset."""
    cams = scene.getTrainCameras()
    wvt = torch.stack([corr.device_camera(c, c.uid, POSE_ANCHOR).world_view_transform for c in cams])
    np.savez(os.path.join(scene.model_path, f"point_cloud/iteration_{iteration}", "train_poses.npz"),
             omega=corr.omega.detach().cpu().numpy(), nu=corr.nu.detach().cpu().numpy(),
             world_view_transform=wvt.cpu().numpy(), angle=np.array([float(c.angle) for c in cams]))


@torch.no_grad()
def save_detector_offset(scene: Scene, det, iteration: int):
    """`point_cloud/iteration_<N>/detector_offset.yml`: the learned offset (`det`, or None) in pixels and in scene units
    at the detector, and the sign convention in words; under `--estimate_offDetector` also the estimate
    (`estimate_px`, `estimate_scene`, relative to the file's offset or a centred detector)."""
    import yaml
    doc = {}
    if det is not None:
        doc = {"offset_px": float(det.offset.detach()[0]), "offset_scene": det.scene_units(scene.scanner_cfg)}
    doc["sign_convention"] = SIGN_CONVENTION
    est = getattr(scene, "offset_estimate", None)
    if est is not None:
        doc["estimate_px"], doc["estimate_scene"] = est["offset_px"], est["offset_scene"]
    if getattr(scene, "use_offDetector", False):
        # the learned offset acts on top of the scanner file's (or the estimate's): the total, in the file's units
        cfg = scene.scanner_cfg
        learned = det.scene_units(cfg) if det is not None else 0.0
        doc["offDetector_u"] = (float(cfg.get("offDetector", [0.0, 0.0])[0]) - learned) / scene.scene_scale
    with open(os.path.join(scene.model_path, f"point_cloud/iteration_{iteration}", "detector_offset.yml"), "w") as f:
        yaml.dump(doc, f, default_flow_style=False, sort_keys=False)


class _ViewGrad:
    """One view's rows of a batched render's screen-space gradients, in the shape `add_densification_stats` reads."""

    def __init__(self, grad):
        self.grad = grad


def rank_checkpoint_path(path: str, rank: int, world: int) -> str:
    """`chkpntN.pth` for a single-GPU run, `chkpntN_rank{r}.pth` for rank r of a Gaussian-sharded run (any existing
    `_rank{k}` suffix of the given path is replaced, so the same --start_checkpoint works on every rank)."""
    import re
    if world == 1:
        return path
    stem, ext = os.path.splitext(path)
    stem = re.sub(r"_rank\d+$", "", stem)
    return f"{stem}_rank{rank}{ext}"


def total_gaussians(gaussians: GaussianModel, world: int) -> int:
    n = int(gaussians.get_xyz.shape[0])
    if world == 1:
        return n
    t = torch.tensor([n], device="cuda", dtype=torch.int64)
    torch.distributed.all_reduce(t)
    return int(t.item())


def write_eval_yaml(model_path: str, iteration: int, ev: dict):
    """`eval/iter_xxxxxx/eval3d.yml` + `eval2d_render_{train,test}.yml` with the reference's keys (`train.py:283-330`)."""
    import yaml
    out = os.path.join(model_path, "eval", f"iter_{iteration:06d}")
    os.makedirs(out, exist_ok=True)
    d3 = {k: float(v) for k, v in ev.items() if k.endswith("_3d")}
    with open(os.path.join(out, "eval3d.yml"), "w") as f:
        yaml.dump(d3, f, default_flow_style=False, sort_keys=False)
    for name in ("train", "test"):
        d2 = {k.replace(f"_{name}", ""): float(v) for k, v in ev.items() if k.endswith(f"_2d_{name}")}
        if d2:
            with open(os.path.join(out, f"eval2d_render_{name}.yml"), "w") as f:
                yaml.dump(d2, f, default_flow_style=False, sort_keys=False)


def write_cfg_args(model_path: str, model, pipe, opt, extra: dict, pose: PoseParams | None = None,
                   detector: DetectorParams | None = None):
    """`<model_path>/cfg_args`: the Namespace repr the reference's test.py evaluates (`arguments/__init__.py:74-95`,
    written by `utils/log_utils.py:28-29`), with the reference's field names, next to a JSON copy.  The pose settings
    are added (flat, and as "pose" in the JSON) only when `pose.pose_refine` is on, the detector settings (as "detector")
    only when `detector.detector_offset_refine` is on."""
    from argparse import Namespace
    pose_fields = asdict(pose) if pose is not None and pose.pose_refine else {}
    det_fields = asdict(detector) if detector is not None and detector.detector_offset_refine else {}
    flat = {**asdict(model), **asdict(pipe), **asdict(opt), **pose_fields, **det_fields, **extra}
    with open(os.path.join(model_path, "cfg_args"), "w") as f:
        f.write(str(Namespace(**flat)))
    doc = {"model": asdict(model), "pipe": asdict(pipe), "opt": asdict(opt)}
    if pose_fields:
        doc["pose"] = pose_fields
    if det_fields:
        doc["detector"] = det_fields
    with open(os.path.join(model_path, "cfg_args.json"), "w") as f:
        json.dump(doc, f, indent=1)


def save_sharded(scene: Scene, gaussians: GaussianModel, iteration: int, queryfunc, rank: int):
    """`Scene.save` for a Gaussian-sharded run: all ranks take part (the volume query is a collective), rank 0
    writes ONE merged `point_cloud.pickle` + the volumes, in the layout `test.py` reads."""
    import pickle
    out = os.path.join(scene.model_path, "point_cloud/iteration_{}".format(iteration))
    merged = gather_point_cloud(gaussians)
    vol_pred = queryfunc(gaussians)["vol"] if queryfunc is not None else None
    if rank == 0:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "point_cloud.pickle"), "wb") as f:
            pickle.dump(merged, f, pickle.HIGHEST_PROTOCOL)
        if vol_pred is not None:
            np.save(os.path.join(out, "vol_gt.npy"), scene.vol_gt.detach().cpu().numpy())
            np.save(os.path.join(out, "vol_pred.npy"), vol_pred.detach().cpu().numpy())
    # rank 0 alone does the file I/O: nobody may run ahead into the next exchange (the peer-memory kernel waits a
    # bounded time for late ranks), and any reduction that gave up since the last check is reported here
    torch.distributed.barrier()
    sharded.check_peer_exchange()


def _add_dataclass_args(parser, cls, skip=()):
    for name, f in cls.__dataclass_fields__.items():
        if name in skip:
            continue
        default = f.default
        if isinstance(default, bool):
            parser.add_argument("--" + name, default=default, action="store_true")
        else:
            typ = float if (default is None or isinstance(default, float)) else type(default)
            parser.add_argument("--" + name, default=default, type=typ)


def parse_args(argv=None):
    """-> (argparse namespace, ModelParams, PipelineParams, OptimizationParams, PoseParams) of the command line; the
    namespace's `detector_params` holds the DetectorParams."""
    ap = argparse.ArgumentParser(description="Train R2-Gaussian on one scene (H100-native pipeline)")
    ap.add_argument("-s", "--source_path", required=True)
    ap.add_argument("-m", "--model_path", default="")
    _add_dataclass_args(ap, ModelParams, skip=("source_path", "model_path"))
    _add_dataclass_args(ap, PipelineParams)
    _add_dataclass_args(ap, OptimizationParams)
    _add_dataclass_args(ap, PoseParams)
    _add_dataclass_args(ap, DetectorParams)
    ap.add_argument("--test_iterations", nargs="+", type=int, default=[5000, 10000, 20000, 30000])
    ap.add_argument("--save_iterations", nargs="+", type=int, default=[])
    ap.add_argument("--checkpoint_iterations", nargs="+", type=int, default=[])
    ap.add_argument("--start_checkpoint", type=str, default=None)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--peer_exchange", action="store_true",
                    help="multi-GPU: sum partial images / volumes with the NVLink peer-memory kernel instead of NCCL")
    ap.add_argument("--batch_size", type=int, default=1,
                    help="train views per optimizer step (1 .. number of train views); schedules stay in steps")
    ap.add_argument("--use_offDetector", action="store_true",
                    help="train through the scanner's offDetector (every camera's projection matrix carries it)")
    ap.add_argument("--estimate_offDetector", action="store_true",
                    help="estimate the horizontal detector offset from the train views (on top of the file's under "
                         "--use_offDetector) and train through it")
    ap.add_argument("--use_view_geometry", action="store_true",
                    help="train through each view's own DSO, DSD, offOrigin and offDetector (the projection frames' "
                         "keys; helical scans, calibrated benches); implies --use_offDetector")
    a = ap.parse_args(argv)
    pick = lambda cls: cls(**{k: getattr(a, k) for k in cls.__dataclass_fields__})
    model, pipe, opt, pose = pick(ModelParams), pick(PipelineParams), pick(OptimizationParams), pick(PoseParams)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if pose.pose_refine and world > 1:
        ap.error("--pose_refine is not supported with Gaussian sharding (WORLD_SIZE > 1): every rank would hold only "
                 "its shard's part of the camera-matrix gradients; train on one GPU")
    why = batch_refusal(a.batch_size, pose.pose_refine, world, pipe.compute_cov3D_python)
    if why is not None:
        ap.error(why)
    a.detector_params = pick(DetectorParams)
    why = detector_refusal(a.detector_params.detector_offset_refine, pose.pose_refine, world)
    if why is not None:
        ap.error(why)
    try:
        why = view_geometry_refusal(a.use_view_geometry, a.estimate_offDetector, world, a.batch_size, a.source_path)
    except (OSError, ValueError, KeyError) as e:
        why = f"--use_view_geometry: cannot read the train views of {a.source_path}: {e}"
    if why is not None:
        ap.error(why)
    if a.batch_size > 1:
        try:
            n_train = train_view_count(a.source_path)
        except (OSError, ValueError, KeyError) as e:
            ap.error(f"--batch_size: cannot count the train views of {a.source_path}: {e}")
        if a.batch_size > n_train:
            ap.error(f"--batch_size {a.batch_size} exceeds the scene's {n_train} train views")
    return a, model, pipe, opt, pose


def main(argv=None):
    a, model, pipe, opt, pose = parse_args(argv)
    model.source_path = os.path.abspath(model.source_path)
    if not model.model_path:
        model.model_path = os.path.join("./output", os.path.basename(model.source_path.rstrip("/")))
    os.makedirs(model.model_path, exist_ok=True)
    if int(os.environ.get("RANK", "0")) == 0:
        write_cfg_args(model.model_path, model, pipe, opt,
                       {"test_iterations": a.test_iterations, "save_iterations": a.save_iterations,
                        "checkpoint_iterations": a.checkpoint_iterations, "start_checkpoint": a.start_checkpoint,
                        "quiet": False, "config": None, "detect_anomaly": False,
                        **({"batch_size": a.batch_size} if a.batch_size > 1 else {}),
                        **({"use_offDetector": True} if a.use_offDetector else {}),
                        **({"estimate_offDetector": True} if a.estimate_offDetector else {}),
                        **({"use_view_geometry": True} if a.use_view_geometry else {})}, pose, a.detector_params)
    random.seed(a.seed), np.random.seed(a.seed), torch.manual_seed(a.seed)     # safe_state (`general_utils.py:61-63`)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:                      # launched by torchrun: one process per GPU, Gaussians sharded by index
        import torch.distributed as dist
        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        sharded.enable()                       # Gaussian sharding is an explicit opt-in of render() / query()
        if a.peer_exchange:
            from .sharded import enable_peer_exchange
            enable_peer_exchange(True)
    hist = training(model, opt, pipe, set(a.test_iterations) | {opt.iterations}, set(a.save_iterations),
                    set(a.checkpoint_iterations), a.start_checkpoint, pose_params=pose, batch_size=a.batch_size,
                    detector_params=a.detector_params, use_offDetector=a.use_offDetector,
                    estimate_offDetector=a.estimate_offDetector, use_view_geometry=a.use_view_geometry)
    final = hist["eval"].get(opt.iterations, {})
    if world > 1:
        import torch.distributed as dist
        from .sharded import enable_peer_exchange
        enable_peer_exchange(False)
        sharded.enable(on=False)
        rank0 = dist.get_rank() == 0
        dist.barrier()
        dist.destroy_process_group()
        if not rank0:
            return
    n_it = max(hist["iterations"], 1)
    print(json.dumps({"seconds": hist["seconds"], "train_seconds": hist["train_seconds"],
                      "ms_per_iteration": hist["train_seconds"] / n_it * 1e3,       # training steps alone
                      "ms_per_iteration_with_save_and_eval": hist["seconds"] / n_it * 1e3,
                      "steady_ms_per_iteration": hist.get("steady_ms_per_iteration"),
                      "repeated_iterations": hist.get("repeated_iterations", 0),
                      "gaussians": hist["gaussians"], **({"batch_size": a.batch_size} if a.batch_size > 1 else {}),
                      **({"detector_offset_px": hist["detector_offset_px"]} if "detector_offset_px" in hist else {}),
                      **({"detector_estimate_px": hist["detector_estimate_px"]} if "detector_estimate_px" in hist
                         else {}),
                      **final}))


if __name__ == "__main__":
    main()
