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
from .dataset import Scene
from .gaussian_model import GaussianModel
from .metrics import metric_proj, metric_vol
from .render_query import query, render
from . import sharded, train_step
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


@torch.no_grad()
def evaluate(scene: Scene, gaussians: GaussianModel, pipe, with_ssim: bool = True) -> dict:
    """3-D PSNR / SSIM of the queried volume and 2-D PSNR / SSIM of the rendered train and test views, with the
    reference's metric definitions (`train.py:262-330`, `utils/image_utils.py:90-183`)."""
    cfg = scene.scanner_cfg
    vol = query(gaussians, cfg["offOrigin"], cfg["nVoxel"], cfg["sVoxel"], pipe)["vol"]
    out = {"psnr_3d": metric_vol(scene.vol_gt, vol, "psnr")[0]}
    if with_ssim:
        out["ssim_3d"] = metric_vol(scene.vol_gt, vol, "ssim")[0]
    for name, cams in (("train", scene.getTrainCameras()), ("test", scene.getTestCameras())):
        if not cams:
            continue
        imgs = torch.concat([render(c, gaussians, pipe)["render"] for c in cams], 0).permute(1, 2, 0)
        gts = torch.concat([c.original_image.to(imgs.device) for c in cams], 0).permute(1, 2, 0)
        out[f"psnr_2d_{name}"] = metric_proj(gts, imgs, "psnr")[0]
        if with_ssim:
            out[f"ssim_2d_{name}"] = metric_proj(gts, imgs, "ssim")[0]
    return out


def training(model: ModelParams, opt: OptimizationParams, pipe: PipelineParams, testing_iterations=(),
             saving_iterations=(), checkpoint_iterations=(), checkpoint: str | None = None, init_points=None,
             log=print) -> dict:
    first_iter = 0
    scene = Scene(model.source_path, model.model_path, eval=model.eval, shuffle=False, device="cuda",
                  data_device=model.data_device)
    cfg = scene.scanner_cfg
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
    if checkpoint is not None:
        path = rank_checkpoint_path(checkpoint, rank, world)
        payload = torch.load(path, weights_only=False)
        model_state, first_iter = payload[0], payload[1]
        tag = payload[2] if len(payload) > 2 else {"rank": 0, "world": 1}
        if (tag["rank"], tag["world"]) != (rank, world):
            raise RuntimeError(f"checkpoint {path} was written by rank {tag['rank']} of {tag['world']}; this process is "
                               f"rank {rank} of {world} (a Gaussian-sharded run resumes with the same number of ranks)")
        gaussians.restore(model_state, opt)
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
                                            [float(v) for v in tv_s])
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
        if not stack:
            stack = scene.getTrainCameras().copy()
        cam = stack.pop(random.randint(0, len(stack) - 1))

        densify_due = iteration < opt.densify_until_iter and iteration > opt.densify_from_iter \
            and iteration % opt.densification_interval == 0
        centre = None
        if use_tv:
            centre = (bbox_cpu[0] + tv_s / 2) + (bbox_cpu[1] - tv_s - bbox_cpu[0]) * torch.rand(3)
        if native is not None and (gaussians.get_xyz.shape[0] > 0 or world > 1):
            # fixed launch sequence, no autograd (train_step.py).  At a densification iteration the reference's
            # optimizer.step() comes AFTER the tensors were replaced and therefore applies nothing (their .grad is None,
            # train.py:158-176): the same here.
            gt = cam.original_image.cuda()
            native(cam, gt, centre, apply_update=(iteration < opt.iterations) and not densify_due)
            total = None
            with torch.no_grad():
                if densify_due:
                    native.flush()
                    gaussians.densify_and_prune(opt.densify_grad_threshold, opt.density_min_threshold, opt.max_screen_size,
                                                ds["max_scale"], opt.max_num_gaussians, ds["densify_scale_threshold"], bbox)
        else:
            pkg = render(cam, gaussians, pipe)
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
                pkg = render(cam, gaussians, pipe)
                total = losses.image_loss(pkg["render"], gt, lambda_dssim=opt.lambda_dssim)["total"]
                if use_tv:
                    total = total + opt.lambda_tv * losses.tv_3d_loss(query(gaussians, centre, tv_n, tv_s, pipe)["vol"],
                                                                      reduction="mean")
                total.backward()
            with torch.no_grad():
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
            if native is not None and (iteration in saving_iterations or iteration in checkpoint_iterations or
                                       iteration in testing_iterations or iteration == opt.iterations):
                native.flush()       # the last enqueued iteration is checked (and repeated if it had overflowed)
            if scene.model_path and (iteration in saving_iterations or iteration == opt.iterations):
                log(f"[ITER {iteration}] Saving Gaussians")
                with _aside():
                    if world == 1:
                        scene.save(iteration, queryfunc)
                    else:
                        save_sharded(scene, gaussians, iteration, queryfunc, rank)
            if scene.model_path and iteration in checkpoint_iterations:
                log(f"[ITER {iteration}] Saving Checkpoint")
                with _aside():
                    name = os.path.basename(rank_checkpoint_path(f"chkpnt{iteration}.pth", rank, world))
                    payload = (gaussians.capture(), iteration) if world == 1 else \
                        (gaussians.capture(), iteration, {"rank": rank, "world": world})
                    torch.save(payload, os.path.join(ckpt_dir, name))
                    if world > 1:
                        torch.distributed.barrier()  # no rank runs ahead into the next exchange while others write
            if iteration % 100 == 0:
                history["loss"].append((iteration, float(total) if total is not None else native.total_loss()))
                if world > 1:
                    sharded.check_peer_exchange()    # the loss read-out above synchronised anyway
            if iteration in testing_iterations:
                with _aside():
                    history["eval"][iteration] = evaluate(scene, gaussians, pipe)
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
    return history


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


def write_cfg_args(model_path: str, model, pipe, opt, extra: dict):
    """`<model_path>/cfg_args`: the Namespace repr the reference's test.py evaluates (`arguments/__init__.py:74-95`,
    written by `utils/log_utils.py:28-29`), with the reference's field names, next to a JSON copy."""
    from argparse import Namespace
    flat = {**asdict(model), **asdict(pipe), **asdict(opt), **extra}
    with open(os.path.join(model_path, "cfg_args"), "w") as f:
        f.write(str(Namespace(**flat)))
    with open(os.path.join(model_path, "cfg_args.json"), "w") as f:
        json.dump({"model": asdict(model), "pipe": asdict(pipe), "opt": asdict(opt)}, f, indent=1)


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


def main(argv=None):
    ap = argparse.ArgumentParser(description="Train R2-Gaussian on one scene (H100-native pipeline)")
    ap.add_argument("-s", "--source_path", required=True)
    ap.add_argument("-m", "--model_path", default="")
    _add_dataclass_args(ap, ModelParams, skip=("source_path", "model_path"))
    _add_dataclass_args(ap, PipelineParams)
    _add_dataclass_args(ap, OptimizationParams)
    ap.add_argument("--test_iterations", nargs="+", type=int, default=[5000, 10000, 20000, 30000])
    ap.add_argument("--save_iterations", nargs="+", type=int, default=[])
    ap.add_argument("--checkpoint_iterations", nargs="+", type=int, default=[])
    ap.add_argument("--start_checkpoint", type=str, default=None)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--peer_exchange", action="store_true",
                    help="multi-GPU: sum partial images / volumes with the NVLink peer-memory kernel instead of NCCL")
    a = ap.parse_args(argv)
    pick = lambda cls: cls(**{k: getattr(a, k) for k in cls.__dataclass_fields__})
    model, pipe, opt = pick(ModelParams), pick(PipelineParams), pick(OptimizationParams)
    model.source_path = os.path.abspath(model.source_path)
    if not model.model_path:
        model.model_path = os.path.join("./output", os.path.basename(model.source_path.rstrip("/")))
    os.makedirs(model.model_path, exist_ok=True)
    if int(os.environ.get("RANK", "0")) == 0:
        write_cfg_args(model.model_path, model, pipe, opt,
                       {"test_iterations": a.test_iterations, "save_iterations": a.save_iterations,
                        "checkpoint_iterations": a.checkpoint_iterations, "start_checkpoint": a.start_checkpoint,
                        "quiet": False, "config": None, "detect_anomaly": False})
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
                    set(a.checkpoint_iterations), a.start_checkpoint)
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
                      "gaussians": hist["gaussians"], **final}))


if __name__ == "__main__":
    main()
