"""Evaluate a trained model -- the reference's `test.py` with its `get_combined_args`.

    python -m r2_gaussian_b200.test -m <model> [-s <scene>] [--iteration -1] [--skip_render_train]
        [--skip_render_test] [--skip_recon] [--quiet]

Settings come from what `trainer` recorded: `<model>/cfg_args.json`, plus the run options only the flat
`<model>/cfg_args` carries (such as `use_offDetector` and `use_view_geometry`); without the JSON, `cfg_args` alone, the `Namespace(...)` repr,
read with `ast` (never evaluated).  Options given on the command line win over the file.  `--iteration -1` loads the
largest N among `<model>/point_cloud/iteration_N/` (the reference's `searchForMaxIteration`).

The model is evaluated with the geometry `trainer.evaluate` uses at that iteration: with `iteration_N/train_poses.npz`
(`trainer --pose_refine`) the train views carry their learned corrections, re-formed from the stored omega / nu and
checked bit for bit against the stored `world_view_transform` rows; with `iteration_N/detector_offset.yml`
(`--detector_offset_refine`) both splits carry the learned detector offset.

Writes under `<model>/test/iter_N/`, with the reference's names, keys and order:
  render_train/, render_test/        {i:05d}_gt.npy, {i:05d}_pred.npy ([H, W] float32, one per view)
  eval2d_render_train.yml, eval2d_render_test.yml   psnr_2d, ssim_2d, psnr_2d_projs, ssim_2d_projs
  reconstruction/                    {i:05d}_gt.npy, {i:05d}_pred.npy (the [nx, ny] slice i of the last axis)
  eval3d.yml                         psnr_3d, ssim_3d, ssim_3d_x, ssim_3d_y, ssim_3d_z
  vol_gt.npy, vol_pred.npy, vol_gt.nii.gz, vol_pred.nii.gz
Each `--skip_*` flag skips its work and its files.  Scores come from `metrics.volume_metrics` /
`metrics.projection_metrics`.  Not written: PNG images (matplotlib and torchvision are not dependencies).  The NIfTI
files come from `write_nifti`, a numpy + gzip writer of what SimpleITK writes for the reference's array; byte parity
with SimpleITK is not checked.  GPU only; a Gaussian-sharded run's merged pickle is evaluated on one GPU.
"""
from __future__ import annotations

import argparse
import ast
import gzip
import json
import os
import re
import struct
import sys
import time

import numpy as np

from .trainer import ModelParams, PipelineParams

SETTING_FLAGS = ("source_path", "data_device", "compute_cov3D_python", "debug", "use_offDetector", "use_view_geometry")


def parse_cfg_args(text: str) -> dict:
    """The `Namespace(k=v, ...)` repr `trainer.write_cfg_args` writes -> dict, with `ast.literal_eval` per value."""
    tree = ast.parse(text.strip(), mode="eval").body
    if not (isinstance(tree, ast.Call) and isinstance(tree.func, ast.Name) and tree.func.id == "Namespace"
            and not tree.args):
        raise ValueError("cfg_args: expected a Namespace(key=value, ...) repr")
    return {kw.arg: ast.literal_eval(kw.value) for kw in tree.keywords}


def load_settings(model_path: str) -> dict:
    """The flat settings the trainer recorded under `model_path` (see the module docstring)."""
    js, flat = os.path.join(model_path, "cfg_args.json"), os.path.join(model_path, "cfg_args")
    out = {}
    if os.path.exists(flat):
        with open(flat) as f:
            out = parse_cfg_args(f.read())
    if os.path.exists(js):
        with open(js) as f:
            doc = json.load(f)
        for section in doc.values():
            out.update(section)
    elif not out:
        raise FileNotFoundError(f"no recorded settings: neither {js} nor {flat} exists")
    return out


def iteration_dirs(model_path: str) -> dict:
    """{N: path} of `<model_path>/point_cloud/iteration_N/`."""
    root = os.path.join(model_path, "point_cloud")
    if not os.path.isdir(root):
        raise FileNotFoundError(f"no saved iterations: {root} does not exist")
    found = {}
    for name in os.listdir(root):
        m = re.fullmatch(r"iteration_(\d+)", name)
        if m and os.path.isdir(os.path.join(root, name)):
            found[int(m.group(1))] = os.path.join(root, name)
    return found


def resolve_iteration(model_path: str, iteration: int) -> tuple[int, str]:
    """(N, path of iteration_N/point_cloud.pickle): -1 picks the largest saved N."""
    found = iteration_dirs(model_path)
    if iteration == -1:
        if not found:
            raise FileNotFoundError(f"no saved iterations under {os.path.join(model_path, 'point_cloud')}")
        iteration = max(found)
    if iteration not in found:
        raise FileNotFoundError(f"iteration {iteration} was not saved: "
                                f"{os.path.join(model_path, 'point_cloud', f'iteration_{iteration}')} does not exist")
    pickle_path = os.path.join(found[iteration], "point_cloud.pickle")
    if not os.path.exists(pickle_path):
        raise FileNotFoundError(f"cannot find {pickle_path} for loading")
    return iteration, pickle_path


def parse_args(argv=None):
    """-> (namespace of the command line, merged settings dict)."""
    ap = argparse.ArgumentParser(description="Evaluate a trained R2-Gaussian model: renders, volume, PSNR / SSIM "
                                             "(the reference's test.py)")
    ap.add_argument("-m", "--model_path", required=True, help="output directory of a trainer run")
    ap.add_argument("-s", "--source_path", default=None, help="scene (default: the one the model was trained on)")
    ap.add_argument("--data_device", default=None)
    ap.add_argument("--compute_cov3D_python", action="store_const", const=True, default=None)
    ap.add_argument("--debug", action="store_const", const=True, default=None)
    ap.add_argument("--use_offDetector", action="store_const", const=True, default=None,
                    help="evaluate through the scanner's offDetector (default: as the model was trained)")
    ap.add_argument("--use_view_geometry", action="store_const", const=True, default=None,
                    help="evaluate through each view's own geometry (default: as the model was trained)")
    ap.add_argument("--iteration", default=-1, type=int, help="saved iteration to evaluate (-1: the last one)")
    ap.add_argument("--skip_render_train", action="store_true", default=False)
    ap.add_argument("--skip_render_test", action="store_true", default=False)
    ap.add_argument("--skip_recon", action="store_true", default=False)
    ap.add_argument("--quiet", action="store_true", default=False)
    a = ap.parse_args(argv)
    if not os.path.isdir(a.model_path):
        ap.error(f"model directory {a.model_path} does not exist")
    try:
        settings = load_settings(a.model_path)
    except (OSError, ValueError, SyntaxError) as e:
        ap.error(str(e))
    for k in SETTING_FLAGS:
        if getattr(a, k) is not None:
            settings[k] = getattr(a, k)
    if not settings.get("source_path"):
        ap.error("no scene: the recorded settings name none; pass -s")
    return a, settings


# ---- NIfTI-1 ----------------------------------------------------------------------------------------------------------

NIFTI_HEADER = 348
NIFTI_VOX_OFFSET = 352


def nifti_header(shape_xyz) -> bytes:
    """The 348-byte NIfTI-1 header of a float32 image of ITK size `shape_xyz` (fastest axis first): unit spacing, zero
    origin, identity LPS direction, which NIfTI stores as the RAS affine diag(-1, -1, 1, 1) in both the qform and the
    sform (code 1)."""
    nx, ny, nz = (int(v) for v in shape_xyz)
    h = bytearray(NIFTI_HEADER)
    struct.pack_into("<i", h, 0, NIFTI_HEADER)
    h[38] = ord("r")
    struct.pack_into("<8h", h, 40, 3, nx, ny, nz, 1, 1, 1, 1)
    struct.pack_into("<hhh", h, 70, 16, 32, 0)                       # datatype FLOAT32, bitpix, slice_start
    struct.pack_into("<8f", h, 76, 1.0, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 0.0)   # qfac, spacing
    struct.pack_into("<3f", h, 108, float(NIFTI_VOX_OFFSET), 1.0, 0.0)     # vox_offset, scl_slope, scl_inter
    h[123] = 2 | 8                                                   # xyzt_units: mm, s
    struct.pack_into("<hh", h, 252, 1, 1)                            # qform_code, sform_code: scanner
    struct.pack_into("<6f", h, 256, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0)    # quatern b, c, d (180 deg about z), qoffset
    struct.pack_into("<12f", h, 280, -1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1, 0)   # srow_x, srow_y, srow_z
    h[344:348] = b"n+1\0"
    return bytes(h)


def write_nifti(path: str, vol: np.ndarray):
    """`vol` [nx, ny, nz] as the reference writes it, `sitk.WriteImage(sitk.GetImageFromArray(vol.transpose(2, 0, 1)))`:
    the data are that transposed array's bytes in C order (ITK size [ny, nx, nz]) as float32, gzip-compressed."""
    data = np.ascontiguousarray(np.asarray(vol).transpose(2, 0, 1), dtype="<f4")
    nz, nx, ny = data.shape
    with gzip.open(path, "wb") as f:
        f.write(nifti_header((ny, nx, nz)))
        f.write(b"\0" * (NIFTI_VOX_OFFSET - NIFTI_HEADER))          # no extensions
        f.write(data.tobytes())


# ---- evaluation -------------------------------------------------------------------------------------------------------

class _Clock:
    """Seconds per phase; each phase synchronises the device on both sides."""

    def __init__(self):
        self.seconds = {"render": 0.0, "metrics": 0.0, "write": 0.0}

    def phase(self, name):
        import torch
        clock = self

        class _Phase:
            def __enter__(self):
                torch.cuda.synchronize()
                self.t0 = time.perf_counter()

            def __exit__(self, *exc):
                torch.cuda.synchronize()
                clock.seconds[name] += time.perf_counter() - self.t0
                return False
        return _Phase()


def _dump_yaml(path: str, doc: dict):
    import yaml
    with open(path, "w") as f:
        yaml.dump(doc, f, default_flow_style=False, sort_keys=False)


def _write_slices(path: str, stack: np.ndarray, suffix: str):
    os.makedirs(path, exist_ok=True)
    for i in range(stack.shape[0]):
        np.save(os.path.join(path, f"{i:05d}{suffix}.npy"), stack[i])


def correction_modules(iter_dir: str, scene):
    """(PoseCorrection or None, DetectorOffset or None) of a saved iteration: what `trainer.evaluate` used there."""
    import torch
    import yaml

    from .detector import DetectorOffset
    from .pose import PoseCorrection
    from .trainer import POSE_ANCHOR

    pose = det = None
    poses_path = os.path.join(iter_dir, "train_poses.npz")
    if os.path.exists(poses_path):
        stored = np.load(poses_path)
        cams = scene.getTrainCameras()
        if stored["omega"].shape != (len(cams), 3):
            raise ValueError(f"{poses_path} holds poses of {stored['omega'].shape[0]} train views, the scene has "
                             f"{len(cams)}")
        pose = PoseCorrection(len(cams), device="cuda")
        with torch.no_grad():
            pose.omega.copy_(torch.from_numpy(stored["omega"]))
            pose.nu.copy_(torch.from_numpy(stored["nu"]))
            wvt = torch.stack([pose.device_camera(c, c.uid, POSE_ANCHOR).world_view_transform for c in cams])
        if not np.array_equal(wvt.cpu().numpy().view(np.uint32),
                              np.asarray(stored["world_view_transform"], np.float32).view(np.uint32)):
            raise ValueError(f"{poses_path}: the poses re-formed from omega / nu differ from its stored "
                             "world_view_transform rows")
    offset_path = os.path.join(iter_dir, "detector_offset.yml")
    if os.path.exists(offset_path):
        with open(offset_path) as f:
            doc = yaml.safe_load(f)
        det = DetectorOffset("cuda")
        with torch.no_grad():
            det.offset.fill_(float(doc["offset_px"]))
    return pose, det


def testing(model_path: str, settings: dict, iteration: int = -1, skip_render_train: bool = False,
            skip_render_test: bool = False, skip_recon: bool = False, log=print) -> dict:
    """Evaluate the model saved under `model_path` at `iteration` (-1: the last) -> {"iteration", "path", "eval2d_*",
    "eval3d" (the written scores), "seconds": {"render", "metrics", "write"}}."""
    import torch

    from .dataset import Scene
    from .gaussian_model import GaussianModel
    from .metrics import projection_metrics, volume_metrics
    from .render_query import query, render
    from .trainer import evaluation_cameras

    iteration, pickle_path = resolve_iteration(model_path, iteration)
    pick = lambda cls: cls(**{k: settings[k] for k in cls.__dataclass_fields__ if k in settings})
    model, pipe = pick(ModelParams), pick(PipelineParams)
    scene = Scene(settings["source_path"], model_path, eval=model.eval, shuffle=False, device="cuda",
                  data_device=model.data_device, use_offDetector=bool(settings.get("use_offDetector", False)),
                  use_view_geometry=bool(settings.get("use_view_geometry", False)))
    gaussians = GaussianModel(None)
    gaussians.load_ply(pickle_path)
    scene.gaussians = gaussians
    log(f"Loading trained model at iteration {iteration}")
    pose, det = correction_modules(os.path.dirname(pickle_path), scene)
    save_path = os.path.join(model_path, "test", f"iter_{iteration}")
    os.makedirs(save_path, exist_ok=True)
    clock = _Clock()
    out = {"iteration": iteration, "path": save_path}
    skip = {"train": skip_render_train, "test": skip_render_test}
    with torch.no_grad():
        for split, cams in evaluation_cameras(scene, pose, det):
            if skip[split]:
                continue
            name = f"render_{split}"
            with clock.phase("render"):
                preds = torch.cat([render(c, gaussians, pipe)["render"] for c in cams], 0)
                gts = torch.cat([c.original_image for c in cams], 0).to(preds.device)
            with clock.phase("metrics"):
                ev = projection_metrics(gts, preds)
            with clock.phase("write"):
                _write_slices(os.path.join(save_path, name), gts.cpu().numpy(), "_gt")
                _write_slices(os.path.join(save_path, name), preds.cpu().numpy(), "_pred")
                _dump_yaml(os.path.join(save_path, f"eval2d_{name}.yml"), ev)
            out[f"eval2d_{name}"] = ev
            log(f"{name} complete. psnr_2d: {ev['psnr_2d']}, ssim_2d: {ev['ssim_2d']}.")
        if not skip_recon:
            cfg = scene.scanner_cfg
            with clock.phase("render"):
                vol_pred = query(gaussians, cfg["offOrigin"], cfg["nVoxel"], cfg["sVoxel"], pipe)["vol"]
            with clock.phase("metrics"):
                ev = volume_metrics(scene.vol_gt, vol_pred)
            with clock.phase("write"):
                vg, vp = scene.vol_gt.cpu().numpy(), vol_pred.cpu().numpy()
                rec = os.path.join(save_path, "reconstruction")
                _write_slices(rec, np.moveaxis(vg, 2, 0), "_gt")
                _write_slices(rec, np.moveaxis(vp, 2, 0), "_pred")
                _dump_yaml(os.path.join(save_path, "eval3d.yml"), ev)
                np.save(os.path.join(save_path, "vol_gt.npy"), vg)
                np.save(os.path.join(save_path, "vol_pred.npy"), vp)
                write_nifti(os.path.join(save_path, "vol_gt.nii.gz"), vg)
                write_nifti(os.path.join(save_path, "vol_pred.nii.gz"), vp)
            out["eval3d"] = ev
            log(f"reconstruction complete. psnr_3d: {ev['psnr_3d']}, ssim_3d: {ev['ssim_3d']}")
    out["seconds"] = clock.seconds
    return out


def main(argv=None) -> dict:
    a, settings = parse_args(argv)
    try:
        resolve_iteration(a.model_path, a.iteration)
    except FileNotFoundError as e:
        raise SystemExit(str(e)) from e
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("evaluation needs a CUDA device: rendering and the metrics run on the GPU and have no CPU "
                         "fallback")
    log = (lambda *args: None) if a.quiet else print
    try:
        return testing(a.model_path, settings, a.iteration, a.skip_render_train, a.skip_render_test, a.skip_recon,
                       log=log)
    except (FileNotFoundError, ValueError) as e:
        raise SystemExit(str(e)) from e


if __name__ == "__main__":
    main(sys.argv[1:])
