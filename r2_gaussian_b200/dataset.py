"""Scene I/O in the reference's on-disk formats (SURVEY §8(f) rank 4).

* `read_blender(path, eval)` -- directory with `meta_data.json` (+ `proj_*/*.npy`, `vol_gt.npy`), the layout of
  `r2_gaussian/dataset/dataset_readers.py:43-153`;
* `read_naf(path, eval)` -- NAF pickle (`:196-307`, millimetres -> metres);
* both rescale every length so that the volume of interest becomes [-1, 1]^3 (`scene_scale = 2 / max(sVoxel)`,
  projections multiplied by the same factor) and derive pose / FoV per view exactly like the reference;
* `Camera` exposes the attributes render() reads (`dataset/cameras.py:20-84`); `Scene` the reference's
  (`dataset/__init__.py:26-99`): `getTrainCameras()`, `getTestCameras()`, `vol_gt`, `scanner_cfg`, `bbox`, `save`;
* `init_point_cloud` = `initialize_pcd.py:41-91` (random cloud, or voxels of a given reconstruction above a threshold
  -- the reconstruction itself is passed in: `fdk.fdk` on the GPU, TIGRE's FDK in the reference);
* `write_blender` writes a dataset in that format (used by the tests and by `generate_data`, which makes synthetic
  scenes from a CT volume with the GPU projector of `projector.py` where the reference uses TIGRE's `Ax`).

Device is a parameter everywhere ("cuda" by default like the reference; the CPU tests pass "cpu").
"""
from __future__ import annotations

import json
import math
import os
import pickle
import random
import warnings
from dataclasses import dataclass, field

import numpy as np
import torch

from .scene import VIEW_KEYS, camera_pose, detector_shift, projection_matrix, shifted_projection_matrix, view_scanner

MODE_ID = {"parallel": 0, "cone": 1}
_LENGTH_KEYS = ("dVoxel", "sVoxel", "sDetector", "dDetector", "offOrigin", "offDetector", "DSD", "DSO")


@dataclass
class CameraInfo:
    uid: int
    R: np.ndarray          # w2c rotation, stored transposed (`dataset_readers.py:121-125`)
    T: np.ndarray
    angle: float
    FovY: float
    FovX: float
    image: np.ndarray      # [H, W], already multiplied by scene_scale
    image_path: str | None
    image_name: str
    width: int
    height: int
    mode: int
    scanner_cfg: dict
    view_geometry: dict = field(default_factory=dict)   # the frame's VIEW_KEYS overrides, in scene units


@dataclass
class SceneInfo:
    train_cameras: list
    test_cameras: list
    vol: np.ndarray
    scanner_cfg: dict
    scene_scale: float
    extra: dict = field(default_factory=dict)


def _rescale(cfg: dict) -> float:
    scale = 2.0 / max(cfg["sVoxel"])
    for k in _LENGTH_KEYS:
        cfg[k] = (np.asarray(cfg[k], dtype=np.float64) * scale).tolist()
    return scale


def _camera_info(uid, angle, image, name, path, cfg) -> CameraInfo:
    w2c = np.linalg.inv(camera_pose(cfg, angle))
    # dDetector / sDetector are [v, u]
    fov_x = math.atan2(cfg["sDetector"][1] / 2, cfg["DSD"]) * 2
    fov_y = math.atan2(cfg["sDetector"][0] / 2, cfg["DSD"]) * 2
    return CameraInfo(uid, np.transpose(w2c[:3, :3]), w2c[:3, 3], float(angle), fov_y, fov_x, image, path, name,
                      int(cfg["nDetector"][1]), int(cfg["nDetector"][0]), MODE_ID[cfg["mode"]], cfg)


def scale_scanner(cfg: dict) -> float:
    """Complete `dVoxel` / `dDetector` of a scanner dict in the reference's file format and rescale it in place to
    scene units (what `read_blender` does to `meta_data.json`'s scanner); returns scene_scale."""
    if "dVoxel" not in cfg:
        cfg["dVoxel"] = (np.asarray(cfg["sVoxel"], float) / np.asarray(cfg["nVoxel"], float)).tolist()
    if "dDetector" not in cfg:
        cfg["dDetector"] = (np.asarray(cfg["sDetector"], float) / np.asarray(cfg["nDetector"], float)).tolist()
    return _rescale(cfg)


def frame_geometry(frame: dict, scale: float) -> dict:
    """A projection frame's per-view overrides (`scene.VIEW_KEYS`), rescaled by `scale` as `_rescale` rescales the
    scanner's lengths."""
    return {k: (np.asarray(frame[k], dtype=np.float64) * scale).tolist() for k in VIEW_KEYS if k in frame}


def read_blender(path: str, eval: bool = True, use_view_geometry: bool = False) -> SceneInfo:
    """`use_view_geometry` builds each camera from its frame's overrides (`scene.view_scanner`); without it they are
    only recorded in `CameraInfo.view_geometry`, with one warning naming the flag when a frame carries any."""
    with open(os.path.join(path, "meta_data.json")) as f:
        meta = json.load(f)
    cfg = meta["scanner"]
    scale = scale_scanner(cfg)
    cams = {"train": [], "test": []}
    for split in (("train", "test") if eval else ("train",)):
        offset = len(meta["proj_train"]) if split == "test" else 0
        for i, frame in enumerate(meta["proj_" + split]):
            p = os.path.join(path, frame["file_path"])
            geo = frame_geometry(frame, scale)
            info = _camera_info(i + offset, frame["angle"], np.load(p) * scale, os.path.basename(p).split(".")[0], p,
                                view_scanner(cfg, geo) if use_view_geometry else cfg)
            info.view_geometry = geo
            cams[split].append(info)
    if not use_view_geometry and any(c.view_geometry for c in cams["train"] + cams["test"]):
        warnings.warn(f"{path}: its projection frames carry per-view geometry ({', '.join(VIEW_KEYS)}), which is "
                      "ignored: pass --use_view_geometry (use_view_geometry=True) to use it", stacklevel=2)
    vol = np.load(os.path.join(path, meta["vol"])).astype(np.float32)
    return SceneInfo(cams["train"], cams["test"], vol, cfg, scale)


def read_naf(path: str, eval: bool = True) -> SceneInfo:
    with open(path, "rb") as f:
        data = pickle.load(f)
    mm = lambda v: (np.asarray(v, dtype=np.float64) / 1000).tolist()      # NAF geometry is in millimetres
    cfg = {"DSD": data["DSD"] / 1000, "DSO": data["DSO"] / 1000, "nVoxel": data["nVoxel"], "dVoxel": mm(data["dVoxel"]),
           "sVoxel": mm(np.asarray(data["nVoxel"]) * np.asarray(data["dVoxel"])), "nDetector": data["nDetector"],
           "dDetector": mm(data["dDetector"]),
           "sDetector": mm(np.asarray(data["nDetector"]) * np.asarray(data["dDetector"])),
           "offOrigin": mm(data["offOrigin"]), "offDetector": mm(data["offDetector"]),
           "totalAngle": data["totalAngle"], "startAngle": data["startAngle"], "accuracy": data["accuracy"],
           "mode": data["mode"], "filter": None}
    scale = _rescale(cfg)
    cams = {"train": [], "test": []}
    for split in (("train", "test") if eval else ("train",)):
        if split == "test":
            offset, n = data["numTrain"], data["numVal"]
            part = data["val"] if "val" in data else data[split]
        else:
            offset, n, part = 0, data["numTrain"], data["train"]
        for i in range(n):
            cams[split].append(_camera_info(i + offset, part["angles"][i], part["projections"][i] * scale,
                                            f"{i + offset:04d}", None, cfg))
    return SceneInfo(cams["train"], cams["test"], np.asarray(data["image"], dtype=np.float32), cfg, scale)


def read_scene(source_path: str, eval: bool = True, use_view_geometry: bool = False) -> SceneInfo:
    """`use_view_geometry`: each camera from its frame's per-view geometry (`read_blender`; NAF pickles carry none)."""
    if os.path.exists(os.path.join(source_path, "meta_data.json")):
        return read_blender(source_path, eval, use_view_geometry)
    if source_path.split(".")[-1] in ("pickle", "pkl"):
        return read_naf(source_path, eval)
    raise ValueError(f"Could not recognize scene type: {source_path}.")


def train_view_count(source_path: str) -> int:
    """Number of train views of a scene (either format), without reading its projections."""
    if os.path.exists(os.path.join(source_path, "meta_data.json")):
        with open(os.path.join(source_path, "meta_data.json")) as f:
            return len(json.load(f)["proj_train"])
    if source_path.split(".")[-1] in ("pickle", "pkl"):
        with open(source_path, "rb") as f:
            return int(pickle.load(f)["numTrain"])
    raise ValueError(f"Could not recognize scene type: {source_path}.")


def train_view_dsd(source_path: str) -> list[float]:
    """Each train view's DSD under per-view geometry (its frame's, else the scanner's; file units), without reading
    the projections.  NAF pickles carry one DSD."""
    if os.path.exists(os.path.join(source_path, "meta_data.json")):
        with open(os.path.join(source_path, "meta_data.json")) as f:
            meta = json.load(f)
        return [float(fr.get("DSD", meta["scanner"]["DSD"])) for fr in meta["proj_train"]]
    if source_path.split(".")[-1] in ("pickle", "pkl"):
        with open(source_path, "rb") as f:
            return [float(pickle.load(f)["DSD"])]
    raise ValueError(f"Could not recognize scene type: {source_path}.")


class Camera:
    """What render() needs from a view (`dataset/cameras.py:20-84`), on `device`.  `use_offDetector` puts the scanner's
    offDetector into `projection_matrix` (`scene.detector_shift`), so full_proj_transform, pose corrections, batched
    views and the native training step all see it; off, or with a zero offset, the camera is today's bit for bit."""

    def __init__(self, info: CameraInfo, uid: int | None = None, device="cuda", data_device=None,
                 use_offDetector: bool = False):
        self.uid = info.uid if uid is None else uid
        self.colmap_id = info.uid
        self.R, self.T, self.angle = info.R, info.T, info.angle
        self.FoVx, self.FoVy, self.mode = info.FovX, info.FovY, info.mode
        self.image_name = info.image_name
        self.original_image = torch.from_numpy(np.asarray(info.image, dtype=np.float32))[None].to(data_device or device)
        self.image_height, self.image_width = int(self.original_image.shape[1]), int(self.original_image.shape[2])
        Rt = np.zeros((4, 4))
        Rt[:3, :3] = info.R.transpose()
        Rt[:3, 3] = info.T
        Rt[3, 3] = 1.0
        w2c = np.float32(np.linalg.inv(np.linalg.inv(Rt)))               # getWorld2View2 with zero translate
        self.world_view_transform = torch.tensor(w2c).transpose(0, 1).contiguous().to(device)
        P = projection_matrix(info.FovX, info.FovY, info.mode)
        if use_offDetector:
            P = shifted_projection_matrix(P, *detector_shift(info.scanner_cfg), self.image_width, self.image_height)
        proj = torch.tensor(P, dtype=torch.float32)
        self.projection_matrix = proj.transpose(0, 1).contiguous().to(device)
        self.full_proj_transform = (self.world_view_transform.unsqueeze(0).bmm(self.projection_matrix.unsqueeze(0))
                                    ).squeeze(0).contiguous()
        self.camera_center = self.world_view_transform.inverse()[3, :3].contiguous()


class Scene:
    def __init__(self, source_path: str, model_path: str = "", eval: bool = True, shuffle: bool = True, device="cuda",
                 data_device=None, use_offDetector: bool = False, offDetector_u: float | None = None,
                 use_view_geometry: bool = False):
        """`offDetector_u` (scene units) replaces the scanner's offDetector[0] in a copy of its config, the one every
        camera and `scanner_cfg` then carry (with `use_offDetector`, e.g. an estimated offset).  `use_view_geometry`
        builds every camera from its frame's per-view DSO, DSD, offOrigin and offDetector (`scene.view_scanner`) and
        implies `use_offDetector`; `scanner_cfg`, `bbox` and the grid stay the scanner's."""
        if use_view_geometry and offDetector_u is not None:
            raise ValueError("Scene: offDetector_u (an estimated offset of one fixed circle) cannot be combined with "
                             "use_view_geometry")
        use_offDetector = bool(use_offDetector or use_view_geometry)
        self.use_view_geometry = bool(use_view_geometry)
        self.model_path = model_path
        info = read_scene(source_path, eval, use_view_geometry)
        if offDetector_u is not None:
            from .detector import with_offDetector_u
            info.scanner_cfg = with_offDetector_u(info.scanner_cfg, offDetector_u)
            for c in info.train_cameras + info.test_cameras:
                c.scanner_cfg = info.scanner_cfg
        if shuffle:
            random.shuffle(info.train_cameras)
            random.shuffle(info.test_cameras)
        self.use_offDetector = bool(use_offDetector)
        self.train_cameras = [Camera(c, i, device, data_device, use_offDetector) for i, c in enumerate(info.train_cameras)]
        self.test_cameras = [Camera(c, i, device, data_device, use_offDetector) for i, c in enumerate(info.test_cameras)]
        self.vol_gt = torch.from_numpy(info.vol).float().to(device)
        self.scanner_cfg, self.scene_scale = info.scanner_cfg, info.scene_scale
        off, size = torch.tensor(self.scanner_cfg["offOrigin"]), torch.tensor(self.scanner_cfg["sVoxel"])
        self.bbox = torch.stack([off - size / 2, off + size / 2], dim=0)
        self.gaussians = None

    def getTrainCameras(self):
        return self.train_cameras

    def getTestCameras(self):
        return self.test_cameras

    def save(self, iteration, queryfunc):
        out = os.path.join(self.model_path, "point_cloud/iteration_{}".format(iteration))
        self.gaussians.save_ply(os.path.join(out, "point_cloud.pickle"))
        if queryfunc is not None:
            np.save(os.path.join(out, "vol_gt.npy"), self.vol_gt.detach().cpu().numpy())
            np.save(os.path.join(out, "vol_pred.npy"), queryfunc(self.gaussians)["vol"].detach().cpu().numpy())


def init_point_cloud(scanner_cfg: dict, n_points: int, recon: np.ndarray | None = None, density_thresh: float = 0.05,
                     density_rescale: float = 0.15, random_density_max: float = 1.0, rng=None) -> np.ndarray:
    """[n_points, 4] = (x, y, z, density).  `recon=None` -> uniform random cloud; else sample voxels of `recon` above
    `density_thresh` without replacement (`initialize_pcd.py:41-91`).  `rng` defaults to numpy's global generator,
    which the reference seeds with 0."""
    rnd = np.random if rng is None else rng
    off, size = np.asarray(scanner_cfg["offOrigin"], float), np.asarray(scanner_cfg["sVoxel"], float)
    if recon is None:
        xyz = off[None] + size[None] * (rnd.rand(n_points, 3) - 0.5)
        rho = rnd.rand(n_points) * random_density_max
    else:
        idx = np.argwhere(recon > density_thresh)
        if idx.shape[0] < n_points:
            raise ValueError("Valid voxels less than target number of sampling. Check threshold")
        pick = idx[rnd.choice(len(idx), n_points, replace=False)]
        xyz = pick * np.asarray(scanner_cfg["dVoxel"], float) - size / 2 + off
        rho = recon[pick[:, 0], pick[:, 1], pick[:, 2]] * density_rescale
    return np.concatenate([xyz, rho[:, None]], axis=-1)


def write_blender(path: str, scanner: dict, train: list, test: list, vol: np.ndarray):
    """Write a scene in the reference's directory format.  `train` / `test`: lists of (angle, projection[H,W]) in
    the scanner's own (unscaled) units, or (angle, projection, overrides) with a dict of the frame's per-view geometry
    (`scene.VIEW_KEYS`, unscaled); `scanner` as in `data_generator/synthetic_dataset/scanner/*.yml`."""
    os.makedirs(path, exist_ok=True)
    meta = {"scanner": scanner, "vol": "vol_gt.npy", "bbox": [[-1, -1, -1], [1, 1, 1]], "proj_train": [], "proj_test": []}
    np.save(os.path.join(path, "vol_gt.npy"), np.asarray(vol, dtype=np.float32))
    for split, frames in (("train", train), ("test", test)):
        os.makedirs(os.path.join(path, "proj_" + split), exist_ok=True)
        for i, (angle, proj, *overrides) in enumerate(frames):
            rel = os.path.join("proj_" + split, f"proj_{split}_{i:04d}.npy")
            np.save(os.path.join(path, rel), np.asarray(proj, dtype=np.float32))
            meta["proj_" + split].append({"file_path": rel, "angle": float(angle), **(overrides[0] if overrides else {})})
    with open(os.path.join(path, "meta_data.json"), "w") as f:
        json.dump(meta, f, indent=1)
