"""Synthetic CT scenes: scanner geometry, cameras and Gaussian clouds (NumPy, host side).

Restates the reference's geometry conventions so tests and bench.py can build inputs without the
reference or any dataset:
  * scanner = data_generator/synthetic_dataset/scanner/cone_beam.yml:2-33 (DSD 7, DSO 5, 512^2
    detector of size 4x4, volume 2^3 at 256^3); scene scale 2/max(sVoxel) = 1
    (r2_gaussian/dataset/dataset_readers.py:63).
  * camera pose  = angle2pose (dataset_readers.py:156-191), R/T split (:120-127),
    getWorld2View2 + getProjectionMatrix (utils/graphics_utils.py:81-139), matrices stored transposed
    and multiplied as in dataset/cameras.py:66-84 (so the flat arrays are column-major).
  * Gaussians "init-like" = initialize_pcd.py:50-58 (uniform positions / densities, seed 0) with
    isotropic scales from the mean squared distance to the 3 nearest neighbours
    (gaussian/gaussian_model.py:145-156); "trained-like" perturbs scales and rotations (SURVEY.md 8d).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

MODE_PARALLEL = 0
MODE_CONE = 1


def cone_beam_scanner(n_detector: int = 512, n_voxel: int = 256) -> dict:
    return {
        "mode": "cone", "DSD": 7.0, "DSO": 5.0,
        "nDetector": [n_detector, n_detector], "sDetector": [4.0, 4.0],
        "nVoxel": [n_voxel, n_voxel, n_voxel], "sVoxel": [2.0, 2.0, 2.0],
        "offOrigin": [0.0, 0.0, 0.0], "offDetector": [0.0, 0.0],
    }


def parallel_beam_scanner(n_detector: int = 512, n_voxel: int = 256) -> dict:
    s = cone_beam_scanner(n_detector, n_voxel)
    s["mode"] = "parallel"
    s["sDetector"] = [2.0, 2.0]
    return s


def angle2pose(DSO: float, angle: float) -> np.ndarray:
    """Camera-to-world of the source at `angle` on a circle of radius DSO around z."""
    c1, s1 = math.cos(-math.pi / 2), math.sin(-math.pi / 2)
    R1 = np.array([[1.0, 0.0, 0.0], [0.0, c1, -s1], [0.0, s1, c1]])
    c2, s2 = math.cos(math.pi / 2), math.sin(math.pi / 2)
    R2 = np.array([[c2, -s2, 0.0], [s2, c2, 0.0], [0.0, 0.0, 1.0]])
    ca, sa = math.cos(angle), math.sin(angle)
    R3 = np.array([[ca, -sa, 0.0], [sa, ca, 0.0], [0.0, 0.0, 1.0]])
    T = np.eye(4)
    T[:3, :3] = R3 @ R2 @ R1
    T[:3, 3] = [DSO * ca, DSO * sa, 0.0]
    return T


def projection_matrix(fovx: float, fovy: float, mode: int) -> np.ndarray:
    if mode == MODE_PARALLEL:
        return np.eye(4, dtype=np.float32)
    znear, zfar = 0.01, 100.0
    top = math.tan(fovy / 2) * znear
    right = math.tan(fovx / 2) * znear
    P = np.zeros((4, 4), dtype=np.float32)
    P[0, 0] = 2.0 * znear / (2 * right)
    P[1, 1] = 2.0 * znear / (2 * top)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def detector_shift(scanner_cfg: dict) -> tuple[float, float]:
    """(t_u, t_v): the scanner's `offDetector` in detector pixels, t_u = offDetector[0] / dDetector_u and
    t_v = offDetector[1] / dDetector_v with dDetector_u = sDetector[1] / nDetector[1], dDetector_v = sDetector[0] /
    nDetector[0] (scanner files store nDetector / sDetector as [v, u] but offDetector as [u, v]; only ratios are used,
    so any consistent units do).  A missing offDetector is (0, 0).

    Convention: image pixel (row r, column c) sees the ray that the centred detector has at fractional pixel
    (r - t_v, c + t_u).  In ndc the pixel centre (2c + 1) / W - 1 gains 2 t_u / W and the row's (2r + 1) / H - 1 loses
    2 t_v / H; in the camera intrinsics the x row of the projection matrix (math sense) gains -(2 t_u / W) times its w
    row and the y row +(2 t_v / H) times it (`shifted_projection_matrix`).

    Derivation.  TIGRE (which the reference hands `geo.offDetector = [offDetector[1], offDetector[0]]`,
    r2_gaussian/utils/ct_utils.py::get_geometry_tigre) places detector column iu at
    u = dDetector_u (iu - n_u / 2 + 0.5) + offDetector_u, and image columns run along u: column c holds the ray of the
    centred detector's column c + t_u.  This is the horizontal convention of `detector.py`, with
    `DetectorOffset` s = -t_u (offDetector[0] = -s dDetector_u).  Row iv sits at v = dDetector_v (iv - n_v / 2 + 0.5) +
    offDetector_v, and the reference hands TIGRE `projs[:, ::-1, :]`, so image row r is iv = n_v - 1 - r: row r holds
    the ray of the centred detector's row r - t_v.  The vertical sign rests on that flip and has not been checked
    against TIGRE itself."""
    off = scanner_cfg.get("offDetector", [0.0, 0.0])
    du = float(scanner_cfg["sDetector"][1]) / float(scanner_cfg["nDetector"][1])
    dv = float(scanner_cfg["sDetector"][0]) / float(scanner_cfg["nDetector"][0])
    return float(off[0]) / du, float(off[1]) / dv


def shifted_projection_matrix(P: np.ndarray, t_u: float, t_v: float, W: int, H: int) -> np.ndarray:
    """P' (math sense, float32) of a detector offset by (t_u, t_v) pixels: the x row gains -(2 t_u / W) times the w row
    and the y row +(2 t_v / H) times it, in float64 rounded once.  Cone beam changes P[0,2] and P[1,2] (w row
    (0, 0, 1, 0)), parallel beam P[0,3] and P[1,3] (P = I).  Zero shifts return P unchanged."""
    if t_u == 0.0 and t_v == 0.0:
        return P
    Q = np.asarray(P, np.float64).copy()
    Q[0] -= (2.0 * t_u / W) * Q[3]
    Q[1] += (2.0 * t_v / H) * Q[3]
    return Q.astype(np.float32)


@dataclass
class View:
    """One projection geometry in the layout the rasterizer expects."""
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    viewmatrix: np.ndarray   # [4,4] float32 = world->view, TRANSPOSED (flat == column-major)
    projmatrix: np.ndarray   # [4,4] float32 = view @ proj in the transposed convention
    campos: np.ndarray       # [3]
    mode: int
    angle: float = 0.0
    FoVx: float = 0.0
    FoVy: float = 0.0


# the keys a projection frame of meta_data.json may carry to override the scanner for that view (scanner units)
VIEW_KEYS = ("DSO", "DSD", "offOrigin", "offDetector")


def view_scanner(scanner: dict, frame: dict) -> dict:
    """The scanner of one view: a copy of `scanner` with the frame's `VIEW_KEYS` overrides.  `DSO`, `DSD` and
    `offDetector` replace the scanner's.  The frame's `offOrigin` is where the volume sits during the view (TIGRE's
    per-angle `geo.offOrigin`); the reconstruction grid stays at the scanner's `offOrigin`, so it goes to
    `offOrigin_view` and `camera_pose` translates the camera by offOrigin - offOrigin_view.  A view_scanner dict is a
    valid frame: its own `offOrigin_view` (else `offOrigin`) is taken as the view's."""
    cfg = dict(scanner)
    for k in ("DSO", "DSD"):
        if k in frame:
            cfg[k] = float(frame[k])
    if "offDetector" in frame:
        cfg["offDetector"] = [float(v) for v in frame["offDetector"]]
    pos = frame.get("offOrigin_view", frame.get("offOrigin"))
    if pos is not None:
        cfg["offOrigin_view"] = [float(v) for v in pos]
    return cfg


def camera_pose(scanner: dict, angle: float) -> np.ndarray:
    """Camera-to-world of the view at `angle`: `angle2pose` at the scanner's DSO, translated by offOrigin -
    offOrigin_view when `view_scanner` set a volume position (a zero translation changes no bit)."""
    c2w = angle2pose(scanner["DSO"], angle)
    if "offOrigin_view" in scanner:
        t = (np.asarray(scanner["offOrigin"], np.float64) - np.asarray(scanner["offOrigin_view"], np.float64))
        if np.any(t != 0.0):
            c2w[:3, 3] += t
    return c2w


def make_view(scanner: dict, angle: float, use_offDetector: bool = False) -> View:
    """The view at `angle`.  `use_offDetector` puts the scanner's offDetector into the projection matrix
    (`detector_shift`, `shifted_projection_matrix`); off, or with a zero offset, the view is bit for bit the centred
    one.  A `view_scanner` dict gives that view's camera (`camera_pose`)."""
    mode = MODE_CONE if scanner["mode"] == "cone" else MODE_PARALLEL
    c2w = camera_pose(scanner, angle)
    w2c = np.linalg.inv(c2w)
    R = w2c[:3, :3].T  # stored transposed, dataset_readers.py:123-125
    T = w2c[:3, 3]
    Rt = np.zeros((4, 4))
    Rt[:3, :3] = R.T
    Rt[:3, 3] = T
    Rt[3, 3] = 1.0
    Rt = np.float32(np.linalg.inv(np.linalg.inv(Rt)))  # getWorld2View2 with zero translate, unit scale
    fovx = math.atan2(scanner["sDetector"][1] / 2, scanner["DSD"]) * 2
    fovy = math.atan2(scanner["sDetector"][0] / 2, scanner["DSD"]) * 2
    view_t = np.ascontiguousarray(Rt.T.astype(np.float32))
    P = projection_matrix(fovx, fovy, mode)
    if use_offDetector:
        P = shifted_projection_matrix(P, *detector_shift(scanner), int(scanner["nDetector"][1]),
                                      int(scanner["nDetector"][0]))
    proj_t = np.ascontiguousarray(P.T.astype(np.float32))
    full = (view_t.astype(np.float32) @ proj_t.astype(np.float32)).astype(np.float32)
    campos = np.linalg.inv(view_t.astype(np.float64))[3, :3].astype(np.float32)
    if mode == MODE_PARALLEL:
        tx = ty = 1.0
    else:
        tx, ty = math.tan(fovx * 0.5), math.tan(fovy * 0.5)
    return View(int(scanner["nDetector"][0]), int(scanner["nDetector"][1]), tx, ty, view_t,
                np.ascontiguousarray(full), campos, mode, angle, fovx, fovy)


def camera_from_view(view: View, device="cuda"):
    """The attributes render() reads from the reference's `Camera` (`r2_gaussian/dataset/cameras.py:20-70`:
    world_view_transform, full_proj_transform, camera_center, FoVx/FoVy, image size, mode) as device tensors."""
    import types

    import torch
    return types.SimpleNamespace(
        image_height=view.image_height, image_width=view.image_width, FoVx=view.FoVx, FoVy=view.FoVy, mode=view.mode,
        world_view_transform=torch.tensor(view.viewmatrix, device=device),
        full_proj_transform=torch.tensor(view.projmatrix, device=device),
        camera_center=torch.tensor(view.campos, device=device), angle=view.angle)


def make_views(scanner: dict, n_views: int = 50) -> list[View]:
    """Angles linspace(0, 2pi, n+1)[:-1] (data_generator/synthetic_dataset/generate_data.py:47-50)."""
    angles = np.linspace(0.0, 2.0 * math.pi, n_views + 1)[:-1]
    return [make_view(scanner, float(a)) for a in angles]


@dataclass
class Cloud:
    """Activated Gaussian parameters (what render()/query() hand to the extension)."""
    means: np.ndarray      # [P,3] float32
    scales: np.ndarray     # [P,3] float32
    rotations: np.ndarray  # [P,4] float32 (r,x,y,z), normalised
    density: np.ndarray    # [P,1] float32
    meta: dict = field(default_factory=dict)

    @property
    def P(self) -> int:
        return int(self.means.shape[0])


def knn3_mean_sq_dist(xyz: np.ndarray) -> np.ndarray:
    """simple_knn.distCUDA2 semantics: mean squared distance to the 3 nearest neighbours."""
    from scipy.spatial import cKDTree

    tree = cKDTree(xyz.astype(np.float64))
    k = min(4, xyz.shape[0])
    d, _ = tree.query(xyz.astype(np.float64), k=k, workers=-1)
    d = np.atleast_2d(d)
    if k < 2:
        return np.zeros(xyz.shape[0], dtype=np.float32)
    return (d[:, 1:] ** 2).mean(axis=1).astype(np.float32)


def make_cloud(P: int, kind: str = "init", seed: int = 0, s_voxel=(2.0, 2.0, 2.0), density_scale: float = 1.0,
               scale_bound=(0.001, 1.0)) -> Cloud:
    rng = np.random.RandomState(seed)
    s_voxel = np.asarray(s_voxel, dtype=np.float64)
    xyz = (s_voxel * (rng.rand(P, 3) - 0.5)).astype(np.float32)
    dens = (rng.rand(P, 1) * density_scale).astype(np.float32)
    dist2 = np.maximum(knn3_mean_sq_dist(xyz), 1e-6)
    iso = np.sqrt(dist2).astype(np.float32)
    # scale_bound = [scale_min, scale_max] * max(sVoxel) = [0.001, 1.0] for the 2^3 volume (train.py:59-61);
    # create_from_pcd clamps to [lo + EPS, hi - EPS] (gaussian_model.py:152-155)
    lo, hi = scale_bound[0] + 1e-5, scale_bound[1] - 1e-5
    iso = np.clip(iso, lo, hi)
    scales = np.repeat(iso[:, None], 3, axis=1).astype(np.float32)
    rots = np.zeros((P, 4), dtype=np.float32)
    rots[:, 0] = 1.0
    if kind == "trained":
        scales = (scales * rng.uniform(0.5, 1.5, size=(P, 3))).astype(np.float32)
        scales = np.clip(scales, lo, hi).astype(np.float32)
        q = rng.randn(P, 4)
        q /= np.linalg.norm(q, axis=1, keepdims=True)
        rots = q.astype(np.float32)
    elif kind != "init":
        raise ValueError(f"unknown cloud kind {kind!r}")
    return Cloud(xyz, scales, rots, dens, {"kind": kind, "seed": seed})


def shard_cloud(cloud: Cloud, rank: int, world: int) -> Cloud:
    """Contiguous index partition of the Gaussians (SURVEY.md 8e): rank r owns [r*P/world, (r+1)*P/world)."""
    P = cloud.P
    lo = (P * rank) // world
    hi = (P * (rank + 1)) // world
    return Cloud(cloud.means[lo:hi].copy(), cloud.scales[lo:hi].copy(), cloud.rotations[lo:hi].copy(),
                 cloud.density[lo:hi].copy(), dict(cloud.meta, shard=(rank, world)))
