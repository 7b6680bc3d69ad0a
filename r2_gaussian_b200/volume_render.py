"""Volume rendering on the GPU: emission-absorption and MIP ray casting over the C ABI (r2x_volume_render,
csrc/r2x_volrender.cu).

    cam = default_camera(vol.shape, 800, 1000)                     # or look_at(position, focal_point, view_up, W, H)
    rgba = render(vol, cam, mode="composite", clim=(0, 1))         # CUDA float32 [1, H, W, 4]
    write_png("volume.png", to_uint8(rgba[0, ..., :3]))

The model, stated in full in include/r2x.h, works in index space: sample vol[i, j, k] sits at the point (i, j, k), the
convention of a numpy array wrapped by pyvista, so the reference's `plot_volume.py` camera positions can be passed
unchanged.  Rays march at `step` voxels through the trilinear field on [0, n-1]^3; the transfer function maps
t = clamp((v - c0) / (c1 - c0), 0, 1) to a colour from an RGB LUT and to opacity t (pyvista's "linear"); composite
rendering corrects the opacity for the step, 1 - (1 - t)^(step / opacity_unit), and composites front to back; MIP
colours the largest sampled value.  No shading, no jitter.  Parity with VTK's pixels is not claimed.  There is no CPU
fallback.
"""
from __future__ import annotations

import math
import struct
import zlib
from dataclasses import dataclass

import numpy as np

from .mesh import _device_volume

CAMERA_FLOATS = 16          # R2X_VR_CAMERA_FLOATS
MAX_LUT = 4096
MODES = {"composite": 0, "mip": 1}
GRAY = np.array([[0.0, 0.0, 0.0], [1.0, 1.0, 1.0]])


@dataclass(frozen=True)
class Camera:
    """A camera in index space, built by `look_at`: position P, focal point F, view-up U (as given), the frame
    f = normalize(F - P), r = normalize(f x U), u = r x f (float64), the image size and either a vertical view angle in
    degrees (perspective) or a parallel scale, half the image height in voxels (orthographic)."""
    position: tuple
    focal_point: tuple
    view_up: tuple
    width: int
    height: int
    view_angle: float
    parallel_scale: float | None
    f: np.ndarray
    r: np.ndarray
    u: np.ndarray

    @property
    def parallel(self) -> bool:
        return self.parallel_scale is not None

    @property
    def pitch(self) -> float:
        """Pixel pitch: 2 tan(view_angle / 2) / H (perspective, per unit distance) or 2 S / H (parallel, voxels)."""
        if self.parallel:
            return 2.0 * self.parallel_scale / self.height
        return 2.0 * math.tan(math.radians(self.view_angle) / 2.0) / self.height

    def record(self) -> np.ndarray:
        """The kernel's float32 camera record: P, f, r, u, pitch, 3 zeros."""
        rec = np.zeros(CAMERA_FLOATS, np.float64)
        rec[0:3], rec[3:6], rec[6:9], rec[9:12], rec[12] = self.position, self.f, self.r, self.u, self.pitch
        return rec.astype(np.float32)


def _vec3(v, what) -> np.ndarray:
    a = np.asarray(v, np.float64).reshape(-1)
    if a.shape != (3,) or not np.isfinite(a).all():
        raise ValueError(f"{what} must be 3 finite numbers, got {v}")
    return a


def look_at(position, focal_point, view_up, width: int, height: int, view_angle: float = 30.0,
            parallel_scale: float | None = None) -> Camera:
    """A camera at `position` looking at `focal_point` with `view_up` upwards (need not be unit length or orthogonal
    to the view direction, but must not be parallel to it).  `view_angle` is VTK's vertical view angle in degrees;
    with `parallel_scale` (half the image height in voxels) the projection is orthographic instead."""
    P, F, U = _vec3(position, "position"), _vec3(focal_point, "focal_point"), _vec3(view_up, "view_up")
    width, height = int(width), int(height)
    if width < 1 or height < 1:
        raise ValueError(f"the image must be at least 1 x 1 pixels, got {width} x {height}")
    if parallel_scale is not None:
        parallel_scale = float(parallel_scale)
        if not (math.isfinite(parallel_scale) and parallel_scale > 0):
            raise ValueError(f"parallel_scale must be finite and > 0, got {parallel_scale}")
    view_angle = float(view_angle)
    if not (0.0 < view_angle < 180.0):
        raise ValueError(f"view_angle must be in (0, 180) degrees, got {view_angle}")
    fv = F - P
    nf = float(np.linalg.norm(fv))
    if nf == 0.0:
        raise ValueError("the camera position equals its focal point: no view direction")
    f = fv / nf
    nu = float(np.linalg.norm(U))
    ru = np.cross(f, U)
    nr = float(np.linalg.norm(ru))
    if nu == 0.0 or nr <= 1e-12 * nu:
        raise ValueError(f"view_up {tuple(U)} is parallel to the view direction {tuple(f)}")
    r = ru / nr
    u = np.cross(r, f)
    return Camera(tuple(P.tolist()), tuple(F.tolist()), tuple(U.tolist()), width, height, view_angle, parallel_scale,
                  f, r, u)


def default_camera(shape, width: int, height: int, view_angle: float = 30.0,
                   parallel_scale: float | None = None) -> Camera:
    """Looks at the box centre from direction (1, 1, 1), view-up +z, at the distance where the box's bounding sphere
    (radius: the half diagonal) spans the vertical view angle: half-diagonal / sin(view_angle / 2).  With
    `parallel_scale` the projection is orthographic from the same position."""
    n = np.asarray([int(s) for s in shape], np.float64)
    if n.shape != (3,):
        raise ValueError(f"expected a 3-D shape, got {tuple(shape)}")
    centre = (n - 1) / 2
    dist = float(np.linalg.norm(n - 1)) / 2 / math.sin(math.radians(view_angle) / 2)
    pos = centre + dist * np.ones(3) / math.sqrt(3.0)
    return look_at(pos, centre, (0.0, 0.0, 1.0), width, height, view_angle, parallel_scale)


def orbit(camera: Camera, n: int) -> list:
    """n cameras; frame k's position is the camera's rotated by 360 k / n degrees about the axis through the focal
    point along the view-up (right-handed).  Focal point, view-up, image and projection are kept."""
    n = int(n)
    if n < 1:
        raise ValueError(f"an orbit needs at least 1 frame, got {n}")
    F = np.asarray(camera.focal_point, np.float64)
    k = np.asarray(camera.view_up, np.float64)
    k = k / np.linalg.norm(k)
    v = np.asarray(camera.position, np.float64) - F
    out = []
    for i in range(n):
        th = 2.0 * math.pi * i / n
        c, s = math.cos(th), math.sin(th)
        rot = v * c + np.cross(k, v) * s + k * float(k @ v) * (1.0 - c)     # Rodrigues
        out.append(look_at(F + rot, F, camera.view_up, camera.width, camera.height, camera.view_angle,
                           camera.parallel_scale))
    return out


def lut_from(cmap) -> np.ndarray:
    """A float64 [K, 3] LUT: "gray" (black -> white), a `.npy` path or an array, values in [0, 1], 1 <= K <= 4096."""
    if isinstance(cmap, str):
        if cmap == "gray":
            return GRAY.copy()
        if not cmap.endswith(".npy"):
            raise ValueError(f"cmap must be 'gray' or a .npy file of shape [K, 3], got {cmap!r}")
        cmap = np.load(cmap)
    lut = np.asarray(cmap)
    if lut.ndim != 2 or lut.shape[1] != 3 or not 1 <= lut.shape[0] <= MAX_LUT:
        raise ValueError(f"a LUT has shape [K, 3] with 1 <= K <= {MAX_LUT}, got {lut.shape}")
    if not np.issubdtype(lut.dtype, np.number) or np.iscomplexobj(lut):
        raise ValueError(f"a LUT holds real numbers, got {lut.dtype}")
    lut = lut.astype(np.float64)
    if not (np.isfinite(lut).all() and lut.min() >= 0.0 and lut.max() <= 1.0):
        raise ValueError("LUT values must be finite and in [0, 1]")
    return lut


def default_opacity_unit(shape) -> float:
    """The box diagonal over (mean axis size - 1): sqrt(3) voxels for a cube."""
    n = np.asarray([int(s) for s in shape], np.float64)
    return float(np.linalg.norm(n - 1) / (n.mean() - 1))


def _finite_f32(x) -> bool:
    with np.errstate(over="ignore"):
        return math.isfinite(float(x)) and math.isfinite(float(np.float32(x)))


def check_clim(clim) -> tuple:
    c0, c1 = (float(c) for c in clim)
    if not (_finite_f32(c0) and _finite_f32(c1) and np.float32(c0) < np.float32(c1)
            and _finite_f32(float(np.float32(c1)) - float(np.float32(c0)))):
        raise ValueError(f"clim must be two finite float32 values lo < hi, got {tuple(clim)}")
    return c0, c1


def render(volume, cameras, mode: str = "composite", clim=(0.0, 1.0), lut=None, step: float = 0.5,
           opacity_unit: float | None = None, background=(0.0, 0.0, 0.0)):
    """RGBA frames, CUDA float32 [N, H, W, 4], of `volume` (a CUDA or host tensor or array [nx, ny, nz], every axis
    >= 2) seen by `cameras` (one Camera or a list sharing the image size and projection), in one launch.  `lut` is
    anything `lut_from` takes (default gray); `opacity_unit` defaults to `default_opacity_unit`."""
    import torch

    from ._lib import check, load

    cams = [cameras] if isinstance(cameras, Camera) else list(cameras)
    if not cams or not all(isinstance(c, Camera) for c in cams):
        raise ValueError("render: cameras must be a Camera or a non-empty list of them")
    W, H, par = cams[0].width, cams[0].height, cams[0].parallel
    if any((c.width, c.height, c.parallel) != (W, H, par) for c in cams):
        raise ValueError("render: every camera of one call needs the same image size and projection")
    if mode not in MODES:
        raise ValueError(f"render: mode must be one of {sorted(MODES)}, got {mode!r}")
    c0, c1 = check_clim(clim)
    table = lut_from("gray" if lut is None else lut)
    step = float(step)
    if not (_finite_f32(step) and step > 0):
        raise ValueError(f"render: step must be a finite float > 0, got {step}")
    shape = tuple(int(s) for s in np.shape(volume))
    if len(shape) != 3 or min(shape) < 2:
        raise ValueError(f"render: expected a [nx, ny, nz] volume with every axis >= 2 samples, got shape {shape}")
    unit = default_opacity_unit(shape) if opacity_unit is None else float(opacity_unit)
    if not (_finite_f32(unit) and unit > 0):
        raise ValueError(f"render: opacity_unit must be a finite float > 0, got {unit}")
    bg = np.asarray(background, np.float32).reshape(-1)
    if bg.shape != (3,) or not np.isfinite(bg).all():
        raise ValueError(f"render: background must be 3 finite numbers, got {background}")
    diag = float(np.linalg.norm(np.asarray(shape, np.float64) - 1))
    if diag / float(np.float32(step)) > 2**31 - 1:
        raise ValueError(f"render: step {step} puts more than 2^31 - 1 samples on the box diagonal")
    v = _device_volume(volume, what="render")
    nx, ny, nz = shape
    lib = load()
    with torch.cuda.device(v.device):
        stream = torch.cuda.current_stream(v.device).cuda_stream
        rec = torch.from_numpy(np.stack([c.record() for c in cams])).to(v.device)
        lut_d = torch.from_numpy(table.astype(np.float32)).to(v.device)
        out = torch.empty((len(cams), H, W, 4), dtype=torch.float32, device=v.device)
        check(lib.r2x_volume_render(stream, nx, ny, nz, v.data_ptr(), len(cams), H, W, rec.data_ptr(), int(par),
                                    MODES[mode], c0, c1, lut_d.data_ptr(), len(table), step, unit,
                                    bg.ctypes.data, out.data_ptr()), "r2x_volume_render")
    return out


def to_uint8(rgb):
    """floor(255 clamp(c, 0, 1) + 1/2) as uint8, in the input's precision; a torch tensor stays on its device."""
    if hasattr(rgb, "detach"):
        import torch
        x = rgb.detach()
        return torch.floor(x.clamp(0, 1) * 255 + 0.5).to(torch.uint8)
    x = np.asarray(rgb)
    if not np.issubdtype(x.dtype, np.floating):
        x = x.astype(np.float64)
    return np.floor(np.clip(x, 0, 1) * x.dtype.type(255) + x.dtype.type(0.5)).astype(np.uint8)


def _chunk(kind: bytes, data: bytes) -> bytes:
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)


def write_png(path: str, rgb_uint8) -> None:
    """An 8-bit RGB PNG of a uint8 [H, W, 3] image (numpy or tensor): one IDAT, filter 0 on every row."""
    img = rgb_uint8.detach().cpu().numpy() if hasattr(rgb_uint8, "detach") else np.asarray(rgb_uint8)
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] != 3 or img.shape[0] < 1 or img.shape[1] < 1:
        raise ValueError(f"write_png: expected a uint8 [H, W, 3] image, got {img.dtype} {img.shape}")
    h, w = img.shape[:2]
    raw = np.zeros((h, 1 + 3 * w), np.uint8)
    raw[:, 1:] = img.reshape(h, 3 * w)
    png = (b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0))
           + _chunk(b"IDAT", zlib.compress(raw.tobytes(), 6)) + _chunk(b"IEND", b""))
    with open(path, "wb") as fh:
        fh.write(png)
