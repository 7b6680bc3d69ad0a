"""Per-view pose corrections, fitted through the rasterizer's view- and projection-matrix gradients.

Real scans are not exact: detector shifts, gantry angles and source / detector mounting carry errors that the
dataset files do not record.  `PoseCorrection(n_views)` holds one small rigid correction per view and hands
`render()` cameras whose matrices depend on it, so `loss.backward()` reaches the corrections (with the scene
trainable or frozen).

Convention.  A camera's `world_view_transform` is T^T, where T is the 4x4 world -> camera transform acting on column
vectors (x_cam = T x_world); the rasterizer reads the 16 floats column-major, as the reference stores them.  View i
carries a twist xi_i = (omega_i, nu_i) (rotation vector, translation; both [3], zero at start) and is corrected by a
LEFT perturbation in the camera frame:

    T_i' = exp(xi_i) T_i,   exp(xi) = [[R, V nu], [0, 1]],
    R = I + a K + b K^2,    V = I + b K + c K^2,    K = [omega]_x,   theta = |omega|,
    a = sin(theta) / theta,  b = (1 - cos(theta)) / theta^2,  c = (theta - sin(theta)) / theta^3

(Rodrigues' formula and the SE(3) left Jacobian V; the series of a, b, c is used below theta = 0.1).  So omega rotates
the camera frame about its own axes and nu moves it along them, in scene units.  The corrected camera has

    world_view_transform' = T_i'^T
    full_proj_transform'  = T_i'^T projection_matrix     (the camera's own, as `dataset.Camera` forms it)

both computed with torch ops from (omega_i, nu_i), so autograd carries dL/d(matrices) from the rasterizer to the
parameters.  With zero correction both matrices equal the camera's bit for bit.

`PoseCorrection.device_camera(cam, i, anchor)` is the same map as two small device kernels (libr2xray's
`r2x_pose_apply` / `r2x_pose_grad`): the matrices come from a float64 evaluation rounded once, and the backward is the
exact chain rule through it.  It replaces ~30 torch ops forward and as many backward with one launch each, and it is
what both training paths use (`NativeTrainStep(pose=...)` calls the kernels directly; `trainer --pose_refine`).  Its
gradient rows are written in full, with the `anchor` view's row held at 0: a rigid motion of the scene together with
every camera leaves every image unchanged, so one view fixes the frame.

Pose gradients are not supported together with Gaussian sharding (`sharded.enable`); intrinsics (tan_fovx, detector
offsets) stay as given.
"""
from __future__ import annotations

import copy

import torch
from torch import nn

from ._lib import check, load


def hat(w: torch.Tensor) -> torch.Tensor:
    """[..., 3] -> [..., 3, 3] cross-product matrix: hat(w) @ v = w x v."""
    z = torch.zeros_like(w[..., 0])
    return torch.stack([torch.stack([z, -w[..., 2], w[..., 1]], -1),
                        torch.stack([w[..., 2], z, -w[..., 0]], -1),
                        torch.stack([-w[..., 1], w[..., 0], z], -1)], -2)


def _coefficients(theta2: torch.Tensor):
    """(a, b, c) of the module docstring as functions of theta^2, with finite gradients at theta = 0."""
    small = theta2 < 1e-2
    t2 = torch.where(small, torch.ones_like(theta2), theta2)
    t = torch.sqrt(t2)
    s, co = torch.sin(t), torch.cos(t)
    x = theta2   # Taylor series to theta^6: truncation below 3e-14 for theta^2 < 1e-2
    a = torch.where(small, 1 - x / 6 * (1 - x / 20 * (1 - x / 42)), s / t)
    b = torch.where(small, 0.5 - x / 24 * (1 - x / 30 * (1 - x / 56)), (1 - co) / t2)
    c = torch.where(small, 1.0 / 6 - x / 120 * (1 - x / 42 * (1 - x / 72)), (t - s) / (t2 * t))
    return a, b, c


def se3_exp_minus_identity(omega: torch.Tensor, nu: torch.Tensor) -> torch.Tensor:
    """exp([omega, nu]) - I as a [..., 4, 4] matrix (formed directly, so small twists lose no precision)."""
    K = hat(omega)
    K2 = K @ K
    a, b, c = _coefficients((omega * omega).sum(-1))
    a, b, c = a[..., None, None], b[..., None, None], c[..., None, None]
    eye = torch.eye(3, dtype=omega.dtype, device=omega.device)
    rot = a * K + b * K2                                   # R - I
    trans = ((eye + b * K + c * K2) @ nu[..., None])[..., 0]   # V nu
    out = torch.zeros(omega.shape[:-1] + (4, 4), dtype=omega.dtype, device=omega.device)
    out[..., :3, :3] = rot
    out[..., :3, 3] = trans
    return out


def se3_exp(omega: torch.Tensor, nu: torch.Tensor) -> torch.Tensor:
    """exp([omega, nu]) as a [..., 4, 4] matrix."""
    return torch.eye(4, dtype=omega.dtype, device=omega.device) + se3_exp_minus_identity(omega, nu)


def _as_negative_zero(z: torch.Tensor) -> torch.Tensor:
    """z with every zero turned into -0.0 (other values and the gradient unchanged), so that x + result == x bit for
    bit wherever z == 0: x + (-0.0) is x for every x, x + (+0.0) is not for x = -0.0."""
    return -((-z) + 0.0)


class PoseCorrection(nn.Module):
    """Per-view rigid corrections: `omega` and `nu` ([n_views, 3], zeros), see the module docstring."""

    def __init__(self, n_views: int, device=None, dtype=torch.float32):
        super().__init__()
        self.omega = nn.Parameter(torch.zeros(int(n_views), 3, device=device, dtype=dtype))
        self.nu = nn.Parameter(torch.zeros(int(n_views), 3, device=device, dtype=dtype))

    def matrices(self, cam, i: int) -> tuple[torch.Tensor, torch.Tensor]:
        """(world_view_transform', full_proj_transform') of view `i` for camera `cam`, differentiable in omega, nu."""
        dt = self.omega.dtype
        wvt = cam.world_view_transform.to(dt)
        full = cam.full_proj_transform.to(dt)
        proj = cam.projection_matrix.to(dt)
        d = se3_exp_minus_identity(self.omega[i], self.nu[i])     # exp(xi) - I
        d_wvt = _as_negative_zero(wvt @ d.transpose(0, 1))         # (exp(xi) T)^T - T^T
        return wvt + d_wvt, full + _as_negative_zero(d_wvt @ proj)

    def forward(self, cam, i: int):
        """A copy of `cam` (same attributes) whose matrices carry correction `i`."""
        view, full = self.matrices(cam, i)
        out = copy.copy(cam)
        out.world_view_transform = view
        out.full_proj_transform = full
        out.camera_center = torch.linalg.inv(view.detach())[3, :3].contiguous()
        return out

    def device_camera(self, cam, i: int, anchor: int = 0):
        """A copy of `cam` whose matrices carry correction `i`, formed by the device kernels (module docstring):
        differentiable in omega / nu, whose gradient rows other than `i` -- and row `anchor` (-1: none) always -- are
        0.  float32 CUDA parameters only.  `camera_center` stays the camera's own (the rasterizer never reads it)."""
        view, full = _DevicePose.apply(self.omega, self.nu, int(i), int(anchor), cam.world_view_transform,
                                       cam.full_proj_transform, cam.projection_matrix)
        out = copy.copy(cam)
        out.world_view_transform = view
        out.full_proj_transform = full
        return out


def _matrix(t: torch.Tensor, dev) -> torch.Tensor:
    if t.dtype != torch.float32 or t.device != dev or not t.is_contiguous():
        t = t.to(device=dev, dtype=torch.float32).contiguous()
    if t.numel() != 16:
        raise ValueError("PoseCorrection.device_camera: camera matrices must have 16 entries")
    return t


class _DevicePose(torch.autograd.Function):
    """(omega, nu) -> (world_view_transform', full_proj_transform') of view i through r2x_pose_apply / r2x_pose_grad."""

    @staticmethod
    def forward(ctx, omega, nu, i, anchor, wvt, full, proj):
        for name, p in (("omega", omega), ("nu", nu)):
            if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous() or p.dim() != 2 or p.shape[1] != 3:
                raise RuntimeError(f"PoseCorrection.device_camera: {name} must be a contiguous float32 CUDA [n_views, 3]")
        dev = omega.device
        wvt, full, proj = _matrix(wvt, dev), _matrix(full, dev), _matrix(proj, dev)
        lib = load()
        with torch.cuda.device(dev):
            view_out = torch.empty((4, 4), dtype=torch.float32, device=dev)
            full_out = torch.empty((4, 4), dtype=torch.float32, device=dev)
            check(lib.r2x_pose_apply(torch.cuda.current_stream(dev).cuda_stream, omega.data_ptr(), nu.data_ptr(),
                                     int(omega.shape[0]), i, wvt.data_ptr(), full.data_ptr(), proj.data_ptr(),
                                     view_out.data_ptr(), full_out.data_ptr()), "r2x_pose_apply")
        ctx.i, ctx.anchor = i, anchor
        ctx.save_for_backward(omega, nu, wvt, proj)
        return view_out, full_out

    @staticmethod
    def backward(ctx, g_view, g_full):
        omega, nu, wvt, proj = ctx.saved_tensors
        dev = omega.device
        zero = lambda: torch.zeros((4, 4), dtype=torch.float32, device=dev)
        g_view = zero() if g_view is None else _matrix(g_view, dev)
        g_full = zero() if g_full is None else _matrix(g_full, dev)
        lib = load()
        with torch.cuda.device(dev):
            g_omega, g_nu = torch.empty_like(omega), torch.empty_like(nu)
            check(lib.r2x_pose_grad(torch.cuda.current_stream(dev).cuda_stream, omega.data_ptr(), nu.data_ptr(),
                                    int(omega.shape[0]), ctx.i, ctx.anchor, wvt.data_ptr(), proj.data_ptr(),
                                    g_view.data_ptr(), g_full.data_ptr(), g_omega.data_ptr(), g_nu.data_ptr()),
                  "r2x_pose_grad")
        return g_omega, g_nu, None, None, None, None, None
