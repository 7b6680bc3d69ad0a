"""Pose corrections without a GPU: the matrix-gradient entry point rejects bad arguments before any CUDA call, and
`PoseCorrection` reproduces the camera at zero, matches a float64 restatement of its exponential map and carries
matrix gradients to its parameters as central finite differences say."""
import ctypes
import math
import types

import numpy as np
import pytest
import scipy.linalg
import torch

from r2_gaussian_b200 import _lib, scene
from r2_gaussian_b200.pose import PoseCorrection, se3_exp


def _camera(mode=1, angle=0.7, dtype=torch.float32):
    """A camera as `dataset.Camera` builds it (matrices on the CPU)."""
    sc = scene.cone_beam_scanner(64, 64) if mode == 1 else scene.parallel_beam_scanner(64, 64)
    v = scene.make_view(sc, angle)
    wvt = torch.tensor(v.viewmatrix, dtype=dtype)
    proj = torch.tensor(scene.projection_matrix(v.FoVx, v.FoVy, v.mode).T.copy(), dtype=dtype)
    full = wvt.unsqueeze(0).bmm(proj.unsqueeze(0)).squeeze(0).contiguous()
    return types.SimpleNamespace(world_view_transform=wvt, projection_matrix=proj, full_proj_transform=full,
                                 camera_center=torch.tensor(v.campos, dtype=dtype), image_height=v.image_height,
                                 image_width=v.image_width, FoVx=v.FoVx, FoVy=v.FoVy, mode=v.mode)


# ---- C entry point: argument checks ---------------------------------------------------------------------------------

def _call(lib, P=10, R=0, W=16, H=16, view=1, proj=1, gview=1, gproj=1, pose_scratch=1, pose_bytes=None, act=None,
          cov=None, scales=1, rots=1):
    p = ctypes.c_void_p
    if pose_bytes is None:
        pose_bytes = lib.r2x_raster_backward_pose_scratch_bytes(P)
    nz = lambda x: None if x is None else p(0x1000 * x)   # never dereferenced: the checks come first
    return lib.r2x_raster_backward_pose(
        None, P, R, W, H, nz(1), nz(scales), 1.0, nz(rots), nz(cov), nz(view), nz(proj), None, 1.0, 1.0, None, None,
        None, None, None, None, None, None, None, None, None, None, None, 1, 0, act, nz(gview), nz(gproj),
        nz(pose_scratch), pose_bytes)


@pytest.mark.parametrize("kw,msg", [
    (dict(P=-1), b"bad sizes"), (dict(W=0), b"bad sizes"), (dict(H=-3), b"bad sizes"), (dict(R=-1), b"bad sizes"),
    (dict(view=None), b"null matrix"), (dict(proj=None), b"null matrix"), (dict(gview=None), b"null matrix"),
    (dict(gproj=None), b"null matrix"), (dict(pose_scratch=None), b"pose_scratch"),
    (dict(pose_bytes=8), b"pose_scratch"),
    (dict(act="x", cov=1), b"raw parameters"), (dict(act="x", scales=None), b"raw parameters"),
])
def test_pose_entry_rejects_bad_arguments_before_cuda(kw, msg):
    lib = _lib.load()
    if kw.get("act") == "x":
        kw["act"] = ctypes.byref(_lib.ActivationDesc(0, 0.0, 0.0))
    rc = _call(lib, **kw)
    assert rc == 1, rc
    err = lib.r2x_last_error()
    assert b"r2x_raster_backward_pose" in err and msg in err, err


def test_pose_scratch_grows_with_P():
    lib = _lib.load()
    a, b = lib.r2x_raster_backward_pose_scratch_bytes(256), lib.r2x_raster_backward_pose_scratch_bytes(100_000)
    assert a >= 24 * 4 and b >= math.ceil(100_000 / 256) * 24 * 4 and b > a
    assert lib.r2x_raster_backward_pose_scratch_bytes(0) >= 24 * 4


# ---- PoseCorrection --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", [0, 1])
def test_zero_correction_reproduces_the_camera_bit_for_bit(mode):
    cam = _camera(mode)
    corr = PoseCorrection(3)
    for i in range(3):
        c = corr(cam, i)
        for name in ("world_view_transform", "full_proj_transform"):
            got, want = getattr(c, name), getattr(cam, name)
            assert got.dtype == want.dtype and got.shape == want.shape
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), name
            assert got.requires_grad
        assert c.image_width == cam.image_width and c.mode == cam.mode and c.FoVx == cam.FoVx


def _expm_reference(omega, nu):
    """exp of the twist in float64: Rodrigues for the rotation, the SE(3) left Jacobian for the translation."""
    w = np.asarray(omega, np.float64)
    th = np.linalg.norm(w)
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    if th == 0:
        R, V = np.eye(3), np.eye(3)
    else:
        R = np.eye(3) + math.sin(th) / th * K + (1 - math.cos(th)) / th ** 2 * K @ K
        V = np.eye(3) + (1 - math.cos(th)) / th ** 2 * K + (th - math.sin(th)) / th ** 3 * K @ K
    E = np.eye(4)
    E[:3, :3], E[:3, 3] = R, V @ np.asarray(nu, np.float64)
    return E


@pytest.mark.parametrize("scale", [0.0, 1e-6, 1e-3, 0.05, 0.3, 2.0])
def test_exponential_map_matches_float64_restatement(scale):
    rng = np.random.RandomState(int(scale * 1000) + 1)
    for _ in range(4):
        w, n = rng.randn(3) * scale, rng.randn(3)
        twist = np.zeros((4, 4))
        twist[:3, :3] = [[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]
        twist[:3, 3] = n
        want = scipy.linalg.expm(twist)
        if np.linalg.norm(w) == 0 or np.linalg.norm(w) > 1e-3:   # the closed forms cancel catastrophically in between
            np.testing.assert_allclose(_expm_reference(w, n), want, rtol=0, atol=1e-12)
        got64 = se3_exp(torch.tensor(w), torch.tensor(n)).numpy()
        np.testing.assert_allclose(got64, want, rtol=0, atol=1e-13)
        got32 = se3_exp(torch.tensor(w, dtype=torch.float32), torch.tensor(n, dtype=torch.float32)).numpy()
        np.testing.assert_allclose(got32, want, rtol=0, atol=4e-6 * max(1.0, np.abs(n).max()))


@pytest.mark.parametrize("mode", [0, 1])
def test_correction_applies_a_left_perturbation(mode):
    cam = _camera(mode, dtype=torch.float64)
    corr = PoseCorrection(2, dtype=torch.float64)
    with torch.no_grad():
        corr.omega[1] = torch.tensor([0.01, -0.02, 0.015])
        corr.nu[1] = torch.tensor([0.03, 0.01, -0.05])
    c = corr(cam, 1)
    T = cam.world_view_transform.numpy().T
    E = _expm_reference(corr.omega[1].detach().numpy(), corr.nu[1].detach().numpy())
    np.testing.assert_allclose(c.world_view_transform.detach().numpy(), (E @ T).T, rtol=0, atol=1e-12)
    full = (E @ T).T @ cam.projection_matrix.numpy()
    np.testing.assert_allclose(c.full_proj_transform.detach().numpy(), full, rtol=0, atol=1e-12)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("at_zero", [True, False])
def test_parameter_gradient_matches_central_differences(mode, at_zero):
    """A fixed linear functional of both matrices stands in for the rasterizer's dL/dmatrices."""
    cam = _camera(mode, dtype=torch.float64)
    rng = np.random.RandomState(3 + mode)
    Gv, Gp = torch.tensor(rng.randn(4, 4)), torch.tensor(rng.randn(4, 4))
    corr = PoseCorrection(3, dtype=torch.float64)
    if not at_zero:
        with torch.no_grad():
            corr.omega.copy_(torch.tensor(rng.randn(3, 3) * 0.2))
            corr.nu.copy_(torch.tensor(rng.randn(3, 3) * 0.1))

    def loss():
        c = corr(cam, 2)
        return (c.world_view_transform * Gv).sum() + (c.full_proj_transform * Gp).sum()

    corr.zero_grad()
    loss().backward()
    for p in (corr.omega, corr.nu):
        assert torch.count_nonzero(p.grad[:2]) == 0
        fd = torch.zeros(3, dtype=torch.float64)
        h = 1e-6
        for k in range(3):
            with torch.no_grad():
                p[2, k] += h
                up = loss().item()
                p[2, k] -= 2 * h
                dn = loss().item()
                p[2, k] += h
            fd[k] = (up - dn) / (2 * h)
        np.testing.assert_allclose(p.grad[2].numpy(), fd.numpy(), rtol=1e-6, atol=1e-7 * float(fd.abs().max()))
