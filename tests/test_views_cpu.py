"""Batched views without a GPU: the C ABI exports the calls, sizes its buffers linearly in the number of views and
rejects bad arguments before any CUDA call; the Python entry points check shapes before touching the device."""
import ctypes
import os
import types

import pytest
import torch

from r2_gaussian_b200 import _lib
from r2_gaussian_b200.rasterization import GaussianRasterizationSettings, rasterize_views
from r2_gaussian_b200.render_query import render_views

NEW = ["r2x_raster_views_geom_bytes", "r2x_raster_views_image_bytes", "r2x_raster_forward_views_async",
       "r2x_raster_backward_views"]


def _lib_handle():
    return _lib.load()


def test_abi_exports_the_views_calls():
    lib = ctypes.CDLL(_lib.LIB_PATH) if os.path.exists(_lib.LIB_PATH) else _lib.load()
    for name in NEW:
        assert hasattr(lib, name) and name in _lib.PROTOTYPES


def _padded(P):
    return (max(P, 1) + 255) // 256 * 256


@pytest.mark.parametrize("P,N", [(1, 1), (255, 3), (256, 3), (257, 7), (100_000, 8), (50_000, 50)])
def test_geometry_is_one_record_set_per_view_padded_to_a_cta(P, N):
    """View v's Gaussians are the virtual Gaussians [v Pp, (v + 1) Pp), Pp = P rounded up to 256."""
    lib = _lib_handle()
    assert lib.r2x_raster_views_geom_bytes(P, N) == lib.r2x_raster_geom_bytes(N * _padded(P))


def test_one_view_has_the_single_view_image_layout():
    lib = _lib_handle()
    for P, W, H in ((1, 16, 16), (3000, 100, 100), (100_000, 512, 512), (1500, 1040, 1040)):
        assert lib.r2x_raster_views_image_bytes(P, 1, W, H) == lib.r2x_raster_image_bytes(_padded(P), W, H)


def test_image_state_grows_linearly_in_the_views():
    """The direct path's per-CTA tile table only covers each CTA's own band: N views cost about N times one view
    (a table over the whole stacked grid would cost N^2)."""
    lib = _lib_handle()
    P, W, H = 50_000, 256, 256                        # 256 tiles per view: direct binning up to N = 16
    one = lib.r2x_raster_views_image_bytes(P, 1, W, H)
    for N in (2, 4, 8, 16):
        b = lib.r2x_raster_views_image_bytes(P, N, W, H)
        assert N * one * 0.9 <= b <= N * one * 1.1, (N, b, one)
    # beyond 4096 tiles (radix path) the image buffer holds the tile ranges and the work plan only
    b17, b34 = lib.r2x_raster_views_image_bytes(P, 17, W, H), lib.r2x_raster_views_image_bytes(P, 34, W, H)
    assert b17 < lib.r2x_raster_views_image_bytes(P, 16, W, H) and 1.8 * b17 <= b34 <= 2.2 * b17


def _fwd(lib, P=10, N=2, W=64, H=64, ptr=None, binning=None, cap=0):
    return lib.r2x_raster_forward_views_async(None, P, N, W, H, ptr, ptr, ptr, 1.0, ptr, ptr, ptr, 1.0, 1.0, 1, ptr,
                                              ptr, ptr, ptr, binning, cap, None)


def test_abi_rejects_bad_arguments_before_any_cuda_call():
    lib = _lib_handle()
    fake = ctypes.c_void_p(1 << 20)   # never dereferenced: every case fails its checks first
    assert _fwd(lib, N=0, ptr=fake, binning=fake) != 0 and b"bad N" in lib.r2x_last_error()
    assert _fwd(lib, N=-3, ptr=fake, binning=fake) != 0 and b"bad N" in lib.r2x_last_error()
    # 4097 views of 16 tile rows: 65552 stacked tile rows > 65535
    assert _fwd(lib, N=4097, H=256, ptr=fake, binning=fake) != 0 and b"tile rows" in lib.r2x_last_error()
    assert _fwd(lib, W=0, ptr=fake, binning=fake) != 0 and b"bad P/W/H" in lib.r2x_last_error()
    assert _fwd(lib, ptr=None, binning=fake) != 0 and b"null" in lib.r2x_last_error()
    assert _fwd(lib, ptr=fake, binning=None) != 0 and b"binning" in lib.r2x_last_error()
    rc = lib.r2x_raster_backward_views(None, 10, 0, 100, 64, 64, fake, fake, 1.0, fake, fake, fake, 1.0, 1.0, fake,
                                       fake, fake, fake, fake, fake, fake, fake, fake, fake, fake, fake, 1, 0)
    assert rc != 0 and b"bad N" in lib.r2x_last_error()
    rc = lib.r2x_raster_backward_views(None, 10, 2, 100, 64, 64, fake, fake, 1.0, fake, None, fake, 1.0, 1.0, fake,
                                       fake, fake, fake, fake, fake, fake, fake, fake, fake, fake, fake, 1, 0)
    assert rc != 0 and b"null" in lib.r2x_last_error()
    assert lib.r2x_raster_views_geom_bytes(10, 0) == 0 and lib.r2x_raster_views_image_bytes(10, 0, 64, 64) == 0


def _settings():
    eye = torch.eye(4)
    return GaussianRasterizationSettings(64, 64, 1.0, 1.0, 1.0, eye, eye, torch.zeros(3), False, 1, False)


def _cloud(P=5):
    return torch.zeros(P, 3), torch.ones(P, 1), torch.ones(P, 3), torch.ones(P, 4)


def test_python_checks_shapes_before_the_device():
    m, d, s, r = _cloud()
    eye = torch.eye(4)
    with pytest.raises(ValueError, match="viewmatrices"):
        rasterize_views(m, d, s, r, eye, eye, _settings())                         # not [N,4,4]
    with pytest.raises(ValueError, match="viewmatrices"):
        rasterize_views(m, d, s, r, eye[None][:0], eye[None][:0], _settings())     # N = 0
    with pytest.raises(ValueError, match="projmatrices"):
        rasterize_views(m, d, s, r, eye.expand(3, 4, 4), eye.expand(2, 4, 4), _settings())
    with pytest.raises(ValueError, match="means2D"):
        rasterize_views(m, d, s, r, eye.expand(3, 4, 4), eye.expand(3, 4, 4), _settings(), means2D=torch.zeros(5, 3))
    with pytest.raises(ValueError, match="scales and rotations"):
        rasterize_views(m, d, None, r, eye.expand(3, 4, 4), eye.expand(3, 4, 4), _settings())
    with pytest.raises(RuntimeError, match="CUDA tensor"):                        # right shapes, host tensors
        rasterize_views(m, d, s, r, eye.expand(3, 4, 4).clone(), eye.expand(3, 4, 4).clone(), _settings())


def test_render_views_checks_the_cameras_first():
    def cam(h=64, mode=1, fov=0.5):
        return types.SimpleNamespace(image_height=h, image_width=64, FoVx=fov, FoVy=fov, mode=mode,
                                     world_view_transform=torch.eye(4), full_proj_transform=torch.eye(4),
                                     camera_center=torch.zeros(3))
    m, d, s, r = _cloud()
    pc = types.SimpleNamespace(get_xyz=m, get_density=d, get_scaling=s, get_rotation=r)
    pipe = types.SimpleNamespace(debug=False, compute_cov3D_python=False)
    with pytest.raises(ValueError, match="no camera"):
        render_views([], pc, pipe)
    for other in (cam(h=32), cam(mode=0), cam(fov=0.6)):
        with pytest.raises(ValueError, match="share"):
            render_views([cam(), other], pc, pipe)
    with pytest.raises(ValueError, match="compute_cov3D_python"):
        render_views([cam()], pc, types.SimpleNamespace(debug=False, compute_cov3D_python=True))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        render_views([cam(), cam()], pc, pipe)
