"""ctypes binding of libr2xray.so (C ABI in include/r2x.h).

There is NO fallback: if the shared library is missing or does not export every symbol the header
declares, importing the compute path raises.  `R2X_AUTOBUILD=1` (default) compiles it with nvcc when
the in-tree library is absent or stale.
"""
from __future__ import annotations

import ctypes as C
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libr2xray.so")

ALLOC_FN = C.CFUNCTYPE(C.c_void_p, C.c_size_t, C.c_void_p)

_vp, _i, _f, _ll, _sz = C.c_void_p, C.c_int, C.c_float, C.c_longlong, C.c_size_t

# name -> (restype, argtypes); kept in the order of include/r2x.h
PROTOTYPES = {
    "r2x_last_error": (C.c_char_p, []),
    "r2x_version": (_i, []),
    "r2x_raster_geom_bytes": (_sz, [_i]),
    "r2x_raster_image_bytes": (_sz, [_i, _i, _i]),
    "r2x_voxel_geom_bytes": (_sz, [_i]),
    "r2x_voxel_image_bytes": (_sz, [_i, _i, _i, _i]),
    "r2x_binning_bytes": (_sz, [_ll]),
    "r2x_raster_bwd_scratch_bytes": (_sz, [_ll]),
    "r2x_voxel_bwd_scratch_bytes": (_sz, [_ll]),
    "r2x_raster_forward": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp, _f, _f, _i, _i,
                                _vp, _vp, _vp, _vp, ALLOC_FN, _vp, _i, C.POINTER(_i)]),
    "r2x_raster_forward_async": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp, _f, _f, _i, _i,
                                      _vp, _vp, _vp, _vp, _vp, _ll, _vp]),
    "r2x_raster_backward": (_i, [_vp, _i, _ll, _i, _i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp, _f, _f, _vp,
                                 _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i]),
    "r2x_raster_views_geom_bytes": (_sz, [_i, _i]),
    "r2x_raster_views_image_bytes": (_sz, [_i, _i, _i, _i]),
    "r2x_raster_forward_views_async": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _f, _vp, _vp, _vp, _f, _f, _i, _vp, _vp,
                                            _vp, _vp, _vp, _ll, _vp]),
    "r2x_raster_backward_views": (_i, [_vp, _i, _i, _ll, _i, _i, _vp, _vp, _f, _vp, _vp, _vp, _f, _f, _vp, _vp, _vp, _vp,
                                       _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i]),
    "r2x_raster_render_only": (_i, [_vp, _i, _i, _i, _ll, _vp, _vp, _vp, _vp]),
    "r2x_voxel_render_only": (_i, [_vp, _i, _i, _i, _i, _ll, _vp, _vp, _vp, _vp]),
    "r2x_mark_visible": (_i, [_vp, _i, _vp, _vp, _vp, _vp]),
    "r2x_raster_export": (_i, [_vp, _i, _i, _i, _ll, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "r2x_voxel_forward": (_i, [_vp, _i, _i, _i, _i, _f, _f, _f, _f, _f, _f, _vp, _vp, _vp, _f, _vp, _vp, _i,
                               _vp, _vp, _vp, _vp, _vp, _vp, ALLOC_FN, _vp, _i, C.POINTER(_i)]),
    "r2x_voxel_forward_async": (_i, [_vp, _i, _i, _i, _i, _f, _f, _f, _f, _f, _f, _vp, _vp, _vp, _f, _vp, _vp, _i,
                                     _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ll, _vp]),
    "r2x_voxel_backward": (_i, [_vp, _i, _ll, _i, _i, _i, _f, _f, _f, _f, _f, _f, _vp, _vp, _f, _vp, _vp,
                                _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i]),
    "r2x_voxel_export": (_i, [_vp, _i, _i, _i, _i, _ll, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "r2x_knn_scratch_bytes": (_sz, [_i]),
    "r2x_knn3_mean_dist2": (_i, [_vp, _i, _vp, _vp, _vp, _sz]),
    "r2x_image_loss_scratch_bytes": (_sz, [_i, _i]),
    "r2x_image_loss": (_i, [_vp, _i, _i, _vp, _vp, _f, _f, _vp, _vp, _vp, _sz]),
    "r2x_image_loss_views_scratch_bytes": (_sz, [_i, _i, _i]),
    "r2x_image_loss_views": (_i, [_vp, _i, _i, _i, _vp, _vp, _f, _f, _vp, _vp, _vp, _sz]),
    "r2x_tv3d_scratch_bytes": (_sz, [_i, _i, _i]),
    "r2x_tv3d_loss": (_i, [_vp, _i, _i, _i, _vp, _i, _vp, _vp, _vp, _sz]),
    "r2x_adam_step": (_i, [_vp, _i, _vp, C.c_double, C.c_double, C.c_double, _ll]),
    "r2x_adam_step_sum": (_i, [_vp, _i, _vp, _vp, C.c_double, C.c_double, C.c_double, _ll, _vp, _vp]),
    "r2x_densify_stats": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "r2x_densify_stats_views": (_i, [_vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "r2x_raster_forward_async_raw": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _f, _vp, _vp, _vp, _vp, _f, _f, _i, _vp, _vp, _vp, _vp,
                                          _vp, _ll, _vp, _vp]),
    "r2x_raster_backward_raw": (_i, [_vp, _i, _ll, _i, _i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _f, _f, _vp, _vp, _vp, _vp, _vp,
                                     _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp]),
    "r2x_raster_forward_views_async_raw": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _f, _vp, _vp, _vp, _f, _f, _i, _vp,
                                                _vp, _vp, _vp, _vp, _ll, _vp, _vp]),
    "r2x_raster_backward_views_raw": (_i, [_vp, _i, _i, _ll, _i, _i, _vp, _vp, _f, _vp, _vp, _vp, _f, _f, _vp, _vp, _vp,
                                           _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _vp]),
    "r2x_raster_backward_pose_scratch_bytes": (_sz, [_i]),
    "r2x_raster_backward_pose": (_i, [_vp, _i, _ll, _i, _i, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp, _f, _f, _vp,
                                      _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i,
                                      _vp, _vp, _vp, _vp, _sz]),
    "r2x_pose_apply": (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "r2x_pose_grad": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "r2x_detector_offset_apply": (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    "r2x_detector_offset_grad_scratch_bytes": (_sz, [_i, _i]),
    "r2x_detector_offset_grad": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _sz]),
    "r2x_detector_offset_cost_scratch_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "r2x_detector_offset_cost": (_i, [_vp, _i, _i, _i, _i, _vp, _i, _vp, _vp, C.c_double, C.c_double, C.c_double, _i,
                                      _i, _i, _vp, _vp, _vp, _vp, _vp, _sz]),
    "r2x_voxel_forward_async_raw": (_i, [_vp, _i, _i, _i, _i, _f, _f, _f, _f, _f, _f, _vp, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp,
                                         _vp, _vp, _vp, _ll, _vp, _vp]),
    "r2x_voxel_backward_raw": (_i, [_vp, _i, _ll, _i, _i, _i, _f, _f, _f, _f, _f, _f, _vp, _vp, _f, _vp, _vp, _vp, _vp, _vp, _vp,
                                    _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "r2x_mask_select_scratch_bytes": (_sz, [_i]),
    "r2x_mask_select": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _sz]),
    "r2x_gather_rows": (_i, [_vp, _i, _vp, _vp, _ll]),
    "r2x_fdk_scratch_bytes": (_sz, [_i, _i, _i]),
    "r2x_fdk": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _f, _f, _i, _f, _f, _i, _vp, _f, _f, _i, _i, _i, _f, _f, _f, _f, _f,
                     _f, _vp, _vp, _sz]),
    "r2x_fdk_pad": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _f, _f, _i, _f, _f, _i, _vp, _f, _f, _i, _i, _i, _f, _f, _f, _f,
                         _f, _f, _vp, _vp, _sz, _i]),
    "r2x_fdk_filter": (_i, [_vp, _i, _i, _i, _vp, _f, _f, _i, _f, _vp]),
    "r2x_fdk_backproject": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _i, _f, _i, _i, _i, _f, _f, _f, _f, _f, _f, _vp]),
    "r2x_volume_project": (_i, [_vp, _i, _i, _i, _vp, _f, _f, _f, _f, _f, _f, _i, _i, _i, _vp, _f, _f, _i, _f, _f, _f,
                                _vp]),
    "r2x_volume_backproject_scratch_bytes": (_sz, [_i, _i, _i]),
    "r2x_volume_backproject": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _f, _f, _i, _f, _f, _i, _i, _i, _f, _f, _f, _f, _f,
                                    _f, _f, _vp, _vp, _vp, _sz]),
    "r2x_fdk_views": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _f, _f, _f, _f, _f, _vp, _vp, _vp, _vp,
                           _sz]),
    "r2x_fdk_helical": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _f, _f, _i, _i, _f, _vp, _vp, _vp, C.c_double, C.c_double,
                             C.c_double, C.c_double, C.c_double, C.c_double, _f, _i, _i, _i, _f, _f, _f, _f, _f, _f, _vp,
                             _vp, _sz]),
    "r2x_volume_project_views": (_i, [_vp, _i, _i, _i, _vp, _f, _f, _f, _f, _f, _f, _i, _i, _i, _vp, _i, _f, _vp, _vp,
                                      _vp]),
    "r2x_volume_backproject_views": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _i, _i, _i, _i, _f, _f, _f, _f, _f, _f, _f,
                                          _vp, _vp, _vp, _vp, _vp, _sz]),
    "r2x_tv_prox_scratch_bytes": (_sz, [_i, _i, _i]),
    "r2x_tv_prox": (_i, [_vp, _i, _i, _i, _vp, _f, _i, _i, _vp, _vp, _sz]),
    "r2x_tv_value_scratch_bytes": (_sz, [_i, _i, _i]),
    "r2x_tv_value": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _sz]),
    "r2x_tv_cp_step": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _f, _f, _f, _i, _vp, _vp, _vp]),
    "r2x_projection_prepare_shape": (_i, [_i, _i, _i, C.POINTER(_i)]),
    "r2x_projection_prepare": (_i, [_vp, _i, _i, _i, _i, _vp, C.c_double, C.c_double, _vp]),
    "r2x_zoom_workspace_bytes": (_sz, [_i, _i, _i]),
    "r2x_volume_place": (_i, [_vp, _vp, _vp]),
    "r2x_zoom_cubic": (_i, [_vp, _vp, _i, _i, _i, _vp, _sz, _vp]),
    "r2x_marching_cubes_table": (_i, [_vp, _vp]),
    "r2x_marching_cubes_scratch_bytes": (_sz, [_i, _i, _i]),
    "r2x_marching_cubes_count": (_i, [_vp, _i, _i, _i, _vp, _f, _vp, _vp, _sz]),
    "r2x_marching_cubes_emit": (_i, [_vp, _i, _i, _i, _vp, _f, _ll, _ll, _vp, _vp, _vp, _sz]),
    "r2x_volume_render": (_i, [_vp, _i, _i, _i, _vp, _i, _i, _i, _vp, _i, _i, _f, _f, _vp, _i, _f, _f, _vp, _vp]),
    "r2x_scene_raster_scratch_bytes": (_sz, [_i, _i]),
    "r2x_scene_raster": (_i, [_vp, _i, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _i, _i, _i, _i, _vp, _i, C.c_double, _vp,
                              _vp, _vp, _vp, _sz]),
    "r2x_peer_alloc": (_i, [_sz, C.POINTER(_vp)]),
    "r2x_peer_free": (_i, [_vp]),
    "r2x_ipc_export": (_i, [_vp, _vp]),
    "r2x_ipc_open": (_i, [_vp, C.POINTER(_vp)]),
    "r2x_ipc_close": (_i, [_vp]),
    "r2x_peer_allreduce_sum": (_i, [_vp, _i, _i, _vp, _vp, C.c_uint32, _vp, _ll, _vp]),
    "r2x_peer_allreduce_sum_t": (_i, [_vp, _i, _i, _vp, _vp, C.c_uint32, _vp, _ll, _vp, _ll]),
}


class ActivationDesc(C.Structure):
    """Mirror of `r2x_activation` (include/r2x.h)."""
    _fields_ = [("scale_mode", C.c_int), ("scale_lo", C.c_float), ("scale_hi", C.c_float)]


class GatherDesc(C.Structure):
    """Mirror of `r2x_gather_desc` (include/r2x.h)."""
    _fields_ = [("src0", C.c_void_p), ("src1", C.c_void_p), ("dst", C.c_void_p), ("n0", C.c_longlong), ("width", C.c_int)]


class AdamGroup(C.Structure):
    """Mirror of `r2x_adam_group` (include/r2x.h)."""
    _fields_ = [("param", C.c_void_p), ("grad", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p),
                ("numel", C.c_longlong), ("lr", C.c_float)]

class PlaceDesc(C.Structure):
    """Mirror of `r2x_place_desc` (include/r2x.h)."""
    _fields_ = [("src", C.c_void_p), ("dtype", C.c_int), ("src_shape", C.c_int * 3), ("src_strides", C.c_longlong * 3),
                ("shape", C.c_int * 3), ("offset", C.c_int * 3), ("lo", C.c_double), ("hi", C.c_double)]

_lock = threading.Lock()
_lib = None


class R2XError(RuntimeError):
    pass


def load(autobuild: bool | None = None):
    """Load (building first if allowed and needed) and return the ctypes library handle."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if autobuild is None:
            autobuild = os.environ.get("R2X_AUTOBUILD", "1") != "0"
        if autobuild:
            from . import build as _build
            try:
                if _build.needs_build():
                    _build.build()
            except Exception as e:  # no nvcc on this box: use the prebuilt library if there is one
                if not os.path.exists(LIB_PATH):
                    raise R2XError(f"libr2xray.so is missing and could not be built: {e}") from e
        if not os.path.exists(LIB_PATH):
            raise R2XError(
                f"{LIB_PATH} not found. Build it with `python -m r2_gaussian_b200.build` "
                "(needs nvcc); there is no CPU fallback."
            )
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in PROTOTYPES.items():
            try:
                fn = getattr(lib, name)
            except AttributeError as e:
                raise R2XError(f"libr2xray.so does not export {name}; rebuild it") from e
            fn.restype = res
            fn.argtypes = args
        _lib = lib
        return _lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().r2x_last_error()
        raise R2XError(f"{what} failed (code {rc}): {msg.decode() if msg else '?'}")
