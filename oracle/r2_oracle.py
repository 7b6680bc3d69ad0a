"""ctypes wrapper of the CPU oracle (oracle/r2_oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
reference legs -- never by the product package.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libr2oracle.so")
_lib = None

_f = np.float32
_fp = C.POINTER(C.c_float)
_ip = C.POINTER(C.c_int)
_up = C.POINTER(C.c_uint32)
_u64p = C.POINTER(C.c_uint64)


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "r2_oracle.c")
    if force or not os.path.exists(LIB_PATH) or os.path.getmtime(src) > os.path.getmtime(LIB_PATH):
        cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
        cmd = [cc, "-O2", "-fPIC", "-shared", "-std=c11", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-mavx2",
               "-fopenmp", "-o", LIB_PATH, src, "-lm"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"oracle build failed:\n{r.stderr}")
    return LIB_PATH


def lib():
    global _lib
    if _lib is None:
        try:
            build()
        except Exception:
            if not os.path.exists(LIB_PATH):
                raise
        _lib = C.CDLL(LIB_PATH)
        _lib.orc_raster_forward.restype = C.c_longlong
        _lib.orc_voxel_forward.restype = C.c_longlong
        _lib.orc_raster_preprocess.restype = C.c_longlong
        _lib.orc_voxel_preprocess.restype = C.c_longlong
        _lib.orc_num_threads.restype = C.c_int
    return _lib


def _c(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype)


def _p(a, ptype):
    return None if a is None else a.ctypes.data_as(ptype)


def num_threads() -> int:
    return int(lib().orc_num_threads())


def set_num_threads(n: int):
    lib().orc_set_num_threads(C.c_int(int(n)))


def _take(ptr, n, dtype):
    """Copy n items out of a malloc'ed C array and free it."""
    if n == 0:
        lib().orc_free(ptr)
        return np.zeros(0, dtype=dtype)
    arr = np.ctypeslib.as_array(ptr, shape=(n,)).astype(dtype, copy=True)
    lib().orc_free(ptr)
    return arr


def raster_forward(means, scales, rots, opac, view, proj, W, H, tanfovx, tanfovy, mode, scale_modifier=1.0,
                   cov3D_precomp=None, render=True):
    """Reference forward on the CPU.  Returns a dict of every stage output."""
    L = lib()
    means = _c(means, _f).reshape(-1, 3); P = means.shape[0]
    opac = _c(opac, _f).reshape(-1)
    scales = None if scales is None else _c(scales, _f).reshape(-1, 3)
    rots = None if rots is None else _c(rots, _f).reshape(-1, 4)
    cov_pre = None if cov3D_precomp is None else _c(cov3D_precomp, _f).reshape(-1, 6)
    view = _c(view, _f).reshape(16); proj = _c(proj, _f).reshape(16)
    out = dict(
        image=np.zeros((H, W), _f), radii=np.zeros(P, np.int32), xy=np.zeros((P, 2), _f), depth=np.zeros(P, _f),
        cov3D=np.zeros((P, 6), _f), conic_opacity=np.zeros((P, 4), _f), mu=np.zeros(P, _f),
        tiles_touched=np.zeros(P, np.uint32), rect=np.zeros((P, 4), np.int32), n_contrib=np.zeros((H, W), np.uint32))
    gx, gy = (W + 15) // 16, (H + 15) // 16
    if not render:
        R = L.orc_raster_preprocess(
            C.c_int(P), _p(means, _fp), _p(scales, _fp), C.c_float(scale_modifier), _p(rots, _fp), _p(opac, _fp),
            _p(cov_pre, _fp), _p(view, _fp), _p(proj, _fp), C.c_int(W), C.c_int(H), C.c_float(tanfovx),
            C.c_float(tanfovy), C.c_int(mode), _p(out["radii"], _ip), _p(out["xy"], _fp), _p(out["depth"], _fp),
            _p(out["cov3D"], _fp), _p(out["conic_opacity"], _fp), _p(out["mu"], _fp), _p(out["tiles_touched"], _up),
            _p(out["rect"], _ip))
        out["R"] = int(R)
        return out
    kp, vp, rp = _u64p(), _up(), _up()
    R = L.orc_raster_forward(
        C.c_int(P), _p(means, _fp), _p(scales, _fp), C.c_float(scale_modifier), _p(rots, _fp), _p(opac, _fp),
        _p(cov_pre, _fp), _p(view, _fp), _p(proj, _fp), C.c_int(W), C.c_int(H), C.c_float(tanfovx),
        C.c_float(tanfovy), C.c_int(mode), _p(out["image"], _fp), _p(out["radii"], _ip), _p(out["xy"], _fp),
        _p(out["depth"], _fp), _p(out["cov3D"], _fp), _p(out["conic_opacity"], _fp), _p(out["mu"], _fp),
        _p(out["tiles_touched"], _up), _p(out["rect"], _ip), _p(out["n_contrib"], _up), C.byref(kp), C.byref(vp),
        C.byref(rp))
    R = int(R)
    out["R"] = R
    out["keys"] = _take(kp, R, np.uint64)
    out["point_list"] = _take(vp, R, np.uint32)
    out["ranges"] = _take(rp, gx * gy * 2, np.uint32).reshape(gx * gy, 2)
    return out


def raster_backward(fwd, means, scales, rots, view, proj, W, H, tanfovx, tanfovy, mode, dL_dpix,
                    scale_modifier=1.0, cov3D_precomp=None):
    """Reference backward on the CPU from a `raster_forward` result."""
    L = lib()
    means = _c(means, _f).reshape(-1, 3); P = means.shape[0]
    scales = None if scales is None else _c(scales, _f).reshape(-1, 3)
    rots = None if rots is None else _c(rots, _f).reshape(-1, 4)
    view = _c(view, _f).reshape(16); proj = _c(proj, _f).reshape(16)
    dL = _c(dL_dpix, _f).reshape(H, W)
    g = dict(dL_dmean2D=np.zeros((P, 3), _f), dL_dconic=np.zeros((P, 4), _f), dL_dopacity=np.zeros((P, 1), _f),
             dL_dmu=np.zeros((P, 1), _f), dL_dmean3D=np.zeros((P, 3), _f), dL_dcov3D=np.zeros((P, 6), _f),
             dL_dscale=np.zeros((P, 3), _f), dL_drot=np.zeros((P, 4), _f))
    ranges = _c(fwd["ranges"], np.uint32); pl = _c(fwd["point_list"], np.uint32)
    L.orc_raster_render_backward(
        C.c_int(W), C.c_int(H), C.c_int(P), _p(ranges, _up), _p(pl, _up), _p(fwd["xy"], _fp),
        _p(fwd["conic_opacity"], _fp), _p(fwd["mu"], _fp), _p(dL, _fp), _p(g["dL_dmean2D"], _fp),
        _p(g["dL_dconic"], _fp), _p(g["dL_dopacity"], _fp), _p(g["dL_dmu"], _fp))
    cov = fwd["cov3D"] if cov3D_precomp is None else _c(cov3D_precomp, _f)
    L.orc_raster_preprocess_backward(
        C.c_int(P), _p(means, _fp), _p(fwd["radii"], _ip), _p(scales, _fp), C.c_float(scale_modifier), _p(rots, _fp),
        _p(cov, _fp), C.c_int(0 if cov3D_precomp is not None else 1), _p(view, _fp), _p(proj, _fp), C.c_int(W),
        C.c_int(H), C.c_float(tanfovx), C.c_float(tanfovy), C.c_int(mode), _p(g["dL_dmean2D"], _fp),
        _p(g["dL_dconic"], _fp), _p(g["dL_dmu"], _fp), _p(g["dL_dmean3D"], _fp), _p(g["dL_dcov3D"], _fp),
        _p(g["dL_dscale"], _fp), _p(g["dL_drot"], _fp))
    return g


def voxel_forward(means, scales, rots, opac, nVoxel, sVoxel, center, scale_modifier=1.0, cov3D_precomp=None,
                  render=True):
    L = lib()
    means = _c(means, _f).reshape(-1, 3); P = means.shape[0]
    opac = _c(opac, _f).reshape(-1)
    scales = _c(scales, _f).reshape(-1, 3)
    rots = None if rots is None else _c(rots, _f).reshape(-1, 4)
    cov_pre = None if cov3D_precomp is None else _c(cov3D_precomp, _f).reshape(-1, 6)
    nx, ny, nz = (int(v) for v in nVoxel)
    out = dict(
        vol=np.zeros((nx, ny, nz), _f), radii_x=np.zeros(P, np.int32), radii_y=np.zeros(P, np.int32),
        radii_z=np.zeros(P, np.int32), xyz_vol=np.zeros((P, 3), _f), depth=np.zeros(P, _f), cov3D=np.zeros((P, 6), _f),
        conic_opacity=np.zeros((P, 7), _f), tiles_touched=np.zeros(P, np.uint32), cube=np.zeros((P, 6), np.int32),
        n_contrib=np.zeros((nx, ny, nz), np.uint32))
    gx, gy, gz = (nx + 7) // 8, (ny + 7) // 8, (nz + 7) // 8
    common = [C.c_int(P), _p(means, _fp), _p(scales, _fp), C.c_float(scale_modifier), _p(rots, _fp), _p(opac, _fp),
              _p(cov_pre, _fp), C.c_int(nx), C.c_int(ny), C.c_int(nz), C.c_float(sVoxel[0]), C.c_float(sVoxel[1]),
              C.c_float(sVoxel[2]), C.c_float(center[0]), C.c_float(center[1]), C.c_float(center[2])]
    state = [_p(out["radii_x"], _ip), _p(out["radii_y"], _ip), _p(out["radii_z"], _ip), _p(out["xyz_vol"], _fp),
             _p(out["depth"], _fp), _p(out["cov3D"], _fp), _p(out["conic_opacity"], _fp),
             _p(out["tiles_touched"], _up), _p(out["cube"], _ip)]
    if not render:
        out["R"] = int(L.orc_voxel_preprocess(*common, *state))
        return out
    kp, vp, rp = _u64p(), _up(), _up()
    R = int(L.orc_voxel_forward(*common, _p(out["vol"], _fp), *state, _p(out["n_contrib"], _up), C.byref(kp),
                                C.byref(vp), C.byref(rp)))
    out["R"] = R
    out["keys"] = _take(kp, R, np.uint64)
    out["point_list"] = _take(vp, R, np.uint32)
    out["ranges"] = _take(rp, gx * gy * gz * 2, np.uint32).reshape(gx * gy * gz, 2)
    return out


def voxel_backward(fwd, scales, rots, nVoxel, sVoxel, dL_dvol, scale_modifier=1.0, cov3D_precomp=None):
    L = lib()
    P = fwd["radii_x"].shape[0]
    scales = _c(scales, _f).reshape(-1, 3)
    rots = None if rots is None else _c(rots, _f).reshape(-1, 4)
    nx, ny, nz = (int(v) for v in nVoxel)
    dL = _c(dL_dvol, _f).reshape(nx, ny, nz)
    g = dict(dL_dmean3D_norm=np.zeros((P, 3), _f), dL_dconic3D=np.zeros((P, 6), _f), dL_dopacity=np.zeros((P, 1), _f),
             dL_dmean3D=np.zeros((P, 3), _f), dL_dcov3D=np.zeros((P, 6), _f), dL_dscale=np.zeros((P, 3), _f),
             dL_drot=np.zeros((P, 4), _f))
    ranges = _c(fwd["ranges"], np.uint32); pl = _c(fwd["point_list"], np.uint32)
    L.orc_voxel_render_backward(
        C.c_int(P), C.c_int(nx), C.c_int(ny), C.c_int(nz), C.c_float(sVoxel[0]), C.c_float(sVoxel[1]),
        C.c_float(sVoxel[2]), _p(ranges, _up), _p(pl, _up), _p(fwd["xyz_vol"], _fp), _p(fwd["conic_opacity"], _fp),
        _p(dL, _fp), _p(g["dL_dmean3D_norm"], _fp), _p(g["dL_dconic3D"], _fp), _p(g["dL_dopacity"], _fp))
    cov = fwd["cov3D"] if cov3D_precomp is None else _c(cov3D_precomp, _f)
    L.orc_voxel_preprocess_backward(
        C.c_int(P), _p(fwd["radii_x"], _ip), _p(fwd["radii_y"], _ip), _p(fwd["radii_z"], _ip), _p(scales, _fp),
        C.c_float(scale_modifier), _p(rots, _fp), _p(cov, _fp), C.c_int(0 if cov3D_precomp is not None else 1),
        C.c_int(nx), C.c_int(ny), C.c_int(nz), C.c_float(sVoxel[0]), C.c_float(sVoxel[1]), C.c_float(sVoxel[2]),
        _p(g["dL_dmean3D_norm"], _fp), _p(g["dL_dconic3D"], _fp), _p(g["dL_dmean3D"], _fp), _p(g["dL_dcov3D"], _fp),
        _p(g["dL_dscale"], _fp), _p(g["dL_drot"], _fp))
    return g


def mark_visible(means, view, proj):
    means = _c(means, _f).reshape(-1, 3)
    present = np.zeros(means.shape[0], np.uint8)
    lib().orc_mark_visible(C.c_int(means.shape[0]), _p(means, _fp), _p(_c(view, _f).reshape(16), _fp),
                           _p(_c(proj, _f).reshape(16), _fp), present.ctypes.data_as(C.POINTER(C.c_ubyte)))
    return present.astype(bool)


def knn3_mean_dist2(points):
    """Brute-force restatement of simple_knn._C.distCUDA2 (see orc_knn3_mean_dist2)."""
    pts = _c(points, _f).reshape(-1, 3)
    out = np.zeros(pts.shape[0], _f)
    with np.errstate(over="ignore"):
        lib().orc_knn3_mean_dist2(C.c_int(pts.shape[0]), _p(pts, _fp), _p(out, _fp))
    return out


def knn3_mean_dist2_at(points, idx):
    """knn3_mean_dist2(points)[idx], computed for the points `idx` only (see orc_knn3_mean_dist2_at)."""
    pts = _c(points, _f).reshape(-1, 3)
    q = _c(idx, np.int32).reshape(-1)
    if q.size and (q.min() < 0 or q.max() >= pts.shape[0]):
        raise IndexError("knn3_mean_dist2_at: query index out of range")
    out = np.zeros(q.shape[0], _f)
    with np.errstate(over="ignore"):
        lib().orc_knn3_mean_dist2_at(C.c_int(pts.shape[0]), _p(pts, _fp), C.c_int(q.shape[0]), _p(q, _ip),
                                     _p(out, _fp))
    return out
