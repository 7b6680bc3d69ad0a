"""Shared helpers for the parity tests: scene cases, running our C ABI, the oracle, and the reference project's own
kernels as stored golden records (tests/golden/ref/, see ref_raster)."""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import os

import numpy as np

from r2_gaussian_b200 import scene

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libr2ref.so")
REF_GOLDEN = os.path.join(ROOT, "tests", "golden", "ref")
# Set to a directory to (re)generate the golden records: the reference's kernels (oracle/_ref/libr2ref.so, built by
# oracle/build_ref.sh) are run on the GPU and what the tests compare against is written there, e.g.
#     R2X_RECORD_REF_GOLDEN=/tmp/ref python -m pytest -m gpu tests/test_ref_gpu.py tests/test_parity_baseline_gpu.py
RECORD_DIR = os.environ.get("R2X_RECORD_REF_GOLDEN") or None


def case(name: str):
    """Named small scenes: returns (cloud, view)."""
    kind, beam, P, n = {
        "cone_init_small": ("init", "cone", 3000, 128),
        "cone_trained_small": ("trained", "cone", 3000, 128),
        "parallel_trained_small": ("trained", "parallel", 2000, 96),
        "cone_trained_ragged": ("trained", "cone", 1500, 100),   # detector not a multiple of 16
        "cone_trained_mid": ("trained", "cone", 20000, 256),
        "cone_init_mid": ("init", "cone", 50000, 256),
        "cone_trained_bigdet": ("trained", "cone", 1500, 1040),  # 65 x 65 = 4225 tiles > DIRECT_MAX_TILES: radix path
    }[name]
    sc = scene.cone_beam_scanner(n, 64) if beam == "cone" else scene.parallel_beam_scanner(n, 64)
    view = scene.make_view(sc, 0.37 + 0.1 * len(name))
    cloud = scene.make_cloud(P, kind=kind, seed=len(name))
    return cloud, view


def to_torch(cloud, view, device="cuda", requires_grad=False):
    import torch

    t = dict(
        means=torch.tensor(cloud.means, device=device), scales=torch.tensor(cloud.scales, device=device),
        rots=torch.tensor(cloud.rotations, device=device), dens=torch.tensor(cloud.density, device=device),
    )
    if requires_grad:
        for v in t.values():
            v.requires_grad_(True)
    if view is not None:
        t["view"] = torch.tensor(view.viewmatrix, device=device)
        t["proj"] = torch.tensor(view.projmatrix, device=device)
        t["campos"] = torch.tensor(view.campos, device=device)
    return t


def ours_raster_forward(cloud, view, export=True, cov3D_precomp=None, debug=False):
    import torch
    from r2_gaussian_b200 import _C
    from r2_gaussian_b200._lib import load, check

    t = to_torch(cloud, view)
    empty = torch.Tensor([])
    scales, rots, cov = t["scales"], t["rots"], empty
    if cov3D_precomp is not None:
        scales, rots, cov = empty, empty, torch.tensor(cov3D_precomp, device="cuda")
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(
        t["means"], t["dens"], scales, rots, 1.0, cov, t["view"], t["proj"], view.tanfovx, view.tanfovy,
        view.image_height, view.image_width, t["campos"], False, view.mode, debug)
    t["scales_in"], t["rots_in"], t["cov_in"] = scales, rots, cov
    out = dict(R=R, image=color[0].cpu().numpy(), radii=radii.cpu().numpy(), state=(geom, binning, img), t=t)
    if export:
        lib = load()
        P, W, H = cloud.P, view.image_width, view.image_height
        T = ((W + 15) // 16) * ((H + 15) // 16)
        dev = "cuda"
        xy = torch.empty((P, 2), device=dev); depth = torch.empty(P, device=dev)
        co = torch.empty((P, 4), device=dev); mu = torch.empty(P, device=dev)
        tt = torch.empty(P, dtype=torch.int32, device=dev); po = torch.empty(P, dtype=torch.int32, device=dev)
        keys = torch.empty(max(R, 1), dtype=torch.int64, device=dev)
        pl = torch.empty(max(R, 1), dtype=torch.int32, device=dev)
        ranges = torch.empty((T, 2), dtype=torch.int32, device=dev)
        from r2_gaussian_b200._C import _carved_capacity
        cap = _carved_capacity(binning, R)
        keys = torch.empty(max(cap, 1), dtype=torch.int64, device=dev)
        pl = torch.empty(max(cap, 1), dtype=torch.int32, device=dev)
        rc = lib.r2x_raster_export(torch.cuda.current_stream().cuda_stream, P, W, H, cap, geom.data_ptr(),
                                   binning.data_ptr() if binning.numel() else None, img.data_ptr(), xy.data_ptr(),
                                   depth.data_ptr(), co.data_ptr(), mu.data_ptr(), tt.data_ptr(), po.data_ptr(),
                                   keys.data_ptr(), pl.data_ptr(), ranges.data_ptr())
        check(rc, "r2x_raster_export")
        torch.cuda.synchronize()
        out.update(xy=xy.cpu().numpy(), depth=depth.cpu().numpy(), conic_opacity=co.cpu().numpy(), mu=mu.cpu().numpy(),
                   tiles_touched=tt.cpu().numpy().astype(np.uint32), point_offsets=po.cpu().numpy().astype(np.uint32),
                   keys=keys.cpu().numpy().astype(np.uint64)[:R], point_list=pl.cpu().numpy().astype(np.uint32)[:R],
                   ranges=ranges.cpu().numpy().astype(np.uint32))
    return out


def ours_raster_backward(cloud, view, fwd, dL, debug=False):
    import torch
    from r2_gaussian_b200 import _C

    t = fwd["t"]
    geom, binning, img = fwd["state"]
    radii = torch.tensor(fwd["radii"], device="cuda")
    g = _C.rasterize_gaussians_backward(
        t["means"], radii, t["scales_in"], t["rots_in"], 1.0, t["cov_in"], t["view"], t["proj"], view.tanfovx,
        view.tanfovy, torch.tensor(dL, device="cuda")[None], t["campos"], geom, fwd["R"], binning, img, view.mode, debug)
    names = ["dL_dmean2D", "dL_dopacity", "dL_dmu", "dL_dmean3D", "dL_dcov3D", "dL_dscale", "dL_drot"]
    return {n: x.cpu().numpy() for n, x in zip(names, g)}


def oracle_raster_forward(cloud, view, **kw):
    from oracle import r2_oracle as orc

    return orc.raster_forward(cloud.means, cloud.scales, cloud.rotations, cloud.density, view.viewmatrix,
                              view.projmatrix, view.image_width, view.image_height, view.tanfovx, view.tanfovy,
                              view.mode, **kw)


def oracle_raster_backward(cloud, view, fwd, dL):
    from oracle import r2_oracle as orc

    return orc.raster_backward(fwd, cloud.means, cloud.scales, cloud.rotations, view.viewmatrix, view.projmatrix,
                               view.image_width, view.image_height, view.tanfovx, view.tanfovy, view.mode, dL)


# ---- voxelizer ------------------------------------------------------------------------------
def ours_voxel_forward(cloud, nVoxel, sVoxel, center, export=True, cov3D_precomp=None, debug=False):
    import torch
    from r2_gaussian_b200 import _C
    from r2_gaussian_b200._lib import load, check

    t = to_torch(cloud, None)
    rots, cov = t["rots"], torch.Tensor([])
    if cov3D_precomp is not None:   # the voxelizer needs the scales for its bounding radius either way
        rots, cov = torch.Tensor([]), torch.tensor(cov3D_precomp, device="cuda")
    t["rots_in"], t["cov_in"] = rots, cov
    R, vol, rx, ry, rz, geom, binning, img = _C.voxelize_gaussians(
        t["means"], t["dens"], t["scales"], rots, 1.0, cov, nVoxel[0], nVoxel[1], nVoxel[2],
        sVoxel[0], sVoxel[1], sVoxel[2], center[0], center[1], center[2], False, debug)
    out = dict(R=R, vol=vol.cpu().numpy(), radii_x=rx.cpu().numpy(), radii_y=ry.cpu().numpy(), radii_z=rz.cpu().numpy(),
               state=(geom, binning, img), t=t, radii_t=(rx, ry, rz))
    if export:
        lib = load()
        P = cloud.P
        nx, ny, nz = nVoxel
        T = ((nx + 7) // 8) * ((ny + 7) // 8) * ((nz + 7) // 8)
        dev = "cuda"
        xyz = torch.empty((P, 3), device=dev); depth = torch.empty(P, device=dev); co = torch.empty((P, 7), device=dev)
        tt = torch.empty(P, dtype=torch.int32, device=dev); po = torch.empty(P, dtype=torch.int32, device=dev)
        keys = torch.empty(max(R, 1), dtype=torch.int64, device=dev)
        pl = torch.empty(max(R, 1), dtype=torch.int32, device=dev)
        ranges = torch.empty((T, 2), dtype=torch.int32, device=dev)
        from r2_gaussian_b200._C import _carved_capacity
        cap = _carved_capacity(binning, R)
        keys = torch.empty(max(cap, 1), dtype=torch.int64, device=dev)
        pl = torch.empty(max(cap, 1), dtype=torch.int32, device=dev)
        rc = lib.r2x_voxel_export(torch.cuda.current_stream().cuda_stream, P, nx, ny, nz, cap, geom.data_ptr(),
                                  binning.data_ptr() if binning.numel() else None, img.data_ptr(), xyz.data_ptr(),
                                  depth.data_ptr(), co.data_ptr(), tt.data_ptr(), po.data_ptr(), keys.data_ptr(),
                                  pl.data_ptr(), ranges.data_ptr())
        check(rc, "r2x_voxel_export")
        torch.cuda.synchronize()
        out.update(xyz_vol=xyz.cpu().numpy(), depth=depth.cpu().numpy(), conic_opacity=co.cpu().numpy(),
                   tiles_touched=tt.cpu().numpy().astype(np.uint32), keys=keys.cpu().numpy().astype(np.uint64)[:R],
                   point_list=pl.cpu().numpy().astype(np.uint32)[:R], ranges=ranges.cpu().numpy().astype(np.uint32))
    return out


def ours_voxel_backward(cloud, nVoxel, sVoxel, center, fwd, dL, debug=False):
    import torch
    from r2_gaussian_b200 import _C

    t = fwd["t"]
    geom, binning, img = fwd["state"]
    rx, ry, rz = fwd["radii_t"]
    g = _C.voxelize_gaussians_backward(
        t["means"], rx, ry, rz, t["scales"], t["rots_in"], 1.0, t["cov_in"], torch.tensor(dL, device="cuda"), geom,
        fwd["R"], binning, img, nVoxel[0], nVoxel[1], nVoxel[2], sVoxel[0], sVoxel[1], sVoxel[2], center[0], center[1],
        center[2], debug)
    names = ["dL_dopacity", "dL_dmean3D", "dL_dcov3D", "dL_dscale", "dL_drot"]
    return {n: x.cpu().numpy() for n, x in zip(names, g)}


def oracle_voxel_forward(cloud, nVoxel, sVoxel, center, **kw):
    from oracle import r2_oracle as orc

    return orc.voxel_forward(cloud.means, cloud.scales, cloud.rotations, cloud.density, nVoxel, sVoxel, center, **kw)


def oracle_voxel_backward(cloud, nVoxel, sVoxel, fwd, dL):
    from oracle import r2_oracle as orc

    return orc.voxel_backward(fwd, cloud.scales, cloud.rotations, nVoxel, sVoxel, dL)


# ---- comparison helpers ---------------------------------------------------------------------
def key_multiset_equal(keys_a, keys_b):
    return np.array_equal(np.sort(np.asarray(keys_a, dtype=np.uint64)), np.sort(np.asarray(keys_b, dtype=np.uint64)))


def rel_err(a, b, floor=None):
    """max |a-b| / max(|b|, floor) -- floor defaults to 1e-3 * max|b| (relative to the signal scale)."""
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    if floor is None:
        floor = 1e-3 * (np.abs(b).max() if b.size else 1.0) + 1e-30
    return float((np.abs(a - b) / np.maximum(np.abs(b), floor)).max()) if a.size else 0.0


def grad_mismatch(a, b, rtol=2e-4, atol_rel=2e-5, scale=None):
    """Worst violation of |a-b| <= rtol*|b| + atol_rel*scale (scale defaults to max|b|); <= 1 passes.

    Gradients are sums of thousands of signed float32 terms: the achievable agreement between two
    summation orders (the reference's float atomics are not even run-to-run stable) is relative to the
    magnitude of the terms, not of the (possibly cancelling) sum, hence the absolute part tied to the
    array's scale."""
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    if a.size == 0:
        return 0.0
    if scale is None:
        scale = float(np.abs(b).max())
    tol = rtol * np.abs(b) + atol_rel * scale + 1e-30
    return float((np.abs(a - b) / tol).max())


def assert_grads_close(got: dict, want: dict, keys, rtol=2e-4, atol_rel=2e-5, label=""):
    for k in keys:
        scale = None
        if k == "dL_drot":
            # for isotropic Gaussians the rotation gradient is pure cancellation noise: tie its scale
            # to the scale gradient (same chain, dL/dM times a parameter of order one)
            scale = max(float(np.abs(want[k]).max()), float(np.abs(want["dL_dscale"]).max()))
        m = grad_mismatch(got[k], want[k], rtol, atol_rel, scale)
        assert m <= 1.0, f"{label}{k}: mismatch {m:.3g} x tolerance"


# ---- the reference's outputs, stored -------------------------------------------------------------
# A record keeps, for every array a test compares bit for bit, the SHA-256 of its bytes, and for every array compared
# within a tolerance, max|x| over the whole array, the values at a fixed sample of positions (the largest entries and a
# seeded random set) and sums over blocks that tile the whole array (square / cubic blocks of an image or volume, runs
# of rows of a gradient column): the records stay small however large the scene, and a fault anywhere in an array
# still moves the sum of its block.
N_SAMPLE = 96         # flat positions of an image / volume
N_SAMPLE_ROWS = 20    # rows (Gaussians) of a gradient array
N_BLOCKS = 512        # at most this many blocks of an image / volume
N_ROW_BLOCKS = 16     # runs of rows per gradient column


def _block_sums(a, absolute=False):
    """float64 sums of an image / volume over square (cubic) blocks, the edge a power-of-two multiple of the tile edge
    (16 pixels, 8 voxels) chosen so that there are at most N_BLOCKS; and the element count of each block."""
    a = np.asarray(a, dtype=np.float64)
    a = np.abs(a) if absolute else a
    edge = 16 if a.ndim == 2 else 8
    while np.prod([-(-n // edge) for n in a.shape]) > N_BLOCKS:
        edge *= 2
    nb = [-(-n // edge) for n in a.shape]
    pad = np.zeros([k * edge for k in nb]); pad[tuple(slice(0, n) for n in a.shape)] = a
    cnt = np.zeros_like(pad); cnt[tuple(slice(0, n) for n in a.shape)] = 1.0
    shape = [x for k in nb for x in (k, edge)]
    axes = tuple(range(1, 2 * a.ndim, 2))
    return pad.reshape(shape).sum(axis=axes).reshape(-1), cnt.reshape(shape).sum(axis=axes).reshape(-1)


def _row_block_sums(a, absolute=False):
    """float64 sums of each column of a [rows, k] array over N_ROW_BLOCKS runs of consecutive rows: [blocks, k]."""
    a = np.asarray(a, dtype=np.float64).reshape(len(a), -1)
    a = np.abs(a) if absolute else a
    cuts = np.linspace(0, len(a), N_ROW_BLOCKS + 1).astype(np.int64)
    return np.stack([a[lo:hi].sum(axis=0) for lo, hi in zip(cuts[:-1], cuts[1:])]), np.diff(cuts)


def _digest(a) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


def _sample(a, n):
    a = np.asarray(a).reshape(len(a), -1) if n == N_SAMPLE_ROWS else np.asarray(a).reshape(-1)
    if len(a) <= n:
        return np.arange(len(a), dtype=np.int64)
    mag = np.abs(a.reshape(len(a), -1)).max(axis=1)
    top = np.argsort(-mag, kind="stable")[: n // 4]
    rest = np.setdiff1d(np.arange(len(a)), top)
    pick = np.random.RandomState(0).choice(rest, n - len(top), replace=False)
    return np.sort(np.concatenate([top, pick])).astype(np.int64)


class RefRecord:
    """The reference's outputs for one call, as stored in tests/golden/ref/<name>.npz."""

    def __init__(self, data: dict):
        self.d = data
        self.R = int(data["R"])

    @classmethod
    def from_outputs(cls, res: dict, exact: dict, tolerant: dict, grads: dict | None):
        d = {"R": np.int64(res["R"])}
        for k, a in exact.items():
            d[f"sha_{k}"] = _digest(a)
        for k, a in tolerant.items():
            idx = _sample(a, N_SAMPLE)
            d[f"max_{k}"] = np.float64(np.abs(a).max()) if a.size else np.float64(0.0)
            d[f"idx_{k}"] = idx.astype(np.int32)
            d[f"val_{k}"] = np.asarray(a).reshape(-1)[idx]
            d[f"bsum_{k}"] = _block_sums(a)[0].astype(np.float32)
        for k, a in (grads or {}).items():
            a = np.asarray(a).reshape(len(a), -1)
            idx = _sample(a, N_SAMPLE_ROWS)
            d[f"gmax_{k}"] = np.float64(np.abs(a).max()) if a.size else np.float64(0.0)
            d[f"gidx_{k}"] = idx.astype(np.int32)
            d[f"gval_{k}"] = a[idx]
            d[f"gbsum_{k}"] = _row_block_sums(a)[0].astype(np.float32)
        return cls(d)

    def assert_equal(self, key, a):
        assert np.array_equal(_digest(a), self.d[f"sha_{key}"]), f"{key}: differs from the reference"

    def assert_close(self, key, a, rel=1e-5, abs_=1e-7):
        """|a - ref| <= rel * max|ref| + abs_ at the stored positions, max|a| within the same bar of max|ref|, and every
        block sum within (elements of the block) x that bar of the reference's (the bound the per-element bar implies;
        1e-6 relative allows for the float32 storage of the reference's sums)."""
        scale = float(self.d[f"max_{key}"])
        bar = rel * scale + abs_
        sums, cnt = _block_sums(a)
        flat = np.asarray(a, dtype=np.float64).reshape(-1)
        want = self.d[f"val_{key}"].astype(np.float64)
        err = float(np.abs(flat[self.d[f"idx_{key}"]] - want).max()) if want.size else 0.0
        err = max(err, abs(float(np.abs(flat).max()) - scale) if flat.size else 0.0)
        assert err <= bar, f"{key}: max |ours - ref| = {err:.3g} vs scale {scale:.3g}"
        ref_sums = self.d[f"bsum_{key}"].astype(np.float64)
        over = np.abs(sums - ref_sums) / (cnt * bar + 1e-6 * np.abs(ref_sums) + 1e-30)
        assert over.max(initial=0.0) <= 1.0, f"{key}: block {int(over.argmax())} sum off by {over.max():.3g} x its bar"
        return err / max(scale, 1e-30)

    @property
    def grad_keys(self):
        return [k[5:] for k in self.d if k.startswith("gmax_")]

    def assert_grads_close(self, got: dict, keys, rtol=2e-4, atol_rel=2e-5, label=""):
        """util.assert_grads_close at the stored rows, with the scales of the whole arrays."""
        for k in keys:
            scale = float(self.d[f"gmax_{k}"])
            if k == "dL_drot":
                scale = max(scale, float(self.d["gmax_dL_dscale"]))
            idx = self.d[f"gidx_{k}"]
            a = np.asarray(got[k]).reshape(len(got[k]), -1)
            m = grad_mismatch(a[idx], self.d[f"gval_{k}"], rtol, atol_rel, scale)
            assert m <= 1.0, f"{label}{k}: mismatch {m:.3g} x tolerance"
            # runs of rows: the sum of the per-element tolerances over the run, with sum |ref| taken as sum |ours|
            # (the two differ by far less than the run's tolerance); 1e-6 relative for the float32 storage
            sums, n = _row_block_sums(a)
            babs = _row_block_sums(a, absolute=True)[0]
            ref_sums = self.d[f"gbsum_{k}"].astype(np.float64)
            tol = (rtol + 1e-6) * babs + atol_rel * scale * n[:, None] + 1e-30
            over = np.abs(sums - ref_sums) / tol
            assert over.max(initial=0.0) <= 1.0, f"{label}{k}: a run of rows sums off by {over.max():.3g} x tolerance"


def _save(path, d: dict):
    """One record = a JSON index of (name, dtype, shape) + one byte blob: two zip entries instead of one per array."""
    keys = sorted(d)
    arrs = [np.asarray(d[k]) for k in keys]
    meta = json.dumps([[k, a.dtype.str, list(a.shape)] for k, a in zip(keys, arrs)]).encode()
    blob = np.frombuffer(b"".join(np.ascontiguousarray(a).tobytes() for a in arrs), dtype=np.uint8)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    np.savez_compressed(path, meta=np.frombuffer(meta, dtype=np.uint8), blob=blob)


def _load(path) -> dict:
    assert os.path.exists(path), f"golden record {path} is missing"
    with np.load(path) as z:
        meta, blob = json.loads(z["meta"].tobytes()), z["blob"].tobytes()
    d, off = {}, 0
    for k, dt, shape in meta:
        n = int(np.prod(shape, dtype=np.int64)) * np.dtype(dt).itemsize
        d[k] = np.frombuffer(blob[off:off + n], dtype=dt).reshape(tuple(shape))
        off += n
    return d


def _ref_record(name: str, run, backward: bool):
    if RECORD_DIR and (backward or not os.path.exists(os.path.join(RECORD_DIR, name + ".npz"))):
        rec = run()
        _save(os.path.join(RECORD_DIR, name + ".npz"), rec.d)
        return rec
    # a forward-only call may reuse a full record
    return RefRecord(_load(os.path.join(RECORD_DIR or REF_GOLDEN, name + ".npz")))


def ref_raster(name, cloud, view, dL=None, cov3D_precomp=None) -> RefRecord:
    """The reference rasterizer's outputs for this scene (forward, and backward when dL is given)."""
    def run():
        ref = run_ref_raster(cloud, view, dL, cov3D_precomp=cov3D_precomp)
        vis = ref["radii"] > 0
        exact = {"radii": ref["radii"].astype(np.int32), "tiles_touched": ref["tiles_touched"],
                 "keys": ref["keys"], "keys_sorted": np.sort(ref["keys"]), "point_list": ref["point_list"],
                 "ranges": ref["ranges"]}
        for k in ("depth", "xy", "cov3D", "conic_opacity", "mu"):
            exact[k + "_vis"] = ref[k][vis].view(np.uint32)
        return RefRecord.from_outputs(ref, exact, {"image": ref["image"]}, ref.get("grads"))
    return _ref_record(name, run, dL is not None)


def ref_voxel(name, cloud, nV, sV, ctr, dL=None, cov3D_precomp=None) -> RefRecord:
    """The reference voxelizer's outputs for this grid (forward, and backward when dL is given)."""
    def run():
        ref = run_ref_voxel(cloud, nV, sV, ctr, dL, cov3D_precomp=cov3D_precomp)
        vis = ref["tiles_touched"] > 0
        exact = {k: ref[k].astype(np.int32) for k in ("radii_x", "radii_y", "radii_z")}
        exact.update(tiles_touched=ref["tiles_touched"], keys=ref["keys"], keys_sorted=np.sort(ref["keys"]),
                     point_list=ref["point_list"], ranges=ref["ranges"])
        for k in ("xyz_vol", "depth", "conic_opacity"):
            exact[k + "_vis"] = ref[k][vis].view(np.uint32)
        return RefRecord.from_outputs(ref, exact, {"vol": ref["vol"]}, ref.get("grads"))
    return _ref_record(name, run, dL is not None)


def ref_mark_visible(name, means, view_t, proj_t) -> np.ndarray:
    """The reference's markVisible flags for these (device) points, stored whole (one byte per point)."""
    path = os.path.join(REF_GOLDEN, name + ".npz")
    if RECORD_DIR:
        import torch
        lib = need_ref()
        present = torch.zeros(means.shape[0], dtype=torch.bool, device=means.device)
        p = lambda x: C.c_void_p(x.data_ptr())
        lib.ref_mark_visible(means.shape[0], p(means), p(view_t), p(proj_t), p(present))
        torch.cuda.synchronize()
        out = present.cpu().numpy()
        _save(os.path.join(RECORD_DIR, name + ".npz"), {"present": np.packbits(out), "n": np.int64(out.size)})
        return out
    z = _load(path)
    return np.unpackbits(z["present"])[: int(z["n"])].astype(bool)


def ref_digests(name, run) -> dict:
    """SHA-256 of each array `run()` returns (a dict of tensors / arrays), computed now when recording, else stored."""
    path = os.path.join(REF_GOLDEN, name + ".npz")
    if RECORD_DIR:
        out = {k: np.array(tensor_digest(v)) for k, v in run().items()}
        _save(os.path.join(RECORD_DIR, name + ".npz"), out)
        return {k: str(v) for k, v in out.items()}
    return {k: str(v) for k, v in _load(path).items()}


def tensor_digest(x) -> str:
    if hasattr(x, "detach"):
        x = x.detach().cpu().contiguous().numpy()
    return _digest(np.asarray(x)).tobytes().hex() + f":{np.asarray(x).dtype}:{tuple(np.asarray(x).shape)}"


# ---- the compiled reference (recording only) --------------------------------------------------
_ref = None


def ref_lib():
    global _ref
    if _ref is None:
        if not os.path.exists(REF_LIB):
            return None
        _ref = C.CDLL(REF_LIB)
        _ref.ref_raster_forward.restype = C.c_int
        _ref.ref_voxel_forward.restype = C.c_int
    return _ref


def need_ref():
    lib = ref_lib()
    assert lib is not None, "recording golden records needs oracle/_ref/libr2ref.so (oracle/build_ref.sh)"
    return lib


def _cptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None and t.numel() else None


def run_ref_raster(cloud, view, dL=None, cov3D_precomp=None):
    import torch

    lib = need_ref()
    t = to_torch(cloud, view)
    P, W, H = cloud.P, view.image_width, view.image_height
    dev = "cuda"
    out = torch.zeros((1, H, W), device=dev); radii = torch.zeros(P, dtype=torch.int32, device=dev)
    f = C.c_float
    covp = None if cov3D_precomp is None else torch.tensor(cov3D_precomp, device=dev)
    sc_p = None if covp is not None else _cptr(t["scales"])
    ro_p = None if covp is not None else _cptr(t["rots"])
    R = lib.ref_raster_forward(P, W, H, _cptr(t["means"]), _cptr(t["dens"]), sc_p, f(1.0), ro_p,
                               _cptr(covp), _cptr(t["view"]), _cptr(t["proj"]), _cptr(t["campos"]), f(view.tanfovx),
                               f(view.tanfovy), view.mode, _cptr(out), _cptr(radii))
    torch.cuda.synchronize()
    T = ((W + 15) // 16) * ((H + 15) // 16)
    depth = torch.zeros(P, device=dev); xy = torch.zeros((P, 2), device=dev); cov = torch.zeros((P, 6), device=dev)
    co = torch.zeros((P, 4), device=dev); mu = torch.zeros(P, device=dev)
    tt = torch.zeros(P, dtype=torch.int32, device=dev); po = torch.zeros(P, dtype=torch.int32, device=dev)
    ks = torch.zeros(max(R, 1), dtype=torch.int64, device=dev); pl = torch.zeros(max(R, 1), dtype=torch.int32, device=dev)
    rg = torch.zeros((T, 2), dtype=torch.int32, device=dev); nc = torch.zeros((H, W), dtype=torch.int32, device=dev)
    lib.ref_raster_export(P, W, H, R, _cptr(depth), _cptr(xy), _cptr(cov), _cptr(co), _cptr(mu), _cptr(tt), _cptr(po), None,
                          None, _cptr(ks), _cptr(pl), _cptr(rg), _cptr(nc))
    res = dict(R=R, image=out[0].cpu().numpy(), radii=radii.cpu().numpy(), depth=depth.cpu().numpy(),
               xy=xy.cpu().numpy(), cov3D=cov.cpu().numpy(), conic_opacity=co.cpu().numpy(), mu=mu.cpu().numpy(),
               tiles_touched=tt.cpu().numpy().astype(np.uint32), keys=ks.cpu().numpy().astype(np.uint64)[:R],
               point_list=pl.cpu().numpy().astype(np.uint32)[:R], ranges=rg.cpu().numpy().astype(np.uint32))
    if dL is not None:
        z = lambda *s: torch.zeros(s, device=dev)
        g2, gc, go, gm, g3, gcov, gs, gr = z(P, 3), z(P, 4), z(P, 1), z(P, 1), z(P, 3), z(P, 6), z(P, 3), z(P, 4)
        dLt = torch.tensor(dL, device=dev)
        lib.ref_raster_backward(P, R, W, H, _cptr(t["means"]), sc_p, f(1.0), ro_p, _cptr(covp),
                                _cptr(t["view"]), _cptr(t["proj"]), _cptr(t["campos"]), f(view.tanfovx), f(view.tanfovy),
                                _cptr(radii), _cptr(dLt), _cptr(g2), _cptr(gc), _cptr(go), _cptr(gm), _cptr(g3), _cptr(gcov),
                                _cptr(gs), _cptr(gr), view.mode)
        torch.cuda.synchronize()
        res["grads"] = dict(dL_dmean2D=g2.cpu().numpy(), dL_dopacity=go.cpu().numpy(), dL_dmu=gm.cpu().numpy(),
                            dL_dmean3D=g3.cpu().numpy(), dL_dcov3D=gcov.cpu().numpy(), dL_dscale=gs.cpu().numpy(),
                            dL_drot=gr.cpu().numpy())
    return res


def run_ref_voxel(cloud, nV, sV, ctr, dL=None, cov3D_precomp=None):
    import torch

    lib = need_ref()
    t = to_torch(cloud, None)
    P = cloud.P
    nx, ny, nz = nV
    dev = "cuda"
    f = C.c_float
    vol = torch.zeros(nV, device=dev)
    covp = None if cov3D_precomp is None else torch.tensor(cov3D_precomp, device=dev)
    rx = torch.zeros(P, dtype=torch.int32, device=dev); ry = torch.zeros_like(rx); rz = torch.zeros_like(rx)
    R = lib.ref_voxel_forward(P, nx, ny, nz, f(sV[0]), f(sV[1]), f(sV[2]), f(ctr[0]), f(ctr[1]), f(ctr[2]),
                              _cptr(t["means"]), _cptr(t["dens"]), _cptr(t["scales"]), f(1.0),
                              None if covp is not None else _cptr(t["rots"]), _cptr(covp),
                              _cptr(vol), _cptr(rx), _cptr(ry), _cptr(rz))
    torch.cuda.synchronize()
    T = ((nx + 7) // 8) * ((ny + 7) // 8) * ((nz + 7) // 8)
    depth = torch.zeros(P, device=dev); xyz = torch.zeros((P, 3), device=dev); cov = torch.zeros((P, 6), device=dev)
    co = torch.zeros((P, 7), device=dev)
    tt = torch.zeros(P, dtype=torch.int32, device=dev); po = torch.zeros(P, dtype=torch.int32, device=dev)
    ks = torch.zeros(max(R, 1), dtype=torch.int64, device=dev); pl = torch.zeros(max(R, 1), dtype=torch.int32, device=dev)
    rg = torch.zeros((T, 2), dtype=torch.int32, device=dev)
    lib.ref_voxel_export(P, nx, ny, nz, R, _cptr(depth), _cptr(xyz), _cptr(cov), _cptr(co), _cptr(tt), _cptr(po), None, None,
                         _cptr(ks), _cptr(pl), _cptr(rg), None)
    res = dict(R=R, vol=vol.cpu().numpy(), radii_x=rx.cpu().numpy(), radii_y=ry.cpu().numpy(), radii_z=rz.cpu().numpy(),
               depth=depth.cpu().numpy(), xyz_vol=xyz.cpu().numpy(), conic_opacity=co.cpu().numpy(),
               tiles_touched=tt.cpu().numpy().astype(np.uint32), keys=ks.cpu().numpy().astype(np.uint64)[:R],
               point_list=pl.cpu().numpy().astype(np.uint32)[:R], ranges=rg.cpu().numpy().astype(np.uint32))
    if dL is not None:
        z = lambda *s: torch.zeros(s, device=dev)
        gn, gc, go, g3, gcov, gs, gr = z(P, 3), z(P, 6), z(P, 1), z(P, 3), z(P, 6), z(P, 3), z(P, 4)
        dLt = torch.tensor(dL, device=dev)
        lib.ref_voxel_backward(P, R, nx, ny, nz, f(sV[0]), f(sV[1]), f(sV[2]), f(ctr[0]), f(ctr[1]), f(ctr[2]),
                               _cptr(t["means"]), _cptr(t["scales"]), f(1.0),
                               None if covp is not None else _cptr(t["rots"]), _cptr(covp), _cptr(rx), _cptr(ry),
                               _cptr(rz), _cptr(dLt), _cptr(gn), _cptr(gc), _cptr(go), _cptr(g3), _cptr(gcov), _cptr(gs), _cptr(gr))
        torch.cuda.synchronize()
        res["grads"] = dict(dL_dopacity=go.cpu().numpy(), dL_dmean3D=g3.cpu().numpy(), dL_dcov3D=gcov.cpu().numpy(),
                            dL_dscale=gs.cpu().numpy(), dL_drot=gr.cpu().numpy())
    return res
