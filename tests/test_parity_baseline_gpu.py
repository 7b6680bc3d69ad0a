"""GPU parity AT THE BASELINE CONFIGURATIONS (BASELINE.json configs / SURVEY.md 8d): our kernels, through the
reference-shaped `_C` entry points, against the UNMODIFIED reference CUDA sources (oracle/build_ref.sh), whose
outputs on an H100 are stored in tests/golden/ref/ (util.ref_raster) -- forward and backward.

  raster  100k Gaussians / 512^2 cone beam   (headline; init-like and trained-like cloud, 3 views each)
  raster   50k Gaussians / 256^2             (config 1)
  raster  300k Gaussians / 512^2             (config 3, the cloud the 8 shards are cut from)
  voxel   256^3 over 500k Gaussians          (config 4; RAS/forward.cu:198-395, VOX/forward.cu:58-315)
  voxel   32^3 TV crop over 100k Gaussians   (train.py:128-139)
  + the binding paths cov3D_precomp (PYX/rasterization.py:241-253), markVisible
    (SUB/rasterize_points.cu:166-186) and debug=True (synchronous ABI, allocator callback).

Bars: radii / tiles_touched / multiset of 64-bit (tile | depth bits) keys / per-tile ranges bit-exact;
intensities |ours - ref| <= 1e-5 * max|ref| + 1e-7; gradients |a-b| <= 5e-4 |b| + 5e-5 max|b| (the reference's
float atomics are not order-stable, util.grad_mismatch)."""
import numpy as np
import pytest

import util
from r2_gaussian_b200 import scene

pytestmark = pytest.mark.gpu

GRAD_KEYS_R = ["dL_dmean2D", "dL_dopacity", "dL_dmu", "dL_dmean3D", "dL_dcov3D", "dL_dscale", "dL_drot"]
GRAD_KEYS_V = ["dL_dopacity", "dL_dmean3D", "dL_dcov3D", "dL_dscale", "dL_drot"]
_clouds = {}


def cloud_of(P, kind):
    key = (P, kind)
    if key not in _clouds:
        _clouds.clear()     # keep one big cloud alive at a time
        _clouds[key] = scene.make_cloud(P, kind=kind, seed=0)
    return _clouds[key]


def check_raster(name, cloud, view, backward=True, cov3D_precomp=None, debug=False):
    dL = np.random.RandomState(5).randn(view.image_height, view.image_width).astype(np.float32) if backward else None
    ref = util.ref_raster(name, cloud, view, dL, cov3D_precomp=cov3D_precomp)
    ours = util.ours_raster_forward(cloud, view, cov3D_precomp=cov3D_precomp, debug=debug)
    assert int(ours["R"]) == ref.R
    ref.assert_equal("radii", ours["radii"].astype(np.int32))
    ref.assert_equal("tiles_touched", ours["tiles_touched"])
    vis = ours["radii"] > 0
    for k in ("depth", "xy", "conic_opacity", "mu"):
        ref.assert_equal(k + "_vis", ours[k][vis].view(np.uint32))
    ref.assert_equal("keys_sorted", np.sort(ours["keys"]))
    ref.assert_equal("ranges", ours["ranges"])
    ref.assert_close("image", ours["image"])
    if backward:
        g = util.ours_raster_backward(cloud, view, ours, dL, debug=debug)
        if cov3D_precomp is None:
            ref.assert_grads_close(g, GRAD_KEYS_R, rtol=5e-4, atol_rel=5e-5, label="ours vs ref ")
        else:
            for k in ["dL_dmean2D", "dL_dopacity", "dL_dmu", "dL_dmean3D", "dL_dcov3D"]:
                # each array against its own scale (no dL_drot / dL_dscale coupling)
                ref.assert_grads_close(g, [k], 5e-4, 5e-5, label="ours vs ref ")
            assert not g["dL_dscale"].any() and not g["dL_drot"].any()
    return ours, ref


@pytest.mark.parametrize("kind", ["init", "trained"])
def test_raster_100k_512_cone_three_views(kind):
    """The headline scene of BASELINE.json (100k Gaussians, 512^2 cone beam)."""
    cloud = cloud_of(100_000, kind)
    sc = scene.cone_beam_scanner(512, 256)
    for angle in (0.0, 2.1, 4.4):
        check_raster(f"raster_100k_{kind}_cone512_{angle}", cloud, scene.make_view(sc, angle))


@pytest.mark.parametrize("kind", ["init", "trained"])
def test_raster_50k_256_cone(kind):
    cloud = cloud_of(50_000, kind)
    sc = scene.cone_beam_scanner(256, 256)
    for angle in (0.3, 3.9):
        check_raster(f"raster_50k_{kind}_cone256_{angle}", cloud, scene.make_view(sc, angle))


def test_raster_300k_512_cone():
    cloud = cloud_of(300_000, "trained")
    sc = scene.cone_beam_scanner(512, 256)
    check_raster("raster_300k_trained_cone512_1.0", cloud, scene.make_view(sc, 1.0))


def test_raster_100k_512_parallel():
    cloud = cloud_of(100_000, "trained")
    sc = scene.parallel_beam_scanner(512, 256)
    check_raster("raster_100k_trained_parallel512_0.7", cloud, scene.make_view(sc, 0.7))


def check_voxel(name, cloud, nV, sV, ctr, backward=True, cov3D_precomp=None, debug=False):
    dL = np.random.RandomState(6).randn(*nV).astype(np.float32) if backward else None
    ref = util.ref_voxel(name, cloud, nV, sV, ctr, dL, cov3D_precomp=cov3D_precomp)
    ours = util.ours_voxel_forward(cloud, nV, sV, ctr, cov3D_precomp=cov3D_precomp, debug=debug)
    assert int(ours["R"]) == ref.R
    for k in ["radii_x", "radii_y", "radii_z"]:
        ref.assert_equal(k, ours[k].astype(np.int32))
    ref.assert_equal("tiles_touched", ours["tiles_touched"])
    vis = ours["tiles_touched"] > 0
    ref.assert_equal("xyz_vol_vis", ours["xyz_vol"][vis].view(np.uint32))
    ref.assert_equal("depth_vis", ours["depth"][vis].view(np.uint32))
    ref.assert_equal("keys_sorted", np.sort(ours["keys"]))
    ref.assert_equal("ranges", ours["ranges"])
    ref.assert_close("vol", ours["vol"])
    if backward:
        g = util.ours_voxel_backward(cloud, nV, sV, ctr, ours, dL, debug=debug)
        if cov3D_precomp is None:
            ref.assert_grads_close(g, GRAD_KEYS_V, rtol=5e-4, atol_rel=5e-5, label="ours vs ref ")
        else:
            for k in ["dL_dopacity", "dL_dmean3D", "dL_dcov3D"]:
                ref.assert_grads_close(g, [k], 5e-4, 5e-5, label="ours vs ref ")
    return ours, ref


@pytest.mark.parametrize("kind", ["init", "trained"])
def test_voxel_256_cube_500k(kind):
    """BASELINE config 4: 256^3 volume query over 500k Gaussians (32768 tiles)."""
    cloud = cloud_of(500_000, kind)
    check_voxel(f"voxel_256_500k_{kind}", cloud, (256, 256, 256), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0), backward=(kind == "trained"))


def test_voxel_tv_crop_32_100k():
    """The 32^3 total-variation crop of train.py:128-139 (random centre, crop = volume / 8 per axis)."""
    cloud = cloud_of(100_000, "trained")
    rng = np.random.RandomState(3)
    sV = (0.25, 0.25, 0.25)
    for i in range(3):
        ctr = tuple(float(v) for v in (2.0 - 0.25) * (rng.rand(3) - 0.5))
        check_voxel(f"voxel_tv32_100k_{i}", cloud, (32, 32, 32), sV, ctr)


# ---- binding paths -------------------------------------------------------------------------------
def _precomputed_cov(cloud, view):
    """Sigma3 per Gaussian, bit-identical to what the reference's preprocess computes from scales / rotations
    (the oracle is pinned to it bit for bit, test_ref_gpu.py)."""
    return util.oracle_raster_forward(cloud, view, render=False)["cov3D"]


def test_raster_cov3D_precomp_path():
    cloud = cloud_of(20_000, "trained")
    view = scene.make_view(scene.cone_beam_scanner(256, 256), 0.9)
    cov = _precomputed_cov(cloud, view)
    ours_c, ref_c = check_raster("raster_20k_cone256_0.9_cov3D", cloud, view, cov3D_precomp=cov)
    ours_s, _ = check_raster("raster_20k_cone256_0.9", cloud, view, backward=False)
    np.testing.assert_array_equal(ours_c["radii"], ours_s["radii"])
    np.testing.assert_array_equal(ours_c["image"].view(np.uint32), ours_s["image"].view(np.uint32))


def test_voxel_cov3D_precomp_path():
    """Forward against the reference.  The reference's voxelizer backward cannot run with cov3D_precomp (it needs
    `scales` for the radius, VOX/forward.cu:137, and then differentiates through `rotations`, which are absent:
    VOX/backward.cu:201-211 dereferences a null pointer), so the gradients are checked against the CPU oracle."""
    cloud = cloud_of(20_000, "trained")
    view = scene.make_view(scene.cone_beam_scanner(64, 64), 0.0)
    cov = _precomputed_cov(cloud, view)
    grid = ((64, 64, 64), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0))
    ours, _ = check_voxel("voxel_64_20k_cov3D", cloud, *grid, backward=False, cov3D_precomp=cov)
    ours_s, _ = check_voxel("voxel_64_20k", cloud, *grid, backward=False)
    np.testing.assert_array_equal(ours["vol"].view(np.uint32), ours_s["vol"].view(np.uint32))
    dL = np.random.RandomState(6).randn(*grid[0]).astype(np.float32)
    g = util.ours_voxel_backward(cloud, *grid, ours, dL)
    orc = util.oracle_voxel_forward(cloud, *grid, cov3D_precomp=cov)
    from oracle import r2_oracle as o
    go = o.voxel_backward(orc, cloud.scales, None, grid[0], grid[1], dL, cov3D_precomp=cov)
    util.assert_grads_close(g, go, ["dL_dopacity", "dL_dmean3D", "dL_dcov3D"])
    assert not g["dL_dscale"].any() and not g["dL_drot"].any()


def test_debug_true_synchronous_abi():
    """debug=True takes r2x_raster_forward / r2x_voxel_forward: the variant with the reference's semantics exactly
    (the library learns R, asks the allocator callback for the binning buffer, syncs after every stage)."""
    cloud = cloud_of(20_000, "trained")
    view = scene.make_view(scene.cone_beam_scanner(256, 256), 2.2)
    a, _ = check_raster("raster_20k_cone256_2.2", cloud, view, debug=True)
    b, _ = check_raster("raster_20k_cone256_2.2", cloud, view, backward=False, debug=False)
    np.testing.assert_array_equal(a["image"].view(np.uint32), b["image"].view(np.uint32))
    assert int(a["R"]) == a["R"].capacity          # the synchronous ABI sizes the buffer exactly
    check_voxel("voxel_64_20k_bwd", cloud, (64, 64, 64), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0), debug=True)


def test_mark_visible_matches_reference():
    import torch
    from r2_gaussian_b200.rasterization import GaussianRasterizationSettings, GaussianRasterizer

    cloud = cloud_of(20_000, "trained")
    view = scene.make_view(scene.cone_beam_scanner(256, 256), 1.3)
    t = util.to_torch(cloud, view)
    # move a third of the points behind / onto the near plane (view-space z <= 0.2 fails, RAS/auxiliary.h:143-168)
    means = t["means"].clone()
    cam = torch.tensor(view.campos, device="cuda")
    means[::3] = cam + (means[::3] - cam) * torch.linspace(-0.02, 0.06, means[::3].shape[0], device="cuda")[:, None]
    settings = GaussianRasterizationSettings(view.image_height, view.image_width, view.tanfovx, view.tanfovy, 1.0,
                                             t["view"], t["proj"], t["campos"], False, view.mode, False)
    ours = GaussianRasterizer(settings).markVisible(means)
    present = util.ref_mark_visible("mark_visible_20k", means, t["view"], t["proj"])
    assert ours.dtype == torch.bool and ours.shape == (cloud.P,)
    assert 0 < int(present.sum()) < cloud.P
    np.testing.assert_array_equal(ours.cpu().numpy(), present)
    from oracle import r2_oracle as orc
    np.testing.assert_array_equal(orc.mark_visible(means.cpu().numpy(), view.viewmatrix, view.projmatrix), present)
