"""Pins the CPU oracle (and our kernels) against the UNMODIFIED reference CUDA sources (oracle/build_ref.sh), whose
outputs on an H100 are stored in tests/golden/ref/ (util.ref_raster): bit-exact radii / tiles_touched / sorted 64-bit
keys / point lists, 1e-5 on intensities, gradient agreement within atomics noise."""
import numpy as np
import pytest

import util
from r2_gaussian_b200 import scene

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["cone_trained_small", "parallel_trained_small", "cone_trained_ragged", "cone_init_mid"])
def test_oracle_pinned_to_reference_raster(name):
    cloud, view = util.case(name)
    dL = np.random.RandomState(5).randn(view.image_height, view.image_width).astype(np.float32)
    ref = util.ref_raster(f"raster_{name}", cloud, view, dL)
    orc = util.oracle_raster_forward(cloud, view)
    assert ref.R == orc["R"]
    ref.assert_equal("radii", orc["radii"].astype(np.int32))
    ref.assert_equal("tiles_touched", orc["tiles_touched"].astype(np.uint32))
    vis = orc["radii"] > 0
    for k in ("depth", "xy", "cov3D", "conic_opacity", "mu"):
        ref.assert_equal(k + "_vis", orc[k][vis].astype(np.float32).view(np.uint32))
    ref.assert_equal("keys", orc["keys"].astype(np.uint64))          # sorted order too
    ref.assert_equal("point_list", orc["point_list"].astype(np.uint32))
    ref.assert_equal("ranges", orc["ranges"].astype(np.uint32))
    ref.assert_close("image", orc["image"])
    go = util.oracle_raster_backward(cloud, view, orc, dL)
    ref.assert_grads_close(go, ref.grad_keys, rtol=5e-4, atol_rel=5e-5, label="oracle vs ref ")


@pytest.mark.parametrize("name", ["cone_trained_small", "cone_trained_mid"])
def test_ours_against_reference_raster(name):
    cloud, view = util.case(name)
    dL = np.random.RandomState(5).randn(view.image_height, view.image_width).astype(np.float32)
    ref = util.ref_raster(f"raster_{name}", cloud, view, dL)
    ours = util.ours_raster_forward(cloud, view)
    assert ours["R"] == ref.R
    ref.assert_equal("radii", ours["radii"].astype(np.int32))
    ref.assert_equal("tiles_touched", ours["tiles_touched"])
    ref.assert_equal("keys_sorted", np.sort(ours["keys"]))
    ref.assert_equal("ranges", ours["ranges"])
    ref.assert_close("image", ours["image"])
    g = util.ours_raster_backward(cloud, view, ours, dL)
    ref.assert_grads_close(g, ref.grad_keys, rtol=5e-4, atol_rel=5e-5, label="ours vs ref ")


@pytest.mark.parametrize("grid", [((32, 32, 32), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0)),
                                  ((20, 36, 28), (1.3, 2.0, 1.7), (0.1, -0.05, 0.2))])
def test_oracle_and_ours_against_reference_voxel(grid):
    nV, sV, ctr = grid
    cloud = scene.make_cloud(1500, kind="trained", seed=9)
    dL = np.random.RandomState(6).randn(*nV).astype(np.float32)
    ref = util.ref_voxel(f"voxel_{'x'.join(map(str, nV))}_seed9", cloud, nV, sV, ctr, dL)
    orc = util.oracle_voxel_forward(cloud, nV, sV, ctr)
    ours = util.ours_voxel_forward(cloud, nV, sV, ctr)
    for other in (orc, ours):
        assert other["R"] == ref.R
        for k in ["radii_x", "radii_y", "radii_z"]:
            ref.assert_equal(k, other[k].astype(np.int32))
        ref.assert_equal("tiles_touched", other["tiles_touched"].astype(np.uint32))
        ref.assert_equal("keys_sorted", np.sort(other["keys"].astype(np.uint64)))
        ref.assert_equal("ranges", other["ranges"].astype(np.uint32))
        ref.assert_close("vol", other["vol"])
    ref.assert_equal("keys", orc["keys"].astype(np.uint64))
    ref.assert_equal("point_list", orc["point_list"].astype(np.uint32))
    vis = orc["tiles_touched"] > 0
    ref.assert_equal("conic_opacity_vis", orc["conic_opacity"][vis].astype(np.float32).view(np.uint32))
    go = util.oracle_voxel_backward(cloud, nV, sV, orc, dL)
    g = util.ours_voxel_backward(cloud, nV, sV, ctr, ours, dL)
    ref.assert_grads_close(go, ref.grad_keys, rtol=5e-4, atol_rel=5e-5, label="oracle vs ref ")
    ref.assert_grads_close(g, ref.grad_keys, rtol=5e-4, atol_rel=5e-5, label="ours vs ref ")
