"""CPU tests of the oracle itself (no GPU): against an independent float64 textbook statement of the
math, against the committed golden vectors produced by the compiled reference on the GPU
(tests/golden/), and through the structural properties the pipeline must satisfy."""
import os

import numpy as np
import pytest

import textbook
import util
from oracle import r2_oracle as orc
from r2_gaussian_b200 import scene

GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("name", ["cone_trained_small", "parallel_trained_small"])
def test_preprocess_matches_textbook(name):
    cloud, view = util.case(name)
    f = util.oracle_raster_forward(cloud, view, render=False)
    tb = textbook.project(cloud.means, cloud.scales, cloud.rotations, view.viewmatrix, view.projmatrix,
                          view.image_width, view.image_height, view.tanfovx, view.tanfovy, view.mode)
    vis = f["radii"] > 0
    assert vis.sum() > 0.9 * cloud.P
    np.testing.assert_allclose(f["xy"][vis], tb["xy"][vis], rtol=2e-5, atol=2e-3)
    np.testing.assert_allclose(f["depth"][vis], tb["depth"][vis], rtol=1e-5)
    np.testing.assert_allclose(f["conic_opacity"][vis, :3], tb["conic"][vis], rtol=2e-3, atol=1e-6)
    np.testing.assert_allclose(f["mu"][vis], tb["mu"][vis], rtol=2e-3)
    # radius = ceil(3 sqrt(lambda_max)) : allow the ceil to flip where the float value is within 1e-3 of an integer
    r = tb["radius"][vis]
    ok = (f["radii"][vis] == np.ceil(r)) | (np.abs(r - np.round(r)) < 1e-3)
    assert ok.all()


def test_render_matches_bruteforce_small():
    sc = scene.cone_beam_scanner(48, 32)
    view = scene.make_view(sc, 1.1)
    cloud = scene.make_cloud(300, kind="trained", seed=3)
    f = util.oracle_raster_forward(cloud, view)
    tb = textbook.project(cloud.means, cloud.scales, cloud.rotations, view.viewmatrix, view.projmatrix, 48, 48,
                          view.tanfovx, view.tanfovy, view.mode)
    w = cloud.density[:, 0].astype(np.float64) * tb["mu"]
    img = textbook.render_bruteforce(tb["xy"], tb["conic"], w, 48, 48, mask=f["radii"] > 0)
    # the tiled renderer only evaluates a Gaussian inside its 3-sigma tile rectangle, the brute force
    # everywhere: they differ by the tails outside the rectangle (<= exp(-4.5) w), so compare loosely
    # in the aggregate and tightly at the pixels next to a Gaussian centre
    assert abs(img.sum() - f["image"].sum()) / img.sum() < 5e-3
    np.testing.assert_allclose(f["image"], img, rtol=0.05, atol=0.05 * img.max())


def test_keys_ranges_structure():
    cloud, view = util.case("cone_trained_small")
    f = util.oracle_raster_forward(cloud, view)
    R = f["R"]
    assert R == int(f["tiles_touched"].sum()) == len(f["keys"])
    assert np.all(np.diff(f["keys"].astype(np.uint64)) >= 0) or np.all(f["keys"][1:] >= f["keys"][:-1])
    tiles = (f["keys"] >> np.uint64(32)).astype(np.int64)
    depth_bits = (f["keys"] & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    np.testing.assert_array_equal(depth_bits, f["depth"].view(np.uint32)[f["point_list"]])
    gx = (view.image_width + 15) // 16
    for t in np.unique(tiles):
        a, b = f["ranges"][t]
        assert np.all(tiles[a:b] == t) and (a == 0 or tiles[a - 1] != t) and (b == R or tiles[b] != t)
    # every instance lies inside its Gaussian's rectangle
    g = f["point_list"]
    tx, ty = tiles % gx, tiles // gx
    r = f["rect"][g]
    assert np.all((tx >= r[:, 0]) & (tx < r[:, 2]) & (ty >= r[:, 1]) & (ty < r[:, 3]))
    np.testing.assert_array_equal(np.bincount(g, minlength=cloud.P), f["tiles_touched"])


def test_shard_sum_identity():
    """Additivity (SURVEY.md 8e): the image of the whole cloud equals the sum of the images of a
    partition of it, up to float32 summation order."""
    cloud, view = util.case("cone_trained_small")
    full = util.oracle_raster_forward(cloud, view)["image"].astype(np.float64)
    parts = sum(util.oracle_raster_forward(scene.shard_cloud(cloud, r, 3), view)["image"].astype(np.float64)
                for r in range(3))
    assert np.abs(full - parts).max() <= 1e-5 * np.abs(full).max()
    nV, sV, c = (24, 24, 24), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0)
    fullv = util.oracle_voxel_forward(cloud, nV, sV, c)["vol"].astype(np.float64)
    partv = sum(util.oracle_voxel_forward(scene.shard_cloud(cloud, r, 2), nV, sV, c)["vol"].astype(np.float64)
                for r in range(2))
    assert np.abs(fullv - partv).max() <= 1e-5 * np.abs(fullv).max()


def test_voxel_conic_matches_textbook():
    cloud = scene.make_cloud(500, kind="trained", seed=4)
    nV, sV, c = (32, 32, 32), (2.0, 1.5, 1.0), (0.0, 0.1, -0.1)
    f = util.oracle_voxel_forward(cloud, nV, sV, c, render=False)
    dv = np.array(sV) / np.array(nV)
    inv = textbook.voxel_conic(cloud.scales, cloud.rotations, dv)
    vis = f["tiles_touched"] > 0
    got = f["conic_opacity"][vis]
    exp = np.stack([inv[:, 0, 0], inv[:, 0, 1], inv[:, 0, 2], inv[:, 1, 1], inv[:, 1, 2], inv[:, 2, 2]], 1)[vis]
    np.testing.assert_allclose(got[:, :6], exp, rtol=5e-3, atol=1e-4 * np.abs(exp).max())
    pv = (cloud.means - np.array(c) + np.array(sV) / 2) / dv
    np.testing.assert_allclose(f["xyz_vol"][vis], pv[vis], rtol=1e-5, atol=1e-4)
    rad = np.ceil(3 * cloud.scales.max(1)[:, None] / dv[None])
    soft = np.abs(3 * cloud.scales.max(1)[:, None] / dv[None] - np.round(3 * cloud.scales.max(1)[:, None] / dv[None])) < 1e-3
    got_r = np.stack([f["radii_x"], f["radii_y"], f["radii_z"]], 1)
    assert np.all((got_r[vis] == rad[vis]) | soft[vis])


def test_voxel_single_gaussian_peak_and_edges():
    """One isotropic Gaussian at a voxel centre: peak value = density, symmetric, zero outside its cube."""
    means = np.array([[0.03125, 0.03125, 0.03125]], np.float32)  # centre of voxel (16,16,16) for 32^3 over 2^3
    scales = np.full((1, 3), 0.05, np.float32); rots = np.array([[1, 0, 0, 0]], np.float32); dens = np.array([[0.7]], np.float32)
    f = orc.voxel_forward(means, scales, rots, dens, (32, 32, 32), (2, 2, 2), (0, 0, 0))
    vol = f["vol"]
    assert abs(vol[16, 16, 16] - 0.7) < 1e-6
    assert abs(vol[15, 16, 16] - vol[17, 16, 16]) < 1e-7 and abs(vol[16, 16, 15] - vol[16, 16, 17]) < 1e-7
    expect = 0.7 * np.exp(-0.5 * (0.0625 / 0.05) ** 2)
    assert abs(vol[17, 16, 16] - expect) < 1e-6
    assert f["radii_x"][0] == int(np.ceil(3 * 0.05 / 0.0625))


def test_backward_finite_difference_density():
    """d(sum(dL*image))/d(density) from the oracle backward vs a finite difference of the oracle forward
    (density enters linearly, so this is exact up to the alpha cut)."""
    cloud, view = util.case("cone_trained_small")
    cloud = scene.Cloud(cloud.means[:200], cloud.scales[:200], cloud.rotations[:200], cloud.density[:200] + 0.5)
    dL = np.random.RandomState(0).rand(view.image_height, view.image_width).astype(np.float32)
    f = util.oracle_raster_forward(cloud, view)
    g = util.oracle_raster_backward(cloud, view, f, dL)
    base = float((f["image"].astype(np.float64) * dL).sum())
    for i in [0, 17, 101]:
        c2 = scene.Cloud(cloud.means, cloud.scales, cloud.rotations, cloud.density.copy())
        c2.density[i, 0] *= 1.01
        f2 = util.oracle_raster_forward(c2, view)
        fd = (float((f2["image"].astype(np.float64) * dL).sum()) - base) / (0.01 * cloud.density[i, 0])
        assert abs(fd - g["dL_dopacity"][i, 0]) <= 2e-2 * abs(fd) + 1e-4


def test_golden_vectors():
    """Outputs of the compiled reference (oracle/_ref run on the GPU, tests/golden/make_golden.py) vs the oracle."""
    files = sorted(f for f in os.listdir(GOLD) if f.endswith(".npz") and f.split("_")[0] in ("raster", "voxel")) \
        if os.path.isdir(GOLD) else []
    if not files:
        pytest.skip("no golden vectors committed yet")
    for fn in files:
        z = np.load(os.path.join(GOLD, fn))
        if fn.startswith("raster"):
            f = orc.raster_forward(z["means"], z["scales"], z["rots"], z["dens"], z["view"], z["proj"], int(z["W"]),
                                   int(z["H"]), float(z["tanfovx"]), float(z["tanfovy"]), int(z["mode"]))
            np.testing.assert_array_equal(f["radii"], z["radii"])
            np.testing.assert_array_equal(f["tiles_touched"], z["tiles_touched"])
            np.testing.assert_array_equal(f["keys"], z["keys"])
            np.testing.assert_array_equal(f["point_list"], z["point_list"])
            scale = np.abs(z["image"]).max()
            assert np.abs(f["image"].astype(np.float64) - z["image"]).max() <= 1e-5 * scale + 1e-7
            g = orc.raster_backward(f, z["means"], z["scales"], z["rots"], z["view"], z["proj"], int(z["W"]), int(z["H"]),
                                    float(z["tanfovx"]), float(z["tanfovy"]), int(z["mode"]), z["dL"])
            util.assert_grads_close(g, {k[2:]: z[k] for k in z.files if k.startswith("g_")},
                                    ["dL_dmean2D", "dL_dopacity", "dL_dmean3D", "dL_dscale", "dL_drot"], rtol=5e-4,
                                    atol_rel=5e-5, label=fn + " ")
        else:
            nV = tuple(int(v) for v in z["nVoxel"]); sV = tuple(float(v) for v in z["sVoxel"]); c = tuple(float(v) for v in z["center"])
            f = orc.voxel_forward(z["means"], z["scales"], z["rots"], z["dens"], nV, sV, c)
            for k in ["radii_x", "radii_y", "radii_z", "tiles_touched", "keys", "point_list"]:
                np.testing.assert_array_equal(f[k], z[k])
            scale = np.abs(z["vol"]).max()
            assert np.abs(f["vol"].astype(np.float64) - z["vol"]).max() <= 1e-5 * scale + 1e-7
            g = orc.voxel_backward(f, z["scales"], z["rots"], nV, sV, z["dL"])
            util.assert_grads_close(g, {k[2:]: z[k] for k in z.files if k.startswith("g_")},
                                    ["dL_dopacity", "dL_dmean3D", "dL_dscale", "dL_drot"], rtol=5e-4, atol_rel=5e-5,
                                    label=fn + " ")


def test_knn_oracle_vs_kdtree():
    """orc_knn3_mean_dist2 (the restated simple_knn.distCUDA2) against an independent float64 k-d tree."""
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(11)
    for pts in (rng.normal(size=(1500, 3)), rng.uniform(-1, 1, size=(800, 3)) * [1, 1, 0.01]):
        pts = pts.astype(np.float32)
        got = orc.knn3_mean_dist2(pts)
        d, _ = cKDTree(pts.astype(np.float64)).query(pts.astype(np.float64), k=4)
        ref = (d[:, 1:] ** 2).mean(1)
        assert np.allclose(got, ref, rtol=2e-6, atol=1e-12)
    two = orc.knn3_mean_dist2(np.zeros((2, 3), np.float32))
    assert np.all(two > 1e37)          # fewer than 3 neighbours: FLT_MAX placeholders, as upstream


@pytest.mark.parametrize("name", ["cone_trained_mid", "parallel_trained_small", "cone_trained_ragged"])
def test_torch_cpu_projector_matches_oracle(name):
    """The pure-PyTorch CPU projector (bench.py's cpu_baseline_torch) against the C oracle."""
    from oracle import torch_projector as tp
    cloud, view = util.case(name)
    ref = np.asarray(util.oracle_raster_forward(cloud, view)["image"])
    got = tp.project(cloud.means, cloud.density, cloud.scales, cloud.rotations, view.viewmatrix, view.projmatrix,
                     view.image_width, view.image_height, view.tanfovx, view.tanfovy, view.mode).numpy()
    assert got.shape == (1, view.image_height, view.image_width)
    assert np.abs(got - ref.reshape(got.shape)).max() <= 1e-4 * np.abs(ref).max()
