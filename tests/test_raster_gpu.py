"""GPU parity: our sm_90a rasterizer (through the C ABI) against the CPU oracle.

Bars (BASELINE.json north_star): bit-exact radii / tiles_touched / tile rectangles / depth bits / the
multiset of 64-bit sort keys; pixel intensities within 1e-5 relative (of the image scale -- a pair that
sits exactly on the alpha = 1e-5 cut may flip and moves a pixel by 1e-5 absolute); gradients within
1e-4 relative of the gradient scale (the reference's own float atomics are not order-stable)."""
import numpy as np
import pytest

import util

pytestmark = pytest.mark.gpu

CASES = ["cone_init_small", "cone_trained_small", "parallel_trained_small", "cone_trained_ragged", "cone_trained_mid",
         "cone_trained_bigdet"]


@pytest.mark.parametrize("name", CASES)
def test_forward_matches_oracle(name):
    cloud, view = util.case(name)
    ours = util.ours_raster_forward(cloud, view)
    orc = util.oracle_raster_forward(cloud, view)
    # --- bit-exact territory
    assert ours["R"] == orc["R"]
    np.testing.assert_array_equal(ours["radii"], orc["radii"])
    np.testing.assert_array_equal(ours["tiles_touched"], orc["tiles_touched"])
    vis = orc["radii"] > 0
    np.testing.assert_array_equal(ours["depth"][vis].view(np.uint32), orc["depth"][vis].view(np.uint32))
    np.testing.assert_array_equal(ours["xy"][vis].view(np.uint32), orc["xy"][vis].view(np.uint32))
    np.testing.assert_array_equal(ours["point_offsets"], np.cumsum(orc["tiles_touched"]).astype(np.uint32))
    assert util.key_multiset_equal(ours["keys"], orc["keys"])
    # per-tile ranges identical; our per-tile lists hold the same Gaussians (ascending id instead of depth order)
    np.testing.assert_array_equal(ours["ranges"], orc["ranges"])
    for t in range(orc["ranges"].shape[0]):
        a, b = orc["ranges"][t]
        mine = ours["point_list"][a:b]
        assert np.all(np.diff(mine.astype(np.int64)) > 0), "per-tile list must be strictly ascending in Gaussian id"
        np.testing.assert_array_equal(mine, np.sort(orc["point_list"][a:b]))
    # --- tolerance territory
    np.testing.assert_allclose(ours["conic_opacity"][vis], orc["conic_opacity"][vis], rtol=0, atol=0)
    np.testing.assert_array_equal(ours["mu"][vis].view(np.uint32), orc["mu"][vis].view(np.uint32))
    scale = float(np.abs(orc["image"]).max())
    err = np.abs(ours["image"].astype(np.float64) - orc["image"]).max()
    assert err <= 1e-5 * scale + 1e-7, f"image error {err} vs scale {scale}"


@pytest.mark.parametrize("name", ["cone_trained_small", "parallel_trained_small", "cone_trained_ragged", "cone_trained_bigdet"])
def test_backward_matches_oracle(name):
    cloud, view = util.case(name)
    ours = util.ours_raster_forward(cloud, view, export=False)
    orc = util.oracle_raster_forward(cloud, view)
    rng = np.random.RandomState(7)
    dL = rng.randn(view.image_height, view.image_width).astype(np.float32)
    g = util.ours_raster_backward(cloud, view, ours, dL)
    go = util.oracle_raster_backward(cloud, view, orc, dL)
    util.assert_grads_close(g, go, ["dL_dmean2D", "dL_dopacity", "dL_dmu", "dL_dmean3D", "dL_dcov3D", "dL_dscale", "dL_drot"])


def test_forward_is_deterministic():
    cloud, view = util.case("cone_trained_mid")
    a = util.ours_raster_forward(cloud, view, export=False)["image"]
    b = util.ours_raster_forward(cloud, view, export=False)["image"]
    np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))


def test_backward_is_deterministic():
    cloud, view = util.case("cone_trained_small")
    dL = np.random.RandomState(3).randn(view.image_height, view.image_width).astype(np.float32)
    f = util.ours_raster_forward(cloud, view, export=False)
    g1 = util.ours_raster_backward(cloud, view, f, dL)
    g2 = util.ours_raster_backward(cloud, view, f, dL)
    for k in g1:
        np.testing.assert_array_equal(g1[k].view(np.uint32), g2[k].view(np.uint32))


def test_empty_and_culled_inputs():
    import torch
    from r2_gaussian_b200 import _C

    cloud, view = util.case("cone_trained_small")
    t = util.to_torch(cloud, view)
    # P = 0: zeros, num_rendered 0 (reference SUB/rasterize_points.cu:70-72)
    e3 = torch.zeros((0, 3), device="cuda"); e1 = torch.zeros((0, 1), device="cuda"); e4 = torch.zeros((0, 4), device="cuda")
    R, color, radii, *_ = _C.rasterize_gaussians(e3, e1, e3, e4, 1.0, torch.Tensor([]), t["view"], t["proj"],
                                                 view.tanfovx, view.tanfovy, view.image_height, view.image_width,
                                                 t["campos"], False, view.mode, False)
    assert R == 0 and radii.numel() == 0 and float(color.abs().max()) == 0.0
    # everything behind the near plane: all radii 0, empty image
    far = t["means"].clone(); far[:] = torch.tensor(view.campos, device="cuda")  # at the source => z_view = 0
    R, color, radii, *_ = _C.rasterize_gaussians(far, t["dens"], t["scales"], t["rots"], 1.0, torch.Tensor([]),
                                                 t["view"], t["proj"], view.tanfovx, view.tanfovy, view.image_height,
                                                 view.image_width, t["campos"], False, view.mode, False)
    assert R == 0 and int(radii.max()) == 0 and float(color.abs().max()) == 0.0


def test_cpu_tensor_is_rejected():
    import torch
    from r2_gaussian_b200 import _C

    with pytest.raises(RuntimeError):
        _C.rasterize_gaussians(torch.zeros(4, 3), torch.zeros(4, 1), torch.zeros(4, 3), torch.zeros(4, 4), 1.0,
                               torch.Tensor([]), torch.eye(4), torch.eye(4), 1.0, 1.0, 16, 16, torch.zeros(3), False, 1, False)


def test_async_capacity_overflow_is_reported_and_recovered():
    """The asynchronous C ABI never touches memory beyond the provisioned instance capacity; an
    overflowing call reports it (status[1]) and the engine re-runs with a larger buffer."""
    import torch
    from r2_gaussian_b200.engine import RasterEngine, VoxelEngine

    cloud, view = util.case("cone_trained_small")
    t = util.to_torch(cloud, view)
    ref = util.oracle_raster_forward(cloud, view)
    eng = RasterEngine(cloud.P, view.image_width, view.image_height, "cuda", capacity=512)   # far too small
    args = (t["means"], t["dens"], t["scales"], t["rots"], t["view"], t["proj"], t["campos"], view.tanfovx, view.tanfovy, view.mode)
    eng.forward(*args)
    assert eng.check() is False and eng.capacity >= ref["R"]
    R = eng.fit(*args)
    assert R == ref["R"]
    img = eng.out[0].cpu().numpy()
    assert np.abs(img.astype(np.float64) - ref["image"]).max() <= 1e-5 * np.abs(ref["image"]).max() + 1e-7
    from r2_gaussian_b200 import scene
    cl = scene.make_cloud(1500, kind="trained", seed=9)
    tv = util.to_torch(cl, None)
    vref = util.oracle_voxel_forward(cl, (32, 32, 32), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0))
    ve = VoxelEngine(cl.P, (32, 32, 32), "cuda", capacity=1000)
    vargs = (tv["means"], tv["dens"], tv["scales"], tv["rots"], (2.0, 2.0, 2.0), (0.0, 0.0, 0.0))
    ve.forward(*vargs)
    assert ve.check() is False
    assert ve.fit(*vargs) == vref["R"]
    assert np.abs(ve.out.cpu().numpy().astype(np.float64) - vref["vol"]).max() <= 1e-5 * np.abs(vref["vol"]).max() + 1e-7


def test_host_projector_pipeline_matches_direct_forward():
    """HostProjector (pinned host in / out, three-stream pipeline, deferred capacity check) returns exactly what a
    plain forward returns, for interleaved views, and recovers from a capacity overflow."""
    import torch
    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.engine import HostProjector, RasterEngine
    cloud, _ = util.case("cone_trained_mid")
    scanner = scene.cone_beam_scanner(128)
    views = scene.make_views(scanner, 6)
    P, W, H = cloud.P, 128, 128
    dev = torch.device("cuda")
    pin = lambda a: torch.tensor(a).pin_memory()
    hm, hd, hs, hr = pin(cloud.means), pin(cloud.density), pin(cloud.scales), pin(cloud.rotations)
    hv = [(pin(v.viewmatrix), pin(v.projmatrix), pin(v.campos), v) for v in views]
    eng = RasterEngine(P, W, H, dev)
    dm, dd, ds, dr = (t.to(dev) for t in (hm, hd, hs, hr))
    want = []
    for a, b, c, v in hv:
        eng.fit(dm, dd, ds, dr, a.to(dev), b.to(dev), c.to(dev), v.tanfovx, v.tanfovy, v.mode)
        want.append(eng.out.clone().cpu())
    hp = HostProjector(P, W, H, dev, depth=3, capacity=64)     # far too small: the first requests overflow
    outs = [torch.empty((1, H, W)).pin_memory() for _ in range(12)]
    tickets = []
    for i in range(12):
        a, b, c, v = hv[i % 6]
        tickets.append(hp.submit(hm, hd, hs, hr, a, b, c, v.tanfovx, v.tanfovy, v.mode, outs[i]))
    hp.drain()
    for i in range(12):
        assert torch.equal(outs[i], want[i % 6]), i
    a, b, c, v = hv[3]
    got = hp.project(hm, hd, hs, hr, a, b, c, v.tanfovx, v.tanfovy, v.mode, outs[0])
    assert torch.equal(got, want[3])


def test_speculative_training_forward_defers_the_capacity_check():
    """Training mode (inputs require grad): the forward does not synchronise; num_rendered is an upper bound that the
    backward resolves.  Results equal the synchronous path; a forward whose instance count more than doubled since the
    previous call of the same shape raises CapacityOverflow in the backward, and repeating the step succeeds."""
    import torch
    from r2_gaussian_b200 import _C
    from r2_gaussian_b200.rasterization import GaussianRasterizationSettings, GaussianRasterizer

    cloud, view = util.case("cone_trained_small")

    def run(c):
        t = util.to_torch(c, view, requires_grad=True)
        m2 = torch.zeros_like(t["means"], requires_grad=True)
        s = GaussianRasterizationSettings(view.image_height, view.image_width, view.tanfovx, view.tanfovy, 1.0, t["view"],
                                          t["proj"], t["campos"], False, view.mode, False)
        img, radii = GaussianRasterizer(s)(t["means"], m2, t["dens"], t["scales"], t["rots"])
        return t, img

    key = ("raster", 0, cloud.P, view.image_width, view.image_height)
    _C._Workspace.hints.pop(key, None)
    t1, img1 = run(cloud)                          # first call of the shape: synchronous, sets the hint
    assert key in _C._Workspace.hints
    img1.sum().backward()
    t2, img2 = run(cloud)                          # second call: speculative
    assert torch.equal(img1, img2)
    img2.sum().backward()
    for k in ("means", "dens", "scales", "rots"):
        assert torch.equal(t1[k].grad, t2[k].grad), k
    # same shape, 6x larger Gaussians: far more than twice the instances -> overflow is reported by the backward
    big = type(cloud)(cloud.means, np.clip(cloud.scales * 6.0, 0, 0.9).astype(np.float32), cloud.rotations, cloud.density)
    ref = util.oracle_raster_forward(big, view)
    assert ref["R"] > 2.5 * int(_C._Workspace.hints[key]) and ref["R"] > 12 * cloud.P
    t3, img3 = run(big)
    with pytest.raises(_C.CapacityOverflow):
        img3.sum().backward()
    t4, img4 = run(big)                            # the hint was raised: the repeated step fits
    img4.sum().backward()
    err = np.abs(img4[0].detach().cpu().numpy().astype(np.float64) - ref["image"]).max()
    assert err <= 1e-5 * np.abs(ref["image"]).max() + 1e-7
