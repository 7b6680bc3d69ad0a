"""Batched views: N views of one cloud in one call (r2x_raster_forward_views_async / r2x_raster_backward_views).

Every image of the batch must be bit for bit the single-view forward of that view, radii included, and every
per-Gaussian gradient bit for bit the single-view gradients summed in view order in float32 (acc = g[0]; acc = acc +
g[v]); the per-view dL/dmean2D equals the single view's.  Cases cover both binning paths of the stacked tile grid (the
direct path up to 4096 tiles, the radix path beyond), parallel beam, a detector that is not a multiple of 16 (a partial
tile row at every band edge), Gaussians culled in some views only, P = 0 and a capacity overflow."""
import math
import types

import numpy as np
import pytest
import torch

import util
from r2_gaussian_b200 import _C, engine, scene
from r2_gaussian_b200.rasterization import GaussianRasterizationSettings, GaussianRasterizer, rasterize_views
from r2_gaussian_b200.render_query import render, render_views

pytestmark = pytest.mark.gpu


def _bits(a: torch.Tensor) -> torch.Tensor:
    return a.contiguous().view(torch.int32)


def _bit_equal(a: torch.Tensor, b: torch.Tensor) -> bool:
    return a.shape == b.shape and _bits(a).equal(_bits(b))


def _inputs(cloud, views):
    t = util.to_torch(cloud, None)
    t["views"] = torch.stack([torch.tensor(v.viewmatrix, device="cuda") for v in views])
    t["projs"] = torch.stack([torch.tensor(v.projmatrix, device="cuda") for v in views])
    return t


def _single(t, view, v, dL=None):
    """Single-view forward (the asynchronous C entry point, retried until it fits) and, with dL, its backward."""
    R, color, radii, geom, binning, img = _C.rasterize_gaussians(
        t["means"], t["dens"], t["scales"], t["rots"], 1.0, torch.Tensor([]), t["views"][v], t["projs"][v],
        view.tanfovx, view.tanfovy, view.image_height, view.image_width, torch.zeros(3), False, view.mode, False)
    out = dict(image=color[0], radii=radii)
    if dL is not None:
        g = _C.rasterize_gaussians_backward(
            t["means"], radii, t["scales"], t["rots"], 1.0, torch.Tensor([]), t["views"][v], t["projs"][v],
            view.tanfovx, view.tanfovy, dL[v:v + 1], torch.zeros(3), geom, R, binning, img, view.mode, False)
        out.update(zip(("mean2D", "opacity", "mu", "mean3D", "cov3D", "scale", "rot"), g))
    return out


def _batched(t, views, dL=None):
    v0 = views[0]
    R, images, radii, geom, binning, img = _C.rasterize_views(
        t["means"], t["dens"], t["scales"], t["rots"], 1.0, t["views"], t["projs"], v0.tanfovx, v0.tanfovy,
        v0.image_height, v0.image_width, v0.mode)
    out = dict(images=images, radii=radii, R=int(R))
    if dL is not None:
        g = _C.rasterize_views_backward(t["means"], radii, t["scales"], t["rots"], 1.0, t["views"], t["projs"],
                                        v0.tanfovx, v0.tanfovy, dL, geom, R, binning, img, v0.mode)
        out.update(zip(("mean2D", "opacity", "mean3D", "cov3D", "scale", "rot"), g))
    return out


def _dL(views, seed=0):
    v0 = views[0]
    gen = torch.Generator("cuda").manual_seed(seed)
    return torch.randn((len(views), v0.image_height, v0.image_width), device="cuda", generator=gen)


def _check_forward(cloud, views):
    t = _inputs(cloud, views)
    b = _batched(t, views)
    assert b["images"].shape == (len(views), views[0].image_height, views[0].image_width)
    for v, view in enumerate(views):
        s = _single(t, view, v)
        assert _bit_equal(b["images"][v], s["image"]), f"view {v}: image differs from the single-view render"
        assert b["radii"][v].equal(s["radii"]), f"view {v}: radii differ"
    return t, b


def _check_backward(cloud, views, seed=0):
    t = _inputs(cloud, views)
    dL = _dL(views, seed)
    b = _batched(t, views, dL)
    acc = None
    for v, view in enumerate(views):
        s = _single(t, view, v, dL)
        assert _bit_equal(b["images"][v], s["image"]), f"view {v}: image"
        assert _bit_equal(b["mean2D"][v], s["mean2D"]), f"view {v}: dL/dmean2D differs from the single view's"
        g = {k: s[k] for k in ("opacity", "mean3D", "cov3D", "scale", "rot")}
        acc = {k: x.clone() for k, x in g.items()} if acc is None else {k: acc[k] + g[k] for k in acc}
    for k, want in acc.items():
        assert _bit_equal(b[k], want), f"{k}: not the view-ordered float32 sum of the single-view gradients"
    return b


def _bench_scene():
    sc = scene.cone_beam_scanner(512, 256)
    return scene.make_cloud(100_000, kind="init", seed=0), scene.make_views(sc, 50)


def _mid_scene():
    sc = scene.cone_beam_scanner(256, 256)
    return scene.make_cloud(50_000, kind="init", seed=3), scene.make_views(sc, 50)


@pytest.mark.parametrize("n", [1, 3, 8])
def test_bench_scene_forward_bits(n):
    cloud, views = _bench_scene()
    _check_forward(cloud, views[::max(1, 50 // n)][:n])


@pytest.mark.parametrize("n", [16, 50])
def test_50k_256_forward_bits(n):
    """N = 16: 4096 tiles, the direct path's limit; N = 50: 12800 tiles, the radix path."""
    cloud, views = _mid_scene()
    _check_forward(cloud, views[:n] if n == 50 else views[::3][:n])


def test_parallel_beam_forward_and_backward_bits():
    sc = scene.parallel_beam_scanner(96, 64)
    views = [scene.make_view(sc, a) for a in (0.1, 1.3, 2.9, 4.4)]
    _check_backward(scene.make_cloud(2000, kind="trained", seed=5), views)


def test_ragged_detector_forward_and_backward_bits():
    """200 x 136 pixels: 13 x 9 tiles with a partial last tile row (and column) at every band edge."""
    sc = scene.cone_beam_scanner(200, 64)
    sc["nDetector"] = [200, 136]
    sc["sDetector"] = [4.0 * 200 / 512 * 2, 4.0 * 136 / 512 * 2]
    views = [scene.make_view(sc, a) for a in (0.2, 0.9, 2.5)]
    _check_backward(scene.make_cloud(3000, kind="trained", seed=7), views, seed=1)


def test_culled_in_some_views_only():
    """Gaussians beyond the source circle sit behind the source in the views that face them, in front in others."""
    cloud = scene.make_cloud(3000, kind="trained", seed=11)
    cloud.means[:64] = np.float32([6.0, 0.0, 0.0]) + 0.05 * cloud.means[:64]
    sc = scene.cone_beam_scanner(128, 64)
    views = [scene.make_view(sc, a) for a in (0.0, math.pi, 0.5 * math.pi)]
    _, b = _check_forward(cloud, views)
    r = b["radii"][:, :64]
    assert (r[0] == 0).all() and (r[1] > 0).any(), "the case does not cull in some views only"
    _check_backward(cloud, views, seed=2)


def test_bench_scene_backward_bits():
    cloud, views = _bench_scene()
    _check_backward(cloud, [views[0], views[17], views[34]])


def test_radix_path_backward_bits():
    cloud, views = _mid_scene()
    _check_backward(cloud, views[:20])   # 5120 tiles


def test_one_view_equals_the_single_path():
    cloud, views = _bench_scene()
    b = _check_backward(cloud, views[5:6], seed=4)
    assert b["mean2D"].shape == (1, cloud.P, 3)


def test_empty_cloud():
    sc = scene.cone_beam_scanner(64, 32)
    views = [scene.make_view(sc, a) for a in (0.0, 1.0)]
    cloud = scene.make_cloud(1, kind="trained", seed=0)
    t = _inputs(cloud, views)
    for k in ("means", "scales", "rots", "dens"):
        t[k] = t[k][:0]
    b = _batched(t, views, _dL(views))
    assert b["R"] == 0 and b["images"].abs().sum().item() == 0 and b["radii"].shape == (2, 0)
    assert b["mean2D"].shape == (2, 0, 3) and b["opacity"].shape == (0, 1)


def test_capacity_overflow_repeated():
    """An engine provisioned far too small overflows, grows and re-runs; forcing the overflow again gives the same
    bits, and they are the single-view images."""
    cloud, views = _mid_scene()
    views = views[:6]
    t = _inputs(cloud, views)
    eng = engine.RasterEngine(cloud.P, views[0].image_width, views[0].image_height, capacity=4096)
    results = []
    for _ in range(2):
        eng._reserve(4096)
        args = (t["means"], t["dens"], t["scales"], t["rots"], t["views"], t["projs"], views[0].tanfovx,
                views[0].tanfovy, views[0].mode)
        eng.forward_views(*args)
        assert not eng.check(), "the forward should have overflowed"
        eng.forward_views(*args)
        assert eng.check()
        results.append((eng.forward_views(*args).clone(), eng.views_radii(len(views)).clone()))
    assert _bit_equal(results[0][0], results[1][0]) and results[0][1].equal(results[1][1])
    for v, view in enumerate(views):
        s = _single(t, view, v)
        assert _bit_equal(results[0][0][v], s["image"]) and results[0][1][v].equal(s["radii"])


def test_two_runs_bitwise_equal():
    cloud, views = _mid_scene()
    t = _inputs(cloud, views[:12])
    dL = _dL(views[:12])
    a, b = _batched(t, views[:12], dL), _batched(t, views[:12], dL)
    for k in ("images", "mean2D", "opacity", "mean3D", "cov3D", "scale", "rot"):
        assert _bit_equal(a[k], b[k]), k
    assert a["radii"].equal(b["radii"])


def test_autograd_matches_a_loop_of_single_renders():
    sc = scene.cone_beam_scanner(128, 64)
    views = [scene.make_view(sc, a) for a in (0.3, 1.1, 2.0, 3.7)]
    cloud = scene.make_cloud(4000, kind="trained", seed=9)
    t = _inputs(cloud, views)
    dL = _dL(views, 5)
    v0 = views[0]

    def settings(v):
        return GaussianRasterizationSettings(v0.image_height, v0.image_width, v0.tanfovx, v0.tanfovy, 1.0,
                                             t["views"][v], t["projs"][v], torch.zeros(3, device="cuda"), False,
                                             v0.mode, False)

    leaves = [x.detach().clone().requires_grad_(True) for x in (t["means"], t["dens"], t["scales"], t["rots"])]
    means2D = torch.zeros((len(views), cloud.P, 3), device="cuda", requires_grad=True)
    images, _ = rasterize_views(leaves[0], leaves[1], leaves[2], leaves[3], t["views"], t["projs"], settings(0),
                                means2D=means2D)
    (images * dL).sum().backward()
    loop = [x.detach().clone().requires_grad_(True) for x in (t["means"], t["dens"], t["scales"], t["rots"])]
    loop2D = []
    total = 0
    for v in range(len(views)):
        m2 = torch.zeros((cloud.P, 3), device="cuda", requires_grad=True)
        loop2D.append(m2)
        img, _ = GaussianRasterizer(settings(v))(loop[0], m2, loop[1], loop[2], loop[3])
        total = total + (img[0] * dL[v]).sum()
    total.backward()
    for got, want in zip(leaves, loop):
        scale = want.grad.abs().max().item()
        assert (got.grad - want.grad).abs().max().item() <= 1e-6 * scale, "gradient differs beyond 1e-6 relative"
    for v in range(len(views)):
        assert _bit_equal(means2D.grad[v], loop2D[v].grad)


def test_render_views_matches_render():
    sc = scene.cone_beam_scanner(96, 64)
    cams = [scene.camera_from_view(scene.make_view(sc, a)) for a in (0.4, 2.2, 5.0)]
    cloud = scene.make_cloud(1500, kind="trained", seed=2)
    t = util.to_torch(cloud, None)
    pc = types.SimpleNamespace(get_xyz=t["means"], get_density=t["dens"], get_scaling=t["scales"],
                               get_rotation=t["rots"])
    pipe = types.SimpleNamespace(debug=False, compute_cov3D_python=False)
    out = render_views(cams, pc, pipe)
    assert out["render"].shape == (3, 1, 96, 96) and out["viewspace_points"].shape == (3, cloud.P, 3)
    for v, cam in enumerate(cams):
        one = render(cam, pc, pipe)
        assert _bit_equal(out["render"][v], one["render"]) and out["radii"][v].equal(one["radii"])
        assert out["visibility_filter"][v].equal(one["visibility_filter"])
