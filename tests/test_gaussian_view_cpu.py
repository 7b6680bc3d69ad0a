"""The scene view's ellipsoid kind without a GPU: tests/gaussian_view_oracle.py against closed forms (sphere silhouettes
in both projections, depth, the quaternion's sign and convention, a camera inside, the near plane, the pixel box), the
`show_gaussians` selection and colours of `scene_view.gaussian_ellipsoids`, and the refusals."""
import math
import os
import re

import numpy as np
import pytest
import torch

import gaussian_view_oracle as go
import scene_view_oracle as so
from r2_gaussian_b200 import scene_view as sv
from r2_gaussian_b200 import visualize_scene
from r2_gaussian_b200.volume_render import look_at

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEAR = 1e-3


def _ell(centres, axes, quats, colours=None):
    n = len(centres)
    pos = np.zeros((n, 3, 3))
    pos[:, 0], pos[:, 1] = centres, axes
    meta = np.zeros((n, 2), np.int32)
    meta[:, 0] = go.ELLIPSOID
    attr = np.zeros((n, 12), np.float32)
    attr[:, 0:3] = 0.5 if colours is None else colours
    attr[:, 3:7] = quats
    return pos, meta, attr


def _raster(pos, meta, attr, cam, near=NEAR):
    return go.raster(pos, meta, attr, None, np.array([[0, 0, 0], [1, 1, 1]], np.float32), cam.record()[None],
                     cam.height, cam.width, cam.parallel, near, (1.0, 1.0, 1.0))


def _screen_cam(W, H):
    """Parallel, looking down -z from z = 10, one scene unit per pixel: world (X, Y) lands at screen (X, H - Y)."""
    return look_at((W / 2, H / 2, 10.0), (W / 2, H / 2, 0.0), (0, 1, 0), W, H, parallel_scale=H / 2)


def _kcam(cam):
    return so.Cam(cam.record(), cam.height, cam.width, cam.parallel)


def _z_at(cam, pos, attr, x, y, near=NEAR):
    """The oracle's float64 (covered, depth) of ellipsoid 0 at pixel (x, y)."""
    k = _kcam(cam)
    O, D = go.rays(k, np.array([x]), np.array([y]))
    cov, z = go.hit(go.Ellipsoids(pos[:1], attr[:1]), O, D, near)
    return bool(cov[0]), float(z[0])


def _ids(keys):
    return np.where(keys == so.EMPTY, -1, (keys & np.uint64(0xFFFFFFFF)).astype(np.int64))


def _depth(keys):
    return (keys >> np.uint64(32)).astype(np.uint32).view(np.float32)


@pytest.mark.parametrize("centre,r", [((12.5, 9.5), 4.3), ((7.5, 6.5), 0.6), ((20.31, 11.17), 3.05),
                                      ((3.77, 14.2), 6.4), ((25.0, 3.0), 2.5)])
def test_parallel_sphere_covers_the_pixel_centres_within_its_radius(centre, r):
    W, H = 32, 20
    cam = _screen_cam(W, H)
    cx, sy = centre
    cz = -1.25
    pos, meta, attr = _ell([(cx, H - sy, cz)], [(r, r, r)], [(0.3, -0.5, 0.1, 0.8)])
    keys, _ = _raster(pos, meta, attr, cam)
    ys, xs = np.mgrid[0:H, 0:W]
    dist = np.hypot(xs + 0.5 - cx, ys + 0.5 - sy)
    assert np.abs(dist - r).min() > 1e-9
    assert np.array_equal(keys[0] != so.EMPTY, dist <= r)
    if (cx - 0.5) % 1 == 0 and (sy - 0.5) % 1 == 0:
        hit, z = _z_at(cam, pos, attr, int(cx), int(sy))
        assert hit and abs(z - ((10.0 - cz) - r)) <= 1e-12


@pytest.mark.parametrize("seed", range(4))
def test_perspective_sphere_covers_the_rays_within_its_angular_radius(seed):
    rng = np.random.default_rng(seed)
    W, H = 41, 33
    cam = look_at(rng.uniform(-1, 1, 3) + (6, 0, 0), (0, 0, 0), (0, 0, 1), W, H, 40.0)
    c = rng.uniform(-0.6, 0.6, 3)
    r = rng.uniform(0.3, 1.2)
    pos, meta, attr = _ell([c], [(r, r, r)], [rng.normal(size=4)])
    keys, _ = _raster(pos, meta, attr, cam)
    k = _kcam(cam)
    ys, xs = np.mgrid[0:H, 0:W]
    _, D = go.rays(k, xs.ravel(), ys.ravel())
    v = c - np.asarray(k.P)
    cosang = (D @ v) / (np.linalg.norm(D, axis=1) * np.linalg.norm(v))
    limit = math.cos(math.asin(r / np.linalg.norm(v)))
    sure = np.abs(cosang - limit) > 1e-9
    covered = (keys[0] != so.EMPTY).ravel()
    assert sure.mean() > 0.99 and covered.any() and not covered.all()
    assert np.array_equal(covered[sure], (cosang >= limit)[sure])


def test_quaternion_sign_changes_nothing():
    rng = np.random.default_rng(3)
    n = 12
    c, s, q = rng.uniform(-1, 1, (n, 3)), rng.uniform(0.05, 0.6, (n, 3)), rng.normal(size=(n, 4))
    for cam in (look_at((4, -2, 1.5), (0, 0, 0), (0, 0, 1), 37, 29, 45.0),
                look_at((4, -2, 1.5), (0, 0, 0), (0, 0, 1), 37, 29, parallel_scale=1.8)):
        k1, rgb1 = _raster(*_ell(c, s, q), cam)
        k2, rgb2 = _raster(*_ell(c, s, -q), cam)
        assert (k1 != so.EMPTY).sum() > 50
        assert np.array_equal(k1, k2) and np.array_equal(rgb1, rgb2)


def test_a_quarter_turn_about_z_swaps_the_first_two_axes():
    W, H = 40, 30
    h = math.sqrt(0.5)
    s = np.array([[6.3, 2.2, 3.1], [1.4, 4.7, 0.9]])
    c = np.array([[14.2, 15.3, 0.0], [29.1, 12.6, -2.0]])
    for cam in (_screen_cam(W, H), look_at((20, -25, 30), (20, 15, 0), (0, 0, 1), W, H, 50.0)):
        k = _kcam(cam)
        ys, xs = np.mgrid[0:H, 0:W]
        O, D = go.rays(k, xs.ravel(), ys.ravel())
        masks = []
        for quat, ax in (((1.0, 0.0, 0.0, 0.0), s), ((h, 0.0, 0.0, h), s[:, [1, 0, 2]])):
            pos, meta, attr = _ell(c, ax, [quat] * 2)
            keys, _ = _raster(pos, meta, attr, cam)
            masks.append(keys[0].ravel() != so.EMPTY)
            E = go.Ellipsoids(pos, attr)
            rim = np.zeros(len(O), bool)
            for i in range(2):
                Ei = E.take(np.full(len(O), i))
                e, g = go._local(Ei.R, Ei.k, O - Ei.c), go._local(Ei.R, Ei.k, D)
                A, B, C = go._dot(g, g), go._dot(g, e), go._dot(e, e) - 1.0
                rim |= np.abs(B * B - A * C) <= 1e-9 * (B * B + np.abs(A * C))
            masks.append(rim)
        sure = ~(masks[1] | masks[3])
        assert masks[0].sum() > 20
        assert np.array_equal(masks[0][sure], masks[2][sure])


def test_camera_inside_sees_the_exit_surface_on_every_pixel():
    c, s = np.array([0.2, -0.1, 0.3]), np.array([2.0, 1.5, 1.2])
    q = np.array([0.9, 0.2, -0.3, 0.1])
    pos, meta, attr = _ell([c], [s], [q])
    for cam in (look_at((0.1, 0.0, 0.2), (1, 0.5, 0.3), (0, 0, 1), 31, 23, 100.0),
                look_at((0.4, 0.2, 0.1), (0.4, 0.2, 5.0), (0, 1, 0), 20, 20, 150.0)):
        keys, _ = _raster(pos, meta, attr, cam)
        assert (keys[0] != so.EMPTY).all()
        k = _kcam(cam)
        ys, xs = np.mgrid[0:cam.height, 0:cam.width]
        O, D = go.rays(k, xs.ravel(), ys.ravel())
        R = go.rotation(q[None].astype(np.float32))[0]
        e = ((O - c) @ R) / s
        g = (D @ R) / s
        A, B, C = (g * g).sum(1), (g * e).sum(1), (e * e).sum(1) - 1
        exit_t = (-B + np.sqrt(B * B - A * C)) / A
        _, z = go.hit(go.Ellipsoids(np.repeat(pos, len(O), 0), np.repeat(attr, len(O), 0)), O, D, NEAR)
        assert np.allclose(z, exit_t, rtol=1e-12, atol=0)
        assert np.array_equal(_depth(keys[0]).ravel(), exit_t.astype(np.float32))


def test_an_ellipsoid_across_the_near_plane_shows_its_inside():
    near = 0.5
    cam = look_at((0, 0, 0), (0, 0, 1), (0, 1, 0), 25, 25, 90.0)
    pos, meta, attr = _ell([(0.0, 0.0, 0.6)], [(0.3, 0.3, 0.3)], [(1, 0, 0, 0)])
    k = _kcam(cam)
    box = go.boxes(k, near, go.Ellipsoids(pos, attr))
    assert tuple(box[0]) == (0, 24, 0, 24)             # cut by the near plane: the whole frame
    keys, _ = _raster(pos, meta, attr, cam, near=near)
    hit, z = _z_at(cam, pos, attr, 12, 12, near)
    assert hit and abs(z - 0.9) < 1e-12                # the far side, not the front at 0.3
    ys, xs = np.mgrid[0:25, 0:25]
    O, D = go.rays(k, xs.ravel(), ys.ravel())
    # covered iff the ray meets the sphere and leaves it beyond the near plane
    c = np.array([0.0, 0.0, 0.6]) - np.asarray(k.P)
    dc, dd = D @ c, (D * D).sum(1)
    disc = dc * dc - dd * (c @ c - 0.09)
    far = (dc + np.sqrt(np.maximum(disc, 0))) / dd
    sure = (np.abs(disc) > 1e-9) & (np.abs(far - near) > 1e-9)
    covered = keys[0].ravel() != so.EMPTY
    assert np.array_equal(covered[sure], ((disc >= 0) & (far >= near))[sure])
    assert covered.sum() > 100 and not covered.all()
    # wholly in front of the near plane: nothing, and an empty box
    pos2 = pos.copy()
    pos2[0, 0] = (0.0, 0.0, 0.1)
    assert go.boxes(k, near, go.Ellipsoids(pos2, attr))[0, 1] < 0
    assert (_raster(pos2, meta, attr, cam, near=near)[0] == so.EMPTY).all()


@pytest.mark.parametrize("parallel", [False, True])
def test_the_ray_test_never_covers_a_pixel_outside_the_box(parallel):
    rng = np.random.default_rng(7 + parallel)
    W, H = 47, 35
    n = 400
    c = rng.uniform(-2, 2, (n, 3))
    s = np.exp(rng.uniform(np.log(0.002), np.log(1.5), (n, 3)))    # sub-pixel to larger than the frame
    s[:20] = rng.uniform(1e-4, 5e-3, (20, 3))
    q = rng.normal(size=(n, 4))
    pos, meta, attr = _ell(c, s, q)
    E = go.Ellipsoids(pos, attr)
    kw = {"parallel_scale": 2.5} if parallel else {}
    for eye in ((5, -3, 2), (1.9, 1.2, -0.8), (0.3, 0.2, 0.1)):   # far, close to some, inside some
        cam = look_at(eye, (0, 0, 0), (0, 0, 1), W, H, 60.0, **kw)
        k = _kcam(cam)
        box = go.boxes(k, NEAR, E)
        full = np.tile(np.array([[0, W - 1, 0, H - 1]]), (n, 1))
        prim, xs, ys = go._pairs(full, (0, H, 0, W))
        O, D = go.rays(k, xs, ys)
        cov, _ = go.hit(E.take(prim), O, D, NEAR)
        b = box[prim[cov]]
        inside = (xs[cov] >= b[:, 0]) & (xs[cov] <= b[:, 1]) & (ys[cov] >= b[:, 2]) & (ys[cov] <= b[:, 3])
        assert cov.sum() > 100 and inside.all()
        small = (box[:, 1] - box[:, 0] < 16) & (box[:, 3] - box[:, 2] < 16) & (box[:, 1] >= box[:, 0])
        assert small.any()


@pytest.mark.parametrize("theta", [0.4, 1.1, 2.6])
def test_the_quaternion_is_read_scalar_first_as_the_rasterizer_reads_it(theta):
    """(cos t/2, 0, 0, sin t/2) with its long axis on x appears turned by t about z, along the principal axis of the
    rasterizer's covariance (scalar-last reading, the reference's create_o3d_ellipse, would turn it elsewhere)."""
    from r2_gaussian_b200.gaussian_utils import build_scaling_rotation
    W = H = 64
    cam = _screen_cam(W, H)
    quat = np.array([math.cos(theta / 2), 0.0, 0.0, math.sin(theta / 2)])
    axes = np.array([20.0, 4.0, 4.0])
    pos, meta, attr = _ell([(32.0, 32.0, 0.0)], [axes], [quat])
    keys, _ = _raster(pos, meta, attr, cam)
    ys, xs = np.nonzero(keys[0] != so.EMPTY)
    X, Y = xs + 0.5 - 32.0, -(ys + 0.5 - 32.0)          # world x, y
    mxx, myy, mxy = (X * X).mean(), (Y * Y).mean(), (X * Y).mean()
    image_angle = 0.5 * math.atan2(2 * mxy, mxx - myy)
    L = build_scaling_rotation(torch.from_numpy(axes[None]), torch.from_numpy(quat[None]))
    cov = (L @ L.transpose(1, 2))[0].numpy()
    w, v = np.linalg.eigh(cov[:2, :2])
    cov_angle = math.atan2(v[1, -1], v[0, -1])

    def close(a, b):
        d = (a - b) % math.pi
        return min(d, math.pi - d) < math.radians(1.0)

    assert close(image_angle, theta) and close(cov_angle, theta)
    from scipy.spatial.transform import Rotation
    wrong = Rotation.from_quat(quat).as_matrix() @ np.diag(axes)
    w2, v2 = np.linalg.eigh((wrong @ wrong.T)[:2, :2])
    assert not close(math.atan2(v2[1, -1], v2[0, -1]), theta) or w2[-1] < 0.5 * axes[0] ** 2


class _Model:
    def __init__(self, xyz, dens, scale, rot):
        self.get_xyz, self.get_density = torch.from_numpy(xyz), torch.from_numpy(dens)
        self.get_scaling, self.get_rotation = torch.from_numpy(scale), torch.from_numpy(rot)


def _show_gaussians_selection(m, n_gaussian, sort):
    """numpy restatement of the reference's show_gaussians selection and vertex colour (a stable sort)."""
    d = m.get_density.numpy()[:, 0]
    keep = np.nonzero(d != 0)[0]
    dk = d[keep]
    if sort == "density":
        keep = keep[np.argsort(-dk, kind="stable")]
    elif sort == "scale":
        s = m.get_scaling.numpy()[keep]
        keep = keep[np.argsort(-(((s[:, 0] + s[:, 1]) + s[:, 2]) / np.float32(3)), kind="stable")]
    scale = np.float32(0.95) / dk.max()
    if n_gaussian is not None:
        keep = keep[:n_gaussian]
    return keep, d[keep] * scale


@pytest.mark.parametrize("sort", ["no", "density", "scale"])
@pytest.mark.parametrize("n_gaussian", [None, 7, 10_000])
def test_selection_and_colours_follow_show_gaussians(sort, n_gaussian):
    rng = np.random.default_rng(11)
    n = 300
    dens = rng.random((n, 1)).astype(np.float32)
    dens[rng.random(n) < 0.2] = 0.0
    dens[50:60] = dens[40]                                  # ties
    scale = rng.uniform(0.01, 0.2, (n, 3)).astype(np.float32)
    scale[70:80] = scale[65]
    rot = rng.normal(size=(n, 4)).astype(np.float32)
    rot /= np.linalg.norm(rot, axis=1, keepdims=True)
    m = _Model(rng.normal(size=(n, 3)).astype(np.float32), dens, scale, rot)
    prims, idx = sv.gaussian_ellipsoids(m, n_gaussian, sort)
    keep, grey = _show_gaussians_selection(m, n_gaussian, sort)
    assert np.array_equal(idx.numpy(), keep)
    assert len(prims) == min(n_gaussian or n, int((dens != 0).sum()))
    assert np.array_equal(prims.attr[:, 0].numpy(), grey) and np.array_equal(prims.attr[:, 2].numpy(), grey)
    assert np.array_equal(prims.attr[:, 3:7].numpy(), rot[keep])
    assert np.array_equal(prims.pos[:, 0].numpy(), m.get_xyz.numpy()[keep].astype(np.float64))
    assert np.array_equal(prims.pos[:, 1].numpy(), scale[keep].astype(np.float64))
    assert (prims.meta[:, 0] == sv.ELLIPSOID).all()


def test_ellipsoid_refusals():
    cam = look_at((0, 0, 5), (0, 0, 0), (0, 1, 0), 8, 8)
    good = sv.ellipsoids([[0, 0, 0]], [[1, 1, 1]], [[1, 0, 0, 0]], (1, 0, 0), device="cpu")
    for change, needle in ((lambda p: p.pos.__setitem__((0, 1, 2), 0.0), "semi-axis"),
                           (lambda p: p.pos.__setitem__((0, 1, 0), -1.0), "semi-axis"),
                           (lambda p: p.pos.__setitem__((0, 1, 1), float("inf")), "finite"),
                           (lambda p: p.attr.__setitem__((0, slice(3, 7)), 0.0), "quaternion"),
                           (lambda p: p.meta.__setitem__((0, 0), 5), "kind")):
        bad = sv.Primitives(good.pos.clone(), good.meta.clone(), good.attr.clone())
        change(bad)
        with pytest.raises(ValueError, match=needle):
            sv.render(bad, cam)
    m = _Model(np.zeros((2, 3), np.float32), np.zeros((2, 1), np.float32), np.ones((2, 3), np.float32),
               np.tile(np.float32([1, 0, 0, 0]), (2, 1)))
    with pytest.raises(ValueError, match="density 0"):
        sv.gaussian_ellipsoids(m)
    m.get_density[0] = 1.0
    for kw in ({"n_gaussian": 0}, {"sort_gaussians": "size"}):
        with pytest.raises(ValueError):
            sv.gaussian_ellipsoids(m, **kw)
    header = open(os.path.join(ROOT, "include", "r2x.h")).read()
    assert int(re.search(r"#define R2X_SV_ELLIPSOID (\d+)", header).group(1)) == sv.ELLIPSOID == go.ELLIPSOID


def test_cli_gaussians_parses_and_refuses(tmp_path):
    model = tmp_path / "model"
    model.mkdir()
    out = str(tmp_path / "g.png")
    a = visualize_scene.parse_args(["-m", str(model), "--gaussians", "--output", out])
    assert a.gaussians and a.n_gaussian is None and a.sort_gaussians == "no"
    a = visualize_scene.parse_args(["-m", str(model), "--gaussians", "--sort_gaussians", "density", "--n_gaussian",
                                    "20000", "--output", out])
    assert (a.sort_gaussians, a.n_gaussian) == ("density", 20000)
    assert visualize_scene.parse_args(["-m", str(model), "--output", out]).sort_gaussians == "no"
    vol = tmp_path / "v.npy"
    np.save(vol, np.zeros((4, 4, 4), np.float32))
    bad = [["-s", str(model), "--gaussians", "--output", out],
           ["--vol", str(vol), "--gaussians", "--output", out],
           ["-m", str(model), "--gaussians", "--resolution", "64", "--output", out],
           ["-m", str(model), "--gaussians", "--vol", str(vol), "--output", out],
           ["-m", str(model), "--gaussians", "--n_gaussian", "0", "--output", out],
           ["-m", str(model), "--n_gaussian", "5", "--output", out],
           ["-m", str(model), "--sort_gaussians", "density", "--output", out],
           ["-m", str(model), "--gaussians", "--sort_gaussians", "size", "--output", out]]
    for argv in bad:
        with pytest.raises(SystemExit):
            visualize_scene.parse_args(argv)
