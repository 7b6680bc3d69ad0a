"""The scene view's ellipsoid kind on the GPU against tests/gaussian_view_oracle.py: depth-id keys bit for bit and
colours within 1e-6 on random soups mixing ellipsoids with triangles and lines (odd sizes, both projections), around
the 16-pixel split (a camera inside, near-plane cuts, sub-pixel ellipsoids), orbits equal to single frames, windows of a
500k-Gaussian cloud, and `visualize_scene --gaussians` end to end on a trained model and on a hand-written one."""
import json
import math
import pickle
import shutil

import numpy as np
import pytest
import torch

import gaussian_view_oracle as go
import scene_view_oracle as so
import volume_render_oracle as vo
from r2_gaussian_b200 import scene_view as sv
from r2_gaussian_b200.volume_render import look_at, to_uint8
from test_scene_view_gpu import LUT, _gpu, _soup

pytestmark = pytest.mark.gpu
TOL = 1e-6


def _ellipsoid_rows(rng, n, spread, size):
    pos = np.zeros((n, 3, 3))
    pos[:, 0] = rng.uniform(-spread, spread, (n, 3))
    pos[:, 1] = size * np.exp(rng.uniform(np.log(0.01), 0.0, (n, 3)))
    meta = np.zeros((n, 2), np.int32)
    meta[:, 0] = go.ELLIPSOID
    attr = np.zeros((n, 12), np.float32)
    attr[:, 0:3] = rng.random((n, 3))
    attr[:, 3:7] = rng.normal(size=(n, 4))
    return pos, meta, attr


def _mix(rng, n_tri, n_line, n_ell, spread, size):
    pos, meta, attr, tex = _soup(rng, n_tri, n_line, spread, size)
    ep, em, ea = _ellipsoid_rows(rng, n_ell, spread, size)
    order = rng.permutation(len(pos) + n_ell)                 # ellipsoids interleaved with the other kinds
    return (np.concatenate([pos, ep])[order], np.concatenate([meta, em])[order], np.concatenate([attr, ea])[order],
            tex)


def _compare(pos, meta, attr, tex, cams, near=sv.NEAR, bg=(1.0, 1.0, 1.0), window=None, prims=None):
    prims = _gpu(pos, meta, attr, tex) if prims is None else prims
    rgb, keys = sv.render(prims, cams, background=bg, lut=LUT, near=near, return_keys=True)
    c0 = cams[0]
    recs = np.stack([c.record() for c in cams])
    okeys, orgb = go.raster(pos, meta, attr, tex, LUT, recs, c0.height, c0.width, c0.parallel, near, bg, window)
    k = keys.cpu().numpy().view(np.uint64)
    g = rgb.cpu().numpy()
    if window is not None:
        y0, y1, x0, x1 = window
        k, okeys = k[:, y0:y1, x0:x1], okeys[:, y0:y1, x0:x1]
        g, orgb = g[:, y0:y1, x0:x1], orgb[:, y0:y1, x0:x1]
    assert np.array_equal(k, okeys), int((k != okeys).sum())
    assert np.abs(g - orgb).max() <= TOL
    return k


def _ids(k):
    return (k & np.uint64(0xFFFFFFFF)).astype(np.int64)


@pytest.mark.parametrize("HW", [(17, 23), (15, 16), (16, 17), (33, 31), (1, 40), (48, 1)])
@pytest.mark.parametrize("parallel", [False, True])
def test_mixed_soups_equal_the_oracle(HW, parallel):
    H, W = HW
    rng = np.random.default_rng(H * 100 + W + parallel)
    pos, meta, attr, tex = _mix(rng, 80, 40, 80, 1.0, 0.6)
    kw = {"parallel_scale": 1.6} if parallel else {}
    cams = [look_at((3.5, -2.0, 1.5), (0, 0, 0), (0, 0, 1), W, H, 45.0, **kw),
            look_at((0.2, 0.1, 0.3), (1, 1, 0), (0, 0, 1), W, H, 120.0, **kw)]    # inside the soup: near cuts
    k = _compare(pos, meta, attr, tex, cams)
    if min(H, W) > 1:
        assert (meta[_ids(k[k != so.EMPTY]), 0] == go.ELLIPSOID).any()


@pytest.mark.parametrize("extent", [14.0, 15.5, 16.0, 16.5, 17.0, 31.5, 32.5, 200.0])
def test_boxes_around_the_tile_split(extent):
    """Ellipsoids whose pixel box is just below, at and above 16 pixels and far above it; sub-pixel ones; one holding
    the perspective camera and ones cut by its near plane."""
    W, H = 37, 29
    cam = look_at((W / 2, H / 2, 10.0), (W / 2, H / 2, 0.0), (0, 1, 0), W, H, parallel_scale=H / 2)
    persp = look_at((W / 2 + 3, H / 2 - 4, 30.0), (W / 2, H / 2, 0.0), (0, 1, 0), W, H, 60.0)
    rng = np.random.default_rng(int(extent * 10))
    n = 14
    pos = np.zeros((n + 6, 3, 3))
    pos[:n, 0] = np.stack([rng.uniform(-3, 40, n), rng.uniform(-3, 32, n), rng.uniform(-2, 2, n)], 1)
    # a box of ~extent pixels: 2 s + 3 (one pixel of widening each side, plus the floor)
    pos[:n, 1] = np.stack([np.full(n, (extent - 3) / 2), rng.uniform(1.0, (extent - 3) / 2, n), rng.uniform(1, 5, n)], 1)
    pos[n:n + 3, 0] = rng.uniform(0, 30, (3, 3))
    pos[n:n + 3, 0, 2] = (-1.0, 0.5, 1.5)                                               # in front of cam
    pos[n:n + 3, 1] = rng.uniform(0.05, 0.3, (3, 3))                                   # sub-pixel
    pos[n + 3, 0], pos[n + 3, 1] = (W / 2 + 3, H / 2 - 4, 30.0), (4.0, 6.0, 3.0)       # holds persp's camera
    pos[n + 4, 0], pos[n + 4, 1] = (W / 2 + 3, H / 2 - 4, 30.0 - 0.6), (1.5, 0.8, 0.5999)   # cut by near
    pos[n + 5, 0], pos[n + 5, 1] = (W / 2 + 2, H / 2 - 3, 29.0), (2.0, 1.0, 1.2)      # cut by near, off-axis
    meta = np.zeros((len(pos), 2), np.int32)
    meta[:, 0] = go.ELLIPSOID
    attr = np.zeros((len(pos), 12), np.float32)
    attr[:, 0:3] = rng.random((len(pos), 3))
    attr[:, 3:7] = rng.normal(size=(len(pos), 4))
    phi = rng.uniform(0, 2 * math.pi, n)                  # the sized ones turn about the view axis only
    attr[:n, 3:7] = np.stack([np.cos(phi / 2), 0 * phi, 0 * phi, np.sin(phi / 2)], 1)
    tex = np.zeros((1, 1, 1), np.float32)
    k = _compare(pos, meta, attr, tex, [cam], near=0.05)
    assert (k != so.EMPTY).any()
    kp = _compare(pos, meta, attr, tex, [persp], near=0.05)
    assert (kp != so.EMPTY).all()                            # the camera is inside one of them
    assert set(_ids(kp).ravel().tolist()) & {n + 3, n + 4, n + 5}
    # the tile split itself: which ellipsoids take the tile path in the parallel view
    E = go.Ellipsoids(pos, attr)
    box = go.boxes(so.Cam(cam.record(), H, W, True), 0.05, E)
    big = (box[:, 1] - box[:, 0] >= 16) | (box[:, 3] - box[:, 2] >= 16)
    if extent >= 31.5:
        assert big.any()
    assert (~big[n:n + 3] & (box[n:n + 3, 1] >= box[n:n + 3, 0])).all()


def test_orbit_equals_single_frames_and_is_reproducible():
    rng = np.random.default_rng(5)
    pos, meta, attr, tex = _mix(rng, 200, 60, 300, 1.0, 0.4)
    prims = _gpu(pos, meta, attr, tex)
    cams = sv.scan_orbit(look_at((3, 1, 2), (0, 0, 0), (0, 0, 1), 45, 33, 40.0), 7)
    rgb, keys = sv.render(prims, cams, lut=LUT, return_keys=True)
    rgb2, keys2 = sv.render(prims, cams, lut=LUT, return_keys=True)
    assert torch.equal(keys, keys2) and torch.equal(rgb, rgb2)
    for i, c in enumerate(cams):
        r1, k1 = sv.render(prims, c, lut=LUT, return_keys=True)
        assert torch.equal(k1[0], keys[i]) and torch.equal(r1[0], rgb[i])
    _compare(pos, meta, attr, tex, cams[:3], prims=prims)


def test_trained_cloud_windows_equal_the_oracle():
    from r2_gaussian_b200 import scene
    cloud = scene.make_cloud(500_000, kind="trained", seed=3)
    dens = cloud.density[:, 0]
    colours = np.repeat((dens * (np.float32(0.95) / dens.max()))[:, None], 3, 1)
    prims = sv.ellipsoids(cloud.means, cloud.scales, cloud.rotations, colours)
    W, H = 1000, 800
    cam = sv.default_view(prims, W, H)
    pos, meta, attr = (t.cpu().numpy() for t in (prims.pos, prims.meta, prims.attr))
    tex = np.zeros((1, 1, 1), np.float32)
    for win in ((390, 410, 490, 510), (200, 216, 300, 331), (600, 611, 640, 660), (0, 9, 0, 1000)):
        k = _compare(pos, meta, attr, tex, [cam], window=win, prims=prims)
    close = look_at((0.05, -0.1, 0.02), (1, 1, 0), (0, 0, 1), W, H, 60.0)      # among the Gaussians
    k = _compare(pos, meta, attr, tex, [close], window=(390, 414, 490, 514), prims=prims)
    assert (k != so.EMPTY).mean() > 0.5


# ---- visualize_scene --gaussians end to end -------------------------------------------------------------------------

@pytest.fixture(scope="module")
def trained(tmp_path_factory):
    from r2_gaussian_b200 import generate_data, initialize_pcd, scene, trainer
    from test_volume_render_gpu import _smooth
    tmp = tmp_path_factory.mktemp("gaussian_view")
    n = 32
    np.save(tmp / "vol.npy", _smooth((n, n, n)).clip(0, 1))
    sc = scene.cone_beam_scanner(48, n)
    phys = {k: (np.asarray(v, float) * 2.0).tolist() if k in ("DSD", "DSO", "sDetector", "sVoxel", "offOrigin")
            else v for k, v in sc.items()}
    phys.update({"offDetector": [0.0, 0.0], "filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0,
                 "noise": False})
    (tmp / "scan.yml").write_text("".join(f"{k}: {json.dumps(v)}\n" for k, v in phys.items()))
    data = generate_data.main(["--vol", str(tmp / "vol.npy"), "--scanner", str(tmp / "scan.yml"), "--n_train", "8",
                               "--n_test", "2", "--output", str(tmp / "scene")])
    init = initialize_pcd.main(["--data", data, "--n_points", "3000", "--output", str(tmp / "init.npy")])
    model = tmp / "model"
    trainer.main(["-s", data, "-m", str(model), "--ply_path", init, "--iterations", "100", "--test_iterations", "100",
                  "--save_iterations", "100"])
    return {"scene": data, "model": model, "tmp": tmp}


def _run(argv, capsys):
    from r2_gaussian_b200 import visualize_scene
    capsys.readouterr()
    rep, frames, prims, cams = visualize_scene.run(argv)
    line = capsys.readouterr().out.strip().splitlines()[-1]
    assert json.loads(line) == json.loads(json.dumps(rep))
    imgs = to_uint8(frames).cpu().numpy()
    pngs = [p for p in rep["outputs"] if p.endswith(".png")]
    assert len(pngs) == rep["frames"] == frames.shape[0]
    for p, img in zip(pngs, imgs):
        assert np.array_equal(vo.read_png(p), img), p
    assert torch.equal(frames, sv.render(prims, cams))
    return rep, frames, prims, cams


def test_visualize_scene_gaussians_end_to_end(trained, tmp_path, capsys):
    from r2_gaussian_b200.extract_mesh import load_model
    from r2_gaussian_b200.visualize_scene import parse_args
    model = str(trained["model"])
    rep, frames, prims, cams = _run(["-m", model, "--gaussians", "--sort_gaussians", "density", "--n_gaussian", "500",
                                     "--width", "160", "--height", "120", "--no_images",
                                     "--output", str(tmp_path / "g.png")], capsys)
    _, gaussians, _, _ = load_model(parse_args(["-m", model, "--gaussians", "--output", str(tmp_path / "x.png")]))
    n_kept = int((gaussians.get_density[:, 0] != 0).sum())
    assert rep["gaussians"] == min(500, n_kept) and rep["triangles"] == 0 and rep["cameras"] == 8
    ell, idx = sv.gaussian_ellipsoids(gaussians, 500, "density")
    assert torch.equal(prims.pos[:len(ell)], ell.pos) and torch.equal(prims.attr[:len(ell)], ell.attr)
    dens = gaussians.get_density[idx, 0]
    assert bool((dens[:-1] >= dens[1:]).all())
    _, keys = sv.render(prims, cams, return_keys=True)
    k = keys.cpu().numpy().view(np.uint64)
    assert (_ids(k[k != so.EMPTY]) < len(ell)).sum() > 100
    # every Gaussian, an orbit, and the mesh path's report unchanged
    rep, frames, prims, cams = _run(["-m", model, "--gaussians", "--orbit", "3", "--width", "64", "--height", "48",
                                     "--output", str(tmp_path / "o.png")], capsys)
    assert rep["gaussians"] == n_kept and rep["frames"] == 3
    rep, _, _, _ = _run(["-m", model, "--no_images", "--width", "64", "--height", "48",
                         "--output", str(tmp_path / "m.png")], capsys)
    assert "gaussians" not in rep and rep["triangles"] > 0


def test_three_gaussians_have_their_analytic_colours(trained, tmp_path, capsys):
    """A hand-written model: each Gaussian's centre pixel has the grey of its density lit by the analytic normal of
    the 1-sigma ellipsoid, and the needle turned 60 degrees about z is drawn along its covariance's long axis."""
    from r2_gaussian_b200.gaussian_utils import build_scaling_rotation
    model = tmp_path / "three"
    it = model / "point_cloud" / "iteration_1"
    it.mkdir(parents=True)
    for name in ("cfg_args", "cfg_args.json"):
        if (trained["model"] / name).exists():
            shutil.copy(trained["model"] / name, model / name)
    xyz = np.array([[-0.45, -0.35, 0.0], [0.4, -0.45, 0.05], [-0.35, 0.45, -0.05]], np.float32)
    scale = np.array([[0.12, 0.09, 0.07], [0.3, 0.03, 0.03], [0.1, 0.1, 0.1]], np.float32)
    th = math.radians(60.0)
    rot = np.array([[0.9, 0.3, -0.2, 0.1], [math.cos(th / 2), 0.0, 0.0, math.sin(th / 2)], [1.0, 0.0, 0.0, 0.0]],
                   np.float32)
    density = np.array([0.2, 0.8, 0.5], np.float32)
    blob = {"xyz": xyz, "density": np.log(np.expm1(density.astype(np.float64))).astype(np.float32)[:, None],
            "scale": np.log(scale), "rotation": rot, "scale_bound": None}
    with open(it / "point_cloud.pickle", "wb") as f:
        pickle.dump(blob, f)
    W = H = 200
    rep, frames, prims, cams = _run(["-m", str(model), "--gaussians", "--no_images", "--cam_scale", "0.1",
                                     "--width", str(W), "--height", str(H), "--camera", "0", "0", "4", "0", "0", "0",
                                     "0", "1", "0", "--output", str(tmp_path / "three.png")], capsys)
    assert rep["gaussians"] == 3
    _, keys = sv.render(prims, cams, return_keys=True)
    ids = _ids(keys[0].cpu().numpy().view(np.uint64))
    img = frames[0].cpu().numpy()
    k = so.Cam(cams[0].record(), H, W, False)
    dens = torch.nn.functional.softplus(torch.from_numpy(blob["density"][:, 0])).numpy()
    grey = (dens.astype(np.float32) * (np.float32(0.95) / dens.astype(np.float32).max())).astype(np.float32)
    L = build_scaling_rotation(torch.from_numpy(np.exp(blob["scale"]).astype(np.float64)),
                               torch.from_numpy(rot.astype(np.float64))).numpy()
    for i in range(3):
        sx, sy = so._project(k, so.to_cam(k, xyz[i].astype(np.float64)))
        x, y = int(math.floor(sx)), int(math.floor(sy))
        assert ids[y, x] == i, (i, ids[y, x])
        a, b = so.pixel_ab(k, x, y)
        O = np.asarray(k.P)
        D = np.asarray(k.f) + float(a) * np.asarray(k.r) + float(b) * np.asarray(k.u)
        Si = np.linalg.inv(L[i] @ L[i].T)
        d = O - xyz[i].astype(np.float64)
        A, B, C = D @ Si @ D, D @ Si @ d, d @ Si @ d - 1.0
        t = (-B - math.sqrt(B * B - A * C)) / A
        n = Si @ (d + t * D)
        lam = min(abs(n @ D) / (np.linalg.norm(n) * np.linalg.norm(D)), 1.0)
        assert np.abs(img[y, x] - grey[i] * (0.25 + 0.75 * lam)).max() <= TOL, (i, img[y, x])
    ys, xs = np.nonzero(ids == 1)
    X, Y = xs - xs.mean(), -(ys - ys.mean())
    angle = 0.5 * math.atan2(2 * (X * Y).mean(), (X * X).mean() - (Y * Y).mean())
    w, v = np.linalg.eigh((L[1] @ L[1].T)[:2, :2])
    cov_angle = math.atan2(v[1, -1], v[0, -1])
    for ang in (angle, cov_angle):
        d = (ang - th) % math.pi
        assert min(d, math.pi - d) < math.radians(2.0), math.degrees(ang)
