"""The scene-view rasterizer on the GPU against tests/scene_view_oracle.py: winning ids and depth keys bit for bit and
colours within 1e-6 on random triangle and line soups (odd sizes, around the 16-pixel tile and the large-primitive
split, perspective and parallel, clipped by the near plane), chosen windows of a ~3 M-triangle mesh, orbits equal to
single frames, reproducibility, the size limits, and `visualize_scene` end to end."""
import json
import os

import numpy as np
import pytest
import torch

import scene_view_oracle as so
import volume_render_oracle as vo
from r2_gaussian_b200 import scene_view as sv
from r2_gaussian_b200.volume_render import look_at, to_uint8

pytestmark = pytest.mark.gpu
TOL = 1e-6


def _soup(rng, n_tri, n_line, spread, size, n_tex=2, tex_shape=(7, 5)):
    """Random triangles (flat, mesh, textured) and lines around the origin; `size` scales each primitive."""
    c = rng.uniform(-spread, spread, (n_tri + n_line, 1, 3))
    pos = c + rng.normal(0, 1, (n_tri + n_line, 3, 3)) * rng.uniform(0.05, 1, (n_tri + n_line, 1, 1)) * size
    meta = np.zeros((len(pos), 2), np.int32)
    meta[:n_tri, 0] = rng.integers(0, 3, n_tri)
    meta[n_tri:, 0] = so.LINE
    meta[:, 1] = rng.integers(0, n_tex, len(pos))
    attr = rng.random((len(pos), 12)).astype(np.float32)
    nrm = rng.normal(0, 1, (len(pos), 9))
    attr[:, 3:12] = np.where((meta[:, 0] == so.MESH)[:, None], nrm, attr[:, 3:12])
    attr[n_tri:, 3] = rng.choice([0.5, 1.0, 1.5, 3.0, 7.0], n_line)
    tex = rng.random((n_tex,) + tex_shape).astype(np.float32)
    return pos, meta, attr, tex


def _gpu(pos, meta, attr, tex):
    t = lambda x, dt: torch.as_tensor(np.ascontiguousarray(x), dtype=dt, device="cuda")
    return sv.Primitives(t(pos, torch.float64), t(meta, torch.int32), t(attr, torch.float32), t(tex, torch.float32))


LUT = np.array([[0.1, 0.2, 0.3], [0.9, 0.5, 0.1], [0.4, 1.0, 0.6]], np.float32)


def _compare(pos, meta, attr, tex, cams, near=sv.NEAR, bg=(1.0, 1.0, 1.0), window=None):
    rgb, keys = sv.render(_gpu(pos, meta, attr, tex), cams, background=bg, lut=LUT, near=near, return_keys=True)
    c0 = cams[0]
    recs = np.stack([c.record() for c in cams])
    okeys, orgb = so.raster(pos, meta, attr, tex, LUT, recs, c0.height, c0.width, c0.parallel, near, bg, window)
    k = keys.cpu().numpy().view(np.uint64)
    g = rgb.cpu().numpy()
    if window is not None:
        y0, y1, x0, x1 = window
        k, okeys = k[:, y0:y1, x0:x1], okeys[:, y0:y1, x0:x1]
        g, orgb = g[:, y0:y1, x0:x1], orgb[:, y0:y1, x0:x1]
    assert np.array_equal(k, okeys), int((k != okeys).sum())
    assert np.abs(g - orgb).max() <= TOL
    return k


@pytest.mark.parametrize("HW", [(17, 23), (15, 16), (16, 17), (33, 31), (1, 40), (48, 1)])
@pytest.mark.parametrize("parallel", [False, True])
def test_random_soups_equal_the_oracle(HW, parallel):
    H, W = HW
    rng = np.random.default_rng(H * 100 + W + parallel)
    pos, meta, attr, tex = _soup(rng, 120, 60, 1.0, 0.6)
    kw = {"parallel_scale": 1.6} if parallel else {}
    cams = [look_at((3.5, -2.0, 1.5), (0, 0, 0), (0, 0, 1), W, H, 45.0, **kw),
            look_at((0.2, 0.1, 0.3), (1, 1, 0), (0, 0, 1), W, H, 120.0, **kw)]    # inside the soup: near clipping
    k = _compare(pos, meta, attr, tex, cams)
    assert (k != so.EMPTY).any()


@pytest.mark.parametrize("extent", [14.0, 15.5, 16.0, 16.5, 17.0, 31.5, 32.5, 200.0])
def test_sizes_around_the_tile_and_the_split(extent):
    """Squares and lines whose pixel box is just below, at and above 16 pixels, and far above it."""
    W, H = 37, 29
    cam = look_at((W / 2, H / 2, 10.0), (W / 2, H / 2, 0.0), (0, 1, 0), W, H, parallel_scale=H / 2)
    rng = np.random.default_rng(int(extent * 10))
    pos, meta, attr = [], [], []
    for _ in range(12):
        x0, y0 = rng.uniform(-3, 20, 2)
        q = np.array([[x0, y0, 0], [x0 + extent, y0, 0], [x0 + extent, y0 + extent * 0.7, 0], [x0, y0 + extent * 0.7, 0]])
        q[:, 2] = rng.uniform(-1, 1)
        pos += [q[[0, 1, 2]], q[[2, 3, 0]], np.stack([q[0], q[2], q[0]])]
        meta += [[so.FLAT, 0], [so.TEXTURED, 0], [so.LINE, 0]]
        a = rng.random(12).astype(np.float32)
        a[3:9] = [0, 0, 1, 0, 1, 1]
        b = a.copy()
        b[3:9] = [1, 1, 0, 1, 0, 0]
        ln = a.copy()
        ln[3] = 2.0
        attr += [a, b, ln]
    tex = rng.random((1, 11, 13)).astype(np.float32)
    persp = look_at((W / 2 + 3, H / 2 - 4, 30.0), (W / 2, H / 2, 0.0), (0, 1, 0), W, H, 60.0)
    for c in (cam, persp):
        _compare(np.array(pos), np.array(meta, np.int32), np.array(attr), tex, [c])


def test_orbit_equals_single_frames_and_is_reproducible():
    rng = np.random.default_rng(5)
    pos, meta, attr, tex = _soup(rng, 300, 100, 1.0, 0.4)
    prims = _gpu(pos, meta, attr, tex)
    cams = sv.scan_orbit(look_at((3, 1, 2), (0, 0, 0), (0, 0, 1), 45, 33, 40.0), 7)
    rgb, keys = sv.render(prims, cams, lut=LUT, return_keys=True)
    rgb2, keys2 = sv.render(prims, cams, lut=LUT, return_keys=True)
    assert torch.equal(keys, keys2) and torch.equal(rgb, rgb2)
    for i, c in enumerate(cams):
        r1, k1 = sv.render(prims, c, lut=LUT, return_keys=True)
        assert torch.equal(k1[0], keys[i]) and torch.equal(r1[0], rgb[i])
    _compare(pos, meta, attr, tex, cams[:3])
    # supersampling: the mean of the k x k blocks of the k-times larger render
    big = sv.render(prims, look_at(cams[0].position, cams[0].focal_point, cams[0].view_up, 90, 66, 40.0), lut=LUT)
    ss = sv.render(prims, cams[0], lut=LUT, supersample=2)
    acc = big[:, 0::2, 0::2] + big[:, 0::2, 1::2] + big[:, 1::2, 0::2] + big[:, 1::2, 1::2]
    assert torch.equal(ss, acc / 4.0)


def test_large_mesh_windows_equal_the_oracle():
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "scripts", "gpu"))
    from mesh_bench import cloud_volume
    from r2_gaussian_b200.mesh import marching_cubes
    vol = cloud_volume(256)
    verts, faces = marching_cubes(vol, 0.3 * float(vol.max()))
    assert faces.shape[0] > 3_000_000
    cfg = {"offOrigin": [0.0, 0.0, 0.0], "sVoxel": [2.0, 2.0, 2.0], "nVoxel": [256] * 3}
    prims = sv.mesh_triangles(verts, faces, vol, cfg)
    W, H = 1000, 800
    cam = sv.default_view(prims, W, H)
    rgb, keys = sv.render(prims, cam, return_keys=True)
    pos, meta, attr = (t.cpu().numpy() for t in (prims.pos, prims.meta, prims.attr))
    tex = np.zeros((1, 1, 1), np.float32)
    rec = cam.record()[None]
    k = keys.cpu().numpy().view(np.uint64)
    for win in ((390, 410, 490, 510), (200, 216, 300, 331), (600, 611, 640, 660)):
        okeys, orgb = so.raster(pos, meta, attr, tex, np.array([[0, 0, 0], [1, 1, 1]], np.float32), rec, H, W, False,
                                sv.NEAR, (1.0, 1.0, 1.0), win)
        y0, y1, x0, x1 = win
        assert np.array_equal(k[:, y0:y1, x0:x1], okeys[:, y0:y1, x0:x1]), win
        assert np.abs(rgb.cpu().numpy()[:, y0:y1, x0:x1] - orgb[:, y0:y1, x0:x1]).max() <= TOL
    assert (k != so.EMPTY).mean() > 0.2


def test_limits_accepted_and_refused():
    pos, meta, attr, tex = _soup(np.random.default_rng(9), 4, 2, 0.5, 0.3, n_tex=1, tex_shape=(16384, 3))
    prims = _gpu(pos, meta, attr, tex)
    for W, H in ((16384, 3), (2, 16384)):
        rgb = sv.render(prims, look_at((2, 1, 1), (0, 0, 0), (0, 0, 1), W, H, 30.0))
        assert rgb.shape == (1, H, W, 3)
    with pytest.raises(ValueError, match="16384"):
        sv.render(prims, look_at((2, 1, 1), (0, 0, 0), (0, 0, 1), 16385, 3, 30.0))
    from r2_gaussian_b200._lib import R2XError
    big = sv.Primitives(prims.pos, prims.meta, prims.attr, torch.zeros((1, 16385, 2), device="cuda"))
    with pytest.raises(R2XError, match="texture"):
        sv.render(big, look_at((2, 1, 1), (0, 0, 0), (0, 0, 1), 8, 8, 30.0))
    cams = [look_at((2, 1, 1), (0, 0, 0), (0, 0, 1), 2, 2, 30.0)] * 65535
    assert sv.render(prims, cams).shape == (65535, 2, 2, 3)
    with pytest.raises(R2XError, match="n_frames"):
        sv.render(prims, cams + cams[:1])
    bad = sv.Primitives(prims.pos, prims.meta.clone(), prims.attr, prims.textures)
    bad.meta[0] = torch.tensor([so.TEXTURED, 1], dtype=torch.int32)
    with pytest.raises(ValueError, match="texture"):
        sv.render(bad, cams[0])


# ---- visualize_scene end to end --------------------------------------------------------------------------------------

def _project(cam, X):
    k = so.Cam(cam.record(), cam.height, cam.width, cam.parallel)
    c = so.to_cam(k, X)
    sx, sy = so._project(k, c)
    return int(np.floor(sx)), int(np.floor(sy))


def _run(argv, capsys):
    from r2_gaussian_b200 import visualize_scene
    rep, frames, prims, cams = visualize_scene.run(argv)
    line = capsys.readouterr().out.strip().splitlines()[-1]
    assert json.loads(line) == json.loads(json.dumps(rep))
    imgs = to_uint8(frames).cpu().numpy()
    pngs = [p for p in rep["outputs"] if p.endswith(".png")]
    assert len(pngs) == rep["frames"] == frames.shape[0]
    for p, img in zip(pngs, imgs):
        assert np.array_equal(vo.read_png(p), img), p
    assert torch.equal(frames, sv.render(prims, cams))
    return rep, frames, cams


def _apex_colours(frames, cam, centres, colours, r=2):
    img = frames[0].cpu().numpy()
    for c, col in zip(centres, colours):
        x, y = _project(cam, c)
        patch = img[max(y - r, 0):y + r + 1, max(x - r, 0):x + r + 1].reshape(-1, 3)
        assert (np.abs(patch - np.float32(col)).max(1) == 0).any(), (x, y, col)


@pytest.fixture(scope="module")
def scenes(tmp_path_factory):
    from r2_gaussian_b200 import generate_data, initialize_pcd, scene
    from test_volume_render_gpu import _smooth
    tmp = tmp_path_factory.mktemp("scene_view")
    n = 32
    np.save(tmp / "vol.npy", _smooth((n, n, n)).clip(0, 1))
    out = {}
    for name, off in (("plain", [0.0, 0.0]), ("offset", [0.6, 0.0])):
        sc = scene.cone_beam_scanner(48, n)
        phys = {k: (np.asarray(v, float) * 2.0).tolist() if k in ("DSD", "DSO", "sDetector", "sVoxel", "offOrigin")
                else v for k, v in sc.items()}
        phys.update({"offDetector": off, "filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0,
                     "noise": False})
        (tmp / f"{name}.yml").write_text("".join(f"{k}: {json.dumps(v)}\n" for k, v in phys.items()))
        out[name] = generate_data.main(["--vol", str(tmp / "vol.npy"), "--scanner", str(tmp / f"{name}.yml"),
                                        "--n_train", "8", "--n_test", "2", "--output", str(tmp / name)]
                                       + (["--use_offDetector"] if name == "offset" else []))
    out["init"] = initialize_pcd.main(["--data", out["plain"], "--n_points", "3000", "--output", str(tmp / "init.npy")])
    return out


def test_visualize_scene_end_to_end(scenes, tmp_path, capsys):
    from r2_gaussian_b200.dataset import Scene
    from r2_gaussian_b200.visualize_scene import CAMERA_LUT, camera_colour
    src = scenes["plain"]
    rep, frames, cams = _run(["-s", src, "--width", "160", "--height", "120", "--output", str(tmp_path / "s.png"),
                              "--no_images"], capsys)
    assert rep["source"] == "scene" and rep["cameras"] == 8 and rep["triangles"] > 100 and frames.shape == (1, 120, 160, 3)
    train = Scene(src, eval=False, shuffle=False).getTrainCameras()
    _apex_colours(frames, cams[0], [sv.camera_centre(c) for c in train],
                  [camera_colour(CAMERA_LUT, i, 8) for i in range(8)])
    # every 2nd view, images, an orbit and --save_npy
    rep, frames, cams = _run(["-s", src, "--width", "64", "--height", "48", "--views", "2", "--orbit", "3",
                              "--save_npy", "--output", str(tmp_path / "o.png")], capsys)
    assert rep["cameras"] == 4 and rep["frames"] == 3
    assert np.array_equal(np.load(tmp_path / "o.npy"), frames.cpu().numpy())
    # offset detector, true detector: the image plane at DSD, shifted by offDetector
    rep, frames, cams = _run(["-s", scenes["offset"], "--use_offDetector", "--true_detector", "--width", "96",
                              "--height", "80", "--output", str(tmp_path / "t.png")], capsys)
    assert rep["cameras"] == 8


def test_visualize_scene_with_learned_poses(scenes, tmp_path, capsys):
    from r2_gaussian_b200 import trainer
    from r2_gaussian_b200.dataset import Scene
    from r2_gaussian_b200.pose import PoseCorrection
    from r2_gaussian_b200.trainer import POSE_ANCHOR
    from r2_gaussian_b200.visualize_scene import CAMERA_LUT, camera_colour
    model = tmp_path / "model"
    trainer.main(["-s", scenes["plain"], "-m", str(model), "--ply_path", scenes["init"], "--iterations", "100",
                  "--test_iterations", "100", "--save_iterations", "100", "--pose_refine"])
    capsys.readouterr()
    it = model / "point_cloud" / "iteration_100"
    assert (it / "train_poses.npz").exists()
    # make the learned correction visible: a rotation and a shift, stored as the trainer stores them
    scene = Scene(scenes["plain"], eval=False, shuffle=False)
    cams = scene.getTrainCameras()
    pose = PoseCorrection(len(cams), device="cuda")
    rng = np.random.default_rng(0)
    with torch.no_grad():
        pose.omega.copy_(torch.from_numpy(rng.normal(0, 0.02, (len(cams), 3)).astype(np.float32)))
        pose.nu.copy_(torch.from_numpy(rng.normal(0, 0.3, (len(cams), 3)).astype(np.float32)))
        pose.omega[POSE_ANCHOR] = 0
        pose.nu[POSE_ANCHOR] = 0
        wvt = torch.stack([pose.device_camera(c, c.uid, POSE_ANCHOR).world_view_transform for c in cams])
    stored = dict(np.load(it / "train_poses.npz"))
    stored.update(omega=pose.omega.detach().cpu().numpy(), nu=pose.nu.detach().cpu().numpy(),
                  world_view_transform=wvt.cpu().numpy())
    np.savez(it / "train_poses.npz", **stored)
    rep, frames, vcams = _run(["-m", str(model), "--no_images", "--width", "200", "--height", "160", "--output",
                               str(tmp_path / "m.png")], capsys)
    assert rep["source"] == "model@100" and rep["cameras"] == 8
    with torch.no_grad():
        corrected = [sv.camera_centre(pose.device_camera(c, c.uid, POSE_ANCHOR)) for c in cams]
    nominal = [sv.camera_centre(c) for c in cams]
    cols = [camera_colour(CAMERA_LUT, i, 8) for i in range(8)]
    _apex_colours(frames, vcams[0], corrected, cols)
    _apex_colours(frames, vcams[0], nominal, cols)
    moved = [i for i in range(8) if _project(vcams[0], corrected[i]) != _project(vcams[0], nominal[i])]
    assert len(moved) >= 6
