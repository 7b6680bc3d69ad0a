"""Scene view without a GPU: tests/scene_view_oracle.py against closed forms (fill rule, shared edges, silhouettes,
depth ties, lines, near-plane clipping, textures), the glyph geometry, the CLI's refusals and the ABI's argument
checks."""
import math

import numpy as np
import pytest
import torch
from scipy import ndimage

import mesh_oracle as mo
import scene_view_oracle as so
from r2_gaussian_b200 import scene_view as sv
from r2_gaussian_b200 import visualize_scene
from r2_gaussian_b200.volume_render import look_at


def _screen_cam(W, H):
    """A parallel camera looking down -z with one scene unit per pixel: world (X, Y) lands at screen (X, H - Y)."""
    return look_at((W / 2, H / 2, 10.0), (W / 2, H / 2, 0.0), (0, 1, 0), W, H, parallel_scale=H / 2)


def _tris(tris, kind=so.FLAT):
    tris = np.asarray(tris, np.float64).reshape(-1, 3, 3)
    meta = np.zeros((len(tris), 2), np.int32)
    meta[:, 0] = kind
    attr = np.zeros((len(tris), 12), np.float32)
    attr[:, 0:3] = np.random.default_rng(0).random((len(tris), 3))
    return tris, meta, attr


def _raster(pos, meta, attr, cam, tex=None, lut=((0, 0, 0), (1, 1, 1)), near=1e-3, bg=(1, 1, 1)):
    return so.raster(pos, meta, attr, tex, np.asarray(lut, np.float32), cam.record()[None], cam.height, cam.width,
                     cam.parallel, near, bg)


def _xy_screen(pts, H):
    """Screen points (sx, sy) -> world points of _screen_cam at z = 0."""
    pts = np.asarray(pts, np.float64)
    return np.stack([pts[:, 0], H - pts[:, 1], np.zeros(len(pts))], 1)


def _count(lo, hi):
    return sum(1 for i in range(-2, 200) if lo <= i + 0.5 < hi)


@pytest.mark.parametrize("box", [(2.0, 9.0, 3.0, 7.0), (2.5, 9.5, 3.5, 7.5), (1.5, 1.5, 2.0, 6.0),
                                 (0.25, 12.75, 0.5, 10.5), (3.3, 8.7, 2.1, 6.9)])
def test_square_covers_the_fill_rule_count(box):
    W, H = 16, 12
    x0, x1, y0, y1 = box
    q = _xy_screen([(x0, y0), (x1, y0), (x1, y1), (x0, y1)], H)
    pos, meta, attr = _tris([q[[0, 1, 2]], q[[2, 3, 0]]])
    keys, _ = _raster(pos, meta, attr, _screen_cam(W, H))
    covered = keys[0] != so.EMPTY
    assert covered.sum() == _count(x0, x1) * _count(y0, y1)
    cols = [i for i in range(W) if x0 <= i + 0.5 < x1]
    rows = [j for j in range(H) if y0 <= j + 0.5 < y1]
    expect = np.zeros_like(covered)
    expect[np.ix_(rows, cols)] = True
    assert np.array_equal(covered, expect)


def test_triangles_sharing_an_edge_partition_the_quad():
    rng = np.random.default_rng(1)
    W = H = 24
    cam = _screen_cam(W, H)
    for _ in range(60):
        c = rng.uniform(4, 20, 2)
        ang = np.sort(rng.uniform(0, 2 * np.pi, 4))
        r = rng.uniform(2, 10, 4)
        pts = c + np.stack([r * np.cos(ang), r * np.sin(ang)], 1)
        snap = rng.random(4) < 0.3
        pts[snap] = np.round(pts[snap] * 2) / 2                      # some corners on pixel centres and edges
        e = np.roll(pts, -1, 0) - pts
        turn = e[:, 0] * np.roll(e, -1, 0)[:, 1] - e[:, 1] * np.roll(e, -1, 0)[:, 0]
        if not ((turn > 0).all() or (turn < 0).all()):
            continue                                             # both diagonals split only a convex quad
        q = _xy_screen(pts, H)
        sets = []
        for split in ([(0, 1, 2), (2, 3, 0)], [(0, 1, 3), (1, 2, 3)]):
            pos, meta, attr = _tris([q[list(t)] for t in split])
            keys, _ = _raster(pos, meta, attr, cam)
            sets.append(keys[0])
        for split in ([(0, 1, 2), (2, 3, 0)], [(0, 1, 3), (1, 2, 3)]):
            masks = []
            for t in split:
                pos, meta, attr = _tris([q[list(t)]])
                masks.append(_raster(pos, meta, attr, cam)[0][0] != so.EMPTY)
            assert not (masks[0] & masks[1]).any()
            union = masks[0] | masks[1]
            assert np.array_equal(union, sets[0] != so.EMPTY)
        assert np.array_equal(sets[0] != so.EMPTY, sets[1] != so.EMPTY)


def test_closed_mesh_silhouette_has_no_holes():
    n = 20
    g = np.stack(np.meshgrid(*[np.arange(n)] * 3, indexing="ij"), -1).astype(np.float64)
    vol = 1.0 - np.sqrt(((g - [9.3, 10.1, 9.7]) ** 2 / [36.0, 25.0, 49.0]).sum(-1))
    vol[0], vol[-1], vol[:, 0], vol[:, -1], vol[:, :, 0], vol[:, :, -1] = [-1.0] * 6
    verts, faces = mo.marching_cubes(vol.astype(np.float32), 0.0)
    pos = verts.astype(np.float64)[faces]
    _, meta, attr = _tris(pos)
    for cam in (look_at((40, -30, 25), (9.5, 9.5, 9.5), (0, 0, 1), 64, 48, 30.0),
                look_at((9.5, 9.5, 60), (9.5, 9.5, 9.5), (0, 1, 0), 40, 40, parallel_scale=12.0)):
        keys, _ = _raster(pos, meta, attr, cam)
        covered = keys[0] != so.EMPTY
        assert covered.sum() > 100
        assert np.array_equal(ndimage.binary_fill_holes(covered), covered)


def test_depth_ties_go_to_the_lower_id():
    W, H = 12, 10
    q = _xy_screen([(1, 1), (11, 1), (6, 9)], H)
    pos, meta, attr = _tris([q, q, q[[1, 2, 0]]])
    keys, rgb = _raster(pos, meta, attr, _screen_cam(W, H))
    hit = keys[0] != so.EMPTY
    assert hit.sum() > 20
    assert ((keys[0][hit] & np.uint64(0xFFFFFFFF)) == 0).all()
    assert np.array_equal(rgb[0][hit], np.broadcast_to(attr[0, :3], (hit.sum(), 3)))
    # a nearer triangle wins whatever its id
    nearer = q.copy()
    nearer[:, 2] = 1.0
    pos2, meta2, attr2 = _tris([q, nearer])
    keys2, _ = _raster(pos2, meta2, attr2, _screen_cam(W, H))
    assert ((keys2[0][hit] & np.uint64(0xFFFFFFFF)) == 1).all()


@pytest.mark.parametrize("width", [1.0, 2.0, 3.0])
def test_horizontal_line_covers_the_stated_pixels(width):
    W, H = 20, 12
    ax, bx, y = 3.25, 14.5, 5.5
    a, b = _xy_screen([(ax, y), (bx, y)], H)
    pos = np.zeros((1, 3, 3))
    pos[0, 0], pos[0, 1] = a, b
    meta = np.array([[so.LINE, 0]], np.int32)
    attr = np.zeros((1, 12), np.float32)
    attr[0, :3], attr[0, 3] = (0.2, 0.4, 0.6), width
    keys, rgb = _raster(pos, meta, attr, _screen_cam(W, H))
    r = width / 2
    expect = np.zeros((H, W), bool)
    for j in range(H):
        for i in range(W):
            cx, cy = i + 0.5, j + 0.5
            dx = max(ax - cx, 0.0, cx - bx)
            expect[j, i] = dx * dx + (cy - y) ** 2 <= r * r
    assert np.array_equal(keys[0] != so.EMPTY, expect)
    assert np.allclose(rgb[0][expect], np.float32([0.2, 0.4, 0.6]))


def _cube(c, s):
    corners = np.array([[(i >> 0) & 1, (i >> 1) & 1, (i >> 2) & 1] for i in range(8)], np.float64) * s + c
    quads = [(0, 1, 3, 2), (4, 5, 7, 6), (0, 1, 5, 4), (2, 3, 7, 6), (0, 2, 6, 4), (1, 3, 7, 5)]
    return np.array([corners[[q[0], q[1], q[2]]] for q in quads] + [corners[[q[2], q[3], q[0]]] for q in quads])


def test_near_clipping_camera_inside_the_box():
    pos, meta, attr = _tris(_cube(np.array([-1.0, -1.0, -1.0]), 2.0))
    for cam in (look_at((0.3, -0.2, 0.1), (1, 0.5, 0.3), (0, 0, 1), 41, 33, 100.0),
                look_at((0.0, 0.0, 0.0), (0, 0, 1), (0, 1, 0), 40, 30, 150.0)):
        keys, _ = _raster(pos, meta, attr, cam)
        assert (keys[0] != so.EMPTY).all()
        depth = (keys[0] >> np.uint64(32)).astype(np.uint32).view(np.float32)
        # the exit of the ray P + z (f + a r + b u) from [-1, 1]^3: z is the camera depth
        k = so.Cam(cam.record(), cam.height, cam.width, False)
        ys, xs = np.mgrid[0:cam.height, 0:cam.width]
        a, b = so.pixel_ab(k, xs, ys)
        d = np.asarray(k.f) + a[..., None] * np.asarray(k.r) + b[..., None] * np.asarray(k.u)
        exit_z = ((np.sign(d) - np.asarray(k.P)) / d).min(-1)
        assert np.allclose(depth, exit_z, rtol=1e-6)
    # a triangle half behind the camera is cut at the near plane, not dropped or mirrored
    cam = look_at((0, 0, 0), (0, 0, 1), (0, 1, 0), 30, 30, 90.0)
    tri = np.array([[[-0.2, -0.5, 1.0], [0.2, -0.5, 1.0], [0.0, 0.5, -0.5]]])
    pos, meta, attr = _tris(tri)
    keys, _ = _raster(pos, meta, attr, cam)
    hit = keys[0] != so.EMPTY
    rows = np.nonzero(hit.any(1))[0]
    # the front edge sits at y / z = -0.5, through row 22's centres (a bottom edge: not owned); the cut at the near
    # plane projects far above the top row
    assert rows.min() == 0 and rows.max() == 21 and hit.sum() < hit.size // 2
    # wholly behind: nothing
    pos, meta, attr = _tris(tri * np.array([1, 1, -1]) - np.array([0, 0, 2]))
    assert (_raster(pos, meta, attr, cam)[0] == so.EMPTY).all()


def test_textured_quad_one_texel_per_pixel_is_its_image():
    W, H = 13, 9
    img = np.random.default_rng(2).random((H, W)).astype(np.float32)
    q = _xy_screen([(0, 0), (W, 0), (W, H), (0, H)], H)
    uv = np.array([[0, 0], [1, 0], [1, 1], [0, 1]], np.float64)
    tris = [(0, 1, 2), (2, 3, 0)]
    pos = np.stack([q[list(t)] for t in tris])
    meta = np.array([[so.TEXTURED, 0]] * 2, np.int32)
    attr = np.zeros((2, 12), np.float32)
    attr[:, 3:9] = np.stack([uv[list(t)].reshape(-1) for t in tris])
    keys, rgb = _raster(pos, meta, attr, _screen_cam(W, H), tex=img[None])
    assert (keys[0] != so.EMPTY).all()
    for c in range(3):
        assert np.array_equal(rgb[0, ..., c], img)


def _dataset_camera(scanner, angle, off=False):
    from r2_gaussian_b200.scene import camera_from_view, make_view
    view = make_view(scanner, angle, use_offDetector=off)
    cam = camera_from_view(view, device="cpu")
    cam.image_width, cam.image_height = view.image_width, view.image_height
    return cam


def _scanner(mode="cone", off=(0.0, 0.0)):
    from r2_gaussian_b200.scene import cone_beam_scanner, parallel_beam_scanner
    s = (cone_beam_scanner if mode == "cone" else parallel_beam_scanner)(64, 32)
    s["offDetector"] = list(off)
    return s


def test_glyph_geometry():
    sc = _scanner("cone", off=(0.25, 0.0))
    angle = 0.7
    for off in (False, True):
        cam = _dataset_camera(sc, angle, off)
        c = sv.camera_centre(cam)
        src = np.array([sc["DSO"] * math.cos(angle), sc["DSO"] * math.sin(angle), 0.0])
        assert np.allclose(c, src, atol=1e-5)
        g = sv.camera_glyph(cam, 1.0, (1, 0, 0), plane_depth=sc["DSD"], device="cpu")
        apex = g.pos[4:8, 0].numpy()     # the four apex edges follow the ring
        assert np.allclose(apex, c, atol=0)
        corners = sv.image_plane(cam, sc["DSD"])
        centre = corners.mean(0)
        axis = -src / np.linalg.norm(src)
        shift = centre - (src + sc["DSD"] * axis)
        assert abs(shift @ axis) < 1e-5
        # the image's columns run along the camera's x; the offset moves the plane by offDetector[0] along it
        x_dir = (corners[1] - corners[0]) / np.linalg.norm(corners[1] - corners[0])
        assert np.isclose(shift @ x_dir, 0.25 if off else 0.0, atol=1e-5)
        side = np.linalg.norm(corners[1] - corners[0]), np.linalg.norm(corners[3] - corners[0])
        assert np.allclose(side, (sc["sDetector"][1], sc["sDetector"][0]), atol=1e-5)
    par = _dataset_camera(_scanner("parallel"), 0.3)
    g = sv.camera_glyph(par, 1.5, (0, 1, 0), image=torch.ones(4, 4), device="cpu")
    pos = g.pos.numpy()
    meta = g.meta.numpy()
    seg = pos[meta[:, 0] == sv.LINE][:12]
    d = seg[8:12, 1] - seg[8:12, 0]                    # the four edges joining the two rectangles
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    assert np.allclose(d, d[0], atol=1e-9)
    assert np.allclose(np.linalg.norm(seg[8:12, 1] - seg[8:12, 0], axis=1), 1.5)
    assert (meta[:, 0] == sv.TEXTURED).sum() == 2 and g.textures.shape == (1, 4, 4)


def test_vertex_normals_point_out_of_a_sphere():
    n = 24
    g = np.stack(np.meshgrid(*[np.arange(n)] * 3, indexing="ij"), -1).astype(np.float64)
    centre = np.array([11.5, 11.2, 11.8])
    vol = (8.0 - np.sqrt(((g - centre) ** 2).sum(-1))).astype(np.float32)
    verts, faces = mo.marching_cubes(vol, 0.0)
    nrm = sv.vertex_normals(torch.from_numpy(verts), torch.from_numpy(vol)).numpy()
    radial = verts - centre
    radial /= np.linalg.norm(radial, axis=1, keepdims=True)
    assert np.allclose(np.linalg.norm(nrm, axis=1), 1, atol=1e-5)
    assert (np.sum(nrm * radial, 1) > 0.99).all()


def test_scan_orbit_turns_about_z():
    cam = look_at((3, 0, 1), (0, 0, 0.5), (0, 0, 1), 20, 10)
    o = sv.scan_orbit(cam, 4)
    assert np.allclose(o[1].position, (0, 3, 1)) and np.allclose(o[2].position, (-3, 0, 1))
    assert all(np.allclose(c.focal_point, cam.focal_point) for c in o)


def test_camera_colour_matches_the_reference_ramp():
    lut = np.array([[0, 0, 0], [1, 1, 1]], np.float64)
    assert np.allclose(visualize_scene.camera_colour(lut, 3, 4), 0.75)
    assert np.allclose(visualize_scene.camera_colour(visualize_scene.CAMERA_LUT, 0, 5), (0, 0, 1))


def test_cli_parses_and_refuses(tmp_path):
    scene = tmp_path / "scene"
    scene.mkdir()
    out = str(tmp_path / "o.png")
    a = visualize_scene.parse_args(["-s", str(scene), "--output", out])
    assert (a.mc_thresh, a.cam_scale, a.width, a.height, a.views, a.orbit) == (0.5, 1.0, 1000, 800, 1, None)
    a = visualize_scene.parse_args(["-s", str(scene), "--output", out, "--camera", "3", "0", "0", "0", "0", "0", "0",
                                    "0", "1", "--orbit", "3", "--views", "5", "--true_detector", "--no_images"])
    assert a.orbit == 3 and a.views == 5 and a.true_detector and a.no_images
    lut = tmp_path / "lut.npy"
    np.save(lut, np.random.default_rng(0).random((8, 3)))
    assert visualize_scene.parse_args(["-s", str(scene), "--output", out, "--cmap", str(lut)]).lut.shape == (8, 3)
    bad = [[], ["--output", out], ["-s", str(tmp_path / "missing"), "--output", out],
           ["-s", str(scene), "--output", str(tmp_path / "no" / "o.png")],
           ["-s", str(scene), "--output", out, "--mc_thresh", "nan"],
           ["-s", str(scene), "--output", out, "--cam_scale", "0"],
           ["-s", str(scene), "--output", out, "--width", "0"],
           ["-s", str(scene), "--output", out, "--height", "16385"],
           ["-s", str(scene), "--output", out, "--views", "0"],
           ["-s", str(scene), "--output", out, "--orbit", "0"],
           ["-s", str(scene), "--output", out, "--supersample", "0"],
           ["-s", str(scene), "--output", out, "--cmap", "viridis"],
           ["-s", str(scene), "--output", out, "--camera", "0", "0", "0", "0", "0", "0", "0", "0", "1"],
           ["-s", str(scene), "--output", out, "--background", "2", "0", "0"],
           ["--vol", str(lut), "--output", out, "--true_detector"],
           ["-s", str(scene), "--output", out, "--resolution", "64"]]
    for argv in bad:
        with pytest.raises(SystemExit):
            visualize_scene.parse_args(argv)


def test_render_refuses_bad_input_without_a_device():
    prims = sv.lines([[0, 0, 0]], [[1, 0, 0]], (1, 0, 0), device="cpu")
    cam = look_at((0, 0, 5), (0, 0, 0), (0, 1, 0), 8, 8)
    for kw, needle in (({"supersample": 0}, "supersample"), ({"background": (0, 0)}, "background"),
                       ({"near": 0.0}, "near")):
        with pytest.raises(ValueError, match=needle):
            sv.render(prims, cam, **kw)
    with pytest.raises(ValueError, match="same image size"):
        sv.render(prims, [cam, look_at((0, 0, 5), (0, 0, 0), (0, 1, 0), 9, 8)])
    with pytest.raises(ValueError, match="width"):
        sv.lines([[0, 0, 0]], [[1, 0, 0]], (1, 0, 0), width=0.0, device="cpu")
    with pytest.raises(ValueError, match="colour"):
        sv.lines([[0, 0, 0]], [[1, 0, 0]], (2, 0, 0), device="cpu")


def test_abi_refuses_bad_arguments_before_any_cuda_work():
    import ctypes

    from r2_gaussian_b200._lib import load
    lib = load()
    assert lib.r2x_scene_raster_scratch_bytes(10, 3) == 64 + 10 * 3 * 40
    assert lib.r2x_scene_raster_scratch_bytes(2**31 - 1, 2) == 0
    bg = np.ones(3, np.float32)
    p = 16   # any non-NULL address: the checks return before touching memory

    def call(**kw):
        a = dict(n=1, n_tex=0, th=1, tw=1, tex=None, K=2, F=1, H=8, W=8, par=0, near=1e-3, bg=bg.ctypes.data,
                 nbytes=1 << 20)
        a.update(kw)
        rc = lib.r2x_scene_raster(None, a["n"], p, p, p, a["n_tex"], a["th"], a["tw"], a["tex"], p, a["K"], a["F"],
                                  a["H"], a["W"], p, a["par"], a["near"], a["bg"], p, p, p, a["nbytes"])
        return rc, lib.r2x_last_error().decode()

    nan_bg = np.array([0, np.nan, 0], np.float32)
    for kw, needle in (({"n": 0}, "n_prims"), ({"n": 2**30, "F": 2}, "n_prims"), ({"F": 0}, "n_frames"),
                       ({"F": 65536}, "n_frames"), ({"H": 16385}, "image"), ({"W": 0}, "image"),
                       ({"n_tex": 1}, "tex is NULL"), ({"n_tex": 1, "tex": p, "th": 16385}, "texture"),
                       ({"n_tex": 2**16, "tex": p, "th": 2**8, "tw": 2**7}, "texture"), ({"K": 0}, "K"),
                       ({"K": 4097}, "K"), ({"par": 2}, "parallel"), ({"near": 0.0}, "near"),
                       ({"near": float("inf")}, "near"), ({"bg": nan_bg.ctypes.data}, "background"),
                       ({"nbytes": 64}, "scratch")):
        rc, msg = call(**kw)
        assert rc == 1 and msg.startswith("r2x_scene_raster: bad") and needle in msg, (kw, msg)
    assert ctypes.sizeof(ctypes.c_double) == 8
