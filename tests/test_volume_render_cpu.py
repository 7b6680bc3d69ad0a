"""Volume rendering without a GPU: tests/volume_render_oracle.py against closed forms, camera construction, the PNG
writer, and the refusals of the C ABI, the Python API and `render_volume` before any CUDA work."""
import ctypes as C
import math

import numpy as np
import pytest

import volume_render_oracle as vo
from r2_gaussian_b200 import _lib, render_volume
from r2_gaussian_b200 import volume_render as vr

# plot_volume.py's camera position, focal point and view-up
CPOS = [(-458.0015547298666, -207.26124611865254, 324.4699978427509),
        (129.02644270914504, 111.50694084289574, 98.55158287937994),
        (0.0, 0.0, 79.59633400474613)]


def _mip_expected(vol, axis, lat, up, side):
    vm = vol.max(axis=axis, keepdims=True)
    ii = [None] * 3
    ii[axis], ii[up], ii[side] = np.zeros_like(lat[..., 0]), lat[..., 0], lat[..., 1]
    return vm[tuple(ii)]


# ---- the oracle against closed forms -------------------------------------------------------------------------------------

@pytest.mark.parametrize("axis,sign,step", [(0, 1, 0.5), (1, -1, 0.5), (2, 1, 0.25), (2, -1, 1.0), (0, -1, 0.3)])
def test_constant_volume_along_an_axis(axis, sign, step):
    """Every ray crosses n - 1 voxels: floor((n - 1) / step) + 1 samples of alpha = 1 - (1 - t)^(step / unit)."""
    shape = (7, 9, 6)
    vol = np.full(shape, 0.3, np.float32)
    cam, lat, _ = vo.axis_view(shape, axis, sign)
    unit = vr.default_opacity_unit(shape)
    out = vo.render(vol, [cam], step=step, background=(0.2, 0.4, 0.6))[0]
    alpha = 1 - (1 - float(np.float32(0.3))) ** (vo.rec_step(step) / vo.rec_step(unit))
    K = math.floor((shape[axis] - 1) / vo.rec_step(step))
    T = (1 - alpha) ** (K + 1)
    assert np.allclose(out[..., 3], 1 - T, rtol=0, atol=1e-12)
    assert np.allclose(out[..., :3], (1 - T) * float(np.float32(0.3)) + T * np.float32([0.2, 0.4, 0.6]), atol=1e-12)


def test_all_below_clim_gives_the_exact_background():
    rng = np.random.default_rng(1)
    vol = rng.uniform(-1, 0.2, (9, 8, 10)).astype(np.float32)
    bg = (0.25, 0.5, 0.75)
    cam = vr.default_camera(vol.shape, 24, 20)
    out = vo.render(vol, [cam], clim=(0.2, 1.0), background=bg)[0]
    assert (out[..., :3] == np.float32(bg).astype(np.float64)).all() and (out[..., 3] == 0).all()


@pytest.mark.parametrize("axis,sign", [(a, s) for a in range(3) for s in (1, -1)])
def test_mip_along_an_axis_is_the_max(axis, sign):
    rng = np.random.default_rng(axis * 2 + (sign > 0))
    vol = rng.random((5, 7, 4), dtype=np.float32)
    cam, lat, (up, side) = vo.axis_view(vol.shape, axis, sign)
    out = vo.render(vol, [cam], mode="mip", step=1.0)[0]
    want = _mip_expected(vol, axis, lat, up, side)
    for c in range(3):
        assert np.array_equal(out[..., c], want.astype(np.float64))
    assert (out[..., 3] == 1).all()


def test_stop_rule():
    """An opaque volume stops each ray after the sample that leaves T < 2^-16; A stays below 1."""
    vol = np.full((6, 6, 40), 0.999, np.float32)
    cam, _, _ = vo.axis_view(vol.shape, 2, 1)
    out = vo.render(vol, [cam], step=0.5)[0]
    assert (out[..., 3] > 1 - 2.0 ** -16).all() and (out[..., 3] < 1).all()


# ---- cameras -------------------------------------------------------------------------------------------------------------

def test_pixel_offsets_and_ray_directions():
    cam = vr.look_at((10.0, -3.0, 4.0), (1.0, 2.0, 0.5), (0.3, 0.2, 5.0), 7, 5, view_angle=40.0)
    f, r, u = cam.f, cam.r, cam.u
    assert np.allclose([f @ f, r @ r, u @ u], 1) and np.allclose([f @ r, f @ u, r @ u], 0, atol=1e-15)
    assert np.allclose(np.cross(r, u), -f)            # right-handed: r x u points back at the camera
    p = 2 * math.tan(math.radians(40) / 2) / 5
    assert math.isclose(cam.pitch, p)
    o, d, _, _, _ = vo.ray_setup(cam.record(), 5, 7, False, (4, 4, 4))
    rec = cam.record().astype(np.float64)
    for y, x in [(0, 0), (2, 3), (4, 6), (1, 5)]:
        a, b = (x + 0.5 - 7 / 2) * rec[12], (5 / 2 - y - 0.5) * rec[12]
        want = rec[3:6] + a * rec[6:9] + b * rec[9:12]
        assert np.allclose(d[y * 7 + x], want / np.linalg.norm(want), rtol=0, atol=1e-15)
        assert np.array_equal(o[y * 7 + x], rec[0:3])
    # the top row looks up (+u), the right column looks right (+r)
    assert d[0 * 7 + 3] @ rec[9:12] > 0 and d[2 * 7 + 6] @ rec[6:9] > 0
    par = vr.look_at((10.0, -3.0, 4.0), (1.0, 2.0, 0.5), (0.3, 0.2, 5.0), 7, 5, parallel_scale=3.0)
    assert math.isclose(par.pitch, 2 * 3.0 / 5)
    o, d, _, _, _ = vo.ray_setup(par.record(), 5, 7, True, (4, 4, 4))
    rec = par.record().astype(np.float64)
    assert np.allclose(o[0], rec[0:3] + (0.5 - 3.5) * rec[12] * rec[6:9] + (2.5 - 0.5) * rec[12] * rec[9:12])
    assert (d == rec[3:6]).all()


def test_default_camera():
    shape = (40, 30, 20)
    cam = vr.default_camera(shape, 80, 100)
    centre = (np.asarray(shape) - 1) / 2
    dist = np.linalg.norm(np.asarray(shape) - 1) / 2 / math.sin(math.radians(15))
    assert np.allclose(cam.focal_point, centre)
    assert np.allclose(np.asarray(cam.position) - centre, dist * np.ones(3) / math.sqrt(3))
    assert cam.view_up == (0.0, 0.0, 1.0) and cam.view_angle == 30.0 and not cam.parallel
    assert (cam.width, cam.height) == (80, 100)
    assert np.allclose(cam.f, -np.ones(3) / math.sqrt(3))
    # the bounding sphere spans the view: every corner projects inside the image
    corners = np.array([[i, j, k] for i in (0, shape[0] - 1) for j in (0, shape[1] - 1) for k in (0, shape[2] - 1)])
    rel = corners - np.asarray(cam.position)
    z = rel @ cam.f
    assert (np.abs(rel @ cam.u / z) <= cam.pitch * 50).all() and (np.abs(rel @ cam.r / z) <= cam.pitch * 50).all()
    assert vr.default_opacity_unit((16, 16, 16)) == pytest.approx(math.sqrt(3))


@pytest.mark.parametrize("n", [1, 2, 5, 8, 36])
def test_orbit(n):
    cam = vr.look_at(CPOS[0], CPOS[1], CPOS[2], 16, 20)
    frames = vr.orbit(cam, n)
    F = np.asarray(CPOS[1])
    k = np.asarray(CPOS[2]) / np.linalg.norm(CPOS[2])
    d0 = np.asarray(cam.position) - F
    assert len(frames) == n
    assert np.allclose(frames[0].position, cam.position) and np.allclose(frames[0].u, cam.u)
    for c in frames:
        v = np.asarray(c.position) - F
        assert math.isclose(np.linalg.norm(v), np.linalg.norm(d0), rel_tol=1e-12)
        assert math.isclose(v @ k, d0 @ k, rel_tol=1e-12)                 # height along the axis kept
        assert c.view_up == cam.view_up and c.focal_point == cam.focal_point
        assert (c.width, c.height, c.view_angle, c.parallel_scale) == (16, 20, 30.0, None)
    if n % 2 == 0:
        half = np.asarray(frames[n // 2].position) - F
        perp0 = d0 - (d0 @ k) * k
        assert np.allclose(half - (half @ k) * k, -perp0, atol=1e-9)
    if n >= 4:
        # successive frames turn right-handedly about the view-up
        v1 = np.asarray(frames[1].position) - F
        assert np.cross(d0, v1) @ k > 0


def test_reference_cpos_parses():
    flat = [str(x) for p in CPOS for x in p]
    a = render_volume.parse_args(["--output", "out.png", "--vol", __file__, "--camera", *flat])
    assert a.camera == [float(x) for x in flat]
    assert a.window_size == [800, 1000] and a.mode == "composite" and a.clim == [0.0, 1.0]
    cam = vr.look_at(a.camera[0:3], a.camera[3:6], a.camera[6:9], *a.window_size)
    f = (np.asarray(CPOS[1]) - np.asarray(CPOS[0])) / np.linalg.norm(np.subtract(CPOS[1], CPOS[0]))
    assert np.allclose(cam.f, f)
    # view-up (0, 0, 79.6) is neither unit nor orthogonal to f; u is its unit part orthogonal to f
    U = np.asarray(CPOS[2])
    want_u = U - (U @ f) * f
    assert np.allclose(cam.u, want_u / np.linalg.norm(want_u))
    assert (cam.width, cam.height) == (800, 1000)


def test_look_at_refusals():
    with pytest.raises(ValueError, match="parallel"):
        vr.look_at((0, 0, 0), (0, 0, 5), (0, 0, 2), 4, 4)
    with pytest.raises(ValueError, match="parallel"):
        vr.look_at((0, 0, 0), (0, 0, 5), (0, 0, 0), 4, 4)
    with pytest.raises(ValueError, match="focal point"):
        vr.look_at((1, 2, 3), (1, 2, 3), (0, 0, 1), 4, 4)
    with pytest.raises(ValueError, match="finite"):
        vr.look_at((0, 0, float("nan")), (0, 0, 5), (0, 1, 0), 4, 4)
    with pytest.raises(ValueError, match="view_angle"):
        vr.look_at((0, 0, 0), (0, 0, 5), (0, 1, 0), 4, 4, view_angle=180)
    with pytest.raises(ValueError, match="parallel_scale"):
        vr.look_at((0, 0, 0), (0, 0, 5), (0, 1, 0), 4, 4, parallel_scale=0)
    with pytest.raises(ValueError, match="1 x 1"):
        vr.look_at((0, 0, 0), (0, 0, 5), (0, 1, 0), 0, 4)


# ---- PNG and to_uint8 ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("hw", [(1, 1), (3, 5), (64, 33)])
def test_png_round_trip(tmp_path, hw):
    rng = np.random.default_rng(sum(hw))
    img = rng.integers(0, 256, (*hw, 3), dtype=np.uint8)
    p = str(tmp_path / "x.png")
    vr.write_png(p, img)
    assert np.array_equal(vo.read_png(p), img)


def test_png_refuses_other_images(tmp_path):
    for bad in (np.zeros((4, 4, 3), np.float32), np.zeros((4, 4, 4), np.uint8), np.zeros((4, 4), np.uint8)):
        with pytest.raises(ValueError):
            vr.write_png(str(tmp_path / "x.png"), bad)


def test_to_uint8():
    x = np.array([-1.0, 0.0, 0.5 / 255, 0.49 / 255, 0.5, 1.0, 2.0, 254.5 / 255], np.float64)
    assert vr.to_uint8(x).tolist() == [0, 0, 1, 0, 128, 255, 255, 255]
    assert vr.to_uint8(x).dtype == np.uint8


# ---- refusals before any CUDA work -----------------------------------------------------------------------------------------

def test_abi_refuses_bad_arguments_before_any_cuda_call():
    lib = _lib.load()
    fake = C.c_void_p(256)            # never dereferenced: every call below is refused first
    bg = (C.c_float * 3)(0, 0, 0)
    good = dict(nx=4, ny=4, nz=4, vol=fake, n=1, H=8, W=8, cams=fake, par=0, mode=0, c0=0.0, c1=1.0, lut=fake, K=2,
                step=0.5, unit=1.0, bg=bg, out=fake)

    def call(**kw):
        a = dict(good, **kw)
        rc = lib.r2x_volume_render(None, a["nx"], a["ny"], a["nz"], a["vol"], a["n"], a["H"], a["W"], a["cams"],
                                   a["par"], a["mode"], a["c0"], a["c1"], a["lut"], a["K"], a["step"], a["unit"],
                                   a["bg"], a["out"])
        return rc, lib.r2x_last_error().decode()

    for kw, needle in [(dict(vol=None), "NULL"), (dict(cams=None), "NULL"), (dict(lut=None), "NULL"),
                       (dict(bg=None), "NULL"), (dict(out=None), "NULL"), (dict(out=C.c_void_p(260)), "aligned"),
                       (dict(nx=1), "grid"), (dict(nz=0), "grid"), (dict(n=0), "image"), (dict(H=0), "image"),
                       (dict(W=-3), "image"), (dict(n=65536), "65535"), (dict(H=16 * 65535 + 1), "65535"),
                       (dict(W=16 * 65535 + 1), "65535"), (dict(par=2), "parallel"), (dict(mode=2), "mode"),
                       (dict(mode=-1), "mode"), (dict(K=0), "K"), (dict(K=4097), "K"), (dict(c0=1.0), "clim"),
                       (dict(c0=2.0), "clim"), (dict(c1=float("nan")), "clim"), (dict(c0=-float("inf")), "clim"),
                       (dict(c0=-3e38, c1=3e38), "clim"), (dict(step=0.0), "step"), (dict(step=-1.0), "step"),
                       (dict(step=float("inf")), "step"), (dict(step=1e-12), "2^31"), (dict(unit=0.0), "unit"),
                       (dict(unit=float("nan")), "unit"), (dict(step=1e30, unit=1e-30), "unit"),
                       (dict(bg=(C.c_float * 3)(0, float("inf"), 0)), "background")]:
        rc, msg = call(**kw)
        assert rc == 1 and msg.startswith("r2x_volume_render: bad") and needle in msg, (kw, msg)


def test_python_api_refuses_before_any_gpu_work():
    vol = np.zeros((4, 5, 6), np.float32)
    cam = vr.default_camera(vol.shape, 8, 6)
    cases = [(dict(mode="shaded"), "mode"), (dict(clim=(1, 0)), "clim"), (dict(clim=(0, float("nan"))), "clim"),
             (dict(clim=(0, 1e39)), "clim"), (dict(clim=(0.5, 0.5)), "clim"), (dict(clim=(-3e38, 3e38)), "clim"), (dict(lut=np.zeros((3, 4))), "[K, 3]"),
             (dict(lut=np.zeros((0, 3))), "[K, 3]"), (dict(lut=np.zeros((4097, 3))), "[K, 3]"),
             (dict(lut=np.full((3, 3), 1.5)), "[0, 1]"), (dict(lut=np.full((3, 3), np.nan)), "[0, 1]"),
             (dict(lut="viridis"), "gray"), (dict(step=0), "step"), (dict(step=float("inf")), "step"),
             (dict(step=1e-12), "2^31"), (dict(opacity_unit=-1), "opacity_unit"), (dict(background=(0, 0)), "background"),
             (dict(background=(0, 0, float("nan"))), "background")]
    for kw, needle in cases:
        with pytest.raises(ValueError) as e:
            vr.render(vol, cam, **kw)
        assert needle in str(e.value), (kw, str(e.value))
    for bad in (np.zeros((1, 5, 6), np.float32), np.zeros((4, 5), np.float32), np.zeros((4, 5, 6, 2), np.float32)):
        with pytest.raises(ValueError, match="every axis >= 2"):
            vr.render(bad, vr.default_camera((4, 5, 6), 8, 6))
    with pytest.raises(ValueError, match="same image size"):
        vr.render(vol, [cam, vr.default_camera(vol.shape, 8, 7)])
    with pytest.raises(ValueError, match="same image size and projection"):
        vr.render(vol, [cam, vr.default_camera(vol.shape, 8, 6, parallel_scale=3.0)])
    with pytest.raises(ValueError, match="Camera"):
        vr.render(vol, [])


def _refused(capsys, argv, needle):
    with pytest.raises(SystemExit) as e:
        render_volume.parse_args(argv)
    msg = str(e.value.code) + capsys.readouterr().err
    assert needle in msg, msg


def test_cli_refusals(tmp_path, capsys):
    out = str(tmp_path / "r.png")
    vol = str(tmp_path / "v.npy")
    np.save(vol, np.zeros((8, 8, 9), np.float32))
    model = tmp_path / "model"
    model.mkdir()
    _refused(capsys, ["--output", out], "no volume")
    _refused(capsys, ["--output", out, "--vol", vol, "-m", str(model)], "not both")
    _refused(capsys, ["--output", out, "--vol", vol, "--resolution", "64"], "--resolution applies to -m")
    _refused(capsys, ["--output", out, "--vol", vol, "--iteration", "3"], "--iteration applies to -m")
    _refused(capsys, ["--output", out, "--vol", str(tmp_path / "missing.npy")], "does not exist")
    _refused(capsys, ["--output", str(tmp_path / "nodir" / "r.png"), "--vol", vol], "does not exist")
    for clim in (["1", "0"], ["0", "0"], ["nan", "1"], ["0", "inf"], ["0", "1e39"]):
        _refused(capsys, ["--output", out, "--vol", vol, "--clim", *clim], "--clim")
    for lut in (np.zeros((4, 4)), np.zeros((2, 3, 1)), np.full((4, 3), 1.01), np.full((4, 3), -0.1),
                np.full((4, 3), np.nan), np.zeros((0, 3))):
        p = str(tmp_path / "lut.npy")
        np.save(p, lut)
        _refused(capsys, ["--output", out, "--vol", vol, "--cmap", p], "--cmap")
    _refused(capsys, ["--output", out, "--vol", vol, "--cmap", "viridis"], "--cmap")
    _refused(capsys, ["--output", out, "--vol", vol, "--cmap", str(tmp_path / "none.npy")], "--cmap")
    _refused(capsys, ["--output", out, "--vol", vol, "--camera", "0", "0", "0", "0", "0", "5", "0", "0", "1"],
             "parallel to the view direction")
    _refused(capsys, ["--output", out, "--vol", vol, "--camera", "1", "1", "1", "1", "1", "1", "0", "0", "1"],
             "focal point")
    _refused(capsys, ["--output", out, "--vol", vol, "--step", "0"], "--step")
    _refused(capsys, ["--output", out, "--vol", vol, "--opacity_unit", "-1"], "--opacity_unit")
    _refused(capsys, ["--output", out, "--vol", vol, "--parallel_scale", "nan"], "--parallel_scale")
    _refused(capsys, ["--output", out, "--vol", vol, "--window_size", "0", "10"], "--window_size")
    _refused(capsys, ["--output", out, "--vol", vol, "--orbit", "0"], "--orbit")
    _refused(capsys, ["--output", out, "--vol", vol, "--view_angle", "0"], "--view_angle")
    _refused(capsys, ["--output", out, "--vol", vol, "--background", "0", "inf", "0"], "--background")
    _refused(capsys, ["--output", out, "--vol", vol, "--zero_lower_half", "w"], "--zero_lower_half")
    _refused(capsys, ["--output", out, "--vol", vol, "--mode", "iso"], "--mode")


def test_cli_reads_a_lut_file(tmp_path):
    lut = np.random.default_rng(0).random((256, 3))
    p = str(tmp_path / "viridis.npy")
    np.save(p, lut)
    vol = str(tmp_path / "v.npy")
    np.save(vol, np.zeros((4, 4, 4), np.float32))
    a = render_volume.parse_args(["--output", str(tmp_path / "r.png"), "--vol", vol, "--cmap", p])
    assert np.array_equal(a.lut, lut)
    a = render_volume.parse_args(["--output", str(tmp_path / "r.png"), "--vol", vol])
    assert np.array_equal(a.lut, vr.GRAY)
