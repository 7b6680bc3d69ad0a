"""Volume rendering on the GPU (`volume_render.render`, r2x_volume_render) against tests/volume_render_oracle.py.

1. MIP along all six axis directions, orthographic with unit pixels through voxel centres and step 1, is bit for bit
   `vol.max(axis)`, for random volumes with axes of length 2 and 3, sizes around the kernel's pixel tile (read from
   include/r2x.h) and non-cubic grids.
2. Composite is within 1e-4 per channel of the float64 oracle: random and smooth volumes, perspective and parallel
   cameras, a camera inside the box, rays along box faces and edges and through a corner, LUTs of 1, 2, 3, 256 and
   4096 entries.
3. An N-frame orbit is N single-frame calls bit for bit; two calls give the same bits; rays that miss are exactly the
   background with A = 0.
4. End to end: `render_volume` on a generated scene (-s), on --vol and on a briefly trained model (-m --resolution);
   each PNG decodes to `to_uint8` of the returned frame."""
import json
import os
import re

import numpy as np
import pytest
import torch

import volume_render_oracle as vo
from r2_gaussian_b200 import volume_render as vr

pytestmark = pytest.mark.gpu

HDR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "r2x.h")
TILE = int(re.search(r"#define R2X_VR_TILE (\d+)", open(HDR).read()).group(1))
TOL = 1e-4


def _mip_expected(vol, axis, lat, up, side):
    vm = vol.max(axis=axis, keepdims=True)
    ii = [None] * 3
    ii[axis], ii[up], ii[side] = np.zeros_like(lat[..., 0]), lat[..., 0], lat[..., 1]
    return vm[tuple(ii)]


def _shapes():
    t = TILE
    return [(2, 2, 2), (2, 3, 2), (3, 2, 3), (2, t, 3), (t - 1, 2, t + 1), (t, t, t), (t + 1, t - 1, 2 * t + 1),
            (3, 2 * t, t + 1), (37, 20, 9), (2 * t + 3, 3, 5)]


@pytest.mark.parametrize("shape", _shapes())
def test_mip_along_every_axis_is_the_max_bit_for_bit(shape):
    rng = np.random.default_rng(sum(shape))
    vol = rng.standard_normal(shape).astype(np.float32) * 0.3 + 0.5     # some values outside [0, 1]: clamped by t
    vol_d = torch.from_numpy(vol).cuda()
    for axis in range(3):
        for sign in (1, -1):
            cam, lat, (up, side) = vo.axis_view(shape, axis, sign)
            out = vr.render(vol_d, cam, mode="mip", step=1.0, clim=(0.0, 1.0))[0]
            want = np.clip(_mip_expected(vol, axis, lat, up, side), 0, 1).astype(np.float32)
            got = out.cpu().numpy()
            for c in range(3):
                assert np.array_equal(got[..., c].view(np.uint32), want.view(np.uint32)), (axis, sign, c)
            assert (got[..., 3] == 1).all()


def test_mip_of_the_raw_values_with_a_wide_clim():
    """With clim (0, 1) and values in [0, 1] the gray LUT is the identity: RGB is the maximum itself."""
    rng = np.random.default_rng(5)
    vol = rng.random((19, 33, 17), dtype=np.float32)
    for axis in range(3):
        cam, lat, (up, side) = vo.axis_view(vol.shape, axis, -1)
        got = vr.render(vol, cam, mode="mip", step=1.0)[0].cpu().numpy()
        assert np.array_equal(got[..., 1], _mip_expected(vol, axis, lat, up, side))


def _compare(vol, cams, **kw):
    got = vr.render(vol, cams, **kw).cpu().numpy().astype(np.float64)
    okw = {k: v for k, v in kw.items() if k != "opacity_unit"}
    if "opacity_unit" in kw:
        okw["unit"] = kw["opacity_unit"]
    if okw.get("lut") is None:
        okw.pop("lut", None)
    want = vo.render(np.asarray(vol, np.float32), cams if isinstance(cams, list) else [cams], **okw)
    err = np.abs(got - want).max()
    assert err <= TOL, err
    return got, want, err


def _smooth(shape):
    g = [np.linspace(-1, 1, n) for n in shape]
    X, Y, Z = np.meshgrid(*g, indexing="ij")
    q = (X / 0.8) ** 2 + (Y / 0.6) ** 2 + (Z / 0.7) ** 2
    return (np.clip(1 - q, 0, None) * 0.9 + 0.05 * np.sin(5 * X) * np.cos(3 * Y)).astype(np.float32)


def test_composite_random_and_smooth_volumes_perspective_and_parallel():
    rng = np.random.default_rng(0)
    for vol in (rng.random((24, 20, 28), dtype=np.float32), _smooth((30, 26, 22))):
        persp = vr.default_camera(vol.shape, 37, 33)
        par = vr.default_camera(vol.shape, 35, 31, parallel_scale=25.0)
        for cam in (persp, par):
            _compare(vol, cam)
            _compare(vol, cam, step=0.37, clim=(0.2, 0.8), opacity_unit=2.5, background=(0.1, 0.3, 0.9))
        side = vr.look_at((80.0, 9.5, 12.0), (10.0, 9.5, 11.0), (0.2, 0.1, 1.0), 33, 17, view_angle=25.0)
        _compare(vol, side, step=1.0)


def test_composite_camera_inside_the_box():
    vol = _smooth((32, 30, 28))
    for focal in ((31.0, 29.0, 27.0), (0.0, 15.0, 3.0), (10.0, 10.0, 10.0)):
        cam = vr.look_at((15.2, 14.1, 13.3), focal, (0.0, 0.0, 1.0), 41, 39, view_angle=90.0)
        got, _, _ = _compare(vol, cam)
        assert (got[..., 3] > 0).all()
    _compare(vol, vr.look_at((15.2, 14.1, 13.3), (15.2, 14.1, 40.0), (0.0, 1.0, 0.0), 17, 17, parallel_scale=30.0))


def test_composite_rays_along_faces_edges_and_through_corners():
    rng = np.random.default_rng(2)
    vol = rng.random((13, 17, 11), dtype=np.float32)
    for axis in range(3):
        for sign in (1, -1):
            # the image is 2 pixels larger on each side: rays on the faces and edges, and rays just outside
            cam, lat, _ = vo.axis_view(vol.shape, axis, sign, margin=2)
            got = _compare(vol, cam, step=0.5)[0][0]
            miss = lat[..., 0] < 0
            assert miss.any() and (got[miss][:, 3] == 0).all()
    # perspective views whose central ray runs through a corner, and one that skims an edge
    for corner in ((0.0, 0.0, 0.0), (12.0, 16.0, 10.0), (0.0, 16.0, 10.0)):
        c = np.asarray(corner)
        pos = c + (np.asarray(vol.shape) / 2 - 0.5 - c) * np.array([-1.7, -1.3, -1.1]) + np.array([0.0, 0.0, 0.5])
        _compare(vol, vr.look_at(pos, c, (0.0, 1.0, 1.0), 33, 32, view_angle=20.0))
    _compare(vol, vr.look_at((-20.0, -20.0, 5.0), (12.0, 16.0, 5.0), (0.0, 0.0, 1.0), 32, 16, view_angle=10.0))


@pytest.mark.parametrize("K", [1, 2, 3, 256, 4096])
def test_composite_luts(K):
    rng = np.random.default_rng(K)
    # random entries up to 256; a random 4096-entry table turns t's float32 rounding (~6e-8) into colour errors of
    # (K - 1) x the step between entries (~1e-4), so the largest table is a smooth one, as colour maps are
    lut = rng.random((K, 3)) if K <= 256 else 0.5 + 0.5 * np.sin(np.linspace(0, 6, K)[:, None] + np.arange(3))
    vol = _smooth((20, 24, 18))
    cam = vr.default_camera(vol.shape, 30, 26)
    _compare(vol, cam, lut=lut)
    _compare(vol, cam, lut=lut, clim=(0.1, 0.6))
    got = vr.render(vol, cam, mode="mip", lut=lut).cpu().numpy().astype(np.float64)
    want = vo.render(vol, [cam], mode="mip", lut=lut)
    assert np.abs(got - want).max() <= TOL


def test_orbit_is_single_frames_bit_for_bit_and_reproducible():
    gen = torch.Generator("cuda").manual_seed(3)
    vol = torch.rand((40, 36, 44), generator=gen, device="cuda")
    for mode in ("composite", "mip"):
        for base in (vr.default_camera(vol.shape, 45, 50), vr.default_camera(vol.shape, 45, 50, parallel_scale=40.0)):
            cams = vr.orbit(base, 7)
            many = vr.render(vol, cams, mode=mode)
            again = vr.render(vol, cams, mode=mode)
            assert many.shape == (7, 50, 45, 4)
            assert torch.equal(many.view(torch.int32), again.view(torch.int32))
            for k, c in enumerate(cams):
                one = vr.render(vol, c, mode=mode)
                assert torch.equal(one[0].view(torch.int32), many[k].view(torch.int32)), (mode, k)


def test_rays_that_miss_are_the_background():
    vol = torch.rand((16, 16, 16), device="cuda")
    bg = (0.2, 0.5, 0.7)
    away = vr.look_at((40.0, 40.0, 40.0), (80.0, 80.0, 90.0), (0.0, 0.0, 1.0), 20, 20)
    for mode in ("composite", "mip"):
        out = vr.render(vol, away, mode=mode, background=bg)[0].cpu().numpy()
        assert (out[..., :3] == np.float32(bg)).all() and (out[..., 3] == 0).all()
    # a wide view: the corners of the image miss the box
    wide = vr.default_camera(vol.shape, 64, 64, view_angle=90.0)
    o, d, s0, s1, meets = vo.ray_setup(wide.record(), 64, 64, False, vol.shape)
    assert (~meets).sum() > 100 and meets.sum() > 100
    for mode in ("composite", "mip"):
        out = vr.render(vol, wide, mode=mode, background=bg)[0].cpu().numpy().reshape(-1, 4)
        assert (out[~meets, :3] == np.float32(bg)).all() and (out[~meets, 3] == 0).all()
        if mode == "mip":
            assert (out[meets, 3] == 1).all()


def test_below_clim_is_the_exact_background_and_device_inputs():
    vol = torch.rand((20, 21, 22), device="cuda") * 0.3
    bg = (0.25, 0.5, 0.75)
    out = vr.render(vol, vr.default_camera(vol.shape, 40, 30), clim=(0.3, 1.0), background=bg)[0].cpu().numpy()
    assert (out[..., :3] == np.float32(bg)).all() and (out[..., 3] == 0).all()
    # float64 host input is rounded to float32 first
    v64 = vol.double().cpu().numpy()
    a = vr.render(v64, vr.default_camera(vol.shape, 40, 30), clim=(0.1, 0.3))
    b = vr.render(vol, vr.default_camera(vol.shape, 40, 30), clim=(0.1, 0.3))
    assert torch.equal(a, b)
    bad = vol.clone()
    bad[3, 4, 5] = float("nan")
    with pytest.raises(ValueError, match="render: the volume holds non-finite values"):
        vr.render(bad, vr.default_camera(vol.shape, 8, 8))


# ---- 4. end to end --------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def ellipsoid_scene(tmp_path_factory):
    """A 32^3 generate_data scene of a smooth ellipsoid (16 train, 4 test views of 64^2) with its initial cloud."""
    from r2_gaussian_b200 import generate_data, initialize_pcd, scene
    tmp = tmp_path_factory.mktemp("render_scene")
    n = 32
    np.save(tmp / "vol.npy", _smooth((n, n, n)).clip(0, 1))
    sc = scene.cone_beam_scanner(64, n)
    phys = {k: (np.asarray(v, float) * 2.0).tolist() if k in ("DSD", "DSO", "sDetector", "sVoxel", "offOrigin",
                                                              "offDetector") else v for k, v in sc.items()}
    phys.update({"filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0, "noise": False})
    (tmp / "scanner.yml").write_text("".join(f"{k}: {json.dumps(v)}\n" for k, v in phys.items()))
    src = generate_data.main(["--vol", str(tmp / "vol.npy"), "--scanner", str(tmp / "scanner.yml"), "--n_train", "16",
                              "--n_test", "4", "--output", str(tmp / "data")])
    init = initialize_pcd.main(["--data", src, "--n_points", "3000", "--output", str(tmp / "init.npy")])
    return src, init, tmp


def _run(argv, capsys):
    from r2_gaussian_b200 import render_volume
    rep, frames = render_volume.run(argv)
    line = capsys.readouterr().out.strip().splitlines()[-1]
    assert json.loads(line) == json.loads(json.dumps(rep))
    imgs = vr.to_uint8(frames[..., :3]).cpu().numpy()
    pngs = [p for p in rep["outputs"] if p.endswith(".png")]
    assert len(pngs) == rep["frames"] == frames.shape[0]
    for p, img in zip(pngs, imgs):
        assert np.array_equal(vo.read_png(p), img), p
    return rep, frames


def test_render_volume_end_to_end(ellipsoid_scene, tmp_path, capsys):
    from r2_gaussian_b200 import trainer
    from r2_gaussian_b200.dataset import read_scene
    src, init, tmp = ellipsoid_scene
    rep, frames = _run(["-s", src, "--window_size", "80", "100", "--output", str(tmp_path / "gt.png")], capsys)
    assert rep["source"] == "scene" and rep["shape"] == [32, 32, 32] and rep["mode"] == "composite"
    assert frames.shape == (1, 100, 80, 4) and (rep["width"], rep["height"]) == (80, 100)
    # the same pixels as the API on the scene's volume, and the oracle's
    vol = read_scene(src, eval=False).vol
    cam = vr.default_camera(vol.shape, 80, 100)
    assert torch.equal(frames, vr.render(vol, cam))
    assert np.abs(frames.cpu().numpy() - vo.render(vol, [cam])).max() <= TOL
    assert frames[0, ..., 3].max() > 0.5

    # --vol, the Fig. 1 recipe: plot_volume.py's lower half zeroed along x, MIP, a LUT file, --orbit and --save_npy
    lut = str(tmp_path / "lut.npy")
    np.save(lut, np.random.default_rng(0).random((256, 3)))
    rep, frames = _run(["--vol", str(tmp / "vol.npy"), "--zero_lower_half", "x", "--cmap", lut, "--window_size", "48",
                        "40", "--orbit", "4", "--save_npy", "--output", str(tmp_path / "orbit.png")], capsys)
    assert rep["frames"] == 4 and rep["source"] == "vol"
    assert sorted(os.listdir(tmp_path)) == sorted(["gt.png", "lut.npy", "orbit.npy"] +
                                                  [f"orbit_{k:04d}.png" for k in range(4)])
    assert np.array_equal(np.load(tmp_path / "orbit.npy"), frames.cpu().numpy())
    half = np.load(tmp / "vol.npy")
    half[:16] = 0
    cams = vr.orbit(vr.default_camera(half.shape, 48, 40), 4)
    assert torch.equal(frames, vr.render(half, cams, lut=np.load(lut)))
    cpos = ["-5", "40", "50", "15.5", "15.5", "15.5", "0", "0", "3"]
    rep, frames = _run(["--vol", str(tmp / "vol.npy"), "--mode", "mip", "--camera", *cpos, "--parallel_scale", "20",
                        "--window_size", "30", "20", "--clim", "0.1", "0.9", "--output", str(tmp_path / "mip.png")],
                       capsys)
    cam = vr.look_at((-5, 40, 50), (15.5, 15.5, 15.5), (0, 0, 3), 30, 20, parallel_scale=20.0)
    assert torch.equal(frames, vr.render(np.load(tmp / "vol.npy"), cam, mode="mip", clim=(0.1, 0.9)))

    # a briefly trained model, queried at 40^3
    model = tmp_path / "model"
    trainer.main(["-s", src, "-m", str(model), "--ply_path", init, "--iterations", "200", "--test_iterations", "200",
                  "--save_iterations", "200"])
    capsys.readouterr()
    rep, frames = _run(["-m", str(model), "--resolution", "40", "--window_size", "64", "64", "--output",
                        str(tmp_path / "pred.png")], capsys)
    assert rep["source"] == "model@200" and rep["shape"] == [40, 40, 40]
    assert frames[0, ..., 3].max() > 0.1
