"""`resample.zoom` on the GPU against scipy.ndimage.zoom, copies and reproducibility, `process_raw_data` end to end
against the reference's scipy chains (within 1 float32 ulp) and through `generate_data` into a scene, and a
kingsnake-sized chain (1024 x 1024 x 795 uint8, expand, 256^3) against a windowed float64 restatement."""
import os

import numpy as np
import pytest
import scipy.ndimage as ndimage

import raw_data_oracle as oracle
from test_raw_data_cpu import TARGET, ZOOM_CASES, make_cases, readers, reference_case  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu


def _zoom(x, factors):
    import torch

    from r2_gaussian_b200.resample import zoom

    return zoom(torch.from_numpy(np.ascontiguousarray(x)).cuda(), factors).cpu().numpy()


def _check(x, factors):
    want = ndimage.zoom(x, factors, order=3, mode="nearest")
    got = _zoom(x, factors)
    assert got.shape == want.shape
    err = np.abs(got - want).max()
    assert err <= 1e-12, err


@pytest.mark.parametrize("shape,factors", ZOOM_CASES)
def test_zoom_matches_scipy(shape, factors):
    _check(np.random.default_rng(sum(shape)).random(shape), factors)


# padded row lengths 25, 31 .. 33, 55 .. 57, 64, 281: around the 32-voxel staging tile of the contiguous axis
@pytest.mark.parametrize("nz", [1, 7, 8, 9, 31, 32, 33, 40, 257])
def test_zoom_contiguous_axis_lengths(nz):
    x = np.random.default_rng(nz).random((9, 13, nz))
    _check(x, (1.7, 0.6, 0.8))
    _check(x, (0.5, 2.0, 2.3))


def test_zoom_256_cube_to_97x300x128():
    x = np.random.default_rng(3).random((256, 256, 256))
    _check(x, (97 / 256, 300 / 256, 0.5))


def test_unit_factors_copy_and_runs_repeat_bit_for_bit():
    import torch

    from r2_gaussian_b200.resample import zoom

    x = torch.from_numpy(np.random.default_rng(4).random((37, 41, 45))).cuda()
    assert zoom(x, 1.0).cpu().numpy().tobytes() == x.cpu().numpy().tobytes()
    assert zoom(x.permute(2, 0, 1), (1, 1, 1)).cpu().numpy().tobytes() == x.permute(2, 0, 1).cpu().numpy().tobytes()
    a = zoom(x, (2.1, 0.7, 1.3)).cpu().numpy()
    b = zoom(x, (2.1, 0.7, 1.3)).cpu().numpy()
    assert a.tobytes() == b.tobytes()
    # a strided view zooms as its contiguous copy
    assert zoom(x.permute(2, 0, 1), 0.9).cpu().numpy().tobytes() == \
        zoom(x.permute(2, 0, 1).contiguous(), 0.9).cpu().numpy().tobytes()


def test_placed_sources_match_the_placement_oracle():
    from r2_gaussian_b200 import process_raw_data as prd
    from r2_gaussian_b200.resample import Place, zoom_placed

    rng = np.random.default_rng(5)
    for dtype in (np.uint8, np.uint16, np.float64):
        src = oracle.blob_volume((21, 14, 17), rng, dtype).transpose(2, 0, 1)     # a strided host view
        for place in (prd.normalising_place(src, "t"), prd.cube_place(src.shape, "expand"),
                      prd.cube_place(src.shape, "crop"), Place((30, 12, 25), (4, -1, 2), 3.0, 200.0)):
            for factors in ((1, 1, 1), (0.8, 1.9, 0.45)):
                got = zoom_placed(src, factors, place).cpu().numpy()
                want = ndimage.zoom(oracle.place(src, place), factors, order=3, mode="nearest")
                if factors == (1, 1, 1):
                    assert got.tobytes() == want.tobytes(), (dtype, place)
                else:
                    assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max()), (dtype, place)


# One float32 ulp of the voxel, but never finer than a float32 ulp at 2^-26 (1.8e-15): below that the float64 chains'
# own rounding on [0, 1] data (~1e-16) decides the float32 bits, e.g. the sign of the +-1e-20 ringing in a zero pad.
ULP_FLOOR = float(np.spacing(np.float32(2.0 ** -26)))


def _ulps(got, want):
    """Voxels where two float32 arrays differ, and the largest difference in units of the 1-ulp bar."""
    tol = np.maximum(np.spacing(np.abs(want)).astype(np.float64), ULP_FLOOR)
    return int((got != want).sum()), float((np.abs(got.astype(np.float64) - want) / tol).max())


def test_process_raw_data_end_to_end(tmp_path, readers):  # noqa: F811
    import yaml

    from r2_gaussian_b200 import dataset, generate_data, process_raw_data as prd, scene

    cases = make_cases(str(tmp_path / "raw"), np.random.default_rng(7))
    meta = str(tmp_path / "meta.py")
    oracle.write_metadata(meta, cases)
    out = str(tmp_path / "vols")
    assert len(prd.main(["--metadata", meta, "--output", out, "--target_size", str(TARGET)])) == len(cases)
    for case in cases:
        got = np.load(os.path.join(out, case["output_name"] + ".npy"))
        want = reference_case(case, TARGET).astype(np.float32)
        assert got.dtype == np.float32 and got.shape == want.shape == (TARGET,) * 3
        n_diff, worst = _ulps(got, want)
        print(f"{case['output_name']}: {n_diff} of {got.size} voxels differ from scipy's chain, at most {worst:.2f} ulp")
        assert worst <= 1.0, case["output_name"]
    assert prd.main(["--metadata", meta, "--output", out, "--target_size", str(TARGET)]) == []   # all skipped

    scanner = scene.cone_beam_scanner(32, TARGET)
    scanner.update({"filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0, "noise": False})
    yml = tmp_path / "cone.yml"
    yml.write_text(yaml.safe_dump(scanner))
    case_dir = generate_data.main(["--vol", os.path.join(out, "raw_expand.npy"), "--scanner", str(yml),
                                   "--output", str(tmp_path / "scenes"), "--n_train", "8", "--n_test", "2"])
    info = dataset.read_scene(case_dir, eval=True)
    assert len(info.train_cameras) == 8 and len(info.test_cameras) == 2
    assert np.array_equal(np.asarray(info.vol), np.load(os.path.join(out, "raw_expand.npy")))
    assert all(np.isfinite(c.image).all() and c.image.max() > 0 for c in info.train_cameras)


KINGSNAKE = dict(shape=(1024, 1024, 795), spacing=[0.03174 * 20, 0.03174 * 20, 0.0688 * 20])


def kingsnake_volume():
    """A seeded kingsnake-sized uint8 volume [x, y, z]: smooth blobs plus noise, cheap to make at this size."""
    rng = np.random.default_rng(11)
    nx, ny, nz = KINGSNAKE["shape"]
    gx, gy, gz = (np.linspace(-1, 1, n, dtype=np.float32) for n in (nx, ny, nz))
    blobs = []
    for _ in range(3):
        c, r = rng.uniform(-0.4, 0.4, 3), rng.uniform(0.3, 0.6, 3)
        blobs.append((np.float32(rng.uniform(0.3, 0.6)) * np.exp(-((gx - c[0]) / r[0]) ** 2),
                      np.exp(-((gy - c[1]) / r[1]) ** 2), np.exp(-((gz - c[2]) / r[2]) ** 2)))
    vol = rng.integers(0, 40, (nx, ny, nz), dtype=np.uint8)
    for x0 in range(0, nx, 64):                      # 64 x-slices at a time keeps the float32 temporaries small
        slab = sum(fx[x0:x0 + 64, None, None] * fy[None, :, None] * fz[None, None, :] for fx, fy, fz in blobs)
        vol[x0:x0 + 64] += (slab * np.float32(110.0)).astype(np.uint8)
    return vol


def test_kingsnake_sized_chain_within_20_gb():
    import torch

    from r2_gaussian_b200 import process_raw_data as prd
    from r2_gaussian_b200.resample import zoom_placed

    src = kingsnake_volume()
    place = prd.normalising_place(src, "kingsnake")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    vol = prd.reshape_vol(src, place, KINGSNAKE["spacing"], 256, "expand", zoom_placed)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f"kingsnake-sized chain: peak device memory {peak / 1e9:.2f} GB")
    assert peak <= 20e9
    out = vol.cpu().numpy()
    assert out.shape == (256,) * 3 and np.isfinite(out).all()
    out = out.clip(0.0, 1.0).astype(np.float32)
    assert out.min() >= 0.0 and out.max() <= 1.0 and out.max() > 0.5

    # spot checks against the two zooms restated in float64 on windows of the source
    factors, places = prd.reshape_plan(src.shape, KINGSNAKE["spacing"], 256, "expand")
    resampled = oracle.zoom_shape(src.shape, factors[0])
    cube = places[0]

    def placed_src(i0, i1, i2):
        return (src[np.ix_(i0, i1, i2)].astype(np.float64) - place.lo) / (place.hi - place.lo)

    def cube_values(i0, i1, i2):          # the expanded cube at cube indices: stage-A zoom values or 0
        idx = [np.asarray(i) - o for i, o in zip((i0, i1, i2), cube.offset)]
        inside = [(i >= 0) & (i < n) for i, n in zip(idx, resampled)]
        vals = np.zeros((len(i0), len(i1), len(i2)))
        sub = [i[m] for i, m in zip(idx, inside)]
        if all(len(s) for s in sub):
            box = [(int(s.min()), int(s.max()) + 1) for s in sub]
            a = oracle.zoom_box(placed_src, src.shape, factors[0], box=box, margin=32)
            a = a[np.ix_(*[s - b[0] for s, b in zip(sub, box)])]
            vals[np.ix_(*inside)] = a
        return vals

    for p in [(128, 128, 128), (0, 0, 0), (255, 17, 200), (40, 250, 3), (90, 160, 255)]:
        ref = oracle.zoom_box(cube_values, cube.shape, factors[1], box=[(c, c + 1) for c in p], margin=32)[0, 0, 0]
        want = np.float32(np.clip(ref, 0.0, 1.0))
        assert abs(float(out[p]) - float(want)) <= float(np.spacing(want)), (p, out[p], want)
