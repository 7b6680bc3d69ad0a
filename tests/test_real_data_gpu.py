"""r2x_projection_prepare on the GPU against the numpy restatement and cv2's golden bytes, chunking and
reproducibility, and `generate_real_data` end to end on a FIPS-format scan made from a seeded phantom."""
import json
import os
import random

import numpy as np
import pytest

import real_data_oracle as oracle
from test_real_data_cpu import CASES, golden

pytestmark = pytest.mark.gpu

# fixed before the first run; reached on an H100 80GB HBM3 (700 W): 33.49 and 43.55 dB (DESIGN §8)
VOL_GT_PSNR_BAR = 22.0        # pseudo-GT FDK of 90 views against the phantom, 3D PSNR in dB
TRAIN_PSNR_BAR = 20.0         # fdk-initialised trainer, 1000 iterations, against the pseudo-GT


def _prepare(img, s, rescale, obj):
    import torch

    from r2_gaussian_b200 import generate_real_data as grd

    return grd.prepare(torch.from_numpy(np.ascontiguousarray(img)).cuda(), s, rescale, obj).cpu().numpy()


@pytest.mark.parametrize("name", CASES)
def test_kernel_equals_oracle_and_cv2_golden(name):
    img, s, rescale, obj, want = golden(name)
    got = _prepare(img[None], s, rescale, obj)[0]
    assert got.tobytes() == oracle.prepare(img, s, rescale, obj).tobytes()
    assert got.tobytes() == want.tobytes()


@pytest.mark.parametrize("H0,W0,s", [(1536, 1944, 4), (2368, 2240, 4), (301, 257, 3), (9, 40, 2), (6, 6, 1)])
def test_kernel_equals_oracle_on_stacks(H0, W0, s):
    rng = np.random.default_rng(H0 * W0 + s)
    img = rng.normal(0.4, 0.7, (3, H0, W0)) * 8.0
    got = _prepare(img, s, 400.0, 50)
    for v in range(3):
        assert got[v].tobytes() == oracle.prepare(img[v], s, 400.0, 50).tobytes(), v


def test_chunking_and_repeats_give_the_same_bits(tmp_path):
    from r2_gaussian_b200 import generate_real_data as grd

    rng = np.random.default_rng(5)
    imgs = [rng.normal(0.4, 0.7, (91, 103)) * 8.0 for _ in range(11)]
    oracle.write_fips_case(str(tmp_path), imgs, 0.0, 10.0)
    paths = sorted(str(tmp_path / f) for f in os.listdir(tmp_path) if f.endswith(".mat"))
    ref = grd.prepare_files(paths, 4, 400.0, 50, chunk=11).cpu().numpy()
    for chunk in (1, 3, 4, 32):
        assert grd.prepare_files(paths, 4, 400.0, 50, chunk=chunk).cpu().numpy().tobytes() == ref.tobytes(), chunk
    assert grd.prepare_files(paths, 4, 400.0, 50, chunk=11).cpu().numpy().tobytes() == ref.tobytes()
    for v in (0, 5, 10):
        assert ref[v].tobytes() == oracle.prepare(imgs[v], 4, 400.0, 50).tobytes()


def _phantom(n, rng):
    g = (np.arange(n) + 0.5) / n * 2.0 - 1.0
    x, y, z = np.meshgrid(g, g, g, indexing="ij")
    vol = np.zeros((n, n, n), np.float32)
    for _ in range(6):
        c = rng.uniform(-0.35, 0.35, 3)
        r = rng.uniform(0.15, 0.4, 3)
        vol += rng.uniform(0.2, 0.6) * ((((x - c[0]) / r[0]) ** 2 + ((y - c[1]) / r[1]) ** 2
                                          + ((z - c[2]) / r[2]) ** 2) <= 1.0)
    return vol


def _fips_scan(tmp_path, n=48, views=90, interval=4.0, proj_rescale=400.0, object_scale=50, pixel_mm=1.0):
    """A scan of a seeded phantom in the processed FIPS layout: projected at a detector 4x finer than the one the
    builder makes (256 x 256 raw pixels of pixel_mm / 4), multiplied by proj_rescale / object_scale, moved down 5 rows."""
    import torch

    from r2_gaussian_b200.projector import project

    rng = np.random.default_rng(11)
    vol = _phantom(n, rng)
    dsd, dso = 553.74, 410.66
    fine = 256
    d_raw = pixel_mm / 4 / 1000 * object_scale                     # raw pitch in scene units
    cfg = {"mode": "cone", "DSD": dsd / 1000 * object_scale, "DSO": dso / 1000 * object_scale,
           "nDetector": [fine, fine], "sDetector": [fine * d_raw, fine * d_raw], "nVoxel": [n, n, n],
           "sVoxel": [2.0, 2.0, 2.0], "offOrigin": [0.0, 0.0, 0.0], "offDetector": [0.0, 0.0], "accuracy": 0.5,
           "dVoxel": [2.0 / n] * 3, "dDetector": [d_raw, d_raw]}
    angles = np.concatenate([np.arange(0.0, interval * (views - 1), interval), [interval * (views - 1)]]) / 180 * np.pi
    projs = project(torch.from_numpy(vol).cuda(), angles, cfg).cpu().numpy().astype(np.float64)
    raw = np.zeros_like(projs)
    raw[:, 5:] = projs[:, :-5] * proj_rescale / object_scale
    oracle.write_fips_case(str(tmp_path / "scan"), list(raw), 0.0, interval, dsd=dsd, dso=dso, pixel=pixel_mm / 4)
    return str(tmp_path / "scan"), vol


def test_generate_real_data_end_to_end(tmp_path):
    import torch

    from r2_gaussian_b200 import dataset, generate_real_data as grd, initialize_pcd, trainer
    from r2_gaussian_b200.fdk import fdk
    from r2_gaussian_b200.metrics import metric_vol

    scan, phantom = _fips_scan(tmp_path)
    out = str(tmp_path / "scene")
    state = random.getstate()
    grd.main(["--data", scan, "--output", out, "--n_train", "30", "--n_test", "20", "--nVoxel", "48", "48", "48"])
    assert random.getstate() == state

    with open(os.path.join(out, "meta_data.json")) as f:
        meta = json.load(f)
    assert meta["vol"] == meta["ct"] == "vol_gt.npy"
    assert len(meta["proj_train"]) == 30 and len(meta["proj_test"]) == 20
    assert len(os.listdir(os.path.join(out, "proj_all"))) == 90
    sc = meta["scanner"]
    assert sc["nDetector"] == [64, 64] and sc["mode"] == "cone" and sc["noise"] is True and sc["filter"] is None
    assert sc["totalAngle"] == 356.0 and sc["startAngle"] == 0.0
    info = dataset.read_blender(out)
    assert len(info.train_cameras) == 30 and info.vol.shape == (48, 48, 48)

    # vol_gt is fdk.fdk of proj_all in scene units, clamped, bit for bit
    names = sorted(os.listdir(os.path.join(out, "proj_all")))
    stack = torch.from_numpy(np.stack([np.load(os.path.join(out, "proj_all", n)) for n in names])).cuda()
    scaled = dict(sc)
    scale = dataset.scale_scanner(scaled)
    angles = np.concatenate([np.arange(0.0, 356.0, 4.0), [356.0]]) / 180.0 * np.pi
    vol = fdk(stack * scale, angles, scaled)
    want = torch.where(vol < 0, torch.zeros_like(vol), vol).cpu().numpy()
    got = np.load(os.path.join(out, "vol_gt.npy"))
    assert got.tobytes() == want.tobytes()
    psnr_gt = metric_vol(phantom, got, "psnr")[0]
    print(f"pseudo-GT 3D PSNR against the phantom: {psnr_gt:.2f} dB")
    assert psnr_gt > VOL_GT_PSNR_BAR

    # an existing vol_gt.npy is kept
    np.save(os.path.join(out, "vol_gt.npy"), np.zeros((48, 48, 48), np.float32))
    grd.main(["--data", scan, "--output", out, "--n_train", "30", "--n_test", "20", "--nVoxel", "48", "48", "48"])
    assert not np.load(os.path.join(out, "vol_gt.npy")).any()
    np.save(os.path.join(out, "vol_gt.npy"), got)

    init = initialize_pcd.main(["--data", out, "--recon_method", "fdk", "--n_points", "3000",
                                "--output", str(tmp_path / "init.npy")])
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    model = trainer.ModelParams(source_path=out, model_path="", ply_path=init)
    hist = trainer.training(model, trainer.OptimizationParams(iterations=1000), trainer.PipelineParams(), {1000},
                            set(), log=lambda *a: None)
    psnr_train = hist["eval"][1000]["psnr_3d"]
    print(f"trainer after 1000 iterations, 3D PSNR against the pseudo-GT: {psnr_train:.2f} dB")
    assert psnr_train > TRAIN_PSNR_BAR
