"""The TV kernels on the GPU (r2x_tv_prox through tv.tv_denoise, r2x_tv_value through tv.tv_value) against the float64
statement of tests/tv_oracle.py; GPU FISTA-TV against `fista_tv_solve` over the float64 oracle operators; and FISTA-TV
end to end on a noisy `generate_data` scene, through `python -m r2_gaussian_b200.recon --methods fista_tv` and
`initialize_pcd --recon_method fista_tv --evaluate`."""
import math
import os
import re

import numpy as np
import pytest
import yaml

import backproject_oracle as bo
import tv_oracle as tvo
from test_projector_gpu import _write_inputs
from test_recon_gpu import SOLVER_BOUND, _tiny_case

pytestmark = pytest.mark.gpu

# GPU prox (float32) against the float64 FGP with the same iteration count, relative to max |x|
PROX_BOUND = 1e-5
# r2x_tv_value against the float64 sum of the same float32 volume
VALUE_BOUND = 1e-6


def _torch():
    import torch

    return torch


@pytest.mark.parametrize("nonneg", [True, False])
@pytest.mark.parametrize("shape", [(20, 36, 28), (1, 33, 17), (64, 64, 64)])
def test_prox_matches_float64_fgp(shape, nonneg):
    torch = _torch()
    from r2_gaussian_b200.tv import tv_denoise

    rng = np.random.RandomState(sum(shape))
    v = rng.uniform(-0.3, 1.0, size=shape).astype(np.float32)
    vt = torch.tensor(v, device="cuda")
    for w, niter in ((0.05, 20), (0.2, 7)):
        got = tv_denoise(vt, w, niter, nonneg)
        again = tv_denoise(vt, w, niter, nonneg)
        assert got.view(torch.int32).equal(again.view(torch.int32))          # bitwise reproducible
        want = tvo.fgp(v, w, niter, nonneg)[0]
        err = np.abs(got.cpu().numpy().astype(np.float64) - want).max() / np.abs(want).max()
        print(f"prox {shape} nonneg {nonneg} w {w} niter {niter}: max err / max = {err:.3g}")
        assert err <= PROX_BOUND, err
        if nonneg:
            assert float(got.min()) >= 0.0
    # weight 0: the projection of v, bit for bit
    zero = tv_denoise(vt, 0.0, 5, nonneg)
    want = torch.where(vt < 0, torch.zeros_like(vt), vt) if nonneg else vt
    assert zero.view(torch.int32).equal(want.view(torch.int32))


@pytest.mark.parametrize("shape", [(20, 36, 28), (1, 33, 17), (64, 64, 64), (1, 1, 1)])
def test_value_matches_float64(shape):
    torch = _torch()
    from r2_gaussian_b200.tv import tv_value

    v = np.random.RandomState(3).uniform(0.0, 1.0, size=shape).astype(np.float32)
    got = tv_value(torch.tensor(v, device="cuda"))
    assert got == tv_value(torch.tensor(v, device="cuda"))
    want = tvo.tv_value(v)
    print(f"tv {shape}: {got!r} vs {want!r}")
    assert abs(got - want) <= VALUE_BOUND * max(want, 1e-30) or (want == 0.0 and got == 0.0)


def test_fista_tv_matches_the_oracle_solver():
    torch = _torch()
    from r2_gaussian_b200 import recon

    sc, angles, b = _tiny_case()
    A, At = bo.operators(angles, sc)
    bt = torch.tensor(b, dtype=torch.float32, device="cuda")
    for nonneg in (True, False):
        got, hist = recon.fista_tv(bt, angles, sc, 3, 0.01, 10, nonneg)
        again, _ = recon.fista_tv(bt, angles, sc, 3, 0.01, 10, nonneg)
        assert got.view(torch.int32).equal(again.view(torch.int32))
        want, want_hist = recon.fista_tv_solve(torch.from_numpy(b), A, At, sc["nVoxel"], 3, 0.01, 10, nonneg=nonneg,
                                               prox=tvo.prox, tv=tvo.tv)
        want = want.numpy()
        err = np.abs(got.cpu().numpy().astype(np.float64) - want).max() / np.abs(want).max()
        print(f"fista_tv nonneg {nonneg}: max err / max = {err:.3g}; F {hist[-1]['F']:.6g} vs {want_hist[-1]['F']:.6g}")
        assert err <= SOLVER_BOUND, err
        assert abs(hist[-1]["F"] - want_hist[-1]["F"]) <= 1e-4 * want_hist[-1]["F"]


# ---- a noisy generate_data scene ------------------------------------------------------------------------------------

# psnr_3d margins of FISTA-TV at its defaults over the unregularised methods, in dB (fixed before the first run)
MARGIN_DB = {"fdk": 1.0, "cgls": 1.0, "sart": 0.25}


@pytest.fixture(scope="module")
def noisy_scene(tmp_path_factory):
    """24 train and 6 test views of 96^2 of the round-trip volume on a 48^3 grid, Poisson (1e5) + Gaussian noise."""
    from r2_gaussian_b200 import generate_data

    tmp = tmp_path_factory.mktemp("tv_scene")
    yml, vol_path, *_ = _write_inputs(tmp, noise=True)
    return generate_data.main(["--vol", str(vol_path), "--scanner", str(yml), "--n_train", "24", "--n_test", "6",
                               "--output", str(tmp / "data")])


def test_fista_tv_beats_the_unregularised_methods(noisy_scene):
    torch = _torch()
    from r2_gaussian_b200 import recon
    from r2_gaussian_b200.dataset import read_blender
    from r2_gaussian_b200.metrics import metric_vol

    info = read_blender(noisy_scene, eval=False)
    cfg = info.scanner_cfg
    b = torch.tensor(np.stack([c.image for c in info.train_cameras]), dtype=torch.float32, device="cuda")
    angles = [c.angle for c in info.train_cameras]
    x, hist = recon.fista_tv(b, angles, cfg)
    assert len(hist) == recon.FISTA_NITER
    assert hist[-1]["F"] < hist[0]["F"] and all(math.isfinite(h["F"]) for h in hist)
    assert float(x.min()) >= 0.0
    psnr = {m: metric_vol(info.vol, recon.recon_volume(b, angles, cfg, m).cpu().numpy(), "psnr")[0]
            for m in ("fdk", "sart", "cgls")}
    psnr["fista_tv"] = metric_vol(info.vol, x.cpu().numpy(), "psnr")[0]
    print(f"psnr_3d {psnr}")
    for m, margin in MARGIN_DB.items():
        assert psnr["fista_tv"] >= psnr[m] + margin, (m, psnr)


def test_cli_end_to_end(noisy_scene, tmp_path, capsys):
    from r2_gaussian_b200 import initialize_pcd, recon
    from r2_gaussian_b200.metrics import metric_vol

    out = tmp_path / "trad"
    report = recon.main(["-s", noisy_scene, "-m", str(out), "--methods", "fdk,fista_tv"])
    with open(out / "eval_3d.yml") as f:
        top = yaml.safe_load(f)
    assert list(top) == ["fdk", "fista_tv"] and report["fista_tv"] == top["fista_tv"]
    keys = ["method", "psnr_3d", "ssim_3d", "ssim_3d_x", "ssim_3d_y", "ssim_3d_z", "duration (sec)", "duration (min)"]
    with open(out / "fista_tv" / "eval_3d.yml") as f:
        per = yaml.safe_load(f)
    assert list(per) == keys and per == top["fista_tv"] and per["method"] == "fista_tv"
    vol_gt = np.load(os.path.join(noisy_scene, "vol_gt.npy"))
    assert np.array_equal(np.load(out / "fista_tv" / "ct_gt.npy"), vol_gt)
    pred = np.load(out / "fista_tv" / "ct_pred.npy")
    assert pred.shape == vol_gt.shape and pred.dtype == np.float32
    assert per["psnr_3d"] == metric_vol(vol_gt, pred, "psnr")[0]
    names = sorted(os.listdir(out / "fista_tv" / "projs"))
    assert names == sorted([f"{i:05d}_render.npy" for i in range(6)] + [f"{i:05d}_gt.npy" for i in range(6)])

    capsys.readouterr()
    init = initialize_pcd.main(["--data", noisy_scene, "--recon_method", "fista_tv", "--n_points", "400",
                                "--output", str(tmp_path / "init_tv.npy"), "--evaluate"])
    assert os.path.exists(init)
    psnr = re.findall(r"3D PSNR for initial Gaussians: (\S+)", capsys.readouterr().out)
    assert len(psnr) == 1 and math.isfinite(float(psnr[0])), psnr
