"""The matched backprojector on the GPU (r2_gaussian_b200.projector.backproject over r2x_volume_backproject) against the
float64 transpose oracle and as the adjoint of the GPU projector; CGLS / SART of r2_gaussian_b200.recon against the same
solvers over the oracle operators; and the reconstructions end to end on a `generate_data` scene, through
`python -m r2_gaussian_b200.recon` and `initialize_pcd --recon_method cgls --evaluate`."""
import math
import os
import re

import numpy as np
import pytest
import yaml

import backproject_oracle as bo
import fdk_cases as fc
from test_projector_gpu import ORACLE_CASES, _scanner, _write_inputs

pytestmark = pytest.mark.gpu

# GPU solver (float32 operators) against the same solver over the float64 oracle operators, 3 iterations on the tiny
# case below, relative to the largest voxel (measured 3.1e-7 CGLS, 1.2e-6 SART, 1.1e-6 OS-SART on an H100)
SOLVER_BOUND = 1e-5


def _torch():
    import torch

    return torch


def _rand(shape, seed, lo=0.0):
    return np.random.RandomState(seed).uniform(lo, 1.0, size=shape).astype(np.float32)


@pytest.mark.parametrize("name", sorted(ORACLE_CASES))
def test_backproject_matches_oracle(name):
    torch = _torch()
    from r2_gaussian_b200.projector import backproject

    mode, det, vox, sv, off, acc, angles = ORACLE_CASES[name]
    sc = _scanner(mode, det, vox, sv, off, acc)
    y = _rand((len(angles), *det), len(name))
    got = backproject(torch.tensor(y, device="cuda"), angles, sc).cpu().numpy()
    want = bo.backproject_scene(y, angles, sc)
    assert got.shape == tuple(vox)
    err = np.abs(got.astype(np.float64) - want).max()
    print(f"backproject {name}: max err / max = {err / np.abs(want).max():.3g}")
    assert err <= 1e-5 * np.abs(want).max(), (err, np.abs(want).max())
    assert (got[want == 0.0] == 0.0).all()                            # no ray reaches them: exactly 0


def _dot_gap(sc, angles, x, y):
    torch = _torch()
    from r2_gaussian_b200.projector import backproject, project

    ax = project(torch.tensor(x, device="cuda"), angles, sc).cpu().numpy().astype(np.float64)
    aty = backproject(torch.tensor(y, device="cuda"), angles, sc).cpu().numpy().astype(np.float64)
    lhs, rhs = float((ax * y).sum()), float((x * aty).sum())
    return lhs, rhs


@pytest.mark.parametrize("name", sorted(ORACLE_CASES))
def test_dot_product_small(name):
    mode, det, vox, sv, off, acc, angles = ORACLE_CASES[name]
    sc = _scanner(mode, det, vox, sv, off, acc)
    lhs, rhs = _dot_gap(sc, angles, _rand(vox, 1, 0.1), _rand((len(angles), *det), 2, 0.1))
    print(f"dot {name}: relative gap {abs(lhs - rhs) / lhs:.3g}")
    assert abs(lhs - rhs) <= 1e-5 * lhs, (lhs, rhs)


def test_dot_product_256_cubed_50_views():
    """256^3 grid, 50 cone views of 512^2 (two chunks of views): a footprint that misses rays fails here."""
    sc = fc.scanner("cone", 512, 256)
    angles = fc.full_scan(50)
    lhs, rhs = _dot_gap(sc, angles, _rand((256, 256, 256), 3, 0.1), _rand((50, 512, 512), 4, 0.1))
    print(f"dot 256^3 x 50 x 512^2: relative gap {abs(lhs - rhs) / lhs:.3g}")
    assert abs(lhs - rhs) <= 1e-5 * lhs, (lhs, rhs)


def test_weight_output_and_determinism():
    """40 views (more than one chunk): out_weight is bitwise backproject(ones), and two runs are bitwise equal."""
    torch = _torch()
    from r2_gaussian_b200.projector import backproject

    for mode in ("cone", "parallel"):
        sc = dict(fc.scanner(mode, 64, 40), accuracy=0.5)
        angles = fc.full_scan(40)
        y = torch.rand(40, 64, 64, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
        a, w = backproject(y, angles, sc, weights=True)
        b = backproject(y, angles, sc)
        ones = backproject(torch.ones_like(y), angles, sc)
        assert a.view(torch.int32).equal(b.view(torch.int32))
        assert w.view(torch.int32).equal(ones.view(torch.int32))
        assert float(w.min()) > 0.0                                    # every voxel of this grid is seen


def _tiny_case():
    sc = fc.scanner("cone", 16, 8)
    sc["nDetector"] = [16, 20]
    angles = [0.0, math.pi / 2, 1.1, 2.5, 3.9, 5.2]
    truth = _rand((8, 8, 8), 5)
    from oracle import projector_oracle as po

    b = po.project_scene(truth, angles, sc)
    return sc, angles, b


def test_solvers_match_the_oracle_solvers():
    torch = _torch()
    from r2_gaussian_b200 import recon

    sc, angles, b = _tiny_case()
    A, At = bo.operators(angles, sc)
    bt = torch.tensor(b, dtype=torch.float32, device="cuda")
    runs = {
        "cgls": (lambda: recon.cgls(bt, angles, sc, 3)[0],
                 lambda: recon.cgls_solve(torch.from_numpy(b), A, At, 3)[0]),
        "sart": (lambda: recon.sart(bt, angles, sc, 3),
                 lambda: recon.sart_solve(torch.from_numpy(b), A, At, sc["nVoxel"], 3)),
        "ossart": (lambda: recon.sart(bt, angles, sc, 3, blocksize=4),
                   lambda: recon.sart_solve(torch.from_numpy(b), A, At, sc["nVoxel"], 3, blocksize=4)),
    }
    for name, (gpu, cpu) in runs.items():
        got, again = gpu(), gpu()
        assert got.view(torch.int32).equal(again.view(torch.int32)), name          # bitwise reproducible
        want = cpu().numpy()
        err = np.abs(got.cpu().numpy().astype(np.float64) - want).max() / np.abs(want).max()
        print(f"solver {name}: max err / max = {err:.3g}")
        assert err <= SOLVER_BOUND, (name, err)


# ---- a generate_data scene ------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def clean_scene(tmp_path_factory):
    """The noise-free scene of test_generate_data_end_to_end: 24 train and 6 test views of 96^2, 48^3 grid."""
    from r2_gaussian_b200 import generate_data

    tmp = tmp_path_factory.mktemp("recon_scene")
    yml, vol_path, *_ = _write_inputs(tmp, noise=False)
    return generate_data.main(["--vol", str(vol_path), "--scanner", str(yml), "--n_train", "24", "--n_test", "6",
                               "--output", str(tmp / "data")])


def test_iterative_beats_fdk_at_sparse_views(clean_scene):
    torch = _torch()
    from r2_gaussian_b200 import recon
    from r2_gaussian_b200.dataset import read_blender
    from r2_gaussian_b200.metrics import metric_vol
    from r2_gaussian_b200.projector import project

    info = read_blender(clean_scene, eval=False)
    cfg = info.scanner_cfg
    b = torch.tensor(np.stack([c.image for c in info.train_cameras]), dtype=torch.float32, device="cuda")
    angles = [c.angle for c in info.train_cameras]
    x_cgls, l2 = recon.cgls(b, angles, cfg)
    vols = {"fdk": recon.recon_volume(b, angles, cfg, "fdk"), "sart": recon.recon_volume(b, angles, cfg, "sart"),
            "ossart": recon.recon_volume(b, angles, cfg, "ossart"), "cgls": x_cgls}
    res = {m: float(torch.linalg.vector_norm(project(v, angles, cfg) - b) / torch.linalg.vector_norm(b))
           for m, v in vols.items()}
    psnr = {m: metric_vol(info.vol, v.cpu().numpy(), "psnr")[0] for m, v in vols.items()}
    print(f"residual {res}\npsnr {psnr}\ncgls l2 first {l2[0]:.4g} last {l2[-1]:.4g}")
    assert len(l2) == recon.CGLS_NITER and l2[-1] < 0.5 * l2[0]
    for m in ("sart", "ossart", "cgls"):
        assert res[m] < res["fdk"], (m, res)
        assert psnr[m] > psnr["fdk"], (m, psnr)


def test_cli_end_to_end(clean_scene, tmp_path, capsys):
    from r2_gaussian_b200 import initialize_pcd, recon
    from r2_gaussian_b200.metrics import metric_vol

    out = tmp_path / "trad"
    report = recon.main(["-s", clean_scene, "-m", str(out), "--methods", "fdk,sart,cgls"])
    with open(out / "eval_3d.yml") as f:
        top = yaml.safe_load(f)
    assert list(top) == ["fdk", "sart", "cgls"]
    keys = ["method", "psnr_3d", "ssim_3d", "ssim_3d_x", "ssim_3d_y", "ssim_3d_z", "duration (sec)", "duration (min)"]
    vol_gt = np.load(os.path.join(clean_scene, "vol_gt.npy"))
    for m in ("fdk", "sart", "cgls"):
        with open(out / m / "eval_3d.yml") as f:
            per = yaml.safe_load(f)
        assert list(per) == keys and per == top[m] and per["method"] == m
        assert np.array_equal(np.load(out / m / "ct_gt.npy"), vol_gt)
        pred = np.load(out / m / "ct_pred.npy")
        assert pred.shape == vol_gt.shape and pred.dtype == np.float32
        assert per["psnr_3d"] == metric_vol(vol_gt, pred, "psnr")[0]
        assert math.isfinite(per["ssim_3d"]) and per["duration (sec)"] >= 0.0
        names = sorted(os.listdir(out / m / "projs"))
        assert names == sorted([f"{i:05d}_render.npy" for i in range(6)] + [f"{i:05d}_gt.npy" for i in range(6)])
        assert np.load(out / m / "projs" / "00000_render.npy").shape == (96, 96)
        print(f"cli {m}: psnr {per['psnr_3d']:.3f} ssim {per['ssim_3d']:.4f}")
    assert report["cgls"]["psnr_3d"] == top["cgls"]["psnr_3d"]

    capsys.readouterr()
    init = initialize_pcd.main(["--data", clean_scene, "--recon_method", "cgls", "--n_points", "400",
                                "--output", str(tmp_path / "init_cgls.npy"), "--evaluate"])
    assert os.path.exists(init)
    psnr = re.findall(r"3D PSNR for initial Gaussians: (\S+)", capsys.readouterr().out)
    assert len(psnr) == 1 and math.isfinite(float(psnr[0])), psnr
