"""Helical FDK on the GPU (r2x_fdk_helical through fdk.fdk(helical=True)): within 1e-5 of max of the float64 oracle
(tests/fdk_helical_oracle.py) at odd shapes around the 32 x 4 x 8 backprojection CTA, in both helix directions, with
Ram-Lak and a window, and on a long thin helix whose voxels sit at the edges of the CTAs' view windows; the plain FDK
within 1e-6 of max on a circle at Q = 1; bitwise reproducible; the launch limits; then the helical scene of
test_view_geometry_gpu.py through recon and initialize_pcd + training.  The end-to-end scores are printed and recorded
in DESIGN §8."""
import json
import math
import os

import numpy as np
import pytest

import fdk_helical_oracle as fho

pytestmark = pytest.mark.gpu

ORACLE_BOUND = 1e-5
ANCHOR_BOUND = 1e-6


def _torch():
    import torch

    return torch


def _bits(t):
    return t.contiguous().view(_torch().int32)


def _run(projs, angles, sc, geo, q, name=None):
    from r2_gaussian_b200.fdk import fdk
    return fdk(_torch().from_numpy(projs).cuda(), angles, sc, view_geometry=geo, helical=True, helical_q=q,
               filter=name)


def _check(got, want):
    err = float(np.abs(got.cpu().numpy().astype(np.float64) - want).max())
    assert err <= ORACLE_BOUND * np.abs(want).max(), (err, np.abs(want).max())
    return err


@pytest.mark.parametrize("q", [0.0, 0.5])
@pytest.mark.parametrize("travel,name", [(1.3, "ram_lak"), (-1.1, "hann"), (0.9, "shepp_logan")])
def test_against_the_oracle_at_odd_shapes(q, travel, name):
    sc, angles, geo = fho.helix_case(53, 2.3, travel, nvox=(9, 35, 21), ndet=(11, 17), svox=(1.0, 1.1, 2.2),
                                     sdet=(1.1, 2.6))
    projs = np.random.RandomState(4).uniform(0.0, 1.0, (53, 11, 17)).astype(np.float32)
    got = _run(projs, angles, sc, geo, q, name)
    _check(got, fho.fdk_helical_scene(projs, angles, sc, geo, q, name))
    # shuffled frames give the same volume bit for bit (the views are reconstructed in beta order)
    perm = np.random.RandomState(5).permutation(53)
    again = _run(projs[perm], angles[perm], sc, [geo[i] for i in perm], q, name)
    assert _bits(got).equal(_bits(again))


@pytest.mark.parametrize("q", [0.0, 0.5])
def test_long_thin_helix(q):
    # 20 turns, each CTA's z-run sees about one turn of views: voxels at the edges of the view windows everywhere
    sc, angles, geo = fho.helix_case(600, 20.0, 7.2, nvox=(16, 16, 256), ndet=(8, 16), svox=(1.0, 1.0, 8.0),
                                     sdet=(0.56, 2.0), off=(0.02, -0.03, 0.0))
    projs = np.random.RandomState(6).uniform(0.0, 1.0, (600, 8, 16)).astype(np.float32)
    got = _run(projs, angles, sc, geo, q)
    _check(got, fho.fdk_helical_scene(projs, angles, sc, geo, q))
    assert _bits(got).equal(_bits(_run(projs, angles, sc, geo, q)))


def test_circle_at_q1_is_the_plain_fdk():
    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.fdk import fdk, helix_views
    torch = _torch()
    N = 48
    sc, angles, geo = fho.helix_case(N, 1.0, 0.0, nvox=(33, 37, 27), ndet=(41, 45), svox=(1.0, 1.0, 0.8),
                                     sdet=(2.4, 2.6))
    projs = torch.from_numpy(np.random.RandomState(7).uniform(0.0, 1.0, (N, 41, 45)).astype(np.float32)).cuda()
    got = fdk(projs, angles, sc, view_geometry=geo, helical=True, helical_q=1.0).cpu().numpy()
    want = fdk(projs, angles, sc, view_geometry=geo).cpu().numpy()
    # the slab where both conjugate rays of every view hit the detector well inside its edges
    hx = helix_views(angles, sc, geo)
    tany = float(scene.make_view(sc, 0.0).tanfovy)
    xs, ys, zs = fho.fdk_oracle.voxel_centres(sc["nVoxel"], sc["sVoxel"], sc["offOrigin"])
    X, Y, Z = np.meshgrid(xs, ys, zs, indexing="ij")
    inside = np.ones(X.shape, bool)
    for b in hx.beta:
        zin, _, zc = fho.conjugate_geometry(float(b), X, Y, float(sc["DSO"]), hx.c_x, hx.c_y)
        inside &= (np.abs(Z - hx.z0) < 0.9 * zin * tany) & (np.abs(Z - hx.z0) < 0.9 * zc * tany)
    assert inside.mean() > 0.3
    err = np.abs(got - want)[inside].max()
    assert err <= ANCHOR_BOUND * np.abs(want).max(), (err, np.abs(want).max())


def _abi(N, H, W, nz, beta, helix=None, q=0.5):
    torch = _torch()
    from r2_gaussian_b200 import _lib, scene
    lib = _lib.load()
    sc = scene.cone_beam_scanner(1, 1)
    vs = [scene.make_view(dict(sc, nDetector=[H, W]), float(b)) for b in beta]
    vm = torch.from_numpy(np.stack([v.viewmatrix.reshape(16) for v in vs])).cuda()
    pm = torch.from_numpy(np.stack([v.projmatrix.reshape(16) for v in vs])).cuda()
    projs = torch.ones((N, H, W), device="cuda")
    vol = torch.empty((1, 1, nz), device="cuda")
    nbytes = int(lib.r2x_fdk_scratch_bytes(N, H, W))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    bh = np.ascontiguousarray(beta, np.float64)
    bd = torch.from_numpy(bh).cuda()
    dbd = torch.full((N,), 2.0 * math.pi / N, dtype=torch.float64, device="cuda")
    step = 2.0 * math.pi / N
    helix = helix or (0.0, 0.0, float(bh[0]) - 0.5 * step, float(bh[-1]) + 0.5 * step, 0.0, 0.0)
    rc = lib.r2x_fdk_helical(torch.cuda.current_stream().cuda_stream, N, H, W, projs.data_ptr(), vm.data_ptr(),
                             pm.data_ptr(), float(vs[0].tanfovx), float(vs[0].tanfovy), 1, 0, 5.0, bd.data_ptr(),
                             dbd.data_ptr(), bh.ctypes.data, *helix, q, 1, 1, nz, 0.01, 0.01, 2.0, 0.0, 0.0, 0.0,
                             vol.data_ptr(), scratch.data_ptr(), nbytes)
    torch.cuda.synchronize()
    return rc, vol, lib


def test_launch_limits():
    beta = np.linspace(0.0, 2.0 * math.pi, 5)[:-1]
    rc, vol, lib = _abi(4, 1, 16384, 8, beta)
    assert rc == 0 and bool(_torch().isfinite(vol).all())
    rc, _, lib = _abi(4, 1, 16385, 8, beta)
    assert rc != 0 and "bad W" in lib.r2x_last_error().decode()
    rc, vol, lib = _abi(4, 4, 8, 524280, beta)
    assert rc == 0 and bool(_torch().isfinite(vol).all())
    rc, _, lib = _abi(4, 4, 8, 524281, beta)
    assert rc != 0 and "bad grid" in lib.r2x_last_error().decode()


# ---- end to end through the CLIs on the helical scene of test_view_geometry_gpu.py -------------------------------------

RESULTS = {}


def _record(key, value):
    RESULTS[key] = value
    out = os.environ.get("FDK_HELICAL_RESULTS")
    print(f"[fdk_helical] {key} = {value:.3f}")
    if out:
        with open(out, "w") as f:
            json.dump(RESULTS, f, indent=1, sort_keys=True)


@pytest.fixture(scope="module")
def helical_scene(tmp_path_factory):
    from test_view_geometry_gpu import _tall_phantom, _yml

    from r2_gaussian_b200 import generate_data
    tmp = tmp_path_factory.mktemp("helical")
    np.save(tmp / "vol.npy", _tall_phantom())
    return generate_data.main(["--vol", str(tmp / "vol.npy"), "--scanner", str(_yml(tmp / "h.yml")), "--n_train",
                               "120", "--n_test", "8", "--helical_travel", "3.2", "--output", str(tmp / "data")]), tmp


def _recon(src, out, flags):
    from r2_gaussian_b200 import recon
    return recon.main(["-s", src, "-m", str(out), "--methods", "fdk"] + flags)["fdk"]


# margins from the first H100 run with slack (DESIGN §8: FDK 27.70 dB with --helical at Q = 0.75 against 16.74 without
# the flags; the FDK-initialised training 28.90)
HELICAL_FDK_GAIN = 10.0      # dB above the flagless FDK at least
HELICAL_TRAIN_FLOOR = 26.0   # dB psnr_3d of the FDK-initialised training at least


def test_helical_scene_recon_and_q_table(helical_scene):
    src, tmp = helical_scene
    flagless = _recon(src, tmp / "plain", [])["psnr_3d"]
    _record("helical_fdk_without", flagless)
    reports = {}
    for q in (0.0, 0.25, 0.5, 0.75, 1.0):
        reports[q] = _recon(src, tmp / f"q{q}", ["--use_view_geometry", "--helical", "--helical_q", str(q)])
        _record(f"helical_fdk_q{q:.2f}", reports[q]["psnr_3d"])
    default = _recon(src, tmp / "default", ["--use_view_geometry", "--helical"])
    assert default["helical"] is True
    from r2_gaussian_b200.fdk import HELICAL_Q
    assert default["helical_q"] == HELICAL_Q
    _record("helical_fdk_with", default["psnr_3d"])
    assert default["psnr_3d"] >= flagless + HELICAL_FDK_GAIN, (default["psnr_3d"], flagless)


def test_helical_scene_fdk_initialised_training(helical_scene):
    import random

    import yaml
    torch = _torch()
    from r2_gaussian_b200 import initialize_pcd, test, trainer
    src, tmp = helical_scene
    init = initialize_pcd.main(["--data", src, "--recon_method", "fdk", "--use_view_geometry", "--helical",
                                "--n_points", "4000", "--output", str(tmp / "init_fdk.npy")])
    model = tmp / "model_fdk"
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    trainer.main(["-s", src, "-m", str(model), "--ply_path", init, "--iterations", "1500", "--test_iterations",
                  "1500", "--save_iterations", "1500", "--use_view_geometry"])
    test.main(["-m", str(model), "--skip_render_train", "--skip_render_test"])
    with open(model / "test" / "iter_1500" / "eval3d.yml") as f:
        psnr = float(yaml.safe_load(f)["psnr_3d"])
    _record("helical_train_fdk_init", psnr)
    assert psnr >= HELICAL_TRAIN_FLOOR, psnr
