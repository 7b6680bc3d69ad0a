"""FDK on the GPU (r2_gaussian_b200.fdk over r2x_fdk) against the float64 oracle, through the product path
(render -> fdk vs query), and end to end through `initialize_pcd --recon_method fdk --evaluate`."""
import math
import os
import re
import types

import numpy as np
import pytest

import fdk_cases as fc
from oracle import fdk_oracle
from r2_gaussian_b200 import scene

pytestmark = pytest.mark.gpu


def _torch():
    import torch

    return torch


def _scanner(mode, det_hw, vox, s_voxel, off, s_det=(3.0, 4.0)):
    sc = fc.scanner(mode, 8, 8)
    sc["nDetector"] = list(det_hw)
    if mode == "cone":
        sc["sDetector"] = list(s_det)
    sc["nVoxel"], sc["sVoxel"], sc["offOrigin"] = list(vox), list(s_voxel), list(off)
    return sc


ORACLE_CASES = {
    # cone beam, H != W, non-cubic off-centre grid, unevenly spaced angles
    "cone_uneven": ("cone", (24, 40), (20, 28, 12), (1.6, 1.8, 1.2), (0.1, -0.2, 0.15), 9),
    # parallel beam, H != W, non-cubic off-centre grid, unevenly spaced angles
    "parallel_uneven": ("parallel", (20, 36), (18, 10, 26), (1.4, 1.0, 1.8), (-0.15, 0.1, 0.05), 7),
    # a single view
    "cone_one_view": ("cone", (32, 24), (16, 16, 16), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0), 1),
    # more views than one shared-memory chunk of the backprojection kernel, z not a multiple of its run length
    "cone_many_views": ("cone", (16, 16), (9, 11, 13), (2.0, 2.0, 2.0), (0.05, 0.0, -0.1), 70),
}


@pytest.mark.parametrize("name", sorted(ORACLE_CASES))
def test_cuda_matches_oracle(name):
    torch = _torch()
    from r2_gaussian_b200.fdk import fdk

    mode, det, vox, sv, off, n = ORACLE_CASES[name]
    sc = _scanner(mode, det, vox, sv, off)
    rng = np.random.RandomState(len(name))
    angles = np.sort(rng.uniform(0.0, 2.0 * math.pi, n))
    projs = rng.uniform(0.0, 1.0, size=(n, *det)).astype(np.float32)
    got = fdk(torch.tensor(projs, device="cuda"), angles, sc).cpu().numpy()
    want = fdk_oracle.fdk_scene(projs, angles, sc)
    assert got.shape == tuple(vox)
    err = np.abs(got.astype(np.float64) - want).max()
    assert err <= 1e-4 * np.abs(want).max(), (err, np.abs(want).max())


def _render_views(cloud, sc, angles):
    torch = _torch()
    from r2_gaussian_b200.render_query import render

    t = {k: torch.tensor(v, device="cuda") for k, v in
         (("xyz", cloud.means), ("dens", cloud.density), ("s", cloud.scales), ("r", cloud.rotations))}
    pc = types.SimpleNamespace(get_xyz=t["xyz"], get_density=t["dens"], get_scaling=t["s"], get_rotation=t["r"])
    pipe = types.SimpleNamespace(debug=False, compute_cov3D_python=False)
    with torch.no_grad():
        imgs = [render(scene.camera_from_view(scene.make_view(sc, float(a))), pc, pipe)["render"][0] for a in angles]
    return torch.stack(imgs), pc, pipe


@pytest.mark.parametrize("mode,n_views", sorted(fc.ROUND_TRIP_BOUNDS))
def test_round_trip_render_fdk_query(mode, n_views):
    """fdk(render(cloud)) against query(cloud), with the cloud, sizes and bounds of the CPU round trip."""
    torch = _torch()
    from r2_gaussian_b200.fdk import fdk
    from r2_gaussian_b200.render_query import query

    cloud = fc.round_trip_cloud()
    sc = fc.scanner(mode, fc.ROUND_TRIP_DET, fc.ROUND_TRIP_VOX)
    angles = fc.full_scan(n_views)
    projs, pc, pipe = _render_views(cloud, sc, angles)
    got = fdk(projs, angles, sc).cpu().numpy()
    with torch.no_grad():
        want = query(pc, sc["offOrigin"], sc["nVoxel"], sc["sVoxel"], pipe)["vol"].cpu().numpy()
    err = fc.rel_l2(got, want)
    assert err <= fc.ROUND_TRIP_BOUNDS[(mode, n_views)], err
    assert fc.rel_l2(got[::-1], want) >= 0.5
    assert fc.rel_l2(got[:, :, ::-1], want) >= 0.5


def test_deterministic_and_argument_errors():
    torch = _torch()
    from r2_gaussian_b200.fdk import fdk

    sc = fc.scanner("cone", 64, 40)
    angles = fc.full_scan(30)
    g = torch.Generator("cuda").manual_seed(0)
    projs = torch.rand(30, 64, 64, device="cuda", generator=g)
    a, b = fdk(projs, angles, sc), fdk(projs, angles, sc)
    assert torch.equal(a, b)
    assert a.view(torch.int32).equal(b.view(torch.int32))           # bitwise, signed zeros included
    with pytest.raises(RuntimeError, match="CUDA"):
        fdk(projs.cpu(), angles, sc)
    with pytest.raises(ValueError, match="filter"):
        fdk(projs, angles, dict(sc, filter="shepp_logan"))
    with pytest.raises(ValueError, match="angles"):
        fdk(projs, angles[:-1], sc)
    assert fdk(projs, angles, dict(sc, filter="ram_lak")).equal(a)


def test_fdk_512_cubed_grid():
    """512^3 output (2^27 voxels, 512 MiB): the last voxels are written and agree with the oracle."""
    torch = _torch()
    from r2_gaussian_b200.fdk import fdk

    sc = fc.scanner("cone", 32, 512)
    angles = fc.full_scan(4)
    projs = torch.rand(4, 32, 32, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    vol = fdk(projs, angles, sc)
    small = dict(sc, nVoxel=[2, 2, 2], sVoxel=[2.0 * 2 / 512] * 3, offOrigin=[1.0 - 2.0 / 512] * 3)
    want = fdk_oracle.fdk_scene(projs.cpu().numpy(), angles, small)     # the 2^3 corner block at +x, +y, +z
    got = vol[510:, 510:, 510:].cpu().numpy()
    assert np.abs(got - want).max() <= 1e-4 * max(np.abs(want).max(), 1e-3)
    del vol
    torch.cuda.empty_cache()


def _write_case(tmp_path, n_views=60):
    torch = _torch()
    from r2_gaussian_b200 import dataset
    from r2_gaussian_b200.render_query import query

    cloud = fc.round_trip_cloud()
    sc = fc.scanner("cone", 64, 32)           # sVoxel 2: scene scale 1, so rendered projections are stored as they are
    sc.update({"accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0, "filter": None})
    angles = fc.full_scan(n_views)
    projs, pc, pipe = _render_views(cloud, sc, angles)
    with torch.no_grad():
        vol = query(pc, sc["offOrigin"], sc["nVoxel"], sc["sVoxel"], pipe)["vol"].cpu().numpy()
    case = tmp_path / "fdk_case"
    frames = list(zip(angles, projs.cpu().numpy()))
    dataset.write_blender(str(case), sc, frames, frames[:2], vol)
    return case, sc, angles, projs


def test_initialize_pcd_fdk_end_to_end(tmp_path, capsys):
    from r2_gaussian_b200 import initialize_pcd
    from r2_gaussian_b200.fdk import fdk

    case, sc, angles, projs = _write_case(tmp_path)
    n = 600
    out = initialize_pcd.main(["--data", str(case), "--recon_method", "fdk", "--n_points", str(n), "--evaluate"])
    assert out == str(case / "init_fdk_case.npy")
    pts = np.load(out)
    assert pts.shape == (n, 4)
    lo, hi = np.asarray(sc["offOrigin"]) - 1.0, np.asarray(sc["offOrigin"]) + 1.0
    assert (pts[:, :3] >= lo).all() and (pts[:, :3] <= hi).all()
    vol = fdk(projs, angles, sc).cpu().numpy()
    d = np.asarray(sc["dVoxel"])
    idx = np.rint((pts[:, :3] - lo) / d).astype(int)
    assert np.allclose(idx * d + lo, pts[:, :3], atol=1e-9)
    assert (vol[idx[:, 0], idx[:, 1], idx[:, 2]] > 0.05).all()
    assert np.array_equal(pts[:, 3], vol[idx[:, 0], idx[:, 1], idx[:, 2]] * 0.15)
    assert len({tuple(i) for i in idx}) == n                          # sampled without replacement
    psnr = re.findall(r"3D PSNR for initial Gaussians: (\S+)", capsys.readouterr().out)
    assert len(psnr) == 1 and math.isfinite(float(psnr[0])), psnr
    out2 = initialize_pcd.main(["--data", str(case), "--recon_method", "fdk", "--n_points", str(n), "--output",
                                str(tmp_path / "again.npy")])
    with open(out, "rb") as f1, open(out2, "rb") as f2:
        assert f1.read() == f2.read()


def test_initialize_pcd_fdk_refuses_too_few_views(tmp_path):
    from r2_gaussian_b200 import initialize_pcd

    case, *_ = _write_case(tmp_path, n_views=initialize_pcd.MIN_FDK_VIEWS - 1)
    with pytest.raises(SystemExit, match="train views"):
        initialize_pcd.main(["--data", str(case), "--recon_method", "fdk", "--n_points", "10"])
    assert not os.path.exists(case / "init_fdk_case.npy")
