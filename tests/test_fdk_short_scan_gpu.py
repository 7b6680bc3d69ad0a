"""Short-scan FDK on the GPU (fdk(short_scan=True) over r2x_fdk with R2X_FDK_PARKER) against the float64 oracle,
bitwise reproducibility, the 180-degree parallel case, the render -> fdk -> query round trip at 220 degrees, and
`initialize_pcd --recon_method fdk --short_scan --evaluate` on a generate_data scene."""
import json
import math
import re
import types

import numpy as np
import pytest

import fdk_cases as fc
import fdk_short_scan_oracle as sso
from r2_gaussian_b200 import scene
from test_fdk_short_scan_cpu import PARKER_BOUND, PLAIN_FLOOR, SHORT_ARC, SHORT_VIEWS, arc_angles

pytestmark = pytest.mark.gpu

# 3D PSNR that the Parker-weighted initial cloud of the end-to-end scene must gain over the unweighted one, in dB.
# Fixed from the oracle before any GPU run: on that scene the FDK volume itself gains 6.6 dB (41.1 against 34.5).
INIT_PSNR_MARGIN = 0.25


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
    # cone beam, H != W, non-cubic off-centre grid, unevenly spaced angles over 230 degrees starting at 100
    "cone_uneven": ("cone", (24, 40), (20, 28, 12), (1.6, 1.8, 1.2), (0.1, -0.2, 0.15), 9, 230.0, 100.0),
    # parallel beam, H != W, non-cubic off-centre grid, uneven angles over 190 degrees crossing 360
    "parallel_uneven": ("parallel", (20, 36), (18, 10, 26), (1.4, 1.0, 1.8), (-0.15, 0.1, 0.05), 7, 190.0, 300.0),
    # more views than one shared-memory chunk of the backprojection kernel, z not a multiple of its run length
    "cone_many_views": ("cone", (16, 16), (9, 11, 13), (2.0, 2.0, 2.0), (0.05, 0.0, -0.1), 70, 250.0, 0.0),
}


def _uneven(n, deg, start_deg, seed):
    rng = np.random.RandomState(seed)
    a = np.concatenate([[0.0, 1.0], rng.uniform(0.0, 1.0, n - 2)]) * math.radians(deg)
    return rng.permutation(a) + math.radians(start_deg)


@pytest.mark.parametrize("name", sorted(ORACLE_CASES))
def test_cuda_matches_oracle(name):
    torch = _torch()
    from r2_gaussian_b200.fdk import fdk

    mode, det, vox, sv, off, n, deg, start = ORACLE_CASES[name]
    sc = _scanner(mode, det, vox, sv, off)
    angles = _uneven(n, deg, start, len(name))
    projs = np.random.RandomState(len(name)).uniform(0.0, 1.0, size=(n, *det)).astype(np.float32)
    got = fdk(torch.tensor(projs, device="cuda"), angles, sc, short_scan=True).cpu().numpy()
    want = sso.fdk_short_scan_scene(projs, angles, sc)
    assert got.shape == tuple(vox)
    err = np.abs(got.astype(np.float64) - want).max()
    assert err <= 1e-4 * np.abs(want).max(), (err, np.abs(want).max())


def test_deterministic_and_plain_path_unchanged():
    torch = _torch()
    from r2_gaussian_b200.fdk import fdk

    sc = fc.scanner("cone", 64, 40)
    angles = arc_angles(220.0, 30)
    projs = torch.rand(30, 64, 64, device="cuda", generator=torch.Generator("cuda").manual_seed(0))
    a, b = fdk(projs, angles, sc, short_scan=True), fdk(projs, angles, sc, short_scan=True)
    assert a.view(torch.int32).equal(b.view(torch.int32))           # bitwise, signed zeros included
    plain = fdk(projs, angles, sc)
    assert fdk(projs, angles, sc, short_scan=False).view(torch.int32).equal(plain.view(torch.int32))
    assert not a.equal(plain)
    with pytest.raises(ValueError, match="full circle"):
        fdk(projs, fc.full_scan(30), sc, short_scan=True)


def test_parallel_180_matches_plain_fdk():
    torch = _torch()
    from r2_gaussian_b200.fdk import fdk

    sc = fc.scanner("parallel", 48, 32)
    angles = arc_angles(180.0, 40, 0.7)
    projs = torch.rand(40, 48, 48, device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    got, want = fdk(projs, angles, sc, short_scan=True), fdk(projs, angles, sc)
    assert float((got - want).abs().max()) <= 1e-5 * float(want.abs().max())


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


def test_round_trip_render_fdk_query_220_cone():
    """fdk(render(cloud), short_scan=True) against query(cloud), with the CPU round trip's views and bounds."""
    torch = _torch()
    from r2_gaussian_b200.fdk import fdk
    from r2_gaussian_b200.render_query import query

    sc = fc.scanner("cone", fc.ROUND_TRIP_DET, fc.ROUND_TRIP_VOX)
    angles = arc_angles(SHORT_ARC, SHORT_VIEWS, 0.3)
    projs, pc, pipe = _render_views(fc.round_trip_cloud(), sc, angles)
    with torch.no_grad():
        want = query(pc, sc["offOrigin"], sc["nVoxel"], sc["sVoxel"], pipe)["vol"].cpu().numpy()
    err = fc.rel_l2(fdk(projs, angles, sc, short_scan=True).cpu().numpy(), want)
    plain = fc.rel_l2(fdk(projs, angles, sc).cpu().numpy(), want)
    print(f"220-degree round trip: short scan {err:.4f}, plain {plain:.4f}")
    assert err <= PARKER_BOUND, err
    assert plain >= PLAIN_FLOOR, plain


def _short_scan_scene(tmp_path):
    """generate_data at 220 degrees (24 train, 6 test views of 96^2, 48^3 grid, no noise) of the round-trip cloud, from
    a scanner yml in physical units (scene scale 0.5)."""
    torch = _torch()
    from r2_gaussian_b200 import generate_data
    from r2_gaussian_b200.render_query import query

    sc = scene.cone_beam_scanner(96, 48)
    phys = {k: (np.asarray(v, float) * 2.0).tolist() if k in ("DSD", "DSO", "sDetector", "sVoxel", "offOrigin",
                                                              "offDetector") else v for k, v in sc.items()}
    phys.update({"filter": None, "accuracy": 0.5, "totalAngle": SHORT_ARC, "startAngle": 30.0, "noise": False})
    yml = tmp_path / "short.yml"
    yml.write_text("".join(f"{k}: {json.dumps(v)}\n" for k, v in phys.items()))
    _, pc, pipe = _render_views(fc.round_trip_cloud(), sc, [0.0])
    with torch.no_grad():
        vol = query(pc, sc["offOrigin"], sc["nVoxel"], sc["sVoxel"], pipe)["vol"].cpu().numpy()
    np.save(tmp_path / "vol.npy", vol)
    return generate_data.main(["--vol", str(tmp_path / "vol.npy"), "--scanner", str(yml), "--n_train", "24",
                               "--n_test", "6", "--output", str(tmp_path / "data")])


def test_initialize_pcd_and_recon_short_scan_end_to_end(tmp_path, capsys):
    import yaml

    from r2_gaussian_b200 import initialize_pcd, recon

    case = _short_scan_scene(tmp_path)
    psnr = {}
    for flag in ([], ["--short_scan"]):
        capsys.readouterr()
        initialize_pcd.main(["--data", case, "--recon_method", "fdk", "--n_points", "2000", "--evaluate", "--output",
                             str(tmp_path / f"init{len(flag)}.npy"), *flag])
        found = re.findall(r"3D PSNR for initial Gaussians: (\S+)", capsys.readouterr().out)
        assert len(found) == 1
        psnr[bool(flag)] = float(found[0])
    print(f"initial-cloud 3D PSNR: short scan {psnr[True]:.3f}, plain {psnr[False]:.3f}")
    assert psnr[True] >= psnr[False] + INIT_PSNR_MARGIN, psnr

    out = tmp_path / "trad"
    report = recon.main(["-s", case, "-m", str(out), "--methods", "fdk,sart", "--short_scan"])
    with open(out / "fdk" / "eval_3d.yml") as f:
        per = yaml.safe_load(f)
    assert per["short_scan"] is True and per == report["fdk"]
    with open(out / "sart" / "eval_3d.yml") as f:
        assert "short_scan" not in yaml.safe_load(f)
    plain = recon.main(["-s", case, "-m", str(tmp_path / "plain"), "--methods", "fdk"])
    assert "short_scan" not in plain["fdk"]
    print(f"recon fdk psnr_3d: short scan {per['psnr_3d']:.3f}, plain {plain['fdk']['psnr_3d']:.3f}")
    assert per["psnr_3d"] > plain["fdk"]["psnr_3d"]
