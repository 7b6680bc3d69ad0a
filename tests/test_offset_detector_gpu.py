"""The scanner's detector offset (offDetector) on the GPU: the offset projector, backprojector, FDK and half-fan FDK
against the float64 oracle (tests/offset_detector_oracle.py) at a fractional (t_u, t_v); consistency with render() of
offset cameras; the integer-shift identities; the half-fan weights on a quarter-width offset; and generate_data ->
initialize_pcd -> trainer end to end with `--use_offDetector`."""
import json
import math
import os
import random

import numpy as np
import pytest

import fdk_cases as fc
import offset_detector_oracle as oo
import projector_cases as pc
from test_projector_gpu import FDK_ROUND_TRIP_BOUND, ORACLE_CASES, _cloud_tensors, _query, _scanner
from r2_gaussian_b200 import scene

pytestmark = pytest.mark.gpu

SHIFT = (2.4, -1.7)          # (t_u, t_v) in pixels
# half-fan FDK against unweighted offset FDK on a quarter-width offset over 360 degrees (psnr_3d, dB)
HALF_FAN_GAIN_DB = 3.0
# half-fan FDK against FDK of the centred detector on the same scene
HALF_FAN_LOSS_DB = 3.0


def _torch():
    import torch

    return torch


def _offset(sc, t_u, t_v):
    du = sc["sDetector"][1] / sc["nDetector"][1]
    dv = sc["sDetector"][0] / sc["nDetector"][0]
    return dict(sc, offDetector=[t_u * du, t_v * dv])


@pytest.mark.parametrize("name", ["cone_acc05", "parallel_acc05", "cone_acc1"])
def test_offset_projector_matches_oracle(name):
    torch = _torch()
    from r2_gaussian_b200.projector import project

    mode, det, vox, sv, off, acc, angles = ORACLE_CASES[name]
    sc = _offset(_scanner(mode, det, vox, sv, off, acc), *SHIFT)
    vol = np.random.RandomState(len(name)).uniform(0.0, 1.0, size=vox).astype(np.float32)
    got = project(torch.tensor(vol, device="cuda"), angles, sc, use_offDetector=True).cpu().numpy()
    want = oo.project_scene(vol, angles, sc)
    err = np.abs(got.astype(np.float64) - want).max()
    print(f"project {name}: max err / max = {err / np.abs(want).max():.3g}")
    assert err <= 1e-5 * np.abs(want).max(), (err, np.abs(want).max())
    assert (got[want == 0.0] == 0.0).all()


@pytest.mark.parametrize("name", ["cone_acc05", "parallel_acc05"])
def test_offset_backprojector_matches_oracle_and_is_the_adjoint(name):
    torch = _torch()
    from r2_gaussian_b200.projector import CTOperator, backproject, project

    mode, det, vox, sv, off, acc, angles = ORACLE_CASES[name]
    sc = _offset(_scanner(mode, det, vox, sv, off, acc), *SHIFT)
    rng = np.random.RandomState(2)
    y = rng.uniform(0.1, 1.0, (len(angles), *det)).astype(np.float32)
    x = rng.uniform(0.1, 1.0, vox).astype(np.float32)
    got = backproject(torch.tensor(y, device="cuda"), angles, sc, use_offDetector=True).cpu().numpy()
    want = oo.backproject_scene(y, angles, sc)
    err = np.abs(got.astype(np.float64) - want).max()
    print(f"backproject {name}: max err / max = {err / np.abs(want).max():.3g}")
    assert err <= 1e-5 * np.abs(want).max(), (err, np.abs(want).max())
    ax = project(torch.tensor(x, device="cuda"), angles, sc, use_offDetector=True).cpu().numpy().astype(np.float64)
    lhs, rhs = float((ax * y).sum()), float((x * got.astype(np.float64)).sum())
    print(f"dot {name}: relative gap {abs(lhs - rhs) / lhs:.3g}")
    assert abs(lhs - rhs) <= 1e-5 * lhs, (lhs, rhs)
    # the operator's weights come from the same launch
    op = CTOperator(angles, sc, "cuda", use_offDetector=True)
    vol, wgt = op.At(torch.tensor(y, device="cuda"), slice(None), True)
    assert torch.equal(vol.cpu(), torch.from_numpy(got))
    ones = oo.backproject_scene(np.ones_like(y), angles, sc)
    assert np.abs(wgt.cpu().numpy() - ones).max() <= 1e-5 * ones.max()


@pytest.mark.parametrize("mode,half_fan", [("cone", False), ("parallel", False), ("cone", True), ("parallel", True)])
def test_offset_fdk_matches_oracle(mode, half_fan):
    torch = _torch()
    from r2_gaussian_b200.fdk import fdk

    det, vox = (24, 40), (20, 28, 12)
    sc = _scanner(mode, det, vox, (1.6, 1.8, 1.2), (0.1, -0.2, 0.15), 0.5)
    sc = _offset(sc, 9.4 if half_fan else SHIFT[0], SHIFT[1])
    rng = np.random.RandomState(5)
    angles = fc.full_scan(12) + 0.2
    projs = rng.uniform(0.0, 1.0, size=(12, *det)).astype(np.float32)
    got = fdk(torch.tensor(projs, device="cuda"), angles, sc, use_offDetector=True, half_fan=half_fan).cpu().numpy()
    want = oo.fdk_scene(projs, angles, sc, half_fan=half_fan)
    err = np.abs(got.astype(np.float64) - want).max()
    print(f"fdk {mode} half_fan={half_fan}: max err / max = {err / np.abs(want).max():.3g}")
    assert err <= 1e-4 * np.abs(want).max(), (err, np.abs(want).max())


@pytest.mark.parametrize("op", ["project", "backproject", "fdk", "fdk_short_scan"])
@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_zero_offset_is_the_centred_result_bit_for_bit(mode, op):
    """offDetector = [0, 0] with use_offDetector=True adds exact zeros to every ray and cosine weight: each output is
    the centred one bit for bit (the backprojector's weights included)."""
    torch = _torch()
    from r2_gaussian_b200.fdk import fdk
    from r2_gaussian_b200.projector import backproject, project

    det, vox = (24, 40), (20, 28, 12)
    sc = dict(_scanner(mode, det, vox, (1.6, 1.8, 1.2), (0.1, -0.2, 0.15), 0.5), offDetector=[0.0, 0.0])
    rng = np.random.RandomState(7)
    angles = np.linspace(0.0, math.radians(240.0), 21)[:-1] if op == "fdk_short_scan" else fc.full_scan(12) + 0.2
    x = torch.tensor(rng.uniform(0.0, 1.0, vox).astype(np.float32), device="cuda")
    y = torch.tensor(rng.uniform(0.0, 1.0, (len(angles), *det)).astype(np.float32), device="cuda")
    run = {"project": lambda off: (project(x, angles, sc, use_offDetector=off),),
           "backproject": lambda off: backproject(y, angles, sc, weights=True, use_offDetector=off),
           "fdk": lambda off: (fdk(y, angles, sc, use_offDetector=off),),
           "fdk_short_scan": lambda off: (fdk(y, angles, sc, short_scan=True, use_offDetector=off),)}[op]
    for centred, offset in zip(run(False), run(True)):
        assert float(centred.abs().max()) > 0.0
        assert torch.equal(centred.view(torch.int32), offset.view(torch.int32))


def test_offset_short_scan_fdk_takes_a_vertical_offset():
    """Parker-weighted FDK with a vertical offset against the centred short scan of the row-moved projections."""
    torch = _torch()
    from r2_gaussian_b200.fdk import fdk

    sc = fc.scanner("cone", 32, 16)
    k = 3
    angles = np.linspace(0.0, math.radians(240.0), 41)[:-1]
    projs = np.random.RandomState(0).uniform(0.0, 1.0, (40, 32, 32)).astype(np.float32)
    projs[:, :k] = 0.0
    projs[:, -k:] = 0.0
    moved = np.zeros_like(projs)
    moved[:, k:] = projs[:, :-k]                                          # offDetector v = k rows: k rows down
    got = fdk(torch.tensor(moved, device="cuda"), angles, _offset(sc, 0.0, k), short_scan=True,
              use_offDetector=True).cpu().numpy()
    want = fdk(torch.tensor(projs, device="cuda"), angles, sc, short_scan=True).cpu().numpy()
    assert np.abs(got - want).max() <= 1e-4 * np.abs(want).max()


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_integer_offsets_move_the_projections(mode):
    torch = _torch()
    from r2_gaussian_b200.projector import project

    mode_, det, vox, sv, off, acc, angles = ORACLE_CASES[f"{mode}_acc05"]
    sc = _scanner(mode, det, vox, sv, off, acc)
    vol = torch.tensor(np.random.RandomState(1).uniform(0.0, 1.0, vox).astype(np.float32), device="cuda")
    base = project(vol, angles, sc).cpu().numpy()
    top = np.abs(base).max()
    assert np.array_equal(project(vol, angles, sc, use_offDetector=True).cpu().numpy(), base)
    for k in (1, 3):
        got = project(vol, angles, _offset(sc, k, 0), use_offDetector=True).cpu().numpy()
        assert np.abs(got[..., :-k] - base[..., k:]).max() <= 1e-5 * top              # k columns to smaller index
        got = project(vol, angles, _offset(sc, 0, k), use_offDetector=True).cpu().numpy()
        assert np.abs(got[:, k:, :] - base[:, :-k, :]).max() <= 1e-5 * top            # k rows to larger index


def _render_offset(pcl, pipe, sc, angles):
    torch = _torch()
    from r2_gaussian_b200.render_query import render

    with torch.no_grad():
        return torch.stack([render(scene.camera_from_view(scene.make_view(sc, float(a), use_offDetector=True)), pcl,
                                   pipe)["render"][0] for a in angles])


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_render_of_offset_cameras_is_the_offset_projection(mode):
    from r2_gaussian_b200.projector import project

    pcl, pipe = _cloud_tensors(fc.round_trip_cloud())
    sc = _offset(fc.scanner(mode, pc.ROUND_TRIP_DET, pc.ROUND_TRIP_VOX), *SHIFT)
    angles = list(pc.ROUND_TRIP_ANGLES)
    want = _render_offset(pcl, pipe, sc, angles).cpu().numpy()
    vol = _query(pcl, pipe, sc)
    err = pc.rel_l2(project(vol, angles, sc, use_offDetector=True).cpu().numpy(), want)
    centred = pc.rel_l2(project(vol, angles, sc | {"offDetector": [0.0, 0.0]}).cpu().numpy(), want)
    print(f"render vs offset projection {mode}: {err:.4f} (centred projector {centred:.4f})")
    assert err <= pc.ROUND_TRIP_BOUND, err
    assert centred >= 2 * pc.ROUND_TRIP_BOUND, centred


def test_render_offset_fdk_query_round_trip():
    torch = _torch()
    from r2_gaussian_b200.fdk import fdk

    pcl, pipe = _cloud_tensors(fc.round_trip_cloud())
    sc = _offset(fc.scanner("cone", fc.ROUND_TRIP_DET, fc.ROUND_TRIP_VOX), *SHIFT)
    angles = fc.full_scan(180)
    projs = _render_offset(pcl, pipe, sc, angles)
    want = _query(pcl, pipe, sc).cpu().numpy()
    got = fdk(projs, angles, sc, use_offDetector=True).cpu().numpy()
    err = fc.rel_l2(got, want)
    with pytest.warns(UserWarning, match="ignored"):
        ignored = fc.rel_l2(fdk(projs, angles, sc).cpu().numpy(), want)
    print(f"render -> offset fdk -> query: {err:.4f} (offset ignored {ignored:.4f})")
    assert err <= FDK_ROUND_TRIP_BOUND, err
    assert ignored > err


def _phantom(n):
    """A ball of radius 0.9 (density 0.5) holding two denser balls, one of them far off the axis."""
    g = (np.arange(n) + 0.5) / n * 2.0 - 1.0
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    vol = 0.5 * (X ** 2 + Y ** 2 + Z ** 2 <= 0.81)
    vol += 0.5 * ((X - 0.55) ** 2 + Y ** 2 + Z ** 2 <= 0.04)
    vol += 0.3 * (X ** 2 + (Y + 0.2) ** 2 + (Z - 0.1) ** 2 <= 0.05)
    return vol.astype(np.float32)


def _yml(tmp_path, name, n_det, n_vox, off_px=(0.0, 0.0), total=360.0):
    sc = scene.cone_beam_scanner(n_det, n_vox)
    phys = {k: (np.asarray(v, float) * 2.0).tolist() if k in ("DSD", "DSO", "sDetector", "sVoxel", "offOrigin")
            else v for k, v in sc.items()}
    du, dv = phys["sDetector"][1] / n_det, phys["sDetector"][0] / n_det
    phys["offDetector"] = [off_px[0] * du, off_px[1] * dv]
    phys.update({"filter": None, "accuracy": 0.5, "totalAngle": total, "startAngle": 0.0, "noise": False})
    yml = tmp_path / f"{name}.yml"
    yml.write_text("".join(f"{k}: {json.dumps(v)}\n" for k, v in phys.items()))
    return yml


def test_half_fan_fdk_on_a_quarter_width_offset(tmp_path):
    """A 360-degree scan with the detector shifted by a quarter of its width: half-fan FDK against the unweighted offset
    FDK and against FDK of the centred detector."""
    torch = _torch()
    from r2_gaussian_b200 import generate_data
    from r2_gaussian_b200.dataset import read_scene
    from r2_gaussian_b200.fdk import fdk
    from r2_gaussian_b200.metrics import metric_vol

    n_det, n_vox = 96, 48
    np.save(tmp_path / "vol.npy", _phantom(n_vox))
    res = {}
    for name, off in (("centred", (0.0, 0.0)), ("offset", (n_det / 4, 0.0))):
        case = generate_data.main(["--vol", str(tmp_path / "vol.npy"), "--scanner", str(_yml(tmp_path, name, n_det, n_vox, off)),
                                   "--n_train", "90", "--n_test", "2", "--output", str(tmp_path / name),
                                   "--use_offDetector"])
        info = read_scene(case, eval=False)
        projs = torch.from_numpy(np.stack([c.image for c in info.train_cameras])).cuda()
        angles = [c.angle for c in info.train_cameras]
        variants = {"plain": {}} if name == "centred" else {"plain": {}, "half_fan": {"half_fan": True}}
        for v, kw in variants.items():
            vol = fdk(projs, angles, info.scanner_cfg, use_offDetector=True, **kw)
            res[name, v] = float(metric_vol(torch.from_numpy(info.vol).cuda(), vol, "psnr")[0])
    print("half fan psnr_3d: " + ", ".join(f"{k}: {v:.2f}" for k, v in res.items()))
    assert res["offset", "half_fan"] >= res["offset", "plain"] + HALF_FAN_GAIN_DB, res
    assert res["offset", "half_fan"] >= res["centred", "plain"] - HALF_FAN_LOSS_DB, res


def _train(path, init, model_path, use_offDetector, iterations):
    import torch

    from r2_gaussian_b200 import trainer
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    model = trainer.ModelParams(source_path=path, model_path=str(model_path), ply_path=init)
    opt = trainer.OptimizationParams(iterations=iterations)
    h = trainer.training(model, opt, trainer.PipelineParams(), {iterations}, set(), log=lambda *a: None,
                         use_offDetector=use_offDetector)
    return h["eval"][iterations]["psnr_3d"]


def test_generate_initialize_train_with_an_offset_detector(tmp_path, capsys):
    """generate_data, initialize_pcd and trainer with --use_offDetector on a scanner offset by (2.5, -2) pixels: within
    1.5 dB of the same scene without the offset, and well above training that ignores the offset."""
    from r2_gaussian_b200 import generate_data, initialize_pcd
    from test_projector_gpu import _write_inputs

    _, vol_path, *_ = _write_inputs(tmp_path, noise=False)
    it = 2000
    runs = {}
    for name, off in (("plain", (0.0, 0.0)), ("offset", (2.5, -2.0))):
        yml = _yml(tmp_path, name, pc.ROUND_TRIP_DET, pc.ROUND_TRIP_VOX, off)
        switch = ["--use_offDetector"] if name == "offset" else []
        case = generate_data.main(["--vol", str(vol_path), "--scanner", str(yml), "--n_train", "24", "--n_test", "6",
                                   "--output", str(tmp_path / name), *switch])
        init = initialize_pcd.main(["--data", case, "--recon_method", "fdk", "--n_points", "2000",
                                    "--output", str(tmp_path / f"init_{name}.npy"), *switch])
        runs[name, True] = _train(case, init, tmp_path / f"m_{name}", bool(switch), it)
        if name == "offset":
            runs[name, False] = _train(case, init, tmp_path / f"m_{name}_ignored", False, it)
    print("offset detector training psnr_3d: " + ", ".join(f"{k}: {v:.2f}" for k, v in runs.items()))
    assert runs["offset", True] >= runs["plain", True] - 1.5, runs
    assert runs["offset", True] >= runs["offset", False] + 3.0, runs
