"""r2x_mar_inpaint on the GPU, bit for bit against the numpy model (tests/mar_oracle.py): widths around the CTA size up
to the limit, random and edge traces, whole-trace rows, priors below eps, in place, repeats, grids around a boundary
and a stack past 2^31 samples; `mar.reduce_metal` against the host rules; then `python -m r2_gaussian_b200.reduce_metal`
and `recon --mar` on a cone-beam metal scene from tests/mar_cases.py, end to end."""
import os
import random

import numpy as np
import pytest
import yaml

import mar_oracle as mo

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]


def _t(x, dtype=np.float32):
    import torch

    return torch.from_numpy(np.ascontiguousarray(x, dtype)).cuda()


def _run(p, m, tau, d, P=None, eps=1e-3, trace=True):
    import torch

    from r2_gaussian_b200.mar import inpaint

    tr = torch.empty(p.shape, dtype=torch.uint8, device="cuda") if trace else None
    out = inpaint(_t(p), _t(m), tau, d, None if P is None else _t(P), eps, trace=tr)
    return out.cpu().numpy(), None if tr is None else tr.cpu().numpy()


def _case(rng, n, H, W):
    p = rng.normal(1.0, 0.5, (n, H, W)).astype(np.float32)
    m = np.zeros((n, H, W), np.float32)
    u = rng.random((n, H, W))
    m[u < 0.05] = 1.0                                       # scattered trace
    for v in range(n):
        for r in range(H):
            k = (v * H + r) % 6
            if k == 1:
                m[v, r, :max(1, W // 5)] = 1.0              # a run at the left edge
            elif k == 2:
                m[v, r, W - max(1, W // 7):] = 1.0          # and at the right edge
            elif k == 3:
                m[v, r] = 1.0                               # the whole row
            elif k == 4:
                m[v, r] = 0.0                               # none
    P = rng.uniform(0.0, 2.0, (n, H, W)).astype(np.float32)
    P[rng.random(P.shape) < 0.05] = 1e-6                    # below eps
    return p, m, P


@pytest.mark.parametrize("W", [1, 2, 3, 255, 256, 257, 2368, 16384])
@pytest.mark.parametrize("prior", [False, True])
def test_equals_the_oracle_bit_for_bit(W, prior):
    rng = np.random.default_rng(W * 2 + prior)
    n, H = (2, 3) if W < 4096 else (1, 6)
    p, m, P = _case(rng, n, H, W)
    for d in (0, 2):
        got, tr = _run(p, m, 0.5, d, P if prior else None)
        want, wtr = mo.inpaint(p, m, 0.5, d, P if prior else None)
        assert got.tobytes() == want.tobytes() and tr.tobytes() == wtr.tobytes(), (W, prior, d)
    got, tr = _run(p, m, 0.5, 1, P if prior else None, trace=False)
    assert tr is None and got.tobytes() == mo.inpaint(p, m, 0.5, 1, P if prior else None)[0].tobytes()


def test_one_past_the_width_limit_is_refused():
    import torch

    from r2_gaussian_b200.mar import inpaint

    x = torch.zeros((1, 1, 16385), device="cuda")
    with pytest.raises(ValueError, match="16384"):
        inpaint(x, x.clone(), 0.5, 1)


def test_special_values_outside_the_trace_and_large_dilations():
    rng = np.random.default_rng(1)
    p, m, P = _case(rng, 3, 4, 300)
    u = rng.random(p.shape)
    p[u < 0.03] = np.nan
    p[(u >= 0.03) & (u < 0.05)] = np.inf
    p[(u >= 0.05) & (u < 0.07)] = -0.0
    p.view(np.uint32)[u > 0.99] = 0x7FC12345
    m[(u > 0.5) & (u < 0.52)] = np.nan
    for d in (0, 7, 299, 300, 1 << 30):
        for prior in (None, P):
            got, tr = _run(p, m, 0.5, d, prior)
            want, wtr = mo.inpaint(p, m, 0.5, min(d, 300), prior)
            assert got.tobytes() == want.tobytes() and tr.tobytes() == wtr.tobytes(), d


def test_in_place_equals_out_of_place_and_repeats_give_the_same_bits():
    import torch

    from r2_gaussian_b200.mar import inpaint

    rng = np.random.default_rng(2)
    p, m, P = _case(rng, 20, 16, 512)
    for prior in (None, _t(P)):
        ref = inpaint(_t(p), _t(m), 0.5, 2, prior)
        again = inpaint(_t(p), _t(m), 0.5, 2, prior)
        assert ref.cpu().numpy().tobytes() == again.cpu().numpy().tobytes()
        y = _t(p)
        assert inpaint(y, _t(m), 0.5, 2, prior, out=y) is y
        assert y.cpu().numpy().tobytes() == ref.cpu().numpy().tobytes()
    rows = [0, 7, 15]
    want, _ = mo.inpaint(p, m, 0.5, 2, P, rows=rows)
    assert inpaint(_t(p), _t(m), 0.5, 2, _t(P)).cpu().numpy()[:, rows].tobytes() == want.tobytes()


@pytest.mark.parametrize("rows", [65535, 65536, 65537])
def test_grid_around_a_boundary(rows):
    rng = np.random.default_rng(rows)
    p, m, P = _case(rng, rows // 97 + 1, 97, 5)
    p, m, P = p.reshape(-1, 5)[:rows], m.reshape(-1, 5)[:rows], P.reshape(-1, 5)[:rows]
    p, m, P = p.reshape(1, rows, 5), m.reshape(1, rows, 5), P.reshape(1, rows, 5)
    got, tr = _run(p, m, 0.5, 1, P)
    want, wtr = mo.inpaint(p, m, 0.5, 1, P)
    assert got.tobytes() == want.tobytes() and tr.tobytes() == wtr.tobytes()


def test_view_windows_give_the_same_bits(monkeypatch):
    from r2_gaussian_b200 import mar

    rng = np.random.default_rng(3)
    p, m, P = _case(rng, 11, 5, 70)
    whole = mar.inpaint(_t(p), _t(m), 0.5, 1, _t(P)).cpu().numpy()
    monkeypatch.setattr(mar, "_MAX_ROWS", 3 * 5)            # windows of 3 views
    assert mar.inpaint(_t(p), _t(m), 0.5, 1, _t(P)).cpu().numpy().tobytes() == whole.tobytes()


def test_past_2_31_samples_in_place():
    import torch

    from r2_gaussian_b200.mar import inpaint

    n, H, W = 721, 1600, 1900
    assert n * H * W > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn((n, H, W), device="cuda", generator=g)
    m = (torch.rand((n, H, W), device="cuda", generator=g) < 0.02).to(torch.float32)
    rows = [0, 1, 799, 1598, H - 1]
    views = [0, 360, n - 1]
    before, mb = x[views][:, rows].cpu().numpy(), m[views][:, rows].cpu().numpy()
    inpaint(x, m, 0.5, 2, out=x)
    got = x[views][:, rows].cpu().numpy()
    del x, m
    torch.cuda.empty_cache()
    assert got.tobytes() == mo.inpaint(before, mb, 0.5, 2)[0].tobytes()


# ---- reduce_metal and the CLIs on a cone-beam metal scene --------------------------------------------------------------

@pytest.fixture(scope="module")
def metal_scene(tmp_path_factory):
    import mar_cases

    tmp = tmp_path_factory.mktemp("mar")
    path, tissue, metal, mask = mar_cases.metal_scene(str(tmp / "metal"))
    return path, mask, tmp


def _stacks(path):
    import torch

    from r2_gaussian_b200.dataset import read_scene

    info = read_scene(path)
    st = lambda cams: torch.from_numpy(np.stack([c.image for c in cams]).astype(np.float32)).cuda()
    return (info, st(info.train_cameras), [c.angle for c in info.train_cameras], st(info.test_cameras),
            [c.angle for c in info.test_cameras])


def test_reduce_metal_against_the_host_rules(metal_scene):
    import torch

    from r2_gaussian_b200 import mar
    from r2_gaussian_b200.fdk import fdk
    from r2_gaussian_b200.projector import project

    path, mask, _ = metal_scene
    info, ptr, atr, pte, ate = _stacks(path)
    cfg = info.scanner_cfg
    tau = mar.TRACE_TAU * min(cfg["dVoxel"])
    res = mar.reduce_metal(ptr, atr, cfg, method="nmar", mask=mask, extra=[(pte, ate)])
    assert torch.equal(res.mask.cpu(), torch.from_numpy(mask))
    for p, ang, (got, tr) in ((ptr, atr, (res.projs, res.trace)), (pte, ate, res.extra[0][:2])):
        mp = project(torch.from_numpy(mask.astype(np.float32)).cuda(), ang, cfg).cpu().numpy()
        rows = [5, 31, 40]
        _, want_tr = mo.inpaint(p.cpu().numpy(), mp, tau, mar.TRACE_DILATE, rows=rows)
        assert tr.cpu().numpy()[:, rows].tobytes() == want_tr.tobytes()
        assert tr.any()
        outside = tr.cpu().numpy() == 0
        assert got.cpu().numpy()[outside].tobytes() == p.cpu().numpy()[outside].tobytes()
    assert res.trace_fraction == pytest.approx(float(res.trace.float().mean()))
    # the prior: the float64 rules on the LI volume of the same mask
    li = mar.reduce_metal(ptr, atr, cfg, method="li", mask=mask)
    vol_li = fdk(li.projs, atr, cfg)
    want, *_ = mo.nmar_prior(vol_li.cpu().numpy(), mask)
    got = mar.nmar_prior(vol_li, torch.from_numpy(mask).cuda()).cpu().numpy()
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=0)
    # segmentation: FDK > threshold
    vol0 = fdk(ptr, atr, cfg)
    t = 0.6 * float(vol0.max())
    seg = mar.reduce_metal(ptr, atr, cfg, method="li", threshold=t)
    assert np.array_equal(seg.mask.cpu().numpy(), mo.segment(vol0.cpu().numpy(), t))
    rec = mar.reinsert(torch.zeros_like(vol0), vol0, seg.mask)
    assert np.array_equal(rec.cpu().numpy(), mo.reinsert(0 * vol0.cpu().numpy(), vol0.cpu().numpy(),
                                                         seg.mask.cpu().numpy()))


def test_no_metal_is_refused_and_nothing_written(metal_scene):
    from r2_gaussian_b200 import mar, reduce_metal as rm

    path, mask, tmp = metal_scene
    info, ptr, atr, *_ = _stacks(path)
    with pytest.raises(ValueError, match="empty"):
        mar.reduce_metal(ptr, atr, info.scanner_cfg, mask=np.zeros_like(mask))
    with pytest.raises(ValueError, match="threshold 1e\\+06"):
        mar.reduce_metal(ptr, atr, info.scanner_cfg, threshold=1e6)
    out = str(tmp / "none")
    with pytest.raises(ValueError, match="threshold"):
        rm.main(["-s", path, "--output", out, "--metal_threshold", "1e6"])
    assert not os.path.exists(out)


def test_scene_cli_and_recon_end_to_end(metal_scene, capsys):
    import torch

    from r2_gaussian_b200 import initialize_pcd, mar, recon, reduce_metal as rm, trainer
    from r2_gaussian_b200.dataset import read_scene

    path, mask, tmp = metal_scene
    np.save(os.path.join(path, "init_x.npy"), np.zeros((3, 4), np.float32))
    np.save(tmp / "mask.npy", mask)
    out = rm.main(["-s", path, "--output", str(tmp / "fixed"), "--metal_mask", str(tmp / "mask.npy")])
    assert "init_x.npy" in capsys.readouterr().out and not os.path.exists(os.path.join(out, "init_x.npy"))
    with open(os.path.join(path, "meta_data.json"), "rb") as a, open(os.path.join(out, "meta_data.json"), "rb") as b:
        assert a.read() == b.read()
    assert np.array_equal(np.load(os.path.join(out, "metal_mask.npy")), mask)
    with open(os.path.join(out, "mar.yml")) as f:
        rep = yaml.safe_load(f)
    assert rep["method"] == "nmar" and rep["metal_voxels"] == int(mask.sum())
    assert 0 < rep["trace_fraction_train"] < 1 and 0 < rep["trace_fraction_test"] < 1
    info, ptr, atr, pte, ate = _stacks(path)
    res = mar.reduce_metal(ptr, atr, info.scanner_cfg, mask=mask, extra=[(pte, ate)])
    fixed = read_scene(out)
    got = np.stack([c.image for c in fixed.test_cameras])
    np.testing.assert_allclose(got, res.extra[0][0].cpu().numpy(), rtol=1e-6, atol=1e-7)   # test views, train mask

    base = recon.main(["-s", path, "-m", str(tmp / "plain"), "--methods", "fdk"])
    assert "psnr_3d_outside_metal" not in base["fdk"] and "mar" not in base["fdk"]
    base_again = recon.main(["-s", path, "-m", str(tmp / "plain2"), "--methods", "fdk"])
    assert base_again["fdk"]["psnr_3d"] == base["fdk"]["psnr_3d"]
    scores = {}
    for m in ("li", "nmar"):
        r = recon.main(["-s", path, "-m", str(tmp / m), "--methods", "fdk", "--mar", m, "--metal_mask",
                        str(tmp / "mask.npy")])["fdk"]
        assert r["mar"] == m and r["metal_voxels"] == int(mask.sum()) and 0 < r["trace_fraction"] < 1
        scores[m] = r["psnr_3d_outside_metal"]
    ct = np.load(os.path.join(tmp / "plain", "fdk", "ct_pred.npy"))
    scores["fdk"] = mo.psnr_outside_metal(np.load(os.path.join(path, "vol_gt.npy")), ct, mask)
    print(f"psnr_3d_outside_metal: {scores}")
    # measured on an H100 80GB HBM3: 21.99 dB without MAR, 24.21 dB with NMAR (DESIGN §8); the margin is under half
    # that gain
    assert scores["nmar"] > scores["fdk"] + 1.0

    init = initialize_pcd.main(["--data", out, "--n_points", "2000", "--output", str(tmp / "init.npy")])
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    model = trainer.ModelParams(source_path=out, model_path="", ply_path=init)
    hist = trainer.training(model, trainer.OptimizationParams(iterations=100), trainer.PipelineParams(), {100}, set(),
                            log=lambda *a: None)
    assert np.isfinite(hist["eval"][100]["psnr_3d"])
