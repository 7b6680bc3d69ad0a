"""Metal-trace inpainting without a GPU: the numpy model (tests/mar_oracle.py) against closed forms, the float64 host
rules, and the refusals of the C ABI, `mar.inpaint` / `mar.reduce_metal`, `python -m r2_gaussian_b200.reduce_metal`
and `recon --mar`."""
import json
import os

import numpy as np
import pytest

import mar_oracle as mo
from r2_gaussian_b200 import _lib, mar

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")


def _runs_trace(W, runs):
    m = np.zeros(W, np.float32)
    for a, b in runs:
        m[a:b] = 1.0
    return m


def test_dilation_clips_at_the_row_ends_and_equals_a_direct_search():
    rng = np.random.default_rng(0)
    for W in (1, 2, 3, 17, 64):
        for d in (0, 1, 2, 5, W, W + 3):
            m = (rng.random(W) < 0.1).astype(np.float32)
            t = mo.trace_row(m, 0.5, d)
            for c in range(W):
                assert t[c] == any(m[k] > 0.5 for k in range(W) if abs(k - c) <= d)
    t = mo.trace_row(_runs_trace(8, [(0, 1)]), 0.5, 3)
    assert t.tolist() == [True] * 4 + [False] * 4
    t = mo.trace_row(_runs_trace(8, [(7, 8)]), 0.5, 2)
    assert t.tolist() == [False] * 5 + [True] * 3


def test_a_linear_row_is_reproduced_inside_any_trace():
    rng = np.random.default_rng(1)
    W = 200
    p = (np.float32(3.0) + np.arange(W, dtype=np.float32) * np.float32(0.0625)).astype(np.float32)
    for _ in range(20):
        m = (rng.random(W) < 0.15).astype(np.float32)
        m[:2] = m[-2:] = 0.0                                 # both ends stay outside the dilated trace
        out, t = mo.inpaint_row(p, m, 0.5, 1)
        np.testing.assert_allclose(out, p, rtol=4e-7, atol=0)
    # gaps of a power of two: s and every product are exact, so the line comes back bit for bit
    for a, b in [(1, 4), (10, 17), (100, 131)]:
        m = _runs_trace(W, [(a, b)])
        out, t = mo.inpaint_row(p, m, 0.5, 0)
        assert out.tobytes() == p.tobytes()
        P = np.full(W, 2.0, np.float32)
        out, _ = mo.inpaint_row(p, m, 0.5, 0, P)
        assert out.tobytes() == p.tobytes()


def test_traces_touching_either_edge_take_the_one_sided_value():
    p = np.arange(10, dtype=np.float32) + np.float32(1)
    out, _ = mo.inpaint_row(p, _runs_trace(10, [(0, 3)]), 0.5, 0)
    assert out[:3].tolist() == [4.0] * 3 and out[3:].tobytes() == p[3:].tobytes()
    out, _ = mo.inpaint_row(p, _runs_trace(10, [(8, 10)]), 0.5, 1)
    assert out[7:].tolist() == [7.0] * 3 and out[:7].tobytes() == p[:7].tobytes()
    P = np.array([1, 1, 1, 2, 2, 2, 2, 2, 4, 4], np.float32)
    out, _ = mo.inpaint_row(p, _runs_trace(10, [(0, 3)]), 0.5, 0, P)
    assert out[:3].tolist() == [2.0, 2.0, 2.0]                      # q[3] = 4 / 2, times Pe = 1


def test_an_all_trace_row_is_copied_or_becomes_the_prior():
    p = np.array([1, np.nan, 3, -np.inf], np.float32)
    m = np.ones(4, np.float32)
    out, t = mo.inpaint_row(p, m, 0.5, 0)
    assert t.all() and out.tobytes() == p.tobytes()
    P = np.array([0.5, 1e-9, np.nan, 7], np.float32)
    out, _ = mo.inpaint_row(p, m, 0.5, 0, P, eps=1e-3)
    assert out.tobytes() == np.array([0.5, 1e-3, 1e-3, 7], np.float32).tobytes()


def test_pixels_outside_the_trace_keep_their_bits_nan_and_inf_included():
    rng = np.random.default_rng(2)
    W = 64
    p = rng.normal(0, 1, W).astype(np.float32)
    p[[0, 5, 9, 30, 63]] = [np.nan, np.inf, -np.inf, -0.0, np.nan]
    p.view(np.uint32)[40] = 0x7FC12345
    m = _runs_trace(W, [(12, 20), (45, 50)])
    P = rng.uniform(0.5, 2.0, W).astype(np.float32)
    for prior in (None, P):
        out, t = mo.inpaint_row(p, m, 0.5, 1, prior)
        assert out[~t].tobytes() == p[~t].tobytes()


def test_no_trace_returns_the_input_bit_for_bit():
    rng = np.random.default_rng(3)
    p = rng.normal(0, 1, (3, 4, 33)).astype(np.float32)
    p.flat[:4] = [np.nan, np.inf, -0.0, 1e-45]
    m = rng.uniform(0, 1, p.shape).astype(np.float32)
    for prior in (None, rng.uniform(0, 1, p.shape).astype(np.float32)):
        out, tr = mo.inpaint(p, m, 1.0, 0, prior)
        assert out.tobytes() == p.tobytes() and not tr.any()


def test_the_prior_classes_and_reinsertion():
    x = np.array([[[0.0, 0.05, 1.0, 1.2, 0.9, 3.0, 5.0, 0.4]]], np.float32)
    mask = np.zeros_like(x, bool)
    mask[0, 0, 6] = True
    prior, s, mean = mo.nmar_prior(x, mask)
    # non-metal above 0.1 * 3: 1.0, 1.2, 0.9, 3.0, 0.4 -> lower median 1.0; tissue [0.5, 1.5): 1.0, 1.2, 0.9
    assert s == 1.0 and mean == pytest.approx(31 / 30)
    np.testing.assert_allclose(prior[0, 0], [0, 0, mean, mean, mean, 3.0, mean, 0], rtol=1e-7)
    assert mo.reinsert(np.zeros(3), np.arange(3.0), np.array([0, 1, 0], bool)).tolist() == [0, 1, 0]
    m = np.zeros((7, 7, 7), bool)
    m[3, 3, 3] = True
    assert mo.dilate(m).sum() == 125


def test_the_gpu_host_rules_equal_the_float64_restatement_on_the_cpu():
    import torch

    rng = np.random.default_rng(4)
    x = rng.gamma(2.0, 0.3, (12, 13, 14)).astype(np.float32)
    mask = x > 1.8
    want, *_ = mo.nmar_prior(x, mask)
    got = mar.nmar_prior(torch.from_numpy(x), torch.from_numpy(mask)).numpy()
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=0)
    assert ((got == 0) == (want == 0)).all()
    gt = rng.uniform(0, 1, x.shape)
    assert mar.psnr_outside_metal(gt, x, mask) == pytest.approx(mo.psnr_outside_metal(gt, x, mask), rel=1e-12)


# ---- refusals ---------------------------------------------------------------------------------------------------------

def _abi(n=2, H=3, W=8, p=1 << 20, m=2 << 20, tau=0.5, d=1, P=None, eps=1e-3, out=3 << 20, trace=None):
    lib = _lib.load()
    rc = lib.r2x_mar_inpaint(None, n, H, W, p, m, tau, d, P, eps, out, trace)
    return rc, (lib.r2x_last_error() or b"").decode()


@pytest.mark.parametrize("kw,what", [
    (dict(p=None), "pointer"), (dict(m=None), "pointer"), (dict(out=None), "pointer"),
    (dict(n=0), "shape"), (dict(H=0), "shape"), (dict(W=0), "shape"), (dict(n=-1), "shape"),
    (dict(n=1 << 16, H=1 << 15), "n * H"), (dict(W=16385), "R2X_MAR_MAX_W"),
    (dict(tau=float("nan")), "bad tau"), (dict(tau=float("inf")), "bad tau"),
    (dict(eps=0.0), "bad eps"), (dict(eps=-1.0), "bad eps"), (dict(eps=float("inf")), "bad eps"),
    (dict(eps=float("nan")), "bad eps"), (dict(d=-1), "bad d"),
    (dict(out=(1 << 20) + 4), "overlaps p"), (dict(out=(2 << 20) + 4), "overlaps m or P"),
    (dict(P=(3 << 20) + 8), "overlaps m or P"),
    (dict(trace=(1 << 20) + 1), "trace overlaps"), (dict(trace=(3 << 20) + 1), "trace overlaps"),
    (dict(trace=(2 << 20) + 1), "trace overlaps"), (dict(P=4 << 20, trace=(4 << 20) + 3), "trace overlaps"),
])
def test_c_abi_refuses_bad_arguments_before_any_cuda_work(kw, what):
    rc, msg = _abi(**kw)
    assert rc == 1 and "r2x_mar_inpaint" in msg and what in msg, msg


def test_inpaint_refuses_bad_inputs():
    import torch

    with pytest.raises(ValueError, match="CUDA float32"):
        mar.inpaint(np.zeros((2, 2, 2), np.float32), np.zeros((2, 2, 2), np.float32), 0.5, 1)
    with pytest.raises(ValueError, match="CUDA float32"):
        mar.inpaint(torch.zeros((2, 2, 2)), torch.zeros((2, 2, 2)), 0.5, 1)


def test_reduce_metal_refuses_before_any_cuda_work():
    import torch

    cfg = {"nVoxel": [4, 4, 4], "dVoxel": [0.5] * 3}
    x = torch.zeros((2, 3, 4))
    with pytest.raises(ValueError, match="method"):
        mar.reduce_metal(x, [0, 1], cfg, method="nmar2", threshold=1.0)
    for k in ("view_geometry", "helical"):
        with pytest.raises(ValueError, match="not supported"):
            mar.reduce_metal(x, [0, 1], cfg, threshold=1.0, **{k: [{}] if k == "view_geometry" else True})
    with pytest.raises(TypeError, match="unexpected"):
        mar.reduce_metal(x, [0, 1], cfg, threshold=1.0, accuracy=2)
    with pytest.raises(ValueError, match="exactly one"):
        mar.reduce_metal(x, [0, 1], cfg)
    with pytest.raises(ValueError, match="exactly one"):
        mar.reduce_metal(x, [0, 1], cfg, threshold=1.0, mask=np.ones((4, 4, 4), bool))
    with pytest.raises(ValueError, match="shape"):
        mar.reduce_metal(x, [0, 1], cfg, mask=np.ones((4, 4, 5), bool))
    with pytest.raises(RuntimeError, match="CUDA"):
        mar.reduce_metal(x, [0, 1], cfg, threshold=1.0)


def _scene(tmp_path, frame_extra=None):
    src = tmp_path / "scene"
    (src / "proj_train").mkdir(parents=True)
    (src / "proj_test").mkdir()
    frames = {"proj_train": [], "proj_test": []}
    for i in range(4):
        split = "proj_train" if i % 2 == 0 else "proj_test"
        rel = f"{split}/{split}_{i:04d}.npy"
        np.save(src / rel, np.ones((6, 8), np.float32))
        frames[split].append({"file_path": rel, "angle": 0.1 * i, **(frame_extra or {})})
    np.save(src / "vol_gt.npy", np.zeros((4, 4, 4), np.float32))
    (src / "meta_data.json").write_text(json.dumps({"scanner": {"nVoxel": [4, 4, 4]}, "vol": "vol_gt.npy", **frames}))
    return src


def test_scene_cli_refusals(tmp_path):
    from r2_gaussian_b200 import reduce_metal as rm

    src = _scene(tmp_path)
    out = str(tmp_path / "out")
    with pytest.raises(SystemExit):
        rm.main(["-s", str(src), "--output", out])                                   # neither threshold nor mask
    with pytest.raises(SystemExit):
        rm.main(["-s", str(src), "--output", out, "--metal_threshold", "1", "--metal_mask", "m.npy"])
    with pytest.raises(SystemExit):
        rm.main(["-s", str(src), "--output", out, "--metal_threshold", "1", "--method", "nmar2"])
    naf = tmp_path / "scan.pickle"
    naf.write_bytes(b"\x80\x04N.")
    with pytest.raises(ValueError, match="NAF pickle"):
        rm.main(["-s", str(naf), "--output", out, "--metal_threshold", "1"])
    with pytest.raises(ValueError, match="is the source"):
        rm.main(["-s", str(src), "--output", str(src), "--metal_threshold", "1"])
    taken = tmp_path / "taken"
    taken.mkdir()
    (taken / "meta_data.json").write_text("{}")
    with pytest.raises(ValueError, match="already holds"):
        rm.main(["-s", str(src), "--output", str(taken), "--metal_threshold", "1"])
    helical = _scene(tmp_path / "h", {"offOrigin": [0, 0, 0.1]})
    with pytest.raises(ValueError, match="per-view geometry"):
        rm.main(["-s", str(helical), "--output", out, "--metal_threshold", "1"])
    np.save(tmp_path / "bad.npy", np.ones((4, 4, 5), bool))
    with pytest.raises(ValueError, match="shape"):
        rm.main(["-s", str(src), "--output", out, "--metal_mask", str(tmp_path / "bad.npy")])
    np.save(tmp_path / "float.npy", np.ones((4, 4, 4), np.float32))
    with pytest.raises(ValueError, match="bool"):
        rm.main(["-s", str(src), "--output", out, "--metal_mask", str(tmp_path / "float.npy")])
    assert not os.path.exists(out)


@pytest.mark.parametrize("args,what", [
    (["--metal_threshold", "1"], "--mar only"), (["--metal_mask", "m.npy"], "--mar only"),
    (["--mar", "nmar"], "exactly one"), (["--mar", "li", "--metal_threshold", "1", "--metal_mask", "m.npy"],
                                          "exactly one"),
    (["--mar", "nmar", "--metal_threshold", "1", "--use_view_geometry"], "--use_view_geometry"),
    (["--mar", "nmar", "--metal_threshold", "1", "--use_view_geometry", "--helical"], "--mar cannot"),
    (["--mar", "nmar", "--metal_threshold", "nan"], "finite"),
])
def test_recon_refuses_bad_mar_flags(tmp_path, args, what):
    from r2_gaussian_b200 import recon

    with pytest.raises(SystemExit, match=what):
        recon.main(["-s", str(tmp_path / "missing"), "-m", str(tmp_path / "o"), "--methods", "fdk", *args])
    assert not os.path.exists(tmp_path / "o")


def test_recon_refuses_an_unknown_mar_method(tmp_path):
    from r2_gaussian_b200 import recon

    with pytest.raises(SystemExit):
        recon.main(["-s", str(tmp_path / "missing"), "-m", str(tmp_path / "o"), "--mar", "nmar2",
                    "--metal_threshold", "1"])
