"""r2x_remove_stripes on the GPU, bit for bit against the numpy model (tests/stripe_oracle.py): view counts and widths
around both passes' tiles up to the view limit, special values, in place, repeats, row splits, a stack past 2^31
samples and the closed form; then `python -m r2_gaussian_b200.remove_stripes` on a striped generate_data scene and
`generate_real_data --remove_stripes` on a striped FIPS-format scan, end to end."""
import json
import os
import random

import numpy as np
import pytest

import stripe_oracle as so
from test_stripes_cpu import clean_with_offsets

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore::RuntimeWarning")]


def _run(x, K, **kw):
    import torch

    from r2_gaussian_b200.stripes import remove_stripes

    return remove_stripes(torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda(), K, **kw).cpu().numpy()


def _sort_tile(n):
    """Pass A's column tile at n views (csrc/r2x_stripes.cu): min(32, 8192 / P)."""
    P = 1 << max(0, (n - 1).bit_length())
    return min(32, 8192 // P)


def _cases():
    out = []
    for n in (1, 2, 3, 31, 32, 33, 721, 8192):
        tw = _sort_tile(n)
        for W in sorted({max(1, tw - 1), tw, tw + 1, 255, 256, 257}):
            for K in sorted({1, 3, 21, 255, 2 * W + 1}):
                if K <= 255 and K // 2 <= W and n * W * K <= 6e7:
                    out.append((n, W, K))
    return out


@pytest.mark.parametrize("n,W,K", _cases())
def test_equals_the_oracle_bit_for_bit(n, W, K):
    rng = np.random.default_rng(n * 7919 + W * 31 + K)
    x = rng.normal(0.0, 1.0, (n, 1, W)).astype(np.float32)
    x[:, :, ::3] = np.round(x[:, :, ::3] * 4) / 4                     # ties in every third column
    assert _run(x, K).tobytes() == so.remove_stripes(x, K).tobytes()


@pytest.mark.parametrize("K", [1, 3, 21])
def test_ties_signed_zeros_infinities_and_nans(K):
    rng = np.random.default_rng(K)
    x = rng.integers(-3, 4, (37, 3, 50)).astype(np.float32)
    m = rng.random(x.shape)
    x[m < 0.1] = -0.0
    x[(m >= 0.1) & (m < 0.15)] = np.inf
    x[(m >= 0.15) & (m < 0.2)] = -np.inf
    u = x.view(np.uint32)
    nan = (m >= 0.2) & (m < 0.26)
    u[nan] = rng.choice(np.array([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFFFFFFF, 0x7FFFFFFF], np.uint32), nan.sum())
    assert _run(x, K).tobytes() == so.remove_stripes(x, K).tobytes()


def test_in_place_repeats_and_row_splits_give_the_same_bits():
    import torch

    from r2_gaussian_b200.stripes import remove_stripes

    rng = np.random.default_rng(4)
    x = torch.from_numpy(rng.normal(0, 1, (100, 12, 300)).astype(np.float32)).cuda()
    ref = remove_stripes(x, 21)
    assert remove_stripes(x, 21).cpu().numpy().tobytes() == ref.cpu().numpy().tobytes()
    parts = [remove_stripes(x[:, a:b].contiguous(), 21) for a, b in ((0, 1), (1, 5), (5, 12))]
    assert torch.cat(parts, dim=1).cpu().numpy().tobytes() == ref.cpu().numpy().tobytes()
    y = x.clone()
    assert remove_stripes(y, 21, out=y) is y
    assert y.cpu().numpy().tobytes() == ref.cpu().numpy().tobytes()
    assert ref.cpu().numpy()[:, 3].tobytes() == so.remove_stripes(x.cpu().numpy(), 21, rows=[3]).tobytes()


def test_view_limit_is_accepted_and_one_more_refused():
    import torch

    from r2_gaussian_b200.stripes import remove_stripes

    x = torch.from_numpy(np.random.default_rng(5).normal(0, 1, (8192, 2, 3)).astype(np.float32)).cuda()
    assert remove_stripes(x, 5).cpu().numpy().tobytes() == so.remove_stripes(x.cpu().numpy(), 5).tobytes()
    with pytest.raises(ValueError, match="8192"):
        remove_stripes(torch.zeros((8193, 1, 4), device="cuda"), 3)


def test_past_2_31_samples_in_place():
    import torch

    from r2_gaussian_b200.stripes import remove_stripes

    n, H, W = 721, 1600, 1900
    assert n * H * W > 2 ** 31
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn((n, H, W), device="cuda", generator=g)
    rows = [0, 1, 799, 1598, H - 1]
    before = x[:, rows].cpu().numpy()
    remove_stripes(x, 21, out=x)
    got = x[:, rows].cpu().numpy()
    del x
    torch.cuda.empty_cache()
    assert got.tobytes() == so.remove_stripes(before, 21).tobytes()


def test_closed_form_on_the_gpu():
    rng = np.random.default_rng(7)
    clean, striped = clean_with_offsets(rng, 90, 200, 21, 25)
    x = np.stack([striped, striped[::-1]], axis=1)
    want = np.stack([clean, clean[::-1]], axis=1)
    assert _run(x, 21).tobytes() == want.tobytes()


# ---- a striped generate_data scene ---------------------------------------------------------------------------------

def _add_stripes(views, frac, rng, amp):
    """Constant per-pixel offsets, amp * N(0, 1), on `frac` of the detector columns, the same in every view."""
    H, W = views[0].shape
    cols = rng.choice(W, max(1, int(round(frac * W))), replace=False)
    d = np.zeros((H, W), np.float32)
    d[:, cols] = (amp * rng.standard_normal((H, len(cols)))).astype(np.float32)
    return [(v + d).astype(np.float32) for v in views]


@pytest.fixture(scope="module")
def striped_scene(tmp_path_factory):
    from r2_gaussian_b200 import generate_data
    from test_projector_gpu import _write_inputs

    tmp = tmp_path_factory.mktemp("stripes")
    yml, vol_path, *_ = _write_inputs(tmp, noise=False)
    clean = generate_data.main(["--vol", str(vol_path), "--scanner", str(yml), "--n_train", "24", "--n_test", "6",
                                "--output", str(tmp / "clean")])
    with open(os.path.join(clean, "meta_data.json")) as f:
        meta = json.load(f)
    rels = [fr["file_path"] for s in ("proj_train", "proj_test") for fr in meta[s]]
    views = [np.load(os.path.join(clean, r)) for r in rels]
    amp = 0.05 * float(max(v.max() for v in views))
    striped = str(tmp / "striped")
    for r, v in zip(rels, _add_stripes(views, 0.1, np.random.default_rng(8), amp)):
        os.makedirs(os.path.dirname(os.path.join(striped, r)), exist_ok=True)
        np.save(os.path.join(striped, r), v)
    for f in ("meta_data.json", meta["vol"]):
        with open(os.path.join(clean, f), "rb") as a, open(os.path.join(striped, f), "wb") as b:
            b.write(a.read())
    return clean, striped, rels, tmp


def test_scene_cli_end_to_end(striped_scene, capsys):
    import torch

    from r2_gaussian_b200 import initialize_pcd, recon, remove_stripes as rs, trainer
    from r2_gaussian_b200.stripes import remove_stripes

    clean, striped, rels, tmp = striped_scene
    np.save(os.path.join(striped, "init_x.npy"), np.zeros((3, 4), np.float32))
    out = rs.main(["-s", striped, "--output", str(tmp / "fixed")])
    assert "init_x.npy" in capsys.readouterr().out
    assert not os.path.exists(os.path.join(out, "init_x.npy")) and not os.path.exists(os.path.join(out, "proj_all"))
    with open(os.path.join(striped, "meta_data.json"), "rb") as a, open(os.path.join(out, "meta_data.json"), "rb") as b:
        assert a.read() == b.read()
    union = np.stack([np.load(os.path.join(striped, r)) for r in rels]).astype(np.float32)
    want = remove_stripes(torch.from_numpy(union).cuda()).cpu().numpy()           # the default window
    for i, r in enumerate(rels):
        got = np.load(os.path.join(out, r))
        assert got.dtype == np.float32 and got.tobytes() == want[i].tobytes(), r

    scores = {}
    for name, src in (("clean", clean), ("striped", striped), ("fixed", out)):
        scores[name] = recon.main(["-s", src, "-m", str(tmp / f"recon_{name}"), "--methods", "fdk"])["fdk"]["psnr_3d"]
    print(f"fdk psnr_3d: {scores}")
    assert scores["fixed"] > scores["striped"]

    init = initialize_pcd.main(["--data", out, "--n_points", "3000", "--output", str(tmp / "init.npy")])
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    model = trainer.ModelParams(source_path=out, model_path="", ply_path=init)
    hist = trainer.training(model, trainer.OptimizationParams(iterations=200), trainer.PipelineParams(), {200}, set(),
                            log=lambda *a: None)
    assert np.isfinite(hist["eval"][200]["psnr_3d"])


# ---- generate_real_data --remove_stripes on a striped FIPS-format scan -----------------------------------------------

def fips_stripes(raw):
    """The raw views with constant per-pixel offsets (5 % of the largest raw value) on 10 % of the built detector's 64
    columns, each covering the 4 raw columns one built column is made from."""
    amp = 0.05 * float(max(r.max() for r in raw))
    rng = np.random.default_rng(9)
    d = np.zeros_like(raw[0])
    for c in rng.choice(64, 6, replace=False):
        d[:, 4 * c:4 * c + 4] = amp * rng.standard_normal((d.shape[0], 1))
    return [r + d for r in raw]


def test_generate_real_data_removes_stripes_end_to_end(tmp_path):
    import scipy.io
    import torch

    import real_data_oracle as rdo
    from r2_gaussian_b200 import generate_real_data as grd
    from r2_gaussian_b200.metrics import metric_vol
    from r2_gaussian_b200.stripes import remove_stripes
    from test_real_data_gpu import _fips_scan

    scan, phantom = _fips_scan(tmp_path)
    names = sorted(f for f in os.listdir(scan) if f.endswith(".mat"))
    raw = [scipy.io.loadmat(os.path.join(scan, f))["img"] for f in names]
    rdo.write_fips_case(str(tmp_path / "striped"), fips_stripes(raw), 0.0, 4.0, dsd=553.74, dso=410.66, pixel=1.0 / 4)
    args = ["--data", str(tmp_path / "striped"), "--n_train", "30", "--n_test", "20", "--nVoxel", "48", "48", "48"]
    plain = grd.main([*args, "--output", str(tmp_path / "plain")])
    # 3, not the default 5: on this 64-pixel detector a 5-column window loses more than it gains (DESIGN §8)
    fixed = grd.main([*args, "--output", str(tmp_path / "fixed"), "--remove_stripes", "3"])

    stack = grd.prepare_files(sorted(os.path.join(tmp_path / "striped", f) for f in names), 4, 400.0, 50)
    want = remove_stripes(stack, 3).cpu().numpy()
    got = np.stack([np.load(os.path.join(fixed, "proj_all", f.replace(".mat", ".npy"))) for f in names])
    assert got.tobytes() == want.tobytes()
    with open(os.path.join(fixed, "meta_data.json")) as f:
        meta = json.load(f)
    fr = meta["proj_train"][3]
    i = names.index(os.path.basename(fr["file_path"]).replace(".npy", ".mat"))
    assert np.load(os.path.join(fixed, fr["file_path"])).tobytes() == want[i].tobytes()

    psnr = {k: metric_vol(phantom, np.load(os.path.join(p, "vol_gt.npy")), "psnr")[0]
            for k, p in (("plain", plain), ("fixed", fixed))}
    print(f"pseudo-GT psnr_3d against the phantom: {psnr}")
    assert psnr["fixed"] > psnr["plain"]
