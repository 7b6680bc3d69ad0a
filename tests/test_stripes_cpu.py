"""Stripe removal without a GPU: the numpy model (tests/stripe_oracle.py) against sarepy's procedure and its exact
properties, the scratch query, and the refusals of the C ABI, `stripes.remove_stripes` and both CLIs."""
import json
import os

import numpy as np
import pytest

import stripe_oracle as so
from r2_gaussian_b200 import _lib, stripes

pytestmark = pytest.mark.filterwarnings("ignore::RuntimeWarning")


def _finite(rng, n, W, levels=None):
    x = rng.normal(0.0, 1.0, (n, W)).astype(np.float32)
    if levels:                                    # ties within and across columns
        x = np.round(x * levels).astype(np.float32) / np.float32(levels)
    x[x == 0] = np.float32(0.25)                  # no +-0 ties: sarepy's argsort sees them equal, the model does not
    return x


def clean_with_offsets(rng, n, W, K, n_striped):
    """(clean, striped): every column of clean is one profile f(v); striped adds a constant to n_striped columns, placed
    so that no reflected window of K columns holds more than h of them.  Values are multiples of 2^-10: exact sums."""
    h = K // 2
    f = rng.permutation(n).astype(np.float32) / np.float32(1024) + np.float32(1)
    clean = np.repeat(f[:, None], W, axis=1)
    for _ in range(1000):
        cols = rng.choice(W, n_striped, replace=False)
        mark = np.zeros(W, int)
        mark[cols] = 1
        ext = mark[so.reflect_index(W, h)]
        if np.lib.stride_tricks.sliding_window_view(ext, K).sum(axis=1).max() <= h:
            break
    else:
        raise AssertionError("no admissible stripe placement")
    d = np.zeros(W, np.float32)
    d[cols] = rng.integers(-200, 200, n_striped).astype(np.float32) / np.float32(1024)
    d[cols[d[cols] == 0]] = np.float32(1 / 1024)
    return clean, clean + d[None, :]


@pytest.mark.parametrize("n,W,K,levels", [(50, 97, 21, None), (7, 5, 3, None), (33, 40, 11, 4), (16, 3, 7, 2),
                                          (1, 9, 5, None), (64, 64, 129, 8)])
def test_oracle_equals_sarepy_on_finite_data(n, W, K, levels):
    rng = np.random.default_rng(n * 1000 + W + K)
    S = _finite(rng, n, W, levels)
    assert so.sinogram(S, K).tobytes() == so.sarepy(S, K).tobytes()


def test_size_one_is_the_identity_bit_for_bit():
    rng = np.random.default_rng(1)
    x = rng.normal(0, 1, (9, 4, 13)).astype(np.float32)
    x.flat[:8] = [np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-45, -1e-45]
    x.view(np.uint32).flat[8] = 0x7FC12345                           # a NaN with a payload
    assert so.remove_stripes(x, 1).tobytes() == x.tobytes()


def test_view_shuffle_shuffles_the_output():
    rng = np.random.default_rng(2)
    x = rng.permutation(40 * 3 * 30).astype(np.float32).reshape(40, 3, 30) - 600   # distinct values
    p = rng.permutation(40)
    for K in (3, 21):
        assert so.remove_stripes(x[p], K).tobytes() == so.remove_stripes(x, K)[p].tobytes()


def test_power_of_two_scaling_is_exact():
    rng = np.random.default_rng(3)
    x = rng.normal(0, 1, (20, 2, 31)).astype(np.float32)
    for s in (0.25, 8.0, -2.0):
        got = so.remove_stripes(np.float32(s) * x, 5)
        if s > 0:
            assert got.tobytes() == (np.float32(s) * so.remove_stripes(x, 5)).tobytes()
        else:                                                       # a negative scale reverses the order: no claim
            assert np.isin(got, np.float32(s) * x).all()


@pytest.mark.parametrize("n,W,K,n_striped", [(50, 97, 21, 5), (30, 64, 11, 10), (12, 40, 3, 6)])
def test_closed_form_offsets_are_removed_bit_for_bit(n, W, K, n_striped):
    rng = np.random.default_rng(W + K)
    clean, striped = clean_with_offsets(rng, n, W, K, n_striped)
    assert so.sinogram(striped, K).tobytes() == clean.tobytes()
    assert so.sarepy(striped, K).tobytes() == clean.tobytes()


def test_scratch_query_needs_no_gpu():
    lib = _lib.load()
    assert lib.r2x_remove_stripes_scratch_bytes(721, 2368, 2240) == 6 * 721 * 2368 * 2240
    assert lib.r2x_remove_stripes_scratch_bytes(8192, 1, 1) == 6 * 8192
    assert stripes.scratch_bytes(3, 4, 5) == 360
    for bad in [(0, 1, 1), (8193, 1, 1), (1, 0, 1), (1, 1, 0), (1, 1 << 16, 1 << 15), (-1, 5, 5)]:
        assert lib.r2x_remove_stripes_scratch_bytes(*bad) == 0, bad


def _abi(n=4, H=3, W=8, K=3, inp=1 << 20, out=2 << 20, scratch=4 << 20, nbytes=None):
    lib = _lib.load()
    nbytes = 6 * n * H * W if nbytes is None else nbytes
    rc = lib.r2x_remove_stripes(None, n, H, W, K, inp, out, scratch, nbytes)
    return rc, (lib.r2x_last_error() or b"").decode()


@pytest.mark.parametrize("kw,what", [
    (dict(inp=None), "pointer"), (dict(out=None), "pointer"), (dict(scratch=None), "pointer"),
    (dict(n=0), "bad n"), (dict(n=8193), "bad n"), (dict(H=0), "shape"), (dict(W=0), "shape"),
    (dict(H=1 << 16, W=1 << 15, n=1, nbytes=1 << 40), "2^31"),
    (dict(K=0), "bad K"), (dict(K=2), "bad K"), (dict(K=257), "bad K"), (dict(K=-1), "bad K"),
    (dict(W=2, K=7), "h = (K - 1) / 2"), (dict(nbytes=6 * 4 * 3 * 8 - 1), "too small"),
    (dict(scratch=(4 << 20) + 4), "aligned"), (dict(out=(1 << 20) + 4), "overlaps in"),
    (dict(scratch=(1 << 20) + 64), "overlaps in or out"), (dict(scratch=(2 << 20) - 16), "overlaps in or out"),
])
def test_c_abi_refuses_bad_arguments_before_any_cuda_work(kw, what):
    rc, msg = _abi(**kw)
    assert rc == 1 and "r2x_remove_stripes" in msg and what in msg, msg


def test_c_abi_view_limit_and_largest_window_pass_the_checks():
    # the checks that precede CUDA work accept these: the first refusal left is the deliberately short scratch
    assert "too small" in _abi(n=8192, nbytes=0)[1]
    assert "too small" in _abi(W=127, K=255, nbytes=0)[1]
    assert "too small" in _abi(W=1, K=3, nbytes=0)[1]


def test_remove_stripes_refuses_bad_inputs():
    import torch

    with pytest.raises(ValueError, match="CUDA float32"):
        stripes.remove_stripes(np.zeros((2, 2, 2), np.float32))
    with pytest.raises(ValueError, match="CUDA float32"):
        stripes.remove_stripes(torch.zeros((2, 2, 2)))
    for bad in (0, 2, 20, 257, -3, 2.5, True):
        with pytest.raises(ValueError, match="odd integer"):
            stripes.check_size(bad)
    with pytest.raises(ValueError, match="detector width"):
        stripes.check_size(11, 4)
    assert stripes.check_size(9, 4) == 9


def _scene(tmp_path, shapes=((6, 8),) * 4):
    src = tmp_path / "scene"
    (src / "proj_train").mkdir(parents=True)
    (src / "proj_test").mkdir()
    frames = {"proj_train": [], "proj_test": []}
    for i, s in enumerate(shapes):
        split = "proj_train" if i % 2 == 0 else "proj_test"
        rel = f"{split}/{split}_{i:04d}.npy"
        np.save(src / rel, np.ones(s, np.float32))
        frames[split].append({"file_path": rel, "angle": 0.1 * i})
    np.save(src / "vol_gt.npy", np.zeros((4, 4, 4), np.float32))
    (src / "meta_data.json").write_text(json.dumps({"scanner": {}, "vol": "vol_gt.npy", **frames}))
    return src


def test_scene_cli_refusals(tmp_path):
    from r2_gaussian_b200 import remove_stripes as rs

    src = _scene(tmp_path)
    out = str(tmp_path / "out")
    for bad in ("20", "0", "257", "-1"):
        with pytest.raises(ValueError, match="odd integer"):
            rs.main(["-s", str(src), "--output", out, "--size", bad])
    naf = tmp_path / "scan.pickle"
    naf.write_bytes(b"\x80\x04N.")
    with pytest.raises(ValueError, match="NAF pickle"):
        rs.main(["-s", str(naf), "--output", out])
    with pytest.raises(ValueError, match="is the source"):
        rs.main(["-s", str(src), "--output", str(src)])
    taken = tmp_path / "taken"
    taken.mkdir()
    (taken / "meta_data.json").write_text("{}")
    with pytest.raises(ValueError, match="already holds"):
        rs.main(["-s", str(src), "--output", str(taken)])
    with pytest.raises(ValueError, match="share one 2-D shape"):
        rs.main(["-s", str(_scene(tmp_path / "b", ((6, 8), (6, 8), (6, 9)))), "--output", out])
    with pytest.raises(ValueError, match="detector width"):
        rs.main(["-s", str(src), "--output", out, "--size", "19"])
    assert not os.path.exists(out)


def test_generate_real_data_refuses_a_bad_size_before_reading(tmp_path):
    from r2_gaussian_b200 import generate_real_data as grd

    for bad in ("4", "0", "301"):
        with pytest.raises(ValueError, match="odd integer"):
            grd.main(["--data", str(tmp_path / "missing"), "--output", str(tmp_path / "o"), "--remove_stripes", bad])
    assert not os.path.exists(tmp_path / "o")
