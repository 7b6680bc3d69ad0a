"""The training-step edge cases (tests/train_edge_cases.py) without a GPU: each sits on the side of the limit it claims,
with the limits read from the CUDA sources; the float64 statements agree with independent restatements; float32
emulations of the kernels' operation sequences pass the per-element bars, and planted mistakes fail them; the kNN
oracle's subset entry is the full oracle; and the new refusals happen before any CUDA call."""
import ctypes

import numpy as np
import pytest
import torch

import train_edge_cases as te
from oracle import r2_oracle as orc
from r2_gaussian_b200 import _lib

FAKE = ctypes.c_void_p(1 << 20)   # never dereferenced: every call below fails its checks first
f32, f64 = np.float32, np.float64


def test_limits_are_read_from_the_sources():
    k = te.K
    assert (k["LT"], k["LH"], k["LE"], k["IMAGE_LOSS_MAX_H"]) == (16, 5, 26, 65535 * 16)
    assert (k["SSIM_REDUCE_THREADS"], k["TV_REDUCE_THREADS"], k["TV_THREADS"], k["ADAM_THREADS"]) == (1024, 1024, 256, 256)
    assert (k["ADAM_GRID_PER_SM"], k["VIEWS_MAX_N"], k["GATHER_THREADS"], k["GATHER_GRID_PER_SM"]) == (16, 65535, 256, 8)
    assert (k["SCAN_TILE"], k["R2X_ADAM_MAX_GROUPS"], k["R2X_GATHER_MAX_TENSORS"], k["KNN_MAX_G"]) == (1024, 8, 16, 128)
    assert [te.knn_grid(P) for P in (1, 2, 3, 16, 17, 2 * 128 ** 3, 2 * 128 ** 3 + 1)] == [1, 1, 2, 2, 3, 128, 128]


def test_every_case_claims_something():
    for case in te.ALL_CASES.values():
        assert case.claims and case.boundary, case.name


@pytest.mark.parametrize("name", sorted(te.ALL_CASES))
def test_case_lands_where_it_claims(name):
    case = te.ALL_CASES[name]
    assert te.claim_failures(case) == [], (case.boundary, te.claim_failures(case))


def test_sm_claims_move_with_the_device():
    """A case past the grid cap on 132 SMs is not past it on a device with twice as many: the GPU test fails there."""
    assert te.claim_failures(te.ADAM_CASES["adam_past_cap"], 264) != []
    assert te.claim_failures(te.GATHER_CASES["gather_past_cap"], 1024) != []


# ---- image loss -------------------------------------------------------------------------------------------------------

def test_taps_are_the_reference_window():
    """make_window()'s literals are the reference's float32 1-D window (loss_utils.py:45-52, torch's float32 sum)."""
    import math
    g = torch.tensor([math.exp(-((x - 5) ** 2) / float(2 * 1.5 ** 2)) for x in range(11)])
    assert np.array_equal(te.ssim_taps().view(np.uint32), (g / g.sum()).numpy().view(np.uint32))


def _direct_total(x, y, w_l1, w_d):
    """The loss by explicit 2-D loops over the zero-padded window (torch float64 scalars, autograd-able)."""
    g = torch.tensor(te.ssim_taps(), dtype=torch.float64)
    H, W = x.shape
    C1, C2 = 0.01 ** 2, 0.03 ** 2
    s = 0.0
    for i in range(H):
        for j in range(W):
            acc = [0.0] * 5
            for a in range(-5, 6):
                for b in range(-5, 6):
                    if 0 <= i + a < H and 0 <= j + b < W:
                        w = g[a + 5] * g[b + 5]
                        u, v = x[i + a, j + b], y[i + a, j + b]
                        acc = [acc[0] + w * u, acc[1] + w * v, acc[2] + w * u * u, acc[3] + w * v * v, acc[4] + w * u * v]
            m1, m2, e11, e22, e12 = acc
            s = s + ((2 * m1 * m2 + C1) * (2 * (e12 - m1 * m2) + C2)) / (
                (m1 * m1 + m2 * m2 + C1) * (e11 - m1 * m1 + e22 - m2 * m2 + C2))
    return w_l1 * (x - y).abs().mean() + w_d * (1 - s / (H * W)), s / (H * W)


@pytest.mark.parametrize("H,W,content", [(6, 7, "random"), (1, 3, "random"), (4, 4, "identical"), (3, 12, "scaled50")])
def test_ssim_statement_is_the_direct_loops(H, W, content):
    x, y = te.image_pair(H, W, content, H * W)
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    total, s = _direct_total(xt, torch.tensor(y, dtype=torch.float64), 1.0, 0.25)
    total.backward()
    l1, ssim, tot, grad, bound = te.ssim_f64(torch.from_numpy(x), torch.from_numpy(y), 1.0, 0.25)
    assert abs(ssim - s.item()) <= 1e-12 and abs(tot - total.item()) <= 1e-12
    assert torch.allclose(grad, xt.grad, rtol=1e-9, atol=1e-14)
    assert bool((bound > 0).all())


def _fma(a, b, c):
    return (np.asarray(a, f64) * np.asarray(b, f64) + np.asarray(c, f64)).astype(f32)


def _wsum(t, g, axis, n):
    """The kernel's 11-tap pass along `axis` over a zero-padded array: fma in tap order, n outputs."""
    acc = np.zeros(tuple(n if a == axis else s for a, s in enumerate(t.shape)), f32)
    for k in range(11):
        acc = _fma(g[k], np.take(t, np.arange(k, k + n), axis=axis), acc)
    return acc


def ssim_grad_emulated(x, y, w_l1, w_d):
    """The kernels' float32 sequence (ssim_stats_body, ssim_grad_body) in numpy, fma emulated in float64."""
    g, LH = te.ssim_taps(), te.K["LH"]
    H, W = x.shape
    P = lambda t: np.pad(t, LH)                                         # noqa: E731
    conv = lambda t: _wsum(_wsum(P(t), g, 1, W), g, 0, H)              # noqa: E731  horizontal, then vertical
    mu1, mu2, e11, e22, e12 = conv(x), conv(y), conv(x * x), conv(y * y), conv(x * y)
    C1, C2 = f32(0.01) * f32(0.01), f32(0.03) * f32(0.03)
    m1s, m2s, m12 = mu1 * mu1, mu2 * mu2, mu1 * mu2
    s11, s22, s12 = e11 - m1s, e22 - m2s, e12 - m12
    A1, A2, B1, B2 = f32(2) * m12 + C1, f32(2) * s12 + C2, m1s + m2s + C1, s11 + s22 + C2
    inv = f32(1) / (B1 * B2)
    S = A1 * A2 * inv
    M2 = -S / B2
    M3 = f32(2) * A1 * inv
    M1 = f32(2) * mu2 * A2 * inv - f32(2) * mu1 * S / B1 - f32(2) * mu1 * M2 - mu2 * M3
    a, b, d = conv(M1), conv(M2), conv(M3)
    sgn = np.sign(x - y).astype(f32)
    inv_n = f32(1.0 / (H * W))
    return inv_n * (f32(w_l1) * sgn - f32(w_d) * (a + f32(2) * x * b + y * d))


@pytest.mark.parametrize("H,W,content", [(37, 29, "random"), (5, 6, "random"), (33, 17, "scaled50"),
                                         (27, 26, "identical"), (6, 5, "constant")])
def test_ssim_emulation_passes_the_bar_and_a_border_error_fails_it(H, W, content):
    x, y = te.image_pair(H, W, content, 3 * H + W)
    _, _, _, g64, bound = te.ssim_f64(torch.from_numpy(x), torch.from_numpy(y), 1.0, 0.25)
    g64, bar = g64.numpy(), te.SSIM_K * te.U * bound.numpy()
    emu = ssim_grad_emulated(x, y, 1.0, 0.25).astype(f64)
    assert (np.abs(emu - g64) <= bar).all(), float((np.abs(emu - g64) / bar).max())
    if content in ("random", "scaled50") and min(H, W) > 2:
        # 1e-4 max|g| on the border pixels only: inside the old bar (2e-4 max|g|), outside the per-pixel one
        bad = emu.copy()
        border = np.ones_like(bad, bool)
        border[1:-1, 1:-1] = False
        bad[border] += 1e-4 * np.abs(g64).max()
        assert np.abs(bad - g64).max() <= 2e-4 * np.abs(g64).max()
        assert (np.abs(bad - g64) > bar).any()


# ---- image-loss refusals ----------------------------------------------------------------------------------------------

def test_image_loss_refuses_a_grid_taller_than_the_launch_limit():
    lib = _lib.load()
    Hmax = te.K["IMAGE_LOSS_MAX_H"]
    n1 = lib.r2x_image_loss_scratch_bytes(Hmax + 1, 1)
    assert lib.r2x_image_loss(None, Hmax + 1, 1, FAKE, FAKE, 1.0, 0.25, FAKE, FAKE, FAKE, n1) != 0
    err = lib.r2x_last_error()
    assert b"r2x_image_loss" in err and b"H too large" in err, err
    nv = lib.r2x_image_loss_views_scratch_bytes(2, Hmax + 1, 1)
    assert lib.r2x_image_loss_views(None, 2, Hmax + 1, 1, FAKE, FAKE, 1.0, 0.25, FAKE, FAKE, FAKE, nv) != 0
    err = lib.r2x_last_error()
    assert b"r2x_image_loss_views" in err and b"H too large" in err, err
    # H = IMAGE_LOSS_MAX_H passes the H check (and fails the next one, a null scratch)
    assert lib.r2x_image_loss(None, Hmax, 1, FAKE, FAKE, 1.0, 0.25, FAKE, FAKE, None, n1) != 0
    assert b"null pointer" in lib.r2x_last_error()
    assert lib.r2x_image_loss_views(None, 2, Hmax, 1, FAKE, FAKE, 1.0, 0.25, FAKE, FAKE, None, nv) != 0
    assert b"null pointer" in lib.r2x_last_error()


# ---- TV ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 5, 6), (3, 1, 4), (1, 1, 9), (4, 5, 3)])
@pytest.mark.parametrize("mean", [True, False])
def test_tv_statement_is_autograd(shape, mean):
    case = te.Case("t", "tv", "", (), dict(shape=shape), seed=sum(shape))
    v = te.tv_volume(case)
    t = torch.tensor(v, dtype=torch.float64, requires_grad=True)
    tv = sum(t.diff(dim=a).abs().sum() for a in range(3))
    nx, ny, nz = shape
    tot = (nx - 1) * ny * nz + nx * (ny - 1) * nz + nx * ny * (nz - 1)
    loss = tv / tot if mean else tv
    loss.backward()
    want = te.tv_value_f64(v, mean)
    assert (np.isnan(want) and np.isnan(loss.item())) or abs(want - loss.item()) <= 1e-12 * max(1.0, abs(want))
    exact = te.tv_grad_exact(v, mean)
    assert np.array_equal(exact.astype(f64), t.grad.numpy().astype(f32).astype(f64)) or \
        np.abs(exact - t.grad.numpy()).max() <= 2 ** -24 * np.abs(t.grad.numpy()).max()
    if shape == (1, 1, 1):
        assert exact.tolist() == [[[0.0]]] and t.grad.item() == 0.0 and (np.isnan(want) == mean)


# ---- Adam -------------------------------------------------------------------------------------------------------------

B1, B2, EPS = 0.9, 0.999, 1e-15


def adam_emulated(p, m, v, g, lr, step, g2=None, float_one_minus=False, bias_on_v=False):
    """adam_kernel's float32 sequence in numpy (fma emulated in float64); the two planted mistakes: 1 - beta formed in
    float32, and the bias correction of v (1 / bc2) applied to sqrt(v) in place of 1 / sqrt(bc2)."""
    bc1, bc2 = 1.0 - B1 ** step, 1.0 - B2 ** step
    omb1, omb2 = (f32(1) - f32(B1), f32(1) - f32(B2)) if float_one_minus else (f32(1.0 - B1), f32(1.0 - B2))
    isb = f32(1.0 / bc2) if bias_on_v else f32(1.0 / np.sqrt(bc2))
    gs = g + g2 if g2 is not None else g
    m1 = _fma(omb1, gs - m, m)
    v1 = _fma(omb2, gs * gs, f32(B2) * v)
    den = np.sqrt(v1) * isb + f32(EPS)
    ss = f32(lr) * f32(1.0 / bc1)
    return p - ss * (m1 / den), m1, v1


def _adam_fails(got, want, bars):
    return [name for name, a, w, b in zip("pmv", got, want, bars) if not (np.abs(a.astype(f64) - w) <= b).all()]


@pytest.mark.parametrize("grad", te.ADAM_GRADS)
@pytest.mark.parametrize("step", te.ADAM_STEPS)
@pytest.mark.parametrize("two", [False, True])
def test_adam_emulation_passes_the_bars(grad, step, two):
    rng = np.random.RandomState(step)
    p, m, v, g = te.adam_state(3000, grad, rng, step)
    g2 = te.adam_state(3000, grad, rng, step)[3] if two else None
    lr = f32(1e-3)
    with np.errstate(under="ignore"):
        want, bars = te.adam_f64(p, m, v, g, float(lr), B1, B2, EPS, step, g2)
        got = adam_emulated(p, m, v, g, lr, step, g2)
    assert _adam_fails(got, want, bars) == []


@pytest.mark.parametrize("mistake,step,fails", [("float_one_minus", 1, "mv"), ("bias_on_v", 1, "p"),
                                                ("bias_on_v", 10000, "p")])
def test_planted_adam_mistakes_fail_the_bars(mistake, step, fails):
    rng = np.random.RandomState(5)
    p, m, v, g = te.adam_state(3000, "normal", rng, step)
    lr = f32(1e-3)
    want, bars = te.adam_f64(p, m, v, g, float(lr), B1, B2, EPS, step)
    got = adam_emulated(p, m, v, g, lr, step, **{mistake: True})
    assert set(fails) <= set(_adam_fails(got, want, bars))


def test_adam_refuses_more_groups_than_one_launch_takes():
    lib = _lib.load()
    n = te.K["R2X_ADAM_MAX_GROUPS"] + 1
    arr = (_lib.AdamGroup * n)()
    for a in arr:
        a.param = a.grad = a.exp_avg = a.exp_avg_sq = FAKE.value
        a.numel, a.lr = 10, 1e-3
    assert lib.r2x_adam_step(None, n, ctypes.cast(arr, ctypes.c_void_p), B1, B2, EPS, 1) != 0
    assert b"r2x_adam_step: too many groups" in lib.r2x_last_error()
    assert lib.r2x_adam_step_sum(None, n, ctypes.cast(arr, ctypes.c_void_p), None, B1, B2, EPS, 1, None, None) != 0
    assert b"r2x_adam_step: too many groups" in lib.r2x_last_error()


# ---- densification statistics -----------------------------------------------------------------------------------------

def test_densify_statement_is_the_scalar_loop():
    case = te.Case("d", "densify", "", (), dict(P=37, N=4), seed=3)
    radii, grad2d, (mr, acc, den) = te.densify_inputs(case)
    got = te.densify_f32(radii, grad2d, mr, acc, den)
    for i in range(37):
        a, b, c = mr[i], acc[i], den[i]
        for v in range(4):
            if radii[v, i] > 0:
                gx, gy = grad2d[v, i, 0], grad2d[v, i, 1]
                a = max(a, f32(radii[v, i]))
                b = f32(b + f32(np.sqrt(f32(f32(gx * gx) + f32(gy * gy)))))
                c = f32(c + f32(1))
        assert (got[0][i], got[1][i], got[2][i]) == (a, b, c), i
    vis = (radii > 0).sum(0)
    assert (vis[::3] == 0).all() and (vis[1::3] == 4).all() and ((vis > 0) & (vis < 4)).any()


# ---- kNN --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", ["knn_129", "knn_elongated", "knn_lattice"])
def test_knn_subset_oracle_is_the_full_oracle(name):
    pts = te.knn_points(te.KNN_CASES[name])
    full = orc.knn3_mean_dist2(pts)
    idx = te.knn_queries(pts, 300, 1)
    assert len(idx) <= 300
    assert np.array_equal(orc.knn3_mean_dist2_at(pts, idx).view(np.uint32), full[idx].view(np.uint32))
    assert np.array_equal(orc.knn3_mean_dist2_at(pts, np.arange(len(pts))).view(np.uint32), full.view(np.uint32))
    with pytest.raises(IndexError):
        orc.knn3_mean_dist2_at(pts, [len(pts)])
