"""The training-step kernels on the GPU at their edge shapes and launch limits (tests/train_edge_cases.py) against their
float64 or exact statements: the image loss and its gradient per pixel (single and batched), the TV loss and its
gradient bit for bit, one Adam step per element (plain, with a second gradient, through FusedAdam), the densification
statistics bit for bit, row compaction against torch indexing and the 3-NN distances against the brute-force oracle,
bit for bit.  Besides the bars, each checks the exact properties: a batched view is the single-image call bit for bit,
two runs are bitwise equal, a call without a gradient gives the same loss, and a guarded call changes nothing."""
import ctypes

import numpy as np
import pytest

import train_edge_cases as te
from oracle import r2_oracle as orc

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

B1, B2, EPS = 0.9, 0.999, 1e-15


def _lib():
    from r2_gaussian_b200 import _lib as L
    return L, L.load()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _bits(t):
    return t.contiguous().view(torch.int32)


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def test_claims_hold_on_this_device():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    bad = {n: te.claim_failures(c, sms) for n, c in te.ALL_CASES.items()}
    assert {n: f for n, f in bad.items() if f} == {}, sms


# ---- image loss -------------------------------------------------------------------------------------------------------

def image_loss(x, y, w_l1, w_d, grad=True):
    L, lib = _lib()
    H, W = x.shape
    nb = lib.r2x_image_loss_scratch_bytes(H, W)
    scratch = torch.empty(nb, dtype=torch.uint8, device="cuda")
    out = torch.full((3,), float("nan"), device="cuda")
    g = torch.full_like(x, float("nan")) if grad else None
    L.check(lib.r2x_image_loss(_st(), H, W, _p(x), _p(y), w_l1, w_d, _p(out), _p(g), _p(scratch), nb), "r2x_image_loss")
    return out, g


def image_loss_views(x, y, w_l1, w_d, grad=True):
    L, lib = _lib()
    N, H, W = x.shape
    nb = lib.r2x_image_loss_views_scratch_bytes(N, H, W)
    scratch = torch.empty(nb, dtype=torch.uint8, device="cuda")
    out = torch.full((N, 3), float("nan"), device="cuda")
    g = torch.full_like(x, float("nan")) if grad else None
    L.check(lib.r2x_image_loss_views(_st(), N, H, W, _p(x), _p(y), w_l1, w_d, _p(out), _p(g), _p(scratch), nb),
            "r2x_image_loss_views")
    return out, g


def _check_against_f64(x, y, lam, out, grad, what):
    """The existing value bars of test_image_loss_matches_torch and the per-pixel gradient bar of te.ssim_f64."""
    from test_train_gpu import torch_ssim
    l1, s64, total, g64, bound = te.ssim_f64(x, y, 1.0, lam)
    tf32 = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    s32 = torch_ssim(x[None], y[None]).item()
    torch.backends.cudnn.allow_tf32 = tf32
    bar = max(5e-6, 3.0 * abs(s32 - s64))
    got_l1, got_s, got_t = (float(v) for v in out.tolist())
    assert abs(got_s - s64) <= bar, (what, got_s, s64, bar)
    assert abs(got_t - total) <= 2e-6 * max(1.0, abs(total)) + lam * bar, (what, got_t, total)
    # mean|x - y|: float32 per-CTA sums of 256 terms (a 5-level shuffle tree, then 8 warps in order: 13 roundings) and
    # one rounding each of the difference and the result: 15 u of the mean, or the existing 1e-6 where that is larger
    assert abs(got_l1 - l1) <= max(1e-6, 15 * te.U * l1), (what, got_l1, l1)
    err = (grad.double() - g64).abs()
    lim = te.SSIM_K * te.U * bound
    worst = (err / lim).max().item()
    assert bool((err <= lim).all()), (what, worst, int((err > lim).sum()))


def _pair(case, n=None):
    x, y = te.image_pair(case.q["H"], case.q["W"], case.content, case.seed, n)
    return torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()


@pytest.mark.parametrize("lam", [0.25, 0.0])
@pytest.mark.parametrize("name", sorted(te.IMAGE_CASES))
def test_image_loss_case(name, lam):
    case = te.IMAGE_CASES[name]
    x, y = _pair(case)
    out, g = image_loss(x, y, 1.0, lam)
    _check_against_f64(x, y, lam, out, g, name)
    out2, g2 = image_loss(x, y, 1.0, lam)
    assert torch.equal(_bits(out), _bits(out2)) and torch.equal(_bits(g), _bits(g2))
    out3, _ = image_loss(x, y, 1.0, lam, grad=False)
    assert torch.equal(_bits(out), _bits(out3))
    if case.content == "identical" and lam == 0.0:
        assert bool((g == 0).all())                                   # sign(0) = 0
    # view 0 of a batched call (its second image different) is the single-image call
    xs, ys = torch.stack([x, y.flip(0)]), torch.stack([y, x])
    ov, gv = image_loss_views(xs, ys, 1.0, lam)
    assert torch.equal(_bits(ov[0]), _bits(out)) and torch.equal(_bits(gv[0]), _bits(g))
    o1, g1 = image_loss(xs[1].contiguous(), ys[1].contiguous(), 1.0, lam)
    assert torch.equal(_bits(ov[1]), _bits(o1)) and torch.equal(_bits(gv[1]), _bits(g1))


@pytest.mark.parametrize("name", sorted(te.VIEWS_CASES))
def test_image_loss_views_case(name):
    case = te.VIEWS_CASES[name]
    N = case.q["N"]
    x, y = _pair(case, N)
    out, g = image_loss_views(x, y, 1.0, 0.25)
    out_n, _ = image_loss_views(x, y, 1.0, 0.25, grad=False)
    assert torch.equal(_bits(out), _bits(out_n))
    check = range(N) if N <= 7 else (0, N // 2, N - 1)
    for v in check:
        o1, g1 = image_loss(x[v].contiguous(), y[v].contiguous(), 1.0, 0.25)
        assert torch.equal(_bits(out[v]), _bits(o1)) and torch.equal(_bits(g[v]), _bits(g1)), v
        if N <= 7:
            _check_against_f64(x[v], y[v], 0.25, out[v], g[v], (name, v))
    assert bool(torch.isfinite(out).all()) and bool(torch.isfinite(g).all())


# ---- TV ---------------------------------------------------------------------------------------------------------------

def tv3d(vol, mean, grad=True):
    L, lib = _lib()
    nx, ny, nz = vol.shape
    nb = lib.r2x_tv3d_scratch_bytes(nx, ny, nz)
    scratch = torch.empty(nb, dtype=torch.uint8, device="cuda")
    out = torch.full((1,), -1.0, device="cuda")
    g = torch.full_like(vol, float("nan")) if grad else None
    L.check(lib.r2x_tv3d_loss(_st(), nx, ny, nz, _p(vol), int(mean), _p(out), _p(g), _p(scratch), nb), "r2x_tv3d_loss")
    return out, g


@pytest.mark.parametrize("mean", [True, False])
@pytest.mark.parametrize("name", sorted(te.TV_CASES))
def test_tv_case(name, mean):
    case = te.TV_CASES[name]
    v = te.tv_volume(case)
    vol = torch.from_numpy(v).cuda()
    out, g = tv3d(vol, mean)
    want = te.tv_value_f64(v, mean)
    got = out.item()
    if np.isnan(want):
        assert np.isnan(got)
    else:
        assert abs(got - want) <= 2e-6 * max(1.0, abs(want)), (got, want)
    exact = te.tv_grad_exact(v, mean)
    assert np.array_equal(g.cpu().numpy().view(np.uint32), exact.view(np.uint32)), \
        int((g.cpu().numpy() != exact).sum())
    out2, _ = tv3d(vol, mean, grad=False)
    assert torch.equal(_bits(out), _bits(out2))


# ---- Adam -------------------------------------------------------------------------------------------------------------

def _adam_groups(case):
    """Per group (p, m, v, g, g2-or-None, lr) as float32 numpy: odd groups of the `_sum` form take no second gradient."""
    rng = np.random.RandomState(case.seed)
    step = case.q["step"]
    out = []
    for i, n in enumerate(case.q["numels"]):
        p, m, v, g = te.adam_state(n, case.content, rng, step)
        g2 = te.adam_state(n, case.content, rng, step)[3] if i % 2 == 0 else None
        out.append((p, m, v, g, g2, np.float32(10.0 ** -(2 + i % 3))))
    return out


def _adam_call(groups, step, form, guard=None):
    L, lib = _lib()
    dev = [tuple(torch.from_numpy(a.copy()).cuda() if a is not None else None for a in gr[:5]) for gr in groups]
    arr = (L.AdamGroup * len(groups))()
    g2s = (ctypes.c_void_p * len(groups))()
    for k, ((p, m, v, g, g2), gr) in enumerate(zip(dev, groups)):
        arr[k].param, arr[k].grad, arr[k].exp_avg, arr[k].exp_avg_sq = (t.data_ptr() for t in (p, g, m, v))
        arr[k].numel, arr[k].lr = p.numel(), float(gr[5])
        g2s[k] = g2.data_ptr() if (g2 is not None and form == "sum") else None
    a = ctypes.cast(arr, ctypes.c_void_p)
    if form == "plain":
        rc = lib.r2x_adam_step(_st(), len(groups), a, B1, B2, EPS, step)
    else:
        grads2 = ctypes.cast(g2s, ctypes.c_void_p) if form == "sum" else None
        rc = lib.r2x_adam_step_sum(_st(), len(groups), a, grads2, B1, B2, EPS, step, _p(guard), None)
    L.check(rc, "r2x_adam_step")
    return [tuple(t.cpu().numpy() for t in d[:3]) for d in dev]


def _assert_adam(groups, got, step, use_g2, what):
    for i, ((p, m, v, g, g2, lr), (gp, gm, gv)) in enumerate(zip(groups, got)):
        with np.errstate(under="ignore"):
            want, bars = te.adam_f64(p, m, v, g, float(lr), B1, B2, EPS, step, g2 if use_g2 else None)
        for name, a, w, b in zip("pmv", (gp, gm, gv), want, bars):
            err = np.abs(a.astype(np.float64) - w)
            assert (err <= b).all(), (what, i, name, int((err > b).sum()), float((err / b).max()))


@pytest.mark.parametrize("name", [n for n, c in sorted(te.ADAM_CASES.items()) if c.kind == "adam"])
def test_adam_case(name):
    case = te.ADAM_CASES[name]
    groups, step = _adam_groups(case), case.q["step"]
    plain = _adam_call(groups, step, "plain")
    _assert_adam(groups, plain, step, False, name)
    summed = _adam_call(groups, step, "sum")
    _assert_adam(groups, summed, step, True, name)
    # grads2 = NULL is r2x_adam_step bit for bit; an overflow word set changes nothing
    nul = _adam_call(groups, step, "null")
    for a, b in zip(plain, nul):
        assert all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(a, b))
    guard = torch.tensor([5, 1], dtype=torch.int32, device="cuda")
    kept = _adam_call(groups, step, "sum", guard)
    for gr, k in zip(groups, kept):
        assert all(np.array_equal(x.view(np.uint32), y.view(np.uint32)) for x, y in zip(gr[:3], k))


@pytest.mark.parametrize("name", [n for n, c in sorted(te.ADAM_CASES.items()) if c.kind == "fused_adam"])
def test_fused_adam_case(name):
    """8, 9 and 17 parameters: one, two and three launches; two steps, each against float64 from its own state."""
    from r2_gaussian_b200.optim import FusedAdam
    case = te.ADAM_CASES[name]
    rng = np.random.RandomState(case.seed)
    params = [torch.nn.Parameter(torch.from_numpy(rng.normal(0, 1, n).astype(np.float32)).cuda())
              for n in case.q["numels"]]
    lrs = [float(np.float32(10.0 ** -(2 + i % 3))) for i in range(len(params))]
    opt = FusedAdam([{"params": [p], "lr": lr} for p, lr in zip(params, lrs)], lr=0.0, eps=EPS)
    for step in (1, 2):
        groups = []
        for p, lr in zip(params, lrs):
            g = rng.normal(0, 1, p.numel()).astype(np.float32)
            p.grad = torch.from_numpy(g).cuda()
            st = opt.state[p]
            m = st["exp_avg"].cpu().numpy() if st else np.zeros(p.numel(), np.float32)
            v = st["exp_avg_sq"].cpu().numpy() if st else np.zeros(p.numel(), np.float32)
            groups.append((p.detach().cpu().numpy(), m, v, g, None, np.float32(lr)))
        opt.step()
        got = [(p.detach().cpu().numpy(), opt.state[p]["exp_avg"].cpu().numpy(), opt.state[p]["exp_avg_sq"].cpu().numpy())
               for p in params]
        _assert_adam(groups, got, step, False, (name, step))


def test_fused_adam_4M_25_steps_against_torch_adam():
    from r2_gaussian_b200.optim import FusedAdam
    torch.manual_seed(0)
    n = te.ADAM_CASES["adam_4M"].q["numels"][0]
    p_ref = [torch.nn.Parameter(torch.randn(n, device="cuda")), torch.nn.Parameter(torch.randn(1000, device="cuda"))]
    p_our = [torch.nn.Parameter(p.detach().clone()) for p in p_ref]
    lrs = [1e-3, 1e-2]
    o_ref = torch.optim.Adam([{"params": [p], "lr": lr} for p, lr in zip(p_ref, lrs)], lr=0.0, eps=EPS)
    o_our = FusedAdam([{"params": [p], "lr": lr} for p, lr in zip(p_our, lrs)], lr=0.0, eps=EPS)
    for it in range(25):
        for pr, po in zip(p_ref, p_our):
            g = torch.randn_like(pr) * (0.1 + it)
            g[::7] = 0.0
            pr.grad, po.grad = g.clone(), g.clone()
        o_ref.step()
        o_our.step()
    for pr, po in zip(p_ref, p_our):
        assert (pr - po).abs().max().item() <= 2e-6 * pr.abs().max().item()
        for k in ("exp_avg", "exp_avg_sq"):
            a, b = o_ref.state[pr][k], o_our.state[po][k]
            assert (a - b).abs().max().item() <= 2e-6 * a.abs().max().item(), k


# ---- densification statistics -----------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(te.DENSIFY_CASES))
def test_densify_case(name):
    L, lib = _lib()
    case = te.DENSIFY_CASES[name]
    radii, grad2d, stats = te.densify_inputs(case)
    N, P = radii.shape
    want = te.densify_f32(radii, grad2d, *stats)
    r, g2 = torch.from_numpy(radii).cuda(), torch.from_numpy(grad2d).cuda()
    eq = lambda a, w: np.array_equal(a.cpu().numpy().view(np.uint32), w.view(np.uint32))   # noqa: E731
    # the batched kernel, and N single-view launches in view order
    got = [torch.from_numpy(s.copy()).cuda() for s in stats]
    L.check(lib.r2x_densify_stats_views(_st(), N, P, _p(r), _p(g2), *(_p(t) for t in got), None, None), "views")
    assert all(eq(a, w) for a, w in zip(got, want))
    seq = [torch.from_numpy(s.copy()).cuda() for s in stats]
    for v in range(N):
        L.check(lib.r2x_densify_stats(_st(), P, _p(r[v]), _p(g2[v]), *(_p(t) for t in seq), None, None), "single")
    assert all(eq(a, w) for a, w in zip(seq, want))
    # a set overflow word in either guard, or both, changes nothing
    ok = torch.tensor([3, 0], dtype=torch.int32, device="cuda")
    bad = torch.tensor([3, 1], dtype=torch.int32, device="cuda")
    for g0, g1 in ((bad, None), (None, bad), (bad, bad), (ok, bad)):
        kept = [torch.from_numpy(s.copy()).cuda() for s in stats]
        L.check(lib.r2x_densify_stats_views(_st(), N, P, _p(r), _p(g2), *(_p(t) for t in kept), _p(g0), _p(g1)), "g")
        L.check(lib.r2x_densify_stats(_st(), P, _p(r[0]), _p(g2[0]), *(_p(t) for t in kept), _p(g0), _p(g1)), "g")
        assert all(eq(a, s) for a, s in zip(kept, stats))


# ---- row compaction ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(te.MASK_CASES))
def test_mask_select_case(name):
    from r2_gaussian_b200 import compact
    mask = torch.from_numpy(te.mask_bytes(te.MASK_CASES[name])).cuda()
    idx, count = compact.select_rows(mask)
    want = torch.nonzero(mask).flatten().to(torch.int32)
    k = int(count.item())
    assert k == want.numel()
    assert torch.equal(idx[:k], want)


def _gather_inputs(case):
    rng = np.random.RandomState(case.seed)
    layout, rows = te.gather_rows_n0(case)
    src = []
    for (n0, n1, has1), w in zip(layout, case.q["widths"]):
        a = torch.from_numpy(rng.normal(0, 1, (n0, w)).astype(np.float32)).cuda()
        b = torch.from_numpy(rng.normal(0, 1, (n1, w)).astype(np.float32)).cuda() if has1 else None
        full = torch.cat([a, b if b is not None else torch.zeros(n1, w, device="cuda")])
        src.append((a, b, full))
    nsel = case.q["nsel"]
    sel = None if nsel is None else torch.from_numpy(rng.randint(0, rows, nsel).astype(np.int32)).cuda()
    return src, sel, rows if nsel is None else nsel


@pytest.mark.parametrize("name", sorted(te.GATHER_CASES))
def test_gather_rows_case(name):
    L, lib = _lib()
    case = te.GATHER_CASES[name]
    src, sel, nsel = _gather_inputs(case)
    want = [full[:nsel] if sel is None else full[sel.long()] for _, _, full in src]
    if len(src) > te.K["R2X_GATHER_MAX_TENSORS"]:             # compact.gather_rows splits it into launches
        from r2_gaussian_b200 import compact
        got = compact.gather_rows([(a, b) for a, b, _ in src], sel, nsel)
    else:
        got = [torch.full((nsel, full.shape[1]), float("nan"), device="cuda") for _, _, full in src]
        arr = (L.GatherDesc * len(src))()
        for k, ((a, b, _), out) in enumerate(zip(src, got)):
            arr[k].src0 = a.data_ptr() if a.shape[0] else None
            arr[k].src1 = b.data_ptr() if b is not None else None
            arr[k].dst, arr[k].n0, arr[k].width = out.data_ptr(), a.shape[0], out.shape[1]
        L.check(lib.r2x_gather_rows(_st(), len(src), ctypes.cast(arr, ctypes.c_void_p), _p(sel), nsel), "gather")
    for k, (a, w) in enumerate(zip(got, want)):
        assert torch.equal(_bits(a), _bits(w)), k


# ---- kNN --------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(te.KNN_CASES))
def test_knn_case(name):
    from simple_knn._C import distCUDA2
    case = te.KNN_CASES[name]
    pts = te.knn_points(case)
    got = distCUDA2(torch.from_numpy(pts).cuda()).cpu().numpy()
    if len(pts) <= te.KNN_BRUTE_MAX:
        want, idx = orc.knn3_mean_dist2(pts), np.arange(len(pts))
    else:
        idx = te.knn_queries(pts, te.KNN_QUERIES, case.seed)
        want = orc.knn3_mean_dist2_at(pts, idx)
    assert np.array_equal(got[idx].view(np.uint32), want.view(np.uint32)), (
        int((got[idx] != want).sum()), float(np.abs(got[idx] - want).max()))
