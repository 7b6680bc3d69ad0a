"""The Gaussian-sharded GPU path against a single-process truth, bit for bit.

Ranks are spawned processes in a gloo process group with CUDA tensors; with one device they all share it.  The truth
runs in the pytest process without a process group: per shard, the single-GPU entry points, with the shard images (and
TV volumes) summed in rank order.  Two ranks add each element once, and an empty shard adds +0.0, so the gloo sum is
exact in any order and every comparison is of bits:

* render() / query() after sharded.enable(): image and volume on every rank equal the rank-ordered sum of the shards
  rendered alone, each rank's gradients equal its own shard's; the summed image lies within the float64 statement's
  bar (forward_float64.py) of the whole cloud;
* NativeTrainStep on shards: parameters, Adam moments and steps, max_radii2D and denom equal the autograd iteration over
  the list of shard models, in a cone-beam and a 127 x 125 parallel-beam case, with and without TV, across a
  densification that leaves the ranks with different numbers of Gaussians, with one rank starved of instance capacity
  (the overflow flag that rides with the image makes every rank skip and repeat), and with an empty shard;
* over peer memory (r2x_peer_allreduce_sum between two devices), when two peer-capable GPUs are visible.

Each shard's model is built the way the trainer builds it: 3-NN distances of the full point set, then
shard_init_points and create_from_pcd(dist2=...).  A collective mismatch fails within the 60 s gloo time-out; every
worker is terminated and joined before a test returns."""
import os
import queue
import socket
import time
import traceback
import types
from datetime import timedelta

import numpy as np
import pytest

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

SCALE_BOUND = (0.0005, 0.5)
N_POINTS = 5000
LAM_D, LAM_TV = 0.25, 0.05
TV_N, TV_S = [32, 32, 32], [0.5, 0.5, 0.5]
PIPE = types.SimpleNamespace(compute_cov3D_python=False, debug=False)
RUN_TIMEOUT_S = 300


# ---- scenes (built identically in the workers and the truth) -------------------------------------------------------
def init_points(n=N_POINTS, seed=11):
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(-0.8, 0.8, size=(n, 3))
    dens = rng.uniform(0.05, 0.9, size=(n, 1))
    return np.concatenate([xyz, dens], axis=1).astype(np.float32)


def full_dist2(points):
    """Mean squared 3-NN distances of the FULL point set (the trainer's order: before sharding)."""
    from r2_gaussian_b200.simple_knn import distCUDA2
    return distCUDA2(torch.as_tensor(points[:, :3]).float().cuda()).cpu().numpy()


def shard_model(points, dist2, rank, world):
    from r2_gaussian_b200.gaussian_model import GaussianModel
    from r2_gaussian_b200.sharded import shard_init_points
    from test_train_gpu import _opt_args
    pts, d2 = shard_init_points(points, dist2, rank, world)
    gm = GaussianModel(SCALE_BOUND)
    gm.create_from_pcd(pts[:, :3], pts[:, 3:4], 1.0, dist2=d2)
    gm.training_setup(_opt_args())
    return gm


def train_inputs(beam):
    """test_train_gpu._train_inputs for the cone beam; the same four angles on a 127 x 125 parallel-beam detector."""
    from r2_gaussian_b200 import scene
    from test_train_gpu import _train_inputs
    if beam == "cone":
        return _train_inputs()
    sc = scene.parallel_beam_scanner(128, 64)
    sc["nDetector"] = [125, 127]
    cams = [scene.camera_from_view(scene.make_view(sc, 0.3 + 0.9 * k)) for k in range(4)]
    g = torch.Generator("cuda").manual_seed(9)
    gts = [torch.rand((1, 125, 127), device="cuda", generator=g) * 0.5 for _ in cams]
    centres = [(0.1 * k - 0.15, 0.05 * k, -0.1 + 0.07 * k) for k in range(4)]
    return cams, gts, centres


def fixed_grads(H, W, seed=21):
    g = torch.Generator("cuda").manual_seed(seed)
    return (torch.randn((1, H, W), device="cuda", generator=g),
            torch.randn(tuple(TV_N), device="cuda", generator=g))


_GROUPS = (("xyz", "_xyz"), ("density", "_density"), ("scaling", "_scaling"), ("rotation", "_rotation"))


def model_state(gm):
    """Everything a training iteration changes: parameters, both Adam moments, step counts and the statistics."""
    out = {}
    for name, attr in _GROUPS:
        p = getattr(gm, attr)
        st = gm.optimizer.state[p]
        out[name] = p.detach().cpu().numpy()
        out[name + "_exp_avg"] = st["exp_avg"].cpu().numpy()
        out[name + "_exp_avg_sq"] = st["exp_avg_sq"].cpu().numpy()
        out[name + "_step"] = np.array(float(st["step"]))
    out["max_radii2D"] = gm.max_radii2D.cpu().numpy()
    out["xyz_gradient_accum"] = gm.xyz_gradient_accum.cpu().numpy()
    out["denom"] = gm.denom.cpu().numpy()
    return out


def restore_model(state):
    """A GaussianModel holding `state` (model_state's dictionary): the truth restarts from a worker's saved state."""
    from r2_gaussian_b200.gaussian_model import GaussianModel
    from test_train_gpu import _opt_args
    gm = GaussianModel(SCALE_BOUND)
    n = state["xyz"].shape[0]
    gm.create_from_pcd(state["xyz"], np.full((n, 1), 0.5, np.float32), 1.0, dist2=np.ones(n, np.float32))
    gm.training_setup(_opt_args())
    with torch.no_grad():
        for name, attr in _GROUPS:
            p = getattr(gm, attr)
            p.copy_(torch.from_numpy(state[name]))
            gm.optimizer.state[p] = {"step": torch.tensor(float(state[name + "_step"]), dtype=torch.float32),
                                     "exp_avg": torch.from_numpy(state[name + "_exp_avg"]).cuda(),
                                     "exp_avg_sq": torch.from_numpy(state[name + "_exp_avg_sq"]).cuda()}
    gm.max_radii2D = torch.from_numpy(state["max_radii2D"]).cuda()
    gm.xyz_gradient_accum = torch.from_numpy(state["xyz_gradient_accum"]).cuda()
    gm.denom = torch.from_numpy(state["denom"]).cuda()
    return gm


def _snapshot(gm):
    ts = [gm.max_radii2D, gm.xyz_gradient_accum, gm.denom]
    for _, attr in _GROUPS:
        p = getattr(gm, attr)
        ts += [p.detach(), gm.optimizer.state[p]["exp_avg"], gm.optimizer.state[p]["exp_avg_sq"]]
    return [t.clone() for t in ts]


# ---- worker jobs ----------------------------------------------------------------------------------------------------
def job_render(rank, world, points, dist2, beam):
    """render() + query() of this rank's shard after sharded.enable(), and the backward of one fixed dL/dimage, dL/dvol."""
    from r2_gaussian_b200.render_query import query, render
    gm = shard_model(points, dist2, rank, world)
    cams, _, centres = train_inputs(beam)
    pkg = render(cams[1], gm, PIPE)
    vol = query(gm, centres[1], TV_N, TV_S, PIPE)["vol"]
    dLi, dLv = fixed_grads(int(cams[1].image_height), int(cams[1].image_width))
    ((pkg["render"] * dLi).sum() + (vol * dLv).sum()).backward()
    out = {"image": pkg["render"].detach().cpu().numpy(), "vol": vol.detach().cpu().numpy(),
           "radii": pkg["radii"].cpu().numpy(), "g_means2D": pkg["viewspace_points"].grad.cpu().numpy()}
    for name, attr in _GROUPS:
        out["g_" + name] = getattr(gm, attr).grad.cpu().numpy()
    return out


def _starve(step, which):
    """One page of instances for the raster or the voxel forward, kept for the next call (test_native_train_step_repeats_
    an_overflowed_iteration's recipe, for one forward)."""
    from r2_gaussian_b200 import _C
    lib = step.lib
    if which == "raster":
        step.cap_r = 4096
        step.binning_r = torch.empty(lib.r2x_binning_bytes(4096), dtype=torch.uint8, device="cuda")
        step.scratch_r = torch.empty(lib.r2x_raster_bwd_scratch_bytes(4096), dtype=torch.uint8, device="cuda")
        _C._Workspace.hints[step.key_r] = 1
    else:
        step.cap_v = 4096
        step.binning_v = torch.empty(lib.r2x_binning_bytes(4096), dtype=torch.uint8, device="cuda")
        step.scratch_v = torch.empty(lib.r2x_voxel_bwd_scratch_bytes(4096), dtype=torch.uint8, device="cuda")
        _C._Workspace.hints[step.key_v] = 1
    step._provision = lambda: None


def _densify(gm, rank):
    """densify_and_prune with thresholds taken from this rank's statistics, so that it clones, splits and prunes some
    Gaussians, and differently on every rank.  -> (clones, splits, pruned)."""
    grads = gm.xyz_gradient_accum / gm.denom
    grads = torch.where(grads.isnan(), torch.zeros_like(grads), grads).squeeze(-1)
    max_grad = float(torch.quantile(grads[grads > 0], 0.80 + 0.05 * rank))
    max_s = gm.get_scaling.max(dim=1).values
    hot = grads >= max_grad
    thr = float(torch.quantile(max_s[hot], 0.5))
    min_density = float(torch.quantile(gm.get_density.detach().squeeze(-1), 0.03))
    n0 = int(gm._xyz.shape[0])
    n_clone, n_split = int((hot & (max_s <= thr)).sum()), int((hot & (max_s > thr)).sum())
    with torch.no_grad():
        gm.densify_and_prune(max_grad, min_density, None, None, None, thr, None)
    pruned = n0 + n_clone + n_split - int(gm._xyz.shape[0])
    return n_clone, n_split, pruned


def job_train(rank, world, points, dist2, beam, use_tv, n_it=7, densify_at=None, starve_rank=None, starve_at=None,
              starve=None, empty_rank=None):
    """n_it iterations of NativeTrainStep on this rank's shard; optionally densify after iteration `densify_at`, starve
    rank `starve_rank`'s `starve` forward ("raster" or "voxel") of capacity at iteration `starve_at`, or empty rank
    `empty_rank`'s shard before the first."""
    from r2_gaussian_b200.train_step import NativeTrainStep
    gm = shard_model(points, dist2, rank, world)
    if rank == empty_rank:
        gm.prune_points(torch.ones(gm._xyz.shape[0], dtype=torch.bool, device="cuda"))
        assert gm._xyz.shape[0] == 0
    cams, gts, centres = train_inputs(beam)
    step = NativeTrainStep(gm, LAM_D, LAM_TV if use_tv else 0.0, TV_N, TV_S)
    out = {}
    for i in range(1, n_it + 1):
        k = i % len(cams)
        gm.update_learning_rate(i)
        if i == starve_at:
            step.flush()
            if rank == starve_rank:
                _starve(step, starve)
            before = _snapshot(gm)
            step(cams[k], gts[k], centres[k])
            torch.cuda.synchronize()
            out["starved_unchanged"] = np.array([torch.equal(a, b) for a, b in zip(before, _snapshot(gm))])
            if rank == starve_rank:
                del step._provision
                step.cap_r = step.cap_v = 0
            step.flush()                                        # notices the overflow, repeats the iteration
            out["repeats_after_starve"] = np.array(step.repeats)
        else:
            res = step(cams[k], gts[k], centres[k])
        if i == n_it:
            out["loss"] = np.array(step.total_loss())
            out["image"] = res["render"].cpu().numpy()
            if use_tv:
                out["vol"] = step.vol.cpu().numpy()
        if i == densify_at:
            step.flush()
            out.update({"pre_" + key: v for key, v in model_state(gm).items()})
            out["densified"] = np.array(_densify(gm, rank))
            out.update({"post_" + key: v for key, v in model_state(gm).items()})
    step.flush()
    out["repeats"] = np.array(step.repeats)
    out.update(model_state(gm))
    return out


def job_peer_epochs(rank, world, n=512 * 512, epochs=40):
    """PeerReducer over `epochs` epochs: each epoch's output and the gathered partials (their rank-ordered sum is
    taken by the parent)."""
    import torch.distributed as dist
    from r2_gaussian_b200.peer import PeerReducer
    dev = torch.device("cuda", torch.cuda.current_device())
    red = PeerReducer(n, dev)
    outs, parts = [], []
    out = torch.empty(n, device=dev)
    for ep in range(epochs):
        mine = torch.randn(n, device=dev, generator=torch.Generator(dev).manual_seed(1000 * ep + rank)) * (1 + rank)
        red.partial().copy_(mine)
        red.reduce(out)
        gathered = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(gathered, mine)
        outs.append(out.cpu().numpy())
        parts.append(np.stack([g.cpu().numpy() for g in gathered]))
    ok = red.ok()
    red.close()
    return {"outs": np.stack(outs), "parts": np.stack(parts), "ok": np.array(ok)}


JOBS = {"render": job_render, "train": job_train, "peer_epochs": job_peer_epochs}


def _worker(rank, world, port, job, kw, peer, out_dir, q):
    import torch.distributed as dist
    from r2_gaussian_b200 import sharded
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    try:
        torch.cuda.set_device(rank % torch.cuda.device_count())
        dist.init_process_group("gloo", rank=rank, world_size=world, timeout=timedelta(seconds=60))
        try:
            sharded.enable()
            if peer:
                sharded.enable_peer_exchange(True)
            res = JOBS[job](rank, world, **kw)
            if peer:
                sharded.check_peer_exchange()
                sharded.enable_peer_exchange(False)
            np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **res)
        finally:
            sharded.enable(on=False)
            dist.destroy_process_group()
        q.put((rank, "ok"))
    except BaseException:
        q.put((rank, traceback.format_exc()))
        raise


def _free_port():
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def run_world(tmp_path, world, job, peer=False, **kw):
    """Run JOBS[job] on `world` spawned ranks; -> each rank's results.  Fails on the first rank that reports an error
    or when the ranks do not finish within RUN_TIMEOUT_S; every worker is terminated and joined before returning."""
    import multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    out_dir = tmp_path / f"{job}_{world}_{time.monotonic_ns()}"
    out_dir.mkdir()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, job, kw, peer, str(out_dir), q), daemon=True)
             for r in range(world)]
    try:
        for p in procs:
            p.start()
        deadline = time.monotonic() + RUN_TIMEOUT_S
        done = {}
        while len(done) < world:
            try:
                rank, msg = q.get(timeout=max(deadline - time.monotonic(), 0.1))
            except queue.Empty:
                pytest.fail(f"{job}: ranks {sorted(set(range(world)) - set(done))} did not finish in {RUN_TIMEOUT_S} s")
            if msg != "ok":
                pytest.fail(f"{job}: rank {rank} failed:\n{msg}")
            done[rank] = msg
        for p in procs:
            p.join(timeout=max(deadline - time.monotonic(), 5.0))
            assert p.exitcode == 0, f"{job}: a worker exited with {p.exitcode}"
    finally:
        started = [p for p in procs if p.pid is not None]      # an interrupt can land between two starts
        for p in started:
            if p.is_alive():
                p.terminate()
        for p in started:
            p.join(timeout=10)
            if p.is_alive():
                p.kill()
                p.join()
        q.close()
        q.join_thread()
    return [dict(np.load(out_dir / f"rank{r}.npz")) for r in range(world)]


# ---- the truth ------------------------------------------------------------------------------------------------------
def truth_iteration(models, cam, gt, centre, i, use_tv):
    """test_native_train_step_is_the_autograd_iteration's iteration over a list of shard models: the shard images (and
    TV volumes) summed in rank order before the loss.  -> (total loss, summed image, summed volume or None)."""
    from r2_gaussian_b200 import losses
    from r2_gaussian_b200.render_query import query, render
    for m in models:
        m.update_learning_rate(i)
    pkgs = [render(cam, m, PIPE) for m in models]
    image = pkgs[0]["render"]
    for p in pkgs[1:]:
        image = image + p["render"]
    total = losses.image_loss(image, gt, LAM_D)["total"]
    vol = None
    if use_tv:
        vols = [query(m, centre, TV_N, TV_S, PIPE)["vol"] for m in models]
        vol = vols[0]
        for v in vols[1:]:
            vol = vol + v
        total = total + LAM_TV * losses.tv_3d_loss(vol, "mean")
    total.backward()
    with torch.no_grad():
        for m, pkg in zip(models, pkgs):
            m.update_max_radii(pkg["radii"], pkg["visibility_filter"])
            m.add_densification_stats(pkg["viewspace_points"], pkg["visibility_filter"])
    for m in models:
        m.optimizer.step()
        m.optimizer.zero_grad(set_to_none=True)
    return float(total.detach()), image.detach(), None if vol is None else vol.detach()


def run_truth(models, beam, use_tv, first, last):
    cams, gts, centres = train_inputs(beam)
    res = None
    for i in range(first, last + 1):
        k = i % len(cams)
        res = truth_iteration(models, cams[k], gts[k], centres[k], i, use_tv)
    return res


def assert_state_equal(got, gm, label, prefix=""):
    """A worker's saved state against the truth model `gm`: bits, except xyz_gradient_accum (1e-6 relative, as the
    single-GPU native-step test allows: the autograd path accumulates a torch.norm, the kernel its own)."""
    want = model_state(gm)
    for key, w in want.items():
        g = got[prefix + key]
        if key == "xyz_gradient_accum":
            assert g.shape == w.shape, f"{label}: {key} shape"
            assert np.abs(g - w).max(initial=0.0) <= 1e-6 * np.abs(w).max(initial=0.0), f"{label}: {key}"
        else:
            assert g.shape == w.shape and np.array_equal(g, w), \
                f"{label}: {key} differs ({int((g != w).sum()) if g.shape == w.shape else 'shape'} elements)"


@pytest.fixture(scope="module")
def cloud():
    points = init_points()
    return points, full_dist2(points)


# ---- render() / query() ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("beam", ["cone", "parallel"])
def test_sharded_render_and_query_are_the_rank_ordered_sum(beam, cloud, tmp_path, monkeypatch):
    import forward_float64 as f64
    import grad_float64 as g64
    import util
    from r2_gaussian_b200.render_query import query, render
    points, dist2 = cloud
    ranks = run_world(tmp_path, 2, "render", points=points, dist2=dist2, beam=beam)
    monkeypatch.setenv("R2X_SPECULATIVE", "0")    # the exported stage outputs are those of a complete forward
    cams, _, centres = train_inputs(beam)
    cam = cams[1]
    H, W = int(cam.image_height), int(cam.image_width)
    dLi, dLv = fixed_grads(H, W)
    shards, image, vol, s64, bar = [], None, None, 0.0, 0.0
    for r in range(2):
        gm = shard_model(points, dist2, r, 2)
        pkg = render(cam, gm, PIPE)
        fn = pkg["render"].grad_fn
        fwd = util.raster_export(int(gm._xyz.shape[0]), W, H, fn.num_rendered, *fn.saved_tensors[4:7])
        v = query(gm, centres[1], TV_N, TV_S, PIPE)["vol"]
        ((pkg["render"] * dLi).sum() + (v * dLv).sum()).backward()
        img_r = pkg["render"].detach()
        image = img_r if image is None else image + img_r
        vol = v.detach() if vol is None else vol + v.detach()
        fast = g64.fast_path(fwd["conic_opacity"], fwd["mu"])
        flags = {"fast": fast, "exact": ~fast, "ill": g64.cond2(fwd["conic_opacity"]) > g64.COND_MAX}
        st = f64.raster_statement(fwd["xy"], fwd["conic_opacity"], fwd["mu"], fwd["ranges"], fwd["point_list"], W, H,
                                  "kernel", flags)
        s64, bar = s64 + st["S64"], bar + f64.bar(st)
        held = (st["count_ill"] == 0) if r == 0 else held & (st["count_ill"] == 0)
        reached = f64.judged(st) if r == 0 else reached | f64.judged(st)
        want = {"radii": pkg["radii"].cpu().numpy(), "g_means2D": pkg["viewspace_points"].grad.cpu().numpy()}
        for name, attr in _GROUPS:
            want["g_" + name] = getattr(gm, attr).grad.cpu().numpy()
        shards.append(want)
    image, vol = image.cpu().numpy(), vol.cpu().numpy()
    for r, got in enumerate(ranks):
        assert np.array_equal(got["image"], image), f"rank {r}: image is not render_r0 + render_r1"
        assert np.array_equal(got["vol"], vol), f"rank {r}: volume is not query_r0 + query_r1"
        assert np.array_equal(got["image"].view(np.uint32), ranks[0]["image"].view(np.uint32))
        for key, w in shards[r].items():
            assert np.array_equal(got[key], w), f"rank {r}: {key} differs from its shard's single-process backward"
    # the summed image against the float64 statement of the whole cloud: the sum of the shards' statements
    img = image[0].astype(np.float64)
    half_ulp = 0.5 * np.spacing(np.abs(s64).astype(np.float32)).astype(np.float64)
    assert np.all(img[~reached] == 0.0), "a pixel no pair of either shard reaches is not 0"
    ratio = np.abs(img - s64)[held] / (bar + half_ulp)[held]
    print(f"\nsharded {beam}: {int(held.sum())} pixels judged, worst {ratio.max():.3g} x (bar_0 + bar_1 + 1/2 ulp)")
    assert held.sum() > 0.3 * img.size and ratio.max() <= 1.0


# ---- NativeTrainStep --------------------------------------------------------------------------------------------------
def _check_training(ranks, models, label):
    loss0 = float(ranks[0]["loss"])
    for r, got in enumerate(ranks):
        assert float(got["loss"]) == loss0, f"{label}: rank {r} total_loss differs from rank 0's"
        assert np.array_equal(got["image"], ranks[0]["image"]), f"{label}: rank {r} image"
        if "vol" in got:
            assert np.array_equal(got["vol"], ranks[0]["vol"]), f"{label}: rank {r} volume"
    held = [r for r, g in enumerate(ranks) if g["xyz"].shape[0] > 0]      # an empty shard has no truth model
    assert len(held) == len(models)
    for r, gm in zip(held, models):
        assert int(ranks[r]["repeats"]) == 0 or "repeats_after_starve" in ranks[r]
        assert_state_equal(ranks[r], gm, f"{label}, rank {r}")
    return loss0


@pytest.mark.parametrize("use_tv", [True, False])
@pytest.mark.parametrize("beam", ["cone", "parallel"])
def test_sharded_native_step_is_the_autograd_iteration_over_the_shards(beam, use_tv, cloud, tmp_path):
    points, dist2 = cloud
    ranks = run_world(tmp_path, 2, "train", points=points, dist2=dist2, beam=beam, use_tv=use_tv)
    models = [shard_model(points, dist2, r, 2) for r in range(2)]
    total, image, vol = run_truth(models, beam, use_tv, 1, 7)
    loss = _check_training(ranks, models, f"{beam}, tv {use_tv}")
    assert abs(loss - total) <= 1e-6 * abs(total)
    assert np.array_equal(ranks[0]["image"], image.cpu().numpy())
    if use_tv:
        assert np.array_equal(ranks[0]["vol"], vol.cpu().numpy())


def test_sharded_native_step_rebinds_after_densification(cloud, tmp_path):
    """Densification after iteration 4 (clone, split and prune, different on each rank), then 3 more iterations: each
    rank matches the truth up to iteration 4, and a truth restarted from its post-densification state after that."""
    points, dist2 = cloud
    ranks = run_world(tmp_path, 2, "train", points=points, dist2=dist2, beam="cone", use_tv=True, densify_at=4)
    models = [shard_model(points, dist2, r, 2) for r in range(2)]
    run_truth(models, "cone", True, 1, 4)
    for r, (got, gm) in enumerate(zip(ranks, models)):
        assert_state_equal(got, gm, f"rank {r} before densification", prefix="pre_")
        n_clone, n_split, pruned = (int(v) for v in got["densified"])
        assert n_clone > 0 and n_split > 0 and pruned > 0, f"rank {r}: densified {got['densified']}"
    sizes = [g["post_xyz"].shape[0] for g in ranks]
    assert sizes[0] != sizes[1] and sizes != [g["pre_xyz"].shape[0] for g in ranks], sizes
    models = [restore_model({k[5:]: v for k, v in g.items() if k.startswith("post_")}) for g in ranks]
    total, image, _ = run_truth(models, "cone", True, 5, 7)
    loss = _check_training(ranks, models, "after densification")
    assert abs(loss - total) <= 1e-6 * abs(total)
    assert np.array_equal(ranks[0]["image"], image.cpu().numpy())


@pytest.mark.parametrize("starve", ["raster", "voxel"])
def test_a_starved_rank_makes_every_rank_repeat(starve, cloud, tmp_path):
    """Rank 1's raster (voxel) forward overflows at iteration 2.  Its flag rides with the summed image (volume), so both
    ranks skip the update, both repeat the iteration, and the result is the unstarved truth."""
    points, dist2 = cloud
    ranks = run_world(tmp_path, 2, "train", points=points, dist2=dist2, beam="cone", use_tv=True, n_it=4,
                      starve_rank=1, starve_at=2, starve=starve)
    for r, got in enumerate(ranks):
        assert got["starved_unchanged"].all(), f"rank {r}: the overflowed call changed {np.nonzero(~got['starved_unchanged'])}"
        assert int(got["repeats_after_starve"]) == 1 and int(got["repeats"]) == 1, f"rank {r}: repeats"
    models = [shard_model(points, dist2, r, 2) for r in range(2)]
    total, image, _ = run_truth(models, "cone", True, 1, 4)
    loss = _check_training(ranks, models, "starved rank 1")
    assert abs(loss - total) <= 1e-6 * abs(total)
    assert np.array_equal(ranks[0]["image"], image.cpu().numpy())


@pytest.mark.parametrize("use_tv", [True, False])
def test_an_empty_shard_joins_both_exchanges(use_tv, cloud, tmp_path):
    """World 3 with rank 1's shard pruned to nothing: the empty rank adds +0.0, ranks 0 and 2 match the two-shard
    truth, and all three ranks hold the same image and volume."""
    points, dist2 = cloud
    ranks = run_world(tmp_path, 3, "train", points=points, dist2=dist2, beam="cone", use_tv=use_tv, n_it=5,
                      empty_rank=1)
    assert ranks[1]["xyz"].shape[0] == 0 and int(ranks[1]["repeats"]) == 0
    models = [shard_model(points, dist2, r, 3) for r in (0, 2)]
    total, image, vol = run_truth(models, "cone", use_tv, 1, 5)
    loss = _check_training(ranks, models, f"empty shard, tv {use_tv}")
    assert abs(loss - total) <= 1e-6 * abs(total)
    assert np.array_equal(ranks[1]["image"], image.cpu().numpy())
    if use_tv:
        assert np.array_equal(ranks[1]["vol"], vol.cpu().numpy())


# ---- peer memory between two devices ----------------------------------------------------------------------------------
def _two_peer_devices():
    return torch.cuda.device_count() >= 2 and torch.cuda.can_device_access_peer(0, 1)


@pytest.mark.skipif(not _two_peer_devices(), reason="needs two peer-capable GPUs (one process per device)")
def test_peer_exchange_on_two_devices(cloud, tmp_path):
    """PeerReducer over 40 epochs (double buffering, the flag protocol over real IPC mappings), then the world-2
    NativeTrainStep with enable_peer_exchange(True) against the same truth as over gloo."""
    ranks = run_world(tmp_path, 2, "peer_epochs")
    for r, got in enumerate(ranks):
        assert bool(got["ok"]), f"rank {r}: a peer was reported missing"
        parts = got["parts"]
        want = parts[:, 0] + parts[:, 1]
        assert np.array_equal(got["outs"], want), f"rank {r}: not the rank-ordered sum"
        assert np.array_equal(got["outs"], ranks[0]["outs"])
    points, dist2 = cloud
    ranks = run_world(tmp_path, 2, "train", peer=True, points=points, dist2=dist2, beam="cone", use_tv=True)
    models = [shard_model(points, dist2, r, 2) for r in range(2)]
    total, image, vol = run_truth(models, "cone", True, 1, 7)
    loss = _check_training(ranks, models, "peer exchange")
    assert abs(loss - total) <= 1e-6 * abs(total)
    assert np.array_equal(ranks[0]["image"], image.cpu().numpy())
    assert np.array_equal(ranks[0]["vol"], vol.cpu().numpy())
