"""Secondary measurements for bench.py's `secondary` block (the other BASELINE configurations, next to the headline):

  raster fwd+bwd   100k Gaussians / 512^2 cone beam, forward + backward through the reference-shaped `_C` entry points
  voxel sweep      256^3 volume query over 500k Gaussians (BASELINE config 4), forward, with its HBM roofline
                   B_vox = 56 P + 44 V + 68 R + 4 N (SURVEY.md 8d)
  TV crop          32^3 sub-volume of the 100k cloud, forward + backward (train.py:128-144)
  train iteration  render + fused L1/D-SSIM + 32^3 TV crop query + backward + fused Adam on the headline scene
  fdk              FDK reconstruction, 50 cone-beam views of 512^2 -> 256^3: filter, backprojection, whole call and
                   voxel-view updates/s (no reference arm: the reference uses TIGRE, which is not part of this build)
  project          forward projection of a 256^3 volume into 150 cone-beam views of 512^2 (the reference's synthetic
                   dataset: 50 train + 100 test), samples/s and projections/s, with the card name and power limit
                   (no reference arm: TIGRE's Ax is not part of this build)
  backproject      the matched backprojection (r2x_volume_backproject) of the fdk row's 50 cone-beam views of 512^2
                   into 256^3, with and without its weight output, per view next to the projector's per view on the
                   same views, with the card name and power limit (no reference arm: TIGRE's Atb)
  recon            one CGLS iteration and one SART sweep (50 single-view updates) on the same workload (no reference
                   arm: TIGRE's algs)

each for ours and, where the compiled reference (oracle/_ref/libr2ref.so) is present, for the reference's own CUDA
kernels with the identical protocol (CUDA events per step, L2 flushed between steps).  `python scripts/secondary.py`
prints the block on its own."""
from __future__ import annotations

import ctypes as C
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def measure(dev=None, peak_gbs: float = 3350.0, quick: bool = False, trace=lambda msg: None) -> dict:
    import torch

    import bench
    from r2_gaussian_b200 import _C, losses, scene
    from r2_gaussian_b200.engine import VoxelEngine
    from r2_gaussian_b200.gaussian_model import GaussianModel
    from r2_gaussian_b200.render_query import query, render

    dev = torch.device("cuda") if dev is None else dev
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    sync = lambda: torch.cuda.synchronize(dev)
    E = torch.Tensor([])
    out = {"protocol": "mean of per-step CUDA-event times, 256 MiB L2 flush between steps"}

    def timed(fn, steps=20, warmup=4):
        if quick:
            steps, warmup = max(3, steps // 4), 2
        return float(np.mean(bench.timed_steps(lambda i: fn(i), steps, warmup, flush, sync)))

    class A:
        gaussians = 100000; detector = 512; views = 50; cloud = "init"

    sc, views, cloud = bench.build_scene(A)
    m = torch.tensor(cloud.means, device=dev); s = torch.tensor(cloud.scales, device=dev)
    r = torch.tensor(cloud.rotations, device=dev); d = torch.tensor(cloud.density, device=dev)
    dv = bench.device_views(views, dev)
    dL = torch.randn(1, 512, 512, device=dev, generator=torch.Generator(dev).manual_seed(0))

    ref_path = os.path.join(ROOT, "oracle", "_ref", "libr2ref.so")
    lib = C.CDLL(ref_path) if os.path.exists(ref_path) else None
    vp = lambda t: C.c_void_p(t.data_ptr())
    f = C.c_float
    z = lambda *sh: torch.zeros(sh, device=dev)
    if lib is not None:
        lib.ref_raster_forward.restype = C.c_int
        lib.ref_voxel_forward.restype = C.c_int

    # ---- projector forward + backward ----
    def ours_fb(i):
        v = dv[i % 50]
        R, img, radii, geom, binning, imgb = _C.rasterize_gaussians(m, d, s, r, 1.0, E, v["view"], v["proj"], v["tx"],
                                                                     v["ty"], 512, 512, v["campos"], False, v["mode"], False)
        _C.rasterize_gaussians_backward(m, radii, s, r, 1.0, E, v["view"], v["proj"], v["tx"], v["ty"], dL, v["campos"],
                                        geom, R, binning, imgb, v["mode"], False)

    rb = {"workload": "100k Gaussians, 512x512 cone beam, forward + backward through _C.rasterize_gaussians[_backward]",
          "ours_ms": timed(ours_fb)}
    v0 = dv[0]
    st = _C.rasterize_gaussians(m, d, s, r, 1.0, E, v0["view"], v0["proj"], v0["tx"], v0["ty"], 512, 512, v0["campos"],
                                False, v0["mode"], False)

    def ours_b(i):
        R, img, radii, geom, binning, imgb = st
        _C.rasterize_gaussians_backward(m, radii, s, r, 1.0, E, v0["view"], v0["proj"], v0["tx"], v0["ty"], dL,
                                        v0["campos"], geom, R, binning, imgb, v0["mode"], False)

    rb["ours_backward_only_ms"] = timed(ours_b)
    P = cloud.P
    if lib is not None:
        o = z(1, 512, 512); radii_r = torch.zeros(P, dtype=torch.int32, device=dev)
        g2, gc, go, gm_, g3, gcov, gs, gr = z(P, 3), z(P, 4), z(P, 1), z(P, 1), z(P, 3), z(P, 6), z(P, 3), z(P, 4)

        def ref_fb(i):
            v = dv[i % 50]
            o.zero_(); radii_r.zero_()
            R = lib.ref_raster_forward(P, 512, 512, vp(m), vp(d), vp(s), f(1.0), vp(r), None, vp(v["view"]), vp(v["proj"]),
                                       vp(v["campos"]), f(v["tx"]), f(v["ty"]), int(v["mode"]), vp(o), vp(radii_r))
            for t in (g2, gc, go, gm_, g3, gcov, gs, gr):   # the binding zero-fills the 8 gradient tensors every call
                t.zero_()
            lib.ref_raster_backward(P, R, 512, 512, vp(m), vp(s), f(1.0), vp(r), None, vp(v["view"]), vp(v["proj"]),
                                    vp(v["campos"]), f(v["tx"]), f(v["ty"]), vp(radii_r), vp(dL), vp(g2), vp(gc), vp(go),
                                    vp(gm_), vp(g3), vp(gcov), vp(gs), vp(gr), int(v["mode"]))

        rb["reference_ms"] = timed(ref_fb, 10, 2)
        rb["speedup"] = rb["reference_ms"] / rb["ours_ms"]
    out["raster_fwd_bwd"] = rb
    trace("secondary: raster forward + backward")

    # ---- voxelizer sweep: 256^3 over 500k Gaussians (BASELINE config 4), init-like and trained-like clouds ----
    N = 256 ** 3
    grid = ((2.0, 2.0, 2.0), (0.0, 0.0, 0.0))
    for kind, key in (("init", "voxel_256_500k"), ("trained", "voxel_256_500k_trained")):
        big = scene.make_cloud(500000, kind=kind, seed=0)
        bm = torch.tensor(big.means, device=dev); bs = torch.tensor(big.scales, device=dev)
        br = torch.tensor(big.rotations, device=dev); bd = torch.tensor(big.density, device=dev)
        ve = VoxelEngine(big.P, (256, 256, 256), dev, capacity=28_000_000)
        Rv = ve.fit(bm, bd, bs, br, *grid)
        V = int((ve.radii[0] > 0).logical_and(ve.radii[1] > 0).logical_and(ve.radii[2] > 0).sum().item())
        vx = {"workload": f"256^3 volume query over 500k Gaussians ({kind}-like, seed 0), forward", "num_rendered": int(Rv),
              "visible": V, "ours_ms": timed(lambda i: ve.forward(bm, bd, bs, br, *grid), 10, 2),
              "ours_render_kernel_ms": timed(lambda i: ve.render_only(), 10, 2)}
        alg = 56.0 * big.P + 44.0 * V + 68.0 * Rv + 4.0 * N
        vx["roofline"] = {"bound": "hbm", "algorithmic_bytes": alg, "achieved": alg / (vx["ours_ms"] * 1e-3) / 1e9,
                          "peak": peak_gbs, "unit": "GB/s", "frac": alg / (vx["ours_ms"] * 1e-3) / 1e9 / peak_gbs,
                          "pair_evals": 512.0 * Rv, "pair_evals_per_s": 512.0 * Rv / (vx["ours_render_kernel_ms"] * 1e-3)}
        if lib is not None:
            vol = z(256, 256, 256)
            rx = torch.zeros(big.P, dtype=torch.int32, device=dev); ry = torch.zeros_like(rx); rz = torch.zeros_like(rx)

            def ref_v(i):
                vol.zero_()
                lib.ref_voxel_forward(big.P, 256, 256, 256, f(2.0), f(2.0), f(2.0), f(0.0), f(0.0), f(0.0), vp(bm), vp(bd),
                                      vp(bs), f(1.0), vp(br), None, vp(vol), vp(rx), vp(ry), vp(rz))

            vx["reference_ms"] = timed(ref_v, 5, 1)
            vx["speedup"] = vx["reference_ms"] / vx["ours_ms"]
            mine = ve.forward(bm, bd, bs, br, *grid)
            vx["parity"] = {"max_abs": float((mine - vol).abs().max()), "max_rel_to_max": float((mine - vol).abs().max() / vol.abs().max()),
                            "radii_equal": bool(torch.equal(ve.radii[0], rx) and torch.equal(ve.radii[1], ry) and torch.equal(ve.radii[2], rz))}
            del vol, rx, ry, rz, mine
        out[key] = vx
        trace(f"secondary: {key} (R = {int(Rv)})")
        del ve, bm, bs, br, bd
        torch.cuda.empty_cache()

    # ---- TV crop: 32^3 sub-volume of the 100k cloud, forward + backward ----
    dV = torch.randn(32, 32, 32, device=dev, generator=torch.Generator(dev).manual_seed(1))
    crop = (32, 32, 32, 0.25, 0.25, 0.25, 0.3, -0.4, 0.1)

    def ours_tv(i):
        R, vol_, rx_, ry_, rz_, geom, binning, imgb = _C.voxelize_gaussians(m, d, s, r, 1.0, E, *crop, False, False)
        _C.voxelize_gaussians_backward(m, rx_, ry_, rz_, s, r, 1.0, E, dV, geom, R, binning, imgb, *crop, False)

    tv = {"workload": "32^3 crop (sVoxel 0.25) of the 100k cloud, forward + backward through _C.voxelize_gaussians[_backward]",
          "ours_ms": timed(ours_tv)}
    if lib is not None:
        vol2 = z(32, 32, 32)
        qx = torch.zeros(P, dtype=torch.int32, device=dev); qy = torch.zeros_like(qx); qz = torch.zeros_like(qx)
        gn, gc6, go1, g31, gcv, gs1, gr1 = z(P, 3), z(P, 6), z(P, 1), z(P, 3), z(P, 6), z(P, 3), z(P, 4)
        fc = [f(x) for x in crop[3:]]

        def ref_tv(i):
            vol2.zero_()
            R = lib.ref_voxel_forward(P, 32, 32, 32, *fc, vp(m), vp(d), vp(s), f(1.0), vp(r), None, vp(vol2), vp(qx), vp(qy), vp(qz))
            for t in (gn, gc6, go1, g31, gcv, gs1, gr1):
                t.zero_()
            lib.ref_voxel_backward(P, R, 32, 32, 32, *fc, vp(m), vp(s), f(1.0), vp(r), None, vp(qx), vp(qy), vp(qz), vp(dV),
                                   vp(gn), vp(gc6), vp(go1), vp(g31), vp(gcv), vp(gs1), vp(gr1))

        tv["reference_ms"] = timed(ref_tv, 10, 2)
        tv["speedup"] = tv["reference_ms"] / tv["ours_ms"]
    out["tv_crop_32"] = tv

    trace("secondary: TV crop")
    # ---- one training iteration on the headline scene ----
    scanner = scene.cone_beam_scanner(512)
    cams = [scene.camera_from_view(vw, device=dev) for vw in scene.make_views(scanner, 8)]
    opt_args = types.SimpleNamespace(
        position_lr_init=2e-4, position_lr_final=2e-5, position_lr_max_steps=30000,
        density_lr_init=1e-2, density_lr_final=1e-3, density_lr_max_steps=30000,
        scaling_lr_init=5e-3, scaling_lr_final=5e-4, scaling_lr_max_steps=30000,
        rotation_lr_init=1e-3, rotation_lr_final=1e-4, rotation_lr_max_steps=30000)
    gm = GaussianModel((0.001, 1.0))
    import contextlib
    import io
    with contextlib.redirect_stdout(io.StringIO()):      # create_from_pcd prints like the reference; bench.py prints ONE JSON line
        gm.create_from_pcd(cloud.means, np.maximum(cloud.density, 1e-3), 1.0)
    gm.training_setup(opt_args)
    pipe = types.SimpleNamespace(compute_cov3D_python=False, debug=False)
    with torch.no_grad():
        gts = [render(c, gm, pipe)["render"] * 0.9 for c in cams]
    it = [0]

    def train_iter(_i):
        i = it[0] = it[0] + 1
        gm.update_learning_rate(i)
        pkg = render(cams[i % 8], gm, pipe)
        loss = losses.image_loss(pkg["render"], gts[i % 8], 0.25)["total"]
        vol_ = query(gm, [0.1, 0.0, -0.1], [32, 32, 32], [0.25, 0.25, 0.25], pipe)["vol"]
        loss = loss + 0.05 * losses.tv_3d_loss(vol_, "mean")
        loss.backward()
        with torch.no_grad():
            vis = pkg["visibility_filter"]
            gm.update_max_radii(pkg["radii"], vis)
            gm.add_densification_stats(pkg["viewspace_points"], vis)
        gm.optimizer.step()
        gm.optimizer.zero_grad(set_to_none=True)

    for k in range(5):
        train_iter(k)
    sync()
    import time
    n_it = 10 if quick else 40
    t0 = time.perf_counter()
    for k in range(n_it):
        train_iter(k)
    sync()
    autograd_ms = (time.perf_counter() - t0) / n_it * 1e3
    # the same iteration as a fixed launch sequence (train_step.NativeTrainStep: no autograd graph, no allocation)
    from r2_gaussian_b200.train_step import NativeTrainStep
    native = NativeTrainStep(gm, 0.25, 0.05, [32, 32, 32], [0.25, 0.25, 0.25])

    def native_iter():
        i = it[0] = it[0] + 1
        gm.update_learning_rate(i)
        native(cams[i % 8], gts[i % 8], (0.1, 0.0, -0.1))

    for k in range(5):
        native_iter()
    native.flush()
    sync()
    n_nat = 20 if quick else 200
    t0 = time.perf_counter()
    for k in range(n_nat):
        native_iter()
    native.flush()
    sync()
    native_ms = (time.perf_counter() - t0) / n_nat * 1e3
    out["train_iteration"] = {"workload": "100k Gaussians, 512x512: render + fused L1/D-SSIM + 32^3 TV crop query + backward + "
                                          "fused Adam + densification statistics",
                              "ours_ms_wall": native_ms, "api": "train_step.NativeTrainStep (what trainer.py runs)",
                              "autograd_path_ms_wall": autograd_ms,
                              "autograd_path_api": "GaussianModel / render() / query() / losses / FusedAdam behind autograd",
                              "repeated_iterations": native.repeats}
    trace("secondary: training iteration")

    # ---- FDK reconstruction: 50 views of 512^2 -> 256^3, the reference's cone-beam dataset geometry ----
    out["fdk"] = measure_fdk(dev, timed)
    trace("secondary: fdk")

    # ---- volume projection: the reference's synthetic dataset, 50 train + 100 test cone-beam views of 512^2 ----
    out["project"] = measure_project(dev, timed)
    trace("secondary: project")

    # ---- matched backprojection and the iterative reconstructions on the fdk row's workload ----
    out["backproject"] = measure_backproject(dev, timed)
    trace("secondary: backproject")
    out["recon"] = measure_recon(dev, timed)
    trace("secondary: recon")
    return out


def card(dev) -> dict:
    """Name and power limit of the device the row was measured on (nvidia-smi query; None if it is unavailable)."""
    import subprocess

    import torch

    idx = torch.device(dev).index or 0
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(idx)],
                           capture_output=True, text=True, timeout=20)
        power = float(r.stdout.strip().splitlines()[0])
    except Exception:
        power = None
    return {"gpu": torch.cuda.get_device_name(idx), "power_limit_w": power}


def projector_samples(sc: dict, angles, step: float) -> int:
    """Samples r2x_volume_project evaluates: per ray, the integers k with t_c + k step inside the support box
    offOrigin +- (sVoxel/2 + dVoxel/2) (cone beam: t > 0), from the same slab test in float64."""
    from r2_gaussian_b200 import scene

    n = np.asarray(sc["nVoxel"], np.float64)
    dv = np.asarray(sc["sVoxel"], np.float64) / n
    c = np.asarray(sc["offOrigin"], np.float64)
    total = 0
    for a in angles:
        v = scene.make_view(sc, float(a))
        H, W = v.image_height, v.image_width
        ndx = (2.0 * np.arange(W) + 1.0) / W - 1.0
        ndy = (2.0 * np.arange(H) + 1.0) / H - 1.0
        c2w = np.linalg.inv(v.viewmatrix.astype(np.float64).T)
        if v.mode == scene.MODE_CONE:
            d = np.stack(np.broadcast_arrays(ndx[None, :] * v.tanfovx, ndy[:, None] * v.tanfovy, 1.0), -1)
            o = np.broadcast_to(c2w[:3, 3], d.shape)
        else:
            d = np.broadcast_to(np.array([0.0, 0.0, 1.0]), (H, W, 3))
            o = np.stack(np.broadcast_arrays(ndx[None, :], ndy[:, None], 0.0), -1) @ c2w[:3, :3].T + c2w[:3, 3]
        d = d @ c2w[:3, :3].T
        d = d / np.linalg.norm(d, axis=-1, keepdims=True)
        tc = ((c - o) * d).sum(-1)
        g = (o + tc[..., None] * d - c) / dv + 0.5 * (n - 1.0)
        st = step * d / dv
        lo = np.full(tc.shape, -np.inf)
        hi = np.full(tc.shape, np.inf)
        for ax in range(3):
            nz = st[..., ax] != 0.0
            s_ = np.where(nz, st[..., ax], 1.0)
            k1, k2 = (-1.0 - g[..., ax]) / s_, (n[ax] - g[..., ax]) / s_
            inside = (g[..., ax] > -1.0) & (g[..., ax] < n[ax])
            lo = np.maximum(lo, np.where(nz, np.minimum(k1, k2), np.where(inside, -np.inf, np.inf)))
            hi = np.minimum(hi, np.where(nz, np.maximum(k1, k2), np.where(inside, np.inf, -np.inf)))
        k0 = np.ceil(lo)
        if v.mode == scene.MODE_CONE:
            k0 = np.maximum(k0, np.floor(-tc / step) + 1.0)
        total += int(np.maximum(np.floor(hi) - k0 + 1.0, 0.0).sum())
    return total


def measure_project(dev, timed) -> dict:
    """r2x_volume_project on the reference's synthetic setting: a seeded 256^3 volume, 50 train views at
    linspace(0, 2 pi) and 100 sorted random test views, 512^2 cone beam, accuracy 0.5."""
    import torch

    from r2_gaussian_b200 import _lib, scene

    lib = _lib.load()
    sc = scene.cone_beam_scanner(512, 256)
    rng = np.random.RandomState(0)
    angles = np.concatenate([np.linspace(0.0, 2.0 * np.pi, 51)[:-1], np.sort(rng.rand(100) * 2.0 * np.pi)])
    views = [scene.make_view(sc, float(a)) for a in angles]
    N, H, W, n = len(views), 512, 512, 256
    step = 0.5 * 2.0 / n
    vol = torch.rand(n, n, n, device=dev, generator=torch.Generator(dev).manual_seed(0))
    vm = torch.tensor(np.stack([v.viewmatrix.reshape(16) for v in views]), device=dev)
    projs = torch.empty(N, H, W, device=dev)
    tx, ty = float(views[0].tanfovx), float(views[0].tanfovy)

    def run(_i):
        _lib.check(lib.r2x_volume_project(torch.cuda.current_stream(dev).cuda_stream, n, n, n, vol.data_ptr(), 2.0, 2.0,
                                          2.0, 0.0, 0.0, 0.0, N, H, W, vm.data_ptr(), tx, ty, 1, 0.0, 0.0, step,
                                          projs.data_ptr()), "r2x_volume_project")

    row = {"workload": "forward projection, seeded 256^3 volume -> 150 cone-beam views (50 train + 100 test) of "
                       "512x512 (DSD 7, DSO 5), accuracy 0.5 (r2x_volume_project)",
           "ours_ms": timed(run), "sample_fetch": "__ldg through L1/L2",
           "reference": "none: TIGRE's Ax is not part of this build"}
    samples = projector_samples(sc, angles, step)
    row["samples"] = samples
    row["samples_per_s"] = samples / (row["ours_ms"] * 1e-3)
    row["projections_per_s"] = N / (row["ours_ms"] * 1e-3)
    row.update(card(dev))
    return row


def measure_fdk(dev, timed) -> dict:
    """Filter, backprojection and the whole r2x_fdk call on 50 seeded 512^2 cone-beam views into a 256^3 grid."""
    import torch

    from r2_gaussian_b200 import _lib, scene
    from r2_gaussian_b200.fdk import R2X_FDK_PLAIN

    lib = _lib.load()
    sc = scene.cone_beam_scanner(512, 256)
    views = scene.make_views(sc, 50)
    N, H, W, n = 50, 512, 512, 256
    projs = torch.rand(N, H, W, device=dev, generator=torch.Generator(dev).manual_seed(0))
    vm = torch.tensor(np.stack([v.viewmatrix.reshape(16) for v in views]), device=dev)
    pm = torch.tensor(np.stack([v.projmatrix.reshape(16) for v in views]), device=dev)
    q = torch.empty_like(projs)
    vol = torch.empty(n, n, n, device=dev)
    nbytes = int(lib.r2x_fdk_scratch_bytes(N, H, W))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    stream = lambda: torch.cuda.current_stream(dev).cuda_stream
    tx, ty, dso = float(views[0].tanfovx), float(views[0].tanfovy), float(sc["DSO"])
    grid = (n, n, n, 2.0, 2.0, 2.0, 0.0, 0.0, 0.0)

    def filt(_i):
        _lib.check(lib.r2x_fdk_filter(stream(), N, H, W, projs.data_ptr(), tx, ty, 1, dso, q.data_ptr()), "r2x_fdk_filter")

    def backproject(_i):
        _lib.check(lib.r2x_fdk_backproject(stream(), N, H, W, q.data_ptr(), vm.data_ptr(), pm.data_ptr(), 1, dso, *grid,
                                           vol.data_ptr()), "r2x_fdk_backproject")

    def total(_i):
        _lib.check(lib.r2x_fdk(stream(), N, H, W, projs.data_ptr(), vm.data_ptr(), pm.data_ptr(), tx, ty, 1, 0.0, 0.0,
                               R2X_FDK_PLAIN, None, 0.0, dso, *grid, vol.data_ptr(), scratch.data_ptr(), nbytes),
                   "r2x_fdk")

    row = {"workload": "FDK, 50 cone-beam views of 512x512 (DSD 7, DSO 5) -> 256^3 volume, Ram-Lak filter + voxel-driven "
                       "backprojection (r2x_fdk)",
           "filter_ms": timed(filt), "backproject_ms": timed(backproject), "ours_ms": timed(total),
           "sample_fetch": "__ldg through L1/L2",
           "reference": "none: the reference reconstructs with TIGRE's algs.fdk, which is not part of this build"}
    row["voxel_view_updates_per_s"] = float(n) ** 3 * N / (row["ours_ms"] * 1e-3)
    row["backproject_voxel_view_updates_per_s"] = float(n) ** 3 * N / (row["backproject_ms"] * 1e-3)
    return row


def _recon_workload(dev):
    """The fdk row's geometry (50 cone-beam views of 512^2 at linspace(0, 2 pi), 256^3 grid, accuracy 0.5) with seeded
    projections of a seeded volume, bound to the GPU projector pair."""
    import torch

    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.projector import CTOperator

    sc = dict(scene.cone_beam_scanner(512, 256), accuracy=0.5)
    op = CTOperator(np.linspace(0.0, 2.0 * np.pi, 51)[:-1], sc, dev)
    vol = torch.rand(256, 256, 256, device=dev, generator=torch.Generator(dev).manual_seed(0))
    return op, op.A(vol)


def measure_backproject(dev, timed) -> dict:
    """r2x_volume_backproject with and without out_weight, and r2x_volume_project on the same 50 views."""
    op, b = _recon_workload(dev)
    n = op.N
    row = {"workload": "matched backprojection, 50 cone-beam views of 512x512 (DSD 7, DSO 5) -> 256^3, accuracy 0.5 "
                       "(r2x_volume_backproject: ray table + voxel-driven gather)",
           "ours_ms": timed(lambda _i: op.At(b)), "with_weight_ms": timed(lambda _i: op.At(b, weights=True), 10, 2),
           "project_same_views_ms": timed(lambda _i: op.A(b.new_zeros(op.nvox)), 10, 2),
           "reference": "none: TIGRE's Atb is not part of this build"}
    row["per_view_ms"] = row["ours_ms"] / n
    row["project_per_view_ms"] = row["project_same_views_ms"] / n
    row["backproject_over_project_per_view"] = row["per_view_ms"] / row["project_per_view_ms"]
    row.update(card(dev))
    return row


def measure_recon(dev, timed) -> dict:
    """One CGLS iteration (A, A^T and three float64 reductions) and one SART sweep (50 single-view updates, each a
    one-view projection and a fused one-view backprojection) on the backproject row's workload."""
    import torch

    from r2_gaussian_b200 import recon

    op, b = _recon_workload(dev)
    one = lambda x, views: op.A(torch.ones_like(x), views)
    row = {"workload": "one CGLS iteration and one SART sweep (blocksize 1: 50 view updates) on 50 cone-beam views of "
                       "512x512 -> 256^3 (recon.cgls_solve / recon.sart_solve over projector.CTOperator)",
           "cgls_iteration_ms": timed(lambda _i: recon.cgls_solve(b, op.A, op.At, 1), 5, 1),
           "cgls_setup_ms": timed(lambda _i: recon.cgls_solve(b, op.A, op.At, 0), 5, 1),
           "sart_sweep_ms": timed(lambda _i: recon.sart_solve(b, op.A, op.At, op.nvox, 1), 5, 1),
           "sart_setup_ms": timed(lambda _i: one(b.new_zeros(op.nvox), slice(None)), 5, 1),
           "reference": "none: TIGRE's algs.cgls / algs.sart are not part of this build"}
    # cgls_solve(niter=1) is setup (A^T b) + one iteration; sart_solve(niter=1) is W = 1 / A 1 + one sweep
    row["cgls_iteration_ms"] -= row["cgls_setup_ms"]
    row["sart_sweep_ms"] -= row["sart_setup_ms"]
    row.update(card(dev))
    return row


if __name__ == "__main__":
    print(json.dumps(measure(quick="--quick" in sys.argv)))
