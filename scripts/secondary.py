"""Secondary measurements for bench.py's `secondary` block (the other BASELINE configurations, next to the headline):

  raster fwd+bwd   100k Gaussians / 512^2 cone beam, forward + backward through the reference-shaped `_C` entry points
  voxel sweep      256^3 volume query over 500k Gaussians (BASELINE config 4), forward, with its HBM roofline
                   B_vox = 56 P + 44 V + 68 R + 4 N (SURVEY.md 8d)
  TV crop          32^3 sub-volume of the 100k cloud, forward + backward (train.py:128-144)
  train iteration  render + fused L1/D-SSIM + 32^3 TV crop query + backward + fused Adam on the headline scene

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
    return out


if __name__ == "__main__":
    print(json.dumps(measure(quick="--quick" in sys.argv)))
