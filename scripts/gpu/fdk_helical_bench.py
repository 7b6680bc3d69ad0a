"""Cost of the helical FDK (r2x_fdk_helical through fdk.fdk(helical=True)):

    python scripts/gpu/fdk_helical_bench.py [--reps 10] [--out DIR]

  * scene: the helical test scene of tests/test_fdk_helical_gpu.py (48 x 48 x 96, 120 views of 32 x 64 over two turns)
    through fdk.fdk(helical=True) (host set-up included) and through r2x_fdk_helical alone.
  * circle: pitch 0 on the 50-view 512^2 -> 256^3 circle (scripts/secondary.py's fdk row), r2x_fdk_helical at Q = 1
    against r2x_fdk, alternated: what the weights cost.
  * long: a 256 x 256 x 512 grid, 8 turns x 360 views of 64 x 512 at pitch factor 1 (the source travels one detector
    height at the isocentre per turn).  The fraction of (CTA, view) pairs the view window keeps is counted on the host
    from the kernel's bound; time / fraction estimates the call without the window.  One CGLS iteration (one A and one
    A^T of the per-view projector pair) on the same views and grid, for comparison.  The long call is r2x_fdk_helical
    alone (the host fit and matrices of 2880 views are built once, outside the timing).
Each time is the median of --reps calls timed with CUDA events after a warm-up.  Prints one JSON line with the card
name and power limit (nvidia-smi)."""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _median_ms(fns: dict, reps: int) -> dict:
    import torch
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(reps):
        for k, f in fns.items():          # alternate the variants
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            times[k].append(a.elapsed_time(b))
    return {k: float(np.median(v)) for k, v in times.items()}


def _helix(n_views, turns, travel, nvox, ndet, svox, sdet):
    sc = {"mode": "cone", "DSD": 7.0, "DSO": 5.0, "nDetector": list(ndet), "sDetector": list(sdet),
          "nVoxel": list(nvox), "sVoxel": list(svox), "offOrigin": [0.0, 0.0, 0.0], "offDetector": [0.0, 0.0]}
    angles = np.linspace(0.0, 2.0 * math.pi * turns, n_views + 1)[:-1]
    geo = [{"offOrigin": [0.0, 0.0, travel * (i / n_views - 0.5)]} for i in range(n_views)]
    return sc, angles, geo


def prepared(projs, angles, sc, geo, q: float = 0.5):
    """A closure running r2x_fdk_helical on views already sorted, uploaded and fitted (fdk.fdk without its host
    set-up), and the fitted helix."""
    import torch

    from r2_gaussian_b200 import _lib
    from r2_gaussian_b200.fdk import helix_views
    from r2_gaussian_b200.projector import view_table
    lib, dev = _lib.load(), projs.device
    hx = helix_views(angles, sc, geo)
    views, table = view_table(np.asarray(angles)[hx.order], sc, [geo[i] for i in hx.order])
    N, H, W = projs.shape
    ps = projs.index_select(0, torch.from_numpy(np.ascontiguousarray(hx.order)).to(dev)).contiguous()
    vm = torch.tensor(np.stack([v.viewmatrix.reshape(16) for v in views]), device=dev)
    pm = torch.tensor(np.stack([v.projmatrix.reshape(16) for v in views]), device=dev)
    bh = np.ascontiguousarray(hx.beta)
    bd, dbd = torch.from_numpy(bh).to(dev), torch.from_numpy(np.ascontiguousarray(hx.dbeta)).to(dev)
    vol = torch.empty(*sc["nVoxel"], device=dev)
    nbytes = int(lib.r2x_fdk_scratch_bytes(N, H, W))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    grid = (*sc["nVoxel"], *(float(v) for v in sc["sVoxel"]), *(float(v) for v in sc["offOrigin"]))

    def run():
        _lib.check(lib.r2x_fdk_helical(torch.cuda.current_stream(dev).cuda_stream, N, H, W, ps.data_ptr(),
                                       vm.data_ptr(), pm.data_ptr(), float(table[0, 0]), float(table[0, 1]), 1, 0,
                                       float(table[0, 4]), bd.data_ptr(), dbd.data_ptr(), bh.ctypes.data, hx.z0, hx.h,
                                       hx.beta_lo, hx.beta_hi, hx.c_x, hx.c_y, q, *grid, vol.data_ptr(),
                                       scratch.data_ptr(), nbytes), "fdk_helical")
        return vol
    return run, hx


def window_fraction(sc, hx, tany: float) -> float:
    """The share of (CTA, view) pairs r2x_fdk_helical visits: views whose source height is within
    (DSO + the grid's largest in-plane radius) tan_fovy (1 + 1e-3) of the CTA's 8-voxel z-run."""
    nx, ny, nz = sc["nVoxel"]
    sx, sy, sz = sc["sVoxel"]
    dx, dy, dz = sx / nx, sy / ny, sz / nz
    ox, oy, oz = -0.5 * sx + 0.5 * dx, -0.5 * sy + 0.5 * dy, -0.5 * sz + 0.5 * dz
    r = max(math.hypot(ox + i * (nx - 1) * dx - hx.c_x, oy + j * (ny - 1) * dy - hx.c_y) for i in (0, 1) for j in (0, 1))
    reach = (sc["DSO"] + r) * tany * (1.0 + 1e-3)
    zs = hx.z0 + hx.h * hx.beta
    z0 = oz + 8 * dz * np.arange((nz + 7) // 8)
    keep = (zs[None, :] > z0[:, None] - reach) & (zs[None, :] < z0[:, None] + 7 * dz + reach)
    return float(keep.mean())


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    import torch

    from r2_gaussian_b200 import _lib, scene
    from r2_gaussian_b200.fdk import fdk, helix_views
    from r2_gaussian_b200.projector import CTOperator
    lib = _lib.load()
    dev = torch.device("cuda")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi}

    # scene: the helical test scene through the public call
    from test_view_geometry_gpu import _tall_phantom, _yml

    from r2_gaussian_b200 import generate_data
    from r2_gaussian_b200.dataset import read_scene
    from r2_gaussian_b200.recon import view_geometry_of
    tmpdir = tempfile.TemporaryDirectory()      # removed when the script exits
    tmp = tmpdir.name
    import pathlib
    tp = pathlib.Path(tmp)
    np.save(tp / "vol.npy", _tall_phantom())
    src = generate_data.main(["--vol", str(tp / "vol.npy"), "--scanner", str(_yml(tp / "h.yml")), "--n_train", "120",
                              "--n_test", "8", "--helical_travel", "3.2", "--output", str(tp / "data")])
    info = read_scene(src, eval=False, use_view_geometry=True)
    p = torch.from_numpy(np.stack([np.asarray(c.image, np.float32) for c in info.train_cameras])).cuda()
    ang = [c.angle for c in info.train_cameras]
    vg = view_geometry_of(info.train_cameras, True)
    kernel, _ = prepared(p, ang, info.scanner_cfg, vg)
    res["scene_ms"] = _median_ms({"fdk.fdk": lambda: fdk(p, ang, info.scanner_cfg, view_geometry=vg, helical=True),
                                  "r2x_fdk_helical": kernel}, a.reps)

    # circle: r2x_fdk_helical at pitch 0 against r2x_fdk
    sc = scene.cone_beam_scanner(512, 256)
    N, H, W, n = 50, 512, 512, 256
    angles = np.linspace(0.0, 2.0 * math.pi, N + 1)[:-1]
    views = [scene.make_view(sc, float(t)) for t in angles]
    vm = torch.tensor(np.stack([v.viewmatrix.reshape(16) for v in views]), device=dev)
    pm = torch.tensor(np.stack([v.projmatrix.reshape(16) for v in views]), device=dev)
    projs = torch.rand(N, H, W, device=dev, generator=torch.Generator(dev).manual_seed(0))
    vol_a, vol_b = torch.empty(n, n, n, device=dev), torch.empty(n, n, n, device=dev)
    nbytes = int(lib.r2x_fdk_scratch_bytes(N, H, W))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    hx = helix_views(angles, sc, [{}] * N)
    bh = np.ascontiguousarray(hx.beta)
    bd, dbd = torch.from_numpy(bh).to(dev), torch.from_numpy(np.ascontiguousarray(hx.dbeta)).to(dev)
    tx, ty, dso = float(views[0].tanfovx), float(views[0].tanfovy), float(sc["DSO"])
    grid = (n, n, n, 2.0, 2.0, 2.0, 0.0, 0.0, 0.0)
    st = lambda: torch.cuda.current_stream(dev).cuda_stream
    plain = lambda: _lib.check(lib.r2x_fdk(st(), N, H, W, projs.data_ptr(), vm.data_ptr(), pm.data_ptr(), tx, ty, 1,
                                           0.0, 0.0, 0, None, 0.0, dso, *grid, vol_a.data_ptr(), scratch.data_ptr(),
                                           nbytes), "fdk")
    helical = lambda: _lib.check(lib.r2x_fdk_helical(st(), N, H, W, projs.data_ptr(), vm.data_ptr(), pm.data_ptr(), tx,
                                                     ty, 1, 0, dso, bd.data_ptr(), dbd.data_ptr(), bh.ctypes.data,
                                                     hx.z0, hx.h, hx.beta_lo, hx.beta_hi, hx.c_x, hx.c_y, 1.0, *grid,
                                                     vol_b.data_ptr(), scratch.data_ptr(), nbytes), "fdk_helical")
    res["circle_ms"] = _median_ms({"r2x_fdk": plain, "r2x_fdk_helical": helical}, a.reps)
    res["circle_max_rel_diff_q1"] = float((vol_a - vol_b).abs().max() / vol_a.abs().max())
    del projs, vol_a, vol_b, scratch

    # long: 8 turns x 360 views of 64 x 512 onto 256 x 256 x 512 at pitch factor 1
    sdet_v = 1.6
    travel = 8 * sdet_v * 5.0 / 7.0          # one isocentre detector height per turn
    sc, angles, geo = _helix(2880, 8, travel, (256, 256, 512), (64, 512), (2.0, 2.0, 4.0 + travel), (sdet_v, 4.0))
    N, H, W = 2880, 64, 512
    projs = torch.rand(N, H, W, device=dev, generator=torch.Generator(dev).manual_seed(1))
    call, hx = prepared(projs, angles, sc, geo)
    frac = window_fraction(sc, hx, float(scene.make_view(sc, 0.0).tanfovy))
    t_long = _median_ms({"fdk": call}, max(3, a.reps // 2))["fdk"]
    op = CTOperator(angles, sc, dev, view_geometry=geo)
    x = torch.rand(*sc["nVoxel"], device=dev, generator=torch.Generator(dev).manual_seed(2))
    t_cgls = _median_ms({"cgls_iter": lambda: op.At(op.A(x))}, 3)["cgls_iter"]
    res["long"] = {"views": N, "detector": [H, W], "grid": sc["nVoxel"], "fdk_helical_ms": t_long,
                   "window_fraction": frac, "full_window_estimate_ms": t_long / frac,
                   "cgls_iteration_ms": t_cgls}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "fdk_helical_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
