"""Marching cubes on the GPU (r2x_marching_cubes_count / _emit, `mesh.marching_cubes`):

    python scripts/gpu/mesh_bench.py [--reps 20] [--no-oracle]

Cases: smooth phantoms (three overlapping ellipsoids with a little noise, level 0.5) at 256^3 and 512^3, and the
density `query()` of a trained-like cloud (scene.make_cloud, 200k Gaussians) at 256^3, level at 30 % of its maximum.
Each pass is timed alone with CUDA events, median of --reps, with a 256 MB buffer written before every call so that L2
starts cold; the emit pass reruns on the scratch one count pass filled.  Also printed: triangles per second of count +
emit, the HBM floor of reading the volume twice (once per pass) at the H100 SXM data sheet's 3.35 TB/s, the end-to-end
`mesh.marching_cubes` time (both passes, the host read of the totals, allocations), and the CPU time of the numpy
oracle (tests/mesh_oracle.py) on the same volume, at 256^3 only (its int64 vertex-id array needs 3.2 GB at 512^3).
One JSON line per case and one with the card's name, power limit and SM clocks read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BYTES_PER_S = 3.35e12


def clocks() -> dict:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", "0"], capture_output=True, text=True, timeout=20)
        sm, smax = (float(x) for x in r.stdout.strip().splitlines()[0].split(","))
        return {"sm_clock_mhz": sm, "max_sm_clock_mhz": smax}
    except Exception:
        return {"sm_clock_mhz": None, "max_sm_clock_mhz": None}


def phantom(n, seed):
    import torch
    g = torch.linspace(-1, 1, n, device="cuda")
    X, Y, Z = torch.meshgrid(g, g, g, indexing="ij")
    vol = torch.zeros((n, n, n), device="cuda")
    for (cx, cy, cz), (a, b, c), w in (((0.0, 0.0, 0.0), (0.7, 0.55, 0.6), 1.0), ((0.25, -0.1, 0.2), (0.3, 0.25, 0.35), 0.6),
                                       ((-0.3, 0.2, -0.25), (0.2, 0.3, 0.2), -0.5)):
        q = ((X - cx) / a) ** 2 + ((Y - cy) / b) ** 2 + ((Z - cz) / c) ** 2
        vol += w * torch.clamp(1 - q, min=0)
    gen = torch.Generator("cuda").manual_seed(seed)
    return (vol + 0.02 * torch.randn(vol.shape, generator=gen, device="cuda")).contiguous()


def cloud_volume(n):
    import torch

    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.voxelization import GaussianVoxelizationSettings, GaussianVoxelizer
    c = scene.make_cloud(200_000, kind="trained", seed=3)
    t = lambda x: torch.as_tensor(x, dtype=torch.float32, device="cuda").contiguous()
    vs = GaussianVoxelizationSettings(1.0, n, n, n, 2.0, 2.0, 2.0, 0.0, 0.0, 0.0, False, False)
    with torch.no_grad():
        vol, _ = GaussianVoxelizer(vs)(t(c.means), t(c.density), t(c.scales), t(c.rotations))
    return vol.contiguous()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    import numpy as np
    import torch

    import secondary
    from r2_gaussian_b200 import mesh
    from r2_gaussian_b200._lib import check, load

    if not torch.cuda.is_available():
        raise SystemExit("mesh_bench needs a CUDA device")
    dev = torch.device("cuda")
    lib = load()
    flush = torch.empty(64 << 20, dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream

    def timed(fn):
        fn()
        ms = []
        for _ in range(a.reps):
            flush.fill_(1.0)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            e.synchronize()
            ms.append(s.elapsed_time(e))
        ms.sort()
        return ms[len(ms) // 2]

    cases = [("phantom_256", lambda: phantom(256, 1), 0.5), ("phantom_512", lambda: phantom(512, 2), 0.5),
             ("query_cloud_256", lambda: cloud_volume(256), None)]
    for name, make, level in cases:
        vol = make()
        if level is None:
            level = 0.3 * float(vol.max())
        nx, ny, nz = vol.shape
        nbytes = int(lib.r2x_marching_cubes_scratch_bytes(nx, ny, nz))
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        totals = torch.empty(2, dtype=torch.int64, device=dev)
        count = lambda: check(lib.r2x_marching_cubes_count(stream, nx, ny, nz, vol.data_ptr(), level, totals.data_ptr(),
                                                           scratch.data_ptr(), nbytes), "count")
        count()
        V, T = (int(x) for x in totals.tolist())
        verts = torch.empty((V, 3), dtype=torch.float32, device=dev)
        faces = torch.empty((T, 3), dtype=torch.int32, device=dev)
        emit = lambda: check(lib.r2x_marching_cubes_emit(stream, nx, ny, nz, vol.data_ptr(), level, V, T,
                                                         verts.data_ptr(), faces.data_ptr(), scratch.data_ptr(), nbytes),
                             "emit")
        t_count = timed(count)
        t_emit = timed(emit)
        t_api = timed(lambda: mesh.marching_cubes(vol, level))
        gv, gf = mesh.marching_cubes(vol, level)
        row = {"case": name, "shape": [nx, ny, nz], "level": level, "vertices": V, "triangles": T,
               "count_ms": t_count, "emit_ms": t_emit, "marching_cubes_ms": t_api,
               "triangles_per_s": T / ((t_count + t_emit) * 1e-3),
               "hbm_floor_two_reads_ms": 2 * 4 * vol.numel() / HBM_BYTES_PER_S * 1e3}
        if not a.no_oracle and vol.numel() <= 256 ** 3:
            import mesh_oracle as mo
            host = vol.cpu().numpy()
            mo.marching_cubes(host[:8, :8, :8], level)          # table generation outside the timing
            t0 = time.perf_counter()
            ov, of = mo.marching_cubes(host, level)
            row["oracle_cpu_ms"] = (time.perf_counter() - t0) * 1e3
            row["oracle_equal"] = bool(np.array_equal(gv.cpu().numpy().view(np.uint32), ov.view(np.uint32))
                                       and np.array_equal(gf.cpu().numpy(), of))
        print(json.dumps(row), flush=True)
        del vol, scratch, verts, faces, gv, gf
        torch.cuda.empty_cache()
    print(json.dumps({**secondary.card(dev), **clocks()}))


if __name__ == "__main__":
    main()
