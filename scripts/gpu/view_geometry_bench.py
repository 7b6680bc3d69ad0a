"""Time the CT operators' per-view geometry table against their scalar path, and the scalar path against another build.

    python scripts/gpu/view_geometry_bench.py [--parent_lib OTHER/libr2xray.so] [--rounds 5] [--reps 5] [--out F.json]

Two workloads, each run through the C entry points with the same matrices:
  * FDK, 50 cone-beam views of 512^2 into 256^3: r2x_fdk (scalar) and r2x_fdk_views (a calibrated circle: DSO, DSD and
    offDetector_u jittered per view);
  * the projector, 150 views of 512^2 from 256^3: r2x_volume_project and r2x_volume_project_views (a two-turn helix).
`--parent_lib` also times the scalar entry points of another build of the library (e.g. the parent commit's), in the
same process.  The variants alternate round by round; each time is the median over rounds of the mean of `reps` calls
between CUDA events.  The scalar outputs of the two builds are compared bit for bit.  Prints one JSON line with the
card's name and power limit.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))

from r2_gaussian_b200 import _lib, scene                    # noqa: E402
from r2_gaussian_b200.projector import view_table           # noqa: E402


def _bind(path):
    lib = C.CDLL(path)
    for name in ("r2x_fdk", "r2x_fdk_views", "r2x_volume_project", "r2x_volume_project_views", "r2x_fdk_scratch_bytes"):
        if hasattr(lib, name):
            res, args = _lib.PROTOTYPES[name]
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    return lib


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, limit = (s.strip() for s in out[torch.cuda.current_device()].split(","))
        return name, limit
    except Exception as e:                      # report what could not be read, never a guess
        return torch.cuda.get_device_name(), f"unknown ({e})"


def _time(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def _calibrated(n, sc, seed=3):
    rng = np.random.RandomState(seed)
    du = sc["sDetector"][1] / sc["nDetector"][1]
    return [{"DSO": sc["DSO"] * (1 + 0.02 * rng.uniform(-1, 1)), "DSD": sc["DSD"] * (1 + 0.02 * rng.uniform(-1, 1)),
             "offDetector": [2.0 * du * rng.uniform(-1, 1), 0.0]} for _ in range(n)]


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--parent_lib", default=None)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("view_geometry_bench needs a CUDA device")
    _lib.load()
    libs = {"this": _bind(_lib.LIB_PATH)}
    if a.parent_lib:
        libs["parent"] = _bind(a.parent_lib)
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.RandomState(0)
    sc = scene.cone_beam_scanner(512, 256)
    nvox, size, ctr = sc["nVoxel"], sc["sVoxel"], sc["offOrigin"]
    step = 0.5 * 2.0 / 256
    vol = torch.from_numpy(rng.uniform(0, 1, tuple(nvox)).astype(np.float32)).cuda()

    # FDK: 50 views
    fa = np.linspace(0, 2 * math.pi, 51)[:-1]
    fviews = [scene.make_view(sc, float(t)) for t in fa]
    fvm = torch.from_numpy(np.stack([v.viewmatrix.reshape(16) for v in fviews])).cuda()
    fpm = torch.from_numpy(np.stack([v.projmatrix.reshape(16) for v in fviews])).cuda()
    cviews, ctab = view_table(fa, sc, _calibrated(50, sc))
    cvm = torch.from_numpy(np.stack([v.viewmatrix.reshape(16) for v in cviews])).cuda()
    cpm = torch.from_numpy(np.stack([v.projmatrix.reshape(16) for v in cviews])).cuda()
    ctab_d = torch.from_numpy(ctab).cuda()
    projs = torch.from_numpy(rng.uniform(0, 1, (50, 512, 512)).astype(np.float32)).cuda()
    nbytes = int(libs["this"].r2x_fdk_scratch_bytes(50, 512, 512))
    scratch = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    fout = {k: torch.empty(tuple(nvox), device="cuda") for k in ("this", "parent", "table")}
    v0 = fviews[0]

    def fdk_scalar(k):
        return lambda: _lib.check(libs[k].r2x_fdk(st, 50, 512, 512, projs.data_ptr(), fvm.data_ptr(), fpm.data_ptr(),
                                                  v0.tanfovx, v0.tanfovy, 1, 0.0, 0.0, 0, None, 0.0, 5.0, *nvox, *size,
                                                  *ctr, fout[k].data_ptr(), scratch.data_ptr(), nbytes), "r2x_fdk")

    def fdk_table():
        _lib.check(libs["this"].r2x_fdk_views(st, 50, 512, 512, projs.data_ptr(), cvm.data_ptr(), cpm.data_ptr(), 1, 0,
                                              *nvox, *size, *ctr, ctab_d.data_ptr(), ctab.ctypes.data,
                                              fout["table"].data_ptr(), scratch.data_ptr(), nbytes), "r2x_fdk_views")

    # projector: 150 views, helix of two turns for the table
    pa = np.linspace(0, 4 * math.pi, 151)[:-1]
    pviews = [scene.make_view(sc, float(t)) for t in pa]
    pvm = torch.from_numpy(np.stack([v.viewmatrix.reshape(16) for v in pviews])).cuda()
    helix = [{"offOrigin": [0.0, 0.0, 0.6 * (i / 150 - 0.5)]} for i in range(150)]
    hviews, htab = view_table(pa, sc, helix)
    hvm = torch.from_numpy(np.stack([v.viewmatrix.reshape(16) for v in hviews])).cuda()
    htab_d = torch.from_numpy(htab).cuda()
    pout = {k: torch.empty((150, 512, 512), device="cuda") for k in ("this", "parent", "table")}
    p0 = pviews[0]

    def proj_scalar(k):
        return lambda: _lib.check(libs[k].r2x_volume_project(st, *nvox, vol.data_ptr(), *size, *ctr, 150, 512, 512,
                                                             pvm.data_ptr(), p0.tanfovx, p0.tanfovy, 1, 0.0, 0.0, step,
                                                             pout[k].data_ptr()), "r2x_volume_project")

    def proj_table():
        _lib.check(libs["this"].r2x_volume_project_views(st, *nvox, vol.data_ptr(), *size, *ctr, 150, 512, 512,
                                                         hvm.data_ptr(), 1, step, htab_d.data_ptr(), htab.ctypes.data,
                                                         pout["table"].data_ptr()), "r2x_volume_project_views")

    variants = {"fdk_scalar_this": fdk_scalar("this"), "fdk_table": fdk_table,
                "project_scalar_this": proj_scalar("this"), "project_table": proj_table}
    if "parent" in libs:
        variants["fdk_scalar_parent"] = fdk_scalar("parent")
        variants["project_scalar_parent"] = proj_scalar("parent")
    for fn in variants.values():            # warm every shape
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    order = list(variants)
    for r in range(a.rounds):
        for k in (order if r % 2 == 0 else order[::-1]):
            times[k].append(_time(variants[k], a.reps))
    name, limit = _card()
    rep = {"gpu": name, "power_limit": limit, "rounds": a.rounds, "reps": a.reps,
           "ms_median": {k: float(np.median(v)) for k, v in times.items()},
           "ms_min": {k: float(np.min(v)) for k, v in times.items()},
           "ms_max": {k: float(np.max(v)) for k, v in times.items()}}
    if "parent" in libs:
        rep["fdk_scalar_same_bits"] = bool(torch.equal(fout["this"].view(torch.int32), fout["parent"].view(torch.int32)))
        rep["project_scalar_same_bits"] = bool(torch.equal(pout["this"].view(torch.int32),
                                                           pout["parent"].view(torch.int32)))
    print(json.dumps(rep))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rep, f, indent=1)
    return rep


if __name__ == "__main__":
    main()
