"""Build libr2xray.so (the sm_90a CUDA kernels + C ABI) in-tree with nvcc.

    python -m r2_gaussian_b200.build [--force] [--verbose]

The shared library is written next to this file (git-ignored build product).  No torch headers are involved: the
C ABI takes raw device pointers.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "libr2xray.so")
SOURCES = ["r2x_api.cu", "r2x_binning.cu", "r2x_binning2.cu", "r2x_raster.cu", "r2x_voxel.cu", "r2x_knn.cu", "r2x_train.cu", "r2x_comm.cu", "r2x_compact.cu", "r2x_fdk.cu", "r2x_project.cu", "r2x_backproject.cu", "r2x_pose.cu", "r2x_detector.cu", "r2x_tv.cu", "r2x_prepare.cu", "r2x_zoom.cu", "r2x_mesh.cu", "r2x_volrender.cu", "r2x_scene.cu", "r2x_stripes.cu", "r2x_mar.cu"]
HEADERS = ["r2x_common.cuh", "r2x_matcalc.cuh", "r2x_binning.cuh", "r2x_raster.cuh", "r2x_voxel.cuh", "r2x_project.cuh",
           "../../include/r2x.h"]

NVCC_FLAGS = [
    "-std=c++17", "-O3",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-Xcompiler", "-fPIC", "-Xptxas", "-v",
]


def find_nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; cannot build libr2xray.so")


def _newest(paths):
    return max(os.path.getmtime(p) for p in paths)


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    deps = [os.path.join(CSRC, s) for s in SOURCES] + [os.path.normpath(os.path.join(CSRC, h)) for h in HEADERS]
    return _newest(deps) > os.path.getmtime(LIB)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    nvcc = find_nvcc()
    os.makedirs(OBJ, exist_ok=True)
    hdr_time = _newest([os.path.normpath(os.path.join(CSRC, h)) for h in HEADERS])

    def compile_one(src):
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        if not force and os.path.exists(o) and os.path.getmtime(o) > max(os.path.getmtime(s), hdr_time):
            return o, ""
        cmd = [nvcc, *NVCC_FLAGS, "-c", s, "-o", o]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return o, r.stderr

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        results = list(ex.map(compile_one, SOURCES))
    if verbose:
        for _, log in results:
            if log:
                print(log)
    objs = [o for o, _ in results]
    r = subprocess.run([nvcc, "-shared", "-o", LIB, *objs, "-lcudart"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
