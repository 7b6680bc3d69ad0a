"""The work-plan arithmetic shared by the binning and render kernels (chunk policy per consumer, equal-slice cut of a
tile list; r2_gaussian_b200/csrc/r2x_binning.cuh) is __host__ __device__: tests/host/plan_check.cu is cross-compiled for
sm_90a and its host code run on the CPU."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_chunk_policy_and_equal_slices(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path / "plan_check")
    src = os.path.join(ROOT, "tests", "host", "plan_check.cu")
    r = subprocess.run([nvcc, "-std=c++17", "-O1", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe, src],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "plan_check: ok" in r.stdout
