"""Where the time of `process_raw_data` goes on the GPU, for a backpack-sized and a kingsnake-sized volume.

    python scripts/gpu/raw_data_bench.py [--repeats 3] [--cpu]

The volumes are seeded stand-ins of the reference's largest cases, made in memory (disk reads are not timed):
  * backpack: 512 x 512 x 373 uint16, spacing [0.9766, 0.9766, 1.25], expand -> 500 x 500 x 466 -> 500^3 -> 256^3;
  * kingsnake: 1024 x 1024 x 795 uint8, spacing [0.6348, 0.6348, 1.376], expand -> 650 x 650 x 1094 -> 1094^3 -> 256^3.
Each chain runs once to warm up, then `--repeats` times.  Per case, the best of the repeats of:
  * upload_s: the host-to-device copy of the raw volume in its own dtype, from pageable memory (CUDA events);
  * resample_kernels_s / resize_kernels_s: the two zooms on device-resident sources (fill, 3 prefilter passes,
    gather, and the allocation of their buffers), CUDA events;
  * chain_s: the whole chain from the host array to the float32 cube on the host (min / max, upload, both zooms,
    download, clip, transpose), host clock after a synchronise;
  * peak_GB: torch.cuda.max_memory_allocated over one chain.
With --cpu, also the reference's scipy chain on the backpack case (single-threaded float64, one run).  Prints one JSON
line with the card name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CASES = {
    "backpack": dict(shape=(512, 512, 373), dtype="uint16", spacing=[0.9766, 0.9766, 1.25], transpose=[1, 0, 2]),
    "kingsnake": dict(shape=(1024, 1024, 795), dtype="uint8", spacing=[0.03174 * 20, 0.03174 * 20, 0.0688 * 20],
                      transpose=[0, 1, 2]),
}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def volume(shape, dtype, seed):
    """A seeded raw volume as the reference holds it after fromfile / reshape / transpose(2, 1, 0): a strided view."""
    import numpy as np

    rng = np.random.default_rng(seed)
    nx, ny, nz = shape
    raw = rng.integers(0, 40, (nz, ny, nx), dtype=np.dtype(dtype))
    gz, gy, gx = (np.linspace(-1, 1, n, dtype=np.float32) for n in (nz, ny, nx))
    top = np.iinfo(np.dtype(dtype)).max * 0.8
    for z0 in range(0, nz, 64):
        fz = np.exp(-(gz[z0:z0 + 64] / 0.6) ** 2)[:, None, None]
        raw[z0:z0 + 64] += (fz * np.exp(-(gy / 0.5) ** 2)[None, :, None] * np.exp(-(gx / 0.7) ** 2)[None, None, :]
                            * np.float32(top)).astype(raw.dtype)
    return raw.transpose(2, 1, 0)


def time_case(name, spec, repeats):
    import numpy as np
    import torch

    from r2_gaussian_b200 import process_raw_data as prd
    from r2_gaussian_b200.resample import device_source, zoom_device, zoom_placed

    src = volume(spec["shape"], spec["dtype"], 0)
    case = {"transpose": spec["transpose"], "z_invert": False}

    def chain():
        place = prd.normalising_place(src, name)
        vol = prd.reshape_vol(src, place, spec["spacing"], 256, "expand", zoom_placed)
        return prd._finish(vol, case).astype(np.float32)

    first = chain()                                    # warm-up
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    chain_s = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = chain()
        torch.cuda.synchronize()
        chain_s.append(time.perf_counter() - t0)
    peak = torch.cuda.max_memory_allocated()
    assert out.tobytes() == first.tobytes()

    factors, places = prd.reshape_plan(src.shape, spec["spacing"], 256, "expand")
    place = prd.normalising_place(src, name)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    up, a_s, b_s = [], [], []
    for _ in range(repeats):
        torch.cuda.synchronize()
        ev[0].record()
        dev = device_source(src)                       # the raw volume in its own dtype, pageable host memory
        ev[1].record()
        res = zoom_device(*dev, factors[0], place)
        ev[2].record()
        vol = zoom_placed(res, factors[1], places[0])
        ev[3].record()
        ev[3].synchronize()
        up.append(ev[0].elapsed_time(ev[1]) / 1e3)
        a_s.append(ev[1].elapsed_time(ev[2]) / 1e3)
        b_s.append(ev[2].elapsed_time(ev[3]) / 1e3)
        dev = res = vol = None
    return {"chain_s": round(min(chain_s), 4), "upload_s": round(min(up), 4), "resample_kernels_s": round(min(a_s), 4),
            "resize_kernels_s": round(min(b_s), 4), "peak_GB": round(peak / 1e9, 2),
            "input_GB": round(src.nbytes / 1e9, 3)}


def time_scipy_backpack():
    import numpy as np

    import raw_data_oracle as oracle

    spec = CASES["backpack"]
    src = volume(spec["shape"], spec["dtype"], 0)
    t0 = time.perf_counter()
    data = src.astype(float)
    data = (data - data.min()) / (data.max() - data.min())
    out = oracle.reference_reshape_vol(data.clip(0.0, 1.0), spec["spacing"], 256, "expand").clip(0.0, 1.0)
    np.ascontiguousarray(out.transpose(spec["transpose"])).astype(np.float32)
    return round(time.perf_counter() - t0, 2)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--cpu", action="store_true", help="also time the reference's scipy chain on the backpack case")
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("raw_data_bench needs a CUDA device")
    res = {"card": card()}
    for name, spec in CASES.items():
        res[name] = time_case(name, spec, a.repeats)
    if a.cpu:
        res["backpack"]["scipy_chain_s"] = time_scipy_backpack()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
