"""Render a CT volume to PNG on the GPU -- what the reference's `scripts/plot_volume.py` draws with pyvista / VTK,
with the project's own ray caster (`volume_render`).

    python -m r2_gaussian_b200.render_volume --output out.png [options] SOURCE

SOURCE is one of (as in `extract_mesh`)
    -s <scene>                           the scene's ground-truth volume (vol_gt)
    --vol X.npy [-s <scene>]             any 3-D volume (with -s: of the scene's nVoxel shape)
    -m <model> [--iteration -1] [--resolution N]
                                         the trained model's density queried on the scene's grid, or on N^3 samples

The camera lives in index space (sample vol[i, j, k] at the point (i, j, k)), so plot_volume.py's `cpos` is
`--camera PX PY PZ FX FY FZ UX UY UZ` unchanged; without --camera the view is `volume_render.default_camera`.
`--zero_lower_half x` is plot_volume.py's `volume[:n // 2] = 0`, done on the device.  `--orbit N` writes
<stem>_0000.png ... <stem>_{N-1}.png around the view-up axis; `--save_npy` also writes the float RGBA frames
[N, H, W, 4] to <stem>.npy.  Prints one JSON line: source, shape, mode, frames, width, height, seconds, outputs.
GPU only.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time

import numpy as np

from .extract_mesh import add_source_arguments, check_source_arguments, load_volume

AXES = {"x": 0, "y": 1, "z": 2}


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Volume rendering (emission-absorption or MIP ray casting on the GPU) of "
                                             "a scene's volume, a reconstruction or a trained model, written as PNG")
    ap.add_argument("--output", required=True, help="PNG file to write (with --orbit: the stem of the frame files)")
    add_source_arguments(ap)
    ap.add_argument("--mode", choices=["composite", "mip"], default="composite",
                    help="composite: emission-absorption (default); mip: maximum intensity projection")
    ap.add_argument("--clim", type=float, nargs=2, default=[0.0, 1.0], metavar=("LO", "HI"),
                    help="values mapped to the ends of the colour map and to opacity 0 and 1 (default 0 1)")
    ap.add_argument("--cmap", default="gray", help="'gray' or a .npy LUT of shape [K, 3] with values in [0, 1]")
    ap.add_argument("--window_size", type=int, nargs=2, default=[800, 1000], metavar=("W", "H"),
                    help="image width and height in pixels (default 800 1000, as plot_volume.py)")
    ap.add_argument("--camera", type=float, nargs=9, default=None,
                    metavar=("PX", "PY", "PZ", "FX", "FY", "FZ", "UX", "UY", "UZ"),
                    help="position, focal point and view-up in index space (plot_volume.py's cpos, flattened)")
    ap.add_argument("--view_angle", type=float, default=30.0, help="vertical view angle in degrees (default 30)")
    ap.add_argument("--parallel_scale", type=float, default=None,
                    help="orthographic projection: half the image height in voxels")
    ap.add_argument("--step", type=float, default=0.5, help="sample spacing along a ray, in voxels (default 0.5)")
    ap.add_argument("--opacity_unit", type=float, default=None,
                    help="opacity unit distance in voxels (default: box diagonal / (mean axis size - 1))")
    ap.add_argument("--background", type=float, nargs=3, default=[0.0, 0.0, 0.0], metavar=("R", "G", "B"))
    ap.add_argument("--zero_lower_half", choices=sorted(AXES), default=None,
                    help="set vol[:n // 2] = 0 along this axis to show the inside (plot_volume.py uses x)")
    ap.add_argument("--orbit", type=int, default=None, help="render N frames around the view-up axis")
    ap.add_argument("--save_npy", action="store_true", help="also write the float RGBA frames to <stem>.npy")
    a = ap.parse_args(argv)
    from .volume_render import check_clim, look_at, lut_from

    check_source_arguments(ap, a)
    try:
        check_clim(a.clim)
    except ValueError as e:
        ap.error(f"--clim: {e}")
    try:
        a.lut = lut_from(a.cmap)
    except (OSError, ValueError) as e:
        ap.error(f"--cmap {a.cmap}: {e}")
    w, h = a.window_size
    if w < 1 or h < 1:
        ap.error(f"--window_size must be at least 1 1, got {w} {h}")
    for name in ("step", "opacity_unit", "parallel_scale"):
        val = getattr(a, name)
        if val is not None and not (math.isfinite(val) and val > 0):
            ap.error(f"--{name} must be finite and > 0, got {val}")
    if not 0 < a.view_angle < 180:
        ap.error(f"--view_angle must be in (0, 180) degrees, got {a.view_angle}")
    if not all(math.isfinite(c) for c in a.background):
        ap.error(f"--background must be finite, got {a.background}")
    if a.orbit is not None and a.orbit < 1:
        ap.error(f"--orbit must be >= 1, got {a.orbit}")
    if a.camera is not None:
        if not all(math.isfinite(c) for c in a.camera):
            ap.error("--camera must be 9 finite numbers")
        try:
            look_at(a.camera[0:3], a.camera[3:6], a.camera[6:9], w, h, a.view_angle, a.parallel_scale)
        except ValueError as e:
            ap.error(f"--camera: {e}")
    return a


def run(argv=None):
    """(report, frames): the JSON report and the CUDA float32 [N, H, W, 4] frames it wrote."""
    a = parse_args(argv)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("volume rendering needs a CUDA device: the ray caster runs on the GPU and has no CPU fallback")
    from .mesh import _device_volume
    from .volume_render import default_camera, look_at, orbit, render, to_uint8, write_png

    source, vol, _ = load_volume(a)
    try:
        v = _device_volume(vol, what="render")
        if min(v.shape) < 2:
            raise ValueError(f"render: every axis needs >= 2 samples, got shape {tuple(v.shape)}")
    except ValueError as e:
        raise SystemExit(str(e)) from e
    if a.zero_lower_half is not None:
        ax = AXES[a.zero_lower_half]
        if v is vol:
            v = v.clone()
        v.narrow(ax, 0, v.shape[ax] // 2).zero_()
    w, h = a.window_size
    if a.camera is not None:
        cam = look_at(a.camera[0:3], a.camera[3:6], a.camera[6:9], w, h, a.view_angle, a.parallel_scale)
    else:
        cam = default_camera(v.shape, w, h, a.view_angle, a.parallel_scale)
    cams = orbit(cam, a.orbit) if a.orbit is not None else [cam]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    frames = render(v, cams, mode=a.mode, clim=a.clim, lut=a.lut, step=a.step, opacity_unit=a.opacity_unit,
                    background=a.background)
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
    stem = os.path.splitext(a.output)[0]
    images = to_uint8(frames[..., :3]).cpu().numpy()
    outputs = [a.output] if a.orbit is None else [f"{stem}_{k:04d}.png" for k in range(len(cams))]
    for path, img in zip(outputs, images):
        write_png(path, img)
    if a.save_npy:
        np.save(stem + ".npy", frames.cpu().numpy())
        outputs.append(stem + ".npy")
    report = {"source": source, "shape": [int(n) for n in v.shape], "mode": a.mode, "frames": len(cams), "width": w,
              "height": h, "seconds": seconds, "outputs": outputs}
    print(json.dumps(report))
    return report, frames


def main(argv=None) -> dict:
    return run(argv)[0]


if __name__ == "__main__":
    main(sys.argv[1:])
