"""Draw a scene's scanner geometry to PNG on the GPU -- what the reference's `scripts/visualize_scene.py` shows in an
open3d window, rendered headless with the project's rasterizer (`scene_view`).

    python -m r2_gaussian_b200.visualize_scene --output scene.png [options] SOURCE

SOURCE is one of (as in `extract_mesh`)
    -s <scene>                           vol_gt's mesh and the scene's train cameras
    --vol X.npy [-s <scene>]             the mesh of any volume (with -s: on the scene's grid, with its cameras)
    -m <model> [--iteration -1] [--resolution N]
                                         the trained model's query() mesh, its cameras with the learned pose and detector
                                         corrections, and (thinner) the nominal cameras

    -m <model> --gaussians [--n_gaussian N] [--sort_gaussians {no,density,scale}]
                                         the trained model's Gaussians as shaded 1-sigma ellipsoids (the reference's
                                         show_gaussians) instead of a mesh: those of non-zero density, optionally sorted
                                         by density or mean scale (largest first), the first N of them, gray by density

Drawn: the marching-cubes mesh at --mc_thresh (0.5), the volume's box (red), the unit box [-1, 1]^3 (blue), a frame at
offOrigin, and per drawn train view its frustum in a colour from --cmap, its projection on the image plane (at depth
--cam_scale, or with --true_detector at the detector: DSD from the source, sDetector in size, the offset honoured) and a
small frame (--use_view_geometry: each view's own source and detector).  Without --camera the view is `scene_view.default_view`; --orbit N turns it about the scan axis (+z) and
writes <stem>_0000.png ...; --save_npy also writes the float frames [N, H, W, 3] to <stem>.npy.  Prints one JSON line:
source, triangles, lines, cameras, frames, width, height, seconds, outputs (and with --gaussians: gaussians, the number
drawn).  GPU only.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time

import numpy as np

from .extract_mesh import add_source_arguments, check_source_arguments, load_model, load_volume
from .scene_view import SORT_GAUSSIANS

CAMERA_LUT = np.array([[0.0, 0.0, 1.0], [1.0, 0.0, 0.0]])   # blue -> red: the default camera colours


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Scanner geometry of a scene (volume mesh, boxes, camera frusta and "
                                             "projections) rasterized on the GPU and written as PNG")
    ap.add_argument("--output", required=True, help="PNG file to write (with --orbit: the stem of the frame files)")
    add_source_arguments(ap)
    ap.add_argument("--use_offDetector", action="store_true", help="cameras with the scanner's detector offset")
    ap.add_argument("--use_view_geometry", action="store_true",
                    help="each camera at its own source and detector (the frames' per-view DSO, DSD, offOrigin, "
                         "offDetector: a helix shows as one); implies --use_offDetector")
    ap.add_argument("--mc_thresh", type=float, default=0.5, help="marching-cubes level of the mesh (default 0.5)")
    ap.add_argument("--cam_scale", type=float, default=1.0, help="size of the camera glyphs (default 1.0)")
    ap.add_argument("--width", type=int, default=1000, help="image width in pixels (default 1000)")
    ap.add_argument("--height", type=int, default=800, help="image height in pixels (default 800)")
    ap.add_argument("--camera", type=float, nargs=9, default=None,
                    metavar=("PX", "PY", "PZ", "FX", "FY", "FZ", "UX", "UY", "UZ"),
                    help="position, focal point and view-up in scene units")
    ap.add_argument("--view_angle", type=float, default=30.0, help="vertical view angle in degrees (default 30)")
    ap.add_argument("--orbit", type=int, default=None, help="render N frames turning about the scan axis (+z)")
    ap.add_argument("--views", type=int, default=1, help="draw every k-th train camera (default 1: all)")
    ap.add_argument("--no_images", action="store_true", help="draw the frusta without the projections")
    ap.add_argument("--cmap", default=None, help="a .npy LUT [K, 3] in [0, 1] for the camera colours, or 'gray' "
                                                  "(default: blue -> red)")
    ap.add_argument("--true_detector", action="store_true",
                    help="draw each image plane at the real detector instead of at depth --cam_scale")
    ap.add_argument("--supersample", type=int, default=1, help="k x k box-filter supersampling (default 1: off)")
    ap.add_argument("--background", type=float, nargs=3, default=[1.0, 1.0, 1.0], metavar=("R", "G", "B"))
    ap.add_argument("--save_npy", action="store_true", help="also write the float RGB frames to <stem>.npy")
    ap.add_argument("--gaussians", action="store_true",
                    help="with -m: draw the model's Gaussians as ellipsoids instead of the density's mesh")
    ap.add_argument("--n_gaussian", type=int, default=None, help="with --gaussians: draw at most N (default: all)")
    ap.add_argument("--sort_gaussians", default=None, choices=SORT_GAUSSIANS,
                    help="with --gaussians: which N to draw -- the first in the model ('no', the default), the densest "
                         "or the largest")
    a = ap.parse_args(argv)
    from .mesh import finite_level
    from .scene_view import MAX_SIDE
    from .volume_render import look_at, lut_from

    check_source_arguments(ap, a)
    if not finite_level(a.mc_thresh):
        ap.error(f"--mc_thresh must be a finite float32, got {a.mc_thresh}")
    if not (math.isfinite(a.cam_scale) and a.cam_scale > 0):
        ap.error(f"--cam_scale must be finite and > 0, got {a.cam_scale}")
    if a.supersample < 1:
        ap.error(f"--supersample must be >= 1, got {a.supersample}")
    if not (1 <= a.width * a.supersample <= MAX_SIDE and 1 <= a.height * a.supersample <= MAX_SIDE):
        ap.error(f"--width and --height (times --supersample) must be from 1 to {MAX_SIDE}, got {a.width} {a.height}")
    if a.views < 1:
        ap.error(f"--views must be >= 1, got {a.views}")
    if a.orbit is not None and a.orbit < 1:
        ap.error(f"--orbit must be >= 1, got {a.orbit}")
    if not 0 < a.view_angle < 180:
        ap.error(f"--view_angle must be in (0, 180) degrees, got {a.view_angle}")
    if not all(math.isfinite(c) and 0 <= c <= 1 for c in a.background):
        ap.error(f"--background must be 3 numbers in [0, 1], got {a.background}")
    try:
        a.lut = CAMERA_LUT if a.cmap is None else lut_from(a.cmap)
    except (OSError, ValueError) as e:
        ap.error(f"--cmap {a.cmap}: {e}")
    if a.camera is not None:
        if not all(math.isfinite(c) for c in a.camera):
            ap.error("--camera must be 9 finite numbers")
        try:
            look_at(a.camera[0:3], a.camera[3:6], a.camera[6:9], a.width, a.height, a.view_angle)
        except ValueError as e:
            ap.error(f"--camera: {e}")
    if (a.true_detector or a.use_offDetector or a.use_view_geometry) and a.source_path is None and a.model_path is None:
        ap.error("--true_detector, --use_offDetector and --use_view_geometry need cameras: give -s <scene> or -m <model>")
    if a.gaussians:
        if a.model_path is None:
            ap.error("--gaussians draws a trained model's Gaussians: give -m <model>")
        if a.resolution is not None or a.vol is not None:
            ap.error("--gaussians draws no volume: --resolution and --vol do not apply")
        if a.n_gaussian is not None and a.n_gaussian < 1:
            ap.error(f"--n_gaussian must be >= 1, got {a.n_gaussian}")
    elif a.n_gaussian is not None or a.sort_gaussians is not None:
        ap.error("--n_gaussian and --sort_gaussians apply to --gaussians")
    if a.sort_gaussians is None:
        a.sort_gaussians = "no"
    return a


def camera_colour(lut, i: int, n: int) -> np.ndarray:
    """The LUT colour of view i of n, at t = i / n (the reference's cmap(i / n)), interpolated as volume_render's."""
    K = len(lut)
    if K == 1:
        return lut[0]
    pos = i / n * (K - 1)
    j = min(int(math.floor(pos)), K - 2)
    w = pos - j
    return (1 - w) * lut[j] + w * lut[j + 1]


def _cameras(a):
    """(list of (nominal, drawn) dataset cameras of the drawn train views, their Scene or None) -- drawn carries the
    model's learned corrections with -m, else it is the nominal camera."""
    from .dataset import Scene

    if a.model_path is None:
        if a.source_path is None:
            return [], None
        scene = Scene(a.source_path, eval=False, shuffle=False, device="cuda", use_offDetector=a.use_offDetector,
                      use_view_geometry=a.use_view_geometry)
        cams = scene.getTrainCameras()
        return [(c, c) for c in cams[::a.views]], scene
    from .test import correction_modules, load_settings, resolve_iteration
    from .trainer import evaluation_cameras

    settings = load_settings(a.model_path)
    source = a.source_path or settings.get("source_path")
    off = a.use_offDetector or bool(settings.get("use_offDetector", False))
    per_view = a.use_view_geometry or bool(settings.get("use_view_geometry", False))
    scene = Scene(source, eval=False, shuffle=False, device="cuda", use_offDetector=off, use_view_geometry=per_view)
    _, pickle_path = resolve_iteration(a.model_path, a.iteration)
    try:
        pose, det = correction_modules(os.path.dirname(pickle_path), scene)
    except ValueError as e:
        raise SystemExit(str(e)) from e
    import torch
    with torch.no_grad():
        corrected = dict(evaluation_cameras(scene, pose, det))["train"]
    nominal = scene.getTrainCameras()
    return list(zip(nominal, corrected))[::a.views], scene


def build(a, vol, cfg, gaussians=None):
    """(primitives, triangles, cameras, Gaussians drawn or None) of everything the CLI draws: the mesh of `vol`, or
    with `gaussians` (a GaussianModel) their ellipsoids."""
    from .mesh import marching_cubes
    from .scene_view import (BLUE, LINE_WIDTH, RED, axes, box, camera_glyph, concat, gaussian_ellipsoids,
                             mesh_triangles)

    if gaussians is None:
        verts, faces = marching_cubes(vol, a.mc_thresh)
        parts, n_tris, n_gauss = [mesh_triangles(verts, faces, vol, cfg)], int(faces.shape[0]), None
    else:
        ell, _ = gaussian_ellipsoids(gaussians, a.n_gaussian, a.sort_gaussians)
        parts, n_tris, n_gauss = [ell], 0, len(ell)
    if cfg is not None:
        parts += [box(cfg["offOrigin"], cfg["sVoxel"], RED), box((0, 0, 0), (2, 2, 2), BLUE),
                  axes(cfg["offOrigin"], float(cfg["sVoxel"][0]) / 2)]
    else:
        n = np.asarray(vol.shape, np.float64)
        parts.append(box((n - 1) / 2, n - 1, RED))
    pairs, scene = _cameras(a)
    n_all = len(scene.getTrainCameras()) if scene is not None else 0
    depth = float(scene.scanner_cfg["DSD"]) if (scene is not None and a.true_detector) else None
    for i, (nom, cam) in enumerate(pairs):
        col = camera_colour(a.lut, i * a.views, n_all)
        img = None if a.no_images else cam.original_image[0]
        if depth is not None and scene.use_view_geometry:   # the view's own DSD, from its field of view
            depth = float(scene.scanner_cfg["sDetector"][1]) / 2.0 / math.tan(float(nom.FoVx) / 2.0)
        parts.append(camera_glyph(cam, a.cam_scale, col, image=img, plane_depth=depth))
        if a.model_path is not None:
            parts.append(camera_glyph(nom, a.cam_scale, col, plane_depth=depth, width=LINE_WIDTH / 2))
    return concat(*parts), n_tris, len(pairs), n_gauss


def run(argv=None):
    """(report, frames, primitives, cameras): the JSON report, the CUDA float32 [N, H, W, 3] frames it wrote and what
    they were rendered from."""
    a = parse_args(argv)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("the scene view needs a CUDA device: the rasterizer runs on the GPU and has no CPU fallback")
    from .scene_view import LINE, default_view, render, scan_orbit
    from .volume_render import look_at, to_uint8, write_png

    if a.gaussians:
        source, gaussians, cfg, _ = load_model(a)
        vol = None
    else:
        (source, vol, cfg), gaussians = load_volume(a), None
    try:
        prims, n_tris, n_cams, n_gauss = build(a, vol, cfg, gaussians)
    except ValueError as e:
        raise SystemExit(str(e)) from e
    if a.camera is not None:
        cam = look_at(a.camera[0:3], a.camera[3:6], a.camera[6:9], a.width, a.height, a.view_angle)
    else:
        cam = default_view(prims, a.width, a.height, a.view_angle)
    cams = scan_orbit(cam, a.orbit) if a.orbit is not None else [cam]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    frames = render(prims, cams, background=a.background, supersample=a.supersample)
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
    stem = os.path.splitext(a.output)[0]
    images = to_uint8(frames).cpu().numpy()
    outputs = [a.output] if a.orbit is None else [f"{stem}_{k:04d}.png" for k in range(len(cams))]
    for path, img in zip(outputs, images):
        write_png(path, img)
    if a.save_npy:
        np.save(stem + ".npy", frames.cpu().numpy())
        outputs.append(stem + ".npy")
    report = {"source": source, "triangles": n_tris, "lines": int((prims.meta[:, 0] == LINE).sum()),
              "cameras": n_cams, "frames": len(cams), "width": a.width, "height": a.height, "seconds": seconds,
              "outputs": outputs}
    if n_gauss is not None:
        report["gaussians"] = n_gauss
    print(json.dumps(report))
    return report, frames, prims, cams


def main(argv=None) -> dict:
    return run(argv)[0]


if __name__ == "__main__":
    main(sys.argv[1:])
