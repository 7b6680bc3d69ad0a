"""Extract an isosurface mesh of a CT volume and write it as PLY -- what the reference's `scripts/visualize_scene.py
--mc_thresh` computes through `create_vol_mesh` (skimage's marching cubes), on the GPU.

    python -m r2_gaussian_b200.extract_mesh --output mesh.ply [--level 0.5] SOURCE

SOURCE is one of
    -s <scene>                           the scene's ground-truth volume (vol_gt), in scene units
    --vol X.npy -s <scene>               any volume of the scene's nVoxel shape (recon's ct_pred.npy, test's
                                         vol_pred.npy), in scene units
    --vol X.npy                          any 3-D volume, in index space
    -m <model> [--iteration -1] [--resolution N]
                                         the trained model's density queried on the scene's grid, or on N^3 samples
                                         over the same box (finer than the scanner grid if N is larger), in scene units

Scene units place each sample at its voxel centre (`mesh.to_scene`).  The model's scene is the one it was trained on
(its recorded settings) unless -s names another.  Pose and detector corrections do not change the volume.  Prints one
JSON line: source, level, shape, vertices, triangles, seconds.  GPU only.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Isosurface mesh (marching cubes on the GPU) of a scene's volume, a "
                                             "reconstruction or a trained model, written as binary PLY")
    ap.add_argument("--output", required=True, help="PLY file to write")
    ap.add_argument("--level", type=float, default=0.5, help="iso level: samples > level are inside (default 0.5)")
    add_source_arguments(ap)
    a = ap.parse_args(argv)
    from .mesh import finite_level

    if not finite_level(a.level):
        ap.error(f"--level must be a finite float32, got {a.level}")
    check_source_arguments(ap, a)
    return a


def add_source_arguments(ap):
    """The volume source options: -s, --vol, -m, --iteration, --resolution."""
    ap.add_argument("-s", "--source_path", default=None, help="scene directory or NAF pickle")
    ap.add_argument("--vol", default=None, help=".npy volume [nx, ny, nz]")
    ap.add_argument("-m", "--model_path", default=None, help="output directory of a trainer run")
    ap.add_argument("--iteration", type=int, default=-1, help="with -m: saved iteration (-1: the last one)")
    ap.add_argument("--resolution", type=int, default=None, help="with -m: query N^3 samples instead of nVoxel")


def check_source_arguments(ap, a):
    """Refuse (ap.error) conflicting or missing sources, options that do not apply to the source, missing paths and a
    missing --output directory."""
    if a.model_path is not None and a.vol is not None:
        ap.error("give either -m or --vol, not both")
    if a.model_path is None and a.vol is None and a.source_path is None:
        ap.error("no volume: give -s <scene>, --vol X.npy [-s <scene>] or -m <model>")
    if a.resolution is not None and a.model_path is None:
        ap.error("--resolution applies to -m (a model can be queried on any grid; a stored volume cannot)")
    if a.resolution is not None and a.resolution < 2:
        ap.error(f"--resolution must be >= 2, got {a.resolution}")
    if a.model_path is None and a.iteration != -1:
        ap.error("--iteration applies to -m")
    for path, what in ((a.vol, "--vol"), (a.source_path, "-s"), (a.model_path, "-m")):
        if path is not None and not os.path.exists(path):
            ap.error(f"{what} {path} does not exist")
    out_dir = os.path.dirname(os.path.abspath(a.output))
    if not os.path.isdir(out_dir):
        ap.error(f"--output: directory {out_dir} does not exist")


def _read_volume(path: str) -> np.ndarray:
    vol = np.load(path)
    if vol.ndim != 3:
        raise SystemExit(f"--vol {path}: expected a 3-D volume, got shape {vol.shape}")
    return vol


def load_volume(a):
    """(source label, volume (array or CUDA tensor), scanner_cfg of the grid or None for index space)."""
    from .dataset import read_scene

    if a.model_path is None:
        cfg = None
        if a.source_path is not None:
            info = read_scene(a.source_path, eval=False)
            cfg = info.scanner_cfg
        if a.vol is None:
            return "scene", info.vol, cfg
        vol = _read_volume(a.vol)
        if cfg is not None and tuple(vol.shape) != tuple(int(n) for n in cfg["nVoxel"]):
            raise SystemExit(f"--vol {a.vol} has shape {tuple(vol.shape)}, the scene's nVoxel is "
                             f"{tuple(int(n) for n in cfg['nVoxel'])}")
        return "vol", vol, cfg
    return _model_volume(a)


def load_model(a):
    """(source label, GaussianModel of the saved iteration, scanner_cfg of the model's scene, recorded settings) of
    -m: the scene is the one the model was trained on unless -s names another."""
    from .dataset import read_scene
    from .gaussian_model import GaussianModel
    from .test import load_settings, resolve_iteration

    try:
        settings = load_settings(a.model_path)
        iteration, pickle_path = resolve_iteration(a.model_path, a.iteration)
    except (OSError, ValueError, SyntaxError) as e:
        raise SystemExit(str(e)) from e
    source = a.source_path or settings.get("source_path")
    if not source:
        raise SystemExit("no scene: the model's recorded settings name none; pass -s")
    if not os.path.exists(source):
        raise SystemExit(f"the model's scene {source} does not exist; pass -s")
    cfg = dict(read_scene(source, eval=False).scanner_cfg)
    gaussians = GaussianModel(None)
    gaussians.load_ply(pickle_path)
    return f"model@{iteration}", gaussians, cfg, settings


def _model_volume(a):
    import torch

    from .render_query import query
    from .trainer import PipelineParams

    source, gaussians, cfg, settings = load_model(a)
    if a.resolution is not None:
        cfg["nVoxel"] = [int(a.resolution)] * 3
    pipe = PipelineParams(**{k: settings[k] for k in PipelineParams.__dataclass_fields__ if k in settings})
    with torch.no_grad():
        vol = query(gaussians, cfg["offOrigin"], cfg["nVoxel"], cfg["sVoxel"], pipe)["vol"]
    return source, vol, cfg


def main(argv=None) -> dict:
    a = parse_args(argv)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("mesh extraction needs a CUDA device: marching cubes runs on the GPU and has no CPU fallback")
    from .mesh import marching_cubes, to_scene, write_ply

    source, vol, cfg = load_volume(a)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    try:
        verts, faces = marching_cubes(vol, a.level)
    except ValueError as e:
        raise SystemExit(str(e)) from e
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
    v = to_scene(verts, cfg) if cfg is not None else verts.cpu().numpy()
    write_ply(a.output, v, faces)
    report = {"source": source, "level": a.level, "shape": [int(n) for n in vol.shape], "vertices": int(len(v)),
              "triangles": int(faces.shape[0]), "seconds": seconds, "output": a.output}
    if faces.shape[0] == 0:
        print(f"warning: the surface at level {a.level} is empty (no sample on one side of it)", file=sys.stderr)
    print(json.dumps(report))
    return report


if __name__ == "__main__":
    main(sys.argv[1:])
