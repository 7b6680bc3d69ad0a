"""Reduce metal artifacts in an existing scene: LI-MAR or NMAR (`mar.reduce_metal`) of its projections.

    python -m r2_gaussian_b200.reduce_metal -s <scene> --output DIR [--method nmar|li]
        (--metal_threshold T | --metal_mask M.npy) [--use_offDetector]

The metal is segmented once, from the FDK of the scene's `proj_train` views (`FDK > T` in scene-scaled units, or the
bool nVoxel-shaped mask M.npy), and the train and test views are corrected with that one mask.  They are written to
the same relative paths under `--output` as float32: pixels outside the metal trace are the source file's bits, pixels
inside it the corrected value in the file's units.  `meta_data.json` is copied byte for byte and the `vol` / `ct`
files are copied, so the trainer, `initialize_pcd` and `recon` open the output unchanged.  Two files are added:
`metal_mask.npy` (bool, nVoxel) and `mar.yml` (method, threshold or mask file, metal voxel count, trace fraction per
split, whole-trace detector rows).  `init_*.npy` point clouds are not copied: they were sampled from the uncorrected
views.  MAR removes the metal from the data by design, so a model trained on the output has none: `metal_mask.npy` is
what to reinsert the metal with, or to mask it out.  Helical and per-view-geometry scenes are refused.
"""
from __future__ import annotations

import argparse
import glob
import json
import os
import shutil

import numpy as np

from .mar import METHODS


def load_mask(path: str):
    mask = np.load(path)
    if mask.dtype != np.bool_:
        raise ValueError(f"--metal_mask {path}: expected a bool array, got {mask.dtype}")
    return mask


def reduce_scene_metal(source: str, output: str, method: str = "nmar", threshold=None, mask_path=None,
                       use_offDetector: bool = False) -> str:
    if method not in METHODS:
        raise ValueError(f"--method must be one of {', '.join(METHODS)}, got {method!r}")
    if (threshold is None) == (mask_path is None):
        raise ValueError("give exactly one of --metal_threshold and --metal_mask")
    if source.split(".")[-1] in ("pickle", "pkl") or os.path.isfile(source):
        raise ValueError(f"{source}: reduce_metal takes a scene directory with meta_data.json, not a NAF pickle")
    meta_path = os.path.join(source, "meta_data.json")
    if not os.path.isfile(meta_path):
        raise ValueError(f"{source}: no meta_data.json")
    if os.path.realpath(output) == os.path.realpath(source):
        raise ValueError(f"--output {output} is the source scene; write the corrected scene elsewhere")
    if os.path.exists(os.path.join(output, "meta_data.json")):
        raise ValueError(f"--output {output} already holds a meta_data.json; choose an empty directory")
    with open(meta_path) as f:
        meta = json.load(f)
    from .scene import VIEW_KEYS

    for split in ("proj_train", "proj_test"):
        for fr in meta.get(split, []):
            keys = [k for k in VIEW_KEYS if k in fr]
            if keys:
                raise ValueError(f"{source}: frame {fr['file_path']} carries per-view geometry ({', '.join(keys)}); "
                                 "metal artifact reduction of helical and per-view-geometry scans is not supported")
    if not meta.get("proj_train"):
        raise ValueError(f"{source}: meta_data.json lists no proj_train views")
    mask = load_mask(mask_path) if mask_path is not None else None
    nvox = [int(v) for v in meta["scanner"]["nVoxel"]]
    if mask is not None and list(mask.shape) != nvox:
        raise ValueError(f"--metal_mask {mask_path}: shape {list(mask.shape)}, the scene's nVoxel is {nvox}")

    import torch

    if not torch.cuda.is_available():
        raise RuntimeError("reduce_metal needs a CUDA device: the correction runs on the GPU, with no CPU fallback")
    import yaml

    from .dataset import read_scene
    from .mar import reduce_metal

    info = read_scene(source, eval=True)
    cfg, scale = info.scanner_cfg, info.scene_scale
    splits = {"proj_train": info.train_cameras, "proj_test": info.test_cameras}
    stacks = {k: torch.from_numpy(np.stack([np.asarray(c.image, np.float32) for c in cams])).cuda()
              for k, cams in splits.items() if cams}
    extra = [(stacks["proj_test"], [c.angle for c in info.test_cameras])] if "proj_test" in stacks else []
    res = reduce_metal(stacks["proj_train"], [c.angle for c in info.train_cameras], cfg, method=method,
                       threshold=threshold, mask=mask, extra=extra, use_offDetector=use_offDetector)
    results = {"proj_train": (res.projs, res.trace, res.trace_fraction, res.all_trace_rows)}
    if extra:
        results["proj_test"] = res.extra[0]

    os.makedirs(output, exist_ok=True)
    report = {"method": method}
    report.update({"metal_threshold": float(threshold)} if threshold is not None else
                  {"metal_mask": os.path.abspath(mask_path)})
    report["metal_voxels"] = int(res.mask.sum())
    for split, (corrected, trace, frac, rows) in results.items():
        corrected, trace = corrected.cpu().numpy(), trace.cpu().numpy().astype(bool)
        for fr, v, t in zip(meta[split], corrected, trace):
            src = np.load(os.path.join(source, fr["file_path"])).astype(np.float32)
            dst = os.path.join(output, fr["file_path"])
            os.makedirs(os.path.dirname(dst), exist_ok=True)
            np.save(dst, np.where(t, (v / np.float32(scale)).astype(np.float32), src))
        report[f"trace_fraction_{split[5:]}"] = frac
        report[f"all_trace_rows_{split[5:]}"] = rows
    for rel in sorted({meta[k] for k in ("vol", "ct") if k in meta}):
        os.makedirs(os.path.dirname(os.path.join(output, rel)), exist_ok=True)
        shutil.copyfile(os.path.join(source, rel), os.path.join(output, rel))
    shutil.copyfile(meta_path, os.path.join(output, "meta_data.json"))
    np.save(os.path.join(output, "metal_mask.npy"), res.mask.cpu().numpy())
    with open(os.path.join(output, "mar.yml"), "w") as f:
        yaml.dump(report, f, default_flow_style=False, sort_keys=False)
    skipped = sorted(os.path.basename(p) for p in glob.glob(os.path.join(source, "init_*.npy")))
    print(f"Reduced metal artifacts ({method}, {report['metal_voxels']} metal voxels) in {source} into {output}")
    print("Not copied: " + (", ".join(skipped) if skipped else "init_*.npy point clouds") + " (sampled from the "
          "uncorrected views); run initialize_pcd on the corrected scene. A model trained on it has no metal: "
          "metal_mask.npy is what to reinsert or mask with.")
    return output


def main(argv=None) -> str:
    ap = argparse.ArgumentParser(description="Reduce metal artifacts in a scene's projections (LI-MAR or NMAR, "
                                             "metal-trace inpainting on the GPU) and write the corrected scene")
    ap.add_argument("-s", "--source_path", required=True, help="scene directory (meta_data.json)")
    ap.add_argument("--output", required=True, help="directory for the corrected scene (must not hold a scene)")
    ap.add_argument("--method", default="nmar", choices=METHODS, help="nmar (default) or li")
    g = ap.add_mutually_exclusive_group(required=True)
    g.add_argument("--metal_threshold", type=float, default=None, metavar="T",
                   help="metal = FDK of the train views > T (scene-scaled units)")
    g.add_argument("--metal_mask", default=None, metavar="M.npy", help="a bool nVoxel-shaped metal mask")
    ap.add_argument("--use_offDetector", default=False, action="store_true",
                    help="reconstruct and project through the scanner's offDetector")
    a = ap.parse_args(argv)
    return reduce_scene_metal(a.source_path, a.output, a.method, a.metal_threshold, a.metal_mask, a.use_offDetector)


if __name__ == "__main__":
    main()
