"""Measure a scan's horizontal detector offset (centre-of-rotation offset) from its train projections.

    python -m r2_gaussian_b200.estimate_offset -s <scene dir | NAF pickle> [--use_offDetector] [--max_shift PX]
        [--output offset.yml]

Runs `detector.estimate_offset` (the GPU conjugate-ray search) on the scene's train views and prints, or writes to
`--output`, the fields of the trainer's `detector_offset.yml`: `offset_px` (the DetectorOffset convention, relative
to the scanner file's offset under `--use_offDetector`, else to a centred detector), `offset_scene` (scene units at
the detector), the sign convention, and `offDetector_u`, the total offDetector[0] a scanner file would carry, in the
file's units; then `n_pairs`, `n_samples` and `cost_min`.  The scene's files are not changed: put `offDetector_u` into
the scanner file, or pass `--estimate_offDetector` to initialize_pcd, recon or trainer.
"""
from __future__ import annotations

import argparse
import os
import sys


def report(est: dict, scene_scale: float) -> dict:
    """The detector_offset.yml fields of an `estimate_offset` result on a scene-unit scanner."""
    from .detector import SIGN_CONVENTION
    return {"offset_px": est["offset_px"], "offset_scene": est["offset_scene"], "sign_convention": SIGN_CONVENTION,
            "offDetector_u": est["offDetector_u"] / scene_scale, "n_pairs": est["n_pairs"],
            "n_samples": est["n_samples"], "cost_min": est["cost_min"]}


def estimate_scene(info, use_offDetector: bool = False, max_shift=None) -> dict:
    """`detector.estimate_offset` of the train views of a `read_scene` result."""
    import numpy as np
    import torch

    from .detector import estimate_offset
    cams = info.train_cameras
    projs = torch.from_numpy(np.stack([np.asarray(c.image, np.float32) for c in cams])).cuda()
    return estimate_offset(projs, [float(c.angle) for c in cams], info.scanner_cfg, use_offDetector=use_offDetector,
                           max_shift=max_shift)


def estimated_scanner(info, use_offDetector: bool = False, log=print) -> tuple[dict, dict]:
    """`--estimate_offDetector` of initialize_pcd, recon and trainer: (a copy of the scene's scene-unit scanner whose
    offDetector[0] is the estimated total, to be used with use_offDetector on; the estimate).  Logs the estimate."""
    from .detector import OffsetEstimateError, with_offDetector_u
    try:
        est = estimate_scene(info, use_offDetector)
    except OffsetEstimateError as e:
        raise SystemExit(f"--estimate_offDetector: {e}") from e
    log(f"estimated detector offset: {est['offset_px']:+.4f} px, offDetector_u = "
        f"{est['offDetector_u'] / info.scene_scale:.6g} ({est['n_pairs']} conjugate pairs)")
    return with_offDetector_u(info.scanner_cfg, est["offDetector_u"]), est


def main(argv=None) -> dict:
    ap = argparse.ArgumentParser(description="Estimate the horizontal detector offset of a scene from its train "
                                             "projections (GPU conjugate-ray search)")
    ap.add_argument("-s", "--source_path", required=True, help="scene directory or NAF pickle")
    ap.add_argument("--use_offDetector", default=False, action="store_true",
                    help="estimate relative to the scanner's offDetector (default: relative to a centred detector)")
    ap.add_argument("--max_shift", type=float, default=None, help="search range in pixels (default: W / 4)")
    ap.add_argument("--output", default=None, help="write the result to this yml")
    a = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("estimate_offset needs a CUDA device: the search runs on the GPU and has no CPU fallback")
    import yaml

    from .dataset import read_scene
    from .detector import OffsetEstimateError
    info = read_scene(os.path.abspath(a.source_path), eval=False)
    try:
        est = estimate_scene(info, a.use_offDetector, a.max_shift)
    except OffsetEstimateError as e:
        raise SystemExit(str(e)) from e
    doc = report(est, info.scene_scale)
    text = yaml.dump(doc, default_flow_style=False, sort_keys=False)
    if a.output:
        os.makedirs(os.path.dirname(os.path.abspath(a.output)), exist_ok=True)
        with open(a.output, "w") as f:
            f.write(text)
    print(text, end="")
    return doc


if __name__ == "__main__":
    main(sys.argv[1:])
