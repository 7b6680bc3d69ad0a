"""Remove ring artifacts from an existing scene: stripe removal (`stripes.remove_stripes`) of its projections.

    python -m r2_gaussian_b200.remove_stripes -s <scene> --output <dir> [--size 5]

For scenes that already exist: the published prebuilt ones, `generate_data` scenes, calibrated ones.  The union of the
scene's `proj_train` and `proj_test` files is corrected as one stack on the GPU (the method ignores view order) and
written to the same relative paths under `--output` as float32.  `meta_data.json` is copied byte for byte and the
`vol` / `ct` files are copied, so the output opens wherever the source does.  `init_*.npy` point clouds are not copied:
they were sampled from a reconstruction of the striped views; run `initialize_pcd` on the output.  `proj_all/` is
neither read nor written.  The scene's `vol_gt` keeps whatever rings it has; only `generate_real_data
--remove_stripes` rebuilds a pseudo ground truth from corrected views.
"""
from __future__ import annotations

import argparse
import glob
import json
import os
import shutil

import numpy as np

from .stripes import DEFAULT_SIZE, check_size


def remove_scene_stripes(source: str, output: str, size: int = DEFAULT_SIZE) -> str:
    size = check_size(size)
    if source.split(".")[-1] in ("pickle", "pkl") or os.path.isfile(source):
        raise ValueError(f"{source}: remove_stripes takes a scene directory with meta_data.json, not a NAF pickle")
    meta_path = os.path.join(source, "meta_data.json")
    if not os.path.isfile(meta_path):
        raise ValueError(f"{source}: no meta_data.json")
    if os.path.realpath(output) == os.path.realpath(source):
        raise ValueError(f"--output {output} is the source scene; write the corrected scene elsewhere")
    if os.path.exists(os.path.join(output, "meta_data.json")):
        raise ValueError(f"--output {output} already holds a meta_data.json; choose an empty directory")
    with open(meta_path) as f:
        meta = json.load(f)
    rels = [fr["file_path"] for split in ("proj_train", "proj_test") for fr in meta.get(split, [])]
    if not rels:
        raise ValueError(f"{source}: meta_data.json lists no proj_train or proj_test views")
    views = [np.load(os.path.join(source, r)) for r in rels]
    for r, v in zip(rels, views):
        if v.ndim != 2 or v.shape != views[0].shape:
            raise ValueError(f"{source}: {r} has shape {v.shape}, the first view {rels[0]} {views[0].shape}; "
                             "the views must share one 2-D shape")
    check_size(size, views[0].shape[1])

    import torch

    if not torch.cuda.is_available():
        raise RuntimeError("remove_stripes needs a CUDA device: the correction runs on the GPU, with no CPU fallback")
    from .stripes import remove_stripes

    stack = torch.from_numpy(np.stack(views).astype(np.float32)).cuda()
    host = remove_stripes(stack, size, out=stack).cpu().numpy()

    os.makedirs(output, exist_ok=True)
    for r, v in zip(rels, host):
        os.makedirs(os.path.dirname(os.path.join(output, r)), exist_ok=True)
        np.save(os.path.join(output, r), v)
    for rel in sorted({meta[k] for k in ("vol", "ct") if k in meta}):
        os.makedirs(os.path.dirname(os.path.join(output, rel)), exist_ok=True)
        shutil.copyfile(os.path.join(source, rel), os.path.join(output, rel))
    shutil.copyfile(meta_path, os.path.join(output, "meta_data.json"))
    skipped = sorted(os.path.basename(p) for p in glob.glob(os.path.join(source, "init_*.npy")))
    print(f"Removed stripes (size {size}) from {len(rels)} views of {source} into {output}")
    print("Not copied: " + (", ".join(skipped) if skipped else "init_*.npy point clouds") + " (sampled from the "
          "striped views); run initialize_pcd on the corrected scene. The copied vol_gt keeps any rings it has.")
    return output


def main(argv=None) -> str:
    ap = argparse.ArgumentParser(description="Remove ring artifacts from a scene's projections (sorting-based stripe "
                                             "removal on the GPU) and write the corrected scene")
    ap.add_argument("-s", "--source_path", required=True, help="scene directory (meta_data.json)")
    ap.add_argument("--output", required=True, help="directory for the corrected scene (must not hold a scene)")
    ap.add_argument("--size", default=DEFAULT_SIZE, type=int,
                    help="median window across detector columns, odd, 1 to 255 (1 changes nothing)")
    a = ap.parse_args(argv)
    return remove_scene_stripes(a.source_path, a.output, a.size)


if __name__ == "__main__":
    main()
