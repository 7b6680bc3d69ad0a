"""The recovery scenes of the horizontal detector offset, shared by test_detector_offset_gpu.py and
scripts/gpu/detector_offset_bench.py so that both run the same recipe: the 48^3 generate_data scene of the end-to-end
tests (24 train / 6 test views of 96^2, cone beam, no noise), once as generated and once with every projection moved
`shift` columns towards larger index, each initialised by FDK of its own views."""
import os
import random
import shutil

import numpy as np

SHIFT = 3
ITERATIONS = 2000


def recovery_scenes(tmp, shift=SHIFT) -> dict:
    """-> {"plain": (case dir, init .npy), "shifted": (case dir, init .npy)} under the directory `tmp` (a pathlib.Path)."""
    from r2_gaussian_b200 import generate_data, initialize_pcd
    from test_projector_gpu import _write_inputs
    yml, vol_path, *_ = _write_inputs(tmp, noise=False)
    plain = generate_data.main(["--vol", str(vol_path), "--scanner", str(yml), "--n_train", "24", "--n_test", "6",
                                "--output", str(tmp / "data")])
    shifted = str(tmp / "shifted")
    shutil.copytree(plain, shifted)
    generate_data.shift_projections(shifted, shift)
    out = {}
    for name, path in (("plain", plain), ("shifted", shifted)):
        init = initialize_pcd.main(["--data", path, "--recon_method", "fdk", "--n_points", "2000",
                                    "--output", str(tmp / f"init_{name}.npy")])
        out[name] = (path, init)
    return out


def train(path, init, model_path, detector_params, iterations=ITERATIONS) -> dict:
    """The trainer from seed 0 with default settings, evaluated (and saved when `model_path`) at the last iteration."""
    import torch

    from r2_gaussian_b200 import trainer
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    model = trainer.ModelParams(source_path=path, model_path=str(model_path), ply_path=init)
    opt = trainer.OptimizationParams(iterations=iterations)
    return trainer.training(model, opt, trainer.PipelineParams(), {iterations},
                            {iterations} if model_path else set(), log=lambda *a: None,
                            detector_params=detector_params)
