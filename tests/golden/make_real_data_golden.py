"""Write tests/golden/real_data/cases.npz: seeded raw projections and what the reference's numpy + cv2.resize chain
makes of them, at the shapes the real-scan preparation must get right.  Needs cv2 (opencv-python on x86-64, whose
INTER_LINEAR float32 resize runs the IPP path by default); run from the repository root:

    python tests/golden/make_real_data_golden.py

Per case <name>: <name>_img (float64 [H0, W0]), <name>_params ([subsample, proj_rescale, object_scale]) and
<name>_out (float32, the reference's bytes; for a height / width difference of 1, where the reference's crop is empty,
the uncropped cv2.resize result, which is what a difference of 1 is meant to give).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import real_data_oracle  # noqa: E402

# name: (H0, W0, subsample)
CASES = {
    "divisible": (64, 72, 4),        # 16 x 18, one column cropped on each side
    "not_divisible": (67, 81, 4),    # 16 x 20 from non-integer ratios
    "odd_crop": (61, 83, 3),         # 20 x 27: difference 7, a non-square 20 x 21 result
    "diff_one": (70, 64, 4),         # 17 x 16: nothing is cropped
    "no_subsample": (32, 40, 1),
    "ratio_5": (97, 131, 5),         # 19 x 26: 97 / 19 and 131 / 26, neither an integer
    "half": (64, 72, 2),             # both ratios exactly 2
}
PROJ_RESCALE, OBJECT_SCALE = 400.0, 50


def main():
    import cv2

    rng = np.random.default_rng(20261017)
    rec = {}
    for name, (H0, W0, s) in CASES.items():
        img = rng.normal(0.5, 0.6, (H0, W0)) * PROJ_RESCALE / OBJECT_SCALE
        img[0, :3] = (-0.0, 0.0, -1e-300)
        out = real_data_oracle.reference_chain(img, s, PROJ_RESCALE, OBJECT_SCALE)
        if out.size == 0:      # the reference's empty crop: keep cv2's resize itself
            p = real_data_oracle.shift_up(real_data_oracle.scale_clamp(img, PROJ_RESCALE, OBJECT_SCALE))
            out = cv2.resize(p, [int(W0 / s), int(H0 / s)])
        rec[name + "_img"] = img
        rec[name + "_params"] = np.array([s, PROJ_RESCALE, OBJECT_SCALE], np.float64)
        rec[name + "_out"] = np.ascontiguousarray(out, np.float32)
    os.makedirs(os.path.join(HERE, "real_data"), exist_ok=True)
    np.savez_compressed(os.path.join(HERE, "real_data", "cases.npz"), **rec)
    print({k: v.shape for k, v in rec.items() if k.endswith("_out")})


if __name__ == "__main__":
    main()
