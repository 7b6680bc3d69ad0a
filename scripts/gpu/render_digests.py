#!/usr/bin/env python
"""Write the SHA-256 digests of the forward images of tests/render_digest_cases.py (tests/golden/render_digests.json).

    python scripts/gpu/render_digests.py [--root DIR] [--out FILE]

--root imports r2_gaussian_b200 from another checkout (with its library built), so that the digests can be taken from
the build a change must reproduce bit for bit; the cases themselves always come from this checkout's tests/.  Prints
the JSON object and writes it to --out when given."""
from __future__ import annotations

import argparse
import json
import os
import sys

HERE_ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=HERE_ROOT, help="checkout whose r2_gaussian_b200 renders the images")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    root = os.path.abspath(args.root)
    sys.path.insert(0, os.path.join(HERE_ROOT, "tests"))
    sys.path.insert(0, root)

    import torch

    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device"}))
        return 1
    import r2_gaussian_b200
    assert os.path.dirname(os.path.abspath(r2_gaussian_b200.__file__)) == os.path.join(root, "r2_gaussian_b200")
    import render_digest_cases as rdc

    out = dict(gpu=torch.cuda.get_device_name(0), images={})
    for name, cloud, view in rdc.cases():
        out["images"][name] = rdc.render(cloud, view)
    s = json.dumps(out, indent=1, sort_keys=True)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(s + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
