"""Forward images whose exact bits are pinned by tests/golden/render_digests.json.

The forward render sums every pixel in a fixed order (8 slices of the chunk, each in increasing Gaussian order, then the
slices and the chunks in order), so its image is a deterministic function of the inputs.  A change to how the render
kernel maps pixels to lanes, or to how it shares work between them, must leave that image unchanged bit for bit; these
cases pin it on the headline scene and at the work-plan, render-path and binning boundaries of tests/regime_cases.py.

`scripts/gpu/render_digests.py` writes the digests; `tests/test_render_bits_gpu.py` checks them.
"""
from __future__ import annotations

import functools
import hashlib

import numpy as np

import regime_cases as rc
import util
from r2_gaussian_b200 import scene

BENCH_VIEWS = (0, 17, 34)


@functools.lru_cache(maxsize=1)
def cases() -> tuple:
    """(name, cloud, view) of every pinned forward, in a fixed order."""
    out = []
    sc = scene.cone_beam_scanner(512, 256)           # the bench.py scene: 100k init-like Gaussians, 512^2 cone beam
    views = scene.make_views(sc, 50)
    cloud = scene.make_cloud(100_000, kind="init", seed=0)
    for v in BENCH_VIEWS:
        out.append((f"bench_view{v}", cloud, views[v]))
    for c in rc.engineered_cases():                  # per-tile counts, the 41-chunk tile, fast/exact limits, CTA totals
        if c.kind == "raster":
            out.append((c.name, c.cloud, c.view))
    for P in (1, 255, 256, 257):                     # partial and single preprocess CTAs
        out.append((f"P{P}", scene.make_cloud(P, kind="trained", seed=P), rc.parallel_view(96, 80)))
    for name in ("det_7x5", "det_656x400", "cone_trained_bigdet"):   # a partial tile, T = 1025, the radix path
        cloud, view = util.case(name)
        out.append((name, cloud, view))
    return tuple(out)


def image_digest(image: np.ndarray) -> str:
    """SHA-256 of the float32 image's bytes (row-major, little-endian)."""
    a = np.ascontiguousarray(image, dtype="<f4")
    return hashlib.sha256(a.tobytes()).hexdigest()


def render(cloud, view) -> dict:
    out = util.ours_raster_forward(cloud, view, export=False)
    return dict(sha256=image_digest(out["image"]), shape=list(out["image"].shape), R=int(out["R"]))
