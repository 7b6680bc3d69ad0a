"""GPU builder of metal scenes for the MAR tests and scripts/gpu/mar_bench.py: a soft-tissue phantom with two metal rods
on one grid, each part projected with `projector.project`, combined per pixel by a three-bin beam-hardening model

    p = -ln sum_k w_k exp(-a_k p_t - b_k p_m),   w = (0.3, 0.4, 0.3), a = (1.3, 1.0, 0.8) g, b = (3.0, 1.0, 0.4) g

(p_t, p_m the projections of the tissue and metal volumes in scene units, g their conversion to attenuation), then
Poisson counts at an absolute I0, floored at one count, and written with `dataset.write_blender` in the scene units
of the middle bin (p / g).  vol_gt is tissue + metal.  Test and bench infrastructure, not a generator option."""
from __future__ import annotations

import numpy as np

W_BINS = (0.3, 0.4, 0.3)
A_BINS = (1.3, 1.0, 0.8)
B_BINS = (3.0, 1.0, 0.4)


def phantom(n_vox: int, metal_density: float = 3.0):
    """(tissue, metal, mask) on an n_vox^3 grid over [-1, 1]^3: an elliptic cylinder of soft tissue (0.2) with two
    bone-like inserts (0.4) and a low-contrast one (0.25), and two metal rods of `metal_density`."""
    c = (np.arange(n_vox) + 0.5) / n_vox * 2.0 - 1.0
    x, y, z = np.meshgrid(c, c, c, indexing="ij")
    tissue = np.zeros((n_vox,) * 3, np.float32)
    body = ((x / 0.8) ** 2 + (y / 0.6) ** 2 <= 1.0) & (np.abs(z) <= 0.8)
    tissue[body] = 0.2
    for cx, cy, r, v in ((0.0, 0.35, 0.1, 0.4), (-0.45, -0.15, 0.08, 0.4), (0.1, -0.3, 0.12, 0.25)):
        tissue[body & ((x - cx) ** 2 + (y - cy) ** 2 <= r * r)] = v
    mask = ((((x - 0.3) ** 2 + y ** 2) <= 0.06 ** 2) | (((x + 0.25) ** 2 + (y - 0.05) ** 2) <= 0.05 ** 2)) \
        & (np.abs(z) <= 0.6)
    tissue[mask] = 0.0
    metal = np.where(mask, np.float32(metal_density), np.float32(0)).astype(np.float32)
    return tissue, metal, mask


def polychromatic(p_t, p_m, g: float, I0: float | None, rng):
    """The beam-hardening model on torch stacks, then Poisson counts at I0 (None: no noise); in units of p / g."""
    import torch

    s = torch.zeros_like(p_t, dtype=torch.float64)
    for w, a, b in zip(W_BINS, A_BINS, B_BINS):
        s += w * torch.exp(-(a * g) * p_t.double() - (b * g) * p_m.double())
    if I0 is not None:
        counts = torch.from_numpy(rng.poisson((I0 * s).cpu().numpy())).to(s.device, torch.float64)
        s = torch.clamp(counts, min=1.0) / I0
    return (-torch.log(s) / g).to(torch.float32)


def metal_scene(path: str, n_det: int = 64, n_vox: int = 64, n_train: int = 60, n_test: int = 10, g: float = 6.0,
                I0: float | None = 1e4, metal_density: float = 3.0, mono: bool = False, seed: int = 0):
    """Write a cone-beam metal scene to `path`; returns (path, tissue, metal, mask).  `mono` writes the ideal
    monochromatic projections p_t + p_m instead (no hardening, no noise)."""
    import torch

    from r2_gaussian_b200.dataset import write_blender
    from r2_gaussian_b200.projector import project
    from r2_gaussian_b200.scene import cone_beam_scanner

    sc = cone_beam_scanner(n_det, n_vox)                  # sVoxel 2: scene units are the file's units
    sc.update({"filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0})
    tissue, metal, mask = phantom(n_vox, metal_density)
    rng = np.random.default_rng(seed)
    train = np.linspace(0, 2 * np.pi, n_train, endpoint=False)
    test = np.sort(rng.uniform(0, 2 * np.pi, n_test))
    cfg = dict(sc, dVoxel=[2.0 / n_vox] * 3, dDetector=[4.0 / n_det] * 2)
    views = {}
    for split, ang in (("train", train), ("test", test)):
        p_t = project(torch.from_numpy(tissue).cuda(), ang, cfg)
        p_m = project(torch.from_numpy(metal).cuda(), ang, cfg)
        p = (p_t + p_m) if mono else polychromatic(p_t, p_m, g, I0, rng)
        views[split] = list(zip(ang, p.cpu().numpy()))
    write_blender(path, sc, views["train"], views["test"], tissue + metal)
    return path, tissue, metal, mask
