"""Drop-in package: the import name the reference's r2_gaussian/gaussian/render_query.py:14-19 uses.

`from xray_gaussian_rasterization_voxelization import GaussianRasterizationSettings, GaussianRasterizer,
GaussianVoxelizationSettings, GaussianVoxelizer` resolves to the H100-native implementation, so the
reference's render()/query()/train.py/test.py run unchanged with this repository on PYTHONPATH.
"""
from r2_gaussian_b200 import _C  # noqa: F401  (same attribute the reference package exposes)
from r2_gaussian_b200.rasterization import GaussianRasterizationSettings, GaussianRasterizer
from r2_gaussian_b200.voxelization import GaussianVoxelizationSettings, GaussianVoxelizer

__all__ = [
    "GaussianRasterizationSettings",
    "GaussianRasterizer",
    "GaussianVoxelizationSettings",
    "GaussianVoxelizer",
]
