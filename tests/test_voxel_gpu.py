"""GPU parity: our sm_90a voxelizer (through the C ABI) against the CPU oracle."""
import numpy as np
import pytest

import util
from r2_gaussian_b200 import scene

pytestmark = pytest.mark.gpu

GRIDS = {
    "full32": ((32, 32, 32), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0), 1500, "trained"),
    "ragged": ((20, 36, 28), (1.3, 2.0, 1.7), (0.1, -0.05, 0.2), 1200, "trained"),
    "tvcrop": ((32, 32, 32), (0.25, 0.25, 0.25), (0.31, -0.42, 0.13), 20000, "init"),   # train.py:128-139 style crop
    "full64": ((64, 64, 64), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0), 8000, "trained"),
    # 18 x 17 x 17 = 5202 tiles > DIRECT_MAX_TILES: two-level direct binning (5 x 5 x 5 supertiles, ragged edges)
    "manytiles": ((144, 136, 136), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0), 1200, "trained"),
    # the same grid through the radix-sort binning (R2X_VOXEL_BINNING=radix; also what grids beyond 512^3 take)
    "manytiles_radix": ((144, 136, 136), (2.0, 2.0, 2.0), (0.0, 0.0, 0.0), 1200, "trained"),
}


@pytest.fixture(autouse=True)
def _binning_mode(request, monkeypatch):
    name = getattr(getattr(request.node, "callspec", None), "params", {}).get("name", "")
    if str(name).endswith("_radix"):
        monkeypatch.setenv("R2X_VOXEL_BINNING", "radix")
    else:
        monkeypatch.delenv("R2X_VOXEL_BINNING", raising=False)


def _cloud(P, kind, seed):
    return scene.make_cloud(P, kind=kind, seed=seed)


@pytest.mark.parametrize("name", list(GRIDS))
def test_forward_matches_oracle(name):
    nV, sV, ctr, P, kind = GRIDS[name]
    cloud = _cloud(P, kind, len(name))
    ours = util.ours_voxel_forward(cloud, nV, sV, ctr)
    orc = util.oracle_voxel_forward(cloud, nV, sV, ctr)
    assert ours["R"] == orc["R"]
    for k in ["radii_x", "radii_y", "radii_z", "tiles_touched"]:
        np.testing.assert_array_equal(ours[k], orc[k])
    vis = orc["tiles_touched"] > 0
    np.testing.assert_array_equal(ours["xyz_vol"][vis].view(np.uint32), orc["xyz_vol"][vis].view(np.uint32))
    np.testing.assert_array_equal(ours["depth"][vis].view(np.uint32), orc["depth"][vis].view(np.uint32))
    assert util.key_multiset_equal(ours["keys"], orc["keys"])
    np.testing.assert_array_equal(ours["ranges"], orc["ranges"])
    np.testing.assert_allclose(ours["conic_opacity"][vis], orc["conic_opacity"][vis], rtol=2e-6, atol=0)
    scale = float(np.abs(orc["vol"]).max()) if orc["R"] else 1.0
    err = np.abs(ours["vol"].astype(np.float64) - orc["vol"]).max()
    assert err <= 1e-5 * scale + 1e-7, f"volume error {err} vs scale {scale}"


@pytest.mark.parametrize("name", ["full32", "ragged", "tvcrop", "manytiles", "manytiles_radix"])
def test_backward_matches_oracle(name):
    nV, sV, ctr, P, kind = GRIDS[name]
    cloud = _cloud(P, kind, len(name))
    ours = util.ours_voxel_forward(cloud, nV, sV, ctr, export=False)
    orc = util.oracle_voxel_forward(cloud, nV, sV, ctr)
    dL = np.random.RandomState(11).randn(*nV).astype(np.float32)
    g = util.ours_voxel_backward(cloud, nV, sV, ctr, ours, dL)
    go = util.oracle_voxel_backward(cloud, nV, sV, orc, dL)
    util.assert_grads_close(g, go, ["dL_dopacity", "dL_dmean3D", "dL_dcov3D", "dL_dscale", "dL_drot"])


@pytest.mark.parametrize("grid,P,kind", [((160, 152, 144), 40000, "init"), ((136, 200, 72), 30000, "trained"),
                                         ((256, 256, 256), 120000, "init")])
def test_two_level_binning_is_bit_identical_to_the_radix_path(grid, P, kind, monkeypatch):
    """Per-tile lists (ranges, point_list), the volume and the gradients from the two-level direct binning are
    the radix path's, bit for bit: both produce every list in ascending Gaussian index."""
    cloud = _cloud(P, kind, 3)
    sV, ctr = (2.0, 2.0, 2.0), (0.0, 0.0, 0.0)
    dL = np.random.RandomState(4).randn(*grid).astype(np.float32)
    monkeypatch.delenv("R2X_VOXEL_BINNING", raising=False)
    a = util.ours_voxel_forward(cloud, grid, sV, ctr)
    ga = util.ours_voxel_backward(cloud, grid, sV, ctr, a, dL)
    monkeypatch.setenv("R2X_VOXEL_BINNING", "radix")
    b = util.ours_voxel_forward(cloud, grid, sV, ctr)
    gb = util.ours_voxel_backward(cloud, grid, sV, ctr, b, dL)
    assert a["R"] == b["R"] and a["R"] > 0
    np.testing.assert_array_equal(a["ranges"], b["ranges"])
    np.testing.assert_array_equal(a["point_list"], b["point_list"])
    np.testing.assert_array_equal(a["keys"], b["keys"])
    np.testing.assert_array_equal(a["vol"].view(np.uint32), b["vol"].view(np.uint32))
    for k in ga:
        np.testing.assert_array_equal(ga[k].view(np.uint32), gb[k].view(np.uint32))


def test_deterministic():
    nV, sV, ctr, P, kind = GRIDS["full32"]
    cloud = _cloud(P, kind, 5)
    a = util.ours_voxel_forward(cloud, nV, sV, ctr, export=False)
    b = util.ours_voxel_forward(cloud, nV, sV, ctr, export=False)
    np.testing.assert_array_equal(a["vol"].view(np.uint32), b["vol"].view(np.uint32))
    dL = np.random.RandomState(2).randn(*nV).astype(np.float32)
    g1 = util.ours_voxel_backward(cloud, nV, sV, ctr, a, dL)
    g2 = util.ours_voxel_backward(cloud, nV, sV, ctr, a, dL)
    for k in g1:
        np.testing.assert_array_equal(g1[k].view(np.uint32), g2[k].view(np.uint32))


def test_requires_scales():
    import torch
    from r2_gaussian_b200 import _C
    from r2_gaussian_b200._lib import R2XError

    m = torch.zeros((8, 3), device="cuda")
    with pytest.raises(R2XError):
        _C.voxelize_gaussians(m, torch.ones((8, 1), device="cuda"), torch.Tensor([]), torch.Tensor([]), 1.0,
                              torch.ones((8, 6), device="cuda"), 16, 16, 16, 2.0, 2.0, 2.0, 0.0, 0.0, 0.0, False, False)
