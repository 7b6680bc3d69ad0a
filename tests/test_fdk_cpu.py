"""The FDK definition (oracle/fdk_oracle.py) on the CPU: amplitude pinned by an analytic ball, geometry pinned by a round
trip through the rasterizer and voxelizer oracles; argument checks of the C ABI and of fdk() that need no GPU."""
import ctypes
import math

import numpy as np
import pytest

import fdk_cases as fc
from oracle import fdk_oracle
from oracle import r2_oracle as orc
from r2_gaussian_b200 import scene


def test_ball_amplitude():
    """Uniform ball, density 1, radius 0.5, cone beam, exact chord-length projections: the centre reconstructs to 1."""
    sc = fc.scanner("cone", 64, 32)
    angles = fc.full_scan(180)
    vol = fdk_oracle.fdk_scene(fc.ball_projections(sc, angles), angles, sc)
    centre = vol[13:19, 13:19, 13:19]          # voxel centres within 0.19 of the origin
    assert abs(centre.mean() - 1.0) <= 0.02, centre.mean()
    assert np.abs(centre - 1.0).max() <= 0.02, np.abs(centre - 1.0).max()
    assert np.abs(vol[:3]).max() <= 0.05       # outside the ball (|x| > 0.8)


def oracle_round_trip(mode: str, n_views: int):
    cloud = fc.round_trip_cloud()
    sc = fc.scanner(mode, fc.ROUND_TRIP_DET, fc.ROUND_TRIP_VOX)
    angles = fc.full_scan(n_views)
    projs = []
    for a in angles:
        v = scene.make_view(sc, float(a))
        projs.append(orc.raster_forward(cloud.means, cloud.scales, cloud.rotations, cloud.density, v.viewmatrix,
                                        v.projmatrix, v.image_width, v.image_height, v.tanfovx, v.tanfovy,
                                        v.mode)["image"])
    got = fdk_oracle.fdk_scene(np.stack(projs), angles, sc)
    want = orc.voxel_forward(cloud.means, cloud.scales, cloud.rotations, cloud.density, sc["nVoxel"], sc["sVoxel"],
                             sc["offOrigin"])["vol"]
    return got, want


@pytest.mark.parametrize("mode,n_views", sorted(fc.ROUND_TRIP_BOUNDS))
def test_round_trip_through_rasterizer_and_voxelizer(mode, n_views):
    """fdk(raster(cloud)) ~ voxel(cloud); a volume flipped along x or z is far off, so a wrong detector orientation or
    axis order fails."""
    got, want = oracle_round_trip(mode, n_views)
    err = fc.rel_l2(got, want)
    assert err <= fc.ROUND_TRIP_BOUNDS[(mode, n_views)], err
    assert fc.rel_l2(got[::-1], want) >= 0.5
    assert fc.rel_l2(got[:, :, ::-1], want) >= 0.5


def test_ramp_filter_taps():
    """One bright pixel in an otherwise empty row gives back the filter kernel: h0 * D at the pixel, -D / (pi^2 k^2 D^2)
    at odd distances, 0 at even ones, no wrap-around."""
    W, D = 16, 2.0 / 16
    p = np.zeros((1, 1, W))
    p[0, 0, 0] = 1.0
    q = fdk_oracle.filter_projections(p, 1.0, 1.0, 0, 1.0)[0, 0]
    k = np.arange(W)
    want = np.where(k % 2 == 1, -1.0 / (np.pi ** 2 * np.maximum(k, 1) ** 2 * D), 0.0)
    want[0] = 1.0 / (4.0 * D)
    np.testing.assert_allclose(q, want, rtol=1e-12, atol=1e-12)


def test_abi_rejects_bad_arguments_before_any_cuda_call():
    from r2_gaussian_b200 import _lib

    lib = _lib.load()
    assert lib.r2x_fdk_scratch_bytes(50, 512, 512) >= 50 * 512 * 512 * 4
    dummy = ctypes.c_void_p(16)
    base = dict(N=2, H=8, W=8, mode=1, su=0.0, sv=0.0, weighting=0, w=None, arc=0.0, dso=5.0, n=4, s=2.0, nbytes=1 << 20)

    def call(**kw):
        a = dict(base, **kw)
        return lib.r2x_fdk(None, a["N"], a["H"], a["W"], dummy, dummy, dummy, 0.3, 0.3, a["mode"], a["su"], a["sv"],
                           a["weighting"], a["w"], a["arc"], a["dso"], a["n"], a["n"], a["n"], a["s"], a["s"], a["s"], 0.0,
                           0.0, 0.0, dummy, dummy, a["nbytes"])

    for kw in (dict(N=0), dict(H=0), dict(W=0), dict(n=0), dict(mode=2), dict(dso=0.0), dict(s=0.0),
               dict(su=math.nan), dict(sv=math.inf), dict(weighting=3), dict(weighting=-1),
               dict(weighting=2, su=0.0), dict(weighting=2, su=4.0), dict(weighting=2, su=-4.0)):
        assert call(**kw) != 0, kw
        assert b"bad" in lib.r2x_last_error(), kw
    assert call(nbytes=16) != 0                                 # scratch too small
    assert b"scratch" in lib.r2x_last_error()


def test_fdk_rejects_host_tensors():
    torch = pytest.importorskip("torch")
    from r2_gaussian_b200.fdk import fdk

    sc = fc.scanner("cone", 8, 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        fdk(torch.zeros(2, 8, 8), [0.0, 1.0], sc)
