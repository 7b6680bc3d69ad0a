"""The projector definition (oracle/projector_oracle.py) on the CPU: amplitude pinned by a cube of ones and an analytic
ball, geometry pinned by a round trip through the voxelizer and rasterizer oracles; argument checks of the C ABI and of
project() that need no GPU; the noise model of generate_data."""
import ctypes
import math

import numpy as np
import pytest

import fdk_cases as fc
import projector_cases as pc
from oracle import projector_oracle as po
from oracle import r2_oracle as orc


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_cube_amplitude(mode):
    """A centred cube of ones: the central ray at 0 and pi/2 crosses sVoxel of density 1."""
    sc = fc.scanner(mode, 64, 32)
    sc["nDetector"] = [65, 65]                     # odd: the central pixel's ray goes through the volume centre
    p = po.project_scene(np.ones((32, 32, 32), np.float32), [0.0, math.pi / 2], sc)
    np.testing.assert_allclose(p[:, 32, 32], 2.0, rtol=0.01)


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_ball_against_exact_chords(mode):
    sc = fc.scanner(mode, 64, 64)
    angles = [0.0, 0.7, 2.1]
    got = po.project_scene(pc.ball_volume(64), angles, sc)
    err = pc.rel_l2(got, fc.ball_projections(sc, angles))
    assert err <= pc.BALL_BOUND, err


def _round_trip(mode):
    cloud = fc.round_trip_cloud()
    sc = fc.scanner(mode, pc.ROUND_TRIP_DET, pc.ROUND_TRIP_VOX)
    vol = orc.voxel_forward(cloud.means, cloud.scales, cloud.rotations, cloud.density, sc["nVoxel"], sc["sVoxel"],
                            sc["offOrigin"])["vol"]
    return sc, vol, pc.raster_views(cloud, sc, pc.ROUND_TRIP_ANGLES)


@pytest.mark.parametrize("mode", ["cone", "parallel"])
def test_round_trip_through_voxelizer_and_rasterizer(mode):
    """project(voxel(cloud)) ~ raster(cloud) for an off-centre, anisotropic, rotated cloud; a flipped or transposed
    volume, or the negated angles, are far off, so a wrong axis order, orientation or angle sign fails."""
    sc, vol, want = _round_trip(mode)
    err = pc.rel_l2(po.project_scene(vol, pc.ROUND_TRIP_ANGLES, sc), want)
    assert err <= pc.ROUND_TRIP_BOUND, err
    for name, v, angles in pc.flipped_variants(vol, list(pc.ROUND_TRIP_ANGLES)):
        off = pc.rel_l2(po.project_scene(np.ascontiguousarray(v), angles, sc), want)
        assert off >= 0.5, (name, off)


def test_abi_rejects_bad_arguments_before_any_cuda_call():
    from r2_gaussian_b200 import _lib

    lib = _lib.load()
    dummy = ctypes.c_void_p(16)
    base = dict(n=4, vol=dummy, s=2.0, c=0.0, N=2, H=8, W=8, vm=dummy, tan=0.3, mode=1, su=0.0, sv=0.0, step=0.25,
                out=dummy)

    def call(**kw):
        a = dict(base, **kw)
        return lib.r2x_volume_project(None, a["n"], a["n"], a["n"], a["vol"], a["s"], a["s"], a["s"], a["c"], a["c"],
                                      a["c"], a["N"], a["H"], a["W"], a["vm"], a["tan"], a["tan"], a["mode"], a["su"],
                                      a["sv"], a["step"], a["out"])

    bad = (dict(n=0), dict(N=0), dict(H=0), dict(W=0), dict(H=65535 * 32 + 1), dict(mode=2), dict(mode=-1),
           dict(s=0.0), dict(s=-1.0), dict(s=math.inf), dict(s=math.nan), dict(c=math.nan), dict(tan=0.0),
           dict(tan=math.inf), dict(step=0.0), dict(step=-0.1), dict(step=math.nan), dict(step=math.inf),
           dict(vol=None), dict(vm=None), dict(out=None), dict(su=math.nan), dict(su=-math.inf), dict(sv=math.nan),
           dict(sv=math.inf))
    for kw in bad:
        assert call(**kw) != 0, kw
        assert b"r2x_volume_project: bad" in lib.r2x_last_error(), kw


def test_project_argument_errors():
    torch = pytest.importorskip("torch")
    from r2_gaussian_b200.projector import project

    sc = fc.scanner("cone", 8, 4)
    vol = torch.zeros(4, 4, 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        project(vol, [0.0, 1.0], sc)
    with pytest.raises(RuntimeError, match="CUDA"):
        project(vol, [0.0, 1.0], dict(fc.scanner("parallel", 8, 4), accuracy=1.0))
    for cfg, match in ((dict(sc, nVoxel=[4, 4, 5]), "nVoxel"), (dict(sc, accuracy=0.0), "accuracy"),
                       (dict(sc, accuracy=-0.5), "accuracy"), (dict(sc, offDetector=[0.1, 0.0]), "offDetector"),
                       (dict(sc, offDetector=[0.0, -0.2]), "offDetector"),
                       (dict(fc.scanner("parallel", 8, 4), sDetector=[2.0, 3.0]), "sDetector")):
        with pytest.raises(ValueError, match=match):
            project(vol, [0.0, 1.0], cfg)


# ---- noise model of generate_data -------------------------------------------------------------------------------------

def _clean(shape=(6, 20, 24), seed=3):
    return np.random.RandomState(seed).uniform(0.5, 2.5, size=shape).astype(np.float32)


def test_noise_is_seeded():
    from r2_gaussian_b200.generate_data import add_noise

    p = _clean()
    a = add_noise(p, 1e4, [0, 10], np.random.RandomState(0))
    b = add_noise(p, 1e4, [0, 10], np.random.RandomState(0))
    c = add_noise(p, 1e4, [0, 10], np.random.RandomState(1))
    assert a.dtype == np.float32 and a.shape == p.shape
    assert a.tobytes() == b.tobytes()
    assert a.tobytes() != c.tobytes()
    assert (a >= 0.0).all()


def test_noise_clamps_to_nonnegative():
    from r2_gaussian_b200.generate_data import add_noise

    p = _clean()
    p[:, :4] = 0.0                                            # I ~ I0 there: half the noisy values would be < 0
    out = add_noise(p, 1e3, [0, 30], np.random.RandomState(0))
    assert (out >= 0.0).all() and (out[:, :4] == 0.0).any()


def test_noise_is_unbiased_for_a_large_dose():
    """gaussian_noise = [0, 0], I0 = 1e7: the per-pixel std is m / sqrt(I0 exp(-p/m)) <= 0.0009 m, so the mean over the
    stack is within 6 standard errors (plus the O(m / I0) log bias) of the clean mean."""
    from r2_gaussian_b200.generate_data import add_noise

    p = _clean()
    I0, m = 1e7, float(p.max())
    out = add_noise(p, I0, [0, 0], np.random.RandomState(0)).astype(np.float64)
    sigma = m / math.sqrt(I0 * math.exp(-1.0))
    bound = 6.0 * sigma / math.sqrt(p.size) + 10.0 * m / (I0 * math.exp(-1.0))
    assert abs(out.mean() - p.mean()) <= bound, (out.mean() - p.mean(), bound)
    assert np.abs(out - p).max() <= 8.0 * sigma
