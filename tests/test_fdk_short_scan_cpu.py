"""Short-scan FDK (Parker weights) on the CPU: the sign of the fan angle against make_view's geometry, the arc and
interval rule of `fdk.short_scan_views`, the float64 oracle's round trip at 220 degrees, the 180-degree parallel case,
and every refusal before any CUDA call (Python, both command lines, the C ABI)."""
import ctypes
import math

import numpy as np
import pytest

import fdk_cases as fc
import fdk_short_scan_oracle as sso
from oracle import fdk_oracle
from oracle import r2_oracle as orc
from r2_gaussian_b200 import scene
from r2_gaussian_b200.fdk import short_scan_views

# 220-degree cone round trip with the cloud, grid and detector of test_fdk_cpu's round trip, at 31 views (the view
# density of its 50-view full scan).  Bounds measured with the oracle: Parker 0.088, unweighted 0.237.
SHORT_VIEWS, SHORT_ARC = 31, 220.0
PARKER_BOUND, PLAIN_FLOOR = 0.095, 0.2


def arc_angles(deg, n, start=0.0):
    return np.linspace(0.0, math.radians(deg), n + 1)[:-1] + start


def _ray(sc, theta, u):
    """Source and unit direction in world space, float64, of the mid-row ray at camera-frame slope u = ndc_x tan_fovx,
    from the pose make_view is built from (checked against its float32 viewmatrix)."""
    c2w = scene.angle2pose(sc["DSO"], theta)
    vm = np.linalg.inv(scene.make_view(sc, theta).viewmatrix.astype(np.float64).T)
    assert np.abs(vm - c2w).max() < 1e-5
    d = c2w[:3, :3] @ np.array([u, 0.0, 1.0])
    return c2w[:3, 3], d / np.linalg.norm(d)


def _line_distance(o1, d1, o2, d2):
    """0 when the two rays lie on the same line."""
    return max(np.linalg.norm(np.cross(d1, d2)), np.linalg.norm(np.cross(o2 - o1, d1)))


@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_conjugate_ray_and_weights_against_make_view(sign):
    sc = fc.scanner("cone", 64, 32)
    v = scene.make_view(sc, 0.0)
    W, arc = 64, math.radians(SHORT_ARC)
    gam = sign * sso.fan_angles(W, v.tanfovx, v.mode)
    rng = np.random.RandomState(3)
    worst, checked = 0.0, 0
    for beta, j in zip(rng.uniform(0.0, arc, 200), rng.randint(0, W, 200)):
        g = gam[j]
        o1, d1 = _ray(sc, 1.1 + beta, math.tan(-sign * g))             # ndc_x(j) tan_fovx, from gamma
        o2, d2 = _ray(sc, 1.1 + beta + math.pi + 2.0 * g, math.tan(sign * g))
        worst = max(worst, _line_distance(o1, d1, o2, d2))
        conj = beta + math.pi + 2.0 * g
        if conj <= arc:
            s = sso.parker_weights(beta, g, arc) + sso.parker_weights(conj, -g, arc)
            assert abs(s - 1.0) <= 1e-12, (beta, g, s)
            checked += 1
    assert checked > 20
    if sign > 0:
        assert worst <= 1e-9, worst
    else:
        assert worst > 1e-3, worst


def test_rays_measured_once_have_weight_one():
    """Neither (beta + pi + 2 gamma) nor (beta - pi + 2 gamma) is on the arc: w = 1."""
    arc = math.radians(SHORT_ARC)
    gam = sso.fan_angles(64, 2.0 / 7.0, 1)
    beta = np.linspace(0.0, arc, 500)
    b, g = np.meshgrid(beta, gam, indexing="ij")
    once = (b + math.pi + 2.0 * g > arc) & (b - math.pi + 2.0 * g < 0.0)
    assert once.sum() > 100
    np.testing.assert_array_equal(sso.parker_weights(b, g, arc)[once], 1.0)


@pytest.mark.parametrize("deg,n,start", [(220.0, 40, 0.0), (220.0, 17, 1.3), (300.0, 60, -2.0), (200.0, 9, 5.9)])
def test_arc_and_intervals_of_uniform_scans(deg, n, start):
    vw, arc = short_scan_views(arc_angles(deg, n, start), 0, 1.0)
    assert abs(arc - math.radians(deg)) <= 1e-12
    np.testing.assert_allclose(vw[:, 1], math.radians(deg) / n, rtol=0, atol=1e-12)
    np.testing.assert_allclose(vw[:, 0], (np.arange(n) + 0.5) * math.radians(deg) / n, rtol=0, atol=1e-12)


def test_arc_across_two_pi_shuffled_and_irregular():
    ref, arc = short_scan_views(arc_angles(220.0, 30), 1, 0.3)
    crossing = np.mod(arc_angles(220.0, 30, math.radians(300.0)), 2.0 * math.pi)   # 300 ... 160 degrees
    got, arc2 = short_scan_views(crossing, 1, 0.3)
    assert abs(arc2 - arc) <= 1e-12
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-12)
    perm = np.random.RandomState(0).permutation(30)
    shuffled, _ = short_scan_views(crossing[perm], 1, 0.3)
    np.testing.assert_array_equal(shuffled, got[perm])
    rng = np.random.RandomState(1)
    irregular = np.sort(rng.uniform(0.0, math.radians(230.0), 25))
    irregular = np.append(irregular, irregular[4])                                   # two views at the same angle
    vw, arc3 = short_scan_views(irregular, 0, 1.0)
    assert abs(vw[:, 1].sum() - arc3) <= 1e-12
    assert vw[4, 1] == vw[-1, 1] and vw[4, 0] == vw[-1, 0]
    assert (vw[:, 1] > 0).all()


def _round_trip(angles):
    cloud = fc.round_trip_cloud()
    sc = fc.scanner("cone", fc.ROUND_TRIP_DET, fc.ROUND_TRIP_VOX)
    projs = []
    for a in angles:
        v = scene.make_view(sc, float(a))
        projs.append(orc.raster_forward(cloud.means, cloud.scales, cloud.rotations, cloud.density, v.viewmatrix,
                                        v.projmatrix, v.image_width, v.image_height, v.tanfovx, v.tanfovy,
                                        v.mode)["image"])
    want = orc.voxel_forward(cloud.means, cloud.scales, cloud.rotations, cloud.density, sc["nVoxel"], sc["sVoxel"],
                             sc["offOrigin"])["vol"]
    return np.stack(projs), sc, want


def test_oracle_round_trip_220_cone():
    angles = arc_angles(SHORT_ARC, SHORT_VIEWS, 0.3)
    projs, sc, want = _round_trip(angles)
    got = sso.fdk_short_scan_scene(projs, angles, sc)
    err = fc.rel_l2(got, want)
    assert err <= PARKER_BOUND, err
    assert fc.rel_l2(fdk_oracle.fdk_scene(projs, angles, sc), want) >= PLAIN_FLOOR
    assert fc.rel_l2(got[::-1], want) >= 0.5


def test_ball_amplitude_short_scan():
    """The analytic ball of test_ball_amplitude at 220 degrees: the centre reconstructs to 1 with the same tolerance
    (the unweighted FDK of the same views misses it)."""
    sc = fc.scanner("cone", 64, 32)
    angles = arc_angles(SHORT_ARC, 110)
    projs = fc.ball_projections(sc, angles)
    centre = sso.fdk_short_scan_scene(projs, angles, sc)[13:19, 13:19, 13:19]
    assert abs(centre.mean() - 1.0) <= 0.02, centre.mean()
    assert np.abs(centre - 1.0).max() <= 0.02, np.abs(centre - 1.0).max()
    plain = fdk_oracle.fdk_scene(projs, angles, sc)[13:19, 13:19, 13:19]
    assert np.abs(plain - 1.0).max() > 0.02


def test_parallel_180_equals_plain_fdk():
    sc = fc.scanner("parallel", 24, 12)
    angles = arc_angles(180.0, 20, 0.4)
    projs = np.random.RandomState(5).uniform(0.0, 1.0, size=(20, 24, 24))
    vw, arc = short_scan_views(angles, 0, 1.0)
    np.testing.assert_array_equal(sso.parker_weights(vw[:, :1], np.zeros((1, 24)), arc), 1.0)
    got = sso.fdk_short_scan_scene(projs, angles, sc)
    want = fdk_oracle.fdk_scene(projs, angles, sc)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()


def test_refusals():
    with pytest.raises(ValueError, match=r"arc of 200\.00 degrees.*at least 211\.89"):
        short_scan_views(arc_angles(200.0, 30), 1, 2.0 / 7.0)
    short_scan_views(arc_angles(212.0, 30), 1, 2.0 / 7.0)
    short_scan_views(arc_angles(180.0, 30), 0, 1.0)
    with pytest.raises(ValueError, match=r"arc of 179\.00 degrees.*at least 180\.00"):
        short_scan_views(arc_angles(179.0, 30), 0, 1.0)
    with pytest.raises(ValueError, match="full circle"):
        short_scan_views(fc.full_scan(30), 1, 2.0 / 7.0)
    with pytest.raises(ValueError, match="at least 2 views"):
        short_scan_views([0.5], 1, 2.0 / 7.0)


def test_fdk_short_scan_rejects_host_tensors():
    torch = pytest.importorskip("torch")
    from r2_gaussian_b200.fdk import fdk

    sc = fc.scanner("cone", 8, 4)
    with pytest.raises(RuntimeError, match="CUDA"):
        fdk(torch.zeros(2, 8, 8), [0.0, 1.0], sc, short_scan=True)


@pytest.mark.parametrize("method", ["random", "cgls", "fista_tv", "volume"])
def test_initialize_pcd_refuses_short_scan_without_fdk(method, tmp_path):
    from r2_gaussian_b200 import initialize_pcd

    with pytest.raises(SystemExit, match="--short_scan applies to --recon_method fdk only"):
        initialize_pcd.main(["--data", str(tmp_path / "none"), "--recon_method", method, "--short_scan"])


def test_recon_refuses_short_scan_without_fdk(tmp_path):
    from r2_gaussian_b200 import recon

    with pytest.raises(SystemExit, match="--short_scan applies to the fdk method"):
        recon.main(["-s", str(tmp_path / "none"), "-m", str(tmp_path / "out"), "--methods", "sart,cgls",
                    "--short_scan"])
    with pytest.raises(ValueError, match="short_scan applies to fdk only"):
        recon.recon_volume(None, [0.0, 1.0], {}, "cgls", short_scan=True)


def test_abi_rejects_bad_arguments_before_any_cuda_call():
    from r2_gaussian_b200 import _lib

    lib = _lib.load()
    dummy = ctypes.c_void_p(16)
    tx = 0.3
    base = dict(N=2, H=8, W=8, mode=1, su=0.0, dso=5.0, n=4, s=2.0, w=dummy, arc=math.radians(220.0), nbytes=1 << 20)

    def call(**kw):
        a = dict(base, **kw)
        return lib.r2x_fdk(None, a["N"], a["H"], a["W"], dummy, dummy, dummy, tx, tx, a["mode"], a["su"], 0.0, 1, a["w"],
                           a["arc"], a["dso"], a["n"], a["n"], a["n"], a["s"], a["s"], a["s"], 0.0, 0.0, 0.0, dummy, dummy,
                           a["nbytes"])

    for kw in (dict(N=0), dict(N=1), dict(H=0), dict(W=0), dict(n=0), dict(mode=2), dict(dso=0.0), dict(s=0.0),
               dict(w=None), dict(arc=0.0), dict(arc=2.0 * math.pi), dict(arc=float("nan")),
               dict(arc=math.pi + 2.0 * math.atan(tx) - 1e-3), dict(mode=0, arc=math.pi - 1e-3), dict(su=0.5),
               dict(su=-1.0)):
        assert call(**kw) != 0, kw
        assert b"bad" in lib.r2x_last_error(), kw
    assert call(nbytes=16) != 0                                 # scratch too small
    assert b"scratch" in lib.r2x_last_error()
