"""Helical FDK without a GPU: the oracle's conjugate geometry against the rasterizer's matrices, the normalisation of
its weights, the helix fit against generate_data's helices, and the refusals of the Python layer, the command lines and
the C ABI before any CUDA work."""
import ctypes
import math

import numpy as np
import pytest
import torch

import fdk_helical_oracle as fho
import view_geometry_oracle as vgo
from r2_gaussian_b200 import fdk, scene


def _helix(sc, angles, geo):
    return fdk.helix_views(angles, sc, geo)


def _source(hx, beta, dso):
    return np.array([dso * math.cos(beta) + hx.c_x, dso * math.sin(beta) + hx.c_y, hx.z0 + hx.h * beta])


def test_conjugates_are_collinear_and_nu0_is_the_ndc_row():
    sc, angles, geo = fho.helix_case(60, 2.0, 1.4)
    hx = _helix(sc, angles, geo)
    dso, rng = float(sc["DSO"]), np.random.RandomState(0)
    tany = float(scene.make_view(sc, 0.0).tanfovy)
    for _ in range(200):
        beta = rng.uniform(hx.beta_lo, hx.beta_hi)
        x = rng.uniform(-0.6, 0.6, 3) + np.asarray(sc["offOrigin"])
        zin, gam, zc = (float(v) for v in fho.conjugate_geometry(beta, np.array(x[0]), np.array(x[1]), dso, hx.c_x,
                                                                   hx.c_y))
        s0, s1 = _source(hx, beta, dso), _source(hx, beta + math.pi + 2.0 * gam, dso)
        d0, d1 = x[:2] - s0[:2], s1[:2] - x[:2]
        assert abs(d0[0] * d1[1] - d0[1] * d1[0]) <= 1e-12 * np.dot(d0, d0) ** 0.5 * np.dot(d1, d1) ** 0.5 + 1e-12
        assert np.dot(d0, d1) > 0                                     # x lies between the two sources
        assert zc == pytest.approx(np.linalg.norm(d1) * math.cos(gam), rel=1e-12, abs=1e-12)
        # each candidate's nu is minus the ndc row of x in the camera of a view at that angle
        for bk, depth in ((beta, zin), (beta + math.pi + 2.0 * gam, zc)):
            zs = hx.z0 + hx.h * bk
            pos = [sc["offOrigin"][0] - hx.c_x, sc["offOrigin"][1] - hx.c_y, sc["offOrigin"][2] - zs]
            v = scene.make_view(scene.view_scanner(sc, {"offOrigin": pos}), float(bk), True)
            pm = v.projmatrix.astype(np.float64).reshape(16)
            ndc_y = fho.fdk_oracle._row(pm, 1, *x) / (fho.fdk_oracle._row(pm, 3, *x) + 1e-7)
            nu = (x[2] - zs) / (depth * tany)
            assert nu == pytest.approx(-ndc_y, rel=2e-5, abs=2e-6), (bk, nu, ndc_y)


@pytest.mark.parametrize("q", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("travel", [1.4, -0.9, 0.0])
def test_weights_of_a_line_sum_to_one(q, travel):
    sc, angles, geo = fho.helix_case(90, 3.0 if travel else 1.0, travel)
    hx = _helix(sc, angles, geo)
    dso, rng = float(sc["DSO"]), np.random.RandomState(1)
    tany = float(scene.make_view(sc, 0.0).tanfovy)
    checked = 0
    for _ in range(300):
        beta = rng.uniform(hx.beta_lo, hx.beta_hi)
        x = rng.uniform(-0.6, 0.6, 3) + np.asarray(sc["offOrigin"])
        X, Y, Z = (np.array(v) for v in x)
        zin, gam, zc = fho.conjugate_geometry(beta, X, Y, dso, hx.c_x, hx.c_y)
        members = [float(b) for b, _, ok in fho.candidates(beta, gam, zin, zc, hx) if ok]
        ws = [float(fho.weights(b, X, Y, Z, hx, dso, tany, q)) for b in members]
        if sum(ws) == 0.0:
            continue
        checked += 1
        assert sum(ws) == pytest.approx(1.0, abs=1e-12), (members, ws)
    assert checked > 50


def test_circle_with_q1_halves_every_ray_seen_twice():
    sc, angles, geo = fho.helix_case(72, 1.0, 0.0, sdet=(1.6, 2.6))
    hx = _helix(sc, angles, geo)
    assert hx.h == 0.0 and hx.beta_hi - hx.beta_lo == pytest.approx(2.0 * math.pi)
    assert np.allclose(hx.dbeta, 2.0 * math.pi / 72)
    dso, rng = float(sc["DSO"]), np.random.RandomState(2)
    tany = float(scene.make_view(sc, 0.0).tanfovy)
    seen = 0
    for _ in range(400):
        beta = rng.uniform(hx.beta_lo, hx.beta_hi)
        x = rng.uniform(-0.6, 0.6, 3) + np.asarray(sc["offOrigin"])
        X, Y, Z = (np.array(v) for v in x)
        zin, gam, zc = fho.conjugate_geometry(beta, X, Y, dso, hx.c_x, hx.c_y)
        nu0, nuc = (Z - hx.z0) / (zin * tany), (Z - hx.z0) / (zc * tany)
        if abs(nu0) < 1.0 and abs(nuc) < 1.0:
            seen += 1
            assert float(fho.weights(beta, X, Y, Z, hx, dso, tany, 1.0)) == 0.5
    assert seen > 100


def _generated(n, total_deg, start_deg, travel, off=(0.0, 0.0, 0.3)):
    from r2_gaussian_b200.generate_data import helical_offsets, train_angles
    cfg = {"totalAngle": total_deg, "startAngle": start_deg, "offOrigin": list(off)}
    angles = train_angles(cfg, n)
    return angles, helical_offsets(cfg, angles, travel)


@pytest.mark.parametrize("travel", [3.2, -2.0])
def test_helix_fit_recovers_generate_data(travel):
    sc = scene.cone_beam_scanner(16, 8)
    sc["offOrigin"] = [0.0, 0.0, 0.3]
    angles, geo = _generated(120, 720.0, 30.0, travel)
    h_want = -travel / math.radians(720.0)
    z0_want = travel * (30.0 / 720.0 + 0.5)
    rng = np.random.RandomState(3)
    for a in (angles, np.mod(angles, 2.0 * math.pi)):
        perm = rng.permutation(len(a))
        for ang, g in ((a, geo), (a[perm], [geo[i] for i in perm])):
            hx = fdk.helix_views(ang, sc, g)
            assert np.all(np.diff(hx.beta) > 0)
            # the fitted helix places each view's source where its camera puts it
            assert hx.h == pytest.approx(h_want, rel=1e-9)
            zs = sc["offOrigin"][2] - np.array([g[i]["offOrigin"][2] for i in hx.order])
            assert np.abs(hx.z0 + hx.h * hx.beta - zs).max() < 1e-9
            assert np.allclose(np.mod(hx.beta - np.asarray(ang)[hx.order], 2 * math.pi) % (2 * math.pi), 0.0,
                               atol=1e-9) or np.allclose(np.cos(hx.beta - np.asarray(ang)[hx.order]), 1.0)
            if ang is angles:
                assert hx.z0 == pytest.approx(z0_want, abs=1e-9)
                assert list(hx.order) == list(range(len(a)))
            assert hx.beta_hi - hx.beta_lo == pytest.approx(4.0 * math.pi)
            assert hx.dbeta.sum() == pytest.approx(4.0 * math.pi)


def test_helix_fit_refusals():
    sc, angles, geo = fho.helix_case(40, 1.5, 1.0)
    fdk.helix_views(angles, sc, geo)

    def refused(msg, a=angles, g=geo, s=sc):
        with pytest.raises(ValueError, match=msg):
            fdk.helix_views(a, s, g)

    bent = [dict(g) for g in geo]
    bent[7] = {"offOrigin": [geo[7]["offOrigin"][0], geo[7]["offOrigin"][1], geo[7]["offOrigin"][2] + 0.01]}
    refused("not affine", g=bent)
    refused("DSO varies", g=[dict(g, DSO=5.0 + 0.01 * (i % 2)) for i, g in enumerate(geo)])
    refused("DSD varies", g=[dict(g, DSD=7.0 + 0.01 * (i % 2)) for i, g in enumerate(geo)])
    refused("offDetector varies", g=[dict(g, offDetector=[0.01 * (i % 2), 0.0]) for i, g in enumerate(geo)])
    refused("detector is offset", g=[dict(g, offDetector=[0.02, 0.0]) for g in geo])
    refused("x / y varies", g=[{"offOrigin": [0.05 + 0.01 * (i % 2), *g["offOrigin"][1:]]} for i, g in enumerate(geo)])
    short_sc, short_a, short_g = fho.helix_case(40, 0.8, 1.0)
    refused("at least 360", short_a, short_g, short_sc)
    refused("cone beam only", s=dict(sc, mode="parallel"))
    refused("at least 2 views", angles[:1], geo[:1])
    refused("advance monotonically", np.concatenate([angles[:20], angles[20:][::-1]]), geo)


def test_fdk_refuses_before_any_cuda_work():
    sc, angles, geo = fho.helix_case(40, 1.5, 1.0)
    p = torch.zeros(40, *sc["nDetector"])
    for kw, msg in (({"short_scan": True}, "helical cannot be combined with short_scan"),
                    ({"half_fan": True, "use_offDetector": True}, "helical cannot be combined with half_fan"),
                    ({"helical_q": 1.5}, "helical_q must be in"), ({"helical_q": -0.1}, "helical_q must be in")):
        with pytest.raises(ValueError, match=msg):
            fdk.fdk(p, angles, sc, view_geometry=geo, helical=True, **kw)
    with pytest.raises(ValueError, match="helical needs view_geometry"):
        fdk.fdk(p, angles, sc, helical=True)
    with pytest.raises(ValueError, match="DSO varies"):
        fdk.fdk(p, angles, sc, view_geometry=[dict(g, DSO=5.0 + 0.01 * i) for i, g in enumerate(geo)], helical=True)
    # without the flag a helical table is refused as before, with a pointer to the flag
    with pytest.raises(ValueError, match="cgls, sart, fista_tv or cp_tv") as e:
        fdk.fdk(p, angles, sc, view_geometry=geo)
    assert "helical=True" in str(e.value)
    # a valid call gets as far as the device check
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        fdk.fdk(p, angles, sc, view_geometry=geo, helical=True, filter="hann")


def _helical_scene(tmp_path, name="h", bend=False):
    sc = vgo.file_scanner()
    n = 24
    frames = []
    for i in range(n):
        z = 2.0 * (i / n - 0.5) + (0.02 if bend and i == 5 else 0.0)
        frames.append((4.0 * math.pi * i / n, {"offOrigin": [0.0, 0.0, z]}))
    return vgo.write_scene(str(tmp_path / name), sc, frames)


def test_command_lines_refuse_before_any_cuda_work(tmp_path):
    from r2_gaussian_b200 import initialize_pcd, recon

    src = _helical_scene(tmp_path)
    out = str(tmp_path / "o")
    cases = ((["--use_view_geometry", "--helical", "--short_scan"], "--helical cannot be combined with --short_scan"),
             (["--use_view_geometry", "--helical", "--half_fan", "--use_offDetector"],
              "--helical cannot be combined with --half_fan"),
             (["--use_view_geometry", "--helical", "--estimate_offDetector"],
              "--helical cannot be combined with --estimate_offDetector"),
             (["--helical"], "--helical needs --use_view_geometry"),
             (["--use_view_geometry", "--helical_q", "0.5"], "--helical_q applies with --helical only"),
             (["--use_view_geometry", "--helical", "--helical_q", "1.5"], "--helical_q must be in"))
    for flags, msg in cases:
        with pytest.raises(SystemExit, match=msg):
            recon.main(["-s", src, "-m", out, "--methods", "fdk", *flags])
        with pytest.raises(SystemExit, match=msg):
            initialize_pcd.main(["--data", src, "--recon_method", "fdk", *flags])
    with pytest.raises(SystemExit, match="applies to the fdk method"):
        recon.main(["-s", src, "-m", out, "--methods", "cgls", "--use_view_geometry", "--helical"])
    with pytest.raises(SystemExit, match="applies to --recon_method fdk only"):
        initialize_pcd.main(["--data", src, "--recon_method", "cgls", "--use_view_geometry", "--helical"])
    # the fit's refusals reach the command line before any CUDA work
    with pytest.raises(SystemExit, match="--helical: fdk helical: the volume's z is not affine"):
        initialize_pcd.main(["--data", _helical_scene(tmp_path, "bent", True), "--recon_method", "fdk",
                             "--use_view_geometry", "--helical"])
    # without the flag the helical scene is refused as before, with a pointer to the flag
    with pytest.raises(SystemExit, match="--recon_method cgls") as e:
        initialize_pcd.main(["--data", src, "--recon_method", "fdk", "--use_view_geometry"])
    assert "--helical" in str(e.value)


def test_abi_refuses_before_any_cuda_call():
    from r2_gaussian_b200 import _lib

    lib = _lib.load()
    d = ctypes.c_void_p(16)
    N = 4
    beta = np.array([0.0, 1.6, 3.2, 4.8])

    def call(b=beta, mode=1, weighting=0, q=0.5, helix=(0.1, 0.05, -0.8, 5.6, 0.0, 0.0), dev=d, W=8, nz=4,
             scratch=1 << 30, n=N):
        return lib.r2x_fdk_helical(None, n, 8, W, d, d, d, 0.3, 0.3, mode, weighting, 5.0, dev, d,
                                   b.ctypes.data if b is not None else None, *helix, q, 4, 4, nz, 2.0, 2.0, 2.0, 0.0,
                                   0.0, 0.0, d, d, scratch)

    def refused(msg, **kw):
        assert call(**kw) != 0
        assert msg in lib.r2x_last_error().decode(), lib.r2x_last_error().decode()

    refused("bad mode (cone beam only", mode=0)
    refused("bad pointer (beta, dbeta or beta_host NULL)", dev=None)
    refused("bad pointer (beta, dbeta or beta_host NULL)", b=None)
    refused("bad weighting (the filter field only", weighting=1)
    refused("bad weighting (the filter field only", weighting=2 | 0x100)
    refused("bad weighting (the filter field only", weighting=0x500)
    for i in range(6):
        for bad in (float("nan"), float("inf")):
            h = [0.1, 0.05, -0.8, 5.6, 0.0, 0.0]
            h[i] = bad
            refused("bad helix", helix=tuple(h))
    refused("bad Q", q=1.5)
    refused("bad Q", q=-0.01)
    refused("bad Q", q=float("nan"))
    refused("bad beta", b=np.array([0.0, 1.6, 1.6, 4.8]))
    refused("bad beta", b=np.array([0.0, 1.6, float("nan"), 4.8]))
    refused("bad arc (needs beta_lo", helix=(0.1, 0.05, 0.1, 5.6, 0.0, 0.0))
    refused("bad arc (needs beta_lo", helix=(0.1, 0.05, -0.8, 4.8, 0.0, 0.0))
    refused("bad arc (beta_hi - beta_lo must be at least 2 pi", helix=(0.1, 0.05, -0.1, 5.0, 0.0, 0.0))
    refused("bad N/H/W", n=0)
    refused("bad W", W=16385)
    refused("bad grid (too large)", nz=524281)
    refused("bad scratch", scratch=16)
    # r2x_fdk and r2x_fdk_views keep their refusals
    assert lib.r2x_fdk(None, N, 8, 8, d, d, d, 0.3, 0.3, 1, 0.0, 0.0, 3, d, 0.0, 5.0, 4, 4, 4, 2.0, 2.0, 2.0, 0.0, 0.0,
                       0.0, d, d, 1 << 30) != 0
    assert "bad weighting" in lib.r2x_last_error().decode()
