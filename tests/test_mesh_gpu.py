"""Marching cubes on the GPU (`mesh.marching_cubes`, r2x_marching_cubes_*) against tests/mesh_oracle.py.

1. Equality: faces equal and vertices equal bit for bit with the oracle for all 256 cube cases, random volumes whose
   sizes straddle the kernels' word and CTA sizes (read from csrc/r2x_mesh.cu), values exactly at the level, constant
   volumes, axes of length 1 and 2 and non-cubic grids.
2. Mesh quality: a 128^3 random zero-border volume is closed and oriented; an analytic sphere at 128^3 has area and
   enclosed volume within 0.1 %; two calls give the same bits.
3. A 1024^3 checkerboard needs more than 2^31 vertices: refused with both counts before any output is allocated.
4. End to end: `extract_mesh` on a generated scene's vol_gt, on recon's FDK volume and on a briefly trained model."""
import json
import math
import os
import re

import numpy as np
import pytest
import torch

import mesh_oracle as mo
from r2_gaussian_b200 import mesh

pytestmark = pytest.mark.gpu

SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "r2_gaussian_b200", "csrc",
                   "r2x_mesh.cu")


def _constexpr(name):
    return int(re.search(rf"constexpr int {name} = (\d+);", open(SRC).read()).group(1))


WORD = 32
CTA_SAMPLES = _constexpr("MC_THREADS")                                   # count / emit: one word per warp
CLASSIFY_SAMPLES = CTA_SAMPLES * _constexpr("MC_CLASSIFY_WORDS")         # classify: MC_CLASSIFY_WORDS words per warp


def _same(vol, level=0.5):
    verts, faces = mesh.marching_cubes(vol, level)
    ov, of = mo.marching_cubes(np.asarray(vol, np.float32) if not isinstance(vol, torch.Tensor)
                               else vol.float().cpu().numpy(), level)
    gv, gf = verts.cpu().numpy(), faces.cpu().numpy()
    assert gv.shape == ov.shape and gf.shape == of.shape, (gv.shape, ov.shape, gf.shape, of.shape)
    assert np.array_equal(gv.view(np.uint32), ov.view(np.uint32))
    assert np.array_equal(gf, of)
    return gv, gf


def test_all_256_cases():
    rng = np.random.default_rng(7)
    total = 0
    for c in range(256):
        vol = np.empty((2, 2, 2), np.float32)
        for b in range(8):
            inside = (c >> b) & 1
            vol[b & 1, (b >> 1) & 1, (b >> 2) & 1] = rng.uniform(0.51, 2.0) if inside else rng.uniform(-1.0, 0.5)
        _, f = _same(vol)
        total += len(f)
    assert total == 820


def _shapes():
    s, c = CTA_SAMPLES, CLASSIFY_SAMPLES
    return [(1, 1, WORD - 1), (1, 1, WORD), (1, 1, WORD + 1), (2, 2, WORD + 1), (3, 5, WORD - 1),
            (1, 2, s // 2 - 1), (2, 2, s // 4 + 1), (4, 4, s // 16), (2, 4, s // 8 + 1), (3, 3, c // 9 + 1),
            (4, 8, c // 32), (4, 8, c // 32 + 1), (7, 11, 13), (9, 9, 33), (33, 31, 32), (17, 65, 5), (64, 3, 63)]


@pytest.mark.parametrize("shape", _shapes())
def test_random_volumes_around_the_tile_sizes(shape):
    rng = np.random.default_rng(sum(shape))
    _same(rng.random(shape, dtype=np.float32))


def test_values_exactly_at_the_level():
    rng = np.random.default_rng(3)
    vol = (rng.integers(0, 3, (23, 19, 37)) * 0.25).astype(np.float32)      # 0, 0.25, 0.5: ties at level 0.25
    v, f = _same(vol, 0.25)
    assert len(f) > 0
    vol = np.full((5, 6, 7), 0.5, np.float32)
    vol[2, 3, 4] = 1.0
    v, f = _same(vol, 0.5)
    assert len(f) == 8


@pytest.mark.parametrize("value", [0.0, 0.5, 1.0])
def test_constant_volumes_are_empty(value):
    v, f = mesh.marching_cubes(torch.full((9, 10, 11), value, device="cuda"), 0.5)
    assert v.shape == (0, 3) and f.shape == (0, 3) and v.dtype == torch.float32 and f.dtype == torch.int32


@pytest.mark.parametrize("shape", [(1, 1, 1), (1, 1, 2), (2, 1, 1), (1, 7, 9), (6, 1, 5), (4, 9, 1), (2, 2, 2),
                                   (2, 5, 2), (1, 2, 40), (2, 40, 1)])
def test_short_axes(shape):
    rng = np.random.default_rng(len(shape) + sum(shape))
    _same(rng.random(shape, dtype=np.float32))


def test_non_cubic_grids_and_inputs():
    rng = np.random.default_rng(11)
    vol = rng.random((20, 36, 28))                                 # float64 host array: rounded to float32 first
    _same(vol.astype(np.float32))
    g64 = mesh.marching_cubes(vol, 0.5)
    g32 = mesh.marching_cubes(torch.from_numpy(vol.astype(np.float32)).cuda(), 0.5)
    assert torch.equal(g64[0], g32[0]) and torch.equal(g64[1], g32[1])
    _same(torch.from_numpy(rng.random((37, 8, 50), dtype=np.float32)).cuda(), 0.3)


def test_refusals_on_the_device():
    for bad in (float("nan"), float("inf"), -float("inf")):
        vol = torch.rand(40, 40, 40, device="cuda")
        vol[11, 22, 33] = bad
        with pytest.raises(ValueError, match="non-finite"):
            mesh.marching_cubes(vol)
        with pytest.raises(ValueError, match="non-finite"):
            mesh.marching_cubes(vol.cpu().double().numpy())
    with pytest.raises(ValueError, match="finite"):
        mesh.marching_cubes(torch.rand(4, 4, 4, device="cuda"), float("inf"))


# ---- 2. mesh quality ---------------------------------------------------------------------------------------------------

def test_random_128_is_closed_and_oriented():
    gen = torch.Generator("cuda").manual_seed(5)
    vol = torch.rand((128, 128, 128), generator=gen, device="cuda")
    for ax in range(3):
        vol.select(ax, 0).zero_()
        vol.select(ax, 127).zero_()
    v, f = mesh.marching_cubes(vol, 0.5)
    fn = f.cpu().numpy()
    assert len(fn) > 10 ** 6
    assert mo.directed_edge_defects(fn) == 0
    assert len(np.unique(fn)) == len(v)
    assert mo.signed_volume(v.cpu().numpy(), fn) > 0


def test_sphere_128_area_and_volume():
    n, r = 128, 0.35 * 128
    g = torch.arange(n, device="cuda", dtype=torch.float64) - (n - 1) / 2
    X, Y, Z = torch.meshgrid(g, g, g, indexing="ij")
    vol = (r - torch.sqrt(X * X + Y * Y + Z * Z)).float()
    v, f = _same(vol, 0.0)
    assert mo.directed_edge_defects(f) == 0 and mo.euler_characteristic(v, f) == 2
    da = mo.area(v, f) / (4 * math.pi * r * r) - 1
    dv = mo.signed_volume(v, f) / (4 / 3 * math.pi * r ** 3) - 1
    print(f"sphere r = {r} at {n}^3: area {da:+.4%}, volume {dv:+.4%}")
    assert abs(da) < 1e-3 and abs(dv) < 1e-3


def test_two_calls_give_the_same_bits():
    gen = torch.Generator("cuda").manual_seed(9)
    vol = torch.rand((96, 80, 112), generator=gen, device="cuda")
    a, b = mesh.marching_cubes(vol, 0.6), mesh.marching_cubes(vol, 0.6)
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32)) and torch.equal(a[1], b[1])


# ---- 3. int32 overflow -------------------------------------------------------------------------------------------------

def test_overflow_is_refused_with_both_counts():
    n = 1024
    p = torch.arange(n, device="cuda", dtype=torch.uint8) % 2
    vol = ((p[:, None, None] + p[None, :, None] + p[None, None, :]) % 2).float()    # every edge is cut
    del p
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    want_v = 3 * (n - 1) * n * n
    want_t = 4 * (n - 1) ** 3                   # every cube: 4 separated corners
    with pytest.raises(ValueError) as e:
        mesh.marching_cubes(vol, 0.5)
    msg = str(e.value)
    assert str(want_v) in msg and str(want_t) in msg, msg
    # the scratch (0.625 bytes per sample) and small reductions, no output (~89 GB)
    assert torch.cuda.max_memory_allocated() - before < 2 * n ** 3
    del vol, e
    torch.cuda.empty_cache()


# ---- 4. end to end -------------------------------------------------------------------------------------------------------

def _read_ply(path):
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii")
    nv = int(re.search(r"element vertex (\d+)", head).group(1))
    nf = int(re.search(r"element face (\d+)", head).group(1))
    body = data[end:]
    assert len(body) == 12 * nv + 13 * nf
    v = np.frombuffer(body, "<f4", 3 * nv).reshape(nv, 3)
    rec = np.frombuffer(body[12 * nv:], dtype=[("n", "u1"), ("idx", "<i4", (3,))], count=nf)
    assert (rec["n"] == 3).all()
    return v, rec["idx"].copy()


@pytest.fixture(scope="module")
def ellipsoid_scene(tmp_path_factory):
    """A 48^3 generate_data scene of a smooth ellipsoid that stays clear of the border (24 train, 4 test views of
    96^2), with its initial cloud."""
    from r2_gaussian_b200 import generate_data, initialize_pcd, scene
    tmp = tmp_path_factory.mktemp("mesh_scene")
    n = 48
    g = (np.arange(n) + 0.5) / n * 2 - 1
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    q = (X / 0.6) ** 2 + (Y / 0.45) ** 2 + ((Z - 0.1) / 0.5) ** 2
    vol = np.clip(1.0 - q, 0.0, None).astype(np.float32) * 0.8
    np.save(tmp / "vol.npy", vol)
    sc = scene.cone_beam_scanner(96, n)
    phys = {k: (np.asarray(v, float) * 2.0).tolist() if k in ("DSD", "DSO", "sDetector", "sVoxel", "offOrigin",
                                                              "offDetector") else v for k, v in sc.items()}
    phys.update({"filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0, "noise": False})
    (tmp / "scanner.yml").write_text("".join(f"{k}: {json.dumps(v)}\n" for k, v in phys.items()))
    src = generate_data.main(["--vol", str(tmp / "vol.npy"), "--scanner", str(tmp / "scanner.yml"), "--n_train", "24",
                              "--n_test", "4", "--output", str(tmp / "data")])
    init = initialize_pcd.main(["--data", src, "--n_points", "5000", "--output", str(tmp / "init.npy")])
    return src, init, tmp


LEVEL = 0.3


def _extract(argv, capsys):
    from r2_gaussian_b200 import extract_mesh
    rep = extract_mesh.main(argv)
    line = capsys.readouterr().out.strip().splitlines()[-1]
    assert json.loads(line)["triangles"] == rep["triangles"]
    return rep


def _check_scene_mesh(path, cfg, closed=True):
    v, f = _read_ply(path)
    assert len(f) > 0
    lo = np.asarray(cfg["offOrigin"]) - np.asarray(cfg["sVoxel"]) / 2
    hi = lo + np.asarray(cfg["sVoxel"])
    assert (v >= lo).all() and (v <= hi).all()
    if closed:
        assert mo.directed_edge_defects(f) == 0
    return mo.signed_volume(v, f)


def test_extract_mesh_end_to_end(ellipsoid_scene, tmp_path, capsys):
    from r2_gaussian_b200 import recon, trainer
    from r2_gaussian_b200.dataset import read_scene
    src, init, _ = ellipsoid_scene
    cfg = read_scene(src, eval=False).scanner_cfg
    gt = _extract(["-s", src, "--level", str(LEVEL), "--output", str(tmp_path / "gt.ply")], capsys)
    assert gt["source"] == "scene" and gt["shape"] == [48, 48, 48]
    vol_gt = _check_scene_mesh(str(tmp_path / "gt.ply"), cfg)
    assert vol_gt > 0

    recon.main(["-s", src, "-m", str(tmp_path / "recon"), "--methods", "fdk"])
    capsys.readouterr()
    fdk = _extract(["--vol", str(tmp_path / "recon" / "fdk" / "ct_pred.npy"), "-s", src, "--level", str(LEVEL),
                    "--output", str(tmp_path / "fdk.ply")], capsys)
    assert fdk["source"] == "vol"
    _check_scene_mesh(str(tmp_path / "fdk.ply"), cfg, closed=False)

    model = tmp_path / "model"
    trainer.main(["-s", src, "-m", str(model), "--ply_path", init, "--iterations", "600", "--test_iterations", "600",
                  "--save_iterations", "600"])
    capsys.readouterr()
    pred = _extract(["-m", str(model), "--resolution", "96", "--level", str(LEVEL), "--output",
                     str(tmp_path / "pred.ply")], capsys)
    assert pred["source"] == "model@600" and pred["shape"] == [96, 96, 96]
    vol_pred = _check_scene_mesh(str(tmp_path / "pred.ply"), cfg, closed=False)
    # recorded, not judged: how close the trained field's surface encloses the ground truth's
    with capsys.disabled():
        print(f"\nenclosed volume at level {LEVEL}: vol_gt mesh {vol_gt:.6f}, model mesh at 96^3 {vol_pred:.6f} "
              f"({vol_pred / vol_gt - 1:+.2%}); gt {gt['triangles']}, fdk {fdk['triangles']}, model "
              f"{pred['triangles']} triangles")
    # index space when no scene is given
    ix = _extract(["--vol", str(tmp_path / "recon" / "fdk" / "ct_gt.npy"), "--level", str(LEVEL), "--output",
                   str(tmp_path / "ix.ply")], capsys)
    v, _ = _read_ply(str(tmp_path / "ix.ply"))
    assert ix["triangles"] == gt["triangles"] and v.min() >= 0 and v.max() <= 47
