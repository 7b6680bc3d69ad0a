"""Marching cubes without a GPU: the generated case table against tests/mesh_oracle.py's independent derivation and
against the rules that make the mesh closed and oriented (include/r2x.h), the oracle's meshes, the PLY writer,
`to_scene`, the CLI's refusals and the C ABI's argument checks."""
import ctypes as C
import math
import os

import numpy as np
import pytest

import mesh_oracle as mo
from r2_gaussian_b200 import _lib, extract_mesh, mesh


def _library_table():
    lib = _lib.load()
    ntri = np.zeros(256, np.int32)
    edges = np.zeros(256 * 15, np.int8)
    _lib.check(lib.r2x_marching_cubes_table(ntri.ctypes.data, edges.ctypes.data), "r2x_marching_cubes_table")
    return ntri, edges.reshape(256, 15)


# ---- the case table ---------------------------------------------------------------------------------------------------

def test_library_table_equals_the_oracles():
    ntri, edges = _library_table()
    ontri, oedges = mo.case_table()
    assert np.array_equal(ntri, ontri)
    assert np.array_equal(edges, oedges)
    # the counts the rule gives: no case above 5 triangles, 820 in all
    assert ntri.max() <= 5 and int(ntri.sum()) == 820
    assert np.bincount(ntri, minlength=6).tolist() == [2, 16, 50, 80, 76, 32]
    assert ntri[0] == 0 and ntri[255] == 0
    for c in range(256):
        assert (edges[c, 3 * ntri[c]:] == -1).all()
        assert ((edges[c, :3 * ntri[c]] >= 0) & (edges[c, :3 * ntri[c]] < 12)).all()


def _cut_edges(case):
    inside = [(case >> b) & 1 for b in range(8)]
    return {e for e, (p, q) in enumerate(mo.EDGES) if inside[p] != inside[q]}


def test_every_case_obeys_the_face_rule():
    """On each face the table's boundary segments are the face rule's: each run of inside corners cut off by the
    segment joining the two cut edges that bound it, so diagonal inside corners are separated."""
    _, edges = _library_table()
    ntri, _ = _library_table()
    for c in range(256):
        tris = edges[c, :3 * ntri[c]].reshape(-1, 3).astype(int)
        directed = [(t[i], t[(i + 1) % 3]) for t in tris for i in range(3)]
        boundary = {d for d in directed if (d[1], d[0]) not in directed}
        # every directed boundary edge of the case's triangles lies in one cube face and is a face-rule segment
        want = set(mo.face_segments(c))
        assert boundary == want, c
        # the vertices are the cut edges, each used
        assert set(tris.reshape(-1).tolist()) == _cut_edges(c), c
        inside = [(c >> b) & 1 for b in range(8)]
        for cyc, fe in zip(mo.FACES, mo.FACE_EDGES):
            segs = [s for s in want if s[0] in fe and s[1] in fe]
            runs = sum(1 for i in range(4) if inside[cyc[i]] and not inside[cyc[(i + 1) % 4]])
            assert len(segs) == runs, (c, cyc)


def test_no_fan_diagonal_lies_in_a_face():
    ntri, edges = _library_table()
    for c in range(256):
        tris = edges[c, :3 * ntri[c]].reshape(-1, 3).astype(int)
        directed = [(t[i], t[(i + 1) % 3]) for t in tris for i in range(3)]
        interior = {frozenset(d) for d in directed if (d[1], d[0]) in directed}
        for d in interior:
            a, b = tuple(d)
            assert not mo.on_one_face(a, b), (c, a, b)


def test_triangles_wind_from_inside_to_outside():
    """Each triangle's normal points away from the cube's inside corners (single-corner cases)."""
    ntri, edges = _library_table()
    for b in range(8):
        for case, sign in ((1 << b, 1.0), (255 ^ (1 << b), -1.0)):
            assert ntri[case] == 1
            mid = {e: (mo.CORNERS[p] + mo.CORNERS[q]) / 2.0 for e, (p, q) in enumerate(mo.EDGES)}
            v0, v1, v2 = (mid[int(e)] for e in edges[case, :3])
            normal = np.cross(v1 - v0, v2 - v0)
            away = (v0 + v1 + v2) / 3 - mo.CORNERS[b]
            assert sign * float(normal @ away) > 0, (case, b)


# ---- the oracle's meshes ---------------------------------------------------------------------------------------------

def _zero_border(v):
    v[0] = v[-1] = 0
    v[:, 0] = v[:, -1] = 0
    v[:, :, 0] = v[:, :, -1] = 0
    return v


@pytest.mark.parametrize("seed", range(30))
def test_random_zero_border_volumes_are_closed_and_oriented(seed):
    rng = np.random.default_rng(seed)
    shape = tuple(int(n) for n in rng.integers(4, 11, 3))
    vol = _zero_border(rng.random(shape, dtype=np.float32))
    verts, faces = mo.marching_cubes(vol, 0.5)
    assert len(faces) > 0
    assert mo.directed_edge_defects(faces) == 0
    assert faces.min() >= 0 and faces.max() < len(verts)
    assert len(np.unique(faces)) == len(verts)          # every vertex is used: no welding pass needed
    assert mo.signed_volume(verts, faces) > 0


def _sphere(n, r):
    g = np.arange(n) - (n - 1) / 2
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    return (r - np.sqrt(X * X + Y * Y + Z * Z)).astype(np.float32)


def _torus(n, R, r):
    g = np.arange(n) - (n - 1) / 2
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    q = np.sqrt(X * X + Y * Y) - R
    return (r - np.sqrt(q * q + Z * Z)).astype(np.float32)


def test_euler_characteristic_of_a_sphere_and_a_torus():
    v, f = mo.marching_cubes(_sphere(40, 14.0), 0.0)
    assert mo.directed_edge_defects(f) == 0 and mo.euler_characteristic(v, f) == 2
    v, f = mo.marching_cubes(_torus(48, 13.0, 5.0), 0.0)
    assert mo.directed_edge_defects(f) == 0 and mo.euler_characteristic(v, f) == 0


def test_sphere_area_and_volume_converge():
    errs = []
    for n in (48, 64):
        r = 0.35 * n
        v, f = mo.marching_cubes(_sphere(n, r), 0.0)
        errs.append((mo.area(v, f) / (4 * math.pi * r * r) - 1, mo.signed_volume(v, f) / (4 / 3 * math.pi * r ** 3) - 1))
    (a48, v48), (a64, v64) = errs
    assert -2e-3 < a48 < 0 and -3e-3 < v48 < 0
    assert abs(a64) < abs(a48) and abs(v64) < abs(v48)


def test_oracle_vertex_arithmetic_is_float32_without_fma():
    vol = np.zeros((2, 1, 1), np.float32)
    vol[0, 0, 0], vol[1, 0, 0] = np.float32(0.1), np.float32(0.7)
    v, f = mo.marching_cubes(vol, 0.3)
    t = (np.float32(0.3) - np.float32(0.1)) / (np.float32(0.7) - np.float32(0.1))
    assert v.dtype == np.float32 and len(f) == 0
    assert v.tolist() == [[float(np.float32(0.0) + t), 0.0, 0.0]]


# ---- PLY, to_scene -----------------------------------------------------------------------------------------------------

def _read_ply(path):
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").splitlines()
    assert header[0] == "ply" and header[1] == "format binary_little_endian 1.0"
    nv = int(next(h for h in header if h.startswith("element vertex")).split()[-1])
    nf = int(next(h for h in header if h.startswith("element face")).split()[-1])
    assert "property list uchar int vertex_indices" in header
    body = data[end:]
    verts = np.frombuffer(body, "<f4", 3 * nv).reshape(nv, 3)
    rec = np.frombuffer(body[12 * nv:], dtype=[("n", "u1"), ("idx", "<i4", (3,))], count=nf)
    assert len(body) == 12 * nv + 13 * nf
    assert (rec["n"] == 3).all()
    return verts, rec["idx"].copy()


def test_ply_round_trip(tmp_path):
    v, f = mo.marching_cubes(_sphere(12, 4.0), 0.0)
    p = str(tmp_path / "m.ply")
    mesh.write_ply(p, v, f)
    rv, rf = _read_ply(p)
    assert np.array_equal(rv, v) and np.array_equal(rf, f)


def test_ply_of_an_empty_mesh(tmp_path):
    p = str(tmp_path / "empty.ply")
    mesh.write_ply(p, np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32))
    rv, rf = _read_ply(p)
    assert rv.shape == (0, 3) and rf.shape == (0, 3)


def test_ply_refuses_dangling_indices(tmp_path):
    with pytest.raises(ValueError):
        mesh.write_ply(str(tmp_path / "x.ply"), np.zeros((2, 3), np.float32), np.array([[0, 1, 2]], np.int32))


def test_to_scene_places_samples_at_voxel_centres():
    cfg = {"offOrigin": [0.1, -0.2, 0.3], "sVoxel": [2.0, 1.0, 0.5], "nVoxel": [4, 5, 8]}
    v = np.array([[0, 0, 0], [3, 4, 7], [1.5, 2.25, 0.5]], np.float32)
    got = mesh.to_scene(v, cfg)
    d = np.array(cfg["sVoxel"]) / np.array(cfg["nVoxel"])
    want = np.array(cfg["offOrigin"]) - np.array(cfg["sVoxel"]) / 2 + (v.astype(np.float64) + 0.5) * d
    assert got.dtype == np.float64 and np.array_equal(got, want)
    # the first and last samples sit half a voxel inside the box
    assert np.allclose(got[0], np.array(cfg["offOrigin"]) - np.array(cfg["sVoxel"]) / 2 + d / 2)
    assert np.allclose(got[1], np.array(cfg["offOrigin"]) + np.array(cfg["sVoxel"]) / 2 - d / 2)


# ---- CLI refusals -----------------------------------------------------------------------------------------------------

def _scene(tmp_path):
    from r2_gaussian_b200 import scene
    from r2_gaussian_b200.dataset import write_blender
    rng = np.random.RandomState(0)
    sc = scene.cone_beam_scanner(16, 8)
    sc.update({"filter": None, "accuracy": 0.5, "totalAngle": 360.0, "startAngle": 0.0, "noise": False})
    frames = [(0.4 * k, rng.rand(16, 16).astype(np.float32)) for k in range(3)]
    src = str(tmp_path / "scene")
    write_blender(src, sc, frames[:2], frames[2:], rng.rand(8, 8, 8).astype(np.float32))
    return src


def _refused(capsys, argv, needle):
    with pytest.raises(SystemExit) as e:
        extract_mesh.load_volume(extract_mesh.parse_args(argv))
    msg = str(e.value.code) + capsys.readouterr().err
    assert needle in msg, msg


def test_cli_refusals(tmp_path, capsys):
    src = _scene(tmp_path)
    out = str(tmp_path / "m.ply")
    vol = str(tmp_path / "v.npy")
    np.save(vol, np.zeros((8, 8, 9), np.float32))
    model = tmp_path / "model"
    model.mkdir()
    _refused(capsys, ["--output", out], "no volume")
    _refused(capsys, ["--output", out, "--vol", vol, "-m", str(model)], "not both")
    _refused(capsys, ["--output", out, "-s", src, "--resolution", "64"], "--resolution applies to -m")
    _refused(capsys, ["--output", out, "--vol", vol, "--iteration", "3"], "--iteration applies to -m")
    _refused(capsys, ["--output", out, "-m", str(model), "--resolution", "1"], "--resolution must be >= 2")
    for bad in ("nan", "inf", "1e39"):
        _refused(capsys, ["--output", out, "-s", src, "--level", bad], "finite")
    _refused(capsys, ["--output", out, "--vol", str(tmp_path / "missing.npy")], "does not exist")
    _refused(capsys, ["--output", str(tmp_path / "nodir" / "m.ply"), "-s", src], "does not exist")
    _refused(capsys, ["--output", out, "--vol", vol, "-s", src], "nVoxel")
    _refused(capsys, ["--output", out, "-m", str(model)], "no recorded settings")
    np.save(vol, np.zeros((8, 8), np.float32))
    _refused(capsys, ["--output", out, "--vol", vol], "3-D")


def test_cli_sources_without_a_gpu(tmp_path):
    """-s and --vol -s read the scene's grid; --vol alone is index space."""
    src = _scene(tmp_path)
    out = str(tmp_path / "m.ply")
    label, vol, cfg = extract_mesh.load_volume(extract_mesh.parse_args(["--output", out, "-s", src]))
    assert label == "scene" and vol.shape == (8, 8, 8) and cfg["nVoxel"] == [8, 8, 8]
    p = str(tmp_path / "v.npy")
    np.save(p, np.ones((8, 8, 8), np.float64))
    label, vol, cfg2 = extract_mesh.load_volume(extract_mesh.parse_args(["--output", out, "--vol", p, "-s", src]))
    assert label == "vol" and cfg2["sVoxel"] == cfg["sVoxel"]
    label, vol, cfg3 = extract_mesh.load_volume(extract_mesh.parse_args(["--output", out, "--vol", p]))
    assert label == "vol" and cfg3 is None


def test_python_refuses_before_any_gpu_work():
    with pytest.raises(ValueError, match="finite"):
        mesh.marching_cubes(np.zeros((2, 2, 2), np.float32), float("nan"))
    with pytest.raises(ValueError, match="finite"):
        mesh.marching_cubes(np.zeros((2, 2, 2), np.float32), 1e39)
    with pytest.raises(ValueError, match=r"\[nx, ny, nz\]"):
        mesh.marching_cubes(np.zeros((2, 2), np.float32), 0.5)


# ---- C ABI argument checks ---------------------------------------------------------------------------------------------

def test_abi_refuses_bad_arguments_before_any_cuda_call():
    lib = _lib.load()
    fake = C.c_void_p(256)           # never dereferenced: every call below is refused first
    big = (2048, 1024, 1024)         # 2^31 samples
    assert lib.r2x_marching_cubes_scratch_bytes(*big) == 0
    assert lib.r2x_marching_cubes_scratch_bytes(0, 4, 4) == 0
    assert lib.r2x_marching_cubes_scratch_bytes(1291, 1291, 1291) == 0     # 2^31 + 4.4e6 samples
    assert lib.r2x_marching_cubes_scratch_bytes(1290, 1290, 1290) > 0      # 2^31 - 7.9e5
    n = lib.r2x_marching_cubes_scratch_bytes(1024, 1024, 1024)
    assert 0.625 * 1024 ** 3 <= n <= 0.626 * 1024 ** 3
    rc = lib.r2x_marching_cubes_count(None, *big, fake, 0.5, fake, fake, 1 << 40)
    assert rc == 1 and b"2^31" in lib.r2x_last_error()
    rc = lib.r2x_marching_cubes_emit(None, *big, fake, 0.5, 10, 10, fake, fake, fake, 1 << 40)
    assert rc == 1 and b"2^31" in lib.r2x_last_error()
    rc = lib.r2x_marching_cubes_count(None, 4, 4, 0, fake, 0.5, fake, fake, 1 << 20)
    assert rc == 1 and b"bad grid" in lib.r2x_last_error()
    rc = lib.r2x_marching_cubes_count(None, 4, 4, 4, None, 0.5, fake, fake, 1 << 20)
    assert rc == 1 and b"NULL" in lib.r2x_last_error()
    rc = lib.r2x_marching_cubes_count(None, 4, 4, 4, fake, 0.5, None, fake, 1 << 20)
    assert rc == 1 and b"NULL" in lib.r2x_last_error()
    rc = lib.r2x_marching_cubes_count(None, 4, 4, 4, fake, float("inf"), fake, fake, 1 << 20)
    assert rc == 1 and b"level" in lib.r2x_last_error()
    rc = lib.r2x_marching_cubes_count(None, 4, 4, 4, fake, 0.5, fake, fake, 16)
    assert rc == 1 and b"scratch" in lib.r2x_last_error()
    rc = lib.r2x_marching_cubes_emit(None, 4, 4, 4, fake, 0.5, 1, 0, None, None, fake, 1 << 20)
    assert rc == 1 and b"NULL" in lib.r2x_last_error()
    rc = lib.r2x_marching_cubes_emit(None, 4, 4, 4, fake, 0.5, -1, 0, fake, fake, fake, 1 << 20)
    assert rc == 1 and b"negative" in lib.r2x_last_error()
    # totals past int32 indices: R2X_ERR_OVERFLOW, nothing written
    rc = lib.r2x_marching_cubes_emit(None, 4, 4, 4, fake, 0.5, 2 ** 31, 5, fake, fake, fake, 1 << 20)
    assert rc == 3 and b"int32" in lib.r2x_last_error()
    rc = lib.r2x_marching_cubes_emit(None, 4, 4, 4, fake, 0.5, 5, 2 ** 31, fake, fake, fake, 1 << 20)
    assert rc == 3
    assert lib.r2x_marching_cubes_table(None, None) == 1
