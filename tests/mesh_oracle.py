"""An independent numpy statement of the marching cubes in include/r2x.h (r2x_marching_cubes_*).

`case_table()` derives the table from the face rule with geometry (face cycles oriented by cross products, loops
walked on edge pairs), separately from the C++ generator in csrc/r2x_mesh.cu.  `marching_cubes(vol, level)` is a
vectorised float32 extractor that returns the same ordered arrays as the GPU: vertices by owning sample, then axis;
triangles by cube, then table order; float32 vertex arithmetic without FMA, so the vertices agree bit for bit.

Mesh checks used by the tests: `directed_edge_defects` (a closed, consistently oriented mesh has every directed edge
once and its reverse once), `euler_characteristic`, `area` and `signed_volume`.
"""
from __future__ import annotations

import numpy as np

CORNERS = np.array([[b & 1, (b >> 1) & 1, (b >> 2) & 1] for b in range(8)])
# axis-major edge numbering: (lower corner, upper corner), lower corners ascending within an axis
EDGES = [(b, b | (1 << a)) for a in range(3) for b in range(8) if not (b >> a) & 1]
EDGE_AXIS = np.array([a for a in range(3) for _ in range(4)])
EDGE_LOWER = np.array([lo for lo, _ in EDGES])
_EDGE_OF = {frozenset(e): i for i, e in enumerate(EDGES)}
MAX_TRI = 5


def _faces():
    """The six faces as corner 4-cycles, counter-clockwise seen from outside the cube."""
    out = []
    for a in range(3):
        for side in (0, 1):
            corners = [b for b in range(8) if ((b >> a) & 1) == side]
            centre = CORNERS[corners].mean(axis=0)
            # order around the face centre by angle, then orient by the outward normal
            u, v = [x for x in range(3) if x != a]
            ang = [np.arctan2(CORNERS[b][v] - centre[v], CORNERS[b][u] - centre[u]) for b in corners]
            cyc = [corners[i] for i in np.argsort(ang)]
            p = CORNERS[cyc].astype(float)
            normal = np.cross(p[1] - p[0], p[2] - p[1])
            outward = np.zeros(3)
            outward[a] = 1.0 if side else -1.0
            if normal @ outward < 0:
                cyc = cyc[::-1]
            out.append(cyc)
    return out


FACES = _faces()
FACE_EDGES = [frozenset(_EDGE_OF[frozenset((c[i], c[(i + 1) % 4]))] for i in range(4)) for c in FACES]


def on_one_face(e0: int, e1: int) -> bool:
    return any(e0 in f and e1 in f for f in FACE_EDGES)


def face_segments(case: int) -> list[tuple[int, int]]:
    """Directed segments (from, to) of the face rule: per face, each run of inside corners along the cycle is cut off
    by the segment from the cut edge where the cycle enters the run to the cut edge where it leaves it."""
    inside = [(case >> b) & 1 for b in range(8)]
    segs = []
    for cyc in FACES:
        # start the walk at an outside corner so that every run is contiguous in the walk
        if all(inside[b] for b in cyc):
            continue
        start = next(i for i in range(4) if not inside[cyc[i]])
        walk = cyc[start:] + cyc[:start] + [cyc[start]]
        enter = None
        for p, q in zip(walk[:-1], walk[1:]):
            e = _EDGE_OF[frozenset((p, q))]
            if not inside[p] and inside[q]:
                enter = e
            elif inside[p] and not inside[q]:
                segs.append((enter, e))
    return segs


def case_loops(case: int) -> list[list[int]]:
    """The closed loops of the face segments, in order of their smallest edge, each starting at its smallest edge."""
    nxt = {}
    for a, b in face_segments(case):
        assert a not in nxt, (case, "edge starts two segments")
        nxt[a] = b
    assert sorted(nxt) == sorted(nxt.values()), (case, "segments do not close")
    loops, seen = [], set()
    for e in sorted(nxt):
        if e in seen:
            continue
        loop = [e]
        while nxt[loop[-1]] != e:
            loop.append(nxt[loop[-1]])
        seen.update(loop)
        loops.append(loop)
    return loops


def fan(loop: list[int]) -> list[tuple[int, int, int]]:
    """Fan of a loop from the first vertex (walking from its smallest edge) whose diagonals leave every face."""
    n = len(loop)
    for r in range(n):
        rot = loop[r:] + loop[:r]
        if not any(on_one_face(rot[0], rot[i]) for i in range(2, n - 1)):
            return [(rot[0], rot[i], rot[i + 1]) for i in range(1, n - 1)]
    raise ValueError(f"no fan apex for loop {loop}")


def case_table() -> tuple[np.ndarray, np.ndarray]:
    """(ntri[256] int32, edges[256, 15] int8 with -1 padding)."""
    ntri = np.zeros(256, np.int32)
    edges = np.full((256, 3 * MAX_TRI), -1, np.int8)
    for c in range(256):
        tris = [t for loop in case_loops(c) for t in fan(loop)]
        if len(tris) > MAX_TRI:
            raise ValueError(f"case {c}: {len(tris)} triangles")
        ntri[c] = len(tris)
        edges[c, :3 * len(tris)] = np.asarray(tris, np.int8).reshape(-1)
    return ntri, edges


_TABLE = None


def table():
    global _TABLE
    if _TABLE is None:
        _TABLE = case_table()
    return _TABLE


def marching_cubes(vol, level=0.5, x_offset: int = 0) -> tuple[np.ndarray, np.ndarray]:
    """(verts float32 [V, 3], faces int32 [T, 3]) of include/r2x.h's marching cubes; float64 input is rounded to
    float32 first, level too.  With `x_offset`, `vol` is the slab of x-planes x_offset, x_offset + 1, ... of a larger
    grid: vertex x coordinates are float32(x_offset + i) + t, as the full grid's."""
    v = np.ascontiguousarray(np.asarray(vol), dtype=np.float32)
    if v.ndim != 3:
        raise ValueError("marching_cubes: expected a 3-D volume")
    lv = np.float32(level)
    nx, ny, nz = v.shape
    inside = v > lv
    cut = np.zeros((nx, ny, nz, 3), bool)
    cut[:-1, :, :, 0] = inside[:-1] != inside[1:]
    cut[:, :-1, :, 1] = inside[:, :-1] != inside[:, 1:]
    cut[:, :, :-1, 2] = inside[:, :, :-1] != inside[:, :, 1:]
    flat = cut.reshape(-1)
    vid = np.cumsum(flat, dtype=np.int64).reshape(cut.shape) - 1
    idx = np.nonzero(flat)[0]
    s, a = idx // 3, idx % 3
    i, j, k = s // (ny * nz), (s // nz) % ny, s % nz
    p0 = np.stack([i, j, k], axis=1)
    p1 = p0.copy()
    p1[np.arange(len(a)), a] += 1
    x0 = v[i, j, k]
    x1 = v[p1[:, 0], p1[:, 1], p1[:, 2]]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        t = (lv - x0) / (x1 - x0)
    verts = (p0 + np.array([x_offset, 0, 0], np.int64)).astype(np.float32)
    rows = np.arange(len(a))
    verts[rows, a] = verts[rows, a] + t
    if min(nx, ny, nz) < 2:
        return verts, np.zeros((0, 3), np.int32)
    ins = inside.astype(np.int32)
    case = np.zeros((nx - 1, ny - 1, nz - 1), np.int32)
    for b, (dx, dy, dz) in enumerate(CORNERS):
        case |= ins[dx:nx - 1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz] << b
    ntri, edges = table()
    n = ntri[case].reshape(-1)
    cube = np.repeat(np.arange(n.size), n)
    if cube.size == 0:
        return verts, np.zeros((0, 3), np.int32)
    first = np.cumsum(n) - n
    m = np.arange(cube.size) - np.repeat(first, n)
    ci, cj, ck = np.unravel_index(cube, case.shape)
    cs = case[ci, cj, ck]
    faces = np.empty((cube.size, 3), np.int64)
    for col in range(3):
        e = edges[cs, 3 * m + col].astype(np.int64)
        lo = CORNERS[EDGE_LOWER[e]]
        faces[:, col] = vid[ci + lo[:, 0], cj + lo[:, 1], ck + lo[:, 2], EDGE_AXIS[e]]
    return verts, faces.astype(np.int32)


# ---- mesh checks ------------------------------------------------------------------------------------------------------

def directed_edge_defects(faces) -> int:
    """Directed edges that do not appear exactly once with their reverse exactly once (0 for a closed, consistently
    oriented, edge-manifold mesh)."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(f) == 0:
        return 0
    p = np.concatenate([f[:, 0], f[:, 1], f[:, 2]])
    q = np.concatenate([f[:, 1], f[:, 2], f[:, 0]])
    n = int(f.max()) + 1
    key, count = np.unique(p * n + q, return_counts=True)
    rev = q * n + p
    pos = np.searchsorted(key, rev)
    found = (pos < len(key)) & (key[np.minimum(pos, len(key) - 1)] == rev)
    rev_count = np.where(found, count[np.minimum(pos, len(key) - 1)], 0)
    own = count[np.searchsorted(key, p * n + q)]
    return int(np.count_nonzero((own != 1) | (rev_count != 1)))


def euler_characteristic(verts, faces) -> int:
    f = np.asarray(faces, np.int64)
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
    n_edges = len(np.unique(e, axis=0))
    n_verts = len(np.unique(f)) if len(f) else 0
    return n_verts - n_edges + len(f)


def area(verts, faces) -> float:
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    return float(0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1).sum())


def signed_volume(verts, faces) -> float:
    """Sum of v0 . (v1 x v2) / 6: the enclosed volume of a closed mesh wound counter-clockwise seen from outside."""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)
