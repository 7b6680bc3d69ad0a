"""Scene view on the GPU: a depth-tested rasterizer for triangles, line segments and ellipsoids over the C ABI
(r2x_scene_raster, csrc/r2x_scene.cu), the glyphs of the reference's `scripts/visualize_scene.py`, and a trained
model's Gaussians as ellipsoids (the reference's `show_gaussians`).

    prims = concat(mesh_triangles(verts, faces, vol, cfg), box(cfg["offOrigin"], cfg["sVoxel"], RED),
                   camera_glyph(cam, 1.0, colour, image=cam.original_image[0]))
    rgb = render(prims, default_view(prims, 1000, 800))             # CUDA float32 [1, H, W, 3]
    write_png("scene.png", to_uint8(rgb[0]))

The model, stated in full in include/r2x.h: scene units; the volume renderer's camera record; clipping against the
near plane and a 2^20-pixel guard band; vertices snapped to 1/256 pixel and int64 edge functions with a top-left fill
rule, so coverage is exact; lines cover the pixels whose centre lies within w/2 pixels of the projected segment;
perspective-correct float64 depth rounded to float32 in a 64-bit atomicMin with the primitive id, so the nearest
primitive wins, ties go to the lower id and two calls give the same bits.  Mesh triangles get a two-sided headlight
Lambert shade from gradient vertex normals, image planes a nearest-texel lookup through a LUT.  Ellipsoids are
analytic: each pixel's ray meets the quadric in float64 (exact silhouette and depth, one record per ellipsoid), shaded
with the same headlight from the analytic normal.  There is no CPU fallback.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

from .volume_render import Camera, look_at, lut_from

FLAT, MESH, TEXTURED, LINE, ELLIPSOID = 0, 1, 2, 3, 4   # R2X_SV_FLAT, _MESH, _TEXTURED, _LINE, _ELLIPSOID
ATTR = 12                                    # R2X_SV_ATTR
MAX_SIDE = 16384                             # R2X_SV_MAX_SIDE
NEAR = 1e-3
MESH_COLOUR = (0.7, 0.7, 0.7)                # the reference's create_vol_mesh
RED, GREEN, BLUE = (1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0)
WHITE = (1.0, 1.0, 1.0)                      # open3d's background
LINE_WIDTH = 1.5
VIEW_DIRECTION = np.array([1.0, 1.0, 1.0]) / math.sqrt(3.0)


@dataclass
class Primitives:
    """Device tensors: pos float64 [n, 3, 3], meta int32 [n, 2] (kind, texture index), attr float32 [n, 12] (as
    include/r2x.h lays them out) and textures float32 [n_tex, th, tw] or None."""
    pos: object
    meta: object
    attr: object
    textures: object = None

    def __len__(self) -> int:
        return int(self.pos.shape[0])


def _device(device):
    import torch
    return torch.device(device if device is not None else "cuda")


def _make(pos, kind, attr, tex_index=None, textures=None, device=None) -> Primitives:
    import torch
    dev = _device(device)
    pos = torch.as_tensor(np.asarray(pos, np.float64).reshape(-1, 3, 3), device=dev)
    n = pos.shape[0]
    meta = torch.zeros((n, 2), dtype=torch.int32, device=dev)
    meta[:, 0] = kind
    if tex_index is not None:
        meta[:, 1] = torch.as_tensor(np.asarray(tex_index, np.int32), device=dev)
    a = torch.zeros((n, ATTR), dtype=torch.float32, device=dev)
    attr = torch.as_tensor(attr, dtype=torch.float32, device=dev)
    a[:, :attr.shape[-1]] = attr
    return Primitives(pos, meta, a, textures)


def _colour(c) -> np.ndarray:
    c = np.asarray(c, np.float64).reshape(-1)
    if c.shape != (3,) or not (np.isfinite(c).all() and c.min() >= 0 and c.max() <= 1):
        raise ValueError(f"a colour is 3 numbers in [0, 1], got {c}")
    return c


def lines(a, b, colour, width: float = LINE_WIDTH, device=None) -> Primitives:
    """Segments a[i] -> b[i] ([L, 3] each) of one colour (or [L, 3] colours) and `width` pixels."""
    a, b = np.asarray(a, np.float64).reshape(-1, 3), np.asarray(b, np.float64).reshape(-1, 3)
    if not (math.isfinite(width) and width > 0):
        raise ValueError(f"a line width is finite and > 0, got {width}")
    cols = np.asarray(colour, np.float64).reshape(-1, 3)
    cols = np.broadcast_to(np.stack([_colour(c) for c in cols]), (len(a), 3))
    pos = np.zeros((len(a), 3, 3))
    pos[:, 0], pos[:, 1] = a, b
    attr = np.concatenate([cols, np.full((len(a), 1), width)], 1)
    return _make(pos, LINE, attr, device=device)


def box(center, extent, colour, width: float = LINE_WIDTH, device=None) -> Primitives:
    """The 12 edges of the axis-aligned box of `center` and side lengths `extent`."""
    c, e = np.asarray(center, np.float64), np.asarray(extent, np.float64)
    corners = c + (np.array([[(i >> 0) & 1, (i >> 1) & 1, (i >> 2) & 1] for i in range(8)]) - 0.5) * e
    edges = [(i, i | 1 << ax) for i in range(8) for ax in range(3) if not i >> ax & 1]
    return lines(corners[[i for i, _ in edges]], corners[[j for _, j in edges]], colour, width, device)


def axes(origin, size: float, rotation=None, width: float = LINE_WIDTH, device=None) -> Primitives:
    """A coordinate frame: x red, y green, z blue, each `size` long from `origin` along the columns of `rotation`
    (default the world axes).  open3d draws arrows; these are lines."""
    o = np.asarray(origin, np.float64)
    R = np.eye(3) if rotation is None else np.asarray(rotation, np.float64)
    return lines(np.repeat(o[None], 3, 0), o + size * R.T, np.array([RED, GREEN, BLUE]), width, device)


def _view_geometry(view):
    """(c2w [4, 4], P [4, 4] in math convention, parallel) of a dataset camera, float64."""
    wvt = view.world_view_transform.detach().double().cpu().numpy()
    full = view.full_proj_transform.detach().double().cpu().numpy().reshape(4, 4)
    c2w = np.linalg.inv(wvt.T)
    P = (np.linalg.inv(wvt) @ full).T
    return c2w, P, int(view.mode) == 0


def image_plane(view, depth: float) -> np.ndarray:
    """The world corners [4, 3] (top-left, top-right, bottom-right, bottom-left of the image) of the camera's image
    rectangle at camera depth `depth`: ndc (+-1, +-1) through the camera's projection, so a principal point moved by
    --use_offDetector or a learned detector offset moves the rectangle.  Camera y points down the image."""
    c2w, P, _ = _view_geometry(view)
    out = []
    for nx, ny in ((-1, -1), (1, -1), (1, 1), (-1, 1)):
        w = P[3, 2] * depth + P[3, 3]
        x = (nx * w - P[0, 2] * depth - P[0, 3]) / P[0, 0]
        y = (ny * w - P[1, 2] * depth - P[1, 3]) / P[1, 1]
        out.append(c2w[:3, :3] @ np.array([x, y, depth]) + c2w[:3, 3])
    return np.array(out)


def camera_centre(view) -> np.ndarray:
    return _view_geometry(view)[0][:3, 3]


def camera_glyph(view, scale: float, colour, image=None, plane_depth: float | None = None,
                 width: float = LINE_WIDTH, device=None) -> Primitives:
    """The glyph of a dataset camera (`world_view_transform`, `full_proj_transform`, `mode`): its frustum in `colour`
    with the image rectangle at depth `plane_depth` (default `scale`, the reference's) -- a pyramid from the source,
    or for a parallel beam the detector rectangle at the source plane and at that depth joined by four parallel
    edges --, `image` (a [H, W] projection, normalised by its maximum) as a texture on the rectangle, and a coordinate
    frame of size scale / 12 at the camera centre."""
    depth = float(scale if plane_depth is None else plane_depth)
    if not (math.isfinite(depth) and depth > 0):
        raise ValueError(f"camera_glyph: the image plane depth must be finite and > 0, got {depth}")
    c2w, _, parallel = _view_geometry(view)
    far = image_plane(view, depth)
    ring = [0, 1, 2, 3]
    a, b = [far[i] for i in ring], [far[(i + 1) % 4] for i in ring]
    if parallel:
        near = far - depth * c2w[:3, 2]
        a += [near[i] for i in ring] + [near[i] for i in ring]
        b += [near[(i + 1) % 4] for i in ring] + [far[i] for i in ring]
    else:
        a += [c2w[:3, 3]] * 4
        b += [far[i] for i in ring]
    parts = [lines(a, b, colour, width, device)]
    if image is not None:
        import torch
        img = torch.as_tensor(image, device=_device(device)).detach().to(torch.float32)
        if img.dim() != 2:
            raise ValueError(f"camera_glyph: expected a [H, W] image, got shape {tuple(img.shape)}")
        m = img.max()
        tex = img / m if float(m) > 0 else img
        uv = np.array([[0.0, 0.0], [1.0, 0.0], [1.0, 1.0], [0.0, 1.0]])
        tris = [(0, 1, 2), (2, 3, 0)]
        pos = np.stack([far[list(t)] for t in tris])
        attr = np.zeros((2, 9))
        attr[:, 3:9] = np.stack([uv[list(t)].reshape(-1) for t in tris])
        parts.append(_make(pos, TEXTURED, attr, tex_index=[0, 0], textures=tex[None].contiguous(), device=device))
    parts.append(axes(c2w[:3, 3], scale / 12.0, c2w[:3, :3], width, device))
    return concat(*parts)


def vertex_normals(verts, vol):
    """Unit normals [V, 3] (float32, index space, pointing from high to low values) of marching-cubes vertices: the
    central-difference gradient of the samples (one-sided at the border, numpy's `gradient`) interpolated trilinearly
    at the vertex, which lies on a grid edge, so this is the interpolation along that edge -- the normals skimage's
    marching_cubes returns.  Element-wise torch operations and gathers, no atomics: deterministic on any device."""
    import torch
    v = torch.as_tensor(vol).to(torch.float32)
    p = torch.as_tensor(verts, device=v.device).to(torch.float64)
    grads = torch.stack(torch.gradient(v), -1)                    # [nx, ny, nz, 3]
    n = torch.tensor(v.shape, device=v.device)
    i0 = torch.minimum(torch.floor(p).long().clamp(min=0), (n - 2).clamp(min=0))
    w = (p - i0).clamp(0, 1)
    g = torch.zeros((p.shape[0], 3), dtype=torch.float64, device=v.device)
    for corner in range(8):
        o = torch.tensor([corner & 1, corner >> 1 & 1, corner >> 2 & 1], device=v.device)
        idx = torch.minimum(i0 + o, n - 1)
        wt = torch.prod(torch.where(o.bool(), w, 1 - w), 1)
        g += wt[:, None] * grads[idx[:, 0], idx[:, 1], idx[:, 2]].to(torch.float64)
    nrm = torch.linalg.vector_norm(g, dim=1, keepdim=True)
    return torch.where(nrm > 0, -g / nrm.clamp(min=1e-300), torch.zeros_like(g)).to(torch.float32)


def mesh_triangles(verts, faces, vol, scanner_cfg: dict | None = None, colour=MESH_COLOUR, device=None) -> Primitives:
    """Shaded triangles of a marching-cubes mesh (verts in index space, faces [T, 3]) of `vol`: in scene units
    (`mesh.to_scene`) with a scanner, else in index space, with `vertex_normals` (scaled by 1 / dVoxel, so they stay
    normal to the surface in scene units)."""
    import torch

    from .mesh import to_scene
    f = torch.as_tensor(faces).long()
    normals = vertex_normals(verts, vol).to(torch.float64)
    if scanner_cfg is not None:
        pos = torch.as_tensor(to_scene(verts, scanner_cfg))
        d = torch.as_tensor(np.asarray(scanner_cfg["sVoxel"], np.float64) / np.asarray(scanner_cfg["nVoxel"], np.float64))
        normals = normals / d.to(normals.device)
        normals = normals / torch.linalg.vector_norm(normals, dim=1, keepdim=True).clamp(min=1e-300)
    else:
        pos = torch.as_tensor(verts).detach().to(torch.float64)
    dev = _device(device)
    pos, f, normals = pos.to(dev), f.to(dev), normals.to(dev)
    attr = torch.zeros((f.shape[0], ATTR), dtype=torch.float32, device=dev)
    attr[:, 0:3] = torch.as_tensor(_colour(colour), dtype=torch.float32, device=dev)
    attr[:, 3:12] = normals[f].reshape(-1, 9).to(torch.float32)
    meta = torch.zeros((f.shape[0], 2), dtype=torch.int32, device=dev)
    meta[:, 0] = MESH
    return Primitives(pos[f].contiguous(), meta, attr, None)


def ellipsoids(centres, axes, quaternions, colours, device=None) -> Primitives:
    """Solid ellipsoids { c + R diag(s) v : |v| <= 1 }: centres and semi-axes [n, 3], quaternions [n, 4] in the
    model's (w, x, y, z) order (R is `gaussian_utils.build_rotation`'s; the kernel normalises them), colours [n, 3]
    or one colour.  Built on the device from tensors or arrays, with no per-ellipsoid host work."""
    import torch
    dev = _device(device)
    c = torch.as_tensor(centres, device=dev).detach().to(torch.float64).reshape(-1, 3)
    n = c.shape[0]
    s = torch.as_tensor(axes, device=dev).detach().to(torch.float64).reshape(n, 3)
    q = torch.as_tensor(quaternions, device=dev).detach().to(torch.float32).reshape(n, 4)
    col = torch.as_tensor(colours, device=dev).detach().to(torch.float32)
    pos = torch.zeros((n, 3, 3), dtype=torch.float64, device=dev)
    pos[:, 0], pos[:, 1] = c, s
    meta = torch.zeros((n, 2), dtype=torch.int32, device=dev)
    meta[:, 0] = ELLIPSOID
    attr = torch.zeros((n, ATTR), dtype=torch.float32, device=dev)
    attr[:, 0:3] = col.reshape(-1, 3).expand(n, 3)
    attr[:, 3:7] = q
    return Primitives(pos, meta, attr, None)


SORT_GAUSSIANS = ("no", "density", "scale")


def gaussian_ellipsoids(gaussians, n_gaussian: int | None = None, sort_gaussians: str = "no"):
    """(Primitives, indices): the 1-sigma ellipsoids of a model's Gaussians by the rules of the reference's
    `show_gaussians`, on the model's device.  Keeps the Gaussians whose density (`get_density[:, 0]`) is not 0; sorts
    them by density ("density") or by the mean activated scale ((s0 + s1) + s2) / 3 in float32 ("scale"), largest
    first, or keeps the model's order ("no"); draws the first `n_gaussian` (all if None or more than there are).  The
    sort is stable, so ties keep the model's order; the reference's `argsort()[::-1]` may order exact ties differently.
    Each is gray at t = density * (0.95 / max density) in float32 (the maximum over every kept Gaussian, as the
    reference's vertex colour) and oriented by `get_rotation` in the model's (w, x, y, z) order -- the orientation the
    rasterizer and voxelizer use.  `indices` (int64, on the device) are the drawn Gaussians' rows in the model."""
    import torch
    if sort_gaussians not in SORT_GAUSSIANS:
        raise ValueError(f"sort_gaussians must be one of {SORT_GAUSSIANS}, got {sort_gaussians!r}")
    if n_gaussian is not None and int(n_gaussian) < 1:
        raise ValueError(f"n_gaussian must be >= 1 or None, got {n_gaussian}")
    with torch.no_grad():
        dens = gaussians.get_density[:, 0].detach()
        idx = torch.nonzero(dens != 0).squeeze(1)
        if idx.numel() == 0:
            raise ValueError("gaussian_ellipsoids: every Gaussian has density 0; nothing to draw")
        kept = dens[idx]
        scale = torch.tensor(0.95, dtype=torch.float32, device=dens.device) / kept.max().to(torch.float32)
        if sort_gaussians != "no":
            if sort_gaussians == "density":
                key = kept
            else:
                s = gaussians.get_scaling.detach()[idx].to(torch.float32)
                key = ((s[:, 0] + s[:, 1]) + s[:, 2]) / 3.0
            idx = idx[torch.sort(key, descending=True, stable=True).indices]
        if n_gaussian is not None:
            idx = idx[:int(n_gaussian)]
        grey = (dens[idx].to(torch.float32) * scale)[:, None].expand(-1, 3)
        prims = ellipsoids(gaussians.get_xyz.detach()[idx], gaussians.get_scaling.detach()[idx],
                           gaussians.get_rotation.detach()[idx], grey, device=dens.device)
    return prims, idx


def concat(*parts) -> Primitives:
    """One primitive list, in the order given (ties in depth go to the earlier part); textures are stacked and their
    indices renumbered.  Textures of one list share a size."""
    import torch
    parts = [p for p in parts if p is not None and len(p)]
    if not parts:
        raise ValueError("concat: nothing to draw")
    metas, texs, n_tex = [], [], 0
    for p in parts:
        m = p.meta.clone()
        if p.textures is not None:
            m[:, 1] += n_tex
            texs.append(p.textures)
            n_tex += p.textures.shape[0]
        metas.append(m)
    if texs and any(t.shape[1:] != texs[0].shape[1:] for t in texs):
        raise ValueError("concat: the textures of one list must share a size")
    return Primitives(torch.cat([p.pos for p in parts]), torch.cat(metas), torch.cat([p.attr for p in parts]),
                      torch.cat(texs) if texs else None)


def points(prims: Primitives) -> np.ndarray:
    """Every point a primitive uses (two per segment, three per triangle), float64 [M, 3]; an ellipsoid gives the two
    opposite corners of its axis-aligned bounding box (half sides sqrt(sum_j (R_ij s_j)^2))."""
    import torch

    from .gaussian_utils import build_rotation
    kind = prims.meta[:, 0]
    ell = kind == ELLIPSOID
    pos = prims.pos.detach()
    parts = [pos[kind == LINE, :2].reshape(-1, 3), pos[(kind != LINE) & ~ell].reshape(-1, 3)]
    if bool(ell.any()):
        e = pos[ell]
        R = build_rotation(prims.attr[ell, 3:7].detach().to(torch.float64))
        half = torch.sqrt(((R * e[:, 1, None, :]) ** 2).sum(2))
        parts += [e[:, 0] - half, e[:, 0] + half]
    return torch.cat(parts).cpu().numpy()


def default_view(prims: Primitives, width: int, height: int, view_angle: float = 30.0) -> Camera:
    """Looks at the centre of the bounding sphere of everything drawn (the centre of its bounding box, radius the
    largest distance from it) from direction (1, 1, 1), view-up +z, at the distance where the sphere spans the
    vertical view angle: radius / sin(view_angle / 2)."""
    p = points(prims)
    centre = (p.min(0) + p.max(0)) / 2
    radius = float(np.sqrt(((p - centre) ** 2).sum(1)).max()) or 1.0
    dist = radius / math.sin(math.radians(view_angle) / 2)
    return look_at(centre + dist * VIEW_DIRECTION, centre, (0.0, 0.0, 1.0), width, height, view_angle)


def scan_orbit(camera: Camera, n: int) -> list:
    """n cameras turned by 360 k / n degrees about the scan's rotation axis (+z) through the focal point; the
    position and the view-up turn together."""
    n = int(n)
    if n < 1:
        raise ValueError(f"an orbit needs at least 1 frame, got {n}")
    F = np.asarray(camera.focal_point, np.float64)
    v, up = np.asarray(camera.position, np.float64) - F, np.asarray(camera.view_up, np.float64)
    out = []
    for i in range(n):
        th = 2.0 * math.pi * i / n
        c, s = math.cos(th), math.sin(th)
        R = np.array([[c, -s, 0.0], [s, c, 0.0], [0.0, 0.0, 1.0]])
        out.append(look_at(F + R @ v, F, R @ up, camera.width, camera.height, camera.view_angle,
                           camera.parallel_scale))
    return out


def _check(prims: Primitives):
    import torch
    n = len(prims)
    if n < 1:
        raise ValueError("render: nothing to draw")
    if prims.pos.dtype != torch.float64 or tuple(prims.pos.shape) != (n, 3, 3):
        raise ValueError("render: pos must be float64 [n, 3, 3]")
    if prims.meta.dtype != torch.int32 or tuple(prims.meta.shape) != (n, 2):
        raise ValueError("render: meta must be int32 [n, 2]")
    if prims.attr.dtype != torch.float32 or tuple(prims.attr.shape) != (n, ATTR):
        raise ValueError(f"render: attr must be float32 [n, {ATTR}]")
    kind = prims.meta[:, 0]
    if not bool(((kind >= FLAT) & (kind <= ELLIPSOID)).all()):
        raise ValueError("render: a primitive kind is not 0 (flat), 1 (mesh), 2 (textured), 3 (line) or 4 (ellipsoid)")
    if not bool(torch.isfinite(prims.pos).all()) or not bool(torch.isfinite(prims.attr).all()):
        raise ValueError("render: positions and attributes must be finite")
    ell = kind == ELLIPSOID
    if bool(ell.any()):
        if not bool((prims.pos[ell, 1] > 0).all()):
            raise ValueError("render: every ellipsoid semi-axis must be finite and > 0")
        if not bool((prims.attr[ell, 3:7] != 0).any(1).all()):
            raise ValueError("render: an ellipsoid's quaternion is all zero")
    w = prims.attr[:, 3][kind == LINE]
    if w.numel() and not bool((w > 0).all()):
        raise ValueError("render: every line width must be > 0")
    t = prims.meta[:, 1][kind == TEXTURED]
    n_tex = 0 if prims.textures is None else int(prims.textures.shape[0])
    if t.numel() and not bool(((t >= 0) & (t < n_tex)).all()):
        raise ValueError(f"render: a textured triangle names a texture outside 0 .. {n_tex - 1}")


def render(prims: Primitives, cameras, background=WHITE, supersample: int = 1, lut=None, near: float = NEAR,
           return_keys: bool = False):
    """RGB frames, CUDA float32 [N, H, W, 3], of `prims` seen by `cameras` (one Camera or a list sharing the image
    size and projection), in one launch.  `lut` (anything `volume_render.lut_from` takes, default gray) colours the
    textures.  `supersample` k renders k H x k W pixels (the same cameras, pitch / k) and returns the mean of each
    k x k block, summed row by row in float32 then divided by k^2.  `return_keys` also returns the depth-id keys
    (int64 holding the uint64 bits) of the rendered (supersampled) pixels."""
    import torch

    from ._lib import check, load

    cams = [cameras] if isinstance(cameras, Camera) else list(cameras)
    if not cams or not all(isinstance(c, Camera) for c in cams):
        raise ValueError("render: cameras must be a Camera or a non-empty list of them")
    W, H, par = cams[0].width, cams[0].height, cams[0].parallel
    if any((c.width, c.height, c.parallel) != (W, H, par) for c in cams):
        raise ValueError("render: every camera of one call needs the same image size and projection")
    k = int(supersample)
    if k < 1 or max(W, H) * k > MAX_SIDE:
        raise ValueError(f"render: supersample must be >= 1 with k W and k H <= {MAX_SIDE}, got {supersample}")
    if k > 1:
        cams = [look_at(c.position, c.focal_point, c.view_up, W * k, H * k, c.view_angle, c.parallel_scale)
                for c in cams]
    bg = np.asarray(background, np.float32).reshape(-1)
    if bg.shape != (3,) or not np.isfinite(bg).all():
        raise ValueError(f"render: background must be 3 finite numbers, got {background}")
    near = float(near)
    if not (math.isfinite(near) and near > 0):
        raise ValueError(f"render: near must be finite and > 0, got {near}")
    table = lut_from("gray" if lut is None else lut)
    _check(prims)
    dev = prims.pos.device
    n, F, Hk, Wk = len(prims), len(cams), H * k, W * k
    lib = load()
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        rec = torch.from_numpy(np.stack([c.record() for c in cams])).to(dev)
        lut_d = torch.from_numpy(table.astype(np.float32)).to(dev)
        tex = prims.textures
        n_tex, th, tw = (0, 1, 1) if tex is None else (int(tex.shape[0]), int(tex.shape[1]), int(tex.shape[2]))
        tex = None if tex is None else tex.to(dev, torch.float32).contiguous()
        nbytes = int(lib.r2x_scene_raster_scratch_bytes(n, F))
        scratch = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=dev)
        keys = torch.empty((F, Hk, Wk), dtype=torch.int64, device=dev)
        rgb = torch.empty((F, Hk, Wk, 3), dtype=torch.float32, device=dev)
        check(lib.r2x_scene_raster(stream, n, prims.pos.contiguous().data_ptr(), prims.meta.contiguous().data_ptr(),
                                   prims.attr.contiguous().data_ptr(), n_tex, th, tw,
                                   None if tex is None else tex.data_ptr(), lut_d.data_ptr(), len(table), F, Hk, Wk,
                                   rec.data_ptr(), int(par), near, bg.ctypes.data, keys.data_ptr(), rgb.data_ptr(),
                                   scratch.data_ptr(), nbytes), "r2x_scene_raster")
    if k > 1:
        acc = torch.zeros((F, H, W, 3), dtype=torch.float32, device=dev)
        for i in range(k):
            for j in range(k):
                acc += rgb[:, i::k, j::k]
        rgb = acc / float(k * k)
    return (rgb, keys) if return_keys else rgb
