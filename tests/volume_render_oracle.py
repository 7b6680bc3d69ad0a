"""Float64 numpy statement of the volume rendering model of include/r2x.h (r2x_volume_render), vectorised over rays.

The ray set-up and the sample points repeat the kernel's float64 operations in the kernel's order (the kernel uses
explicit round-to-nearest operations, no FMA), so every ray meets the box, gets its sample count and samples the
same points as on the GPU.  From there on the oracle stays in float64 where the kernel is float32: the interpolation
weights, the trilinear blend, the transfer function, the LUT and the compositing.  The stop rule is the kernel's:
after the first sample that leaves T < 2^-16.
"""
import numpy as np

T_STOP = 2.0 ** -16


def ray_setup(rec, H, W, parallel, shape, pixels=None):
    """(o [R, 3], d [R, 3], s_in [R], s_out [R], meets [R]) for the H * W rays of one float32 camera record,
    row-major from the top-left pixel, or for the flat pixel indices `pixels` (y W + x) only."""
    rec = np.asarray(rec, np.float32).astype(np.float64)
    P, f, r, u, p = rec[0:3], rec[3:6], rec[6:9], rec[9:12], rec[12]
    if pixels is None:
        y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    else:
        px = np.asarray(pixels, np.int64)
        y, x = (px // W).astype(np.float64), (px % W).astype(np.float64)
    a = (((x + 0.5) - 0.5 * W) * p).reshape(-1, 1)
    b = (((0.5 * H - y) - 0.5) * p).reshape(-1, 1)
    if parallel:
        o = (P + a * r) + b * u
        d = np.broadcast_to(f, o.shape).copy()
    else:
        d = (f + a * r) + b * u
        norm = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
        d = d / norm[:, None]
        o = np.broadcast_to(P, d.shape).copy()
    hi = np.asarray(shape, np.float64) - 1
    s0 = np.zeros(len(o))
    s1 = np.full(len(o), np.inf)
    inside = np.ones(len(o), bool)
    with np.errstate(divide="ignore", invalid="ignore"):
        for c in range(3):
            zero = d[:, c] == 0
            inside &= ~zero | ((o[:, c] >= 0) & (o[:, c] <= hi[c]))
            ta, tb = (-o[:, c]) / d[:, c], (hi[c] - o[:, c]) / d[:, c]
            s0 = np.where(zero, s0, np.maximum(s0, np.minimum(ta, tb)))
            s1 = np.where(zero, s1, np.minimum(s1, np.maximum(ta, tb)))
    meets = inside & (s1 >= s0) & np.isfinite(s1)
    return o, d, s0, s1, meets


def rec_step(step):
    """A float32 argument of the kernel, as float64."""
    return float(np.float32(step))


def sample_counts(s0, s1, meets, step):
    """floor((s_out - s_in) / step) + 1 for rays that meet the box, 0 otherwise."""
    n = np.zeros(len(s0), np.int64)
    n[meets] = np.floor((s1[meets] - s0[meets]) / rec_step(step)).astype(np.int64) + 1
    return n


def trilinear(vol, pts):
    """Values of the trilinear field at points already clamped into the box, cell i0 = min(floor(p), n - 2)."""
    hi = np.asarray(vol.shape, np.float64) - 1
    i0 = np.minimum(np.floor(pts), hi - 1)
    w = pts - i0
    i = i0.astype(np.int64)
    v = vol.astype(np.float64)
    out = 0.0
    for dx in (0, 1):
        for dy in (0, 1):
            for dz in (0, 1):
                wt = ((w[:, 0] if dx else 1 - w[:, 0]) * (w[:, 1] if dy else 1 - w[:, 1])
                      * (w[:, 2] if dz else 1 - w[:, 2]))
                out = out + wt * v[i[:, 0] + dx, i[:, 1] + dy, i[:, 2] + dz]
    return out


def transfer(v, c0, c1):
    c0, c1 = float(np.float32(c0)), float(np.float32(c1))
    return np.clip((v - c0) / (c1 - c0), 0.0, 1.0)


def lut_colour(lut, t):
    lut = np.asarray(lut, np.float32).astype(np.float64)
    K = len(lut)
    if K == 1:
        return np.broadcast_to(lut[0], (len(t), 3)).copy()
    pos = t * (K - 1)
    j = np.minimum(np.floor(pos), K - 2).astype(np.int64)
    w = (pos - j)[:, None]
    return (1 - w) * lut[j] + w * lut[j + 1]


def render_frame(vol, rec, H, W, parallel, mode="composite", clim=(0.0, 1.0), lut=((0, 0, 0), (1, 1, 1)), step=0.5,
                 unit=None, background=(0.0, 0.0, 0.0), pixels=None):
    """float64 [H, W, 4] RGBA of one camera record; with `pixels` (flat indices y W + x) float64 [len(pixels), 4] of
    those pixels only, so that a subset of a 10^6-row image stays cheap."""
    vol = np.asarray(vol, np.float32)
    shape = vol.shape
    n_ = np.asarray(shape, np.float64)
    if unit is None:
        unit = float(np.linalg.norm(n_ - 1) / (n_.mean() - 1))
    step64, expo = rec_step(step), rec_step(step) / rec_step(unit)
    bg = np.asarray(background, np.float32).astype(np.float64)
    o, d, s0, s1, meets = ray_setup(rec, H, W, parallel, shape, pixels)
    n = sample_counts(s0, s1, meets, step)
    R = len(o)
    hi = n_ - 1
    C = np.zeros((R, 3))
    T = np.ones(R)
    m = np.full(R, -np.inf)
    active = meets.copy()
    k = 0
    while True:
        active &= k < n
        idx = np.nonzero(active)[0]
        if len(idx) == 0:
            break
        s = s0[idx] + k * step64
        pts = np.clip(o[idx] + s[:, None] * d[idx], 0.0, hi)
        v = trilinear(vol, pts)
        if mode == "mip":
            m[idx] = np.maximum(m[idx], v)
        else:
            t = transfer(v, *clim)
            al = 1.0 - (1.0 - t) ** expo
            col = lut_colour(lut, t)
            C[idx] += (T[idx] * al)[:, None] * col
            T[idx] *= 1.0 - al
            active[idx[T[idx] < T_STOP]] = False
        k += 1
    out = np.zeros((R, 4))
    out[:, :3] = bg
    if mode == "mip":
        out[meets, :3] = lut_colour(lut, transfer(m[meets], *clim))
        out[meets, 3] = 1.0
    else:
        out[meets, :3] = C[meets] + T[meets, None] * bg
        out[meets, 3] = 1.0 - T[meets]
    return out if pixels is not None else out.reshape(H, W, 4)


def render(vol, cameras, **kw):
    """float64 [N, H, W, 4] for a list of `volume_render.Camera`s."""
    return np.stack([render_frame(vol, c.record(), c.height, c.width, c.parallel, **kw) for c in cameras])


# ---- test helpers ------------------------------------------------------------------------------------------------------

def axis_view(shape, axis, sign, margin=0):
    """A parallel camera looking along sign * e_axis with unit pixels through voxel centres: every pixel's ray runs
    along a grid line of the other two axes (or, with `margin` extra pixels on each side, misses the box), so with
    step 1 the samples sit exactly on voxels.  Returns (camera, lateral [H, W, 2] int indices of the two other axes
    (-1 when the ray misses), the two axes)."""
    from r2_gaussian_b200 import volume_render as vr
    n = np.asarray(shape, np.int64)
    up, side = (axis + 1) % 3, (axis + 2) % 3
    H, W = int(n[up]) + 2 * margin, int(n[side]) + 2 * margin
    centre = (n - 1) / 2.0
    pos = centre.copy()
    pos[axis] -= sign * (n[axis] + 5)
    U = np.zeros(3)
    U[up] = 1.0
    cam = vr.look_at(pos, centre, U, W, H, parallel_scale=H / 2.0)
    o, _, _, _, meets = ray_setup(cam.record(), H, W, True, shape)
    lat = np.full((H * W, 2), -1, np.int64)
    lat[meets] = np.rint(o[meets][:, [up, side]]).astype(np.int64)
    assert np.array_equal(o[meets][:, [up, side]], lat[meets])
    return cam, lat.reshape(H, W, 2), (up, side)


def read_png(path):
    """uint8 [H, W, 3] of an 8-bit RGB PNG with filter 0 on every row; every chunk's CRC is checked."""
    import struct
    import zlib
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, chunks = 8, []
    while pos < len(data):
        (length,) = struct.unpack(">I", data[pos:pos + 4])
        kind, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + length]
        (crc,) = struct.unpack(">I", data[pos + 8 + length:pos + 12 + length])
        assert crc == zlib.crc32(kind + body) & 0xFFFFFFFF, kind
        chunks.append((kind, body))
        pos += 12 + length
    assert [k for k, _ in chunks][0] == b"IHDR" and chunks[-1] == (b"IEND", b"")
    w, h, depth, colour, comp, filt, interlace = struct.unpack(">IIBBBBB", chunks[0][1])
    assert (depth, colour, comp, filt, interlace) == (8, 2, 0, 0, 0)
    raw = np.frombuffer(zlib.decompress(b"".join(b for k, b in chunks if k == b"IDAT")), np.uint8).reshape(h, 1 + 3 * w)
    assert (raw[:, 0] == 0).all()
    return raw[:, 1:].reshape(h, w, 3).copy()
