"""Numpy restatement of the texture bake (nm_texture.cu, DESIGN 4.12): the atlas layout, every texel's query in fp32 in the
kernel's order, the scatter, the ring, the quantisation and the corner uvs, plus the textured OBJ text and a PNG reader."""
import math
import struct
import zlib

import numpy as np

f32 = np.float32
MIN_N, MAX_N, MAX_SIDE = 2, 64, 16384


def layout(F, N):
    """(Q, rows, W, H); ValueError where nm_texture_layout rejects."""
    if not MIN_N <= N <= MAX_N:
        raise ValueError(f"texels per triangle leg N = {N} outside [{MIN_N}, {MAX_N}]")
    if not 0 <= F < 2 ** 31:
        raise ValueError(f"face count {F} outside [0, 2^31)")
    C, P = N + 2, (F + 1) // 2
    Q = math.isqrt(P)
    Q += Q * Q < P
    rows = -(-P // Q) if Q else 0
    W, H = Q * C, rows * C
    if W > MAX_SIDE or H > MAX_SIDE:
        raise ValueError(f"a {W} x {H} atlas exceeds {MAX_SIDE} texels per side")
    return Q, rows, W, H


def largest_n(F):
    """The largest N whose atlas fits, or None."""
    ok = [N for N in range(MIN_N, MAX_N + 1) if _fits(F, N)]
    return max(ok) if ok else None


def _fits(F, N):
    try:
        layout(F, N)
        return True
    except ValueError:
        return False


def patch(N):
    """(i, j) of the K = N(N+1)/2 texels of one face in texel order (row j, then i) and the corner slot (0, 1, 2 or -1)."""
    ij = np.array([(i, j) for j in range(N) for i in range(N - j)], np.int64)
    i, j = ij[:, 0], ij[:, 1]
    corner = np.full(len(ij), -1)
    corner[(i == 0) & (j == 0)] = 0
    corner[(j == 0) & (i == N - 1)] = 1
    corner[(i == 0) & (j == N - 1)] = 2
    return i, j, corner


def pixel(f, i, j, N, Q):
    """Atlas pixel (x, y) of texel (i, j) of face f (arrays broadcast)."""
    C = N + 2
    f = np.asarray(f, np.int64)
    c = f // 2
    x0, y0 = (c % Q) * C, (c // Q) * C
    h1 = (f % 2) == 1
    return x0 + np.where(h1, C - 1 - i, i), y0 + np.where(h1, C - 1 - j, j)


def texels(F, N, f0=0, f1=None):
    """Per texel of faces [f0, f1): face, i, j, corner slot, pixel x, y."""
    f1 = F if f1 is None else f1
    Q = layout(F, N)[0]
    i, j, corner = patch(N)
    K = len(i)
    f = np.repeat(np.arange(f0, f1, dtype=np.int64), K)
    i, j, corner = np.tile(i, f1 - f0), np.tile(j, f1 - f0), np.tile(corner, f1 - f0)
    x, y = pixel(f, i, j, N, Q)
    return f, i, j, corner, x, y


def queries(v, n, faces, N, mode, c, f0=0, f1=None):
    """(a, d, xy) of nm_debug_texture_rays: a = the ray origins p - c*d (mode 0) or the points p (mode 1), d = -n."""
    v, n, faces = np.asarray(v, f32), np.asarray(n, f32), np.asarray(faces, np.int64)
    f, i, j, corner, x, y = texels(len(faces), N, f0, f1)
    idx = faces[f]                                            # (T, 3)
    w1 = i.astype(f32) / f32(N - 1)
    w2 = j.astype(f32) / f32(N - 1)
    w0 = (f32(1) - w1) - w2
    V0, V1, V2 = v[idx[:, 0]], v[idx[:, 1]], v[idx[:, 2]]
    N0, N1, N2 = n[idx[:, 0]], n[idx[:, 1]], n[idx[:, 2]]
    p = (w0[:, None] * V0 + w1[:, None] * V1) + w2[:, None] * V2
    m = (w0[:, None] * N0 + w1[:, None] * N1) + w2[:, None] * N2
    with np.errstate(all="ignore"):
        ln = np.sqrt((m[:, 0] * m[:, 0] + m[:, 1] * m[:, 1]) + m[:, 2] * m[:, 2])
        ok = np.isfinite(ln) & (ln > 0)
        nn = m / np.where(ok, ln, f32(1))[:, None]
    kmax = np.where((w0 >= w1) & (w0 >= w2), 0, np.where(w1 >= w2, 1, 2))
    nn = np.where(ok[:, None], nn, n[idx[np.arange(len(f)), kmax]])
    cs = corner >= 0
    vc = idx[np.arange(len(f)), np.maximum(corner, 0)]
    p = np.where(cs[:, None], v[vc], p)
    nn = np.where(cs[:, None], n[vc], nn)
    d = -nn
    a = p - f32(c) * d if mode == 0 else p
    return a.astype(f32), d.astype(f32), np.stack([x, y], 1).astype(np.int32)


def ring(F, N):
    """Per ring texel: face, (i, j) with i + j = N in half 0's coordinates, pixel x, y."""
    Q = layout(F, N)[0]
    f = np.repeat(np.arange(F, dtype=np.int64), N + 1)
    i = np.tile(np.arange(N + 1), F)
    j = N - i
    x, y = pixel(f, i, j, N, Q)
    return f, i, j, x, y


def assemble(F, N, rgb, xy):
    """The float atlas from every texel's colour rgb (T,3) at its pixel xy (T,2): scatter, rings, zeros elsewhere."""
    Q, _, W, H = layout(F, N)
    atlas = np.zeros((H, W, 3), f32)
    atlas[xy[:, 1], xy[:, 0]] = np.asarray(rgb, f32)
    f, i, j, x, y = ring(F, N)
    ax, ay = pixel(f, np.maximum(i - 1, 0), j, N, Q)          # clamped where the neighbour does not exist (unused there)
    bx, by = pixel(f, i, np.maximum(j - 1, 0), N, Q)
    a, b = atlas[ay, ax], atlas[by, bx]
    both = ((i > 0) & (j > 0))[:, None]
    atlas[y, x] = np.where(both, (a + b) * f32(0.5), np.where((i > 0)[:, None], a, b))
    return atlas


def quantise(atlas):
    return np.floor(np.fmin(np.fmax(np.asarray(atlas, f32), f32(0)), f32(1)) * f32(255) + f32(0.5)).astype(np.uint8)


def uv(F, N):
    """(F,3,2): the centre of each corner texel, u = (x + 0.5)/W, v = 1 - (y + 0.5)/H."""
    Q, _, W, H = layout(F, N)
    f = np.repeat(np.arange(F), 3)
    k = np.tile(np.arange(3), F)
    x, y = pixel(f, np.where(k == 1, N - 1, 0), np.where(k == 2, N - 1, 0), N, Q)
    u = (x.astype(f32) + f32(0.5)) / f32(W)
    w = f32(1) - (y.astype(f32) + f32(0.5)) / f32(H)
    return np.stack([u, w], 1).astype(f32).reshape(F, 3, 2)


def first_corner(faces, V):
    """Per vertex: the lowest 3f + k that references it, or -1."""
    flat = np.asarray(faces, np.int64).reshape(-1)
    out = np.full(V, -1, np.int64)
    order = np.arange(len(flat))[::-1]
    out[flat[order]] = order                                  # the last write (lowest index) wins
    return out


def continuous_pixel(f, w1, w2, N, Q):
    """Atlas coordinates (x, y) in texel-centre units of the surface point with barycentrics (1-w1-w2, w1, w2) of face f:
    a bilinear lookup there reads the texel grid the bake wrote."""
    C = N + 2
    f = np.asarray(f, np.int64)
    c = f // 2
    x0, y0 = (c % Q) * C, (c // Q) * C
    s, t = np.asarray(w1, np.float64) * (N - 1), np.asarray(w2, np.float64) * (N - 1)
    h1 = (f % 2) == 1
    return x0 + np.where(h1, C - 1 - s, s), y0 + np.where(h1, C - 1 - t, t)


def bilinear_taps(x, y):
    """The up to four texels (x, y) integer arrays (n,4) a bilinear lookup reads with nonzero weight, and the weights."""
    x0, y0 = np.floor(x).astype(np.int64), np.floor(y).astype(np.int64)
    fx, fy = x - x0, y - y0
    tx = np.stack([x0, x0 + 1, x0, x0 + 1], 1)
    ty = np.stack([y0, y0, y0 + 1, y0 + 1], 1)
    w = np.stack([(1 - fx) * (1 - fy), fx * (1 - fy), (1 - fx) * fy, fx * fy], 1)
    return tx, ty, w


def obj_text(v, f, d, n, uvs, mtl_name):
    """The textured OBJ, formatted in python like mesh._export_obj_python."""
    r = lambda a: [[repr(x) for x in row] for row in np.asarray(a, f32).astype(np.float64).tolist()]
    out = [f"mtllib {mtl_name}\n"]
    vr, dr = r(v), r(d) if len(d) else []
    for k, row in enumerate(vr):
        out.append("v " + " ".join(row) + (" " + " ".join(dr[k]) if len(dr) > k else "") + "\n")
    out.extend("vt " + " ".join(row) + "\n" for row in r(np.asarray(uvs, f32).reshape(-1, 2)))
    out.extend("vn " + " ".join(row) + "\n" for row in r(n))
    out.append("usemtl texture\n")
    for fi, tri in enumerate(np.asarray(f).tolist()):
        out.append("f" + "".join(f" {a + 1}/{3 * fi + k + 1}/{a + 1}" for k, a in enumerate(tri)) + "\n")
    return "".join(out)


def read_png(path):
    """(H,W,3) uint8 of an 8-bit RGB PNG whose scanlines all use filter 0 (what mesh.write_png writes)."""
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat, ihdr = 8, b"", None
    while pos < len(data):
        ln, tag = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + ln]
        assert struct.unpack(">I", data[pos + 8 + ln:pos + 12 + ln])[0] == zlib.crc32(tag + body) & 0xFFFFFFFF, tag
        if tag == b"IHDR":
            ihdr = struct.unpack(">IIBBBBB", body)
        elif tag == b"IDAT":
            idat += body
        pos += 12 + ln
    W, H, depth, ctype, _, _, interlace = ihdr
    assert (depth, ctype, interlace) == (8, 2, 0)
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(H, 1 + 3 * W)
    assert (raw[:, 0] == 0).all()
    return raw[:, 1:].reshape(H, W, 3).copy()
