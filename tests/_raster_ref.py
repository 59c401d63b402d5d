"""Numpy restatement of the mesh rasterizer (nm_raster.cu, DESIGN 4.13): projection, culling, snapping, exact coverage with the
top-left rule, perspective-correct weights, the (depth, face) key, and the resolve with vertex colours or the 4.12 atlas, in
fp32 in the kernel's order (int64 / float64 where the kernel uses them).  `top_left` and `perspective` switch off the two rules
the tests show are needed."""
import numpy as np

import _texture_ref as T

f32 = np.float32
MAX_SCREEN = f32(2.0 ** 20)
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def project(verts, pose, H, W, focal, z_near):
    """Per vertex: (z, X, Y) fp32 and whether the vertex culls its faces."""
    v = np.asarray(verts, f32).reshape(-1, 3)
    P = np.asarray(pose, f32).reshape(3, 4)
    R, t = P[:, :3], P[:, 3]
    focal, z_near = f32(focal), f32(z_near)
    half_w, half_h = f32(W * 0.5), f32(H * 0.5)
    with np.errstate(all="ignore"):
        d = v - t
        p = [(d[:, 0] * R[0, j] + d[:, 1] * R[1, j]) + d[:, 2] * R[2, j] for j in range(3)]
        z = -p[2]
        X = half_w + focal * (p[0] / z)
        Y = half_h - focal * (p[1] / z)
        cull = ~(z > z_near) | ~np.isfinite(z) | ~np.isfinite(X) | ~np.isfinite(Y) | (np.abs(X) > MAX_SCREEN) | \
            (np.abs(Y) > MAX_SCREEN)
    return z.astype(f32), X.astype(f32), Y.astype(f32), cull


def setup(verts, faces, pose, H, W, focal, z_near):
    """Per face: snapped corners xs, ys (F,3) int64, depths z (F,3), culled (F,), and the clipped box of pixel samples
    c0, c1, r0, r1 (empty where c0 > c1 or r0 > r1; culled and zero-area faces get an empty box)."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    z, X, Y, vcull = project(verts, pose, H, W, focal, z_near)
    culled = vcull[f].any(1)
    with np.errstate(all="ignore"):
        xs = np.where(culled[:, None], 0, np.rint(X[f] * f32(256))).astype(np.int64)
        ys = np.where(culled[:, None], 0, np.rint(Y[f] * f32(256))).astype(np.int64)
    area = (xs[:, 1] - xs[:, 0]) * (ys[:, 2] - ys[:, 0]) - (ys[:, 1] - ys[:, 0]) * (xs[:, 2] - xs[:, 0])
    c0 = np.maximum(-((-xs.min(1)) >> 8), 0)
    c1 = np.minimum(xs.max(1) >> 8, W - 1)
    r0 = np.maximum(-((-ys.min(1)) >> 8), 0)
    r1 = np.minimum(ys.max(1) >> 8, H - 1)
    empty = culled | (area == 0)
    c0, r0 = np.where(empty, 1, c0), np.where(empty, 1, r0)
    c1, r1 = np.where(empty, 0, c1), np.where(empty, 0, r1)
    return dict(xs=xs, ys=ys, z=z[f], culled=culled, c0=c0, c1=c1, r0=r0, r1=r1)


def edges(S, fi, c, r, top_left=True):
    """(covered, E (n,3) int64, A (n,)) of samples (c, r) of faces fi."""
    xs, ys = S["xs"][fi], S["ys"][fi]
    px, py = np.asarray(c, np.int64) * 256, np.asarray(r, np.int64) * 256
    E, dx, dy = [], [], []
    for k in range(3):
        a, b = (k + 1) % 3, (k + 2) % 3
        ddx, ddy = xs[:, b] - xs[:, a], ys[:, b] - ys[:, a]
        E.append(ddx * (py - ys[:, a]) - ddy * (px - xs[:, a]))
        dx.append(ddx)
        dy.append(ddy)
    E, dx, dy = np.stack(E, 1), np.stack(dx, 1), np.stack(dy, 1)
    A = E.sum(1)
    s = np.where(A < 0, -1, 1)
    E, dx, dy, A = E * s[:, None], dx * s[:, None], dy * s[:, None], A * s
    tl = (dy > 0) | ((dy == 0) & (dx > 0)) if top_left else np.zeros(E.shape, bool)
    covered = ((E > 0) | ((E == 0) & tl)).all(1)
    return covered, E, A


def weights(S, fi, E, A, perspective=True):
    """(w (n,3), z_pix (n,)) fp32 of covered samples."""
    with np.errstate(all="ignore"):
        l = (E.astype(np.float64) / A.astype(np.float64)[:, None]).astype(f32)
        zk = S["z"][fi]
        a = l / zk if perspective else l * f32(1)
        s = (a[:, 0] + a[:, 1]) + a[:, 2]
        w = a / s[:, None]
        if not perspective:                          # affine weights, depth interpolated linearly
            return w.astype(f32), ((l[:, 0] * zk[:, 0] + l[:, 1] * zk[:, 1]) + l[:, 2] * zk[:, 2]).astype(f32)
        return w.astype(f32), (f32(1) / s).astype(f32)


def samples(S, face_chunk=1 << 14):
    """Yield (face, c, r) of every pixel sample inside a face's box, chunk by chunk of faces."""
    F = len(S["c0"])
    bw = np.maximum(S["c1"] - S["c0"] + 1, 0)
    bh = np.maximum(S["r1"] - S["r0"] + 1, 0)
    n = bw * bh
    for f0 in range(0, F, face_chunk):
        sl = slice(f0, min(F, f0 + face_chunk))
        cnt = n[sl]
        if cnt.sum() == 0:
            continue
        fi = np.repeat(np.arange(sl.start, sl.stop), cnt)
        start = np.repeat(np.cumsum(cnt) - cnt, cnt)
        off = np.arange(len(fi)) - start
        yield fi, S["c0"][fi] + off % bw[fi], S["r0"][fi] + off // bw[fi]


def keys(S, H, W, top_left=True, perspective=True):
    """The per-pixel (H*W,) uint64 minimum of (bits of z_pix) << 32 | face, EMPTY where no face covers."""
    out = np.full(H * W, EMPTY, np.uint64)
    for fi, c, r in samples(S):
        cov, E, A = edges(S, fi, c, r, top_left)
        fi, c, r, E, A = fi[cov], c[cov], r[cov], E[cov], A[cov]
        if not len(fi):
            continue
        _, z = weights(S, fi, E, A, perspective)
        k = (z.view(np.uint32).astype(np.uint64) << np.uint64(32)) | fi.astype(np.uint64)
        np.minimum.at(out, r * W + c, k)
    return out


def coverage_counts(S, H, W, top_left=True):
    """(H*W,) how many faces cover each sample, with no depth test."""
    out = np.zeros(H * W, np.int64)
    for fi, c, r in samples(S):
        cov, _, _ = edges(S, fi, c, r, top_left)
        np.add.at(out, (r * W + c)[cov], 1)
    return out


def texture_coords(w1, w2, N):
    """Patch coordinates (s, t) of the lookup and its taps: (i, j) (n,) int64 and the four tap weights (n,4) fp32 for taps
    (i,j), (i+1,j), (i,j+1), (i+1,j+1)."""
    w1 = np.fmin(np.fmax(np.asarray(w1, f32), f32(0)), f32(1))
    w2 = np.fmin(np.fmax(np.asarray(w2, f32), f32(0)), f32(1))
    sm = w1 + w2
    k = np.where(sm > f32(1), f32(1) / np.where(sm > 0, sm, f32(1)), f32(1))
    w1 = np.where(sm > f32(1), w1 * k, w1)
    w2 = np.where(sm > f32(1), w2 * k, w2)
    S_ = f32(N - 1)
    s = np.fmin(w1 * S_, S_)
    t = np.fmin(w2 * S_, S_ - s)
    a, b = np.floor(s), np.floor(t)
    fx, fy = s - a, t - b
    one = f32(1)
    tw = np.stack([(one - fx) * (one - fy), fx * (one - fy), (one - fx) * fy, fx * fy], 1).astype(f32)
    return s.astype(f32), t.astype(f32), a.astype(np.int64), b.astype(np.int64), tw


def texture_lookup(atlas, F, N, fi, w1, w2):
    """(n,3) fp32: the bilinear lookup of nm_raster.cu, taps of weight 0 skipped."""
    Q = T.layout(F, N)[0]
    _, _, i, j, tw = texture_coords(w1, w2, N)
    out = np.zeros((len(fi), 3), f32)
    for k in range(4):
        x, y = T.pixel(fi, i + (k & 1), j + (k >> 1), N, Q)
        ok = tw[:, k] > 0
        val = np.zeros((len(fi), 3), f32)
        val[ok] = atlas[y[ok], x[ok]]
        out = np.where(ok[:, None], out + tw[:, k:k + 1] * val, out).astype(f32)
    return out


def rasterize(verts, faces, pose, H, W, focal, *, z_near=1e-3, colors=None, atlas=None, N=0, background=(0, 0, 0),
              top_left=True, perspective=True):
    """(rgb (H,W,3), depth (H,W), face (H,W) int32, counts (covered, drawn, culled)) as nm_rasterize_mesh writes them."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    S = setup(verts, f, pose, H, W, focal, z_near)
    key = keys(S, H, W, top_left, perspective) if len(f) else np.full(H * W, EMPTY, np.uint64)
    cov = key != EMPTY
    rgb = np.tile(np.asarray(background, f32), (H * W, 1))
    depth = np.zeros(H * W, f32)
    face = np.full(H * W, -1, np.int32)
    idx = np.nonzero(cov)[0]
    if len(idx):
        fi = (key[idx] & np.uint64(0xFFFFFFFF)).astype(np.int64)
        c, r = idx % W, idx // W
        _, E, A = edges(S, fi, c, r, top_left)
        w, z = weights(S, fi, E, A, perspective)
        if atlas is not None:
            rgb[idx] = texture_lookup(np.asarray(atlas, f32), len(f), N, fi, w[:, 1], w[:, 2])
        elif colors is not None:
            col = np.asarray(colors, f32)[f[fi]]                                   # (n,3 corners,3)
            rgb[idx] = (w[:, 0:1] * col[:, 0] + w[:, 1:2] * col[:, 1]) + w[:, 2:3] * col[:, 2]
        focal = f32(focal)
        x = (c.astype(f32) - f32(W * 0.5)) / focal
        y = -(r.astype(f32) - f32(H * 0.5)) / focal
        depth[idx] = z * np.sqrt((x * x + y * y) + f32(1))
        face[idx] = fi
    culled = int(S["culled"].sum())
    counts = (int(cov.sum()), len(f) - culled, culled)
    return rgb.reshape(H, W, 3), depth.reshape(H, W), face.reshape(H, W), counts
