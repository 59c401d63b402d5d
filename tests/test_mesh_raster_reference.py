"""The mesh rasterizer's semantics (DESIGN 4.13) without a device: the numpy restatement (_raster_ref) against an independent
float64 ray caster (Moller-Trumbore on get_ray_bundle's rays) on meshes of the C marching-cubes oracle and hand-built ones;
watertight coverage of a grid with mixed diagonals and windings, which fails without the top-left rule; the lower face id
on ties; bilinear taps that stay in the face's patch or ring (4.12); argument rejections of nm_rasterize_mesh without a
device."""
import ctypes as C

import numpy as np
import pytest
import torch

import _raster_ref as R
import _texture_ref as T
from oracle import nerf_oracle as O
from test_mesh_decimate_reference import mesh as analytic_mesh

f32 = np.float32
H = W = 96
FOCAL = float(0.5 * W / np.tan(0.5 * 0.6911112))


def pose(theta, phi=-30.0, radius=4.0):
    return O.pose_spherical(theta, phi, radius).numpy()[:3, :4].astype(f32)


def camera64(P):
    P = np.asarray(P, np.float64)
    return P[:, :3], P[:, 3]


def on_grid(v, P, focal=FOCAL):
    """The vertices moved along their camera ray so that they project onto the 1/256-pixel grid: the snap then moves nothing,
    and the rasterizer and a float64 ray caster can agree to fp32 precision."""
    Rm, t = camera64(P)
    p = (np.asarray(v, np.float64) - t) @ Rm
    z = -p[:, 2]
    X = np.round((W * 0.5 + focal * p[:, 0] / z) * 256) / 256
    Y = np.round((H * 0.5 - focal * p[:, 1] / z) * 256) / 256
    q = np.stack([(X - W * 0.5) * z / focal, -(Y - H * 0.5) * z / focal, -z], 1)
    return (q @ Rm.T + t).astype(f32)


def raycast(v, f, P, z_near, colors, focal=FOCAL):
    """float64 brute force: per pixel the nearest hit (t > 0) among the faces with every corner beyond z_near, both windings.
    Returns (face (H*W,), t, second-nearest t, colour (H*W,3) by the hit's barycentrics)."""
    Rm, t0 = camera64(P)
    o, d = O.get_ray_bundle(H, W, focal, torch.from_numpy(np.asarray(P, np.float64)))
    o, d = o.numpy(), d.numpy().reshape(-1, 3)
    v = np.asarray(v, np.float64)
    z = -((v - t0) @ Rm)[:, 2]
    keep = np.nonzero((z[f] > z_near).all(1))[0]
    A, B, Cc = v[f[keep, 0]], v[f[keep, 1]], v[f[keep, 2]]
    e1, e2 = B - A, Cc - A
    best = np.full(H * W, -1, np.int64)
    tb, t2 = np.full(H * W, np.inf), np.full(H * W, np.inf)
    uv = np.zeros((H * W, 2))
    for p0 in range(0, H * W, 512):
        dd = d[p0:p0 + 512, None, :]
        pv = np.cross(dd, e2[None])
        det = (e1[None] * pv).sum(-1)
        with np.errstate(all="ignore"):
            inv = 1.0 / det
            tv = (o - A)[None]
            u = (tv * pv).sum(-1) * inv
            qv = np.cross(tv, e1[None])
            w = (dd * qv).sum(-1) * inv
            t = (e2[None] * qv).sum(-1) * inv
        hit = (det != 0) & (u >= 0) & (w >= 0) & (u + w <= 1) & (t > 0)
        t = np.where(hit, t, np.inf)
        order = np.argsort(t, 1)[:, :2]
        rows = np.arange(len(t))
        k = order[:, 0]
        tb[p0:p0 + 512] = t[rows, k]
        t2[p0:p0 + 512] = t[rows, order[:, 1]] if t.shape[1] > 1 else np.inf
        best[p0:p0 + 512] = np.where(np.isfinite(t[rows, k]), keep[k], -1)
        uv[p0:p0 + 512] = np.stack([u[rows, k], w[rows, k]], 1)
    col = np.asarray(colors, np.float64)
    fb = np.maximum(best, 0)
    rgb = (1 - uv.sum(1))[:, None] * col[f[fb, 0]] + uv[:, 0:1] * col[f[fb, 1]] + uv[:, 1:2] * col[f[fb, 2]]
    return best, tb, t2, rgb


def near_edges(v, f, P, z_near, tol=2.0 / 256, focal=FOCAL):
    """(H*W,) whether the pixel sample lies within tol pixels of a projected edge of a face that is not culled."""
    Rm, t0 = camera64(P)
    p = (np.asarray(v, np.float64) - t0) @ Rm
    z = -p[:, 2]
    X, Y = W * 0.5 + focal * p[:, 0] / z, H * 0.5 - focal * p[:, 1] / z
    keep = (z[f] > z_near).all(1)
    segs = np.concatenate([f[keep][:, [0, 1]], f[keep][:, [1, 2]], f[keep][:, [2, 0]]])
    a = np.stack([X[segs[:, 0]], Y[segs[:, 0]]], 1)
    b = np.stack([X[segs[:, 1]], Y[segs[:, 1]]], 1)
    c, r = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    s = np.stack([c.reshape(-1), r.reshape(-1)], 1)
    out = np.zeros(H * W, bool)
    ab = b - a
    L2 = np.maximum((ab * ab).sum(1), 1e-300)
    for p0 in range(0, H * W, 256):
        q = s[p0:p0 + 256, None, :] - a[None]
        h = np.clip((q * ab[None]).sum(-1) / L2[None], 0, 1)
        dist = np.linalg.norm(q - h[..., None] * ab[None], axis=-1)
        out[p0:p0 + 256] = (dist < tol).any(1)
    return out


def _world(name, scale=0.05):
    v, _, f = analytic_mesh(name)
    v = (v - v.mean(0)) * f32(scale)
    return v.astype(f32), np.asarray(f, np.int64)


def _quads():
    """Two overlapping squares, the second in front of and tilted against the first, and two triangles that pass through
    each other."""
    v = np.array([[-.6, -.6, 0], [.4, -.6, 0], [.4, .4, 0], [-.6, .4, 0],
                  [-.2, -.3, .3], [.7, -.3, .1], [.7, .6, .2], [-.2, .6, .4],
                  [-.9, .5, -.3], [-.1, .9, .4], [-.5, -.2, .2],
                  [-.8, .8, .35], [-.2, .3, -.4], [-.3, .9, -.1]], f32)
    f = np.array([[0, 1, 2], [0, 2, 3], [4, 5, 6], [4, 6, 7], [8, 9, 10], [11, 12, 13]], np.int64)
    return v, f


CASES = {
    "sphere": (lambda: _world("sphere"), pose(30.0), 1e-3),
    "torus": (lambda: _world("torus", 0.03), pose(200.0, -60.0), 1e-3),
    "quads": (_quads, pose(75.0, -20.0, 3.0), 1e-3),
    # the camera 0.75 from the centre of a sphere of radius 0.5: the faces nearer than 0.35 are culled
    "close_up": (lambda: _world("sphere"), pose(10.0, -10.0, 0.75), 0.35),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_matches_a_float64_ray_caster(name):
    make, P, z_near = CASES[name]
    v, f = make()
    v = on_grid(v, P)
    col = np.random.default_rng(5).random((len(v), 3)).astype(f32)
    rgb, depth, face, counts = R.rasterize(v, f, P, H, W, FOCAL, z_near=z_near, colors=col)
    best, t, t2, ref_rgb = raycast(v, f, P, z_near, col)
    if name == "close_up":
        assert counts[2] > 0, counts
    assert counts[1] + counts[2] == len(f) and counts[0] == int((face >= 0).sum())
    with np.errstate(invalid="ignore"):                 # inf - inf where a ray hits nothing
        ok = ~near_edges(v, f, P, z_near) & ~(np.abs(t2 - t) <= 1e-5 * t)
    face, depth, rgb = face.reshape(-1), depth.reshape(-1), rgb.reshape(-1, 3)
    assert ok.sum() > 0.3 * H * W, ok.sum()
    assert np.array_equal(face[ok], best[ok]), int((face[ok] != best[ok]).sum())
    hit = ok & (best >= 0)
    assert hit.sum() > 300
    assert np.allclose(depth[hit], t[hit], rtol=1e-5, atol=0), np.abs(depth[hit] / t[hit] - 1).max()
    assert np.abs(rgb[hit] - ref_rgb[hit]).max() < 1e-5
    assert (depth[~(face >= 0)] == 0).all()


def test_ray_caster_rejects_an_affine_rasterizer():
    """Without the perspective correction the depth (and the colours) drift from the ray caster's."""
    make, P, z_near = CASES["quads"]
    v, f = make()
    v = on_grid(v, P)
    col = np.random.default_rng(5).random((len(v), 3)).astype(f32)
    _, depth, face, _ = R.rasterize(v, f, P, H, W, FOCAL, z_near=z_near, colors=col, perspective=False)
    best, t, t2, _ = raycast(v, f, P, z_near, col)
    ok = (~near_edges(v, f, P, z_near) & (best >= 0) & (face.reshape(-1) == best))
    assert not np.allclose(depth.reshape(-1)[ok], t[ok], rtol=1e-5, atol=0)


def grid_mesh(G=64, cell=3, seed=0):
    """A G x G grid of cells of `cell` pixels, two triangles per cell with a random diagonal and random windings, corners on
    pixel samples (x/z exact: z is 1 or 2), in front of the identity camera."""
    rng = np.random.default_rng(seed)
    n = G + 1
    Wd = G * cell + 8
    ii, jj = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    X = 4 + jj.reshape(-1) * cell
    Y = 4 + ii.reshape(-1) * cell
    z = rng.choice([1.0, 2.0], n * n)
    v = np.stack([(X - Wd * 0.5) * z, -(Y - Wd * 0.5) * z, -z], 1).astype(f32)
    faces = []
    for i in range(G):
        for j in range(G):
            a, b, c, d = i * n + j, i * n + j + 1, (i + 1) * n + j + 1, (i + 1) * n + j
            tris = [[a, b, c], [a, c, d]] if rng.random() < 0.5 else [[a, b, d], [b, c, d]]
            for tr in tris:
                faces.append(tr[::-1] if rng.random() < 0.3 else tr)
    P = np.concatenate([np.eye(3, dtype=f32), np.zeros((3, 1), f32)], 1)
    return v, np.asarray(faces, np.int64), P, Wd


@pytest.mark.parametrize("seed", [0, 1])
def test_grid_is_covered_exactly_once(seed):
    v, f, P, Wd = grid_mesh(seed=seed)
    S = R.setup(v, f, P, Wd, Wd, 1.0, 1e-3)
    assert not S["culled"].any()
    cnt = R.coverage_counts(S, Wd, Wd).reshape(Wd, Wd)
    inner = cnt[5:Wd - 5, 5:Wd - 5]                   # the samples strictly inside the grid's border
    assert (inner == 1).all(), np.unique(inner, return_counts=True)
    bad = R.coverage_counts(S, Wd, Wd, top_left=False).reshape(Wd, Wd)[5:Wd - 5, 5:Wd - 5]
    assert (bad != 1).any()
    # the depth-tested image is the same: every interior sample has its one face
    _, _, face, counts = R.rasterize(v, f, P, Wd, Wd, 1.0, colors=np.zeros((len(v), 3), f32))
    assert (face[5:Wd - 5, 5:Wd - 5] >= 0).all() and counts == (int((cnt > 0).sum()), len(f), 0)


def test_ties_go_to_the_lower_face():
    v, f = _world("sphere")
    P = pose(30.0)
    g = np.concatenate([f, f[::-1]])               # every face twice; face k and face 2F-1-k are the same triangle
    _, depth, face, _ = R.rasterize(v, g, P, H, W, FOCAL, colors=np.zeros((len(v), 3), f32))
    _, depth1, face1, _ = R.rasterize(v, f, P, H, W, FOCAL, colors=np.zeros((len(v), 3), f32))
    assert np.array_equal(face, face1) and np.array_equal(depth.view(np.int32), depth1.view(np.int32))


@pytest.mark.parametrize("N", [2, 3, 8, 64])
def test_texture_taps_stay_in_the_patch_and_ring(N):
    v, f = _world("torus", 0.06)
    P = pose(120.0, -45.0)
    F = len(f)
    S = R.setup(v, f, P, H, W, FOCAL, 1e-3)
    key = R.keys(S, H, W)
    idx = np.nonzero(key != R.EMPTY)[0]
    fi = (key[idx] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    _, E, A = R.edges(S, fi, idx % W, idx // W)
    w, _ = R.weights(S, fi, E, A)
    rng = np.random.default_rng(N)
    # and adversarial weights: at the corners and edges, one ulp past them, outside [0, 1]
    e = np.float32(1e-7)
    w1 = np.concatenate([w[:, 1], rng.random(4000).astype(f32), [0, 1, 1 - e, e, 1 + e, -e, 0.5 + e, 0.5, 2, -1, 1]]).astype(f32)
    w2 = np.concatenate([w[:, 2], rng.random(4000).astype(f32), [0, 0, e, 1 - e, 0, 0, 0.5, 0.5 + e, 2, 0.5, 1e-30]]).astype(f32)
    ff = np.concatenate([fi, rng.integers(0, F, 4000 + 11)])
    s, t, i, j, tw = R.texture_coords(w1, w2, N)
    assert len(fi) > 1000
    for k in range(4):
        ti, tj = i + (k & 1), j + (k >> 1)
        nz = tw[:, k] > 0
        assert ((ti[nz] >= 0) & (tj[nz] >= 0) & (ti[nz] + tj[nz] <= N)).all(), (N, k)
    # the lookup point is continuous_pixel's, its taps bilinear_taps' (where the weights need no rescaling)
    Q = T.layout(F, N)[0]
    plain = (w1 >= 0) & (w2 >= 0) & (w1 + w2 <= 1)
    x, y = T.continuous_pixel(ff[plain], w1[plain], w2[plain], N, Q)
    cx, cy = T.continuous_pixel(ff[plain], s[plain] / f32(max(N - 1, 1)), t[plain] / f32(max(N - 1, 1)), N, Q)
    assert np.abs(x - cx).max() < 1e-4 and np.abs(y - cy).max() < 1e-4
    tx, ty, bw = T.bilinear_taps(x, y)
    for k in range(4):
        nz = bw[:, k] > 1e-3
        px, py = T.pixel(ff[plain][nz], 0, 0, N, Q)
        C_ = N + 2
        lx, ly = tx[nz, k] - (px - px % C_), ty[nz, k] - (py - py % C_)
        h1 = ff[plain][nz] % 2 == 1
        pi, pj = np.where(h1, C_ - 1 - lx, lx), np.where(h1, C_ - 1 - ly, ly)
        assert ((pi >= 0) & (pj >= 0) & (pi + pj <= N)).all()
    # a whole image: the restatement's lookups read only the atlas values of the faces they resolve to
    atlas = np.zeros((T.layout(F, N)[3], T.layout(F, N)[2], 3), f32)
    ft, it, jt, _, xt, yt = T.texels(F, N)
    atlas[yt, xt] = (ft % 7)[:, None] / 7.0
    rf, _, _, rx, ry = T.ring(F, N)
    atlas[ry, rx] = (rf % 7)[:, None] / 7.0
    rgb, _, face, _ = R.rasterize(v, f, P, H, W, FOCAL, atlas=atlas, N=N)
    m = face >= 0
    assert np.abs(rgb[m] - ((face[m] % 7) / 7.0)[:, None]).max() < 1e-5


def _lib():
    from nerfmeshes_b200 import _lib as L
    return L.load()


def test_rasterize_rejects_bad_arguments_without_a_device():
    lib = _lib()
    P = C.c_void_p(16)                       # never dereferenced: every call below fails its argument checks first
    cnt = (C.c_int64 * 3)()
    pose_ = (C.c_float * 12)(*np.eye(3, 4, dtype=f32).reshape(-1))
    bg = (C.c_float * 3)()
    err = lambda: lib.nm_last_error().decode()

    def rejects(text, h=None, v=P, V=10, f=P, F=10, pose=pose_, H=8, W=8, focal=10.0, z_near=1e-3, mode=0, rgb_in=P, atlas=P,
                N=4, bg=bg, rgb=P, depth=P, face=P, counts=cnt):
        rc = lib.nm_rasterize_mesh(h, v, V, f, F, pose, H, W, focal, z_near, mode, rgb_in, atlas, N, bg, rgb, depth, face, counts,
                                   None)
        assert rc != 0 and text in err(), (text, rc, err())

    rejects("negative size", V=-1)
    rejects("negative size", F=-1)
    rejects("2^31", V=2 ** 31)
    rejects("2^31", F=2 ** 31)
    for kw in (dict(pose=None), dict(bg=None), dict(counts=None)):
        rejects("null pose, background or counts", **kw)
    for kw in (dict(H=0), dict(W=0), dict(H=16385), dict(W=16385), dict(H=-3)):
        rejects("outside [1, 16384]", **kw)
    for x in (0.0, -1.0, float("inf"), float("nan")):
        rejects("focal length", focal=x)
        rejects("z_near", z_near=x)
    rejects("mode 2", mode=2)
    rejects("mode -1", mode=-1)
    rejects("N = 1 outside", mode=1, N=1)
    rejects("N = 65 outside", mode=1, N=65)
    rejects("largest N that fits", mode=1, F=200000, N=64)
    rejects("null vertex pointer", v=None)
    rejects("null face pointer", f=None)
    rejects("null vertex colour pointer", rgb_in=None)
    rejects("null atlas pointer", mode=1, atlas=None)
    rejects("null handle")
    rejects("null handle", N=0)                                   # N is a texture argument: mode 0 ignores it
    rejects("null handle", rgb_in=None, rgb=None)                 # no colour output, no colour source needed
    rejects("null handle", mode=1, atlas=None, rgb=None, N=8)
    rejects("null handle", v=None, f=None, V=0, F=0, rgb_in=None, atlas=None)
    rejects("null handle", rgb=None, depth=None, face=None)
