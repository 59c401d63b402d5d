"""The texture bake's layout and outputs without a device (DESIGN 4.12): the numpy restatement (_texture_ref) gives every face
texels of its own and a ring no triangle or other ring touches, exact corner queries and uvs on corner texel centres, and a
bilinear lookup anywhere inside a triangle reads only that face's texels and ring.  nm_texture_layout equals the restatement,
rejections included; nm_bake_texture rejects bad arguments before it needs a device; the textured OBJ writer matches a python
formatter byte for byte and reduces to nm_export_obj's file; the PNG round-trips through zlib."""
import ctypes as C

import numpy as np
import pytest

import _texture_ref as T
from test_mesh_decimate_reference import mesh as analytic_mesh

CASES = [(1, 2), (2, 2), (3, 3), (7, 4), (10, 8), (33, 5), (101, 17), (250, 64)]


def owner_map(F, N):
    """Per atlas pixel: the face whose triangle owns it (>= 0), the face whose ring it is (-2 - f), or -1."""
    _, _, W, H = T.layout(F, N)
    own = np.full((H, W), -1, np.int64)
    f, _, _, _, x, y = T.texels(F, N)
    assert (own[y, x] == -1).all()
    np.add.at(own, (y, x), 1 + f)                              # -1 + 1 + f: a pixel hit twice would not equal f
    rf, _, _, rx, ry = T.ring(F, N)
    assert (own[ry, rx] == -1).all(), "a ring texel lies in a triangle"
    np.add.at(own, (ry, rx), -1 - rf)
    return own


@pytest.mark.parametrize("F,N", CASES)
def test_texels_and_rings_are_disjoint(F, N):
    Q, rows, W, H = T.layout(F, N)
    assert Q * Q >= (F + 1) // 2 and (Q - 1) ** 2 < (F + 1) // 2 and rows * Q >= (F + 1) // 2
    f, i, j, _, x, y = T.texels(F, N)
    K = N * (N + 1) // 2
    assert len(f) == F * K and (i + j <= N - 1).all()
    assert ((0 <= x) & (x < W) & (0 <= y) & (y < H)).all()
    px = y * W + x
    assert len(np.unique(px)) == len(px), "two texels share a pixel"
    rf, _, _, rx, ry = T.ring(F, N)
    rp = ry * W + rx
    assert len(np.unique(rp)) == len(rp), "two rings share a pixel"
    assert not np.isin(rp, px).any(), "a ring texel lies in a triangle"
    # texel t of face f is number f*K + j*N - j(j-1)/2 + i
    assert np.array_equal(f * K + j * N - j * (j - 1) // 2 + i, np.arange(F * K))
    # the two halves' coordinate sums: half 0 <= N - 1 and ring N; half 1 >= N + 3 and ring N + 2; nothing on N + 1
    C_ = N + 2
    cs = (x % C_) + (y % C_)
    assert (np.where(f % 2 == 0, cs <= N - 1, cs >= N + 3)).all()
    rcs = (rx % C_) + (ry % C_)
    assert (rcs == np.where(rf % 2 == 0, N, N + 2)).all()


@pytest.mark.parametrize("name", ["sphere", "torus"])
@pytest.mark.parametrize("N", [2, 3, 8])
def test_corner_queries_are_the_vertices_own(name, N):
    v, n, f = analytic_mesh(name)
    c = 0.0123
    for mode in (0, 1):
        a, d, _ = T.queries(v, n, f, N, mode, c)
        _, _, _, corner, _, _ = T.texels(len(f), N)
        k = corner >= 0
        vc = f[np.repeat(np.arange(len(f)), N * (N + 1) // 2)[k], corner[k]]
        dirs = -n[vc]
        assert np.array_equal(d[k].view(np.int32), dirs.view(np.int32))
        want = v[vc] - np.float32(c) * dirs if mode == 0 else v[vc]          # mesh_appearance's fp32 product and difference
        assert np.array_equal(a[k].view(np.int32), want.view(np.int32))
        assert np.isfinite(a).all() and np.isfinite(d).all()
        ln = np.linalg.norm(d.astype(np.float64), axis=1)
        assert np.abs(ln - 1).max() < 1e-5


def test_degenerate_normals_fall_back_to_the_heaviest_corner():
    v = np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0]])
    n = np.float32([[0, 0, 1], [0, 0, -1], [np.nan, 0, 0]])
    a, d, _ = T.queries(v, n, np.int32([[0, 1, 2]]), 5, 1, 0.0)
    i, j, corner = T.patch(5)
    w1, w2 = i / 4, j / 4
    heavy = np.where((1 - w1 - w2 >= w1) & (1 - w1 - w2 >= w2), 0, np.where(w1 >= w2, 1, 2))
    nonfinite = np.isnan(d).any(1)
    # every texel with weight on corner 2 has a NaN sum; the texels between corners 0 and 1 with equal weights cancel
    assert np.array_equal(d[~nonfinite], -n[heavy][~nonfinite])
    assert (heavy[nonfinite] == 2).all()


@pytest.mark.parametrize("F,N", CASES)
def test_uvs_are_corner_texel_centres(F, N):
    Q, _, W, H = T.layout(F, N)
    uv = T.uv(F, N).astype(np.float64)
    _, _, _, corner, x, y = T.texels(F, N)
    k = corner >= 0
    cx, cy = x[k].reshape(F, 3), y[k].reshape(F, 3)
    order = np.argsort(corner[k].reshape(F, 3), 1)
    cx, cy = np.take_along_axis(cx, order, 1), np.take_along_axis(cy, order, 1)
    assert np.abs(uv[..., 0] * W - 0.5 - cx).max() < 1e-3
    assert np.abs((1 - uv[..., 1]) * H - 0.5 - cy).max() < 1e-3


@pytest.mark.parametrize("F,N", CASES)
def test_bilinear_reads_stay_in_the_face(F, N):
    Q = T.layout(F, N)[0]
    own = owner_map(F, N)
    rng = np.random.default_rng(F * 100 + N)
    m = 64
    f = np.repeat(np.arange(F), m)
    b = rng.dirichlet((1, 1, 1), size=F * m)
    b = np.concatenate([b, np.tile([[0.5, 0.5, 0.0], [0.0, 0.5, 0.5], [0.5, 0.0, 0.5], [1 / 3, 1 / 3, 1 / 3]], (F, 1))])
    f = np.concatenate([f, np.repeat(np.arange(F), 4)])       # edge midpoints and centroids as well
    x, y = T.continuous_pixel(f, b[:, 1], b[:, 2], N, Q)
    tx, ty, w = T.bilinear_taps(x, y)
    used = w > 0
    H, W = own.shape
    assert ((tx[used] >= 0) & (tx[used] < W) & (ty[used] >= 0) & (ty[used] < H)).all()
    o = own[np.clip(ty, 0, H - 1), np.clip(tx, 0, W - 1)]
    ff = np.broadcast_to(f[:, None], o.shape)
    assert ((o == ff) | (o == -2 - ff))[used].all(), "a bilinear tap with nonzero weight left its face"


def test_assemble_ring_and_quantise():
    F, N = 5, 4
    rng = np.random.default_rng(3)
    _, _, _, _, x, y = T.texels(F, N)
    rgb = rng.uniform(-0.2, 1.2, size=(len(x), 3)).astype(np.float32)
    atlas = T.assemble(F, N, rgb, np.stack([x, y], 1))
    assert np.array_equal(atlas[y, x], rgb)
    Q = T.layout(F, N)[0]
    rf, ri, rj, rx, ry = T.ring(F, N)
    for f, i, j, px, py in zip(rf, ri, rj, rx, ry):
        nb = [atlas[yy, xx] for ok, (xx, yy) in ((i > 0, T.pixel(f, i - 1, j, N, Q)), (j > 0, T.pixel(f, i, j - 1, N, Q))) if ok]
        want = (nb[0] + nb[1]) * np.float32(0.5) if len(nb) == 2 else nb[0]
        assert np.array_equal(atlas[py, px], want)
    own = owner_map(F, N)
    assert (atlas[own == -1] == 0).all()
    q = T.quantise(np.float32([[-1, 0, 0.5, 1 / 510, 1.5 / 255, 1, 2, np.nan]]))
    assert q.tolist() == [[0, 0, 128, 1, 2, 255, 255, 0]]


def _lib():
    from nerfmeshes_b200 import _lib as L
    return L.load()


def test_layout_matches_the_restatement():
    lib = _lib()
    out = (C.c_int64 * 4)()
    err = lambda: lib.nm_last_error().decode()
    for F in (0, 1, 2, 3, 4, 5, 17, 100, 1001, 65536, 123457, 2 ** 20, 200000, 2 ** 25 + 2):
        for N in (1, 2, 3, 8, 16, 17, 49, 50, 64, 65):
            try:
                want = T.layout(F, N)
            except ValueError:
                want = None
            rc = lib.nm_texture_layout(F, N, out)
            if want is None:
                assert rc != 0, (F, N)
                msg = err()
                if not 2 <= N <= 64:
                    assert f"N = {N} outside [2, 64]" in msg
                else:
                    best = T.largest_n(F)
                    assert ("largest N that fits" in msg and msg.endswith(f" is {best}")) if best else "even at N = 2" in msg, msg
            else:
                assert rc == 0 and tuple(out) == want, (F, N, tuple(out), want)
    assert T.largest_n(200000) == 49 and T.largest_n(2 ** 25 + 2) is None
    assert lib.nm_texture_layout(-1, 8, out) != 0 and lib.nm_texture_layout(2 ** 31, 8, out) != 0
    assert lib.nm_texture_layout(10, 8, None) != 0


def test_bake_rejects_bad_arguments_without_a_device():
    lib = _lib()
    P = C.c_void_p(16)                       # never dereferenced: every call below fails its argument checks first
    cnt = (C.c_int64 * 4)()
    nf = (C.c_float * 2)(0.0, 4.0)
    err = lambda: lib.nm_last_error().decode()

    def rejects(text, h=None, v=P, n=P, V=10, f=P, F=10, N=8, mode=0, flags=0, atlas=P, u8=P, uv=P, rgb=P, counts=cnt, bounds=nf):
        rc = lib.nm_bake_texture(h, v, n, V, f, F, N, mode, 0, flags, 0.01, bounds, atlas, u8, uv, rgb, counts, None)
        assert rc != 0 and text in err(), (rc, err())

    rejects("N = 1 outside", N=1)
    rejects("N = 65 outside", N=65)
    rejects("largest N that fits", F=200000, N=64)
    rejects("negative size", V=-1)
    rejects("negative size", F=-1)
    rejects("2^31", V=2 ** 31)
    rejects("2^31", F=2 ** 31)
    rejects("mode 2", mode=2)
    rejects("null counts", counts=None)
    for kw in (dict(v=None), dict(n=None)):
        rejects("null vertex pointer", **kw)
    rejects("null vertex colour pointer", rgb=None)
    rejects("null face pointer", f=None)
    for kw in (dict(atlas=None), dict(u8=None), dict(uv=None)):
        rejects("null atlas or uv pointer", **kw)
    rejects("null near/far", bounds=None)
    rejects("NM_FLAG_TEACHER_T", flags=4)
    rejects("null handle")
    rejects("null handle", v=None, n=None, f=None, V=0, F=0, atlas=None, u8=None, uv=None, rgb=None)
    rejects("null handle", f=None, F=0, atlas=None, u8=None, uv=None)          # F = 0 needs no face or atlas pointers
    a = (C.c_float * 3)()
    rc = lib.nm_debug_texture_rays(None, P, P, 10, P, 10, 8, 0, 0.0, 3, 11, a, a, None, None)
    assert rc != 0 and "face range [3, 11)" in err()


def _random_obj(seed):
    rng = np.random.default_rng(seed)
    V, F = 40, 30
    v = rng.normal(size=(V, 3)).astype(np.float32) * np.float32(10) ** rng.integers(-6, 18, size=(V, 3)).astype(np.float32)
    v[0] = [np.nan, np.inf, -np.inf]
    v[1] = [0.0, -0.0, 1e-4]
    n = rng.normal(size=(V, 3)).astype(np.float32)
    d = rng.uniform(size=(V, 3)).astype(np.float32)
    f = rng.integers(0, V, size=(F, 3)).astype(np.int32)
    uv = rng.uniform(size=(F, 3, 2)).astype(np.float32)
    return v, f, d, n, uv


def _write_textured(path, v, f, d, n, uv, mtl):
    ptr = lambda a: C.c_void_p(a.ctypes.data) if a.size else None
    from nerfmeshes_b200 import _lib as L
    L.check(_lib().nm_export_obj_textured(str(path).encode(), ptr(v), len(v), ptr(f), len(f), ptr(d), len(d), ptr(n), len(n),
                                          ptr(uv), mtl.encode()))


@pytest.mark.parametrize("seed", [0, 1])
def test_textured_obj_matches_python_formatter(tmp_path, seed):
    v, f, d, n, uv = _random_obj(seed)
    p = tmp_path / "m.obj"
    _write_textured(p, v, f, d, n, uv, "m.mtl")
    assert p.read_bytes() == T.obj_text(v, f, d, n, uv, "m.mtl").encode()


def test_textured_obj_reduces_to_the_plain_obj(tmp_path):
    from nerfmeshes_b200 import mesh
    v, f, d, n, uv = _random_obj(2)
    _write_textured(tmp_path / "t.obj", v, f, d, n, uv, "t.mtl")
    mesh.export_obj(v, f, d, n, str(tmp_path / "p.obj"))
    kept = []
    for line in (tmp_path / "t.obj").read_text().splitlines(keepends=True):
        if line.startswith(("mtllib ", "usemtl ", "vt ")):
            continue
        if line.startswith("f "):
            line = "f" + "".join(f" {a}//{c}" for a, _, c in (t.split("/") for t in line.split()[1:])) + "\n"
        kept.append(line)
    assert "".join(kept).encode() == (tmp_path / "p.obj").read_bytes()


def test_png_and_mtl(tmp_path):
    from nerfmeshes_b200 import mesh
    rng = np.random.default_rng(4)
    atlas = rng.integers(0, 256, size=(30, 20, 3), dtype=np.uint8)
    mesh.write_png(str(tmp_path / "a.png"), atlas)
    assert np.array_equal(T.read_png(str(tmp_path / "a.png")), atlas)
    v, f, d, n, _ = _random_obj(5)
    uv = T.uv(len(f), 4)
    paths = mesh.export_textured_obj(v, f, d, n, uv, atlas, str(tmp_path / "mesh.obj"))
    assert paths == (str(tmp_path / "mesh.obj"), str(tmp_path / "mesh.mtl"), str(tmp_path / "mesh.png"))
    assert (tmp_path / "mesh.mtl").read_text().splitlines() == [
        "newmtl texture", "Ka 1.0 1.0 1.0", "Kd 1.0 1.0 1.0", "Ks 0.0 0.0 0.0", "illum 1", "map_Kd mesh.png"]
    assert (tmp_path / "mesh.obj").read_text().startswith("mtllib mesh.mtl\n")
    assert (tmp_path / "mesh.obj").read_bytes() == T.obj_text(v, f, d, n, uv, "mesh.mtl").encode()
    assert np.array_equal(T.read_png(str(tmp_path / "mesh.png")), atlas)
