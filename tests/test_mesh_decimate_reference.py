"""Quadric-error decimation's semantics (DESIGN 4.11) without a device: the numpy restatement (_decimate_ref) on meshes of the
C marching-cubes oracle (a sphere, a torus, two spheres, a surface cut by the grid border) and hand-built meshes keeps a
consistently oriented manifold of the same Euler characteristic, the locked vertices bit for bit and every face's
orientation, ends at T or T - 1 faces unless no collapse is legal, and keeps the sphere close to the analytic surface.  One
round's collapses commute.  Without the link condition, or without the fold-over test, the corresponding check fails.
Argument checks of nm_mesh_decimate without a device."""
import ctypes as C

import numpy as np
import pytest

import _decimate_ref as D
from oracle import mc


def _sphere(c, r):
    return lambda P: r - np.linalg.norm(P - np.asarray(c), axis=-1)


def _torus(c, R, r):
    def f(P):
        d = P - np.asarray(c)
        return r - np.sqrt((np.sqrt(d[..., 0] ** 2 + d[..., 1] ** 2) - R) ** 2 + d[..., 2] ** 2)
    return f


FIELDS = {
    # name: (field of index coordinates, grid points per axis, Euler characteristic, closed)
    "sphere": (_sphere((15.3, 15.7, 16.1), 10.0), 32, 2, True),
    "torus": (_torus((20.2, 19.8, 20.3), 11.0, 4.0), 41, 0, True),
    "two_spheres": ((lambda a, b: lambda P: np.maximum(a(P), b(P)))(_sphere((9.2, 9.9, 10.3), 6.5), _sphere((24.1, 23.2, 22.7), 5.5)),
                    33, 4, True),
    # a sphere cut by the grid's first plane: an open disk, its border vertices locked
    "border": (_sphere((3.2, 16.1, 15.9), 9.0), 32, 1, False),
}


def _mesh(name):
    field, n, _, _ = FIELDS[name]
    g = np.stack(np.meshgrid(*[np.arange(n, dtype=np.float64)] * 3, indexing="ij"), -1)
    v, f, nrm = mc.marching_cubes(field(g).astype(np.float32), 0.0)
    return v, nrm, f


_MESHES = {}


def mesh(name):
    if name not in _MESHES:
        _MESHES[name] = _mesh(name)
    return _MESHES[name]


def edge_counts(f):
    f = np.asarray(f, np.int64)
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    V = int(f.max()) + 1 if len(f) else 1
    _, dcnt = np.unique(d[:, 0] * V + d[:, 1], return_counts=True)
    u = np.sort(d, 1)
    _, ucnt = np.unique(u[:, 0] * V + u[:, 1], return_counts=True)
    return ucnt, dcnt


def euler(f):
    f = np.asarray(f, np.int64)
    ucnt, _ = edge_counts(f)
    return len(np.unique(f)) - len(ucnt) + len(f)


def check(name, v0, f0, v, f, src, surface=True):
    """The invariants of decimation; AssertionError if one fails.  surface: the mesh still approximates the field's zero
    level (not a mesh decimated until no collapse is legal, which can end as two faces back to back)."""
    field, _, chi, closed = FIELDS[name]
    ucnt, dcnt = edge_counts(f)
    assert dcnt.max() == 1, "consistent orientation"
    assert set(ucnt) <= ({2} if closed else {1, 2}), "manifold"
    assert not ((f[:, 0] == f[:, 1]) | (f[:, 1] == f[:, 2]) | (f[:, 0] == f[:, 2])).any(), "no repeated index"
    assert euler(f) == euler(f0) == chi, "Euler characteristic"
    lock = D.locks(f0, len(v0))
    kept = np.zeros(len(v0), bool)
    kept[src] = True
    assert kept[lock].all(), "locked vertices survive"
    at = np.full(len(v0), -1)
    at[src] = np.arange(len(src))
    assert np.array_equal(v[at[np.flatnonzero(lock)]].view(np.int32), v0[lock].view(np.int32)), "locked vertices unmoved"
    if not surface:
        return
    # no flipped face: no face's winding normal turned more than 120 degrees away from the surface's outward normal (down
    # the field's gradient).  A fold-over reverses a face (cosine near -1); a thin face of a correct mesh can lean past 90.
    P = v.astype(np.float64)
    fn = D.cross(P[f[:, 0]], P[f[:, 1]], P[f[:, 2]])
    c = P[f].mean(1)
    h = 1e-4
    grad = np.stack([(field(c + h * e) - field(c - h * e)) / (2 * h) for e in np.eye(3)], 1)
    cos = D.dot(fn, -grad) / np.sqrt(D.dot(fn, fn) * D.dot(grad, grad))
    assert (cos > -0.5).all(), "flipped face"


@pytest.mark.parametrize("name", sorted(FIELDS))
@pytest.mark.parametrize("frac", [0.5, 0.1, 0.0])
def test_invariants(name, frac):
    v0, n0, f0 = mesh(name)
    T = int(frac * len(f0))
    v, n, f, src, counts = D.decimate(v0, n0, f0, T)
    assert counts == (len(v), len(f), counts[2], len(v0) - len(v)) and len(f) == len(f0) - 2 * counts[3]
    check(name, v0, f0, v, f, src, surface=frac > 0)
    if frac > 0:
        assert len(f) in (T, T - 1), (len(f), T)
    else:
        assert len(f) > 0 and counts[2] > 3               # stopped for lack of legal collapses
    same = np.all(v.view(np.int32) == v0[src].view(np.int32), 1)
    assert np.array_equal(n[same].view(np.int32), n0[src][same].view(np.int32)), "unmoved vertices keep their normal"
    np.testing.assert_allclose(np.linalg.norm(n[~same], axis=1), 1.0, atol=1e-6)


def test_sphere_stays_on_the_surface():
    field = FIELDS["sphere"][0]
    v0, n0, f0 = mesh("sphere")
    for frac, tol in ((0.5, 0.05), (0.1, 0.25)):
        v, n, f, src, _ = D.decimate(v0, n0, f0, int(frac * len(f0)))
        assert np.abs(field(v.astype(np.float64))).max() < tol, frac
        # and the moved vertices' normals point outwards
        P = v.astype(np.float64) - np.asarray((15.3, 15.7, 16.1))
        assert (np.sum(n * P, 1) > 0).all()


def test_target_at_or_above_face_count_is_the_identity():
    v0, n0, f0 = mesh("torus")
    for T in (len(f0), len(f0) + 1, 10 ** 9):
        v, n, f, src, counts = D.decimate(v0, n0, f0, T)
        assert counts == (len(v0), len(f0), 0, 0)
        assert np.array_equal(v.view(np.int32), v0.view(np.int32)) and np.array_equal(n.view(np.int32), n0.view(np.int32))
        assert np.array_equal(f, f0) and np.array_equal(src, np.arange(len(v0)))
    for T in (len(f0) - 1, len(f0) - 2, len(f0) - 5):            # odd and even F - T: one collapse removes two faces
        v, n, f, src, counts = D.decimate(v0, n0, f0, T)
        assert len(f) in (T, T - 1) and counts[3] == (len(f0) - T + 1) // 2


def test_one_round_commutes():
    for name in ("sphere", "border"):
        v0, n0, f0 = mesh(name)
        V = len(v0)
        lock, Q0 = D.locks(f0, V), D.vertex_quadrics(v0, f0, V)
        r = D.select(v0, Q0, f0, lock, V, 0)
        k = int(r["sel"].sum())
        assert k > 10
        outs = []
        for order in (None, np.arange(k), np.arange(k)[::-1], np.random.default_rng(3).permutation(k)):
            pos, Q, rem = v0.copy(), Q0.copy(), np.zeros(V, bool)
            fw = D.apply(pos, Q, f0, rem, r) if order is None else D.apply_sequential(pos, Q, f0, rem, r, order)
            outs.append((pos, Q, fw, rem))
        for pos, Q, fw, rem in outs[1:]:
            assert np.array_equal(pos.view(np.int32), outs[0][0].view(np.int32)) and np.array_equal(Q, outs[0][1])
            assert np.array_equal(fw, outs[0][2]) and np.array_equal(rem, outs[0][3])


def _fails(name, T, **kw):
    v0, n0, f0 = mesh(name)
    try:
        v, n, f, src, _ = D.decimate(v0, n0, f0, T, **kw)
        check(name, v0, f0, v, f, src, surface=T > 0)
    except AssertionError:
        return True
    return False


def test_the_checks_have_teeth():
    half = len(mesh("torus")[2]) // 2
    assert not _fails("torus", 0) and not _fails("torus", half)
    assert _fails("torus", 0, link=False)                    # collapses through the hole change the topology
    assert _fails("torus", half, fold=False)                 # a face folds over


def test_hand_cases():
    # a bipyramid with 40 equator vertices: the apexes have 40 faces (above the cap) and stay; the equator collapses
    k = 40
    t = 2 * np.pi * np.arange(k) / k
    v0 = np.concatenate([np.stack([5 * np.cos(t), 5 * np.sin(t), np.zeros(k)], 1), [[0, 0, 3], [0, 0, -3]]]).astype(np.float32)
    i = np.arange(k)
    f0 = np.concatenate([np.stack([i, (i + 1) % k, np.full(k, k)], 1), np.stack([(i + 1) % k, i, np.full(k, k + 1)], 1)]).astype(np.int32)
    n0 = np.zeros_like(v0)
    assert D.locks(f0, len(v0)).tolist() == [False] * k + [True, True]
    v, n, f, src, counts = D.decimate(v0, n0, f0, 0)
    assert src[-2:].tolist() == [k, k + 1] and np.array_equal(v[-2:], v0[-2:]) and counts[3] > 0
    ucnt, dcnt = edge_counts(f)
    assert set(ucnt) == {2} and dcnt.max() == 1 and euler(f) == 2
    # a face with a repeated index locks its vertices; they and their rows stay
    v0, n0, f0 = mesh("sphere")
    g = np.concatenate([f0, [[5, 5, 9]]]).astype(np.int32)
    lock = D.locks(g, len(v0))
    assert lock[5] and lock[9]
    v, n, f, src, _ = D.decimate(v0, n0, g, len(g) // 4)
    assert 5 in src and 9 in src and [int(np.flatnonzero(src == 5)[0])] * 2 + [int(np.flatnonzero(src == 9)[0])] in f.tolist()
    # empty and face-less meshes
    e = np.zeros((0, 3), np.float32)
    assert D.decimate(e, e, np.zeros((0, 3), np.int32), 0)[4] == (0, 0, 0, 0)
    one = np.ones((3, 3), np.float32)
    assert D.decimate(one, one, np.zeros((0, 3), np.int32), 0)[4] == (3, 0, 0, 0)


def test_rejected_arguments_without_a_device():
    from nerfmeshes_b200 import _lib as L
    lib = L.load()
    P = C.c_void_p(16)                       # never dereferenced: every call below fails its argument checks first
    cnt = (C.c_int64 * 4)()
    err = lambda: lib.nm_last_error().decode()

    def rejects(text, h=None, v=P, n=P, V=10, f=P, F=10, T=0, vo=P, no=P, fo=P, counts=cnt):
        rc = lib.nm_mesh_decimate(h, v, n, V, f, F, T, vo, no, fo, None, counts, None)
        assert rc != 0 and text in err(), (rc, err())

    rejects("negative size", V=-1)
    rejects("negative size", F=-1)
    rejects("negative target_faces", T=-1)
    rejects("2^31", V=2 ** 31)
    rejects("2^31", F=2 ** 31)
    rejects("3F", F=2 ** 30)
    rejects("null counts", counts=None)
    for kw in (dict(v=None), dict(n=None), dict(vo=None), dict(no=None)):
        rejects("null vertex pointer", **kw)
    for kw in (dict(f=None), dict(fo=None)):
        rejects("null face pointer", **kw)
    rejects("null handle")
    rejects("null handle", v=None, n=None, vo=None, no=None, f=None, fo=None, V=0, F=0)
    rejects("null handle", f=None, fo=None, F=0)             # F = 0 needs no face pointers
