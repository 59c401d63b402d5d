"""Numpy restatement of quadric-error decimation (nm_mesh_decimate, DESIGN 4.11), bit for bit.

Every floating-point value is computed with the operations of nm_decimate.cu in the same order: elementwise numpy double
arithmetic is one IEEE operation per step, like the kernels built with -fmad=false.  Sums whose order matters go through
np.add.at over the faces in ascending index (never np.sum, which sums pairwise).  Rounds are vectorised: the selected
collapses have disjoint closed neighbourhoods, so applying them at once equals applying them one by one in any order
(apply_sequential, which the tests compare).  `link=False` / `fold=False` drop one legality rule, to show that the checks
fail without it."""
import numpy as np
from scipy.sparse import coo_matrix

VALENCE_CAP = 32
DET_MIN = 1e-12
NO_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)


def cross(p0, p1, p2):
    """(p1 - p0) x (p2 - p0) in double, rows."""
    e1, e2 = p1 - p0, p2 - p0
    return np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                     e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)


def dot(a, b):
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


def qcost(q, p):
    """x^T Q x for x = (p, 1), clamped at 0 (q: (n,10) rows, p: (n,3) double)."""
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    r0 = ((q[:, 0] * x + q[:, 1] * y) + q[:, 2] * z) + q[:, 3]
    r1 = ((q[:, 1] * x + q[:, 4] * y) + q[:, 5] * z) + q[:, 6]
    r2 = ((q[:, 2] * x + q[:, 5] * y) + q[:, 7] * z) + q[:, 8]
    r3 = ((q[:, 3] * x + q[:, 6] * y) + q[:, 8] * z) + q[:, 9]
    c = ((r0 * x + r1 * y) + r2 * z) + r3
    return np.where(c > 0.0, c, 0.0)


def lists(fw, V):
    """Vertex -> face lists: (start (V+1,), faces), each list ascending; a face appears once per corner at the vertex."""
    vert = fw.reshape(-1).astype(np.int64)
    face = np.repeat(np.arange(len(fw), dtype=np.int64), 3)
    order = np.lexsort((face, vert))
    deg = np.bincount(vert, minlength=V)
    return np.concatenate([[0], np.cumsum(deg)]).astype(np.int64), face[order]


def ragged(start, vs):
    """For each vertex of vs its list positions: (owner index into vs, position)."""
    cnt = start[vs + 1] - start[vs]
    owner = np.repeat(np.arange(len(vs)), cnt)
    first = np.repeat(np.cumsum(cnt) - cnt, cnt)
    return owner, start[vs][owner] + (np.arange(int(cnt.sum())) - first)


def locks(fw, V):
    """More than VALENCE_CAP face corners, a face with a repeated index, or an edge with other than two faces."""
    f = fw.astype(np.int64)
    lock = np.bincount(f.reshape(-1), minlength=V) > VALENCE_CAP
    rep = (f[:, 0] == f[:, 1]) | (f[:, 1] == f[:, 2]) | (f[:, 0] == f[:, 2])
    lock[f[rep].reshape(-1)] = True
    g = f[~rep]
    e = np.concatenate([g[:, [0, 1]], g[:, [1, 2]], g[:, [2, 0]]])
    e.sort(1)
    keys, cnt = np.unique(e[:, 0] * V + e[:, 1], return_counts=True)
    bad = keys[cnt != 2]
    lock[bad // V] = True
    lock[bad % V] = True
    return lock


def vertex_quadrics(pos, fw, V):
    """Q_v = sum over v's faces of non-zero area, ascending face index, of area [n n^T, n d; d d^2] (10 unique entries)."""
    P = pos.astype(np.float64)
    f = fw.astype(np.int64)
    p0 = P[f[:, 0]]
    c = cross(p0, P[f[:, 1]], P[f[:, 2]])
    ln = np.sqrt(dot(c, c))
    ok = ln > 0.0
    with np.errstate(invalid="ignore", divide="ignore"):
        nx, ny, nz = c[:, 0] / ln, c[:, 1] / ln, c[:, 2] / ln
    d = -((nx * p0[:, 0] + ny * p0[:, 1]) + nz * p0[:, 2])
    a = 0.5 * ln
    q = np.stack([a * (nx * nx), a * (nx * ny), a * (nx * nz), a * (nx * d), a * (ny * ny), a * (ny * nz), a * (ny * d),
                  a * (nz * nz), a * (nz * d), a * (d * d)], 1)
    Q = np.zeros((V, 10), np.float64)
    np.add.at(Q, f[ok].reshape(-1), np.repeat(q[ok], 3, axis=0))
    return Q


def candidates(fw, lock, V):
    """Candidate edges (a, b), a < b, both unlocked, numbered by (a, b): the kernel's per-vertex numbering."""
    f = fw.astype(np.int64)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    e.sort(1)
    e = e[~lock[e[:, 0]] & ~lock[e[:, 1]]]
    keys = np.unique(e[:, 0] * V + e[:, 1])
    return keys // V, keys % V


def positions(Q, pos, a, b):
    """(double position, cost) of the cheapest of a, b, the midpoint and the quadric's minimiser (if |det| > DET_MIN and
    within one cell, L-inf, of the midpoint); ties go to the earlier point."""
    q = Q[a] + Q[b]
    pa, pb = pos[a].astype(np.float64), pos[b].astype(np.float64)
    mid = (pa + pb) * 0.5
    best, cost = pa.copy(), qcost(q, pa)
    for p in (pb, mid):
        c = qcost(q, p)
        t = c < cost
        best[t], cost[t] = p[t], c[t]
    c00, c01, c02 = q[:, 4] * q[:, 7] - q[:, 5] * q[:, 5], q[:, 2] * q[:, 5] - q[:, 1] * q[:, 7], q[:, 1] * q[:, 5] - q[:, 2] * q[:, 4]
    c11, c12, c22 = q[:, 0] * q[:, 7] - q[:, 2] * q[:, 2], q[:, 1] * q[:, 2] - q[:, 0] * q[:, 5], q[:, 0] * q[:, 4] - q[:, 1] * q[:, 1]
    det = (q[:, 0] * c00 + q[:, 1] * c01) + q[:, 2] * c02
    r0, r1, r2 = -q[:, 3], -q[:, 6], -q[:, 8]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        s = np.stack([((c00 * r0 + c01 * r1) + c02 * r2) / det, ((c01 * r0 + c11 * r1) + c12 * r2) / det,
                      ((c02 * r0 + c12 * r1) + c22 * r2) / det], 1)
        ok = (np.abs(det) > DET_MIN) & np.all(np.abs(s - mid) <= 1.0, 1)
        c = qcost(q, np.where(ok[:, None], s, mid))
    t = ok & (c < cost)
    best[t], cost[t] = s[t], c[t]
    return best, cost


def _no_fold(pos, fw, start, flist, v, other, p):
    """Per edge: every face of v without `other` keeps n_old . n_new > 0 with v at p (double)."""
    owner, k = ragged(start, v)
    faces = flist[k]
    t = fw[faces].astype(np.int64)
    live = ~np.any(t == other[owner][:, None], 1)
    owner, t = owner[live], t[live]
    P = pos.astype(np.float64)
    c = [P[t[:, j]] for j in range(3)]
    n_old = cross(*c)
    c = [np.where((t[:, j] == v[owner])[:, None], p[owner], c[j]) for j in range(3)]
    n_new = cross(*c)
    bad = ~(dot(n_old, n_new) > 0.0)
    return np.bincount(owner[bad], minlength=len(v)) == 0


def select(pos, Q, fw, lock, V, target, link=True, fold=True):
    """One round's candidates: dict with a, b, key, newpos (float32), the faces of every edge, and sel (after the trim)."""
    F = len(fw)
    start, flist = lists(fw, V)
    deg = start[1:] - start[:-1]
    a, b = candidates(fw, lock, V)
    E = len(a)
    # the two faces of each edge (ascending) and their opposite vertices
    f = fw.astype(np.int64)
    fe = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    fid = np.tile(np.arange(F), 3)
    fe.sort(1)
    ek = fe[:, 0] * V + fe[:, 1]
    order = np.lexsort((fid, ek))
    ek, fid = ek[order], fid[order]
    first = np.searchsorted(ek, a * V + b)
    last = np.searchsorted(ek, a * V + b, side="right") - 1
    f1, f2 = fid[np.minimum(first, len(fid) - 1)], fid[np.maximum(last, 0)]
    opp = lambda g: f[g].sum(1) - a - b
    legal = (opp(f1) != opp(f2)) & (deg[a] + deg[b] - 4 <= VALENCE_CAP)
    if link and E:
        rows = np.concatenate([f[:, 0], f[:, 1], f[:, 2], f[:, 1], f[:, 2], f[:, 0]])
        cols = np.concatenate([f[:, 1], f[:, 2], f[:, 0], f[:, 0], f[:, 1], f[:, 2]])
        keep = rows != cols
        A = coo_matrix((np.ones(int(keep.sum()), np.int8), (rows[keep], cols[keep])), shape=(V, V)).tocsr()
        A.data[:] = 1
        common = np.asarray(A[a].multiply(A[b]).sum(1)).reshape(-1)
        legal &= common == 2
    best, cost = positions(Q, pos, a, b)
    newpos = best.astype(np.float32)
    if fold and E:
        p = newpos.astype(np.float64)
        legal &= _no_fold(pos, fw, start, flist, a, b, p) & _no_fold(pos, fw, start, flist, b, a, p)
    key = (cost.astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.arange(E, dtype=np.uint64)
    key[~legal] = NO_KEY
    m = np.full(V, NO_KEY, np.uint64)
    np.minimum.at(m, a[legal], key[legal])
    np.minimum.at(m, b[legal], key[legal])
    emin = key.copy()
    for ends in (a, b):
        owner, k = ragged(start, ends)
        np.minimum.at(emin, owner, m[f[flist[k]]].min(1))
    sel = legal & (emin == key)
    n_sel = int(sel.sum())
    need = (F - target + 1) // 2
    if n_sel > need:
        sel &= key <= np.sort(key[sel])[need - 1]
    return dict(a=a, b=b, key=key, newpos=newpos, faces=np.stack([f1, f2], 1), sel=sel, selected=n_sel, legal=legal)


def apply(pos, Q, fw, removed, r):
    """All of a round's selected collapses at once: b -> a, a's position and quadric, the edge's two faces die."""
    s = r["sel"]
    A, B = r["a"][s], r["b"][s]
    pos[A] = r["newpos"][s]
    Q[A] = Q[A] + Q[B]
    removed[B] = True
    vmap = np.arange(len(pos))
    vmap[B] = A
    dead = np.zeros(len(fw), bool)
    dead[r["faces"][s].reshape(-1)] = True
    return vmap[fw][~dead].astype(np.int32)


def apply_sequential(pos, Q, fw, removed, r, order):
    """The same collapses one at a time, in the order of `order` (indices into the selected edges)."""
    idx = np.flatnonzero(r["sel"])[order]
    fw = fw.astype(np.int64).copy()
    dead = np.zeros(len(fw), bool)
    for e in idx:
        a, b = int(r["a"][e]), int(r["b"][e])
        pos[a] = r["newpos"][e]
        Q[a] = Q[a] + Q[b]
        removed[b] = True
        hb = np.any(fw == b, 1) & ~dead
        both = hb & np.any(fw == a, 1)
        dead |= both
        rows = hb & ~both
        fw[rows] = np.where(fw[rows] == b, a, fw[rows])
    return fw[~dead].astype(np.int32)


def finish(verts, normals, pos, fw, removed):
    """Surviving vertices in input order, normals (input row if the position kept its bits, else the normalised sum of the
    faces' winding normals in ascending face index), faces re-indexed, source."""
    V = len(verts)
    keep = ~removed
    new = np.arange(V) - (np.cumsum(removed) - removed)
    moved = np.any(pos.view(np.int32) != verts.view(np.int32), 1)
    n = normals.copy()
    if moved.any():
        P = pos.astype(np.float64)
        f = fw.astype(np.int64)
        c = cross(P[f[:, 0]], P[f[:, 1]], P[f[:, 2]])
        s = np.zeros((V, 3), np.float64)
        np.add.at(s, f.reshape(-1), np.repeat(c, 3, axis=0))
        ln = np.sqrt(dot(s, s))
        upd = moved & (ln > 0.0)
        n[upd] = (s[upd] / ln[upd, None]).astype(np.float32)
    return pos[keep].copy(), n[keep], new[fw.astype(np.int64)].astype(np.int32).reshape(-1, 3), np.flatnonzero(keep).astype(np.int32)


def decimate(verts, normals, faces, target, link=True, fold=True, max_rounds=None, on_round=None):
    """-> (verts, normals, faces, source, counts = (V', F', rounds, collapses)) like Engine.mesh_decimate.  on_round(state)
    is called after every round with the intermediate (pos, fw, removed)."""
    verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 3)
    normals = np.ascontiguousarray(normals, np.float32).reshape(-1, 3)
    fw = np.ascontiguousarray(faces, np.int32).reshape(-1, 3)
    V = len(verts)
    pos, removed = verts.copy(), np.zeros(V, bool)
    rounds = collapses = 0
    if target < len(fw):
        lock = locks(fw, V)
        Q = vertex_quadrics(pos, fw, V)
        while len(fw) > target and (max_rounds is None or rounds < max_rounds):
            r = select(pos, Q, fw, lock, V, target, link, fold)
            n = int(r["sel"].sum())
            if n == 0:
                break
            fw = apply(pos, Q, fw, removed, r)
            rounds += 1
            collapses += n
            if on_round is not None:
                on_round(pos, fw, removed)
    vo, no, fo, src = finish(verts, normals, pos, fw, removed)
    return vo, no, fo, src, (len(vo), len(fo), rounds, collapses)
