"""numpy restatement of the sparse density sweep (DESIGN 4.10) on a DENSE volume: which points the sweep evaluates, which
blocks it activates, in how many rounds, and the volume it leaves (true values where evaluated, +-inf elsewhere).

Grid of n0 x n1 x n2 points, block edge B cells.  Block b of an axis covers cells [b*B, min((b+1)*B, n-1)); its closed point
set is points [b*B, min((b+1)*B, n-1)]; the lattice is the indices min(b*B, n-1), b = 0 .. number of blocks.
  1. the lattice points are evaluated;
  2. a block whose 8 lattice corners do not agree in value > iso is active; an inactive block has its corners' sign;
  3. every point of an active block's closed point set, dilated by `dilate` points per axis and clipped, is evaluated;
  4. an inactive block with an evaluated point of the other sign in its closed point set becomes active; 3-4 repeat until a
     round activates nothing (a round = one pass of 3 over a non-empty set of newly active blocks);
  5. unevaluated points become +inf where their block's sign is inside (> iso), -inf otherwise.
`dilate` and `max_rounds` exist so that tests can show what breaks without the one-point dilation or the fixpoint."""
import numpy as np


def blocks_per_axis(n, B):
    return (n - 1 + B - 1) // B


def lattice_indices(n, B):
    return np.minimum(np.arange(blocks_per_axis(n, B) + 1) * B, n - 1)


def _closed_block_any(x, B):
    """any() of a bool volume over every block's closed point set -> (nb0, nb1, nb2)."""
    for axis in range(3):
        n = x.shape[axis]
        nb = blocks_per_axis(n, B)
        half_open = np.logical_or.reduceat(x, np.arange(nb) * B, axis=axis)       # [b*B, (b+1)*B), the last one to the end
        x = half_open | np.take(x, lattice_indices(n, B)[1:], axis=axis)          # ... and the closing plane
    return x


def sparse_sweep(dense, iso, B, dilate=1, max_rounds=None):
    """-> dict(evaluated bool (n0,n1,n2), active bool (nb0,nb1,nb2), sign bool (nb0,nb1,nb2), rounds, filled float32 volume,
    lattice float32 (the lattice values, flat in lattice order))."""
    dense = np.asarray(dense, np.float32)
    n = dense.shape
    iso = np.float32(iso)
    inside = dense > iso
    lat = [lattice_indices(m, B) for m in n]
    nb = [blocks_per_axis(m, B) for m in n]
    evaluated = np.zeros(n, bool)
    evaluated[np.ix_(*lat)] = True
    corners = inside[np.ix_(*lat)].astype(np.int32)
    cnt = sum(corners[a:a + nb[0], b:b + nb[1], c:c + nb[2]] for a in (0, 1) for b in (0, 1) for c in (0, 1))
    sign = cnt == 8
    active = (cnt != 0) & (cnt != 8)
    new, rounds = active.copy(), 0
    while new.any() and (max_rounds is None or rounds < max_rounds):
        for b in np.argwhere(new):
            box = tuple(slice(max(int(b[a]) * B - dilate, 0), min(int(lat[a][b[a] + 1]) + dilate, n[a] - 1) + 1) for a in range(3))
            evaluated[box] = True
        rounds += 1
        other_than_outside = _closed_block_any(evaluated & inside, B)
        other_than_inside = _closed_block_any(evaluated & ~inside, B)
        new = ~active & np.where(sign, other_than_inside, other_than_outside)
        active |= new
    of_point = [np.minimum(np.arange(m) // B, k - 1) for m, k in zip(n, nb)]
    point_sign = sign[np.ix_(*of_point)]
    filled = np.where(evaluated, dense, np.where(point_sign, np.float32(np.inf), np.float32(-np.inf))).astype(np.float32)
    return dict(evaluated=evaluated, active=active, sign=sign, rounds=rounds, filled=filled, lattice=dense[np.ix_(*lat)].reshape(-1))


def mesh_subset(dense_mesh, sparse_mesh):
    """Checks that the sparse mesh (verts, faces, normals) is the dense one with rows deleted: every sparse vertex row (and
    its normal) is a dense row bit for bit, in the dense order, and the sparse faces are dense faces, re-indexed, in order.
    Returns (kept vertex mask (V,), kept face mask (F,)) over the dense arrays."""
    dv, df, dn = (np.asarray(x) for x in dense_mesh)
    sv, sf, sn = (np.asarray(x) for x in sparse_mesh)
    assert np.isfinite(sv).all() and np.isfinite(sn).all(), "non-finite vertex or normal"
    key = lambda v: [r.tobytes() for r in np.ascontiguousarray(v, np.float32)]
    where = {k: i for i, k in enumerate(key(dv))}
    assert len(where) == len(dv), "dense vertex rows are not unique"
    idx = np.array([where.get(k, -1) for k in key(sv)], np.int64)
    assert (idx >= 0).all(), f"{int((idx < 0).sum())} sparse vertices are not dense vertices"
    assert (np.diff(idx) > 0).all(), "vertex order differs"
    assert np.array_equal(np.asarray(sn, np.float32).view(np.int32), np.asarray(dn, np.float32)[idx].view(np.int32)), "normals differ"
    vkeep = np.zeros(len(dv), bool)
    vkeep[idx] = True
    fkeep = vkeep[df].all(1) if len(df) else np.zeros(0, bool)
    assert np.array_equal(idx[sf] if len(sf) else np.zeros((0, 3), np.int64), df[fkeep]), "faces differ"
    return vkeep, fkeep


def whole_components(dense_mesh, vkeep, fkeep):
    """Checks that the kept part is a union of whole connected components of the dense mesh.  Returns (sizes in faces of the
    kept components, of the missing ones), each sorted descending."""
    from _components_ref import labels_and_sizes
    dv, df, _ = (np.asarray(x) for x in dense_mesh)
    labels, sizes = labels_and_sizes(len(dv), df)
    roots = np.flatnonzero((labels == np.arange(len(dv))) & (sizes > 0))
    kept_faces = np.bincount(labels[df[fkeep][:, 0]], minlength=len(dv)) if fkeep.any() else np.zeros(len(dv), np.int64)
    kept_verts = np.bincount(labels[vkeep], minlength=len(dv))
    all_verts = np.bincount(labels, minlength=len(dv))
    for r in roots:
        assert kept_faces[r] in (0, sizes[r]), f"component {r}: {kept_faces[r]} of {sizes[r]} faces kept"
        assert kept_verts[r] == (all_verts[r] if kept_faces[r] else 0), f"component {r}: vertices and faces disagree"
    kept = np.sort(sizes[roots][kept_faces[roots] > 0])[::-1]
    missing = np.sort(sizes[roots][kept_faces[roots] == 0])[::-1]
    return kept, missing
