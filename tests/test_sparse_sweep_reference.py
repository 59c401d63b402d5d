"""The sparse sweep's semantics (DESIGN 4.10) on analytic volumes, without a device: the numpy restatement
(_sparse_sweep_ref) leaves a volume whose marching-cubes mesh (oracle/mc_oracle.c) is finite, is the dense mesh with rows
deleted bit for bit, and misses only whole components of the dense mesh, namely those that fit between lattice points and
touch no block the sweep reached.  Without the one-point dilation, or without the rounds after the first, the same checks fail."""
import numpy as np
import pytest

import _sparse_sweep_ref as S
from oracle import mc


def _grid(shape):
    return np.meshgrid(*[np.arange(m, dtype=np.float64) for m in shape], indexing="ij")


def sphere(shape, c, r):
    X, Y, Z = _grid(shape)
    return r - np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2)


def torus(shape, c, R, r):
    X, Y, Z = _grid(shape)
    return r - np.sqrt((np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2) - R) ** 2 + (Z - c[2]) ** 2)


def capsule(shape, a, b, r):
    P = np.stack(_grid(shape), -1)
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    t = np.clip(((P - a) @ (b - a)) / ((b - a) @ (b - a)), 0.0, 1.0)
    return r - np.linalg.norm(P - (a + t[..., None] * (b - a)), axis=-1)


N = (41, 41, 41)
VOLUMES = {
    # name: (field, block edge)
    "sphere": (lambda: sphere(N, (20.3, 20.1, 19.7), 12.0), 8),
    "torus": (lambda: torus(N, (20.2, 19.8, 23.2), 12.0, 3.5), 8),
    # a shell: two nested surfaces, two components
    "nested_spheres": (lambda: np.minimum(sphere(N, (20.3, 20.1, 19.7), 15.0), -sphere(N, (20.3, 20.1, 19.7), 9.0)), 8),
    # a sphere that contains no lattice point, next to one that does
    "sub_block_sphere": (lambda: np.maximum(sphere(N, (28.2, 27.9, 28.1), 9.0), sphere(N, (12.1, 11.9, 12.2), 2.6)), 8),
    # a thin rod that leaves the sphere's seed blocks along a diagonal
    "rod": (lambda: np.maximum(sphere(N, (16.2, 15.9, 16.1), 5.0), capsule(N, (16.2, 15.9, 16.1), (37.4, 35.2, 33.1), 1.3)), 8),
    "boundary": (lambda: sphere(N, (3.2, 20.1, 36.9), 8.0), 8),
    # the last block of every axis is clipped; a small sphere inside those blocks holds one lattice point
    "not_a_multiple": (lambda: np.maximum(sphere((45, 38, 43), (22.3, 18.1, 21.7), 13.0), sphere((45, 38, 43), (41.0, 34.0, 40.0), 2.4)), 8),
    "block_16": (lambda: torus((45, 38, 43), (22.2, 18.8, 21.4), 12.0, 6.0), 16),
    "block_4": (lambda: np.maximum(sphere(N, (28.2, 27.9, 28.1), 9.0), sphere(N, (10.1, 9.9, 10.2), 1.6)), 4),
    # one block per axis: its corners are the grid's
    "grid_smaller_than_block_all_outside": (lambda: sphere((6, 7, 5), (2.6, 3.1, 2.2), 1.7), 8),
    "grid_smaller_than_block_mixed": (lambda: sphere((6, 7, 5), (0.4, 0.3, 0.2), 3.6), 8),
}


def _meshes(vol, B, **kw):
    vol = vol.astype(np.float32)
    r = S.sparse_sweep(vol, 0.0, B, **kw)
    return mc.marching_cubes(vol, 0.0), mc.marching_cubes(r["filled"], 0.0), r


def _check(vol, B, **kw):
    dense, sparse, r = _meshes(vol, B, **kw)
    vkeep, fkeep = S.mesh_subset(dense, sparse)
    kept, missing = S.whole_components(dense, vkeep, fkeep)
    return dense, sparse, r, kept, missing


@pytest.mark.parametrize("name", sorted(VOLUMES))
def test_sparse_mesh_is_whole_components_of_the_dense_mesh(name):
    field, B = VOLUMES[name]
    dense, sparse, r, kept, missing = _check(field(), B)
    ev, filled = r["evaluated"], r["filled"]
    assert np.array_equal(filled[ev], field().astype(np.float32)[ev]) and np.isinf(filled[~ev]).all()
    expect_missing = {"sub_block_sphere": 1, "block_4": 1, "grid_smaller_than_block_all_outside": 1}.get(name, 0)
    assert len(missing) == expect_missing, (kept, missing)
    if name == "grid_smaller_than_block_all_outside":
        assert len(sparse[0]) == 0 and r["rounds"] == 0 and not r["active"].any() and len(dense[0]) > 0
        return
    assert len(kept) >= 1 and len(sparse[1]) == kept.sum()
    if expect_missing:
        assert missing[0] < kept.min()                       # the small sphere is what is missing
    if name == "grid_smaller_than_block_mixed":
        assert ev.all() and r["rounds"] == 1
    if name in ("nested_spheres", "not_a_multiple"):
        assert len(kept) == 2
    if name == "rod":
        assert len(kept) == 1 and r["rounds"] >= 3           # followed block by block well past the seeds
        seeds = S.sparse_sweep(field().astype(np.float32), 0.0, B, max_rounds=0)["active"]
        assert r["active"].sum() > seeds.sum()
    if name == "boundary":
        assert ev[0].any()                                   # the open surface reaches the grid's first plane
    assert r["evaluated"].sum() < r["evaluated"].size or min(field().shape) <= B


def test_inactive_blocks_have_no_mixed_cell_and_one_sign_per_point():
    for name, (field, B) in VOLUMES.items():
        vol = field().astype(np.float32)
        r = S.sparse_sweep(vol, 0.0, B)
        inside = r["filled"] > 0
        # where the filled volume and the dense one disagree in sign there is no evaluated point: the sign of an
        # unevaluated point is its block's, and all blocks that contain it agree
        n = vol.shape
        for shift in ((0, 0, 0), (1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1)):
            of_point = [np.minimum(np.maximum(np.arange(m) - s, 0) // B, S.blocks_per_axis(m, B) - 1) for m, s in zip(n, shift)]
            other = r["sign"][np.ix_(*of_point)]
            act = r["active"][np.ix_(*of_point)]
            assert np.array_equal(other[~r["evaluated"]], inside[~r["evaluated"]]), (name, shift)
            assert not act[~r["evaluated"]].any(), (name, shift)
        # every cell with corners on both sides of iso in the FILLED volume has all 8 corners evaluated
        c = [inside[a:n[0] - 1 + a, b:n[1] - 1 + b, d:n[2] - 1 + d] for a in (0, 1) for b in (0, 1) for d in (0, 1)]
        e = [r["evaluated"][a:n[0] - 1 + a, b:n[1] - 1 + b, d:n[2] - 1 + d] for a in (0, 1) for b in (0, 1) for d in (0, 1)]
        mixed = np.any(c, 0) & ~np.all(c, 0)
        assert np.all(e, 0)[mixed].all(), name


def _fails(vol, B, **kw):
    try:
        _check(vol, B, **kw)
    except AssertionError:
        return True
    return False


def test_the_checks_have_teeth():
    # without the one-point dilation the normals' central differences reach +-inf
    assert _fails(VOLUMES["sphere"][0](), 8, dilate=0)
    # stopping after the seeds' round cuts the rod where it leaves the seed blocks
    assert _fails(VOLUMES["rod"][0](), 8, max_rounds=1)
    assert not _fails(VOLUMES["rod"][0](), 8)


def test_rounds_and_monotonicity():
    vol = VOLUMES["rod"][0]().astype(np.float32)
    full = S.sparse_sweep(vol, 0.0, 8)
    prev = None
    for k in range(full["rounds"] + 2):
        r = S.sparse_sweep(vol, 0.0, 8, max_rounds=k)
        assert r["rounds"] == min(k, full["rounds"])
        if prev is not None:
            assert (r["evaluated"] | ~prev["evaluated"]).all() and (r["active"] | ~prev["active"]).all()
        prev = r
    assert np.array_equal(prev["filled"].view(np.int32), full["filled"].view(np.int32))
