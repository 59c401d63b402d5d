"""Sparse density sweep (nm_sparse_sweep_lattice / nm_sparse_sweep_run, DESIGN 4.10): argument checks without a device;
on the GPU the evaluated mask, the active blocks, the round count and the filled volume against the numpy restatement
(_sparse_sweep_ref) run on the dense grid_sigma volume, bit for bit, at every precision, block edge and chunk size; the
lattice iso level; and through extract_geometry the sparse mesh as whole components of the dense mesh."""
import ctypes as C
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import _sparse_sweep_ref as S

PREC = {"exact": 0, "fast": 1, "fp32": 2}
LIMIT = 1.2


# ----------------------------------------------------------------------------------------------------------------- CPU
def test_rejected_arguments_without_a_device():
    from nerfmeshes_b200 import _lib as L
    lib = L.load()
    P = C.c_void_p(16)                       # never dereferenced: every call below fails its argument checks first
    out = (C.c_int64 * 5)()
    err = lambda: lib.nm_last_error().decode()

    def rejects(text, h=None, lin=(P, P, P), n=(64, 64, 64), block=8, vol=P, host=out):
        rc = lib.nm_sparse_sweep_lattice(h, *lin, *n, block, vol, host, None)
        assert rc != 0 and text in err(), (rc, err())
        rc = lib.nm_sparse_sweep_run(h, *lin, *n, block, 32.0, vol, host, None)
        assert rc != 0 and text in err(), (rc, err())

    for block in (0, 1, 2, 3, 5, 12, 32, -8):
        rejects("is not one of 4, 8, 16", block=block)
    for n in ((1, 64, 64), (64, 1, 64), (64, 64, 0), (-3, 64, 64)):
        rejects("fewer than 2 points", n=n)
    rejects("2^31 points or more", n=(2048, 1024, 1024))
    rejects("2^31 points or more", n=(46341, 46341, 2))
    for kw in (dict(lin=(None, P, P)), dict(lin=(P, None, P)), dict(lin=(P, P, None)), dict(vol=None), dict(host=None)):
        rejects("null pointer", **kw)
    rejects("null handle")


# ----------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def models():
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import LEGO_CFG
    return {name: nm.NeRFModel.from_npz(LEGO_CFG, load_npz(f"weights_{name}_nerf.npz")).eval() for name in ("lego", "fern")}


def engine(model, prec):
    model.precision = PREC[prec]
    return model._engine()


def tables(shape):
    return [torch.linspace(-LIMIT, LIMIT, n) for n in shape]


def sweep(eng, shape, B, iso_level=32.0, chunk=None):
    """-> (volume, iso, counts, evaluated mask, block states) of one sparse sweep, on the host."""
    old = os.environ.pop("NM_SPARSE_CHUNK_POINTS", None)
    if chunk:
        os.environ["NM_SPARSE_CHUNK_POINTS"] = str(chunk)
    try:
        out = torch.full(shape, float("nan"), dtype=torch.float32, device=eng.device)
        iso, counts = eng.sparse_sweep(tables(shape), iso_level, B, out)
        mask, state = eng.debug_sparse_state(shape, B)
        eng.check_flags()
    finally:
        os.environ.pop("NM_SPARSE_CHUNK_POINTS", None)
        if old is not None:
            os.environ["NM_SPARSE_CHUNK_POINTS"] = old
    return out.cpu().numpy(), iso, counts, mask.cpu().numpy(), state.cpu().numpy()


def same_as_restatement(eng, dense, shape, B, chunks):
    vol, iso, counts, mask, state = sweep(eng, shape, B)
    r = S.sparse_sweep(dense, iso, B)
    assert np.array_equal(mask, r["evaluated"]), "evaluated mask differs"
    assert np.array_equal((state & 2) != 0, r["active"]), "active blocks differ"
    assert np.array_equal((state & 1) != 0, r["sign"]), "block signs differ"
    assert counts == (r["lattice"].size, int(r["active"].sum()), r["active"].size, int(r["evaluated"].sum()), r["rounds"]), counts
    assert np.array_equal(vol.view(np.int32), r["filled"].view(np.int32)), "filled volume differs"
    # every evaluated point holds the dense sweep's sigma, every other point +-inf
    assert np.array_equal(vol[mask].view(np.int32), dense[mask].view(np.int32)) and np.isinf(vol[~mask]).all()
    for chunk in chunks:                         # None: a second run at the default chunk size
        again = sweep(eng, shape, B, chunk=chunk)
        assert np.array_equal(again[0].view(np.int32), vol.view(np.int32)), f"chunk {chunk}: volume differs"
        assert again[2] == counts and np.array_equal(again[3], mask) and np.array_equal(again[4], state), f"chunk {chunk}"
    return counts, r


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["exact", "fast", "fp32"])
@pytest.mark.parametrize("net", ["lego", "fern"])
def test_matches_the_restatement(models, net, prec):
    eng = engine(models[net], prec)
    # exact: every shape (128: 16-byte fill stores; 130: a partial last word; 160) and block edge; the others a subset
    shapes = [(64, 64, 64), (96, 80, 130), (128, 128, 128), (160, 160, 160)] if prec == "exact" else [(64, 64, 64), (96, 80, 130)]
    for shape in shapes:
        dense = eng.grid_sigma(tables(shape)).cpu().numpy()
        for B in (4, 8, 16):
            first = shape == shapes[0] or shape == shapes[1]
            counts, r = same_as_restatement(eng, dense, shape, B, chunks=(3001, None) if first else (100003,))
            print(f"{net} {prec} {shape} B={B}: lattice {counts[0]}, blocks {counts[1]}/{counts[2]}, points {counts[3]}/{dense.size}, "
                  f"rounds {counts[4]}")
            if net == "lego":
                assert 0 < counts[1] < counts[2] and counts[3] < dense.size and counts[4] >= 1
    if net == "lego":
        assert 3001 < counts[3] - counts[0]      # the small chunk was smaller than the point lists it cut


@pytest.mark.gpu
def test_lattice_iso_level(models):
    from nerfmeshes_b200 import mesh
    eng = engine(models["lego"], "exact")
    shape, B = (70, 64, 90), 8
    out = torch.zeros(shape, dtype=torch.float32, device=eng.device)
    mn, mx, sd = eng.sparse_lattice(tables(shape), B, out)
    lat = out.cpu().numpy()[np.ix_(*[S.lattice_indices(n, B) for n in shape])]
    dense = eng.grid_sigma(tables(shape)).cpu().numpy()
    assert np.array_equal(lat.view(np.int32), dense[np.ix_(*[S.lattice_indices(n, B) for n in shape])].view(np.int32))
    assert mn == float(lat.min()) and mx == float(lat.max())
    assert abs(sd - float(lat.astype(np.float64).std())) <= 1e-6 * sd
    for level in (32.0, 1e9, -1e9, float(mn) + 0.5 * sd):
        iso, _ = eng.sparse_sweep(tables(shape), level, B, out)
        want = mesh.clamp_iso_level(level, np.float32(mn), np.float32(mx), np.float32(sd))
        assert iso == float(want), (level, iso, want)
    assert eng.sparse_sweep(tables(shape), 1e9, B, out)[0] == float(np.float32(mx) - np.float32(sd))
    assert eng.sparse_sweep(tables(shape), -1e9, B, out)[0] == float(np.float32(mn) + np.float32(sd))
    eng.check_flags()


def geometry(model, **kw):
    import nerfmeshes_b200 as nm
    v, f, n, d = nm.extract_geometry(model, "cuda", SimpleNamespace(limit=LIMIT, res=256, iso_level=32.0, **kw))
    return (v.numpy(), f.numpy(), n.numpy()), d


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["plain", "super_sampling", "network_normals"])
def test_extract_geometry_256(models, variant, capsys):
    model = models["lego"]
    engine(model, "exact")
    kw = dict(plain={}, super_sampling=dict(super_sampling=3), network_normals=dict(network_normals=True))[variant]
    dense, dd = geometry(model, **kw)
    sparse, sd = geometry(model, sparse_sweep=True, **kw)
    assert "sparse sweep (block 8):" in capsys.readouterr().out
    ev = np.isfinite(sd)
    assert np.array_equal(sd[ev].view(np.int32), dd[ev].view(np.int32)) and 0 < ev.sum() < ev.size
    vkeep, fkeep = S.mesh_subset(dense, sparse)
    kept, missing = S.whole_components(dense, vkeep, fkeep)
    assert len(kept) >= 1 and (len(missing) == 0 or kept[0] > missing[0])       # the largest dense component is there in full
    with capsys.disabled():
        print(f"\nlego 256^3 {variant}: {int(ev.sum())} of {ev.size} points; dense {len(dense[1])} faces in {len(kept) + len(missing)} "
              f"components; missing {len(missing)} components, {int(missing.sum())} faces, largest {missing[:3].tolist()}")
    if variant != "plain":
        return
    # B = 4 and 16 through the same route; with min_component_faces = 256 the floaters the sparse sweep misses are removed
    # from the dense mesh too
    for B in (4, 16):
        sp, _ = geometry(model, sparse_sweep=True, sparse_block=B)
        S.whole_components(dense, *S.mesh_subset(dense, sp))
    fd, _ = geometry(model, min_component_faces=256)
    fs, _ = geometry(model, sparse_sweep=True, min_component_faces=256)
    if len(missing) == 0 or missing[0] < 256:
        for a, b in zip(fd, fs):
            assert np.array_equal(a.view(np.int32), b.view(np.int32))
        verdict = "every missing component has fewer than 256 faces: the filtered meshes are equal"
    else:
        S.whole_components(fd, *S.mesh_subset(fd, fs))
        verdict = f"a missing component has {int(missing[0])} faces: the filtered sparse mesh is whole components of the filtered dense one"
    with capsys.disabled():
        print(f"min_component_faces = 256: {verdict}")


@pytest.mark.gpu
def test_more_than_one_slab_is_refused(models):
    from nerfmeshes_b200 import parallel as par
    A = SimpleNamespace(limit=LIMIT, res=64, iso_level=32.0, sparse_sweep=True)
    fresh = lambda key, numel, dtype, dev: torch.empty(numel, dtype=dtype, device=dev)
    with pytest.raises(NotImplementedError, match="one slab"):
        par._extract_mesh(models["lego"], A, 0, 2, None, fresh)
    # one slab through the sharded entry point: the arrays of extract_geometry (at 64^3 the lattice statistics clamp the iso
    # level differently from the dense ones, so the dense mesh is not the yard-stick here)
    import nerfmeshes_b200 as nm
    v0, f0, n0, _ = nm.extract_geometry(models["lego"], "cuda", A)
    v1, f1, n1, _ = par.extract_geometry_sharded(models["lego"], A, group=par.SINGLE)
    assert len(f0) > 0 and torch.equal(v0, v1) and torch.equal(f0, f1) and torch.equal(n0, n1)


@pytest.mark.gpu
def test_error_paths_on_the_device(models):
    from nerfmeshes_b200 import NmError
    from nerfmeshes_b200.engine import Engine, RenderSettings
    eng = engine(models["lego"], "exact")
    shape = (40, 40, 40)
    out = torch.zeros(shape, dtype=torch.float32, device=eng.device)
    other = torch.zeros(shape, dtype=torch.float32, device=eng.device)
    before = eng.launch_count()
    with pytest.raises(NmError, match="not one of 4, 8, 16"):
        eng.sparse_lattice(tables(shape), 7, out)
    assert eng.launch_count() == before                        # a rejected call launches nothing
    eng.sparse_lattice(tables(shape), 8, out)
    for bad in (lambda: eng.sparse_run(tables(shape), 4, 32.0, out), lambda: eng.sparse_run(tables(shape), 8, 32.0, other),
                lambda: eng.sparse_run(tables((40, 40, 41)), 8, 32.0, torch.zeros((40, 40, 41), device=eng.device))):
        with pytest.raises(NmError, match="call nm_sparse_sweep_lattice with the same grid, block and volume first"):
            bad()
    eng.sparse_run(tables(shape), 8, 32.0, out)                 # the handle works
    bare = Engine({}, None, RenderSettings())                   # no weights loaded
    with pytest.raises(NmError, match="weights of network 0 not loaded"):
        bare.sparse_lattice(tables(shape), 8, out)
    bare.close()
    eng.check_flags()
