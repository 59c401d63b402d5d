"""Super-sampled marching cubes (mesh_nerf.py:95-128, DESIGN 4.3): the coarse grid's topology, faces, normals and centre
vertices, with every edge vertex placed from s extra samples along its edge.  The definition is dense (three volumes,
each refined along one axis); the CUDA path (nm_mc_emit_ss) evaluates the network only at the crossed edges' samples.
  * CPU: the dense definition (tests/mc_ss_oracle.c on top of the procedural oracle) on analytic fields, a hand-built edge that
    crosses three times, and sharded calls;
  * GPU: nm_mc_emit_ss equals the oracle fed with grid_sigma volumes, bit for bit, at every precision; chunking, sparse
    evaluation, shards, convergence on the lego network, and the mesh export end to end.
Parity with PyMarchingCubes' marching_cubes_super_sampling is unpinned: it is not installable here."""
import os

import numpy as np
import pytest
import torch

from oracle import mc
from _mc_ss_ref import marching_cubes_ss

LIMIT = 1.2


def lin(n, s=0):
    return torch.linspace(-LIMIT, LIMIT, n + (n - 1) * s).numpy()


def sample(fn, shape, s):
    """coarse volume and the three fine volumes of fn (float32) on the linspace grid of `shape`"""
    def grid(a, b, c):
        X, Y, Z = np.meshgrid(a.astype(np.float64), b.astype(np.float64), c.astype(np.float64), indexing="ij")
        return fn(X, Y, Z).astype(np.float32)
    l = [lin(n) for n in shape]
    f = [lin(n, s) for n in shape]
    return grid(*l), (grid(f[0], l[1], l[2]), grid(l[0], f[1], l[2]), grid(l[0], l[1], f[2]))


FIELDS = {
    "sphere": lambda X, Y, Z: 0.8 - np.sqrt(X * X + Y * Y + Z * Z),
    "torus": lambda X, Y, Z: 0.25 - np.sqrt((np.sqrt(X * X + Y * Y) - 0.7) ** 2 + Z * Z),
    "two_spheres": lambda X, Y, Z: np.maximum(0.35 - np.sqrt((X - 0.5) ** 2 + Y * Y + Z * Z),
                                              0.35 - np.sqrt((X + 0.5) ** 2 + Y * Y + Z * Z)),
    "quadric": lambda X, Y, Z: 0.64 - (X * X + Y * Y + Z * Z),        # R^2 - |x|^2: curved along every edge
}


def edge_vertices(v):
    """(mask, axis, lower grid point) of the vertices that lie on a grid edge: exactly two integral coordinates (centre
    vertices have none; an edge vertex that rounded onto a grid point is left out)."""
    integral = v == np.round(v)
    mask = integral.sum(1) == 2
    axis = np.argmin(integral, 1)
    lo = np.floor(v).astype(np.int64)
    return mask, axis, lo


def check_refined(v0, v, f0, f, n0, n):
    """faces and normals bit-identical; only edge vertices move, along their axis, inside their edge"""
    assert np.array_equal(f, f0) and np.array_equal(n, n0) and v.shape == v0.shape
    changed = v != v0
    mask, axis, lo = edge_vertices(v0)
    assert changed.sum(1).max(initial=0) <= 1
    rows = np.nonzero(changed.any(1))[0]
    assert mask[rows].all(), "a centre vertex moved"
    ax = axis[rows]
    assert np.array_equal(np.argmax(changed[rows], 1), ax), "a vertex moved off its axis"
    new, old = v[rows, ax], v0[rows, ax]
    base = np.floor(np.minimum(new, old))
    assert (np.maximum(new, old) <= base + 1).all(), "a vertex left its edge"


# ----------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("name", ["sphere", "torus", "two_spheres", "noise"])
def test_oracle_ss_s0_equals_oracle(name):
    if name == "noise":
        vol = np.random.default_rng(3).standard_normal((23, 19, 30)).astype(np.float32)
        iso, fines = 0.1, (vol, vol, vol)
    else:
        vol, fines = sample(FIELDS[name], (40, 40, 40), 0)
        iso = 0.0
    ref = mc.marching_cubes(vol, iso)
    out = marching_cubes_ss(vol, iso, 0, *fines)
    for a, b in zip(ref, out):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("s", [1, 3, 7])
@pytest.mark.parametrize("name", ["sphere", "torus", "two_spheres", "quadric"])
def test_oracle_ss_analytic_fields(name, s):
    vol, fines = sample(FIELDS[name], (33, 30, 36), s)
    v0, f0, n0 = mc.marching_cubes(vol, 0.0)
    v, f, n = marching_cubes_ss(vol, 0.0, s, *fines)
    check_refined(v0, v, f0, f, n0, n)
    assert (v != v0).any()


def _surface_error(v, shape, R=0.8):
    h = np.array([2 * LIMIT / (n - 1) for n in shape])
    x = -LIMIT + v.astype(np.float64) * h
    return np.abs(np.sqrt((x * x).sum(1)) - R) / h.max()       # in voxels


def test_oracle_ss_converges_on_a_curved_field():
    """R^2 - |x|^2 is quadratic along every edge: linear interpolation misses the root by O(h^2 curvature); with s = 3 the
    interpolation interval is 4x shorter, so the error shrinks ~16x.  Measured (24^3 grid, R = 0.8): worst 0.0163 voxel
    at s = 0, 0.00102 at s = 3 (ratio 0.0625); asserted: <= 0.1x."""
    shape = (24, 24, 24)
    vol, _ = sample(FIELDS["quadric"], shape, 0)
    v0, _, _ = mc.marching_cubes(vol, 0.0)
    mask, _, _ = edge_vertices(v0)
    e0 = _surface_error(v0[mask], shape).max()
    _, fines = sample(FIELDS["quadric"], shape, 3)
    v3, _, _ = marching_cubes_ss(vol, 0.0, 3, *fines)
    e3 = _surface_error(v3[mask], shape).max()
    assert e0 > 1e-3
    assert e3 <= 0.1 * e0, (e0, e3)


def test_oracle_ss_first_of_three_crossings():
    """A 2x2x2 volume whose (0,0,0)->(0,0,1) edge, sampled with s = 3, crosses iso three times: the vertex is placed in the
    first crossing's sub-interval [0, 1/4]."""
    iso = np.float32(0.5)
    vol = np.zeros((2, 2, 2), np.float32)
    vol[0, 0, 0] = 1.0
    s = 3
    xf = np.zeros((5, 2, 2), np.float32)
    yf = np.zeros((2, 5, 2), np.float32)
    zf = np.zeros((2, 2, 5), np.float32)
    zf[0, 0, 1:4] = [0.2, 0.9, 0.1]                   # 1.0 | 0.2 0.9 0.1 | 0.0: crossings in sub-intervals 0, 1 and 2
    v0, f0, n0 = mc.marching_cubes(vol, iso)
    v, f, n = marching_cubes_ss(vol, iso, s, xf, yf, zf)
    assert np.array_equal(f, f0) and np.array_equal(n, n0) and v.shape == (3, 3)
    eps = float(np.finfo(np.float32).eps)
    w0 = 1.0 / (eps + abs(1.0 - float(iso)))
    w1 = 1.0 / (eps + abs(float(np.float32(0.2)) - float(iso)))
    want = np.float32((0 + w1 / (w0 + w1)) / (s + 1))
    zrow = np.nonzero((v[:, 0] == 0) & (v[:, 1] == 0) & (v[:, 2] > 0))[0]
    assert zrow.size == 1 and v[zrow[0], 2] == want and 0 < want < 0.25
    # the x and y edges: samples 1.0 | 0 0 0 | 0 cross in the first sub-interval too
    for a in (0, 1):
        row = np.nonzero(v[:, a] > 0)[0]
        assert row.size == 1 and 0 < v[row[0], a] < 0.25


@pytest.mark.parametrize("s", [1, 3])
def test_oracle_ss_shards_concatenate(s):
    rng = np.random.default_rng(11)
    shape = (21, 18, 40)
    vol = rng.standard_normal(shape).astype(np.float32)
    fines = [rng.standard_normal(tuple((n - 1) * (s + 1) + 1 if b == a else n for b, n in enumerate(shape))).astype(np.float32)
             for a in range(3)]
    iso, n0 = 0.05, shape[0]
    v, f, n = marching_cubes_ss(vol, iso, s, *fines)
    cuts = [0, 6, 13, n0]
    vs, fs, ns, base = [], [], [], 0
    for own0, own1 in zip(cuts[:-1], cuts[1:]):
        buf0, buf1 = max(own0 - 1, 0), min(own1 + 2, n0)
        ov, of, on = marching_cubes_ss(vol[buf0:buf1], iso, s, *fines, x_off=buf0, g_nx=n0, own=(own0 - buf0, own1 - buf0),
                                       v_base=base)
        vs.append(ov); fs.append(of); ns.append(on)
        base += ov.shape[0]
    assert np.array_equal(np.concatenate(vs), v) and np.array_equal(np.concatenate(fs), f)
    assert np.array_equal(np.concatenate(ns), n)


# ----------------------------------------------------------------------------------------------------------------- GPU
PREC = {"exact": 0, "fast": 1, "fp32": 2}


@pytest.fixture(scope="module")
def lego_model():
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import LEGO_CFG
    return nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval()


def engine(model, prec):
    model.precision = PREC[prec]
    return model._engine()


def volumes(eng, shape, s):
    """coarse and fine density volumes of the lego fine net from grid_sigma, with the super-sampling tables"""
    from nerfmeshes_b200 import super_sampling_tables
    lins, fines = super_sampling_tables(LIMIT, shape, s)
    coarse = eng.grid_sigma(lins)
    fv = [eng.grid_sigma([fines[a] if b == a else lins[b] for b in range(3)]) for a in range(3)]
    return coarse, fv, lins, fines


def iso_of(eng, vol):
    import nerfmeshes_b200 as nm

    class A:
        iso_level = 32.0
    return float(nm.extract_iso_level(vol, A, eng))


def emit_ss(eng, vol, iso, s, lins, fines):
    n0 = vol.shape[0]
    nv, nt = eng.mc_count(vol, iso, 0, n0, 0, n0)
    v, f, n = eng.mc_emit_ss(vol, iso, 0, n0, 0, n0, nv, nt, 0, s, lins, fines)
    return v.cpu().numpy(), f.cpu().numpy(), n.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["exact", "fast", "fp32"])
def test_point_sigma_equals_grid_sigma(lego_model, prec):
    """The precondition of bit-for-bit parity: the fused MLP computes each point's row independently of its position in
    the launch, so sigma at explicit points equals the grid sweep's sigma at the same coordinates."""
    eng = engine(lego_model, prec)
    shape, s = (12, 10, 9), 3
    coarse, fv, lins, fines = volumes(eng, shape, s)
    for a in range(3):
        axes = [fines[b] if b == a else lins[b] for b in range(3)]
        X, Y, Z = torch.meshgrid(*axes, indexing="ij")
        pts = torch.stack([X, Y, Z], -1).reshape(-1, 3).cuda()
        sig = eng.point_mlp(1, pts, None, sigma_only=True)
        assert torch.equal(sig.reshape(fv[a].shape), fv[a]), f"axis {a}"


CASES = [(shape, s, prec) for shape in [(40, 40, 40), (37, 33, 45), (20, 18, 33)] for s in (1, 2, 3, 7)
         for prec in ("exact", "fast")] + [((17, 15, 19), 3, "fp32")]


@pytest.mark.gpu
@pytest.mark.parametrize("shape,s,prec", CASES)
def test_cuda_ss_equals_oracle(lego_model, shape, s, prec):
    eng = engine(lego_model, prec)
    coarse, fv, lins, fines = volumes(eng, shape, s)
    iso = iso_of(eng, coarse)
    v, f, n = emit_ss(eng, coarse, iso, s, lins, fines)
    ov, of, on = marching_cubes_ss(coarse.cpu().numpy(), iso, s, *[x.cpu().numpy() for x in fv])
    assert v.shape[0] > 50
    assert np.array_equal(v, ov) and np.array_equal(f, of) and np.array_equal(n, on)


@pytest.mark.gpu
def test_cuda_ss_s0_equals_emit(lego_model):
    eng = engine(lego_model, "exact")
    coarse, _, lins, fines = volumes(eng, (37, 33, 45), 0)
    iso = iso_of(eng, coarse)
    v, f, n = emit_ss(eng, coarse, iso, 0, lins, fines)
    n0 = coarse.shape[0]
    nv, nt = eng.mc_count(coarse, iso, 0, n0, 0, n0)
    gv, gf, gn = eng.mc_emit(coarse, iso, 0, n0, 0, n0, nv, nt, 0)
    assert np.array_equal(v, gv.cpu().numpy()) and np.array_equal(f, gf.cpu().numpy()) and np.array_equal(n, gn.cpu().numpy())


@pytest.mark.gpu
def test_cuda_ss_shards(lego_model):
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import parallel
    eng = engine(lego_model, "exact")
    shape, s = (21, 18, 40), 3
    coarse, fv, lins, fines = volumes(eng, shape, s)
    iso = iso_of(eng, coarse)
    v, f, n = emit_ss(eng, coarse, iso, s, lins, fines)
    vol, fvn = coarse.cpu().numpy(), [x.cpu().numpy() for x in fv]
    n0 = shape[0]
    cuts = [0, 6, 13, n0]
    vs, fs, ns, base = [], [], [], 0
    for own0, own1 in zip(cuts[:-1], cuts[1:]):
        buf0, buf1 = max(own0 - 1, 0), min(own1 + 2, n0)
        buf = coarse[buf0:buf1].contiguous()
        nv, nt = eng.mc_count(buf, iso, buf0, n0, own0 - buf0, own1 - buf0)
        gv, gf, gn = eng.mc_emit_ss(buf, iso, buf0, n0, own0 - buf0, own1 - buf0, nv, nt, base, s, lins, fines)
        ov, of, on = marching_cubes_ss(vol[buf0:buf1], iso, s, *fvn, x_off=buf0, g_nx=n0, own=(own0 - buf0, own1 - buf0),
                                       v_base=base)
        assert np.array_equal(gv.cpu().numpy(), ov) and np.array_equal(gf.cpu().numpy(), of)
        assert np.array_equal(gn.cpu().numpy(), on)
        vs.append(gv.cpu()); fs.append(gf.cpu()); ns.append(gn.cpu())
        base += nv
    assert np.array_equal(torch.cat(vs).numpy(), v) and np.array_equal(torch.cat(fs).numpy(), f)
    assert np.array_equal(torch.cat(ns).numpy(), n)

    class A:
        limit, res, iso_level, super_sampling = LIMIT, 24, 32.0, 3
    sv, sf, sn, _ = parallel.extract_geometry_sharded(lego_model, A, group=parallel.SINGLE)
    mv, mf, mn, _ = nm.extract_geometry(lego_model, "cuda", A)
    assert torch.equal(sv, mv) and torch.equal(sf, mf) and torch.equal(sn, mn)


@pytest.mark.gpu
def test_cuda_ss_chunking(lego_model, monkeypatch):
    """Chunks of 37 points (a multiple of neither s nor 64): samples of one vertex straddle network launches."""
    eng = engine(lego_model, "exact")
    shape, s = (40, 40, 40), 7
    coarse, _, lins, fines = volumes(eng, shape, s)
    iso = iso_of(eng, coarse)
    ref = emit_ss(eng, coarse, iso, s, lins, fines)
    for chunk in ("37", "5"):
        monkeypatch.setenv("NM_SS_CHUNK_POINTS", chunk)
        out = emit_ss(eng, coarse, iso, s, lins, fines)
        assert all(np.array_equal(a, b) for a, b in zip(ref, out)), chunk


@pytest.mark.gpu
@pytest.mark.parametrize("s", [1, 3])
def test_cuda_ss_is_sparse(lego_model, s):
    """The network sees s points per owned vertex (centre vertices padded) and nothing else."""
    eng = engine(lego_model, "exact")
    coarse, _, lins, fines = volumes(eng, (40, 40, 40), s)
    iso = iso_of(eng, coarse)
    n0 = coarse.shape[0]
    nv, nt = eng.mc_count(coarse, iso, 0, n0, 0, n0)
    eng.set_timing(True)
    try:
        eng.mc_emit_ss(coarse, iso, 0, n0, 0, n0, nv, nt, 0, s, lins, fines)
        torch.cuda.synchronize()
        _, points, launches = eng.mlp_time_ms()
    finally:
        eng.set_timing(False)
    assert points == s * nv and launches >= 1
    assert points < n0 ** 3


@pytest.mark.gpu
def test_cuda_ss_converges_on_the_network(lego_model):
    """Distances to the s = 63 positions, over edges whose 63 inner samples cross iso exactly once (so s = 0, 3 and 63
    place the vertex at the same crossing).  Measured on the lego fine net at 40^3, iso 32, exact precision (H100 80GB
    HBM3, 700 W): median 0.243 voxel at s = 0, 0.0526 at s = 3 (ratio 0.216) over 4074 edges; asserted: <= 0.3x.  The
    kernel is deterministic, so the ratio only moves with the weights; sigma is far from linear over one voxel, which is
    why s = 0 misses by a quarter voxel and s = 3 does not reach the 1/16 of a quadratic field."""
    eng = engine(lego_model, "exact")
    shape = (40, 40, 40)
    from nerfmeshes_b200 import super_sampling_tables
    coarse, fv63, lins, fines63 = volumes(eng, shape, 63)
    iso = iso_of(eng, coarse)
    v0, _, _ = emit_ss(eng, coarse, iso, 0, lins, super_sampling_tables(LIMIT, shape, 0)[1])
    _, fines3 = super_sampling_tables(LIMIT, shape, 3)
    v3, _, _ = emit_ss(eng, coarse, iso, 3, lins, fines3)
    v63, _, _ = emit_ss(eng, coarse, iso, 63, lins, fines63)
    # crossings per edge along each axis: coarse ends + the 63 inner fine samples
    ncross = []
    for a in range(3):
        c = coarse.movedim(a, 0)
        f = fv63[a].movedim(a, 0)
        inner = f[:-1].reshape(c.shape[0] - 1, 64, *c.shape[1:])[:, 1:]
        seq = torch.cat([c[:-1, None], inner, c[1:, None]], 1) > iso
        ncross.append((seq[:, 1:] != seq[:, :-1]).sum(1).movedim(0, a).cpu().numpy())
    mask, axis, lo = edge_vertices(v0)
    rows = np.nonzero(mask)[0]
    single = np.array([ncross[axis[r]][tuple(lo[r])] == 1 for r in rows])
    rows = rows[single]
    assert rows.size > 500
    ax = axis[rows]
    d0 = np.abs(v0[rows, ax].astype(np.float64) - v63[rows, ax])
    d3 = np.abs(v3[rows, ax].astype(np.float64) - v63[rows, ax])
    m0, m3 = np.median(d0), np.median(d3)
    print(f"median distance to s=63: s=0 {m0:.3g}, s=3 {m3:.3g} (ratio {m3 / m0:.3g}) over {rows.size} edges")
    assert m3 <= 0.3 * m0, (m0, m3)


@pytest.mark.gpu
def test_extract_geometry_super_sampling_end_to_end(lego_model, tmp_path):
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import mesh
    from nerfmeshes_b200.engine import Engine, RenderSettings

    class A:
        limit, res, iso_level, super_sampling = LIMIT, 40, 32.0, 0
        save_dir, mesh_name, cache_name = str(tmp_path), "m0.obj", None
        use_cached_mesh, override_cache_mesh, no_view_dependence = False, False, True
    engine(lego_model, "exact")
    v0, t0, n0, d0 = nm.extract_geometry(lego_model, "cuda", A)
    A.super_sampling = 3
    v3, t3, n3, d3 = nm.extract_geometry(lego_model, "cuda", A)
    w3 = nm.extract_geometry_with_super_sampling(lego_model, "cuda", A)
    assert torch.equal(t3, t0) and torch.equal(n3, n0) and np.array_equal(d3, d0)
    assert v3.shape == v0.shape and not torch.equal(v3, v0) and torch.equal(w3[0], v3)
    # OBJ export and the cache of the refined mesh
    A.super_sampling, A.mesh_name = 0, "m0.obj"
    p0 = mesh.export_marching_cubes(lego_model, A)
    A.super_sampling, A.mesh_name, A.cache_name, A.use_cached_mesh = 3, "m3.obj", "c3.pt", True
    p3 = mesh.export_marching_cubes(lego_model, A)
    lines = lambda p: [ln.split(" ", 1)[0] for ln in open(p).read().splitlines()]
    l0, l3 = lines(p0), lines(p3)
    assert len(l0) == len(l3) and all(l0.count(k) == l3.count(k) for k in ("v", "vn", "f"))
    cached = torch.load(os.path.join(str(tmp_path), "c3.pt"), weights_only=False)
    assert torch.equal(cached[0], v3) and torch.equal(cached[1], t3)
    A.mesh_name = "m3b.obj"
    p3b = mesh.export_marching_cubes(lego_model, A)               # served from the cache
    assert open(p3b).read() == open(p3).read()
    # invalid inputs fail before any launch
    eng = lego_model._engine()
    dens = eng.grid_sigma(mesh.super_sampling_tables(LIMIT, 12, 0)[0])
    iso = iso_of(eng, dens)
    nv, nt = eng.mc_count(dens, iso, 0, 12, 0, 12)
    for s in (-1, 65):
        lins, fines = mesh.super_sampling_tables(LIMIT, 12, max(s, 0))
        before = eng.launch_count()
        with pytest.raises(nm.NmError):
            eng.mc_emit_ss(dens, iso, 0, 12, 0, 12, nv, nt, 0, s, lins, fines)
        assert eng.launch_count() == before
    fresh = Engine(lego_model._nets()[0].arch, lego_model._nets()[1].arch, RenderSettings())
    fresh.load_weights(1, lego_model._nets()[1].state_dict())
    lins, fines = mesh.super_sampling_tables(LIMIT, 12, 3)
    with pytest.raises(nm.NmError):
        fresh.mc_emit_ss(dens, iso, 0, 12, 0, 12, max(nv, 1), nt, 0, 3, lins, fines)
    assert fresh.launch_count() == 0
    fresh.close()
