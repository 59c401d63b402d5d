"""Marching cubes (a15).  The reference's implementation is scikit-image 0.17.2's Lewiner extension, which is absent here:
PARITY UNPINNED at that seam (SURVEY 8c).  What is tested instead:
  * CPU: the procedural C oracle (oracle/mc_oracle.c) on analytic fields — closed manifold, Euler characteristic, vertices
    on straddling grid edges within half a voxel of the surface — and on fields full of ambiguous cells (noise, saddles):
    manifoldness, Lewiner's triangle counts per sub-case, centre vertices exactly in the sub-cases that use them;
  * CPU: the generated lookup tables of the CUDA kernels (tools/gen_mc_tables.py) against the oracle's procedural resolution,
    entry by entry — two independent implementations (python generator vs C) of the same rules;
  * CPU: ownership sharding — concatenated slab outputs ARE the single-volume arrays (vertices, normals, faces);
  * GPU: the CUDA kernels equal the oracle array for array, bit for bit, including sharded calls.
tools/diff_skimage.py is the hook that diffs this against a real scikit-image where one is installed."""
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import mc


def fields(n=40):
    g = np.linspace(-1.2, 1.2, n, dtype=np.float32)
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    sphere = (0.8 - np.sqrt(X * X + Y * Y + Z * Z)).astype(np.float32)
    torus = (0.25 - np.sqrt((np.sqrt(X * X + Y * Y) - 0.7) ** 2 + Z * Z)).astype(np.float32)
    two = np.maximum(0.35 - np.sqrt((X - 0.5) ** 2 + Y * Y + Z * Z), 0.35 - np.sqrt((X + 0.5) ** 2 + Y * Y + Z * Z)).astype(np.float32)
    return dict(sphere=(sphere, 2), torus=(torus, 0), two_spheres=(two, 4)), g


def noise(shape=(24, 20, 28), seed=0, scale=1.0):
    return (np.random.default_rng(seed).standard_normal(shape) * scale).astype(np.float32)


def edge_stats(f):
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    und, cnt = np.unique(np.sort(e, 1), axis=0, return_counts=True)
    _, dcnt = np.unique(e, axis=0, return_counts=True)
    return und.shape[0], cnt, dcnt


@pytest.mark.parametrize("name", ["sphere", "torus", "two_spheres"])
def test_oracle_topology_and_geometry(name):
    fs, g = fields()
    vol, euler = fs[name]
    n = vol.shape[0]
    v, f, nrm = mc.marching_cubes(vol, 0.0)
    n_edges, cnt, dcnt = edge_stats(f)
    assert set(cnt) == {2}, "closed manifold: every edge shared by exactly two triangles"
    assert dcnt.max() == 1, "consistent orientation"
    assert v.shape[0] - n_edges + f.shape[0] == euler
    # every vertex lies on a grid edge whose end points straddle the iso value, strictly between them
    frac = v - np.floor(v)
    on_edge = (frac > 0).sum(1)
    assert on_edge.max() <= 1
    lo = np.floor(v).astype(int)
    hi = np.minimum(lo + (frac > 0), n - 1)
    a, b = vol[lo[:, 0], lo[:, 1], lo[:, 2]], vol[hi[:, 0], hi[:, 1], hi[:, 2]]
    assert bool(((a > 0) != (b > 0))[on_edge == 1].all())
    # within half a voxel of the analytic surface, and (signed-distance fields) the weighted mean IS the linear root
    P = v / (n - 1) * 2.4 - 1.2
    h = 2.4 / (n - 1)
    if name == "sphere":
        assert np.abs(np.linalg.norm(P, axis=1) - 0.8).max() < 0.5 * h
        out = P / np.linalg.norm(P, axis=1, keepdims=True)
        assert (np.sum(nrm * out, 1)).min() > 0.99                  # unit normals point to decreasing values (outward)
        fn = np.cross(P[f[:, 1]] - P[f[:, 0]], P[f[:, 2]] - P[f[:, 0]])
        assert (np.sum(fn * P[f].mean(1), 1) > 0).all()             # triangle winding agrees with the normals
    np.testing.assert_allclose(np.linalg.norm(nrm, axis=1), 1.0, atol=1e-6)


def test_vertex_positions_follow_the_skimage_formula():
    """x + w1/(w0+w1), w = 1/(FLT_EPSILON + |v - iso|) in double, stored as float32 (SURVEY Appendix F)."""
    vol = noise((6, 5, 7), seed=3)
    iso = 0.05
    v, f, n = mc.marching_cubes(vol, iso)
    eps = float(np.finfo(np.float32).eps)
    frac = v - np.floor(v)
    checked = 0
    for p in v[(frac > 0).sum(1) == 1]:
        a = int(np.argmax(p - np.floor(p) > 0))
        lo = np.floor(p).astype(int)
        hi = lo.copy()
        hi[a] += 1
        w0 = 1.0 / (eps + abs(float(vol[tuple(lo)]) - np.float64(np.float32(iso))))
        w1 = 1.0 / (eps + abs(float(vol[tuple(hi)]) - np.float64(np.float32(iso))))
        assert np.float32(lo[a] + w1 / (w0 + w1)) == p[a]
        checked += 1
    assert checked > 50


def test_tables_equal_the_procedural_oracle():
    """Every (sign mask, face decisions, tunnel) variant: the generated CUDA tables vs the oracle's run-time resolution."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_mc_tables as G
    n_variants = 0
    for m in range(256):
        case, mu, amb, vs = G.variants(m)
        for J, v in enumerate(vs):
            for tun in (0, 1):
                o = mc.cell_variant(m, J, tun)
                tris = v["tri_tunnel"] if (tun and v["tri_tunnel"] is not None) else v["tri_none"]
                assert o["tris"] == [x for t in tris for x in t], (m, J, tun)
                assert (o["itest"], o["tunnel_if_I"], o["faces"], o["mu_pos"]) == (v["itest"], v["tunnel_if_I"], amb, int(mu))
                n_variants += 1
    assert n_variants == 2 * 656
    # the header on disk is what the generator produces now
    l1, l2, l3 = G.build()
    hdr = open(os.path.join(ROOT, "nerfmeshes_b200", "csrc", "nm_mc_tables.h")).read()
    assert f"#define NM_MC_N_L2 {len(l2)}" in hdr and f"#define NM_MC_N_L3 {len(l3)}" in hdr


def test_lewiner_subcases_triangle_counts_and_centre_vertices():
    """Lewiner's tilings: triangle count per sub-case, and the c-vertex exactly in 6.1.2, 7.3, 10.2, 12.2, 13.3, 13.4."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_mc_tables as G
    want = {3: {(0,): (2, None), (1,): (4, None)}, 4: {(0,): (2, 6)}, 6: {(0,): (3, 9), (1,): (5, None)},
            7: {(0,): (3, None), (1,): (5, None), (2,): (9, None), (3,): (5, 9)},
            10: {(0,): (4, 8), (1,): (8, None), (2,): (4, None)}, 12: {(0,): (4, 8), (1,): (8, None), (2,): (4, None)}}
    with_c = {(6, 0, True), (7, 2, False), (10, 1, False), (12, 1, False)}
    for m in range(256):
        case, mu, amb, vs = G.variants(m)
        for J, v in enumerate(vs):
            k = bin(J).count("1")
            if case in want:
                none, tun = want[case][(k,)]
                assert len(v["tri_none"]) == none and (v["tri_tunnel"] is None) == (tun is None)
                if tun is not None:
                    assert len(v["tri_tunnel"]) == tun
                assert v["c_none"] == ((case, k, False) in with_c) and v["c_tunnel"] == ((case, k, True) in with_c)
            elif case == 13:
                sizes = sorted(len(lp) for lp in G.trace_loops(m, {f: bool((J >> i) & 1) for i, f in enumerate(amb)}))
                assert v["c_none"] == (max(sizes) >= 8)                          # 13.3 (9-loop), 13.4 (12-loop)
                assert len(v["tri_none"]) == {(3, 3, 3, 3): 4, (3, 3, 6): 6, (3, 9): 10, (12,): 12, (6, 6): 8}[tuple(sizes)]
                if v["tri_tunnel"] is not None:
                    assert sizes == [3, 3, 6] and len(v["tri_tunnel"]) == 10 and not v["c_tunnel"]      # 13.5.2
            else:
                assert not amb and v["tri_tunnel"] is None and not v["c_none"]


@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_on_ambiguous_fields_is_watertight(seed):
    """Noise is full of ambiguous faces / interior ambiguities (all of Lewiner's sub-cases occur): the mesh must still be a
    consistently oriented manifold (boundary only on the volume border), with centre vertices strictly inside their cells."""
    vol = noise(seed=seed)
    v, f, n, st = mc.marching_cubes(vol, 0.1, stats=True)
    n_edges, cnt, dcnt = edge_stats(f)
    assert set(cnt) <= {1, 2} and dcnt.max() == 1
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1)
    und, c = np.unique(e, axis=0, return_counts=True)
    border = und[c == 1]
    P = v[border.reshape(-1)]
    on_border = ((P == 0) | (P == np.array(vol.shape) - 1)).any(1)
    assert on_border.all(), "open edges away from the volume border"
    assert sum(c for k, c in st.items() if "(c)" in k) > 20 and any(k.startswith("4.2") for k in st)
    centre = v[((v - np.floor(v)) > 0).sum(1) == 3]
    sure = sum(c for k, c in st.items() if "(c)" in k and "/" not in k and "[" not in k)     # labels that always use the c-vertex
    maybe = sum(c for k, c in st.items() if "(c)" in k)
    assert sure <= centre.shape[0] <= maybe
    cell = np.floor(centre)
    assert ((centre - cell) > 0).all() and ((centre - cell) < 1).all()
    assert f.max() < v.shape[0] and np.isfinite(v).all() and np.isfinite(n).all()


def test_saddle_cell_resolution_follows_the_face_test():
    """One cell, case 3 (two positive corners diagonal on a face): the asymptotic decider A*C - B*D picks 3.1 (2 triangles,
    corners separated) or 3.2 (4 triangles, joined) — the classic 256-case table always separates."""
    vol = -np.ones((2, 2, 2), np.float32)
    vol[0, 0, 0], vol[0, 1, 1] = 1.0, 1.0            # diagonal on the axis-0 = 0 face: A*C - B*D = 1 - 1 = 0 -> tie band -> joined
    v, f, n = mc.marching_cubes(vol, 0.0)
    assert f.shape[0] == 4
    vol[0, 0, 0], vol[0, 1, 1] = 0.5, 0.5            # 0.25 - 1 < 0: positives weaker than negatives -> separated
    v, f, n = mc.marching_cubes(vol, 0.0)
    assert f.shape[0] == 2
    vol[0, 0, 0], vol[0, 1, 1] = 3.0, 3.0            # 9 - 1 > 0 -> joined
    v, f, n = mc.marching_cubes(vol, 0.0)
    assert f.shape[0] == 4 and v.shape[0] == 6


def test_oracle_shards_concatenate_to_the_single_volume_arrays():
    """x-slab sharding by ownership (SURVEY 8e): with halo planes in the buffer, concatenated shard outputs equal the
    single-volume arrays bit for bit — vertices, normals and faces (globally consistent ids, no duplicates)."""
    for vol, iso in ((fields(36)[0]["torus"][0], 0.0), (noise((19, 9, 11), seed=4), 0.2)):
        n0 = vol.shape[0]
        v, f, n = mc.marching_cubes(vol, iso)
        for cuts in ([0, 7, 8, n0 - 2, n0], [0, n0 // 2, n0]):
            vs, fs, ns, base = [], [], [], 0
            for own0, own1 in zip(cuts[:-1], cuts[1:]):
                last = own1 == n0
                if last:
                    own1 = n0
                elif own1 == cuts[-1]:
                    pass
                buf0, buf1 = max(own0 - 1, 0), min(own1 + 2, n0)
                pv, pf, pn = mc.marching_cubes(vol[buf0:buf1], iso, x_off=buf0, g_nx=n0, own=(own0 - buf0, own1 - buf0), v_base=base)
                vs.append(pv); fs.append(pf); ns.append(pn)
                base += pv.shape[0]
            assert np.array_equal(np.concatenate(vs), v) and np.array_equal(np.concatenate(ns), n)
            assert np.array_equal(np.concatenate(fs), f)


def test_ragged_and_empty_inputs():
    v, f, n = mc.marching_cubes(np.zeros((5, 4, 3), np.float32), 0.5)
    assert v.shape == (0, 3) and f.shape == (0, 3)
    vol = np.zeros((2, 2, 2), np.float32)
    vol[0, 0, 0] = 1.0
    v, f, n = mc.marching_cubes(vol, 0.5)
    assert v.shape == (3, 3) and f.shape == (1, 3)
    np.testing.assert_allclose(sorted(v.sum(1)), [0.5, 0.5, 0.5], atol=1e-6)


# ----------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["sphere", "torus", "two_spheres", "noise", "noise_big", "ragged", "line33", "lego"])
def test_cuda_equals_oracle_bit_for_bit(name):
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200.nerf_api import _engine
    if name == "noise":
        vol, iso = noise((33, 20, 47), seed=0), 0.1
    elif name == "noise_big":
        vol, iso = noise((40, 70, 97), seed=5), -0.3
    elif name == "ragged":
        vol, iso = noise((3, 130, 2), seed=1, scale=40.0), 32.0
    elif name == "line33":
        vol, iso = noise((5, 6, 33), seed=2), 0.0                  # 33 points per line: a second, 1-bit word
    elif name == "lego":
        from conftest import load_npz
        vol, iso = load_npz("golden_lego_grid.npz")["radiance"][..., 3].numpy().copy(), 32.0
    else:
        vol, iso = fields(48)[0][name][0], 0.0
    v, f, n = mc.marching_cubes(vol, iso, x_off=3)
    gv, gf, gn = _engine().marching_cubes(torch.from_numpy(vol).cuda(), iso, x_off=3)
    assert np.array_equal(gv.cpu().numpy(), v)
    assert np.array_equal(gf.cpu().numpy(), f)
    assert np.array_equal(gn.cpu().numpy(), n)
    sv, sf, sn, _ = nm.marching_cubes(vol, iso)                 # the skimage-shaped entry point
    assert sv.shape == v.shape and sf.shape == f.shape


@pytest.mark.gpu
def test_cuda_shards_equal_oracle_shards_and_concatenate():
    from nerfmeshes_b200.nerf_api import _engine
    eng = _engine()
    vol, iso = noise((21, 18, 40), seed=7), 0.05
    n0 = vol.shape[0]
    v, f, n = mc.marching_cubes(vol, iso)
    cuts = [0, 6, 13, n0]
    vs, fs, ns, base = [], [], [], 0
    for own0, own1 in zip(cuts[:-1], cuts[1:]):
        buf0, buf1 = max(own0 - 1, 0), min(own1 + 2, n0)
        buf = torch.from_numpy(vol[buf0:buf1]).cuda().contiguous()
        nv, nt = eng.mc_count(buf, iso, buf0, n0, own0 - buf0, own1 - buf0)
        gv, gf, gn = eng.mc_emit(buf, iso, buf0, n0, own0 - buf0, own1 - buf0, nv, nt, base)
        ov, of, on = mc.marching_cubes(vol[buf0:buf1], iso, x_off=buf0, g_nx=n0, own=(own0 - buf0, own1 - buf0), v_base=base)
        assert np.array_equal(gv.cpu().numpy(), ov) and np.array_equal(gf.cpu().numpy(), of) and np.array_equal(gn.cpu().numpy(), on)
        vs.append(gv); fs.append(gf); ns.append(gn)
        base += nv
    assert np.array_equal(torch.cat(vs).cpu().numpy(), v) and np.array_equal(torch.cat(fs).cpu().numpy(), f)
    assert np.array_equal(torch.cat(ns).cpu().numpy(), n)
    with pytest.raises(Exception):                                   # a missing halo plane is an error, not a silent one-sided normal
        eng.mc_count(torch.from_numpy(vol[0:7]).cuda().contiguous(), iso, 0, n0, 0, 6)


@pytest.mark.gpu
def test_extract_geometry_on_lego_grid():
    """mesh_nerf.extract_geometry end to end on a small grid: sigma sweep -> iso clamp -> MC -> rescale; checked against
    the oracle chain run on the same density."""
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import LEGO_CFG
    from oracle import nerf_oracle as O
    model = nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval()

    class A:
        limit, res, iso_level = 1.2, 40, 32.0
    verts, tris, normals, density = nm.extract_geometry(model, "cuda", A)
    iso = O.extract_iso_level(density, A.iso_level)
    v, f, n = mc.marching_cubes(density, iso)
    assert np.array_equal(tris.numpy(), f)
    np.testing.assert_array_equal(verts.numpy(), (1.2 * (torch.from_numpy(v) / (A.res / 2.0) - 1.0)).numpy())
    assert verts.shape[0] > 1000
    # the sharded entry point as a single shard gives the same mesh
    from nerfmeshes_b200 import parallel as par
    v1, f1, n1, iso1 = par.extract_geometry_sharded(model, A, group=par.SINGLE)
    assert float(iso1) == float(iso) and torch.equal(v1, verts) and torch.equal(f1, tris) and torch.equal(n1, normals)


@pytest.mark.gpu
def test_extract_geometry_keeps_no_buffers_and_launches_what_one_slab_does():
    """extract_geometry is the one-slab case of the sharded pipeline, but in buffers that die with the call (it runs inside
    training processes), and with the kernel launches of the stand-alone stage calls: sweep, statistics, marching cubes."""
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import LEGO_CFG
    from nerfmeshes_b200 import parallel as par
    model = nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval()
    eng = model._engine()

    class A:
        limit, res, iso_level = 1.2, 40, 32.0

    def launches(fn):
        before = eng.launch_count()
        fn()
        return eng.launch_count() - before

    par._MESH_BUFFERS.clear()
    n_single = launches(lambda: nm.extract_geometry(model, "cuda", A))
    assert not par._MESH_BUFFERS
    n_slab = launches(lambda: par.extract_geometry_sharded(model, A, group=par.SINGLE, to_host=False))
    assert par._MESH_BUFFERS and n_single == n_slab > 0

    def stages():
        density = nm.extract_radiance(model, A, "cuda", A.res, sigma_only=True)
        eng.marching_cubes(density, float(nm.extract_iso_level(density, A, eng)))
    assert launches(stages) == n_single


@pytest.mark.gpu
def test_export_marching_cubes_writes_coloured_obj(tmp_path):
    """mesh_nerf.export_marching_cubes (geometry -> view-dependent appearance by ray casting along -normal -> OBJ)."""
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import LEGO_CFG
    model = nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval()

    class A:
        limit, res, iso_level = 1.2, 36, 32.0
        no_view_dependence, view_disparity, view_disparity_max_bound = False, 1e-2, 4e0
        save_dir, mesh_name = str(tmp_path), "mesh.obj"
    path = nm.mesh.export_marching_cubes(model, A)
    lines = open(path).read().splitlines()
    v = [l for l in lines if l.startswith("v ")]
    vn = [l for l in lines if l.startswith("vn ")]
    f = [l for l in lines if l.startswith("f ")]
    assert len(v) == len(vn) > 500 and len(f) > 1000
    cols = np.array([[float(x) for x in l.split()[4:7]] for l in v])
    assert cols.shape[1] == 3 and cols.min() >= 0.0 and cols.max() <= 1.0 + 1e-6 and cols.std() > 0.01
    idx = np.array([[int(t.split("//")[0]) for t in l.split()[1:]] for l in f])
    assert idx.min() == 1 and idx.max() == len(v)
    # the no-view-dependence branch samples the network directly at the vertices
    A.no_view_dependence = True
    verts, tris, normals, _ = nm.extract_geometry(model, "cuda", A)
    d = nm.mesh.mesh_appearance(model, verts, normals, A)
    assert d.shape == (verts.shape[0], 3)
