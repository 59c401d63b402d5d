"""Small-component removal (nm_mesh_components, DESIGN 4.9): the CPU oracle against a plain BFS, its invariances and edge
values, argument checks without a device, and on the GPU the kernel against the oracle bit for bit (analytic volumes,
adversarial meshes, the 256^3 lego mesh), determinism, bad face indices, and the switch in extract_geometry /
export_marching_cubes / extract_geometry_sharded."""
import ctypes as C
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import _components_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _random_mesh(rng, V=60, F=50, unreferenced=10):
    """Faces over the first V - unreferenced vertices (several components), with degenerate and duplicate faces."""
    used = V - unreferenced
    f = rng.integers(0, used, size=(F, 3))
    f[::7, 1] = f[::7, 0]                             # (a, a, b)
    f[::11, 1:] = f[::11, :1]                         # (a, a, a)
    f = np.concatenate([f, f[:5]])                    # duplicate faces
    perm = rng.permutation(V)                         # unreferenced vertices anywhere in the numbering
    v = rng.normal(size=(V, 3)).astype(np.float32)
    n = rng.normal(size=(V, 3)).astype(np.float32)
    return v, n, perm[f].astype(np.int32)


# ----------------------------------------------------------------------------------------------------------------- CPU
def test_oracle_matches_bfs():
    rng = np.random.default_rng(0)
    for trial in range(40):
        V = int(rng.integers(1, 80))
        F = int(rng.integers(0, 60))
        v, n, f = _random_mesh(rng, V, F, unreferenced=int(rng.integers(0, max(V // 3, 1))))
        labels, sizes = R.labels_and_sizes(V, f)
        assert np.array_equal(labels, R.bfs_labels(V, f)), trial
        want = np.zeros(V, np.int64)
        for a, _, _ in f.tolist():
            want[labels[a]] += 1
        assert np.array_equal(sizes, want)
        assert np.all(labels <= np.arange(V)) and np.all(labels[labels] == labels)


def test_oracle_filter_hand_case():
    v = np.arange(24, dtype=np.float32).reshape(8, 3)
    n = -v
    # component {0,1,2,3}: 3 faces (one degenerate); {4}: one face (4,4,4); {5,7}: 2 faces (one duplicate); 6 unreferenced
    f = np.array([[3, 1, 2], [0, 1, 1], [7, 5, 5], [2, 3, 0], [4, 4, 4], [7, 5, 5]], np.int32)
    labels, sizes = R.labels_and_sizes(8, f)
    assert labels.tolist() == [0, 0, 0, 0, 4, 5, 6, 5]
    assert sizes[[0, 4, 5, 6]].tolist() == [3, 1, 2, 0]
    vo, no, fo, counts, _ = R.remove_small_components(v, n, f, 2)
    assert np.array_equal(vo, v[[0, 1, 2, 3, 5, 7]]) and np.array_equal(no, n[[0, 1, 2, 3, 5, 7]])
    assert fo.tolist() == [[3, 1, 2], [0, 1, 1], [5, 4, 4], [2, 3, 0], [5, 4, 4]]
    assert counts == (6, 5, 3, 2)


def test_oracle_invariant_under_vertex_permutation():
    rng = np.random.default_rng(1)
    for _ in range(20):
        v, n, f = _random_mesh(rng, 70, 60, 12)
        perm = rng.permutation(len(v))               # old vertex i becomes perm[i]
        inv = np.argsort(perm)
        for m in (0, 1, 2, 3, 5):
            labels, sizes = R.labels_and_sizes(len(v), f)
            keep = sizes[labels] >= m
            l2, s2 = R.labels_and_sizes(len(v), perm[f])
            keep2 = s2[l2] >= m
            assert np.array_equal(keep2[perm], keep)
            _, _, fo, counts, _ = R.remove_small_components(v, n, f, m)
            vo2, _, fo2, counts2, _ = R.remove_small_components(v[inv], n[inv], perm[f], m)
            assert counts2 == counts and fo2.shape == fo.shape
            assert np.array_equal(vo2, v[inv][keep2])


def test_oracle_edge_values_of_m():
    rng = np.random.default_rng(2)
    v, n, f = _random_mesh(rng, 90, 70, 15)
    vo, no, fo, counts, _ = R.remove_small_components(v, n, f, 0)
    assert np.array_equal(vo, v) and np.array_equal(no, n) and np.array_equal(fo, f) and counts[:2] == (90, len(f))
    vo, no, fo, counts, labels = R.remove_small_components(v, n, f, 1)
    ref = np.zeros(len(v), bool)
    ref[f.reshape(-1)] = True
    assert np.array_equal(vo, v[ref]) and len(fo) == len(f) and counts[2] == counts[3]
    _, sizes = R.labels_and_sizes(len(v), f)
    vo, _, fo, counts, _ = R.remove_small_components(v, n, f, int(sizes.max()) + 1)
    assert vo.shape == (0, 3) and fo.shape == (0, 3) and counts[:2] == (0, 0) and counts[3] == 0 and counts[2] > 0


def test_rejected_arguments_without_a_device():
    from nerfmeshes_b200 import _lib as L
    lib = L.load()
    P = C.c_void_p(16)                       # never dereferenced: every call below fails its argument checks first
    cnt = (C.c_int64 * 4)()
    err = lambda: lib.nm_last_error().decode()

    def rejects(text, h=None, v=P, n=P, V=10, f=P, F=10, m=0, vo=P, no=P, fo=P, counts=cnt):
        rc = lib.nm_mesh_components(h, v, n, V, f, F, m, vo, no, fo, None, counts, None)
        assert rc != 0 and text in err(), (rc, err())

    rejects("negative size", V=-1)
    rejects("negative size", F=-1)
    rejects("negative min_faces", m=-1)
    rejects("2^31", V=2 ** 31)
    rejects("2^31", F=2 ** 31)
    rejects("null counts", counts=None)
    for kw in (dict(v=None), dict(n=None), dict(vo=None), dict(no=None)):
        rejects("null vertex pointer", **kw)
    for kw in (dict(f=None), dict(fo=None)):
        rejects("null face pointer", **kw)
    rejects("null handle")
    rejects("null handle", v=None, n=None, vo=None, no=None, f=None, fo=None, V=0, F=0)
    rejects("null handle", f=None, fo=None, F=0)             # F = 0 needs no face pointers


# ----------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def eng():
    from nerfmeshes_b200.nerf_api import _engine
    return _engine()


@pytest.fixture(scope="module")
def lego_model():
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import LEGO_CFG
    return nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval()


def _same_as_oracle(eng, v, n, f, m, labels=True):
    """The kernel at min_faces m against the oracle, bit for bit; returns the oracle's counts."""
    v, n, f = (np.asarray(x) for x in (v, n, f))
    vo, no, fo, counts, lab = eng.mesh_components(torch.as_tensor(v).cuda(), torch.as_tensor(n).cuda(),
                                                  torch.as_tensor(f).cuda(), m, want_labels=labels)
    rv, rn, rf, rc, rl = R.remove_small_components(v, n, f, m)
    assert counts == rc, (m, counts, rc)
    assert np.array_equal(vo.cpu().numpy().view(np.int32), rv.view(np.int32)), f"m={m}: vertices differ"
    assert np.array_equal(no.cpu().numpy().view(np.int32), rn.view(np.int32)), f"m={m}: normals differ"
    assert np.array_equal(fo.cpu().numpy(), rf), f"m={m}: faces differ"
    if labels:
        assert np.array_equal(lab.cpu().numpy(), rl), f"m={m}: labels differ"
    return rc


# Five separated shapes in a 128^3 grid (index units): four spheres (centre, radius) and a torus (centre, R, r) about z.
SPHERES = [((24.37, 24.21, 24.13), 6.0), ((24.29, 24.41, 70.17), 10.0), ((30.23, 90.31, 30.43), 16.0),
           ((85.19, 85.33, 85.27), 24.0)]
TORUS = ((90.41, 30.17, 40.29), 20.0, 5.0)


def _analytic_volume(n=128):
    x = np.arange(n, dtype=np.float64)
    X, Y, Z = np.meshgrid(x, x, x, indexing="ij")
    fields = [r - np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2) for c, r in SPHERES]
    (cx, cy, cz), Rt, rt = TORUS
    fields.append(rt - np.sqrt((np.sqrt((X - cx) ** 2 + (Y - cy) ** 2) - Rt) ** 2 + (Z - cz) ** 2))
    return np.max(fields, 0).astype(np.float32), fields


@pytest.fixture(scope="module")
def shapes_mesh(eng):
    vol, fields = _analytic_volume()
    v, f, n = eng.marching_cubes(torch.from_numpy(vol), 0.0)
    return v.cpu().numpy(), n.cpu().numpy(), f.cpu().numpy(), fields


@pytest.mark.gpu
def test_analytic_shapes(eng, shapes_mesh):
    v, n, f, fields = shapes_mesh
    labels, sizes = R.labels_and_sizes(len(v), f)
    roots = np.flatnonzero((labels == np.arange(len(v))) & (sizes > 0))
    assert len(roots) == 5
    # every component is the surface of exactly one shape: its vertices lie on that shape's zero level
    idx = np.round(v).astype(np.int64).clip(0, 127)
    owner = np.argmax(np.stack([fl[idx[:, 0], idx[:, 1], idx[:, 2]] for fl in fields]), 0)
    shape_of = {}
    for r in roots:
        own = np.unique(owner[labels == r])
        assert len(own) == 1, own
        shape_of[int(r)] = int(own[0])
    assert sorted(shape_of.values()) == [0, 1, 2, 3, 4]
    s = np.sort(sizes[roots])
    assert len(np.unique(s)) == 5
    # sphere face counts grow with the radius
    by_shape = {shape_of[int(r)]: int(sizes[r]) for r in roots}
    assert by_shape[0] < by_shape[1] < by_shape[2] < by_shape[3]
    thresholds = [0, 1] + [int(s[k] + s[k + 1]) // 2 for k in range(4)] + [int(s[0]), int(s[-1]), int(s[-1]) + 1]
    for m in thresholds:
        counts = _same_as_oracle(eng, v, n, f, m)
        assert counts[2] == 5 and counts[3] == int((s >= m).sum())
        assert counts[1] == int(s[s >= m].sum())


@pytest.mark.gpu
def test_adversarial_meshes(eng, shapes_mesh):
    rng = np.random.default_rng(10)
    # every face its own component (V = 3F)
    F = 1 << 16
    v = rng.normal(size=(3 * F, 3)).astype(np.float32)
    f = np.arange(3 * F, dtype=np.int32).reshape(F, 3)
    for m in (0, 1, 2):
        assert _same_as_oracle(eng, v, v, f, m)[2] == F
    # one triangle strip of 2^20 faces: the deepest union-find, the longest diameter; forwards, reversed, permuted
    F = 1 << 20
    v = rng.normal(size=(F + 2, 3)).astype(np.float32)
    n = rng.normal(size=(F + 2, 3)).astype(np.float32)
    f = (np.arange(F)[:, None] + np.arange(3)[None]).astype(np.int32)
    perm = rng.permutation(F + 2)
    for ff, vv, nn in ((f, v, n), (f[::-1].copy(), v, n), (perm[f].astype(np.int32), v[np.argsort(perm)], n[np.argsort(perm)])):
        for m in (1, F, F + 1):
            c = _same_as_oracle(eng, vv, nn, ff, m)
            assert c[2] == 1 and c[3] == (1 if m <= F else 0)
    # the analytic mesh: vertex indices permuted (hooking order scrambled), faces reversed, degenerate faces and unreferenced
    # vertices added
    v, n, f, _ = shapes_mesh
    perm = rng.permutation(len(v))
    inv = np.argsort(perm)
    pv, pn, pf = v[inv], n[inv], perm[f].astype(np.int32)
    _, sizes = R.labels_and_sizes(len(v), f)
    mid = int(np.median(sizes[sizes > 0]))
    for m in (1, mid, mid + 1):
        _same_as_oracle(eng, pv, pn, pf, m)
        _same_as_oracle(eng, v, n, f[::-1].copy(), m)
    extra = rng.normal(size=(1000, 3)).astype(np.float32)
    uv = np.concatenate([extra[:500], v, extra[500:]])
    un = np.concatenate([extra[:500], n, extra[500:]])
    uf = f + 500
    a = rng.integers(0, len(uv), 300)
    b = rng.integers(0, len(uv), 300)
    degen = np.concatenate([np.stack([a, a, b], 1), np.stack([b, b, b], 1)]).astype(np.int32)
    uf = np.concatenate([uf[:1000], degen, uf[1000:]]).astype(np.int32)
    for m in (0, 1, 2, 3, mid):
        _same_as_oracle(eng, uv, un, uf, m)
    # tiny and empty meshes
    one = np.ones((1, 3), np.float32)
    none_f = np.zeros((0, 3), np.int32)
    assert _same_as_oracle(eng, one, one, none_f, 0) == (1, 0, 0, 0)
    assert _same_as_oracle(eng, one, one, none_f, 1) == (0, 0, 0, 0)
    before = eng.launch_count()
    empty = np.zeros((0, 3), np.float32)
    assert _same_as_oracle(eng, empty, empty, none_f, 0) == (0, 0, 0, 0)
    assert eng.launch_count() == before                         # V = F = 0 launches nothing


@pytest.mark.gpu
def test_deterministic(eng, shapes_mesh):
    v, n, f, _ = shapes_mesh
    perm = np.random.default_rng(11).permutation(len(v))
    args = [torch.as_tensor(x).cuda() for x in (v[np.argsort(perm)], n[np.argsort(perm)], perm[f].astype(np.int32))]
    a = eng.mesh_components(*args, 500, want_labels=True)
    b = eng.mesh_components(*args, 500, want_labels=True)
    assert a[3] == b[3]
    for x, y in zip(a[:3] + a[4:], b[:3] + b[4:]):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


@pytest.mark.gpu
def test_bad_face_index(eng, shapes_mesh):
    from nerfmeshes_b200 import NmError
    v, n, f, _ = shapes_mesh
    for bad in (len(v), -1):
        g = f.copy()
        g[17, 2] = bad
        with pytest.raises(NmError, match=r"mesh components: a face index lies outside \[0, V\)"):
            eng.mesh_components(v, n, g, 1)
        eng.check_flags()                                           # reported once
        _same_as_oracle(eng, v, n, f, 1)                            # the handle works
        with pytest.raises(NmError, match=r"mesh sampler: a face index lies outside \[0, V\)"):
            eng.mesh_sample(v, g, 100, 1)                           # the sampler's own message is unaffected
        eng.check_flags()


@pytest.mark.gpu
@pytest.mark.parametrize("s,net", [(0, False), (0, True), (3, False), (3, True)])
def test_lego_256(lego_model, s, net):
    import nerfmeshes_b200 as nm
    eng = lego_model._engine()
    base = dict(limit=1.2, res=256, iso_level=32.0, super_sampling=s, network_normals=net)
    v0, f0, n0, d0 = nm.extract_geometry(lego_model, "cuda", SimpleNamespace(**base))
    labels, sizes = R.labels_and_sizes(len(v0), f0.numpy())
    comp = np.sort(sizes[(labels == np.arange(len(v0))) & (sizes > 0)])[::-1]
    print(f"lego 256^3 s={s} net={net}: {len(v0)} vertices, {len(f0)} faces, {len(comp)} components, largest {comp[:5].tolist()}")
    for m in sorted({1, 16, 256, int(comp[0]), int(comp[min(1, len(comp) - 1)]) + 1}):
        _same_as_oracle(eng, v0.numpy(), n0.numpy(), f0.numpy(), m)
    m = 16
    v1, f1, n1, d1 = nm.extract_geometry(lego_model, "cuda", SimpleNamespace(**base, min_component_faces=m))
    rv, rn, rf, _, _ = R.remove_small_components(v0.numpy(), n0.numpy(), f0.numpy(), m)
    assert np.array_equal(d1, d0)
    assert np.array_equal(v1.numpy().view(np.int32), rv.view(np.int32)) and np.array_equal(f1.numpy(), rf)
    assert np.array_equal(n1.numpy().view(np.int32), rn.view(np.int32))        # the kept vertices' normals, unchanged


@pytest.mark.gpu
def test_switch_off_is_unchanged(lego_model, tmp_path):
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import mesh
    eng = lego_model._engine()

    def args(**kw):
        return SimpleNamespace(limit=1.2, res=64, iso_level=32.0, no_view_dependence=True, save_dir=str(tmp_path), **kw)
    # today's composition of the primitives: sweep, iso, marching cubes, host rescale
    lins = [torch.linspace(-1.2, 1.2, 64) for _ in range(3)]
    dens = eng.grid_sigma(lins)
    iso = mesh.extract_iso_level(dens, args(), eng)
    vt, ft, nt = eng.marching_cubes(dens, float(iso))
    vt = 1.2 * (vt.cpu() / 32.0 - 1.0)
    outs = [nm.extract_geometry(lego_model, "cuda", a) for a in (args(), args(min_component_faces=0),
                                                                  args(min_component_faces=None))]
    for v, f, n, _ in outs:
        assert torch.equal(v, vt) and torch.equal(f, ft.cpu()) and torch.equal(n, nt.cpu())
    p0 = mesh.export_marching_cubes(lego_model, args(mesh_name="a.obj"))
    p1 = mesh.export_marching_cubes(lego_model, args(mesh_name="b.obj", min_component_faces=0))
    assert open(p0, "rb").read() == open(p1, "rb").read()
    d = mesh.mesh_appearance(lego_model, vt, nt.cpu(), args())
    mesh.export_obj(vt, ft.cpu(), d, nt.cpu(), str(tmp_path / "c.obj"))
    assert open(p0, "rb").read() == open(tmp_path / "c.obj", "rb").read()


@pytest.mark.gpu
def test_switch_on_export_and_cache(lego_model, tmp_path):
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import mesh
    base = dict(limit=1.2, res=96, iso_level=32.0, no_view_dependence=True, save_dir=str(tmp_path))
    v0, f0, n0, _ = nm.extract_geometry(lego_model, "cuda", SimpleNamespace(**base))
    labels, sizes = R.labels_and_sizes(len(v0), f0.numpy())
    m = int(sizes.max())                                       # keep only the largest component(s)
    rv, rn, rf, rc, _ = R.remove_small_components(v0.numpy(), n0.numpy(), f0.numpy(), m)
    A = SimpleNamespace(**base, min_component_faces=m, mesh_name="m.obj", cache_name="c.pt", use_cached_mesh=True,
                        override_cache_mesh=False)
    p = mesh.export_marching_cubes(lego_model, A)
    cached = torch.load(os.path.join(str(tmp_path), "c.pt"), weights_only=False)
    assert np.array_equal(cached[0].numpy(), rv) and np.array_equal(cached[1].numpy(), rf) and np.array_equal(cached[2].numpy(), rn)
    text = open(p).read().splitlines()
    assert sum(ln.startswith("v ") for ln in text) == len(rv) and sum(ln.startswith("f ") for ln in text) == len(rf)
    A.mesh_name = "m2.obj"
    p2 = mesh.export_marching_cubes(lego_model, A)             # served from the cache
    assert open(p2).read() == open(p).read()


@pytest.mark.gpu
@pytest.mark.parametrize("s,net", [(0, False), (2, True)])
def test_sharded_matches_single_gpu(lego_model, s, net):
    from nerfmeshes_b200 import parallel as par
    import nerfmeshes_b200 as nm
    A = SimpleNamespace(limit=1.2, res=64, iso_level=32.0, super_sampling=s, network_normals=net, min_component_faces=40)
    v1, f1, n1, _ = par.extract_geometry_sharded(lego_model, A, group=par.SINGLE)
    v0, f0, n0, _ = nm.extract_geometry(lego_model, "cuda", A)
    assert torch.equal(v0, v1) and torch.equal(f0, f1) and torch.equal(n0, n1)
    A.min_component_faces = 0
    v2, f2, n2, _ = par.extract_geometry_sharded(lego_model, A, group=par.SINGLE)
    rv, rn, rf, _, _ = R.remove_small_components(v2.numpy(), n2.numpy(), f2.numpy(), 40)
    assert np.array_equal(v1.numpy(), rv) and np.array_equal(f1.numpy(), rf) and np.array_equal(n1.numpy(), rn)


@pytest.mark.multigpu
def test_multi_gpu_components():
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs 2 GPUs")
    port = 29800 + os.getpid() % 90
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "_components_multi_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0 and f"COMPONENTS_MULTI_OK {world}" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
