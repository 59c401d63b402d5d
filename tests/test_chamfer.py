"""Chamfer-distance mesh evaluation (DESIGN 4.7): the CPU oracle, load_obj, argument checks, and on the GPU the grid
nearest-neighbour search against the brute-force kernel (bit for bit) and float64, nm_chamfer, nm_mesh_sample, the
validation branch of validation_epoch_end and the pytorch3d stand-ins."""
import ctypes as C
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import _chamfer_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


# ----------------------------------------------------------------------------------------------------------------- CPU
def test_oracle_u01_is_splitmix64():
    # splitmix64 of seed 0, index 0: the first output of the reference generator is 0xE220A8397B1DCDAF
    assert R.u01(0, [0])[0] == np.float32((0xE220A8397B1DCDAF >> 40) / 2 ** 24)
    u = R.u01(12345, np.arange(100000))
    assert u.dtype == np.float32 and u.min() >= 0 and u.max() < 1 and abs(u.mean() - 0.5) < 5e-3


def test_oracle_area_cdf_and_points():
    v = np.array([[0, 0, 0], [3, 0, 0], [0, 4, 0], [1, 1, 1], [2, 2, 2]], np.float32)
    f = np.array([[0, 1, 2], [3, 3, 4], [0, 3, 4], [1, 2, 0]], np.int32)       # face 1 repeats a vertex, face 2 is collinear
    a = R.face_areas(v, f)
    assert a.tolist() == [6.0, 0.0, 0.0, 6.0]
    assert R.area_cdf(v, f).tolist() == [6.0, 6.0, 6.0, 12.0]
    faces = R.sample_faces(v, f, 7, 4000)
    assert set(faces.tolist()) == {0, 3}                                          # zero-area faces are never chosen
    p = R.sample_points(v, f, faces, 7).astype(np.float64)
    assert np.all(p[:, 2] == 0) and np.all(p[:, :2] >= 0) and np.all(p[:, 0] / 3 + p[:, 1] / 4 <= 1 + 1e-6)


def test_oracle_nearest_and_chamfer():
    x = np.array([[0, 0, 0]], np.float32)
    y = np.array([[1, 0, 0], [0, 2, 0]], np.float32)
    assert R.chamfer64(x, y) == (1.0, 2.5)
    rng = np.random.default_rng(0)
    q, p = rng.random((200, 3)), rng.random((300, 3))
    d, i = R.nearest64(q, p)
    full = ((q[:, None] - p[None]) ** 2).sum(-1)
    assert np.allclose(d, full.min(1), rtol=1e-12) and np.array_equal(i, full.argmin(1))


def test_create_mesh_hand_case():
    import nerfmeshes_b200 as nm
    v = torch.tensor([[0.0, 0.0, 0.0], [4.0, 0.0, 0.0], [0.0, 2.0, 0.0], [0.0, 0.0, 6.0]])
    m = nm.create_mesh(v, torch.tensor([[0, 1, 2], [0, 1, 3]]))
    # mean (1, 0.5, 1.5); centred max |.| = 4.5 (the z of vertex 3)
    want = np.array([[-1, -0.5, -1.5], [3, -0.5, -1.5], [-1, 1.5, -1.5], [-1, -0.5, 4.5]]) / 4.5
    assert np.allclose(m.verts_list()[0].numpy(), want, atol=1e-7)
    assert np.allclose(R.create_mesh(v.numpy()), want, atol=1e-12)
    assert m.faces_list()[0].tolist() == [[0, 1, 2], [0, 1, 3]] and not m.isempty() and nm.Meshes([], []).isempty()


def test_load_obj_golden_roundtrip():
    from nerfmeshes_b200.mesh import load_obj
    z = np.load(os.path.join(GOLDEN, "golden_mesh_inputs.npz"))
    v, f = load_obj(os.path.join(GOLDEN, "golden_mesh.obj"))
    assert v.dtype == torch.float32 and f.dtype == torch.int32
    assert np.array_equal(v.numpy(), z["v"]) and np.array_equal(f.numpy(), z["f"])


def test_load_obj_forms(tmp_path):
    from nerfmeshes_b200.mesh import load_obj
    p = tmp_path / "m.obj"
    p.write_text("# comment\nv 0 0 0\nv 1 0 0\nv 1 1 0 0.5 0.5 0.5\nv 0 1 0\nvt 0 0\nvn 0 0 1\n"
                 "f 1/1/1 2/1/1 3/1/1\nf -4//1 -2//1 -1//1\nf 1/1 2/1 3/1 4/1\ng x\nf 4 3 2\n")
    v, f = load_obj(str(p))
    assert v.shape == (4, 3) and v[2].tolist() == [1.0, 1.0, 0.0]
    assert f.tolist() == [[0, 1, 2], [0, 2, 3], [0, 1, 2], [0, 2, 3], [3, 2, 1]]


def test_rejected_arguments_without_a_device():
    from nerfmeshes_b200 import _lib as L
    lib = L.load()
    P = C.c_void_p(16)                       # never dereferenced: every call below fails its argument checks first
    err = lambda: lib.nm_last_error().decode()

    def rejects(rc, text):
        assert rc != 0 and text in err(), (rc, err())

    for fn in (lib.nm_nearest, lib.nm_debug_nearest_brute):
        rejects(fn(None, P, -1, P, 10, P, None, None), "negative size")
        rejects(fn(None, P, 10, P, 0, P, None, None), "empty point set")
        rejects(fn(None, P, 2 ** 31, P, 10, P, None, None), "2^31")
        rejects(fn(None, P, 10, P, 2 ** 31, P, None, None), "2^31")
        rejects(fn(None, P, 10, None, 10, P, None, None), "null point pointer")
        rejects(fn(None, None, 10, P, 10, P, None, None), "null query or output")
        rejects(fn(None, P, 10, P, 10, None, None, None), "null query or output")
        rejects(fn(None, P, 10, P, 10, P, None, None), "null handle")
    rejects(lib.nm_chamfer(None, P, 0, P, 5, P, None), "empty point set")
    rejects(lib.nm_chamfer(None, P, 5, P, 0, P, None), "empty point set")
    rejects(lib.nm_chamfer(None, P, -5, P, 5, P, None), "empty point set")
    rejects(lib.nm_chamfer(None, P, 5, P, 2 ** 31, P, None), "2^31")
    rejects(lib.nm_chamfer(None, P, 5, P, 5, None, None), "null pointer")
    rejects(lib.nm_chamfer(None, P, 5, P, 5, P, None), "null handle")
    rejects(lib.nm_mesh_sample(None, P, 3, P, 0, 10, 0, P, None, None), "empty mesh")
    rejects(lib.nm_mesh_sample(None, P, 0, P, 1, 10, 0, P, None, None), "empty mesh")
    rejects(lib.nm_mesh_sample(None, P, -3, P, 1, 10, 0, P, None, None), "empty mesh")
    rejects(lib.nm_mesh_sample(None, P, 3, P, 1, -1, 0, P, None, None), "negative sample count")
    rejects(lib.nm_mesh_sample(None, P, 3, P, 2 ** 31, 10, 0, P, None, None), "2^31")
    rejects(lib.nm_mesh_sample(None, None, 3, P, 1, 10, 0, P, None, None), "null mesh pointer")
    rejects(lib.nm_mesh_sample(None, P, 3, P, 1, 10, 0, None, None, None), "null output pointer")
    rejects(lib.nm_mesh_sample(None, P, 3, P, 1, 10, 0, P, None, None), "null handle")


def test_chamfer_distance_rejects_unsupported_options():
    import nerfmeshes_b200 as nm
    x = torch.zeros(1, 4, 3)
    for kw in (dict(x_lengths=torch.tensor([4])), dict(weights=torch.ones(1)), dict(x_normals=x), dict(batch_reduction="sum")):
        with pytest.raises(NotImplementedError):
            nm.chamfer_distance(x, x, **kw)


def test_compat_pytorch3d_reexports():
    import nerfmeshes_b200.chamfer as ch
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    try:
        for m in [k for k in sys.modules if k == "pytorch3d" or k.startswith("pytorch3d.")]:
            del sys.modules[m]
        from pytorch3d.loss import chamfer_distance
        from pytorch3d.ops import sample_points_from_meshes
        from pytorch3d.structures import Meshes
    finally:
        sys.path.remove(os.path.join(ROOT, "compat"))
        for m in [k for k in sys.modules if k == "pytorch3d" or k.startswith("pytorch3d.")]:
            del sys.modules[m]
    assert chamfer_distance is ch.chamfer_distance and sample_points_from_meshes is ch.sample_points_from_meshes
    assert Meshes is ch.Meshes


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


@pytest.fixture(scope="module")
def lego_mesh(lego_model):
    import nerfmeshes_b200 as nm
    v, f, _, _ = nm.extract_geometry(lego_model, "cuda", SimpleNamespace(limit=1.2, res=128, iso_level=32.0, super_sampling=0))
    return v, f


def _cuda(a):
    return torch.as_tensor(np.asarray(a, np.float32)).cuda()


def _same_as_brute(eng, q, p):
    q, p = _cuda(q), _cuda(p)
    d, i = eng.nearest(q, p)
    db, ib = eng.debug_nearest_brute(q, p)
    torch.cuda.synchronize()
    assert torch.equal(d.view(torch.int32), db.view(torch.int32)), "distances differ from brute force"
    assert torch.equal(i, ib), f"indices differ from brute force at {int((i != ib).sum())} queries"
    return d.cpu().numpy(), i.cpu().numpy()


def _brute_vs_float64(eng, q, p):
    db, ib = eng.debug_nearest_brute(_cuda(q), _cuda(p))
    d, i = db.cpu().numpy().astype(np.float64), ib.cpu().numpy()
    d64, _ = R.nearest64(q, p)
    assert np.all(np.abs(d - d64) <= 2.0 ** -21 * d64)
    assert np.all(R.dist64(q, p, i) <= d64 * (1 + 2.0 ** -20))


@pytest.mark.gpu
def test_nearest_uniform_and_float64(eng):
    rng = np.random.default_rng(1)
    q, p = rng.random((1 << 15, 3), np.float32), rng.random((1 << 15, 3), np.float32)
    _same_as_brute(eng, q, p)
    _brute_vs_float64(eng, q[:4096], p)


@pytest.mark.gpu
def test_nearest_lego_surface(eng, lego_mesh):
    v, f = lego_mesh
    q = eng.mesh_sample(v, f, 1 << 16, 11).cpu().numpy()
    p = eng.mesh_sample(v, f, 1 << 16, 12).cpu().numpy()
    _same_as_brute(eng, q, p)
    _brute_vs_float64(eng, q[:4096], p)


@pytest.mark.gpu
def test_nearest_lattice_ties(eng):
    g = np.stack(np.meshgrid(*[np.arange(10)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    p = np.concatenate([g, g])[np.random.default_rng(2).permutation(2 * len(g))]         # duplicates, permuted indices
    d, i = _same_as_brute(eng, g, p)
    assert np.all(d == 0)
    assert np.array_equal(i, [np.flatnonzero((p == x).all(1)).min() for x in g])
    h = (np.stack(np.meshgrid(*[np.arange(9)] * 3, indexing="ij"), -1).reshape(-1, 3) + 0.5).astype(np.float32)
    d, i = _same_as_brute(eng, h, p)                                                       # 8 corners x 2 copies tie
    full = ((h[:, None].astype(np.float64) - p[None]) ** 2).sum(-1)
    assert np.all(d == 0.75) and np.array_equal(i, [np.flatnonzero(r == r.min()).min() for r in full])


@pytest.mark.gpu
def test_nearest_adversarial_distributions(eng):
    rng = np.random.default_rng(3)
    u = rng.random((1 << 14, 3), np.float32)
    outlier = np.concatenate([u, np.array([[1e4, -1e4, 1e4]], np.float32)])
    _same_as_brute(eng, u, outlier)                                            # one far outlier
    _same_as_brute(eng, outlier, u)
    t = rng.random((1 << 13, 1), np.float32)
    line = np.concatenate([t, 2 * t, -t], 1).astype(np.float32)
    _same_as_brute(eng, line[: 1 << 12], line[1 << 12:])                       # collinear
    _same_as_brute(eng, rng.random((4096, 3), np.float32), line)
    _same_as_brute(eng, u + np.float32(1e3), (rng.random((1 << 14, 3), np.float32) + np.float32(1e3)))   # offset coordinates
    far = (50 + 10 * rng.random((2048, 3))).astype(np.float32)
    _same_as_brute(eng, far, u)                                                # queries far outside P's box
    _same_as_brute(eng, u[:1], u)                                              # N = 1
    _same_as_brute(eng, u, u[:1])                                              # M = 1
    _same_as_brute(eng, u[:1], u[1:2])
    _same_as_brute(eng, np.zeros((1000, 3), np.float32), np.zeros((500, 3), np.float32))   # all coincident
    _brute_vs_float64(eng, far, u)


@pytest.mark.gpu
def test_nearest_large_point_set(eng):
    rng = np.random.default_rng(4)
    _same_as_brute(eng, rng.random((1 << 13, 3), np.float32), rng.random((1 << 20, 3), np.float32))


@pytest.mark.gpu
def test_chamfer_means(eng, lego_mesh):
    v, f = lego_mesh
    rng = np.random.default_rng(5)
    for x, y in ((rng.random((1 << 15, 3), np.float32), rng.random((20000, 3), np.float32)),
                 (eng.mesh_sample(v, f, 1 << 15, 21).cpu().numpy(), eng.mesh_sample(v, f, 1 << 14, 22).cpu().numpy())):
        X, Y = _cuda(x), _cuda(y)
        m1, m2 = eng.chamfer(X, Y).cpu(), eng.chamfer(X, Y).cpu()
        assert torch.equal(m1, m2)
        dx, _ = eng.nearest(X, Y)
        dy, _ = eng.nearest(Y, X)
        own = (dx.double().cpu().numpy().sum() / len(x), dy.double().cpu().numpy().sum() / len(y))
        assert np.allclose(m1.numpy(), own, rtol=1e-12, atol=0)
        ref = R.chamfer64(x, y)
        assert np.all(np.abs(m1.numpy() - ref) <= 2.0 ** -20 * np.array(ref))
        sw = eng.chamfer(Y, X).cpu()
        assert float(sw.sum()) == float(m1.sum()) and sw[0] == m1[1] and sw[1] == m1[0]


def _test_mesh(rng):
    v = rng.normal(size=(200, 3)).astype(np.float32) * np.float32([1, 2, 0.5])
    f = rng.integers(0, 200, size=(500, 3)).astype(np.int32)
    f[::25, 1] = f[::25, 0]                                                     # zero-area faces
    return v, f


@pytest.mark.gpu
def test_mesh_sample_matches_oracle(eng):
    from scipy.stats import chisquare
    v, f = _test_mesh(np.random.default_rng(6))
    n, seed = 1 << 18, 1234
    p1, f1 = eng.mesh_sample(v, f, n, seed, want_faces=True)
    p2, f2 = eng.mesh_sample(v, f, n, seed, want_faces=True)
    p3 = eng.mesh_sample(v, f, n, seed + 1)
    assert torch.equal(p1, p2) and torch.equal(f1, f2) and not torch.equal(p1, p3)
    pts, fi = p1.cpu().numpy(), f1.cpu().numpy().astype(np.int64)
    assert np.array_equal(pts.view(np.int32), R.sample_points(v, f, fi, seed).view(np.int32))
    area = R.face_areas(v, f)
    cdf = R.area_cdf(v, f)
    total = cdf[-1]
    assert np.all(area[fi] > 0)                                                 # zero-area faces never chosen
    want = R.sample_faces(v, f, seed, n)
    off = fi != want
    lo = np.minimum(fi, want)[off]
    t = R.sample_targets(seed, n, total)[off]
    assert np.all(np.abs(t - cdf[lo]) <= 1e-12 * total), f"{int(off.sum())} samples outside the CDF bracket"
    pos = area > 0
    counts = np.bincount(fi, minlength=len(f))[pos]
    expect = n * area[pos].astype(np.float64) / area[pos].astype(np.float64).sum()
    assert chisquare(counts, expect * counts.sum() / expect.sum()).pvalue > 1e-4


@pytest.mark.gpu
def test_mesh_sample_bad_meshes_and_launch_count(eng):
    from nerfmeshes_b200 import NmError
    v, f = _test_mesh(np.random.default_rng(7))
    for bad in (200, -1):
        g = f.copy()
        g[17, 2] = bad
        with pytest.raises(NmError, match="outside"):
            eng.mesh_sample(v, g, 1000, 1)
    with pytest.raises(NmError, match="area"):
        eng.mesh_sample(v, np.repeat(f[:, :1], 3, 1), 1000, 1)                   # every face degenerate
    eng.mesh_sample(v, f, 1000, 1)                                              # the error was reported once: the handle works
    V, F = _cuda(v), torch.as_tensor(f).cuda()
    out = torch.empty((10, 3), device="cuda")
    lib, h, before = eng.lib, eng._h, eng.launch_count()
    P = C.c_void_p
    assert lib.nm_mesh_sample(h, P(V.data_ptr()), 200, P(F.data_ptr()), 500, -1, 0, P(out.data_ptr()), None, None) != 0
    assert lib.nm_mesh_sample(h, P(V.data_ptr()), 200, P(F.data_ptr()), 0, 10, 0, P(out.data_ptr()), None, None) != 0
    assert lib.nm_mesh_sample(h, P(V.data_ptr()), 200, P(F.data_ptr()), 500, 0, 0, None, None, None) == 0
    assert lib.nm_nearest(h, P(V.data_ptr()), 200, P(V.data_ptr()), 0, P(out.data_ptr()), None, None) != 0
    assert lib.nm_nearest(h, None, 0, P(V.data_ptr()), 200, None, None, None) == 0
    assert lib.nm_chamfer(h, P(V.data_ptr()), 0, P(V.data_ptr()), 200, P(out.data_ptr()), None) != 0
    assert eng.launch_count() == before


class _TargetDataset:
    def __init__(self, target_mesh):
        self.target_mesh = target_mesh


@pytest.mark.gpu
def test_validation_epoch_end_chamfer_branch(lego_mesh):
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from nerfmeshes_b200.lightning import LightningHooks
    from test_gpu_parity import LEGO_CFG

    class Model(LightningHooks, nm.NeRFModel):
        pass

    cfg = {**LEGO_CFG, "experiment.chamfer_loss": True, "experiment.chamfer_sampling_size": 2400}
    model = Model.from_npz(cfg, load_npz("weights_lego_nerf.npz")).eval()
    v, f = lego_mesh
    outputs = [{"log": {"validation/loss": torch.tensor(1.0)}, "val_loss": torch.tensor(1.0)}]
    model.val_dataset = _TargetDataset(nm.Meshes([v], [f]))
    torch.manual_seed(3)
    own = model.validation_epoch_end(outputs)["log"]["validation/chamfer_loss"]
    torch.manual_seed(3)                                  # the public functions, the same draws
    vm, fm, _, _ = nm.extract_geometry(model, "cuda", SimpleNamespace(limit=1.2, res=128, iso_level=32.0, super_sampling=0))
    t = nm.sample_points_from_meshes(nm.create_mesh(v, f), 2400)
    s = nm.sample_points_from_meshes(nm.create_mesh(vm, fm), 2400)
    assert float(own) == float(nm.chamfer_distance(t, s)[0])
    jitter = v + 0.02 * torch.randn(v.shape, generator=torch.Generator().manual_seed(0))
    model.val_dataset = _TargetDataset((jitter, f))
    worse = model.validation_epoch_end(outputs)["log"]["validation/chamfer_loss"]
    assert 0 <= float(own) < float(worse)
    model.val_dataset = _TargetDataset(None)
    with pytest.raises(AssertionError, match="a target mesh .obj must be provided"):
        model.validation_epoch_end(outputs)


@pytest.mark.gpu
def test_compat_functions_match(eng, lego_mesh):
    import nerfmeshes_b200.chamfer as ch
    sys.path.insert(0, os.path.join(ROOT, "compat"))
    try:
        from pytorch3d.loss import chamfer_distance
        from pytorch3d.ops import sample_points_from_meshes
        from pytorch3d.structures import Meshes
    finally:
        sys.path.remove(os.path.join(ROOT, "compat"))
    v, f = lego_mesh
    a = sample_points_from_meshes(Meshes(verts=[v], faces=[f]), 3000, seed=9)
    b = ch.sample_points_from_meshes(ch.Meshes([v], [f]), 3000, seed=9)
    assert torch.equal(a, b)
    assert float(chamfer_distance(a, b[:, ::2])[0]) == float(ch.chamfer_distance(b, b[:, ::2])[0])
