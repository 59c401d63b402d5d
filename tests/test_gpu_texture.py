"""Texture bake on the GPU (nm_bake_texture, DESIGN 4.12): the texel queries against the numpy restatement (_texture_ref) bit
for bit on the analytic meshes and decimated lego meshes, the atlas against the restatement's scatter, ring and quantisation of
the kernel's own texel colours, those colours against the render path, the vertex colours against mesh_appearance (lego NeRF
and BuFF, with and without view dependence), chunk sizes and a second run, the error paths, the switch args.texture_texels in
export_marching_cubes, and the texture's colour error at random surface points against the vertex colours'."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import _texture_ref as T
from test_mesh_decimate_reference import mesh as analytic_mesh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
APPEARANCE = dict(view_disparity=1e-2, view_disparity_max_bound=4.0)


@pytest.fixture(scope="module")
def lego():
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import LEGO_CFG
    return nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval()


@pytest.fixture(scope="module")
def buff():
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import BUFF_CFG
    return nm.BuFFModel.from_npz(BUFF_CFG, load_npz("weights_lego_buff.npz")).cuda().eval()


@pytest.fixture(scope="module")
def eng(lego):
    return lego._engine()


_LEGO = {}


def lego_mesh(lego, res, frac):
    """The lego fine net's iso-32 mesh at res^3 decimated to frac of its faces: world coordinates (what extract_geometry
    returns), CPU tensors."""
    if (res, frac) not in _LEGO:
        import nerfmeshes_b200 as nm
        A = SimpleNamespace(limit=1.2, res=res, iso_level=32.0)
        F = nm.extract_geometry(lego, "cuda", A)[1].shape[0]
        A.decimate_faces = int(frac * F)
        _LEGO[(res, frac)] = nm.extract_geometry(lego, "cuda", A)[:3]
    return _LEGO[(res, frac)]


def same_rays(eng, v, n, f, N, mode, c, f0, f1):
    a, d, xy = eng.debug_texture_rays(v, n, f, N, f0, f1, mode=mode, view_disparity=c)
    ra, rd, rxy = T.queries(np.asarray(v), np.asarray(n), np.asarray(f), N, mode, c, f0, f1)
    assert np.array_equal(a.cpu().numpy().view(np.int32), ra.view(np.int32)), (N, mode, f0, f1, "origins / points differ")
    assert np.array_equal(d.cpu().numpy().view(np.int32), rd.view(np.int32)), (N, mode, f0, f1, "directions differ")
    assert np.array_equal(xy.cpu().numpy(), rxy), (N, mode, f0, f1, "pixels differ")


@pytest.mark.gpu
@pytest.mark.parametrize("N", [2, 3, 8, 17])
def test_rays_match_restatement(eng, lego, N):
    meshes = [analytic_mesh(name) for name in ("sphere", "torus", "two_spheres", "border")]
    meshes += [(v.numpy(), n.numpy(), f.numpy()) for v, f, n in (lego_mesh(lego, 64, 0.1), lego_mesh(lego, 128, 0.02))]
    for v, n, f in meshes:
        F = len(f)
        for mode in (0, 1):
            same_rays(eng, v, n, f, N, mode, 0.0123, 0, F)
        for f0, f1 in ((0, 1), (F // 3, F // 2 + 1), (F - 1, F), (5, 5)):
            same_rays(eng, v, n, f, N, 0, 1e-2, f0, f1)


def _render(model, a, d, mode):
    """The colours mesh_appearance's query gives for queries (a, d): ray origins or points."""
    eng = model._engine()
    if mode == 1:
        return eng.point_mlp(model.get_model()._owner[1], a, d)[:, :3]
    return eng.render_rays(a, d, 0.0, 4.0, buff=hasattr(model, "tree"), want=("rgb",))["rgb"]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
def test_atlas_matches_restatement(eng, lego, mode):
    v, f, n = lego_mesh(lego, 64, 0.1)
    N, F = 8, f.shape[0]
    u8, atlas, uv, rgb, counts = eng.bake_texture(v, n, f, N, mode=mode, which=1, view_disparity=1e-2, near_far=(0.0, 4.0))
    _, _, W, H = T.layout(F, N)
    assert counts == (W, H, F * N * (N + 1) // 2, 0) and atlas.shape == (H, W, 3)
    a, d, xy = eng.debug_texture_rays(v, n, f, N, 0, F, mode=mode, view_disparity=1e-2)
    xy = xy.cpu().numpy()
    texel_rgb = atlas.cpu().numpy()[xy[:, 1], xy[:, 0]]
    # the kernel's texel colours are the render path's colours of its queries
    assert np.array_equal(texel_rgb.view(np.int32), _render(lego, a, d, mode).cpu().numpy().view(np.int32))
    ref = T.assemble(F, N, texel_rgb, xy)
    assert np.array_equal(atlas.cpu().numpy().view(np.int32), ref.view(np.int32))
    assert np.array_equal(u8.cpu().numpy(), T.quantise(ref))
    assert np.array_equal(uv.cpu().numpy().view(np.int32), T.uv(F, N).view(np.int32))


def _bake(model, v, f, n, N, **kw):
    from nerfmeshes_b200 import mesh
    return mesh.bake_texture(model, v, f, n, SimpleNamespace(**APPEARANCE, texture_texels=N, **kw))


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["lego", "buff"])
@pytest.mark.parametrize("nvd", [False, True])
def test_diffuse_equals_mesh_appearance(lego, buff, which, nvd):
    from nerfmeshes_b200 import mesh
    model = lego if which == "lego" else buff
    v, f, n = lego_mesh(lego, 64, 0.1)
    # three vertices no face references, in the middle of the vertex list
    k = v.shape[0] // 2
    extra = torch.tensor([[0.1, 0.2, 0.3], [-0.4, 0.0, 0.25], [0.0, 0.0, 0.0]])
    v = torch.cat([v[:k], extra, v[k:]])
    n = torch.cat([n[:k], torch.nn.functional.normalize(torch.tensor([[0.0, 0.0, 1.0], [1.0, 1.0, 0.0], [0.0, -1.0, 0.0]]), dim=1), n[k:]])
    f = torch.where(f >= k, f + 3, f)
    args = SimpleNamespace(**APPEARANCE, no_view_dependence=nvd)
    want = mesh.mesh_appearance(model, v, n, args)
    u8, uv, diffuse = _bake(model, v, f, n, 8, no_view_dependence=nvd)
    assert np.array_equal(diffuse.view(np.int32), want.view(np.int32))
    # every corner texel of a vertex holds the vertex's colour
    eng = model._engine()
    _, atlas, _, _, counts = eng.bake_texture(v, n, f, 8, mode=int(nvd), which=model.get_model()._owner[1],
                                              flags=eng._flags(False, which == "buff"), view_disparity=1e-2, near_far=(0.0, 4.0))
    assert counts[3] == 3
    ff, _, _, corner, x, y = T.texels(f.shape[0], 8)
    c = corner >= 0
    vid = f.numpy()[ff[c], corner[c]]
    assert np.array_equal(atlas.cpu().numpy()[y[c], x[c]].view(np.int32), want[vid].view(np.int32))
    assert np.array_equal(u8, T.quantise(atlas.cpu().numpy()))


@pytest.mark.gpu
def test_chunk_size_and_second_run(eng, lego, monkeypatch):
    v, f, n = lego_mesh(lego, 96, 0.1)
    runs = []
    for chunk in (None, "1000", "37"):
        if chunk is None:
            monkeypatch.delenv("NM_TEXTURE_CHUNK_TEXELS", raising=False)
        else:
            monkeypatch.setenv("NM_TEXTURE_CHUNK_TEXELS", chunk)
        for mode in (0, 1):
            runs.append(eng.bake_texture(v, n, f, 5, mode=mode, which=1, view_disparity=1e-2, near_far=(0.0, 4.0)))
    runs.append(eng.bake_texture(v, n, f, 5, mode=0, which=1, view_disparity=1e-2, near_far=(0.0, 4.0)))     # a second run
    for i, r in enumerate(runs[2:]):
        base = runs[i % 2]
        assert r[4] == base[4]
        for x, y in zip(r[:4], base[:4]):
            assert torch.equal(x.view(torch.uint8), y.view(torch.uint8))


@pytest.mark.gpu
def test_errors(eng, lego):
    from nerfmeshes_b200 import NmError
    v, n, f = analytic_mesh("sphere")
    for N in (1, 65):
        with pytest.raises(NmError, match=f"N = {N} outside"):
            eng.bake_texture(v, n, f, N, mode=1)
    big = np.zeros((200000, 3), np.int32)
    with pytest.raises(NmError, match="the largest N that fits 200000 faces is 49"):
        eng.bake_texture(v, n, big, 64, mode=1)
    for bad in (len(v), -1):
        g = f.copy()
        g[17, 2] = bad
        before = eng.launch_count()
        with pytest.raises(NmError, match=r"texture bake: a face index lies outside \[0, V\)"):
            eng.bake_texture(v, n, g, 4, mode=1, which=1)
        assert eng.launch_count() - before < 10                    # nothing was rendered
        eng.check_flags()                                          # reported once
        eng.debug_texture_rays(v, n, g, 4, 0, len(g))               # the test hook reports it too, at the next check
        with pytest.raises(NmError, match=r"texture bake: a face index"):
            eng.check_flags()
        eng.check_flags()
    e3 = np.zeros((0, 3), np.float32)
    before = eng.launch_count()
    out = eng.bake_texture(e3, e3, np.zeros((0, 3), np.int32), 8, mode=1, which=1)
    assert out[4] == (0, 0, 0, 0) and eng.launch_count() == before
    # a face-less mesh: every vertex gets its own query
    u8, atlas, uv, rgb, counts = eng.bake_texture(v[:5], n[:5], np.zeros((0, 3), np.int32), 8, mode=1, which=1)
    assert counts == (0, 0, 5, 5) and u8.shape == (0, 0, 3)
    want = eng.point_mlp(1, torch.as_tensor(v[:5]).cuda(), -torch.as_tensor(n[:5]).cuda())[:, :3]
    assert torch.equal(rgb, want)


def _lines(path, *prefixes):
    return [ln for ln in open(path).read().splitlines() if ln.startswith(prefixes)]


@pytest.mark.gpu
def test_export_marching_cubes(lego, tmp_path, capsys):
    from nerfmeshes_b200 import mesh
    base = dict(limit=1.2, res=96, iso_level=32.0, decimate_faces=4000, save_dir=str(tmp_path), **APPEARANCE)
    p0 = mesh.export_marching_cubes(lego, SimpleNamespace(**base, mesh_name="plain.obj"))
    A = SimpleNamespace(**base, mesh_name="tex.obj", texture_texels=8, cache_name="c.pt", use_cached_mesh=True,
                        override_cache_mesh=False)
    p1 = mesh.export_marching_cubes(lego, A)
    assert _lines(p0, "v ", "vn ") == _lines(p1, "v ", "vn ")
    assert _lines(p1, "mtllib ") == ["mtllib tex.mtl"] and _lines(p1, "usemtl ") == ["usemtl texture"]
    v, f, n, _ = torch.load(os.path.join(str(tmp_path), "c.pt"), weights_only=False)
    assert len(_lines(p1, "vt ")) == 3 * f.shape[0] and len(_lines(p1, "f ")) == f.shape[0]
    assert open(str(tmp_path / "tex.mtl")).read().splitlines()[-1] == "map_Kd tex.png"
    u8, uv, diffuse = _bake(lego, v, f, n, 8)
    assert np.array_equal(T.read_png(str(tmp_path / "tex.png")), u8)
    assert open(p1, "rb").read() == T.obj_text(v.numpy(), f.numpy(), diffuse, n.numpy(), uv, "tex.mtl").encode()
    A.mesh_name = "tex2.obj"
    p2 = mesh.export_marching_cubes(lego, A)                     # served from the cache
    assert open(p2).read().replace("tex2.mtl", "tex.mtl") == open(p1).read()
    assert open(str(tmp_path / "tex2.png"), "rb").read() == open(str(tmp_path / "tex.png"), "rb").read()
    # a cached mesh without faces: the untextured OBJ and one line
    torch.save((v[:10], f[:0], n[:10], None), os.path.join(str(tmp_path), "empty.pt"))
    capsys.readouterr()
    p3 = mesh.export_marching_cubes(lego, SimpleNamespace(**{**A.__dict__, "cache_name": "empty.pt", "mesh_name": "e.obj"}))
    assert "no faces" in capsys.readouterr().out
    assert not os.path.exists(str(tmp_path / "e.mtl")) and len(_lines(p3, "v ")) == 10 and not _lines(p3, "mtllib")


@pytest.mark.gpu
def test_switch_off_is_unchanged(lego, tmp_path):
    from nerfmeshes_b200 import mesh
    base = dict(limit=1.2, res=64, iso_level=32.0, save_dir=str(tmp_path), **APPEARANCE)
    paths = [mesh.export_marching_cubes(lego, SimpleNamespace(**base, mesh_name=f"{k}.obj", **kw))
             for k, kw in enumerate(({}, {"texture_texels": 0}, {"texture_texels": None}))]
    ref = open(paths[0], "rb").read()
    assert all(open(p, "rb").read() == ref for p in paths[1:])
    assert sorted(os.listdir(str(tmp_path))) == ["0.obj", "1.obj", "2.obj"]


@pytest.mark.gpu
def test_texture_beats_vertex_colours(lego):
    """128^3 lego mesh decimated to 2 %, N = 8: the texture's mean colour error at random surface points (bilinear lookup)
    is below the vertex colours' (barycentric interpolation), against the appearance ray at each point."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from mesh_texture_bench import surface_errors
    v, f, n = lego_mesh(lego, 128, 0.02)
    eng = lego._engine()
    _, atlas, _, diffuse, _ = eng.bake_texture(v, n, f, 8, view_disparity=1e-2, near_far=(0.0, 4.0))
    err_tex, err_vert = surface_errors(lego, v, f, n, atlas, diffuse, 8, SimpleNamespace(**APPEARANCE), 1 << 18, seed=3)
    print(f"128^3 lego, {f.shape[0]} faces, N = 8: mean abs colour error texture {err_tex:.5f}, vertex colours {err_vert:.5f}")
    assert err_tex < err_vert
