"""The mesh rasterizer on the GPU (nm_rasterize_mesh, DESIGN 4.13): rgb, depth, face ids and counts against the numpy
restatement (_raster_ref) bit for bit on the analytic meshes, the 256^3 lego mesh (full and decimated to 10 %) and that mesh
with a texture from nm_bake_texture, at several image sizes and poses, for every NM_RASTER_BIG_FACE_PIXELS; a face that
covers the frame; a second run and a reversed face order; the error paths; compare_with_nerf end to end."""
import math

import numpy as np
import pytest
import torch

import _raster_ref as R
from test_gpu_texture import APPEARANCE, lego_mesh
from test_mesh_raster_reference import CASES, on_grid

pytestmark = pytest.mark.gpu

f32 = np.float32
LEGO_FOCAL = float(0.5 * 800 / np.tan(0.5 * 0.6911112))
THRESHOLDS = (None, "1", str(2 ** 30))


@pytest.fixture(scope="module")
def lego():
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import LEGO_CFG
    return nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval()


@pytest.fixture(scope="module")
def eng(lego):
    return lego._engine()


_FULL = []


def full_mesh(lego):
    """The lego fine net's iso-32 mesh at 256^3, undecimated: world-coordinate (vertices, faces, normals), CPU tensors."""
    if not _FULL:
        from types import SimpleNamespace

        import nerfmeshes_b200 as nm
        _FULL.append(nm.extract_geometry(lego, "cuda", SimpleNamespace(limit=1.2, res=256, iso_level=32.0))[:3])
    return _FULL[0]


def pose(theta, phi=-30.0, radius=4.0):
    import nerfmeshes_b200 as nm
    return np.asarray(nm.pose_spherical(theta, phi, radius), f32)[:3, :4]


def focal_for(W):
    return float(0.5 * W / np.tan(0.5 * 0.6911112))


def same(eng, monkeypatch, v, f, P, H, W, focal, *, z_near=1e-3, colors=None, atlas=None, N=0, bg=(0.25, 0.5, 1.0)):
    """The GPU image equals the restatement's for every threshold; returns the restatement's (rgb, depth, face, counts)."""
    ref = R.rasterize(v, f, P, H, W, focal, z_near=z_near, colors=colors, atlas=atlas, N=N, background=bg)
    for thr in THRESHOLDS:
        if thr is None:
            monkeypatch.delenv("NM_RASTER_BIG_FACE_PIXELS", raising=False)
        else:
            monkeypatch.setenv("NM_RASTER_BIG_FACE_PIXELS", thr)
        outs, counts = eng.rasterize_mesh(v, f, P, H, W, focal, colors=colors, atlas=atlas, N=N, z_near=z_near, background=bg)
        tag = (H, W, thr)
        assert counts == ref[3], (tag, counts, ref[3])
        assert np.array_equal(outs["face"].cpu().numpy(), ref[2]), (tag, int((outs["face"].cpu().numpy() != ref[2]).sum()))
        assert np.array_equal(outs["depth"].cpu().numpy().view(np.int32), ref[1].view(np.int32)), tag
        assert np.array_equal(outs["rgb"].cpu().numpy().view(np.int32), ref[0].view(np.int32)), tag
    return ref


@pytest.mark.parametrize("name", sorted(CASES))
def test_analytic_meshes_match_restatement(eng, monkeypatch, name):
    make, P, z_near = CASES[name]
    v, f = make()
    col = np.random.default_rng(1).random((len(v), 3)).astype(f32)
    for H, W in ((64, 64), (600, 801)):
        for vv in (v, on_grid(v, P)):
            ref = same(eng, monkeypatch, vv, f, P, H, W, focal_for(W), z_near=z_near, colors=col)
            assert ref[3][0] > 0


def _lego_cases():
    return [((800, 800), pose(30.0)), ((600, 801), pose(150.0, -20.0)), ((64, 64), pose(260.0)),
            ((800, 800), pose(75.0, -35.0, 1.2))]      # a close-up: the camera inside the mesh's bounding sphere


@pytest.mark.parametrize("frac", [1.0, 0.1])
def test_lego_mesh_matches_restatement(eng, lego, monkeypatch, frac):
    v, f, _ = full_mesh(lego) if frac == 1.0 else lego_mesh(lego, 256, frac)
    v, f = v.numpy(), f.numpy().astype(np.int64)
    col = np.random.default_rng(2).random((len(v), 3)).astype(f32)
    for (H, W), P in _lego_cases():
        ref = same(eng, monkeypatch, v, f, P, H, W, LEGO_FOCAL * W / 800, colors=col)
        print(f"lego 256^3 x {frac}: {len(f)} faces, {H}x{W}: counts {ref[3]}")
        assert ref[3][0] > 0


def test_lego_texture_matches_restatement(eng, lego, monkeypatch):
    v, f, n = lego_mesh(lego, 256, 0.1)
    _, atlas, _, _, _ = eng.bake_texture(v, n, f, 4, view_disparity=1e-2, near_far=(0.0, 4.0))
    a = atlas.cpu().numpy()
    v, f = v.numpy(), f.numpy().astype(np.int64)
    for (H, W), P in _lego_cases()[:2] + _lego_cases()[3:]:
        same(eng, monkeypatch, v, f, P, H, W, LEGO_FOCAL * W / 800, atlas=a, N=4)
    # mesh.render_mesh takes the uint8 atlas the bake exports, as /255 in fp32
    from nerfmeshes_b200 import mesh
    u8 = (np.clip(a, 0, 1) * 255 + 0.5).astype(np.uint8)
    out = mesh.render_mesh(lego, v, f, pose(30.0), 200, 200, LEGO_FOCAL / 4, texture=(u8, 4))
    a8 = (torch.from_numpy(u8).cuda().float() / 255.0).cpu().numpy()          # the device's division, not numpy's
    ref = R.rasterize(v, f, pose(30.0), 200, 200, LEGO_FOCAL / 4, atlas=a8, N=4)
    assert np.array_equal(out["rgb"].cpu().numpy().view(np.int32), ref[0].view(np.int32)) and out["counts"] == ref[3]


def test_face_covering_the_frame(eng, monkeypatch):
    """One triangle, 0.5 in front of the camera, far wider than the frame; and the same behind a smaller one."""
    v = np.array([[-40, -40, -0.5], [40, -40, -0.5], [0, 40, -0.5], [-0.1, -0.1, -0.3], [0.1, -0.1, -0.3], [0, 0.1, -0.3]], f32)
    P = np.concatenate([np.eye(3, dtype=f32), np.zeros((3, 1), f32)], 1)
    col = np.random.default_rng(3).random((6, 3)).astype(f32)
    for f in (np.array([[0, 1, 2]]), np.array([[0, 1, 2], [3, 4, 5]]), np.array([[3, 4, 5], [2, 1, 0]])):
        for H, W in ((64, 64), (600, 801)):
            ref = same(eng, monkeypatch, v, f, P, H, W, focal_for(W), colors=col)
            assert (ref[2] >= 0).all()


def test_second_run_and_reversed_faces(eng, lego):
    v, f, _ = lego_mesh(lego, 256, 0.1)
    col = torch.rand((v.shape[0], 3), generator=torch.Generator().manual_seed(4))
    P = pose(30.0)
    a, ca = eng.rasterize_mesh(v, f, P, 800, 800, LEGO_FOCAL, colors=col)
    b, cb = eng.rasterize_mesh(v, f, P, 800, 800, LEGO_FOCAL, colors=col)
    assert ca == cb and all(torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)) for k in a)
    F = f.shape[0]
    c, cc = eng.rasterize_mesh(v, f.flip(0), P, 800, 800, LEGO_FOCAL, colors=col)
    assert cc == ca
    mapped = torch.where(c["face"] >= 0, F - 1 - c["face"], c["face"])
    diff = mapped != a["face"]
    # a different face only where two faces tie in depth at the sample
    assert torch.equal(c["depth"].view(torch.int32), a["depth"].view(torch.int32))
    assert int(diff.sum()) < 50
    assert torch.equal(c["rgb"][~diff].view(torch.int32), a["rgb"][~diff].view(torch.int32))


def test_errors(eng):
    from nerfmeshes_b200 import NmError
    make, P, _ = CASES["sphere"]
    v, f = make()
    col = np.zeros((len(v), 3), f32)
    for kw, text in ((dict(H=0), "outside [1, 16384]"), (dict(W=16385), "outside [1, 16384]"), (dict(focal=0.0), "focal length"),
                     (dict(focal=-2.0), "focal length"), (dict(z_near=0.0), "z_near"), (dict(z_near=math.inf), "z_near")):
        args = dict(H=32, W=32, focal=40.0, z_near=1e-3)
        args.update(kw)
        with pytest.raises(NmError, match=text.replace("[", r"\[")):
            eng.rasterize_mesh(v, f, P, args["H"], args["W"], args["focal"], colors=col, z_near=args["z_near"])
    for N in (1, 65):
        with pytest.raises(NmError, match=f"N = {N} outside"):
            eng.rasterize_mesh(v, f, P, 32, 32, 40.0, atlas=np.zeros((8, 8, 3), f32), N=N)
    with pytest.raises(NmError, match="null vertex colour pointer"):
        eng.rasterize_mesh(v, f, P, 32, 32, 40.0)
    for bad in (len(v), -1):
        g = f.copy()
        g[17, 2] = bad
        before = eng.launch_count()
        with pytest.raises(NmError, match=r"mesh raster: a face index lies outside \[0, V\) \(nothing was drawn\)"):
            eng.rasterize_mesh(v, g, P, 32, 32, 40.0, colors=col)
        assert eng.launch_count() - before <= 4
        eng.check_flags()                                          # reported once
    # nothing drawn: the background, and zero counts (the check raises after the image is written)
    g = f.copy()
    g[3, 0] = len(v) + 5
    outs = {k: torch.full(s, 7, dtype=t, device="cuda") for k, s, t in (("rgb", (32, 32, 3), torch.float32),
                                                                         ("depth", (32, 32), torch.float32),
                                                                         ("face", (32, 32), torch.int32))}
    import ctypes as C
    from nerfmeshes_b200 import _lib as L
    cnt = (C.c_int64 * 3)(9, 9, 9)
    vt, ft = torch.from_numpy(v).cuda(), torch.from_numpy(g).int().cuda()
    ct = torch.from_numpy(col).cuda()
    Pc = np.ascontiguousarray(P, f32)
    bg = (C.c_float * 3)(0.25, 0.5, 0.75)
    assert eng.lib.nm_rasterize_mesh(eng._h, C.c_void_p(vt.data_ptr()), len(v), C.c_void_p(ft.data_ptr()), len(g), Pc.ctypes.data,
                                     32, 32, 40.0, 1e-3, 0, C.c_void_p(ct.data_ptr()), None, 0, bg,
                                     *[C.c_void_p(outs[k].data_ptr()) for k in ("rgb", "depth", "face")], cnt, eng._stream()) == 0
    assert tuple(cnt) == (0, 0, 0)
    assert (outs["face"] == -1).all() and (outs["depth"] == 0).all()
    assert torch.equal(outs["rgb"], torch.tensor([0.25, 0.5, 0.75], device="cuda").expand(32, 32, 3))
    with pytest.raises(NmError, match="mesh raster: a face index"):
        eng.check_flags()
    eng.check_flags()
    # an empty mesh: background, no raster kernel
    e3 = np.zeros((0, 3), f32)
    before = eng.launch_count()
    outs, counts = eng.rasterize_mesh(e3, np.zeros((0, 3), np.int32), P, 20, 30, 40.0, colors=e3, background=(0.1, 0.2, 0.3))
    assert counts == (0, 0, 0) and eng.launch_count() - before == 1
    assert torch.equal(outs["rgb"], torch.tensor([0.1, 0.2, 0.3], device="cuda").expand(20, 30, 3))
    assert (outs["face"] == -1).all() and (outs["depth"] == 0).all()


def test_atlas_must_fit_the_mesh(eng, lego):
    """An atlas baked for another N or another face count would be read past its end: it is rejected before any launch, as
    are an integer atlas at the engine (mesh.render_mesh scales a uint8 one) and a face index that does not fit int32."""
    from nerfmeshes_b200 import NmError, mesh
    v, f, n = lego_mesh(lego, 64, 0.1)
    _, atlas, _, _, _ = eng.bake_texture(v, n, f, 4, view_disparity=1e-2, near_far=(0.0, 4.0))
    P = pose(30.0)
    out, _ = eng.rasterize_mesh(v, f, P, 64, 64, focal_for(64), atlas=atlas, N=4)
    before = eng.launch_count()
    with pytest.raises(NmError, match=r"does not fit .* at N = 5"):
        eng.rasterize_mesh(v, f, P, 64, 64, focal_for(64), atlas=atlas, N=5)
    full = torch.cat([f, f.flip(0)])                            # the same N, more faces than the atlas was baked for
    with pytest.raises(NmError, match=f"does not fit {full.shape[0]} faces at N = 4"):
        eng.rasterize_mesh(v, full, P, 64, 64, focal_for(64), atlas=atlas, N=4)
    with pytest.raises(NmError, match="does not fit"):
        mesh.render_mesh(eng, v, full, P, 64, 64, focal_for(64), texture=(atlas, 4))
    with pytest.raises(NmError, match="torch.uint8 atlas"):
        eng.rasterize_mesh(v, f, P, 64, 64, focal_for(64), atlas=(atlas * 255).to(torch.uint8), N=4)
    wide = f.long()
    wide[5, 1] = 2 ** 32 + 3                                    # an int32 cast would make it vertex 3
    with pytest.raises(NmError, match=r"a face index lies outside \[0, V\)"):
        eng.rasterize_mesh(v, wide, P, 64, 64, focal_for(64), colors=torch.zeros_like(v))
    assert eng.launch_count() == before
    eng.check_flags()
    # the uint8 atlas through render_mesh is the float one over 255
    u8 = (atlas.clamp(0, 1) * 255 + 0.5).to(torch.uint8)
    a = mesh.render_mesh(eng, v, f, P, 64, 64, focal_for(64), texture=(u8, 4))
    b, _ = eng.rasterize_mesh(v, f, P, 64, 64, focal_for(64), atlas=u8.cuda().float() / 255.0, N=4)
    assert torch.equal(a["rgb"], b["rgb"]) and torch.equal(a["face"], out["face"])


def test_compare_with_nerf(lego):
    """The lego 256^3 mesh with mesh_appearance's colours against the NeRF at 4 ring poses, 200 x 200."""
    from types import SimpleNamespace

    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import mesh
    v, f, n = full_mesh(lego)
    diffuse = mesh.mesh_appearance(lego, v, n, SimpleNamespace(**APPEARANCE))
    poses = [nm.pose_spherical(th, -30.0, 4.0) for th in (0.0, 90.0, 180.0, 270.0)]
    r = mesh.compare_with_nerf(lego, v, f, poses, 200, 200, LEGO_FOCAL / 4, 2.0, 6.0, diffuse=diffuse)
    print("compare_with_nerf, lego 256^3, 4 poses, 200x200:", {k: r[k] for k in ("psnr", "psnr_masked", "iou", "depth_mae")},
          r["mean"])
    for k in ("psnr", "psnr_masked", "iou", "depth_mae"):
        assert len(r[k]) == 4 and all(math.isfinite(x) for x in r[k]), (k, r[k])
    # first measured on an H100: mean IoU 0.978 (per view 0.970 to 0.987), mean masked PSNR 18.58 dB (17.46 to 19.09)
    assert r["mean"]["iou"] > 0.95 and min(r["iou"]) > 0.93
    assert r["mean"]["psnr_masked"] > 17.5 and min(r["psnr_masked"]) > 16.5
    assert len(r["both"]) == 4 and min(r["both"]) > 1000
    # a camera looking away from the object: no pixel both cover, NaN for the masked values of that view only
    away = np.asarray(nm.pose_spherical(0.0, -30.0, 4.0), f32).copy()
    away[:3, 0], away[:3, 2] = -away[:3, 0], -away[:3, 2]          # turned half a turn about its own up axis
    r2 = mesh.compare_with_nerf(lego, v, f, [poses[0], away], 200, 200, LEGO_FOCAL / 4, 2.0, 6.0, diffuse=diffuse)
    assert r2["both"][1] == 0 and math.isnan(r2["psnr_masked"][1]) and math.isnan(r2["depth_mae"][1])
    assert r2["mean"]["psnr_masked"] == r2["psnr_masked"][0] and r2["mean"]["depth_mae"] == r2["depth_mae"][0]


def test_compare_with_nerf_rejects_ndc(lego):
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from nerfmeshes_b200 import mesh
    from test_gpu_parity import LEGO_CFG
    fern = nm.NeRFModel.from_npz({**LEGO_CFG, "dataset.use_ndc": True}, load_npz("weights_fern_nerf.npz")).eval()
    v = np.zeros((3, 3), f32)
    with pytest.raises(NotImplementedError, match="NDC"):
        mesh.compare_with_nerf(fern, v, np.array([[0, 1, 2]]), [np.eye(4, dtype=f32)], 8, 8, 10.0, 0.0, 1.0, diffuse=v)
