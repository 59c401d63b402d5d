"""Empty-space skipping on the GPU (NM_FLAG_SKIP_EMPTY, DESIGN 4.15): the grid build and the point lookup against the numpy
restatement (_occupancy_ref); the bit identity of every ray whose skipped samples all have raw sigma <= 0 or NaN, on lego NeRF,
lego BuFF and fern NDC; an all-occupied grid (the dense render, bit for bit) and an all-empty one (no network launch); the
independence from the ray chunk and the network launch size; the error paths; the model-level switch."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _occupancy_ref as R
import _sampler_ref as S

pytestmark = pytest.mark.gpu

f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEGO_FOCAL = float(0.5 * 800 / np.tan(0.5 * 0.6911112))
ALL = ("rgb", "depth", "depth_raw", "acc", "disp", "weights", "mask_weights", "t_vals", "coarse_rgb", "coarse_acc",
       "coarse_disp", "coarse_weights")
BUFF_ALL = ("rgb", "depth", "depth_raw", "acc", "disp", "weights", "mask_weights", "t_vals")
# the skipping render of the lego 64x64 view at the defaults evaluates 0.33 of the network points (0.32 at 800x800, DESIGN
# 4.15); the bound leaves room
LEGO_EVAL_BOUND = 0.45


def _models():
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import BUFF_CFG, LEGO_CFG
    lego = nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval()
    buff = nm.BuFFModel.from_npz(BUFF_CFG, load_npz("weights_lego_buff.npz")).eval()
    fern = nm.NeRFModel.from_npz({**LEGO_CFG, "dataset.use_ndc": True}, load_npz("weights_fern_nerf.npz")).eval()
    return lego, buff, fern


@pytest.fixture(scope="module")
def models():
    return _models()


def pose(theta, phi=-30.0, radius=4.0):
    import nerfmeshes_b200 as nm
    return np.asarray(nm.pose_spherical(theta, phi, radius), f32)


def bits(t):
    return np.ascontiguousarray(t.detach().cpu().numpy(), f32).view(np.int32)


def rows_equal(a, b):
    """per ray: every output value the same bits"""
    x, y = bits(a).reshape(a.shape[0], -1), bits(b).reshape(b.shape[0], -1)
    return (x == y).all(1)


def sigma_at(eng, which, o, d, t):
    """raw sigma of network `which` at o + d*t (fp32, two roundings), with the ray directions as view directions"""
    o, d, t = (np.asarray(v, f32) for v in (o, d, t))
    p = (o[:, None, :] + (d[:, None, :] * t[:, :, None]).astype(f32)).astype(f32)
    dd = np.broadcast_to(d[:, None, :], p.shape)
    out = eng.point_mlp(which, torch.from_numpy(p.reshape(-1, 3).copy()).cuda(), torch.from_numpy(np.ascontiguousarray(dd).reshape(-1, 3)).cuda())
    ev = eng.occupancy_query(which, torch.from_numpy(p.reshape(-1, 3).copy()).cuda())
    return out[:, 3].cpu().numpy().reshape(t.shape), ev.cpu().numpy().reshape(t.shape)


def conservative(eng, which, o, d, t):
    """per ray: every sample the grid skips has raw sigma <= 0 or NaN"""
    sg, ev = sigma_at(eng, which, o, d, t)
    with np.errstate(invalid="ignore"):
        ok = ev | ~(sg > 0)
    return ok.all(1)


def test_build_and_lookup_match_restatement(models):
    lego = models[0]
    eng = lego._engine()
    # the fine net over a cube at G = 200 (two lattice slabs) through nm_grid_sigma; the coarse net over a non-cubic box
    for which, box, G, thr, dil in ((1, (-2.0, -2.0, -2.0, 2.0, 2.0, 2.0), 200, -10.0, 2), (0, (-1.3, -0.7, -1.9, 1.1, 1.6, 0.4), 23, 0.0, 1)):
        lins = [R.lattice(box[a], box[3 + a], G) for a in range(3)]
        for a in range(3):
            assert np.array_equal(lins[a], torch.linspace(box[a], box[3 + a], G + 1, dtype=torch.float32).numpy())
        if which == 1:
            sg = eng.grid_sigma([torch.from_numpy(x) for x in lins]).cpu().numpy()
        else:
            x, y, z = np.meshgrid(*lins, indexing="ij")
            p = torch.from_numpy(np.stack([x, y, z], -1).reshape(-1, 3).copy()).cuda()
            sg = eng.point_mlp(which, p, None, sigma_only=True).cpu().numpy().reshape(G + 1, G + 1, G + 1)
        got = eng.build_occupancy(which, box, G, thr, dil).cpu().numpy().view(np.uint32)
        want = R.build(sg, G, thr, dil)
        assert np.array_equal(got, want), (which, G, int((got != want).sum()))
        occ = R.unpack(got, G)
        assert 0 < occ.mean() < 1, occ.mean()
        rng = np.random.default_rng(G)
        lo, hi = np.asarray(box[:3], f32), np.asarray(box[3:], f32)
        pts = [(lo - 0.2 + rng.random((20000, 3)) * (hi - lo + 0.4)).astype(f32)]
        edge = []                                  # every lattice plane and box face, and a neighbour ulp either side
        for a in range(3):
            for v in lins[a]:
                for w in (v, np.nextafter(v, f32(-1e30)), np.nextafter(v, f32(1e30))):
                    q = pts[0][len(edge) % len(pts[0])].copy()
                    q[a] = w
                    edge.append(q)
        pts.append(np.array(edge, f32))
        nonfin = pts[0][:9].copy()
        for i, v in enumerate((np.nan, np.inf, -np.inf) * 3):
            nonfin[i, i % 3] = v
        pts.append(nonfin)
        P = np.concatenate(pts)
        ev = eng.occupancy_query(which, torch.from_numpy(P).cuda()).cpu().numpy()
        assert np.array_equal(ev, R.evaluated(P, box, G, got))


def _render_pair(eng, fn):
    dense = {k: v.clone() for k, v in fn(False).items()}
    eng.skip_stats()
    skip = {k: v.clone() for k, v in fn(True).items()}
    return dense, skip, eng.skip_stats()


def _check_rays(name, dense, skip, ok, want):
    same = np.ones(len(ok), bool)
    for k in want:
        same &= rows_equal(dense[k], skip[k])
    assert (same | ~ok).all(), f"{name}: {int((~same & ok).sum())} conservative rays differ"
    print(f"{name}: {ok.mean():.4f} of rays conservative, {same.mean():.4f} bit-identical")
    assert ok.mean() > 0.9, ok.mean()


def test_lego_conservative_rays_are_bit_identical(models):
    lego = models[0]
    lego.build_occupancy_grid()
    lego.skip_empty = False
    eng = lego._engine()
    H = W = 64
    P = pose(30.0)
    focal = LEGO_FOCAL * H / 800
    dense, skip, st = _render_pair(eng, lambda s: eng.render_image(P, H, W, focal, 2.0, 6.0, want=ALL, skip_empty=s))
    frac = (st["coarse_evaluated"] + st["fine_evaluated"]) / (st["coarse_seen"] + st["fine_seen"])
    print(f"lego 64x64: evaluated {st}, fraction {frac:.4f}")
    assert st["coarse_seen"] == H * W * 64 and st["fine_seen"] == H * W * 192
    assert frac < LEGO_EVAL_BOUND, frac
    o, d = eng.ray_bundle(P, H, W, focal)
    d = d.reshape(-1, 3).cpu().numpy()
    o = np.broadcast_to(o.cpu().numpy().reshape(1, 3), d.shape)
    t_c = S.stratified(S.linspace(64), 2.0, 6.0, False, False, R=H * W)
    ok = conservative(eng, 0, o, d, t_c) & conservative(eng, 1, o, d, dense["t_vals"].cpu().numpy())
    _check_rays("lego view", dense, skip, ok, ALL)
    # random rays with per-ray origins, some of them starting inside the scene
    g = torch.Generator().manual_seed(5)
    R_ = 4096
    o = (torch.rand(R_, 3, generator=g) * 6 - 3)
    d = torch.nn.functional.normalize(torch.randn(R_, 3, generator=g), dim=1)
    fn = lambda s: eng.render_rays(o.cuda(), d.cuda(), 2.0, 6.0, want=ALL, skip_empty=s)
    dense, skip, _ = _render_pair(eng, fn)
    on, dn = o.numpy(), d.numpy()
    ok = conservative(eng, 0, on, dn, S.stratified(S.linspace(64), 2.0, 6.0, False, False, R=R_)) & \
        conservative(eng, 1, on, dn, dense["t_vals"].cpu().numpy())
    _check_rays("lego random rays", dense, skip, ok, ALL)


def test_buff_and_fern_conservative_rays_are_bit_identical(models):
    _, buff, fern = models
    buff.build_occupancy_grid()
    buff.skip_empty = False
    eng = buff._engine()
    buff._sync_tree(eng)
    H = W = 64
    P = pose(120.0)
    focal = LEGO_FOCAL * H / 800
    dense, skip, st = _render_pair(eng, lambda s: eng.render_image(P, H, W, focal, 2.0, 6.0, buff=True, want=BUFF_ALL, skip_empty=s))
    assert st["fine_seen"] == 0 and st["coarse_seen"] == H * W * 192
    o, d = eng.ray_bundle(P, H, W, focal)
    d = d.reshape(-1, 3).cpu().numpy()
    o = np.broadcast_to(o.cpu().numpy().reshape(1, 3), d.shape)
    _check_rays("buff view", dense, skip, conservative(eng, 0, o, d, dense["t_vals"].cpu().numpy()), BUFF_ALL)

    from conftest import load_npz
    g = load_npz("golden_fern_nerf.npz")
    with pytest.raises(Exception, match="explicit box"):
        fern.build_occupancy_grid()
    fern.build_occupancy_grid(box=(-1.5, -1.5, -1.0, 1.5, 1.5, 1.0))
    fern.skip_empty = False
    eng = fern._engine()
    Hf, Wf, ff = int(g["H"]) // 4, int(g["W"]) // 4, float(g["focal"]) / 4
    Pf = np.asarray(g["pose"], f32)
    dense, skip, st = _render_pair(eng, lambda s: eng.render_image(Pf, Hf, Wf, ff, 0.0, 1.0, ndc=True, want=ALL, skip_empty=s))
    print(f"fern {Hf}x{Wf}: evaluated {st}")
    o, d = eng.ray_bundle(Pf, Hf, Wf, ff, ndc=True)
    o, d = o.reshape(-1, 3).cpu().numpy(), d.reshape(-1, 3).cpu().numpy()
    t_c = S.stratified(S.linspace(64), 0.0, 1.0, False, False, R=Hf * Wf)
    ok = conservative(eng, 0, o, d, t_c) & conservative(eng, 1, o, d, dense["t_vals"].cpu().numpy())
    _check_rays("fern ndc view", dense, skip, ok, ALL)


def test_all_occupied_and_all_empty_grids(models):
    lego = models[0]
    eng = lego._engine()
    H = W = 48
    P = pose(200.0)
    focal = LEGO_FOCAL * H / 800
    for which in (0, 1):
        eng.build_occupancy(which, (-2, -2, -2, 2, 2, 2), 16, float("-inf"), 0)
    dense, skip, st = _render_pair(eng, lambda s: eng.render_image(P, H, W, focal, 2.0, 6.0, want=ALL, skip_empty=s))
    assert st["coarse_evaluated"] == st["coarse_seen"] == H * W * 64 and st["fine_evaluated"] == st["fine_seen"] == H * W * 192
    for k in ALL:
        assert np.array_equal(bits(dense[k]), bits(skip[k])), k
    # an all-empty grid around every sample: no network launch, an empty image
    G = 8
    zero = torch.zeros(eng.occupancy_words(G), dtype=torch.int32, device=eng.device)
    for which in (0, 1):
        eng.set_occupancy(which, (-10, -10, -10, 10, 10, 10), G, zero)
    for white in (False, True):
        eng.configure(white_background=white)
        eng.set_timing(True)
        r = eng.render_image(P, H, W, focal, 2.0, 6.0, want=ALL, skip_empty=True)
        _, pts, launches = eng.mlp_time_ms()
        eng.set_timing(False)
        assert launches == 0 and pts == 0
        assert bool((r["rgb"] == (1.0 if white else 0.0)).all()) and bool((r["acc"] == 0).all()) and bool((r["depth"] == 0).all())
        assert bool((r["weights"] == 0).all())
    eng.configure(white_background=False)
    assert eng.skip_stats()["fine_evaluated"] == 0


def test_independent_of_chunks_and_repeatable(models, tmp_path):
    lego = models[0]
    lego.build_occupancy_grid()
    lego.skip_empty = False
    eng = lego._engine()
    H = W = 40
    P = pose(75.0)
    focal = LEGO_FOCAL * H / 800
    render = lambda: {k: v.clone() for k, v in eng.render_image(P, H, W, focal, 2.0, 6.0, want=ALL, skip_empty=True).items()}
    a = render()
    b = render()
    os.environ["NM_SKIP_CHUNK_POINTS"] = "7777"
    try:
        c = render()
    finally:
        del os.environ["NM_SKIP_CHUNK_POINTS"]
    for k in ALL:
        assert np.array_equal(bits(a[k]), bits(b[k])) and np.array_equal(bits(a[k]), bits(c[k])), k
    # NM_CHUNK_RAYS is read once per process: a child renders with 333-ray chunks
    out = tmp_path / "chunked.npz"
    code = f"""
import sys, numpy as np
sys.path.insert(0, {os.path.join(ROOT, 'tests')!r})
import test_gpu_occupancy as T
lego = T._models()[0]
lego.build_occupancy_grid()
lego.skip_empty = False
eng = lego._engine()
r = eng.render_image(T.pose(75.0), {H}, {W}, {focal!r}, 2.0, 6.0, want=T.ALL, skip_empty=True)
np.savez({str(out)!r}, **{{k: v.cpu().numpy() for k, v in r.items()}})
"""
    env = {**os.environ, "NM_CHUNK_RAYS": "333", "NM_SKIP_CHUNK_POINTS": "1000"}
    subprocess.run([sys.executable, "-c", code], check=True, env=env, cwd=ROOT)
    z = np.load(out)
    for k in ALL:
        assert np.array_equal(z[k].view(np.int32), bits(a[k])), k


def test_error_paths(models):
    import nerfmeshes_b200 as nm
    lego = models[0]
    lego.build_occupancy_grid()
    lego.skip_empty = False
    eng = lego._engine()
    o = torch.tensor([0.0, 0.0, 4.0]).cuda()
    d = torch.nn.functional.normalize(torch.randn(64, 3), dim=1).cuda()
    with pytest.raises(nm.NmError, match="inference"):
        eng.render_rays(o, d, 2.0, 6.0, training=True, skip_empty=True)
    with pytest.raises(nm.NmError, match="inference"):
        eng.render_rays(o, d, 2.0, 6.0, teacher_t=torch.linspace(2, 6, 192).expand(64, 192).contiguous().cuda(), skip_empty=True)
    eng.set_occupancy(1, None, 0, None)
    with pytest.raises(nm.NmError, match="build_occupancy_grid"):
        eng.render_rays(o, d, 2.0, 6.0, skip_empty=True)
    eng._occupancy.add(1)                      # past the binding's own check: the library refuses a missing grid too
    with pytest.raises(nm.NmError, match="no occupancy grid for network 1"):
        eng.render_rays(o, d, 2.0, 6.0, skip_empty=True)
    # weights changed after the build: the model's next skipping render names build_occupancy_grid
    lego.build_occupancy_grid()
    lego.query((o, d, (2.0, 6.0)))
    p = next(lego.model_coarse.parameters())
    with torch.no_grad():
        p.add_(0.0)
    with pytest.raises(nm.NmError, match="build_occupancy_grid"):
        lego.query((o, d, (2.0, 6.0)))
    lego.build_occupancy_grid()
    lego.query((o, d, (2.0, 6.0)))
    lego.train()
    lego.query((o, d, (2.0, 6.0)))             # training renders stay dense
    lego.eval()
    lego.skip_empty = False
    for bad in (dict(box=(0, 0, 0, 0, 1, 1)), dict(res=0), dict(res=2000), dict(dilate=-1), dict(threshold=float("nan"))):
        with pytest.raises(nm.NmError):
            args = dict(box=(-2, -2, -2, 2, 2, 2), res=8, threshold=0.0, dilate=0)
            args.update(bad)
            eng.build_occupancy(0, args["box"], args["res"], args["threshold"], args["dilate"])


def test_model_level_eval_poses(models):
    from nerfmeshes_b200 import eval as ev
    lego = models[0]
    lego.build_occupancy_grid()
    eng = lego._engine()
    assert eng.skip_empty
    H = W = 32
    focal = LEGO_FOCAL * H / 800
    poses = [pose(10.0), pose(190.0, -50.0)]
    res = ev.eval_poses(lego, poses, H, W, focal, 2.0, 6.0)
    for i, P in enumerate(poses):
        r = eng.render_image(P, H, W, focal, 2.0, 6.0, want=["rgb", "disp"], skip_empty=True)
        assert torch.equal(res["rgb"][i], r["rgb"].view(H, W, 3).cpu()) and torch.equal(res["disp"][i], r["disp"].view(H, W).cpu())
    st = eng.skip_stats()
    assert 0 < st["fine_evaluated"] < st["fine_seen"]
    lego.skip_empty = False
    lego._engine()
