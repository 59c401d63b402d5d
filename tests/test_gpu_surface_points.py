"""Surface point clouds on the GPU (nm_surface_points, DESIGN 4.14): the kernel's rows against the numpy restatement
(_surface_ref) bit for bit, fed the same depth_raw / acc / rgb and the directions of eng.ray_bundle, on synthetic maps
through the ABI and on lego NeRF and BuFF renders; a second run; render outputs unchanged by a call; the error paths;
network normals; the native PLY writer against the python formatter; the lego cloud's distance to the 256^3 marching-cubes
mesh; the sharded entry on several GPUs."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _surface_ref as R

pytestmark = pytest.mark.gpu

f32 = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEGO_FOCAL = float(0.5 * 800 / np.tan(0.5 * 0.6911112))


def thr_for(size):
    """dist_threshold 0.002 (a squared distance) scaled with the pixel footprint from 800 pixels to `size`: the default keeps
    no lego pixel at 64^2, where two pixels already lie about 0.09 apart on the surface."""
    return 0.002 * (800.0 / size) ** 2


@pytest.fixture(scope="module")
def lego():
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_parity import LEGO_CFG
    return nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval()


@pytest.fixture(scope="module")
def eng(lego):
    return lego._engine()


def pose(theta, phi=-30.0, radius=4.0):
    import nerfmeshes_b200 as nm
    return np.asarray(nm.pose_spherical(theta, phi, radius), f32)


def bits(t):
    a = t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
    return np.ascontiguousarray(a, f32).view(np.int32)


def same(eng, P, H, W, focal, depth_raw, acc, rgb, **kw):
    """The kernel's rows equal the restatement's; returns them (numpy) and the restatement's keep mask."""
    o, d = eng.ray_bundle(P, H, W, focal)
    ref = R.surface_points(o.cpu().numpy(), d.cpu().numpy(), depth_raw.cpu().numpy(), acc.cpu().numpy(), rgb.cpu().numpy(), H, W,
                           min_acc=kw.get("min_acc", 1.0), step=kw.get("step", 2), dist_threshold=kw.get("dist_threshold", 0.002),
                           min_count_=kw.get("min_count", 15))
    outs, n = eng.surface_points(P, H, W, focal, depth_raw, acc, rgb, **kw)
    tag = (H, W, kw)
    assert n == len(ref[3]), (tag, n, len(ref[3]))
    for k, name in enumerate(("points", "normals", "colors")):
        assert np.array_equal(bits(outs[name]), bits(ref[k])), (tag, name)
    assert np.array_equal(outs["pixel"].cpu().numpy(), ref[3]), tag
    return outs, ref


def synthetic(eng, P, H, W, focal, seed):
    """Depth maps the kernel sees through the ABI: a plane with a step, a NaN / inf sprinkle, acc at and just below 1."""
    rng = np.random.default_rng(seed)
    o, d = eng.ray_bundle(P, H, W, focal)
    o, d = o.cpu().numpy().astype(np.float64), d.cpu().numpy().astype(np.float64)
    n = np.array([0.3, 0.2, 0.9])
    with np.errstate(divide="ignore", invalid="ignore"):
        t = (0.1 - o @ n) / (d @ n)
    t = np.where(np.isfinite(t) & (t > 0), t, 0)
    t[:, W // 3:] += 0.3
    t += rng.normal(0, 1e-3, t.shape) * (rng.random(t.shape) < 0.2)
    t = t.astype(f32)
    flat = t.reshape(-1)
    k = rng.choice(flat.size, size=max(1, flat.size // 50), replace=False)
    flat[k] = rng.choice(np.array([np.nan, np.inf, -np.inf, 0.0], f32), k.size)
    acc = rng.choice(np.array([1.0, 1.0, 1.0, np.nextafter(f32(1), f32(0)), 0.5], f32), t.shape)
    rgb = rng.random((H * W, 3)).astype(f32)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return dev(t.reshape(-1)), dev(acc.reshape(-1)), dev(rgb)


@pytest.mark.parametrize("H,W", [(1, 1), (1, 37), (29, 1), (64, 64), (100, 80), (257, 129)])
def test_synthetic_maps_match_restatement(eng, H, W):
    P = pose(30.0)
    focal = LEGO_FOCAL * max(H, W) / 800
    dr, acc, rgb = synthetic(eng, P, H, W, focal, H * 1000 + W)
    for step in (0, 1, 2, 3, 8):
        for min_acc, thr, mc in ((1.0, 0.002, R.min_count(step, 0.6)), (0.99, 1e-4, 1), (0.5, 0.05, R.min_count(step, 0.3))):
            same(eng, P, H, W, focal, dr, acc, rgb, min_acc=min_acc, step=step, dist_threshold=thr, min_count=mc)


def test_lego_renders_match_restatement(eng):
    """Real depth maps: lego at 64^2, 100 x 80 and one 800^2 pose, at min_acc 1.0, 0.99 and 0.5; a second call gives the same
    bits, and the render's own outputs are the same bits before and after a call."""
    for (H, W), th in (((64, 64), 30.0), ((100, 80), 200.0), ((800, 800), 120.0)):
        P = pose(th)
        focal = LEGO_FOCAL * max(H, W) / 800
        r = eng.render_image(P, H, W, focal, 2.0, 6.0, want=("rgb", "depth", "depth_raw", "acc", "disp"))
        kept = []
        thr = thr_for(max(H, W))
        for min_acc in (1.0, 0.99, 0.5):
            outs, ref = same(eng, P, H, W, focal, r["depth_raw"], r["acc"], r["rgb"], min_acc=min_acc, dist_threshold=thr)
            kept.append(len(ref[3]))
            again, n2 = eng.surface_points(P, H, W, focal, r["depth_raw"], r["acc"], r["rgb"], min_acc=min_acc, dist_threshold=thr)
            assert n2 == len(ref[3]) and all(torch.equal(again[k], outs[k]) for k in outs)
        print(f"lego {H}x{W}: kept at min_acc 1.0 / 0.99 / 0.5: {kept} of {H * W}")
        assert kept[0] <= kept[1] <= kept[2] and kept[0] > 0
        r2 = eng.render_image(P, H, W, focal, 2.0, 6.0, want=("rgb", "depth", "depth_raw", "acc", "disp"))
        for k in r:
            assert np.array_equal(bits(r[k]), bits(r2[k])), k


def test_buff_render_matches_restatement():
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from nerfmeshes_b200 import mesh
    from test_gpu_parity import BUFF_CFG
    buff = nm.BuFFModel.from_npz(BUFF_CFG, load_npz("weights_lego_buff.npz")).eval()
    e = buff._engine()
    poses = [pose(30.0), pose(250.0, -60.0)]
    H, W, focal = 96, 72, LEGO_FOCAL * 96 / 800
    res = mesh.surface_points(buff, poses, H, W, focal, 2.0, 6.0, min_acc=0.99, dist_threshold=thr_for(H))
    off = 0
    for i, P in enumerate(poses):
        r = e.render_image(P, H, W, focal, 2.0, 6.0, buff=True, want=("rgb", "depth_raw", "acc"))
        outs, ref = same(e, P, H, W, focal, r["depth_raw"], r["acc"], r["rgb"], min_acc=0.99, dist_threshold=thr_for(H))
        n = len(ref[3])
        assert res["counts"][i] == n and n > 0
        for k in ("points", "normals", "colors", "pixel"):
            assert torch.equal(res[k][off:off + n], outs[k]), k
        assert (res["view"][off:off + n] == i).all()
        off += n
    assert off == res["points"].shape[0]


def test_surface_points_views_and_pixels(lego, eng):
    """mesh.surface_points concatenates the per-view rows in pose order; view and pixel index back into each view's maps."""
    from nerfmeshes_b200 import mesh
    poses = mesh.surface_ray_poses(3, 2)
    H, W, focal = 48, 40, LEGO_FOCAL * 48 / 800
    res = mesh.surface_points(lego, poses, H, W, focal, 2.0, 6.0, min_acc=0.5, dist_threshold=thr_for(H))
    assert len(res["counts"]) == 6 and sum(res["counts"]) == res["points"].shape[0] > 0
    assert res["view"].dtype == res["pixel"].dtype == torch.int32
    assert torch.equal(res["view"], torch.repeat_interleave(torch.arange(6, device="cuda", dtype=torch.int32),
                                                            torch.tensor(res["counts"], device="cuda")))
    for i, P in enumerate(poses):
        sel = res["view"] == i
        r = eng.render_image(P, H, W, focal, 2.0, 6.0, want=("rgb", "depth_raw", "acc"))
        _, d = eng.ray_bundle(P, H, W, focal)
        pix = res["pixel"][sel].long()
        assert (pix[1:] > pix[:-1]).all()
        assert torch.equal(res["colors"][sel], r["rgb"][pix]) and torch.equal(res["normals"][sel], -d.reshape(-1, 3)[pix])
        assert (r["depth_raw"][pix] > 0).all() and (r["acc"][pix] >= 0.5).all()
    again = mesh.surface_points(lego, poses, H, W, focal, 2.0, 6.0, min_acc=0.5, dist_threshold=thr_for(H))
    assert all(torch.equal(again[k], res[k]) for k in ("points", "normals", "colors", "view", "pixel"))


def test_errors(lego, eng):
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from nerfmeshes_b200 import NmError, mesh
    from test_gpu_parity import LEGO_CFG
    P = pose(30.0)
    r = eng.render_image(P, 16, 16, 22.0, 2.0, 6.0, want=("rgb", "depth_raw", "acc"))
    before = eng.launch_count()
    with pytest.raises(NmError, match=r"step 9 outside \[0, 8\]"):
        eng.surface_points(P, 16, 16, 22.0, r["depth_raw"], r["acc"], r["rgb"], step=9)
    with pytest.raises(NmError, match="min_count 0"):
        eng.surface_points(P, 16, 16, 22.0, r["depth_raw"], r["acc"], r["rgb"], min_count=0)
    with pytest.raises(NmError, match="focal length"):
        eng.surface_points(P, 16, 16, 0.0, r["depth_raw"], r["acc"], r["rgb"])
    with pytest.raises(NmError, match="must hold 16 x 15 pixels"):
        eng.surface_points(P, 16, 15, 22.0, r["depth_raw"], r["acc"], r["rgb"])
    with pytest.raises(ValueError, match="prob_threshold"):
        mesh.surface_points(lego, [P], 16, 16, 22.0, 2.0, 6.0, prob_threshold=1.5)
    assert eng.launch_count() == before
    eng.check_flags()
    fern = nm.NeRFModel.from_npz({**LEGO_CFG, "dataset.use_ndc": True}, load_npz("weights_fern_nerf.npz")).eval()
    with pytest.raises(NotImplementedError, match="NDC"):
        mesh.surface_points(fern, [P], 8, 8, 10.0, 0.0, 1.0)
    # nothing kept: an empty cloud of the right shapes
    res = mesh.surface_points(lego, [P], 16, 16, 22.0, 2.0, 6.0, step=8, prob_threshold=1.0, dist_threshold=0.0)
    assert res["counts"] == [0] and res["points"].shape == (0, 3) and res["view"].shape == (0,)


def test_network_normals(lego, eng, capsys):
    from nerfmeshes_b200 import mesh
    poses = [pose(30.0), pose(160.0, -50.0)]
    H = W = 64
    focal = LEGO_FOCAL * 64 / 800
    a = mesh.surface_points(lego, poses, H, W, focal, 2.0, 6.0, dist_threshold=thr_for(H))
    capsys.readouterr()
    b = mesh.surface_points(lego, poses, H, W, focal, 2.0, 6.0, dist_threshold=thr_for(H), network_normals=True)
    printed = capsys.readouterr().out
    for k in ("points", "colors", "view", "pixel"):
        assert torch.equal(a[k], b[k]), k
    assert a["counts"] == b["counts"] and a["points"].shape[0] > 100
    _, g = lego.density_gradient(a["points"])
    norm = g.norm(dim=1)
    ok = torch.isfinite(norm) & (norm > 0)
    fb = int((~ok).sum())
    assert torch.equal(b["normals"][~ok], a["normals"][~ok])
    assert (b["normals"][ok].norm(dim=1) - 1).abs().max() < 1e-5
    assert torch.allclose(b["normals"][ok], -g[ok] / norm[ok, None], atol=1e-6)
    assert (f"{fb} of {a['points'].shape[0]} surface points" in printed) == (fb > 0), printed
    # the network normal mostly faces the camera: cos(n_net, -d) > 0
    print(f"network normals: {fb} fallbacks; facing the camera: {float(((b['normals'] * a['normals']).sum(1) > 0).float().mean()):.3f}")
    # first measured on an H100: 0.764 (no fallbacks); the points sit at the expected hit distance, where the field's
    # gradient still turns with the thin structures and the partially transparent shell
    assert float(((b["normals"] * a["normals"]).sum(1) > 0).float().mean()) > 0.7


def test_export_ply_native_equals_python(lego, tmp_path):
    from nerfmeshes_b200 import mesh
    res = mesh.surface_points(lego, [pose(30.0)], 64, 64, LEGO_FOCAL * 64 / 800, 2.0, 6.0, min_acc=0.5, dist_threshold=thr_for(64))
    assert res["points"].shape[0] > 0
    for binary in (False, True):
        mesh.export_ply(res["points"], res["colors"], res["normals"], tmp_path / "n.ply", binary=binary)
        mesh._export_ply_python(res["points"], res["colors"], res["normals"], tmp_path / "p.ply", binary=binary)
        data = (tmp_path / "n.ply").read_bytes()
        assert data == (tmp_path / "p.ply").read_bytes()
        assert data == R.ply_bytes(res["points"].cpu().numpy(), res["colors"].cpu().numpy(), res["normals"].cpu().numpy(), binary)
        p, n, c = R.read_ply(data)
        assert np.array_equal(bits(p), bits(res["points"])) and np.array_equal(bits(n), bits(res["normals"]))


def test_export_surface_points(lego, tmp_path):
    from types import SimpleNamespace

    from nerfmeshes_b200 import mesh
    args = SimpleNamespace(save_dir=str(tmp_path), img_size=48, focal=LEGO_FOCAL * 48 / 800, min_acc=0.5, ply_binary=True,
                           dist_threshold=thr_for(48))
    path = mesh.export_surface_points(lego, args)
    assert path == os.path.join(str(tmp_path), "lego-sampling.ply")
    p, n, c = R.read_ply(open(path, "rb").read())
    res = mesh.surface_points(lego, mesh.surface_ray_poses(), 48, 48, args.focal, 2.0, 6.0, min_acc=0.5,
                              dist_threshold=thr_for(48))
    assert res["points"].shape[0] > 0 and np.array_equal(bits(p), bits(res["points"])) and np.array_equal(c, R.quantise(res["colors"].cpu().numpy()))


def test_cloud_lies_on_the_mesh(lego, eng):
    """The 32 ring views at 200 x 200 (dist_threshold scaled to the pixel footprint) against the 256^3 marching-cubes mesh: the distance from every kept point to 2^20 dense
    area-weighted samples of the mesh (nm_mesh_sample, nm_nearest).  The sampling floor is the same distance for a second
    sample set of the mesh itself."""
    from test_gpu_mesh_raster import full_mesh
    from nerfmeshes_b200 import mesh
    v, f, _ = full_mesh(lego)
    samples = eng.mesh_sample(v, f, 1 << 20, 1)
    floor = eng.nearest(eng.mesh_sample(v, f, 1 << 16, 2), samples)[0].sqrt()
    res = mesh.surface_points(lego, mesh.surface_ray_poses(), 200, 200, LEGO_FOCAL / 4, 2.0, 6.0, dist_threshold=thr_for(200))
    d = eng.nearest(res["points"], samples)[0].sqrt()
    q = lambda x, p: float(torch.quantile(x.double()[:1 << 24], p))
    stats = dict(points=int(d.numel()), median=q(d, 0.5), p95=q(d, 0.95), floor_median=q(floor, 0.5), floor_p95=q(floor, 0.95))
    print("surface cloud vs 256^3 mesh, 32 views at 200x200:", stats)
    # first measured on an H100: 78,222 points, median 0.0091 and p95 0.0191 world units, against a sampling floor of 0.0022
    # and 0.0044 (the 256^3 grid spacing is 0.0094)
    assert stats["points"] > 60000
    assert stats["median"] < 0.012 and stats["p95"] < 0.025


@pytest.mark.multigpu
def test_multi_gpu_surface_points():
    world = min(torch.cuda.device_count(), 4)
    if world < 2:
        pytest.skip("needs 2 GPUs")
    port = 29700 + os.getpid() % 90
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "_surface_multi_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0 and f"SURFACE_MULTI_OK {world}" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
