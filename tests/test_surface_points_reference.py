"""The surface point filter's restatement (_surface_ref, DESIGN 4.14) against an independent torch float32 implementation built
from replicate-padded slices, on random and structured depth maps; the min_count formula; the 32 ring poses; both PLY
encodings of the native writer and the python formatter against the restatement's bytes, read back; argument rejections of
nm_surface_points and nm_export_ply without a device."""
import ctypes as C

import numpy as np
import pytest
import torch

import _surface_ref as R

f32 = np.float32
FOCAL = 1111.1111


def camera(H, W, focal=FOCAL, theta=30.0, phi=-30.0, radius=4.0):
    """(o (3,), d (H,W,3)) float32 of the oracle's get_ray_bundle for a ring pose."""
    import nerfmeshes_b200 as nm
    from oracle import nerf_oracle as O
    pose = torch.from_numpy(np.asarray(nm.pose_spherical(theta, phi, radius), f32))
    o, d = O.get_ray_bundle(H, W, focal, pose)
    return o.numpy().astype(f32), d.numpy().astype(f32)


def torch_filter(o, d, depth_raw, acc, rgb, H, W, min_acc, s, thr, min_count):
    """Independent: replicate padding of the (3,H,W) point map stands for the clamped neighbour index."""
    o, d = torch.from_numpy(o), torch.from_numpy(d).reshape(H, W, 3)
    dr, ac = torch.from_numpy(depth_raw).reshape(H, W), torch.from_numpy(acc).reshape(H, W)
    t = torch.where(ac >= torch.tensor(min_acc, dtype=torch.float32), dr, torch.zeros(()))
    P = (o + d * t[..., None]).permute(2, 0, 1).contiguous()                 # (3,H,W)
    Pp = torch.nn.functional.pad(P[None], (s, s, s, s), mode="replicate")[0] if s else P
    cnt = torch.zeros((H, W), dtype=torch.int64)
    th = torch.tensor(thr, dtype=torch.float32)
    for a in range(2 * s + 1):
        for b in range(2 * s + 1):
            e = Pp[:, a:a + H, b:b + W] - P
            cnt += ((e[0] * e[0] + e[1] * e[1]) + e[2] * e[2] < th).long()
    keep = (cnt >= min_count) & (t > 0)
    flat = keep.reshape(-1)
    pts = P.permute(1, 2, 0).reshape(-1, 3)[flat]
    return pts.numpy(), (-d).reshape(-1, 3)[flat].numpy(), torch.from_numpy(rgb).reshape(-1, 3)[flat].numpy(), \
        torch.nonzero(flat).reshape(-1).int().numpy(), cnt.numpy()


def bits(a):
    return np.ascontiguousarray(a, f32).view(np.int32)


def agree(o, d, depth_raw, acc, H, W, *, min_acc=1.0, s=2, thr=0.002, mc=15, rgb=None):
    rgb = np.random.default_rng(3).random((H * W, 3)).astype(f32) if rgb is None else rgb
    ref = R.surface_points(o, d, depth_raw, acc, rgb, H, W, min_acc=min_acc, step=s, dist_threshold=thr, min_count_=mc)
    ind = torch_filter(o, d, np.ascontiguousarray(depth_raw, f32).reshape(-1), np.ascontiguousarray(acc, f32).reshape(-1), rgb,
                       H, W, min_acc, s, thr, mc)
    assert np.array_equal(ref[4], ind[4]), "counts differ"
    for k in range(3):
        assert np.array_equal(bits(ref[k]), bits(ind[k])), k
    assert np.array_equal(ref[3], ind[3])
    return ref


def plane_depth(o, d, normal, offset):
    """t where the rays meet the plane n.x = offset (0 where they miss or go backwards)."""
    n = np.asarray(normal, np.float64)
    den = d.astype(np.float64) @ n
    with np.errstate(divide="ignore", invalid="ignore"):
        t = (offset - o.astype(np.float64) @ n) / den
    return np.where(np.isfinite(t) & (t > 0), t, 0).astype(f32)


def sphere_depth(o, d, c, r):
    oc = o.astype(np.float64) - np.asarray(c, np.float64)
    dd = d.astype(np.float64)
    b = dd @ oc
    q = b * b - (oc @ oc - r * r) * (dd * dd).sum(-1)
    t = (-b - np.sqrt(np.maximum(q, 0))) / (dd * dd).sum(-1)
    return np.where(q > 0, t, 0).astype(f32)


def test_min_count():
    assert R.min_count(2, 0.6) == 15
    from nerfmeshes_b200 import mesh
    assert mesh.surface_min_count(2, 0.6) == 15
    assert mesh.surface_min_count(2, 0.5) == 13 == R.min_count(2, 0.5)      # 24 * 0.5 = 12 exactly: sum > 12 needs 13
    assert mesh.surface_min_count(1, 0.25) == 3                              # 8 * 0.25 = 2 exactly
    assert mesh.surface_min_count(0, 0.6) == 1 and mesh.surface_min_count(3, 1.0) == 49 and mesh.surface_min_count(2, 0.0) == 1
    for s in range(4):
        for p in np.linspace(0, 1, 41):
            size = (2 * s + 1) ** 2 - 1
            m = mesh.surface_min_count(s, float(p))
            assert all((k > size * float(p)) == (k >= m) for k in range(size + 2)), (s, p)
    for bad in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError):
            mesh.surface_min_count(2, bad)


@pytest.mark.parametrize("s", [0, 1, 2, 3])
def test_random_maps(s):
    rng = np.random.default_rng(10 + s)
    for H, W in ((1, 1), (1, 17), (13, 1), (24, 40), (37, 29)):
        o, d = camera(H, W)
        depth = rng.uniform(3.9, 4.1, (H, W)).astype(f32)
        acc = rng.choice(np.array([1.0, np.nextafter(f32(1), f32(0)), 0.5, 0.999, 1.0000001], f32), (H, W))
        for min_acc in (1.0, 0.99, 0.5):
            for thr, mc in ((0.002, R.min_count(s, 0.6)), (1e-4, 1), (2e-5, R.min_count(s, 0.3))):
                agree(o, d, depth, acc, H, W, min_acc=min_acc, s=s, thr=thr, mc=mc)


@pytest.mark.parametrize("s", [0, 1, 2, 3])
def test_structured_maps(s):
    H, W = 32, 48
    o, d = camera(H, W)
    ones = np.ones((H, W), f32)
    mc = R.min_count(s, 0.6)
    plane = plane_depth(o, d, (0.3, 0.2, 0.9), 0.1)
    ref = agree(o, d, plane, ones, H, W, s=s, mc=mc)
    assert ref[5].all(), "a plane facing the camera keeps every pixel"
    step = plane.copy()
    step[:, W // 2:] += 0.5                                      # a depth step
    agree(o, d, step, ones, H, W, s=s, mc=mc)
    ref = agree(o, d, step, ones, H, W, s=s, mc=(2 * s + 1) ** 2)  # every neighbour required: the s columns on each side fail
    cols = ref[5].all(0)
    assert not cols[W // 2 - s:W // 2 + s].any() and cols[:W // 2 - s].all() and cols[W // 2 + s:].all()
    sph = sphere_depth(o, d, (0.0, 0.0, 0.0), 0.04)
    ref = agree(o, d, sph, ones, H, W, s=s, mc=mc)
    assert 0 < ref[5].sum() < (sph > 0).sum() + 1
    agree(o, d, np.zeros((H, W), f32), ones, H, W, s=s, mc=mc)              # nothing hit: nothing kept
    assert not R.surface_points(o, d, np.zeros((H, W), f32), ones, np.zeros((H * W, 3), f32), H, W, step=s)[5].any()
    bad = plane.copy()
    bad[3, 4], bad[10, 10], bad[20, 30], bad[0, 0] = np.nan, np.inf, -np.inf, np.nan
    ref = agree(o, d, bad, ones, H, W, s=s, mc=mc)
    assert not ref[5][3, 4] and not ref[5][10, 10] and not ref[5][20, 30]
    acc = ones.copy()
    acc[::2] = np.nextafter(f32(1), f32(0))                      # just below 1: gated at the default, kept at 0.99
    ref1 = agree(o, d, plane, acc, H, W, s=s, mc=1)
    ref2 = agree(o, d, plane, acc, H, W, s=s, mc=1, min_acc=0.99)
    assert not ref1[5][::2].any() and ref1[5][1::2].all() and ref2[5].all()
    agree(o, d, plane, np.full((H, W), np.nan, f32), H, W, s=s, mc=1)       # NaN acc gates everything


def test_edge_pixels_count_themselves_again():
    """A pixel in a corner sees itself (s+1)^2 times for s = 1 on a plane whose other pixels are far: the clamp repeats it."""
    H = W = 5
    o, d = camera(H, W)
    depth = np.full((H, W), 4.0, f32)
    depth[1:, :] = 5.0
    depth[:, 1:] = 5.0
    *_, cnt, _ = R.surface_points(o, d, depth, np.ones((H, W), f32), np.zeros((H * W, 3), f32), H, W, step=1,
                                  dist_threshold=1e-6, min_count_=1)
    assert cnt[0, 0] == 4


def test_ring_poses():
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import mesh
    P = mesh.surface_ray_poses()
    assert len(P) == 32
    k = 0
    for th in np.linspace(-180, 180, 8, endpoint=False):
        for ph in (-90.0, -30.0, 30.0, 90.0):
            assert np.array_equal(P[k], nm.pose_spherical(float(th), ph, 4.0)), k
            k += 1
    assert np.allclose(np.linalg.norm(np.stack(P)[:, :3, 3], axis=1), 4.0, atol=1e-5)
    assert len(mesh.surface_ray_poses(3, 2, 2.0)) == 6


def cloud(n, seed=0):
    rng = np.random.default_rng(seed)
    p = rng.normal(0, 1, (n, 3)).astype(f32)
    nrm = rng.normal(0, 1, (n, 3)).astype(f32)
    c = rng.uniform(-0.2, 1.2, (n, 3)).astype(f32)
    if n >= 8:
        p[0] = [0.1, 1e-30, -3.5e12]
        nrm[1] = [np.inf, -np.inf, np.nan]
        c[2] = [np.nan, 1.0, 0.0]
        c[3] = [255.0 / 255.0, np.nextafter(f32(1), f32(0)), 1 / 255]
        c[4] = [-np.inf, np.inf, 0.5]
    return p, c, nrm


def test_quantise():
    q = R.quantise(np.array([np.nan, -1.0, 0.0, 0.003, 1 / 255, 0.5, 0.999, 1.0, 2.0, np.inf, -np.inf], f32))
    assert q.tolist() == [0, 0, 0, 0, 1, 127, 254, 255, 255, 255, 0]
    from nerfmeshes_b200 import mesh
    x = np.random.default_rng(1).uniform(-1, 2, 10000).astype(f32)
    assert np.array_equal(mesh.ply_colors(x), R.quantise(x))


@pytest.mark.parametrize("binary", [False, True])
@pytest.mark.parametrize("n", [0, 1, 9, 5000])
def test_ply_bytes(tmp_path, binary, n):
    from nerfmeshes_b200 import mesh
    p, c, nrm = cloud(n, n)
    want = R.ply_bytes(p, c, nrm, binary)
    mesh.export_ply(p, c, nrm, tmp_path / "a.ply", binary=binary)                   # native (float32)
    mesh._export_ply_python(p, c, nrm, tmp_path / "b.ply", binary=binary)
    mesh.export_ply(p.astype(np.float64), c.astype(np.float64), torch.from_numpy(nrm), tmp_path / "c.ply", binary=binary)
    for name in ("a.ply", "b.ply", "c.ply"):
        assert (tmp_path / name).read_bytes() == want, name
    rp, rn, rc = R.read_ply(want)
    assert np.array_equal(bits(rp), bits(p)) and np.array_equal(bits(rn), bits(nrm))
    assert np.array_equal(rc, R.quantise(c))
    if n and not binary:
        head = want.split(b"end_header\n")[0].decode().split("\n")
        assert head[:3] == ["ply", "format ascii 1.0", f"element vertex {n}"]
        assert want.split(b"end_header\n")[1].split(b"\n")[0].decode().count(" ") == 8


def test_rejects_bad_arguments_without_a_device(tmp_path):
    from nerfmeshes_b200 import _lib as L
    lib = L.load()
    P = C.c_void_p(16)                       # never dereferenced: every call below fails its argument checks first
    pose_ = (C.c_float * 12)(*np.eye(3, 4, dtype=f32).reshape(-1))
    cnt = C.c_int64()
    err = lambda: lib.nm_last_error().decode()

    def rejects(text, h=None, pose=pose_, H=8, W=8, focal=10.0, dr=P, acc=P, rgb=P, min_acc=1.0, step=2, thr=0.002, mc=15,
                pts=P, nrm=P, col=P, pix=P, count=C.byref(cnt)):
        rc = lib.nm_surface_points(h, pose, H, W, focal, dr, acc, rgb, min_acc, step, thr, mc, pts, nrm, col, pix, count, None)
        assert rc != 0 and text in err(), (text, rc, err())

    for kw in (dict(H=0), dict(W=0), dict(H=-2)):
        rejects("is empty", **kw)
    rejects("2^31 or more", H=65536, W=32768)
    for st in (-1, 9, 100):
        rejects("step", step=st)
    for m in (0, -5):
        rejects("min_count", mc=m)
    for x in (0.0, -1.0, float("inf"), float("nan")):
        rejects("focal length", focal=x)
    rejects("NaN", min_acc=float("nan"))
    rejects("NaN", thr=float("nan"))
    rejects("null pose or count", pose=None)
    rejects("null pose or count", count=None)
    for k in ("dr", "acc", "rgb"):
        rejects("null depth_raw, acc or rgb", **{k: None})
    for k in ("pts", "nrm", "col"):
        rejects("null output", **{k: None})
    rejects("null handle")
    rejects("null handle", pix=None)                       # the pixel indices are optional
    rejects("null handle", step=0, mc=1)
    rejects("null handle", step=8, mc=1000)                # a min_count no pixel can reach is not an error
    assert lib.nm_export_ply(str(tmp_path / "x.ply").encode(), None, None, None, 3, 0) != 0 and "null" in err()
    assert lib.nm_export_ply(str(tmp_path / "x.ply").encode(), P, P, P, 1, 2) != 0 and "binary" in err()
    assert lib.nm_export_ply(str(tmp_path / "no" / "x.ply").encode(), None, None, None, 0, 0) != 0 and "cannot open" in err()
