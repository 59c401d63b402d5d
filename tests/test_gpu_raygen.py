"""Ray generation and NDC on the device (raygen_kernel, ndc_kernel) against their numpy fp32 restatements
(tests/_raygen_ref.py), bit for bit: no tolerance.

* Engine.ray_bundle, plain and NDC, over image sizes 1x1, 1x7, 7x1, 2x3, 37x53, 756x1008, 800x800 and 4097x4096 (16.8M
  rays: the flat index passes 2^24), focal 13.5, 41.3, 815.13, 1111.1111, 0.37, 1e5, near 1.0, 0.3, 2.7, row shards
  (empty, first row, last row, not aligned to the 256-thread block) and poses: two pose_spherical poses, the identity, a
  3x4 input, a non-orthonormal pose with a large translation, and a pose whose third rotation row is zero (every d_z is 0,
  NDC yields inf and NaN: bits compared where neither side is NaN, NaN required at the same places — CUDA's canonical NaN
  and x86's default NaN differ in their bits).
* Engine.ndc_rays with one shared origin (o_stride 0) and per-ray origins (o_stride 3), n = 1, 255, 256, 257.
* The device's NDC rays equal oracle.nerf_oracle.ndc_rays applied to the device's own plain rays; the plain directions lie
  within 2 TAU_RAY u scale of the oracle's get_ray_bundle (both within TAU_RAY of the float64 truth).
* render_image, NDC off and on, whole and in row shards, equals render_rays on ray_bundle's rays bit for bit.
* Malformed arguments fail without a launch; n = 0 and an empty row range succeed with none.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import _raygen_ref as RR
from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu
NET = O.NetCfg(num_layers=4, hidden_size=128, num_encoding_fn_xyz=6)

_SPH30 = O.pose_spherical(30.0, -30.0, 4.0)
POSES = {
    "spherical_30": _SPH30,
    "spherical_m150": O.pose_spherical(-150.0, -30.0, 4.0),
    "identity": torch.eye(4),
    "3x4": _SPH30.numpy()[:3, :4].copy(),
    "skewed_far": np.array([[0.9, 0.3, -1.7, 1234.5], [0.2, -1.1, 0.4, -987.25], [0.5, 0.6, 1.3, 4321.0]], np.float32),
    "flat_z": np.array([[1.0, 0.0, 0.0, 0.1], [0.0, 1.0, 0.0, 0.2], [0.0, 0.0, 0.0, 3.0]], np.float32),
}
SMALL = [(1, 1), (1, 7), (7, 1), (2, 3), (37, 53)]
FOCALS = [13.5, 41.3, 815.13, 1111.1111, 0.37, 1e5]
NEARS = [1.0, 0.3, 2.7]


def _same(a, b):
    """Bitwise equality, except that NaN only has to be NaN on both sides."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))


def _ndiff(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return int(((a.view(np.uint32) != b.view(np.uint32)) & ~(np.isnan(a) & np.isnan(b))).sum())


@pytest.fixture(scope="module")
def eng():
    import nerfmeshes_b200 as nm
    e = nm.Engine(NET.__dict__, NET.__dict__, nm.RenderSettings(num_coarse=32, num_fine=32))
    e.load_weights(0, O.init_weights(NET, 5))
    e.load_weights(1, O.init_weights(NET, 6))
    yield e
    e.close()


def _check_bundle(eng, pose, H, W, f, rows=None, nears=NEARS):
    r0, r1 = rows if rows is not None else (0, H)
    o, d = eng.ray_bundle(pose, H, W, f, rows=rows)
    eo, ed = RR.raygen32(pose, H, W, f, r0, r1)
    o, d = o.cpu().numpy(), d.cpu().numpy()
    assert _same(o, eo) and _same(d, ed), (H, W, f, rows, _ndiff(d, ed))
    for near in nears:
        on, dn = eng.ray_bundle(pose, H, W, f, ndc=True, ndc_near=near, rows=rows)
        xo, xd = RR.ndc32(H, W, f, near, eo, ed)
        on, dn = on.cpu().numpy(), dn.cpu().numpy()
        assert _same(on, xo) and _same(dn, xd), (H, W, f, near, rows, _ndiff(on, xo), _ndiff(dn, xd))
    return d


def test_ray_bundle_small_images_every_focal_pose_and_near(eng):
    n = 0
    for name, pose in POSES.items():
        for H, W in SMALL:
            for f in FOCALS:
                _check_bundle(eng, pose, H, W, f)
                n += 1
    print(f"{n} small ray bundles bit-exact, plain and NDC at near {NEARS}")


def test_ray_bundle_row_shards(eng):
    """First row, last row, and shards whose first ray and ray count are not multiples of the 256-thread block (the empty
    shard is checked at the C ABI in test_malformed_arguments_fail_without_launching)."""
    pose = POSES["spherical_30"]
    for H, W, f in [(37, 53, 41.3), (756, 1008, 815.13)]:
        for rows in [(0, 1), (H - 1, H), (5, 30), (3, H - 2)]:
            assert (rows[0] * W) % 256 != 0 or rows[0] == 0
            _check_bundle(eng, pose, H, W, f, rows=rows, nears=[1.0, 0.3])


@pytest.mark.parametrize("H,W", [(756, 1008), (800, 800)])
def test_ray_bundle_benchmark_sizes(eng, H, W):
    for name in ("spherical_30", "identity", "skewed_far", "flat_z"):
        for f in (815.13, 1111.1111, 41.3):
            _check_bundle(eng, POSES[name], H, W, f, nears=[1.0, 0.3])


def test_ray_bundle_past_2_24_rays(eng):
    H, W, f = 4097, 4096, 815.13
    assert H * W > 2 ** 24
    _check_bundle(eng, POSES["spherical_m150"], H, W, f, nears=[0.3])
    torch.cuda.empty_cache()


def test_flat_pose_gives_the_same_non_finite_rays(eng):
    H, W, f = 37, 53, 41.3
    for near in NEARS:
        on, dn = eng.ray_bundle(POSES["flat_z"], H, W, f, ndc=True, ndc_near=near)
        on, dn = on.cpu().numpy(), dn.cpu().numpy()
        assert not np.isfinite(on).all() and np.isnan(dn).any()
        _, ed = RR.raygen32(POSES["flat_z"], H, W, f)
        xo, xd = RR.ndc32(H, W, f, near, POSES["flat_z"][:, 3], ed)
        assert _same(on, xo) and _same(dn, xd)


def test_device_ndc_equals_oracle_on_device_rays(eng):
    for name in ("spherical_30", "spherical_m150", "skewed_far"):
        for H, W, f in [(37, 53, 41.3), (756, 1008, 815.13), (800, 800, 1111.1111)]:
            o, d = eng.ray_bundle(POSES[name], H, W, f)
            o, d = o.cpu(), d.cpu()
            ratio = RR.ray_error_ratio(d.numpy(), POSES[name], H, W, f)
            assert ratio <= RR.TAU_RAY, (name, H, W, f, ratio)
            _, od = O.get_ray_bundle(H, W, f, torch.as_tensor(POSES[name]))
            _, scale = RR.ray_truth(POSES[name], H, W, f)
            assert bool((np.abs(d.numpy().astype(np.float64) - od.numpy()) <= 2 * RR.TAU_RAY * RR.U * scale).all())
            for near in (1.0, 0.3, 2.7):
                on, dn = eng.ray_bundle(POSES[name], H, W, f, ndc=True, ndc_near=near)
                ro, rd = O.ndc_rays(H, W, f, near, o.expand(d.shape), d)
                assert _same(on.cpu(), ro) and _same(dn.cpu(), rd), \
                    (name, H, W, f, near, _ndiff(on.cpu(), ro), _ndiff(dn.cpu(), rd))


@pytest.mark.parametrize("n", [1, 255, 256, 257])
def test_ndc_rays_on_caller_rays(eng, n):
    g = np.random.default_rng(n)
    d = g.standard_normal((n, 3)).astype(np.float32)
    d[:, 2] = -np.abs(d[:, 2]) - np.float32(0.05)
    o_all = (g.standard_normal((n, 3)) * 3).astype(np.float32)
    o_one = np.array([0.25, -0.5, 0.75], np.float32)
    for f in (41.3, 815.13, 1111.1111):
        for near in NEARS:
            for o in (o_one, o_all):
                got_o, got_d = eng.ndc_rays(756, 1008, f, near, torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda())
                xo, xd = RR.ndc32(756, 1008, f, near, o, d)
                ro, rd = O.ndc_rays(756, 1008, f, near, torch.from_numpy(np.broadcast_to(o, d.shape).copy()),
                                    torch.from_numpy(d))
                assert _same(got_o.cpu(), xo) and _same(got_d.cpu(), xd), (n, f, near, o.shape)
                assert _same(xo, ro) and _same(xd, rd)


def test_render_image_equals_render_rays_on_its_rays(eng):
    pose = POSES["spherical_30"]
    want = ["rgb", "depth", "acc", "disp"]
    H, W, f = 40, 48, 55.0
    o, d = eng.ray_bundle(pose, H, W, f)
    ref = eng.render_rays(o, d.reshape(-1, 3), 2.0, 6.0, want=want)
    img = eng.render_image(pose, H, W, f, 2.0, 6.0, want=want)
    for k in want:
        assert torch.equal(img[k], ref[k]), k
    part = eng.render_image(pose, H, W, f, 2.0, 6.0, rows=(7, 29), want=want)
    ref_p = eng.render_rays(o, d[7:29].reshape(-1, 3), 2.0, 6.0, want=want)
    for k in want:
        assert torch.equal(part[k], ref_p[k]) and torch.equal(part[k], img[k][7 * W:29 * W]), k
    # NDC, the fern camera at a reduced size: render_image warps with near 1.0, NDC bounds [0, 1]
    H, W, f = 63, 84, 815.13 * 84 / 1008
    pose = np.eye(4, dtype=np.float32)
    pose[0, 3] = 0.1
    on, dn = eng.ray_bundle(pose, H, W, f, ndc=True, ndc_near=1.0)
    ref = eng.render_rays(on.reshape(-1, 3), dn.reshape(-1, 3), 0.0, 1.0, want=want)
    img = eng.render_image(pose, H, W, f, 0.0, 1.0, ndc=True, want=want)
    for k in want:
        assert torch.equal(img[k], ref[k]), ("ndc", k)
    part = eng.render_image(pose, H, W, f, 0.0, 1.0, ndc=True, rows=(11, 40), want=want)
    for k in want:
        assert torch.equal(part[k], img[k][11 * W:40 * W]), ("ndc rows", k)


def test_malformed_arguments_fail_without_launching(eng):
    from nerfmeshes_b200 import _lib
    lib, h, st = eng.lib, eng._h, eng._stream()
    pose = np.ascontiguousarray(POSES["spherical_30"].numpy()[:3, :4])
    buf, buf2 = torch.zeros(64 * 3, device="cuda"), torch.zeros(64 * 3, device="cuda")
    p = lambda x: C.c_void_p(x.data_ptr())
    pp = pose.ctypes.data

    def bundle(H, W, ndc, r0, r1, o, d, pose_p=pp):
        return lib.nm_ray_bundle(h, pose_p, H, W, 41.3, ndc, 1.0, r0, r1, o, d, st)

    def ndc(o_stride, n, o=p(buf), d=p(buf2)):
        return lib.nm_ndc_rays(h, 4, 4, 41.3, 1.0, o, o_stride, d, n, p(buf), p(buf2), st)
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    bad = [lambda: bundle(4, 3, 0, 3, 2, None, p(buf)), lambda: bundle(4, 3, 0, 0, 5, None, p(buf)),
           lambda: bundle(4, 0, 0, 0, 4, None, p(buf)), lambda: bundle(4, 3, 0, -1, 2, None, p(buf)),
           lambda: bundle(4, 3, 1, 0, 4, None, p(buf)), lambda: bundle(4, 3, 0, 0, 4, None, None),
           lambda: bundle(4, 3, 0, 0, 4, None, p(buf), None),
           lambda: ndc(1, 4), lambda: ndc(3, -1), lambda: ndc(0, 4, o=None), lambda: ndc(3, 4, d=None)]
    for call in bad:
        assert call() != 0
        assert lib.nm_last_error()
    nf = (C.c_float * 2)(2.0, 6.0)
    block = _lib.NmRenderOut()
    for r0, r1 in [(3, 2), (0, 5), (-1, 2)]:
        assert lib.nm_render_image(h, pp, 4, 3, 41.3, 0, r0, r1, nf, 0, 0, C.byref(block), st) != 0
        assert lib.nm_render_image_host(h, pp, 4, 3, 41.3, 0, r0, r1, nf, 0, 0, C.byref(block)) != 0
    torch.cuda.synchronize()
    assert eng.launch_count() == n0
    assert ndc(0, 0) == 0 and ndc(3, 0) == 0 and bundle(4, 3, 1, 2, 2, p(buf), p(buf2)) == 0
    torch.cuda.synchronize()
    assert eng.launch_count() == n0
    assert bundle(4, 3, 1, 0, 4, p(buf), p(buf2)) == 0 and ndc(3, 5) == 0
    torch.cuda.synchronize()
    assert eng.launch_count() == n0 + 2
