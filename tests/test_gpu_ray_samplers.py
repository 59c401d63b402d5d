"""The ray samplers of nm_render.cu against their numpy fp32 restatements (tests/_sampler_ref.py), bit for bit: no
tolerance anywhere.

* SamplePDF through the nm_debug_sample_pdf hook over the edge matrix of tests/test_ray_samplers_reference.py (Nc 3, 64,
  256; Nf 1, 2, 31, 33, 128, 256 with Nc = 256, 509 with Nc = 3; R 1, 3, 5 and 4099; perturb on and off; zero, spike,
  equal, ~1e-5 and random weights with u on the cdf knots; uniform, lindisp, all-equal and per-ray depths).
* Stratified sampling through coarse-only renders in training mode (perturbed, lindisp on and off, scalar and per-ray
  bounds), and the engine's default table through an unperturbed [0, 1] render.
* The render's wiring: a two-network training render with perturb and noise resamples its own stratified samples with its
  own coarse weights on the stream seed ^ 0x9e3779b9, in one chunk and in chunks of NM_CHUNK_RAYS rays (seed + r0).
* AABB sampling through nm_ray_voxel_indices_ex, deterministic and random, on the synthetic scenes (entry ties, +-0
  direction components, origins on slab planes, tmin == near, tmax == far, 1 / 32 / 33 / 512 hits, misses), the
  overflow path (reported once, the other rays untouched, the handle usable afterwards), and the argument checks.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _sampler_ref as SR
from conftest import ROOT
from oracle import nerf_oracle as O
from test_ray_samplers_reference import aabb_cases, aabb_scene, line_far, pdf_cases, pdf_inputs, run_aabb_ref

pytestmark = pytest.mark.gpu
NET = O.NetCfg(num_layers=4, hidden_size=128, num_encoding_fn_xyz=6)


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _engine(nc=64, nf=0, fine=False, **kw):
    import nerfmeshes_b200 as nm
    eng = nm.Engine(NET.__dict__, NET.__dict__ if fine else None, nm.RenderSettings(num_coarse=nc, num_fine=nf, **kw))
    eng.load_weights(0, O.init_weights(NET, 3))
    if fine:
        eng.load_weights(1, O.init_weights(NET, 4))
    return eng


# ----------------------------------------------------------------------------------------------------- SamplePDF
def test_sample_pdf_hook_matches_restatement_bit_for_bit():
    eng = _engine()
    n = 0
    for R, Nc, Nf, wk, tk, perturb, seed in pdf_cases():
        t, w, u = pdf_inputs(R, Nc, Nf, wk, tk, perturb, seed)
        got = eng.debug_sample_pdf(torch.from_numpy(t), torch.from_numpy(w), None if u is None else torch.from_numpy(u),
                                   Nf=Nf, perturb=perturb, seed=seed).cpu().numpy()
        ref = SR.sample_pdf(t, w, u, Nf, perturb, seed)
        assert _bits_equal(got, ref), (R, Nc, Nf, wk, tk, perturb, int((got != ref).sum()))
        n += 1
    print(f"SamplePDF hook: {n} cases bit-exact")
    eng.close()


def test_sample_pdf_hook_rejects_bad_arguments_without_launching():
    eng = _engine()
    lib, h, st = eng.lib, eng._h, eng._stream()
    R, Nc, Nf = 5, 64, 128
    t, w = torch.zeros(R * Nc, device="cuda"), torch.ones(R * Nc, device="cuda")
    u, out = torch.zeros(512, device="cuda"), torch.zeros(R * 512, device="cuda")
    p = lambda x: C.c_void_p(x.data_ptr())

    def call(tp, wp, up, r, nc, nf, perturb, op):
        return lib.nm_debug_sample_pdf(h, tp, wp, up, r, nc, nf, perturb, 0, op, st)
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    bad = [(None, p(w), p(u), R, Nc, Nf, 0, p(out)), (p(t), None, p(u), R, Nc, Nf, 0, p(out)),
           (p(t), p(w), p(u), R, Nc, Nf, 0, None), (p(t), p(w), p(u), -1, Nc, Nf, 0, p(out)),
           (p(t), p(w), p(u), R, 2, Nf, 0, p(out)), (p(t), p(w), p(u), R, 257, Nf, 0, p(out)),
           (p(t), p(w), p(u), R, Nc, 0, 0, p(out)), (p(t), p(w), p(u), R, Nc, 513 - Nc, 0, p(out)),
           (p(t), p(w), None, R, Nc, Nf, 0, p(out))]
    for args in bad:
        assert call(*args) != 0, args
        assert lib.nm_last_error()
    assert call(p(t), p(w), p(u), 0, Nc, Nf, 0, p(out)) == 0                   # R = 0: nothing to do
    assert eng.launch_count() == n0
    assert call(p(t), p(w), None, R, Nc, 512 - Nc, 1, p(out)) == 0 and eng.launch_count() == n0 + 1
    eng.close()


# ----------------------------------------------------------------------------------------------------- stratified
def _rays(R, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(R, 3, generator=g) * 0.3, torch.randn(R, 3, generator=g)


@pytest.mark.parametrize("lindisp", [False, True])
def test_stratified_training_render_matches_restatement(lindisp):
    R = 1027
    o, d = _rays(R, 1)
    for Nc in (3, 64, 192):
        eng = _engine(nc=Nc, perturb=True, lindisp=lindisp, noise_std=0.3)
        for seed in (0, 12345, 2 ** 64 - 3):
            tv = eng.render_rays(o.cuda(), d.cuda(), 2.0, 6.0, training=True, seed=seed, want=["t_vals"])["t_vals"].cpu()
            assert _bits_equal(tv.numpy(), SR.stratified(SR.linspace(Nc), 2.0, 6.0, lindisp, True, seed=seed, R=R)), (Nc, seed)
        near = torch.rand(R, generator=torch.Generator().manual_seed(Nc)) + 0.5
        far = near + 3.0
        tv = eng.render_rays(o.cuda(), d.cuda(), near.cuda(), far.cuda(), training=True, seed=9, want=["t_vals"])["t_vals"]
        assert _bits_equal(tv.cpu().numpy(), SR.stratified(SR.linspace(Nc), near.numpy(), far.numpy(), lindisp, True, seed=9))
        eng.close()


def test_default_coarse_table_is_torch_linspace():
    """An engine's own table (no nm_set_tables): an unperturbed render on [0, 1] returns it unchanged."""
    o, d = _rays(4, 2)
    for Nc in (3, 64, 128, 192, 256):
        eng = _engine(nc=Nc)
        tv = eng.render_rays(o.cuda(), d.cuda(), 0.0, 1.0, want=["t_vals"])["t_vals"].cpu().numpy()
        assert _bits_equal(tv, np.broadcast_to(torch.linspace(0, 1, Nc).numpy(), (4, Nc))), Nc
        eng.close()


# ----------------------------------------------------------------------------------------------------- render wiring
def _two_net_expectation(tv, cw, R, chunk, seed, Nc=64, Nf=128):
    """t_vals of a two-network perturbed render: per chunk r0, SamplePDF of stratified(seed + r0) with the coarse weights
    of that call, on the stream (seed + r0) ^ SALT_INVCDF."""
    out = []
    for r0 in range(0, R, chunk):
        n = min(chunk, R - r0)
        s = (seed + r0) % 2 ** 64
        t_c = SR.stratified(SR.linspace(Nc), 2.0, 6.0, False, True, seed=s, R=n)
        out.append(SR.sample_pdf(t_c, cw[r0:r0 + n], None, Nf, True, s ^ SR.SALT_INVCDF))
    return np.concatenate(out)


_WIRING = ("import sys, numpy as np, torch; sys.path.insert(0, %r); sys.path.insert(0, %r + '/tests');"
           "from test_gpu_ray_samplers import _engine, _rays;"
           "eng = _engine(nc=64, nf=128, fine=True, perturb=True, noise_std=0.5); o, d = _rays(2000, 5);"
           "r = eng.render_rays(o.cuda(), d.cuda(), 2.0, 6.0, training=True, seed=int(sys.argv[2]),"
           " want=['t_vals', 'coarse_weights']);"
           "np.savez(sys.argv[1], tv=r['t_vals'].cpu().numpy(), cw=r['coarse_weights'].cpu().numpy())")


@pytest.mark.parametrize("chunk", [None, 700])
def test_two_network_render_resamples_its_own_samples(chunk, tmp_path):
    """The salts and the per-chunk seeds: NM_CHUNK_RAYS is read once per process, so each setting runs in its own."""
    seed = 0x2545F4914F6CDD1D
    path = str(tmp_path / "wiring.npz")
    env = dict(os.environ)
    env.pop("NM_CHUNK_RAYS", None)
    if chunk:
        env["NM_CHUNK_RAYS"] = str(chunk)
    subprocess.run([sys.executable, "-c", _WIRING % (ROOT, ROOT), path, str(seed)], check=True, env=env, timeout=600)
    z = np.load(path)
    tv, cw = z["tv"], z["cw"]
    assert np.isfinite(cw).all() and cw.max() > 0
    assert _bits_equal(tv, _two_net_expectation(tv, cw, 2000, chunk or 2000, seed))


# ----------------------------------------------------------------------------------------------------- AABB
def _aabb_device(eng, vox, o, d, near, far, random, seed):
    import nerfmeshes_b200 as nm
    eng.set_tree(torch.from_numpy(vox))
    eng.voxel_random = bool(random)
    try:
        idx, z = eng.ray_voxel_indices(torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda(), near, far, want_z=True, seed=seed)
    finally:
        eng.voxel_random = False
    return z.cpu().numpy(), idx.cpu().numpy(), nm


def test_aabb_matches_restatement_bit_for_bit():
    engines = {}
    for scene, far, S, random, seed in aabb_cases():
        eng = engines.setdefault(S, _engine(nc=S))
        vox, o, d, near, far0 = aabb_scene(scene)
        far = far0 if far is None else far
        z, idx, _ = _aabb_device(eng, vox, o, d, near, far, random, seed)
        z_ref, idx_ref, hits, over = run_aabb_ref(scene, far, S, random, seed)
        assert not over
        assert _bits_equal(z, z_ref) and np.array_equal(idx, idx_ref), (scene, far, S, random)
        eng.check_flags()
    for eng in engines.values():
        eng.close()


def test_aabb_on_the_lego_tree_random_branch():
    from conftest import load_npz
    g = load_npz("golden_lego_buff.npz")
    vox = load_npz("weights_lego_buff.npz")["voxels"].float().numpy()
    near, far = float(g["bounds"][0]), float(g["bounds"][1])
    eng = _engine(nc=192)
    o, d = g["origin"].numpy()[None], g["dirs"].numpy()
    R = d.shape[0]
    tu = SR.stratified(SR.linspace(192), near, far, False, False, R=R)
    for random, seed in ((0, 0), (1, 11), (1, 2 ** 63 + 5)):
        z, idx, _ = _aabb_device(eng, vox, o, d, near, far, random, seed)
        z_ref, idx_ref, _, _ = SR.aabb(vox, o, d, near, far, 192, SR.linspace(192), tu, random=bool(random), seed=seed)
        assert _bits_equal(z, z_ref) and np.array_equal(idx, idx_ref), (random, seed)
    eng.close()


def test_aabb_overflow_is_reported_once_and_leaves_the_other_rays_alone():
    import nerfmeshes_b200 as nm
    vox, o, d, near, _ = aabb_scene("line")
    far = line_far(600)
    # ray 2 runs along the row (600 hits); the others cross it (1 hit, a few hits) or miss it
    oo = np.array([(3.5, 0.5, -1.0), (10.2, 0.5, -1.0), (-0.5, 0.5, 0.5), (7.5, 0.5, -1.0), (-0.5, 2.5, 0.5)], np.float32)
    dd = np.array([(0.0, -0.0, 1.0), (0.25, 0.0, 1.0), (1.0, 0.0, 0.0), (-0.0, 0.0, 1.0), (1.0, 0.0, 0.0)], np.float32)
    rest = [0, 1, 3, 4]
    for random in (0, 1):
        eng = _engine(nc=192)
        z, idx, _ = _aabb_device(eng, vox, oo, dd, near, far, random, 3)
        with pytest.raises(nm.NmError, match="more than 512"):
            eng.check_flags()
        eng.check_flags()                                  # reported once
        tu = SR.stratified(SR.linspace(192), near, far, False, False, R=oo.shape[0])
        z_ref, idx_ref, hits, over = SR.aabb(vox, oo, dd, near, far, 192, SR.linspace(192), tu, random=bool(random), seed=3)
        assert over and hits[2] == 600 and (hits[rest] <= 512).all() and hits[0] == 1 and hits[4] == 0
        assert _bits_equal(z, z_ref) and np.array_equal(idx, idx_ref)
        if not random:                                     # (the random draws are indexed by ray: no in-place comparison)
            z2, idx2, _ = _aabb_device(eng, vox, oo[rest], dd[rest], near, far, 0, 3)
            eng.check_flags()
            assert _bits_equal(z2, z[rest]) and np.array_equal(idx2, idx[rest])
        # the handle stays usable for everything else
        out = eng.render_rays(torch.from_numpy(oo).cuda(), torch.from_numpy(dd).cuda(), 2.0, 6.0, want=["rgb"])
        eng.check_flags()
        assert torch.isfinite(out["rgb"]).all()
        eng.close()


def test_voxel_indices_reject_bad_arguments():
    import nerfmeshes_b200 as nm
    eng = _engine(nc=64)
    o, d = torch.zeros(3, device="cuda"), torch.ones(6, device="cuda")
    idx = torch.zeros(128, dtype=torch.int32, device="cuda")
    nf = (C.c_float * 2)(1.0, 4.0)
    p = lambda x: C.c_void_p(x.data_ptr())
    call = lambda *a: eng.lib.nm_ray_voxel_indices_ex(eng._h, *a, eng._stream())
    assert call(p(o), 0, p(d), 2, nf, 0, 0, None, p(idx)) != 0          # no voxel list yet
    eng.set_tree(torch.tensor([[[0.0, 0, 0], [1, 1, 1]]]))
    for args in [(None, 0, p(d), 2, nf, 0, 0, None, p(idx)), (p(o), 0, None, 2, nf, 0, 0, None, p(idx)),
                 (p(o), 0, p(d), 2, None, 0, 0, None, p(idx)), (p(o), 0, p(d), 2, nf, 0, 0, None, None),
                 (p(o), 1, p(d), 2, nf, 0, 0, None, p(idx))]:
        assert call(*args) != 0, args
    assert call(p(o), 0, p(d), 2, nf, 0, 0, None, p(idx)) == 0
    with pytest.raises(nm.NmError):
        eng.set_tree(torch.zeros(0, 2, 3))
    eng.close()
