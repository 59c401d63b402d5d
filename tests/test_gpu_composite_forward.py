"""The forward compositor on the GPU.

Hook: `composite_kernel` through nm_debug_composite against the float64 truth of tests/_composite_ref.py over the edge
matrix (S_EDGES + S_EXTRA; R = 1, 127, 128, 129 against the kernel's 128 rays per block, and 4099 once per S; white
background, training, noise 0 / 0.7 with both salts, thr 1e-5 / 0 / 1 / -1; the fourteen FWD_KINDS): continuous outputs
within TAU_FWD * forward_error_scale, NaN / inf where the truth has them, mask and thresholded depth exact outside their
undecided margins, the empty / behind values and the zero weights of gated samples exact; two calls agree bit for bit;
malformed arguments fail without a launch.

Render paths: a teacher-forced render, with the fused compositor and with the two-kernel path, equals the hook fed the
network's raw at fl(o + fl(d t)) bit for bit, at the fused path's group edges, ragged ray counts, both precisions,
empty / saturated / acc = 1 networks, duplicate samples and training noise; a two-network render's coarse maps too, and a
render in several NM_CHUNK_RAYS chunks.

Skipping: with a grid and validation noise, every ray whose skipped samples all have a dense noisy pre-activation <= 0
keeps the dense render's bits."""
import os
import subprocess
import sys

import ctypes as C
import numpy as np
import pytest
import torch

import _composite_ref as CR
import _sampler_ref as SR
from oracle import nerf_oracle as O
from test_composite_adjoint import NOISE, S_ALL
from test_composite_forward_reference import THRS

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NET = O.NetCfg(num_layers=4, hidden_size=128, num_encoding_fn_xyz=6)
OUT = CR.FWD_OUT


def _engine(nc=64, nf=0, **kw):
    import nerfmeshes_b200 as nm
    return nm.Engine(NET.__dict__, NET.__dict__ if nf else None, nm.RenderSettings(num_coarse=nc, num_fine=nf, **kw))


def _hook(eng, raw, t, d, **kw):
    out = eng.debug_composite(torch.from_numpy(np.ascontiguousarray(raw)).cuda(), torch.from_numpy(np.ascontiguousarray(t)).cuda(),
                              torch.from_numpy(np.ascontiguousarray(d)).cuda(), **kw)
    return {k: v.cpu().numpy() for k, v in out.items()}


def _bits(a):
    return np.ascontiguousarray(np.asarray(a, np.float32)).view(np.uint32)


# ----------------------------------------------------------------------------------------------------- hook vs truth
def test_hook_matches_float64_truth_over_the_edge_matrix():
    eng = _engine()
    worst, at = 0.0, None
    K = {n: i for i, n in enumerate(CR.FWD_KINDS)}
    for S in S_ALL:
        cases = []
        for j, (white, training) in enumerate(((0, 0), (1, 0), (0, 1), (1, 1))):
            cases.append(((1, 127, 128, 129)[j], white, training, *NOISE[(S + j) % 3], THRS[(S + j) % 4]))
        cases.append((4099, S % 2, (S // 2) % 2, *NOISE[S % 3], THRS[(S + 1) % 4]))
        for R, white, training, std, seed, thr in cases:
            raw, t, d, kinds = CR.make_forward_rays(R, S, 7919 * S + 31 * R + white, kind_offset=S + R)
            got = _hook(eng, raw, t, d, noise_std=std, seed=seed, white_bg=white, training=training, thr=thr)
            f = CR.composite_forward(raw, t, d, white, training, thr, std, seed)
            sc = CR.forward_error_scale(f, raw, t, white)
            for k in OUT:
                r = CR.forward_ratio(got[k], f.out[k], sc[k])
                if r.max() > worst:
                    i = np.unravel_index(r.argmax(), r.shape)
                    worst, at = float(r.max()), (S, R, white, training, std, thr, k, CR.FWD_KINDS[kinds[i[0]]])
                assert r.max() <= CR.TAU_FWD, (S, R, white, training, std, thr, k, float(r.max()))
            # exact values: empty rays, rays behind the origin, the weights of gated samples
            e = kinds == K["empty"]
            assert (got["acc"][e] == 0).all() and (got["disp"][e] == 0).all() and (got["depth_raw"][e] == 0).all()
            assert (got["rgb"][e] == (1.0 if white else 0.0)).all()
            b = (kinds == K["behind"]) & (f.out["acc"] > 1e-6)           # noise may close every gate of a ray
            assert (got["disp"][b] == np.float32(1e10)).all()
            und = (f.noise != 0) & (np.abs(f.pre) <= CR.GATE_MU * np.abs(f.noise))
            gated = ((f.pre <= 0) | np.isnan(f.pre)) & ~und & np.isfinite(f.w)
            assert (got["weights"][gated] == 0).all(), (S, R)
    print(f"RATIO forward hook-vs-truth {worst:.3e} at S,R,white,training,noise,thr,output,kind = {at}")
    eng.close()


def test_hook_is_deterministic():
    eng = _engine()
    raw, t, d, _ = CR.make_forward_rays(4099, 257, 3)
    a = _hook(eng, raw, t, d, noise_std=0.7, seed=NOISE[1][1], white_bg=True)
    b = _hook(eng, raw, t, d, noise_std=0.7, seed=NOISE[1][1], white_bg=True)
    for k in OUT:
        assert np.array_equal(_bits(a[k]), _bits(b[k])), k
    eng.close()


def test_hook_rejects_bad_arguments_without_launching():
    import nerfmeshes_b200._lib as L
    eng = _engine()
    lib, h = eng.lib, eng._h
    R, S = 5, 40
    buf = torch.zeros(R * S * 4 + 4, device="cuda")
    raw = buf[:R * S * 4]
    t, d = torch.zeros(R * S, device="cuda"), torch.ones(R * 3, device="cuda")
    acc = torch.zeros(R, device="cuda")
    p = lambda x, off=0: C.c_void_p(x.data_ptr() + 4 * off)
    st = eng._stream()
    good = L.NmRenderOut(*[acc.data_ptr() if k == "acc" else None for k in L.OUT_FIELDS])
    extra = L.NmRenderOut(*[acc.data_ptr() if k in ("acc", "coarse_acc") else None for k in L.OUT_FIELDS])

    def call(raw_p, t_p, d_p, n, s, out):
        return lib.nm_debug_composite(h, raw_p, t_p, d_p, n, s, 0.0, 0, 0, 0, 1e-5, None if out is None else C.byref(out), st)
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    bad = [(None, p(t), p(d), R, S, good), (p(raw), None, p(d), R, S, good), (p(raw), p(t), None, R, S, good),
           (p(raw), p(t), p(d), R, S, None), (p(raw), p(t), p(d), R, S, extra), (p(raw), p(t), p(d), -1, S, good),
           (p(raw), p(t), p(d), R, 0, good), (p(raw), p(t), p(d), R, 513, good), (p(buf, 1), p(t), p(d), R, S, good)]
    for args in bad:
        assert call(*args) != 0, args
        assert lib.nm_last_error()
    assert call(p(raw), p(t), p(d), 0, S, good) == 0                 # R = 0: nothing to do
    assert eng.launch_count() == n0
    assert call(p(raw), p(t), p(d), R, S, good) == 0 and eng.launch_count() == n0 + 1
    eng.close()


# ----------------------------------------------------------------------------------------------------- render paths
FUSED_S = (3, 5, 15, 16, 48, 96, 192, 240, 480, 512)
# fc_alpha bias shifts: empty rays, saturated at the first sample, acc around 1
SHIFT = {"empty": -40.0, "saturated": 2e3, "acc_one": 0.6}


def _net_engine(S, shift, precision, noise_std=0.0):
    """an engine whose teacher-forced renders take S samples per ray, and the network slot they run (the fine one when
    S exceeds the coarse sampler's 256)"""
    nc, nf = (S, 0) if S <= 256 else (64, S - 64)
    eng = _engine(nc=nc, nf=nf, precision=precision, noise_std=noise_std)
    which = 1 if nf else 0
    for w in range(which + 1):
        sd = O.init_weights(NET, 100 + S + w)
        sd["fc_alpha.bias"] = sd["fc_alpha.bias"] + SHIFT[shift]
        eng.load_weights(w, sd)
    return eng, which


def _rays(R, S, seed, near=2.0, far=6.0, dup=True):
    rng = np.random.default_rng(seed)
    o = (rng.standard_normal((R, 3)) * 0.3).astype(np.float32)
    d = rng.standard_normal((R, 3)).astype(np.float32) * np.float32(0.8)
    t = np.sort(rng.uniform(near, far, (R, S)).astype(np.float32), 1)
    if dup:
        rep = rng.uniform(size=(R, S)) < 1 / 3
        rep[:, 1:2] = False                 # the first interval stays open: a saturating network saturates there
        for i in range(1, S):
            t[:, i] = np.where(rep[:, i], t[:, i - 1], t[:, i])
    return o, d, t


def _raw_at(eng, which, o, d, t):
    """the network's raw at fl(o + fl(d t)) with view directions d, through the point MLP"""
    p = (o[:, None, :] + (d[:, None, :] * t[:, :, None]).astype(np.float32)).astype(np.float32)
    dd = np.ascontiguousarray(np.broadcast_to(d[:, None, :], p.shape))
    out = eng.point_mlp(which, torch.from_numpy(p.reshape(-1, 3).copy()).cuda(), torch.from_numpy(dd.reshape(-1, 3)).cuda())
    return out.cpu().numpy().reshape(t.shape + (4,))


def _teacher(eng, o, d, t, fused, training, seed):
    os.environ["NM_FUSED_COMPOSITE"] = "1" if fused else "0"
    try:
        out = eng.render_rays(torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda(), 2.0, 6.0, training=training, seed=seed,
                              want=OUT, teacher_t=torch.from_numpy(t).cuda())
        return {k: v.cpu().numpy() for k, v in out.items()}
    finally:
        del os.environ["NM_FUSED_COMPOSITE"]


def _cases_render():
    cases = []
    for i, S in enumerate(FUSED_S):
        rays_per_group = int(np.lcm(S, 64)) // S
        shift = ("acc_one", "empty", "saturated")[i % 3]
        prec = i % 2
        cases.append((S, max(1, rays_per_group + (-1, 0, 1)[i % 3]), shift, prec, i % 4 == 3))
    cases.append((64, 20000, "acc_one", 0, False))                  # the persistent workers wrap many times
    cases.append((192, 4099, "acc_one", 1, True))
    return cases


@pytest.mark.parametrize("S,R,shift,prec,training", _cases_render())
def test_render_paths_equal_the_hook(S, R, shift, prec, training):
    std = 0.7 if training else 0.0
    eng, which = _net_engine(S, shift, prec, noise_std=std)
    o, d, t = _rays(R, S, S * 13 + R)
    seed = 12345
    raw = _raw_at(eng, which, o, d, t)
    want = _hook(eng, raw, t, d, noise_std=std, seed=seed ^ CR.SALT_MAIN, training=training)
    for fused in (True, False):
        got = _teacher(eng, o, d, t, fused, training, seed)
        for k in OUT:
            assert np.array_equal(_bits(got[k]), _bits(want[k])), (S, R, shift, prec, fused, k)
    acc = want["acc"]
    if shift == "empty":
        assert (acc == 0).all()
    elif shift == "saturated":              # alpha_0 = 1 wherever the first interval is not a duplicate
        x0 = raw[:, 0, 3].astype(np.float64) * (t[:, 1] - t[:, 0]) * np.linalg.norm(d.astype(np.float64), axis=1)
        assert (raw[:, :, 3] > 1e3).all() and (x0 >= 20).any() and (want["weights"][x0 >= 20, 0] == 1).all()
    elif R > 100:
        assert (acc < 1).any() and (acc >= 1).any()
    eng.close()


def test_two_network_render_coarse_maps_equal_the_hook():
    import nerfmeshes_b200 as nm
    nc, nf, R = 48, 80, 1001
    eng = nm.Engine(NET.__dict__, NET.__dict__, nm.RenderSettings(num_coarse=nc, num_fine=nf))
    for which in (0, 1):
        sd = O.init_weights(NET, 60 + which)
        sd["fc_alpha.bias"] = sd["fc_alpha.bias"] + 0.6
        eng.load_weights(which, sd)
    o, d, _ = _rays(R, 1, 9)
    seed = 77
    for fused in (True, False):
        os.environ["NM_FUSED_COMPOSITE"] = "1" if fused else "0"
        try:
            out = eng.render_rays(torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda(), 2.0, 6.0, seed=seed,
                                  want=OUT + ("t_vals", "coarse_rgb", "coarse_acc", "coarse_disp", "coarse_weights"))
        finally:
            del os.environ["NM_FUSED_COMPOSITE"]
        out = {k: v.cpu().numpy() for k, v in out.items()}
        t_c = SR.stratified(SR.linspace(nc), 2.0, 6.0, False, False, R=R)
        c = _hook(eng, _raw_at(eng, 0, o, d, t_c), t_c, d, seed=seed ^ CR.SALT_COARSE, want=("rgb", "acc", "disp", "weights"))
        for k in ("rgb", "acc", "disp", "weights"):
            assert np.array_equal(_bits(out["coarse_" + k]), _bits(c[k])), (fused, k)
        tf = out["t_vals"]
        f = _hook(eng, _raw_at(eng, 1, o, d, tf), tf, d, seed=seed ^ CR.SALT_MAIN)
        for k in OUT:
            assert np.array_equal(_bits(out[k]), _bits(f[k])), (fused, k)
    eng.close()


def test_multi_chunk_render_equals_the_hook_per_chunk(tmp_path):
    """NM_CHUNK_RAYS is read once per process: a child renders 1000 rays in chunks of 333, training noise on; chunk c
    draws from seed + r0 ^ the salt"""
    S, R, chunk, seed = 96, 1000, 333, 5
    out = tmp_path / "chunks.npz"
    code = f"""
import sys, numpy as np
sys.path.insert(0, {os.path.join(ROOT, 'tests')!r})
import test_gpu_composite_forward as T
eng, which = T._net_engine({S}, "acc_one", 0, noise_std=0.7)
o, d, t = T._rays({R}, {S}, 4)
r = T._teacher(eng, o, d, t, True, True, {seed})
raw = T._raw_at(eng, which, o, d, t)
np.savez({str(out)!r}, raw=raw, **r)
"""
    subprocess.run([sys.executable, "-c", code], check=True, env={**os.environ, "NM_CHUNK_RAYS": str(chunk)}, cwd=ROOT, timeout=600)
    z = np.load(out)
    eng, _ = _net_engine(S, "acc_one", 0, noise_std=0.7)
    o, d, t = _rays(R, S, 4)
    for r0 in range(0, R, chunk):
        sl = slice(r0, min(R, r0 + chunk))
        want = _hook(eng, z["raw"][sl], t[sl], d[sl], noise_std=0.7, seed=(seed + r0) ^ CR.SALT_MAIN, training=True)
        for k in OUT:
            assert np.array_equal(_bits(z[k][sl]), _bits(want[k])), (r0, k)
    eng.close()


# ----------------------------------------------------------------------------------------------------- skipping + noise
def test_skipping_with_validation_noise_keeps_the_dense_bits():
    """Skipped samples enter the compositor as (0,0,0,-inf): the pass's sigma noise cannot open them.  A ray whose skipped
    samples all have a dense noisy pre-activation <= 0 (outside the noise's undecided margin) keeps every output bit."""
    import nerfmeshes_b200 as nm
    from conftest import load_npz
    from test_gpu_occupancy import ALL, LEGO_FOCAL, pose, rows_equal
    from test_gpu_parity import LEGO_CFG
    std, seed = 0.7, 21
    lego = nm.NeRFModel.from_npz(LEGO_CFG, load_npz("weights_lego_nerf.npz")).eval()
    lego.build_occupancy_grid()
    eng = lego._engine()
    eng.configure(noise_std=std)
    H = W = 64
    P = pose(30.0)
    o, d = eng.ray_bundle(P, H, W, LEGO_FOCAL * H / 800)
    d = d.reshape(-1, 3)
    o = o.reshape(1, 3).expand_as(d).contiguous()
    R = d.shape[0]
    render = lambda s: {k: v.clone() for k, v in eng.render_rays(o, d, 2.0, 6.0, seed=seed, want=ALL, skip_empty=s).items()}
    dense, skip = render(False), render(True)
    on, dn = o.cpu().numpy(), d.cpu().numpy()
    ok = np.ones(R, bool)
    for which, salt, t in ((0, CR.SALT_COARSE, SR.stratified(SR.linspace(64), 2.0, 6.0, False, False, R=R)),
                           (1, CR.SALT_MAIN, dense["t_vals"].cpu().numpy())):
        p = (on[:, None, :] + (dn[:, None, :] * t[:, :, None]).astype(np.float32)).astype(np.float32).reshape(-1, 3)
        ev = eng.occupancy_query(which, torch.from_numpy(p).cuda()).cpu().numpy().reshape(t.shape).astype(bool)
        sg = _raw_at(eng, which, on, dn, t)[..., 3]
        n = CR.sigma_noise(seed ^ salt, R, t.shape[1], std)
        pre = sg + n
        with np.errstate(invalid="ignore"):
            closed = np.isnan(pre) | (pre < -CR.GATE_MU * np.abs(n)) | ((pre <= 0) & (n == 0))
        ok &= (ev | closed).all(1)
    same = np.ones(R, bool)
    for k in ALL:
        same &= rows_equal(dense[k], skip[k])
    bad = int((~same & ok).sum())
    print(f"skipping with noise {std}: {ok.mean():.4f} of rays conservative, {same.mean():.4f} bit-identical, "
          f"{bad} conservative rays differ")
    assert bad == 0, f"{bad} of {int(ok.sum())} conservative rays differ"
    assert ok.mean() > 0.9, ok.mean()
