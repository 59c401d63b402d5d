"""The training compositor adjoint (`composite_backward_kernel`, nm_train.cu, through the nm_debug_composite_backward
hook) against the float64 truth of tests/_composite_ref.py, element by element, and the sigma noise of the training
backward against the forward's, end to end.

Hook: |dout - truth| <= TAU * error_scale for all four components over the edge matrix of tests/test_composite_adjoint.py
(every segment length 1..16 with full, partly filled and empty last lanes; R = 1, 3, 5 against the kernel's 4 rays per
block with every white-background / noise setting, and R = 4099 once per S), seven ray kinds (`make_rays`: random,
sigma <= 0 with exact zeros, e == 0 on the first sample, transmittance through the subnormals to 0, 2^-25 < e < 2^-10,
a tiny positive sigma on the last sample, zero-length intervals), |d| from 0.05 to 20, noise 0 and 0.7 with two seeds.
d sigma must be exactly 0 where the noisy pre-activation is <= 0 outside the noise margin and where e == 0, two calls
must agree bit for bit, and the hook rejects malformed arguments without launching anything.

End to end: training gradients and losses with sigma noise on against autograd through the oracle fed the noise the
device draws (`_composite_ref.sigma_noise`): seed ^ kNoiseSaltCoarse for the coarse pass, seed ^ kNoiseSaltMain for the
fine or only pass.  The same comparison against an oracle fed the two salts swapped must miss its bar by
SWAP_MARGIN — the comparison sees the wiring.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import _composite_ref as CR
from conftest import load_npz
from oracle import nerf_oracle as O
from test_composite_adjoint import NOISE, S_ALL
from test_gpu_parity import BUFF_CFG, _cfg
from test_gpu_train import _leafs, compare, model_grads

pytestmark = pytest.mark.gpu

# The swapped-salt oracle misses the random-init bar (relative L2 6e-3) by at least this factor on every case
# (measured on an H100 80GB HBM3, 700 W limit: 210x two-network NeRF, 111x coarse-only, 106x BuFF; the matching oracle
# sits at 6.1e-4, 4.3e-4, 2.1e-4).
SWAP_MARGIN = 25.0


def _engine():
    import nerfmeshes_b200 as nm
    return nm.Engine(O.NetCfg().__dict__, None, nm.RenderSettings())


def _run(eng, raw, t, d, g, white, std, seed):
    out = eng.debug_composite_backward(torch.from_numpy(raw).cuda(), torch.from_numpy(t).cuda(), torch.from_numpy(d).cuda(),
                                       torch.from_numpy(g).cuda(), noise_std=std, seed=seed, white_bg=white)
    return out.cpu().numpy()


def test_hook_matches_float64_truth_over_the_edge_matrix():
    eng = _engine()
    worst, worst_at = 0.0, None
    for S in S_ALL:
        cases = [(R, white, std, seed) for R in (1, 3, 5) for white in (0, 1) for std, seed in NOISE]
        cases.append((4099, S % 2, *NOISE[S % 3]))
        for R, white, std, seed in cases:
            raw, t, d, g, kinds = CR.make_rays(R, S, 7919 * S + 31 * R + 2 * white + int(std > 0), kind_offset=S + R)
            got = _run(eng, raw, t, d, g, white, std, seed)
            a = CR.composite_adjoint(raw, t, d, g, white, std, seed)
            r = CR.ratio(got, a.dout(), CR.error_scale(a, S))
            assert np.isfinite(got).all(), (S, R, white, std)
            if r.max() > worst:
                i = np.unravel_index(r.argmax(), r.shape)
                worst, worst_at = float(r.max()), (S, R, white, std, CR.KINDS[kinds[i[0]]], int(i[1]), int(i[2]))
            assert r.max() <= CR.TAU, (S, R, white, std, float(r.max()))
            # exact zeros: a closed gate outside the noise margin, and e == 0 (x >= 110: exp(-x) far below 2^-150)
            zero = ((a.pre <= 0) & ~CR.undecided(a)) | (a.x >= 110)
            assert (got[..., 3][zero] == 0).all(), (S, R, white, std)
    print(f"RATIO hook-vs-truth {worst:.3e} at S,R,white,noise,kind,sample,component = {worst_at}")
    eng.close()


def test_hook_is_deterministic():
    eng = _engine()
    raw, t, d, g, _ = CR.make_rays(4099, 257, 3)
    a = _run(eng, raw, t, d, g, 1, 0.7, NOISE[1][1])
    b = _run(eng, raw, t, d, g, 1, 0.7, NOISE[1][1])
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    eng.close()


def test_hook_rejects_bad_arguments_without_launching():
    eng = _engine()
    lib, h = eng.lib, eng._h
    R, S = 5, 40
    buf = torch.zeros(R * S * 4 + 4, device="cuda")
    raw, dout = buf[:R * S * 4], torch.zeros(R * S * 4 + 4, device="cuda")
    t, d, g = torch.zeros(R * S, device="cuda"), torch.ones(R * 3, device="cuda"), torch.ones(R * 3, device="cuda")
    p = lambda x, off=0: C.c_void_p(x.data_ptr() + 4 * off)
    st = eng._stream()

    def call(raw_p, t_p, d_p, g_p, n, s, out_p):
        return lib.nm_debug_composite_backward(h, raw_p, t_p, d_p, g_p, n, s, 0.0, 0, 0, out_p, st)
    ok = (p(raw), p(t), p(d), p(g))
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    bad = [
        (None, p(t), p(d), p(g), R, S, p(dout)), (p(raw), None, p(d), p(g), R, S, p(dout)),
        (p(raw), p(t), None, p(g), R, S, p(dout)), (p(raw), p(t), p(d), None, R, S, p(dout)),
        (*ok, R, S, None), (*ok, -1, S, p(dout)), (*ok, R, 0, p(dout)), (*ok, R, 513, p(dout)),
        (p(buf, 1), p(t), p(d), p(g), R, S, p(dout)), (*ok, R, S, p(dout, 1)),
    ]
    for args in bad:
        assert call(*args) != 0, args
        assert lib.nm_last_error()
    assert call(*ok, 0, S, p(dout)) == 0                    # R = 0: nothing to do
    assert eng.launch_count() == n0
    assert call(*ok, R, S, p(dout)) == 0 and eng.launch_count() == n0 + 1
    eng.close()


# ----------------------------------------------------------------------------------------------------- end to end
def _noise(seed, salt, R, S, std):
    return torch.from_numpy(CR.sigma_noise(seed ^ salt, R, S, std))


def _lift(sd):
    """random init puts raw sigma around 0, where fp32 noise decides relu gates: lift it (as test_gpu_train does)"""
    if "fc_alpha.bias" in sd:
        sd["fc_alpha.bias"] = sd["fc_alpha.bias"] + 0.6
    else:
        sd["fc_out.bias"] = sd["fc_out.bias"] + torch.tensor([0.0, 0.0, 0.0, 0.6])
    return sd


def _rel_l2(got, ref):
    return max(float((got[k].double() - ref[k].double()).norm() / ref[k].double().norm().clamp_min(1e-30)) for k in ref)


NOISE_STD, SEED = 0.7, 4242


@pytest.mark.parametrize("case", ["nerf", "coarse_only", "buff"])
def test_training_noise_matches_oracle_fed_the_device_noise(case):
    import nerfmeshes_b200 as nm
    net = O.NetCfg(num_layers=4, hidden_size=128, num_encoding_fn_xyz=6)
    g = torch.Generator().manual_seed(17)
    if case == "buff":
        z = load_npz("weights_lego_buff.npz")
        gold = load_npz("golden_lego_buff.npz")
        net = O.NetCfg()
        model = nm.BuFFModel.from_npz({**BUFF_CFG, "nerf.train.radiance_field_noise_std": NOISE_STD}, z).cuda().train()
        sdc, sdf = _lift(O.init_weights(net, 23)), None
        model.model.load_state_dict(sdc, strict=False)
        R, nc, nf = 48, 192, 0
        o, d = torch.as_tensor(gold["origin"])[None], torch.as_tensor(gold["dirs"])[:R]
        near, far = float(gold["bounds"][0]), float(gold["bounds"][1])
        voxels = torch.as_tensor(z["voxels"]).float()
    else:
        nc, nf = (24, 40) if case == "nerf" else (32, 0)
        cfg = _cfg(net, net if nf else None, nc=nc, nf=nf, white=case == "nerf")
        cfg["nerf.train.radiance_field_noise_std"] = NOISE_STD
        model = nm.NeRFModel(cfg).cuda().train()
        sdc = _lift(O.init_weights(net, 21))
        sdf = _lift(O.init_weights(net, 22)) if nf else None
        model.model_coarse.load_state_dict(sdc, strict=False)
        if sdf is not None:
            model.model_fine.load_state_dict(sdf, strict=False)
        R = 301
        o = torch.randn(R, 3, generator=g) * 0.3
        d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1) * (0.7 + torch.rand(R, 1, generator=g))
        near, far = 2.0, 6.0
    target = torch.rand(R, 3, generator=g)
    S = nc + nf

    def oracle(salt_c, salt_f):
        """losses and gradients of the oracle fed the noise of the two streams (coarse-or-only pass, fine pass)"""
        rc = O.RenderCfg(num_coarse=nc, num_fine=nf, white_background=case == "nerf", noise_std=NOISE_STD)
        lc_sd = _leafs(sdc)
        if case == "buff":
            b, _, _ = O.buff_forward(lc_sd, net, rc, voxels, o, d, torch.tensor(near), torch.tensor(far),
                                     noise=_noise(SEED, salt_f, R, nc, NOISE_STD))
            loss = torch.nn.functional.mse_loss(b.rgb_map, target)
            loss.backward()
            return loss.item(), None, {k: v.grad for k, v in lc_sd.items() if v.requires_grad}, None
        lf_sd = _leafs(sdf) if sdf is not None else None
        # the coarse pass of a two-network model draws from the coarse salt, a coarse-only model's from the main one
        bc, bf, _, _ = O.nerf_forward(lc_sd, lf_sd, net, net if nf else None, rc, o, d, torch.tensor(near), torch.tensor(far),
                                      noise_c=_noise(SEED, salt_c if nf else salt_f, R, nc, NOISE_STD),
                                      noise_f=_noise(SEED, salt_f, R, S, NOISE_STD) if nf else None)
        lc = torch.nn.functional.mse_loss(bc.rgb_map, target)
        lf = torch.nn.functional.mse_loss(bf.rgb_map, target) if bf is not None else None
        (lc + (lf if lf is not None else 0.0)).backward()
        return (lc.item(), lf.item() if lf is not None else None, {k: v.grad for k, v in lc_sd.items() if v.requires_grad},
                {k: v.grad for k, v in lf_sd.items() if v.requires_grad} if lf_sd is not None else None)

    if case == "buff":
        model.zero_grad(set_to_none=True)
        out = model.forward((o.cuda(), d.cuda(), torch.tensor([near, far])), seed=SEED)
        loss = torch.nn.functional.mse_loss(out.rgb_map, target.cuda())
        loss.backward()
        lc, lf, gc, gf = loss.item(), None, {k: p.grad.cpu() for k, p in model.model.named_parameters()}, None
    else:
        lc, lf, gc, gf = model_grads(model, o.cuda(), d.cuda(), (torch.tensor(near), torch.tensor(far)), target.cuda(), seed=SEED)
    lc_ref, lf_ref, gc_ref, gf_ref = oracle(CR.SALT_COARSE, CR.SALT_MAIN)
    assert abs(lc - lc_ref) <= 1e-5 * abs(lc_ref) and (lf_ref is None or abs(lf - lf_ref) <= 1e-5 * abs(lf_ref)), (lc, lc_ref, lf, lf_ref)
    compare(gc, gc_ref, rel_max=3e-2, rel_l2=6e-3, name=f"{case} coarse")
    good = _rel_l2(gc, gc_ref)
    if gf_ref is not None:
        compare(gf, gf_ref, rel_max=3e-2, rel_l2=6e-3, name=f"{case} fine")
        good = max(good, _rel_l2(gf, gf_ref))
    # the control: the same device gradients against the oracle fed the swapped salts
    _, _, sc_ref, sf_ref = oracle(CR.SALT_MAIN, CR.SALT_COARSE)
    swapped = max(_rel_l2(gc, sc_ref), _rel_l2(gf, sf_ref) if sf_ref is not None else 0.0)
    print(f"RATIO noise-wiring {case}: rel L2 {good:.3e} (bar 6e-3), swapped salts {swapped:.3e} = {swapped / 6e-3:.1f}x the bar")
    assert swapped >= SWAP_MARGIN * 6e-3, (case, swapped)
