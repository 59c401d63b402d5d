"""Training backward (SURVEY §8f-1) against torch autograd on the CPU oracle: dL/dθ of
mse(coarse.rgb_map, target) + mse(fine.rgb_map, target) (src/models/model_nerf.py:88-151), both networks.

Tolerances (floating point; the reference trains in fp32):
  * random-init networks with the sigma bias lifted to +0.6 (random init puts raw sigma around 0, where the relu gate of
    individual samples is decided by fp32 noise): every parameter tensor within 6e-3 relative L2 (and no entry further
    than 3e-2 * max|grad_ref|).
    What sets this floor is not GEMM rounding but relu-gate flips: a hidden unit whose pre-activation is within the
    forward's rounding error of 0 is gated differently by two implementations, which moves that (point, unit) gradient
    entry by 100 %; with a fraction f of such entries the relative L2 difference is ~sqrt(f).  The forward recompute uses
    fp16 hi/lo halves (22 bits, the forward kernel's class) rather than bf16 ones (16 bits), which would flip more gates
  * trained lego checkpoint (sigma up to 4.6e3, saturated alphas, fine samples re-derived on device): relative L2 error
    <= 2e-2 per tensor and cosine >= 0.999 — the forward's own end-to-end difference (test_gpu_parity.py header) moves
    individual fine samples, which a sharp trained field amplifies
  * losses: 1e-5 relative
"""
import numpy as np
import pytest
import torch

from conftest import load_npz
from oracle import nerf_oracle as O
from test_gpu_parity import LEGO_CFG, BUFF_CFG, _cfg

pytestmark = pytest.mark.gpu

# Two runs of the SAME kernels on the same inputs differ only by the order of their fp32 atomic adds (split-K weight gradients,
# the bias row sums folded through shared-memory and global atomics).  Sums of ~1e5 signed terms whose partial sums exceed the
# result, so the tolerance leaves room above fp32 summation-order noise.
ATOMIC_NOISE = 1e-4


def _leafs(sd):
    return {k: (v.clone().float().requires_grad_(True) if k.endswith((".weight", ".bias")) else v.clone()) for k, v in sd.items()}


def oracle_grads(sdc, sdf, net_c, net_f, rc, o, d, near, far, target):
    sdc, sdf = _leafs(sdc), (_leafs(sdf) if sdf is not None else None)
    bc, bf, _, _ = O.nerf_forward(sdc, sdf, net_c, net_f, rc, o, d, near, far)
    lc = torch.nn.functional.mse_loss(bc.rgb_map, target)
    lf = torch.nn.functional.mse_loss(bf.rgb_map, target) if bf is not None else None
    (lc + (lf if lf is not None else 0.0)).backward()
    gc = {k: v.grad for k, v in sdc.items() if v.requires_grad}
    gf = {k: v.grad for k, v in sdf.items() if v.requires_grad} if sdf is not None else None
    return lc.item(), (lf.item() if lf is not None else None), gc, gf


def model_grads(model, o, d, bounds, target, seed=0):
    model.zero_grad(set_to_none=True)
    coarse, fine = model.forward((o, d, bounds), seed=seed)
    lc = torch.nn.functional.mse_loss(coarse.rgb_map, target)
    lf = torch.nn.functional.mse_loss(fine.rgb_map, target) if fine is not None else None
    (lc + (lf if lf is not None else 0.0)).backward()
    nets = model._nets()
    gc = {k: p.grad.cpu() for k, p in nets[0].named_parameters()}
    gf = {k: p.grad.cpu() for k, p in nets[1].named_parameters()} if len(nets) > 1 and nets[1] is not None else None
    return lc.item(), (lf.item() if lf is not None else None), gc, gf


def compare(got, ref, rel_max=None, rel_l2=None, cos=None, name=""):
    assert set(got) == set(ref), (sorted(got), sorted(ref))
    worst, bad, table = 0.0, [], []
    for k in ref:
        a, b = got[k].double().flatten(), ref[k].double().flatten()
        assert a.shape == b.shape, (name, k, a.shape, b.shape)
        scale = float(b.abs().max())
        err = float((a - b).abs().max())
        e2 = float((a - b).norm() / b.norm().clamp_min(1e-30))
        c = float(torch.dot(a, b) / (a.norm() * b.norm()).clamp_min(1e-30))
        table.append(f"  {k:24s} max|ref| {scale:.3e}  max err {err:.3e}  rel L2 {e2:.3e}  cos {c:.6f}")
        worst = max(worst, err / max(scale, 1e-30))
        ok = bool(torch.isfinite(a).all())
        ok &= rel_max is None or err <= rel_max * scale + 1e-10
        ok &= rel_l2 is None or e2 <= rel_l2
        ok &= cos is None or c >= cos or scale == 0.0
        if not ok:
            bad.append(k)
    assert not bad, f"{name}: {len(bad)} tensors outside tolerance {bad}\n" + "\n".join(table)
    return worst


@pytest.mark.parametrize("case", ["nerf256", "tiny_coarse_only", "no_viewdirs_skip2"])
def test_backward_matches_autograd_random_init(case):
    import nerfmeshes_b200 as nm
    if case == "nerf256":
        net_c = net_f = O.NetCfg()
        kw = dict(nc=24, nf=40, white=True)
    elif case == "tiny_coarse_only":
        net_c, net_f = O.NetCfg(num_layers=4, hidden_size=128, skip_step=4, num_encoding_fn_xyz=6, num_encoding_fn_dir=4), None
        kw = dict(nc=32, nf=0, lindisp=True)
    else:
        net_c = net_f = O.NetCfg(num_layers=6, hidden_size=256, skip_step=2, num_encoding_fn_xyz=8, use_viewdirs=False)
        kw = dict(nc=16, nf=17)
    sdc = O.init_weights(net_c, 11)
    sdf = O.init_weights(net_f, 12) if net_f is not None else None
    for sd in (sdc, sdf):        # random init puts raw sigma around 0, where the relu gate (sigma > 0) of individual
        if sd is not None:       # samples is decided by fp32 noise; lift it clear of 0 (closed gates: lego test below)
            if "fc_alpha.bias" in sd:
                sd["fc_alpha.bias"] = sd["fc_alpha.bias"] + 0.6
            else:
                sd["fc_out.bias"] = sd["fc_out.bias"] + torch.tensor([0.0, 0.0, 0.0, 0.6])
    model = nm.NeRFModel(_cfg(net_c, net_f, **kw)).cuda().train()         # _cfg: no jitter / noise -> deterministic samples
    model.model_coarse.load_state_dict(sdc, strict=False)
    if sdf is not None:
        model.model_fine.load_state_dict(sdf, strict=False)
    g = torch.Generator().manual_seed(5)
    R = 301
    o = torch.randn(R, 3, generator=g) * 0.3
    d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1) * (0.7 + torch.rand(R, 1, generator=g))
    target = torch.rand(R, 3, generator=g)
    near, far = torch.tensor(0.5), torch.tensor(3.5)
    rc = O.RenderCfg(num_coarse=kw["nc"], num_fine=kw["nf"], lindisp=kw.get("lindisp", False), white_background=kw.get("white", False))
    lc_ref, lf_ref, gc_ref, gf_ref = oracle_grads(sdc, sdf, net_c, net_f, rc, o, d, near, far, target)
    lc, lf, gc, gf = model_grads(model, o.cuda(), d.cuda(), (near, far), target.cuda())
    assert abs(lc - lc_ref) <= 1e-5 * abs(lc_ref) and (lf_ref is None or abs(lf - lf_ref) <= 1e-5 * abs(lf_ref))
    w = compare(gc, gc_ref, rel_max=3e-2, rel_l2=6e-3, name=f"{case} coarse")
    if gf_ref is not None:
        w = max(w, compare(gf, gf_ref, rel_max=3e-2, rel_l2=6e-3, name=f"{case} fine"))
    print(f"{case}: worst max-err / max|ref| = {w:.2e}")


def test_backward_matches_autograd_lego_checkpoint():
    import nerfmeshes_b200 as nm
    z = load_npz("weights_lego_nerf.npz")
    g = load_npz("golden_lego_nerf.npz")
    model = nm.NeRFModel.from_npz({**LEGO_CFG, "nerf.train.radiance_field_noise_std": 0.0}, z).cuda().train()
    sdc = {k[len("coarse."):]: torch.as_tensor(v) for k, v in z.items() if k.startswith("coarse.")}
    sdf = {k[len("fine."):]: torch.as_tensor(v) for k, v in z.items() if k.startswith("fine.")}
    R = 96
    o, d = torch.as_tensor(g["origin"]), torch.as_tensor(g["dirs"])[:R]
    target = torch.rand(R, 3, generator=torch.Generator().manual_seed(1))
    near, far = float(g["bounds"][0]), float(g["bounds"][1])
    rc = O.RenderCfg()
    lc_ref, lf_ref, gc_ref, gf_ref = oracle_grads(sdc, sdf, O.NetCfg(), O.NetCfg(), rc, o, d, torch.tensor(near), torch.tensor(far), target)
    lc, lf, gc, gf = model_grads(model, o.cuda(), d.cuda(), torch.tensor([near, far]), target.cuda())
    assert abs(lc - lc_ref) <= 1e-4 * abs(lc_ref) and abs(lf - lf_ref) <= 1e-4 * abs(lf_ref)
    compare(gc, gc_ref, rel_l2=2e-2, cos=0.999, name="lego coarse")
    compare(gf, gf_ref, rel_l2=2e-2, cos=0.999, name="lego fine")


def test_fused_loss_backward_equals_autograd_path_and_accumulates():
    """nm_loss_backward (loss + backward in one call) == the autograd.Function path, in TRAINING mode with jitter and
    sigma noise (same seed -> same random stream); a second call without nm_zero_grad doubles the buffers."""
    import nerfmeshes_b200 as nm
    net = O.NetCfg(num_layers=4, hidden_size=128, num_encoding_fn_xyz=6)
    cfg = _cfg(net, net, nc=20, nf=28)
    cfg.update({"nerf.train.perturb": True, "nerf.train.radiance_field_noise_std": 0.3})
    model = nm.NeRFModel(cfg).cuda().train()
    model.model_coarse.load_state_dict(O.init_weights(net, 1), strict=False)
    model.model_fine.load_state_dict(O.init_weights(net, 2), strict=False)
    g = torch.Generator().manual_seed(2)
    R = 777
    o = (torch.randn(3, generator=g) * 0.2).cuda()
    d = torch.randn(R, 3, generator=g).cuda()
    target = torch.rand(R, 3, generator=g).cuda()
    lc, lf, gc, gf = model_grads(model, o, d, (torch.tensor(0.5), torch.tensor(3.0)), target, seed=1234)
    eng = model._engine()
    eng.zero_grad()
    loss = eng.loss_backward(o, d, 0.5, 3.0, target, training=True, seed=1234)
    assert abs(float(loss[0]) - lc) <= 1e-6 * abs(lc) + 1e-9 and abs(float(loss[1]) - lf) <= 1e-6 * abs(lf) + 1e-9
    fused_c = {k: eng.get_grad(0, k, p).cpu() for k, p in model.model_coarse.named_parameters()}
    fused_f = {k: eng.get_grad(1, k, p).cpu() for k, p in model.model_fine.named_parameters()}
    compare(fused_c, gc, rel_max=ATOMIC_NOISE, name="fused coarse")
    compare(fused_f, gf, rel_max=ATOMIC_NOISE, name="fused fine")
    eng.loss_backward(o, d, 0.5, 3.0, target, training=True, seed=1234)            # accumulate
    twice = {k: eng.get_grad(1, k, p).cpu() for k, p in model.model_fine.named_parameters()}
    compare(twice, {k: 2 * v for k, v in gf.items()}, rel_max=ATOMIC_NOISE, name="accumulated")
    # a different seed draws different jitter / noise
    lc2, _, gc2, _ = model_grads(model, o, d, (torch.tensor(0.5), torch.tensor(3.0)), target, seed=99)
    assert lc2 != lc and not torch.equal(gc2["layer1.weight"], gc["layer1.weight"])


def test_direct_and_subchunk_walks_agree(monkeypatch):
    """The backward either reuses what the training forward emitted (whole chunk in the workspace, the default) or walks
    sub-chunks with a recompute each (NM_TRAIN_DIRECT_GB=0, what a chunk beyond the budget gets; 6000 rays x 64 samples take
    two sub-chunks of 16 waves).  Same masks, same operands: they differ by atomic order only."""
    import nerfmeshes_b200 as nm
    net = O.NetCfg()
    cfg = _cfg(net, net, nc=24, nf=40)
    cfg.update({"nerf.train.perturb": True, "nerf.train.radiance_field_noise_std": 0.5})
    model = nm.NeRFModel(cfg).cuda().train()
    model.model_coarse.load_state_dict(O.init_weights(net, 3), strict=False)
    model.model_fine.load_state_dict(O.init_weights(net, 4), strict=False)
    g = torch.Generator().manual_seed(8)
    R = 6000
    o = (torch.randn(3, generator=g) * 0.2).cuda()
    d = torch.randn(R, 3, generator=g).cuda()
    target = torch.rand(R, 3, generator=g).cuda()
    eng = model._engine()

    def run():
        eng.zero_grad()
        loss = eng.loss_backward(o, d, 0.5, 3.0, target, training=True, seed=77)
        return ([float(x) for x in loss[:2]],
                {k: eng.get_grad(0, k, p).cpu() for k, p in model.model_coarse.named_parameters()},
                {k: eng.get_grad(1, k, p).cpu() for k, p in model.model_fine.named_parameters()})
    l_dir, c_dir, f_dir = run()
    monkeypatch.setenv("NM_TRAIN_DIRECT_GB", "0")
    l_sub, c_sub, f_sub = run()
    assert all(abs(a - b) <= 1e-6 * abs(a) for a, b in zip(l_dir, l_sub))      # the loss is an atomic sum of block partials
    compare(c_sub, c_dir, rel_max=ATOMIC_NOISE, name="walks coarse")
    compare(f_sub, f_dir, rel_max=ATOMIC_NOISE, name="walks fine")


def test_buff_backward_matches_autograd():
    import nerfmeshes_b200 as nm
    z = load_npz("weights_lego_buff.npz")
    g = load_npz("golden_lego_buff.npz")
    model = nm.BuFFModel.from_npz({**BUFF_CFG, "nerf.train.radiance_field_noise_std": 0.0}, z).cuda().train()
    sd = _leafs({k[len("coarse."):]: torch.as_tensor(v) for k, v in z.items() if k.startswith("coarse.")})
    R = 48
    o, d = torch.as_tensor(g["origin"])[None], torch.as_tensor(g["dirs"])[:R]
    target = torch.rand(R, 3, generator=torch.Generator().manual_seed(3))
    near, far = float(g["bounds"][0]), float(g["bounds"][1])
    rc = O.RenderCfg(num_coarse=192, num_fine=0)
    b, _, _ = O.buff_forward(sd, O.NetCfg(), rc, torch.as_tensor(z["voxels"]).float(), o, d, torch.tensor(near), torch.tensor(far))
    loss_ref = torch.nn.functional.mse_loss(b.rgb_map, target)
    loss_ref.backward()
    ref = {k: v.grad for k, v in sd.items() if v.requires_grad}
    model.zero_grad(set_to_none=True)
    out = model.forward((o.cuda(), d.cuda(), torch.tensor([near, far])))
    loss = torch.nn.functional.mse_loss(out.rgb_map, target.cuda())
    loss.backward()
    assert abs(loss.item() - loss_ref.item()) <= 1e-4 * loss_ref.item()
    got = {k: p.grad.cpu() for k, p in model.model.named_parameters()}
    compare(got, ref, rel_l2=2e-2, cos=0.999, name="buff")


def test_training_loop_reduces_loss():
    """The reference's optimiser loop (Adam, model_base.py:150-177) on top of the fused forward/backward: fitting a
    constant-colour target must drive the loss down, which exercises weight re-upload after every step."""
    import nerfmeshes_b200 as nm
    torch.manual_seed(0)
    net = O.NetCfg(num_layers=4, hidden_size=128, num_encoding_fn_xyz=6)
    cfg = _cfg(net, net, nc=24, nf=24)
    cfg.update({"nerf.train.perturb": True, "nerf.train.radiance_field_noise_std": 0.1})
    model = nm.NeRFModel(cfg).cuda().train()
    opt = torch.optim.Adam(model.parameters(), lr=2e-3)
    g = torch.Generator().manual_seed(4)
    R = 1024
    o = torch.tensor([0.0, 0.0, 0.0]).cuda()
    d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1).cuda()
    target = torch.tensor([0.8, 0.3, 0.1]).expand(R, 3).contiguous().cuda()
    losses = []
    for step in range(40):
        opt.zero_grad(set_to_none=True)
        coarse, fine = model.forward((o, d, (torch.tensor(0.5), torch.tensor(3.0))))
        loss = torch.nn.functional.mse_loss(coarse.rgb_map, target) + torch.nn.functional.mse_loss(fine.rgb_map, target)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert np.isfinite(losses).all() and losses[-1] < 0.25 * losses[0], losses[::8]


def test_device_side_weight_load_is_bit_identical():
    """nm_load_weights_dev (transpose + fp16 hi/lo stage packing on the device) == the host packer."""
    import nerfmeshes_b200 as nm
    z = load_npz("weights_lego_nerf.npz")
    g = load_npz("golden_lego_nerf.npz")
    rays = (torch.as_tensor(g["origin"]).cuda(), torch.as_tensor(g["dirs"]).cuda(), torch.as_tensor(g["bounds"]))
    model = nm.NeRFModel.from_npz(LEGO_CFG, z).eval()               # CPU parameters -> host path
    with torch.no_grad():
        a = model.query(rays)
        pts = torch.rand(1000, 3).cuda() * 2 - 1
        pa = model.sample_points(pts, pts)
        model.cuda()                                                # CUDA parameters -> device path
        b = model.query(rays)
        pb = model.sample_points(pts, pts)
    assert torch.equal(a.rgb_map, b.rgb_map) and torch.equal(a.depth_map, b.depth_map) and torch.equal(pa, pb)
    close = float((b.rgb_map.cpu() - torch.as_tensor(g["fine_rgb"])).abs().max())
    assert close < 1e-4, close


@pytest.mark.parametrize("shape", [
    dict(M=256, N=63, K=5000),                       # weight gradient (encoding part): K = points, split + atomics
    dict(M=128, N=256, K=70001),
])
def test_tc_gemm_matches_fp64(shape):
    """The backward's weight-gradient GEMM (operand split x = hi + lo, 3 MMAs per product; A as MN-major, B as K-major
    tiles) against an fp64 product.  Errors are measured against the random-walk scale s = sqrt((A*A)(B*B)^T): bf16
    halves (16 significand bits per operand) must stay within 1e-4*s (expected ~2^-17 per term), and the one-pass variant
    (bf16's 8 bits) must be at least 30x worse than the three-pass one — i.e. the two correction passes really
    contribute."""
    import nerfmeshes_b200 as nm
    eng = nm.Engine(O.NetCfg().__dict__, None, nm.RenderSettings())
    M, N, K = shape["M"], shape["N"], shape["K"]
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g) * torch.logspace(-2, 1, K)[None, :]        # wide dynamic range along K
    b = torch.randn(N, K, generator=g)
    ref = a.double() @ b.double().T
    scale = ((a.double() ** 2) @ (b.double() ** 2).T).sqrt()
    A, B = a.T.contiguous().cuda(), b.T.contiguous().cuda()                       # point-major, like dZ and the activations
    worst = {}
    for name, n_passes in (("bf16x3", 3), ("bf16x1", 1)):
        d = eng.debug_gemm(A, B, n_passes=n_passes)
        worst[name] = float(((d.cpu().double() - ref).abs() / scale).max())
    assert worst["bf16x3"] <= 1e-4 and worst["bf16x1"] >= 30 * worst["bf16x3"], (shape, worst)
    d1 = eng.debug_gemm(A, B, n_passes=3)                                          # atomic: a second call accumulates
    d2 = eng.debug_gemm(A, B, n_passes=3, out=d1.clone())
    assert float(((d2.cpu().double() - 2 * ref).abs() / scale).max()) <= 2e-4


def test_backward_tensor_core_vs_cuda_core_yardstick():
    """The same backward with the GEMMs on the tensor cores (default) and in plain fp32 FMAs (NM_PREC_FP32)."""
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import _lib as L
    net = O.NetCfg()
    model = nm.NeRFModel(_cfg(net, net, nc=32, nf=32)).cuda().train()
    sdc, sdf = O.init_weights(net, 21), O.init_weights(net, 22)
    sdc["fc_alpha.bias"] = sdc["fc_alpha.bias"] + 0.6
    sdf["fc_alpha.bias"] = sdf["fc_alpha.bias"] + 0.6
    model.model_coarse.load_state_dict(sdc, strict=False)
    model.model_fine.load_state_dict(sdf, strict=False)
    g = torch.Generator().manual_seed(8)
    R = 1500
    o = (torch.randn(3, generator=g) * 0.2).cuda()
    d = torch.randn(R, 3, generator=g).cuda()
    target = torch.rand(R, 3, generator=g).cuda()
    bounds = (torch.tensor(0.5), torch.tensor(3.0))
    _, _, gc, gf = model_grads(model, o, d, bounds, target, seed=5)
    model.precision = L.PREC_FP32
    _, _, gc32, gf32 = model_grads(model, o, d, bounds, target, seed=5)
    compare(gc, gc32, rel_max=3e-2, rel_l2=6e-3, name="tc vs fp32 coarse")
    compare(gf, gf32, rel_max=3e-2, rel_l2=6e-3, name="tc vs fp32 fine")


@pytest.mark.parametrize("case", ["nerf256", "skip2_no_viewdirs"])
def test_backward_fp32_mode_matches_autograd_per_layer(case):
    """NM_PREC_FP32 (plain fp32 FMAs, the same arithmetic class as torch on the CPU) against autograd through the oracle,
    per parameter tensor: relative L2 <= 5e-3 and cosine >= 0.9999.  A scaling / indexing error confined to
    ONE layer's gradient (1 % gives 1e-2) cannot pass here, and the tensor-core path is tied to this one by
    test_backward_tensor_core_vs_cuda_core_yardstick."""
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import _lib as L
    if case == "nerf256":
        net = O.NetCfg()
        nc, nf = 24, 40
    else:
        net = O.NetCfg(num_layers=6, hidden_size=256, skip_step=2, num_encoding_fn_xyz=8, use_viewdirs=False)
        nc, nf = 16, 17
    sdc, sdf = O.init_weights(net, 31), O.init_weights(net, 32)
    for sd in (sdc, sdf):
        if "fc_alpha.bias" in sd:
            sd["fc_alpha.bias"] = sd["fc_alpha.bias"] + 0.6
        else:
            sd["fc_out.bias"] = sd["fc_out.bias"] + torch.tensor([0.0, 0.0, 0.0, 0.6])
    model = nm.NeRFModel(_cfg(net, net, nc=nc, nf=nf)).cuda().train()
    model.precision = L.PREC_FP32
    model.model_coarse.load_state_dict(sdc, strict=False)
    model.model_fine.load_state_dict(sdf, strict=False)
    g = torch.Generator().manual_seed(6)
    R = 257
    o = torch.randn(R, 3, generator=g) * 0.3
    d = torch.nn.functional.normalize(torch.randn(R, 3, generator=g), dim=-1)
    target = torch.rand(R, 3, generator=g)
    near, far = torch.tensor(0.5), torch.tensor(3.5)
    rc = O.RenderCfg(num_coarse=nc, num_fine=nf)
    lc_ref, lf_ref, gc_ref, gf_ref = oracle_grads(sdc, sdf, net, net, rc, o, d, near, far, target)
    lc, lf, gc, gf = model_grads(model, o.cuda(), d.cuda(), (near, far), target.cuda())
    assert abs(lc - lc_ref) <= 1e-5 * abs(lc_ref) and abs(lf - lf_ref) <= 1e-5 * abs(lf_ref)
    w = max(compare(gc, gc_ref, rel_l2=5e-3, cos=0.9999, name=f"fp32 {case} coarse"), compare(gf, gf_ref, rel_l2=5e-3, cos=0.9999, name=f"fp32 {case} fine"))
    print(f"fp32 {case}: worst max-err / max|ref| = {w:.2e}")


def test_fused_training_step_matches_autograd_route():
    """nerfmeshes_b200.training_step (the reference's training_step body with manual batching, one fused call per chunk)
    == forward/backward through autograd on the same chunks with the same seeds; log values like the reference."""
    import nerfmeshes_b200 as nm
    net = O.NetCfg(num_layers=4, hidden_size=128, num_encoding_fn_xyz=6)
    cfg = _cfg(net, net, nc=16, nf=24)
    cfg.update({"nerf.train.perturb": True, "nerf.train.radiance_field_noise_std": 0.2, "nerf.train.chunksize": 400})
    model = nm.NeRFModel(cfg).cuda().train()
    model.model_coarse.load_state_dict(O.init_weights(net, 5), strict=False)
    model.model_fine.load_state_dict(O.init_weights(net, 6), strict=False)
    g = torch.Generator().manual_seed(12)
    R = 800
    o = (torch.randn(3, generator=g) * 0.2).cuda()
    d = torch.randn(R, 3, generator=g).cuda()
    target = torch.rand(R, 3, generator=g).cuda()
    bounds = (torch.tensor(0.5), torch.tensor(3.0))
    model.zero_grad(set_to_none=True)
    out = nm.training_step(model, (o, d, bounds), target, seed=77)
    fused = {f"{w}.{k}": p.grad.clone().cpu() for w, k, p in model._named_net_params()}
    model.zero_grad(set_to_none=True)
    lc = lf = 0.0
    for i in range(0, R, 400):
        coarse, fine = model.forward((o, d[i:i + 400], bounds), seed=77 + i)
        lc = lc + torch.nn.functional.mse_loss(coarse.rgb_map, target[i:i + 400])
        lf = lf + torch.nn.functional.mse_loss(fine.rgb_map, target[i:i + 400])
    lc, lf = lc / 2, lf / 2
    (lc + lf).backward()
    ref = {f"{w}.{k}": p.grad.cpu() for w, k, p in model._named_net_params()}
    compare(fused, ref, rel_max=ATOMIC_NOISE, name="fused training_step")
    log = out["log"]
    assert abs(log["train/coarse_loss"] - lc.item()) <= 1e-6 * lc.item() and abs(log["train/fine_loss"] - lf.item()) <= 1e-6 * lf.item()
    assert abs(out["loss"] - (lc + lf).item()) <= 1e-6 * out["loss"] and abs(log["train/fine_psnr"] + 10 * np.log10(lf.item())) < 1e-4
