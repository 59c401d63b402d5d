"""The fused MLP kernel's weight ring at every depth, and the sigma-only coarse pass.

* Renders (lego, fern) and point_mlp are bit-identical with the ring capped at 2 and 3 slots (NM_MLP_RING_SLOTS) and at
  the depth the layout allows: the depth changes when stages land, never which products a column sums or in what order.
* A training step's gradients at 2 slots and at full depth agree within the fp32 atomic-order noise of two runs.
* A coarse pass whose caller reads no coarse colour runs the sigma-only program; its weights, acc and disp, and so every
  fine map, are bit-identical to a render that also asks for coarse_rgb (which keeps the full program), with a partial
  last tile group and over a render of several internal chunks.  Networks without view directions keep the full program.
"""
import pytest
import torch

from conftest import load_npz
from oracle import nerf_oracle as O
from test_gpu_parity import LEGO_CFG, _cfg
from test_gpu_train import ATOMIC_NOISE, compare

pytestmark = pytest.mark.gpu

PRECS = ["exact", "fast"]
CAPS = ["2", "3", None]          # None: the layout's own depth


def _model(weights, prec, cfg=LEGO_CFG):
    import nerfmeshes_b200 as nm
    m = nm.NeRFModel.from_npz(cfg, load_npz(weights)).cuda().eval()
    m.precision = {"exact": nm.PREC_EXACT, "fast": nm.PREC_FAST}[prec]
    return m


def _at_caps(monkeypatch, fn):
    outs = []
    for cap in CAPS:
        if cap is None:
            monkeypatch.delenv("NM_MLP_RING_SLOTS", raising=False)
        else:
            monkeypatch.setenv("NM_MLP_RING_SLOTS", cap)
        outs.append(fn())
    monkeypatch.delenv("NM_MLP_RING_SLOTS", raising=False)
    return outs


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("scene", ["lego", "fern"])
def test_render_bit_identical_across_ring_depths(scene, prec, monkeypatch):
    model = _model(f"weights_{scene}_nerf.npz", prec)
    eng = model._engine()
    if scene == "lego":
        pose, H, W, f, near, far, ndc = O.pose_spherical(30.0, -30.0, 4.0), 800, 800, 1111.111, 2.0, 6.0, False
        rows = (380, 403)
    else:
        pose, H, W, f, near, far, ndc = torch.eye(4)[:3], 756, 1008, 815.13, 0.0, 1.0, True
        rows = (360, 377)
    want = ["rgb", "depth", "acc", "disp", "weights", "coarse_weights"]

    def run():
        with torch.no_grad():
            out = eng.render_image(pose, H, W, f, near, far, ndc=ndc, rows=rows, want=want)
            return {k: v.clone() for k, v in out.items()}
    outs = _at_caps(monkeypatch, run)
    for o in outs[1:]:
        for k in want:
            assert torch.equal(o[k], outs[0][k]), (scene, prec, k)
    assert float(outs[0]["acc"].max()) > 0.5


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("sigma_only", [False, True])
def test_point_mlp_bit_identical_across_ring_depths(prec, sigma_only, monkeypatch):
    model = _model("weights_lego_nerf.npz", prec)
    eng = model._engine()
    g = torch.Generator().manual_seed(7)
    M = 64 * 517 + 23
    pts = ((torch.rand(M, 3, generator=g) * 2.4) - 1.2).cuda()
    dirs = torch.nn.functional.normalize(torch.randn(M, 3, generator=g), dim=-1).cuda()
    outs = _at_caps(monkeypatch, lambda: eng.point_mlp(1, pts, dirs, sigma_only=sigma_only).clone())
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


@pytest.mark.parametrize("prec", PRECS)
def test_training_gradients_across_ring_depths(prec, monkeypatch):
    import nerfmeshes_b200 as nm
    z = load_npz("weights_lego_nerf.npz")
    model = nm.NeRFModel.from_npz({**LEGO_CFG, "nerf.train.radiance_field_noise_std": 0.0}, z).cuda().train()
    model.precision = {"exact": nm.PREC_EXACT, "fast": nm.PREC_FAST}[prec]
    eng = model._engine()
    o, d = eng.ray_bundle(O.pose_spherical(30.0, -30.0, 4.0), 800, 800, 1111.111)
    d = d.reshape(-1, 3)[320000:320000 + 1531].contiguous()
    target = torch.rand(d.shape[0], 3, generator=torch.Generator().manual_seed(3)).cuda()

    def step():
        eng.zero_grad()
        loss = eng.loss_backward(o, d, 2.0, 6.0, target, training=True, seed=5)
        grads = [{k: eng.get_grad(i, k, p).cpu() for k, p in net.named_parameters()}
                 for i, net in enumerate((model.model_coarse, model.model_fine))]
        return loss.cpu(), grads
    monkeypatch.setenv("NM_MLP_RING_SLOTS", "2")
    l2, g2 = step()
    monkeypatch.delenv("NM_MLP_RING_SLOTS")
    lm, gm = step()
    assert torch.allclose(l2, lm, rtol=1e-6, atol=0)
    for i in range(2):
        compare(g2[i], gm[i], rel_max=ATOMIC_NOISE, name=f"{prec} net {i}")


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("case", ["lego", "s40_group5", "multi_chunk", "no_viewdirs"])
def test_sigma_only_coarse_pass(case, prec):
    """coarse_rgb requested => full coarse program; not requested => sigma-only: the same fine maps and coarse weights.
    lego: the benchmark's networks; s40_group5: 40 coarse samples per ray, tile groups of 5 and a partial last tile and
    group; multi_chunk: past one internal chunk of 2^20 rays; no_viewdirs: networks with one output layer for rgb and sigma,
    which have no separate sigma program and keep the full one.  The sigma-only point count shows which program ran."""
    import nerfmeshes_b200 as nm
    g = torch.Generator().manual_seed(11)
    if case == "lego":
        model = _model("weights_lego_nerf.npz", prec)
        eng = model._engine()
        o, d = eng.ray_bundle(O.pose_spherical(-60.0, -30.0, 4.0), 800, 800, 1111.111)
        d = d.reshape(-1, 3)[300017:300017 + 4099].contiguous()
        o, near, far, nc = o.reshape(-1, 3)[:1].reshape(3), 2.0, 6.0, 64
    else:
        viewdirs = case != "no_viewdirs"
        net = O.NetCfg(num_layers=4, hidden_size=128, num_encoding_fn_xyz=6, use_viewdirs=viewdirs)
        nc = 40
        model = nm.NeRFModel(_cfg(net, net, nc=nc, nf=56)).cuda().eval()   # S = 40: tile groups of 5
        sds = [O.init_weights(net, 41), O.init_weights(net, 42)]
        for sd in sds:                 # random init leaves raw sigma around 0: lift it so that rays are not empty
            if viewdirs:
                sd["fc_alpha.bias"] = sd["fc_alpha.bias"] + 0.6
            else:
                sd["fc_out.bias"] = sd["fc_out.bias"] + torch.tensor([0.0, 0.0, 0.0, 0.6])
        model.model_coarse.load_state_dict(sds[0], strict=False)
        model.model_fine.load_state_dict(sds[1], strict=False)
        model.precision = {"exact": nm.PREC_EXACT, "fast": nm.PREC_FAST}[prec]
        eng = model._engine()
        R = (1 << 20) + 4099 if case == "multi_chunk" else 1237
        o = (torch.randn(3, generator=g) * 0.2).cuda()
        d = torch.randn(R, 3, generator=g).cuda()
        near, far = 0.5, 3.0
    R = d.shape[0]
    base = ["rgb", "depth", "depth_raw", "acc", "disp", "coarse_acc", "coarse_disp", "coarse_weights"]
    if case != "multi_chunk":
        base += ["weights", "t_vals"]
    with torch.no_grad():
        p0 = eng.sigma_only_points()
        sig = {k: v.clone() for k, v in eng.render_rays(o, d, near, far, seed=3, want=base).items()}
        p1 = eng.sigma_only_points()
        full = {k: v.clone() for k, v in eng.render_rays(o, d, near, far, seed=3, want=base + ["coarse_rgb"]).items()}
        p2 = eng.sigma_only_points()
    assert p1 - p0 == (0 if case == "no_viewdirs" else R * nc), (case, p1 - p0)
    assert p2 == p1
    for k in base:
        assert torch.equal(sig[k], full[k]), (case, prec, k, float((sig[k] - full[k]).abs().max()))
    assert float(full["coarse_acc"].max()) > 0.0 and float(full["acc"].max()) > 0.0
