"""CPU checks of the density-gradient reference (tests/_sigma_grad_ref.py) and of the mesh path's coordinate mapping:

* the hand-written float64 gradient equals central finite differences of truth_forward (float64 encodings) for every
  network of _mlp_ref.NETS, away from relu gates;
* the GPU tolerances of tests/test_gpu_sigma_grad.py flag synthetic faults: the skip layers' PE contribution dropped, the
  include_input block dropped, the cos-derivative's sign flipped, one band's factor doubled (against the exact and fp32
  tolerances; the last two also against fast mode's on the nets it is tested on), and one hi/lo pass of the tensor-core tail's emulation dropped (against the exact-mode
  tolerance, which the emulation with all three passes meets);
* mesh.sweep_coordinates reproduces torch.linspace bit for bit at integer indices and interpolates between them.
"""
import numpy as np
import pytest
import torch

import _mlp_ref as R
import _sigma_grad_ref as SG
from oracle import nerf_oracle as O

from nerfmeshes_b200.mesh import sweep_coordinates


def _pts(M, seed, lim=1.5):
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(M, 3, generator=g, dtype=torch.float64) * 2 - 1) * lim).numpy()


@pytest.mark.parametrize("net", list(R.NETS))
def test_reference_matches_finite_differences(net):
    cfg = R.net_cfg(net)
    sd = O.init_weights(cfg, 7)
    p = _pts(128, 3)
    g, S, _, rec = SG.sigma_grad_ref(cfg, sd, p, enc_dtype=torch.float64)
    fd, same = SG.fd_sigma_grad(cfg, sd, p)
    assert same.sum() >= 32, same.sum()             # points whose relu gates do not change within the stencil
    err = np.abs(fd - g)[same]
    assert (err <= 1e-9 * S[same]).all(), float((err / S[same]).max())


def _fault_ratio(cfg, sd, p, mu, **fault):
    g, S, _, rec = SG.sigma_grad_ref(cfg, sd, p)
    keep = R.gate_margin(rec) >= mu
    gf, _, _, _ = SG.sigma_grad_ref(cfg, sd, p, rec=rec, **fault)
    return R.forward_ratio(gf[keep], g[keep], S[keep])


FAULTS = [dict(drop_skip=True), dict(drop_identity=True), dict(flip_cos=True), dict(double_band=3)]
# what fast mode's looser tolerance still flags on the nets it is tested on (a dropped identity block moves g by ~1e-3 S
# there, too close to TAU_FAST to claim)
FAST_FLAGGED = ("flip_cos", "double_band")


@pytest.mark.parametrize("fault", FAULTS, ids=[next(iter(f)) for f in FAULTS])
@pytest.mark.parametrize("net", list(R.NETS))
def test_tolerances_flag_structural_faults(net, fault):
    cfg = R.net_cfg(net)
    if "drop_skip" in fault and not cfg.skip_layers():
        pytest.skip("no skip layer")
    sd = O.init_weights(cfg, 9)
    p = _pts(256, 4)
    r = _fault_ratio(cfg, sd, p, R.MU_EXACT, **fault)
    assert r > 4 * SG.TAU_EXACT and r > 4 * SG.TAU_FP32, (net, fault, r)
    if net in SG.FAST_NETS and next(iter(fault)) in FAST_FLAGGED:
        r = _fault_ratio(cfg, sd, p, R.MU_FAST, **fault)
        assert r > 2 * SG.TAU_FAST, (net, fault, r)


@pytest.mark.parametrize("net", list(R.NETS))
def test_exact_tolerance_flags_a_dropped_pass(net):
    cfg = R.net_cfg(net)
    sd = O.init_weights(cfg, 9)
    p = _pts(512, 5)
    g, S, _, rec = SG.sigma_grad_ref(cfg, sd, p)
    keep = R.gate_margin(rec) >= R.MU_EXACT
    full, _, _, _ = SG.sigma_grad_ref(cfg, sd, p, rec=rec, drop_pass="none")
    assert R.forward_ratio(full[keep], g[keep], S[keep]) <= SG.TAU_EXACT / 4
    for drop in ("lh", "hl"):
        gf, _, _, _ = SG.sigma_grad_ref(cfg, sd, p, rec=rec, drop_pass=drop)
        r = R.forward_ratio(gf[keep], g[keep], S[keep])
        assert r > SG.TAU_EXACT, (net, drop, r)


@pytest.mark.parametrize("n", [2, 3, 64, 65, 128, 257, 512])
def test_sweep_coordinates_hit_linspace(n):
    lim = 1.2
    lins = [torch.linspace(-lim, lim, n) for _ in range(3)]
    idx = torch.arange(n, dtype=torch.float32)
    v = torch.stack([idx, idx.flip(0), idx.roll(1)], 1)
    x = sweep_coordinates(v, lins)
    assert torch.equal(x[:, 0], lins[0]) and torch.equal(x[:, 1], lins[1].flip(0)) and torch.equal(x[:, 2], lins[2].roll(1))
    # between grid points: the linear interpolation of the tables (float32 arithmetic)
    g = torch.Generator().manual_seed(n)
    vf = torch.rand(1000, 3, generator=g) * (n - 1)
    xf = sweep_coordinates(vf, lins).double().numpy()
    ref = SG.sweep_coordinates_ref(vf.numpy(), [t.numpy() for t in lins])
    assert np.abs(xf - ref).max() <= 4 * np.finfo(np.float32).eps * lim
