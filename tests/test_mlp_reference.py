"""CPU checks of the float64 references in tests/_mlp_ref.py (no GPU needed).

* The fp16 operand split follows numpy float16 semantics: round-to-nearest-even ties, subnormal hi / lo halves, and
  `satfinite` clamping at 65504 where plain conversion overflows.
* The exact-mode emulation of mlp_tc_kernel stays within 2^-19 * A of the float64 truth; the fast-mode emulation is
  further away by the expected fp16 amount (well above 2^-19 * A, below 2^-9 * A).
* The hand-written float64 backward equals torch autograd in float64 on the oracle's own network to 1e-12 relative.
* Sensitivity: the comparators the GPU tests use, at their committed tolerances (_mlp_ref.TAU_*), flag each of these
  synthetic faults applied to the reference: one 64-point K block missing from a weight gradient or from a bias
  gradient, one tensor's gradient scaled by 1 + 3e-3, the rows of the last 128-row tile counted twice, one layer's
  a_hi*b_lo pass missing from the weight-gradient GEMM, and (forward, fast mode) one K-step of one weight block missing.
  So a kernel with one of these bugs cannot pass the GPU tests, without any kernel having to be mutated.
* The entrywise bound tau * s of the tensor-core backward allows less relative L2 error than the 6e-3 of the ray-level
  tests (tests/test_gpu_train.py); the GPU test also holds every tensor to 3e-4 relative L2, 20x below it.
"""
import numpy as np
import pytest
import torch

import _mlp_ref as R
from oracle import nerf_oracle as O


def _inputs(M, seed, far=False):
    g = torch.Generator().manual_seed(seed)
    pts = (torch.rand(M, 3, generator=g) * 2 - 1) * 2.5
    dirs = torch.randn(M, 3, generator=g)
    return pts, dirs


# ----------------------------------------------------------------------------------------------------- number formats
def test_f16_split_matches_numpy_float16():
    x = np.array([1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, -(1.0 + 2.0 ** -11), 2049.0, 2051.0], np.float32)
    assert R.f16_sat(x).tolist() == [1.0, 1.0 + 2.0 ** -9, -1.0, 2048.0, 2052.0]         # ties to even
    assert R.f16_sat(x).tolist() == x.astype(np.float16).astype(np.float64).tolist()
    # subnormal hi (below 2^-14) and subnormal lo: spacing 2^-24
    tiny = np.array([3.3e-6, 1e-4 + 1.3e-8, -7.7e-7], np.float32)
    hi, lo = R.f16_split_sat(tiny)
    assert np.all(np.abs(hi) < 2.0 ** -14 + 2.0 ** -14 * (np.abs(tiny) > 2.0 ** -14))
    assert hi.tolist() == tiny.astype(np.float16).astype(np.float64).tolist()
    assert np.all(np.abs(hi + lo - tiny) <= 2.0 ** -25)
    assert np.all((lo / 2.0 ** -24) == np.round(lo / 2.0 ** -24))                        # lo on the subnormal grid
    # saturation: 65504 is exact, 65519 rounds to it, beyond 65520 plain conversion overflows and satfinite clamps;
    # the lo half then carries the excess (itself saturating)
    big = np.array([65504.0, 65519.0, 65520.0, 1e5, -3e5, 1e9], np.float32)
    hi, lo = R.f16_split_sat(big)
    with np.errstate(over="ignore"):
        assert np.isinf(big[2:].astype(np.float16)).all()
    assert hi.tolist() == [65504.0, 65504.0, 65504.0, 65504.0, -65504.0, 65504.0]
    assert lo.tolist() == [0.0, 15.0, 16.0, 34496.0, -65504.0, 65504.0]
    assert R.f16_sat(np.float32(np.inf)) == 65504.0
    # bf16 (the backward's halves): ties to even
    assert R.bf16_rn(np.array([1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8], np.float32)).tolist() == [1.0, 1.0 + 2.0 ** -6]


# ----------------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize("net", list(R.NETS))
def test_emulation_against_truth(net):
    cfg = R.net_cfg(net)
    sd = O.init_weights(cfg, 3)
    pts, dirs = _inputs(1000, 4)
    truth = R.truth_forward(cfg, sd, pts, dirs)
    ref = O.flexible_nerf_forward(sd, cfg, pts, dirs).numpy()                 # the fp32 oracle: same network
    assert np.abs(truth.out - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max())
    exact = R.emulate_forward(cfg, sd, pts, dirs)
    fast = R.emulate_forward(cfg, sd, pts, dirs, fast=True)
    r_exact = R.forward_ratio(exact.logits, truth.logits, truth.A_logits)
    r_fast = R.forward_ratio(fast.logits, truth.logits, truth.A_logits)
    assert r_exact <= R.EMUL_EXACT_VS_TRUTH, r_exact
    assert 2.0 ** -19 < r_fast < 2.0 ** -9, r_fast
    # act_scale_log2 = 3 is exact scaling in range: same class of agreement
    r3 = R.forward_ratio(R.emulate_forward(cfg, sd, pts, dirs, act_scale_log2=3).logits, truth.logits, truth.A_logits)
    assert r3 <= R.EMUL_EXACT_VS_TRUTH, r3


def test_emulation_models_saturation():
    """Points far outside the domain: the saturating emulation departs from the truth (so a GPU test against it pins the
    kernel's satfinite behaviour), and shifting the range with act_scale_log2 brings it back."""
    cfg = R.net_cfg("tiny")
    sd = O.init_weights(cfg, 3)
    pts, dirs = _inputs(256, 5)
    pts = pts * 1.2e5
    truth = R.truth_forward(cfg, sd, pts, dirs)
    sat = R.emulate_forward(cfg, sd, pts, dirs)
    assert R.forward_ratio(sat.logits, truth.logits, truth.A_logits) > 1e-2
    wide = R.emulate_forward(cfg, sd, pts, dirs, act_scale_log2=3)
    assert R.forward_ratio(wide.logits, truth.logits, truth.A_logits) <= R.EMUL_EXACT_VS_TRUTH


# ----------------------------------------------------------------------------------------------------- backward
def _autograd(cfg, sd, pts, dirs, dout, monkeypatch):
    leafs = {k: torch.as_tensor(v).double().requires_grad_(True) for k, v in sd.items()}
    monkeypatch.setattr(torch, "sigmoid", lambda x: x)           # the oracle's network, rgb logits out
    out = O.flexible_nerf_forward(leafs, cfg, pts.double(), dirs.double())
    monkeypatch.undo()
    (out * torch.as_tensor(dout)).sum().backward()
    return {k: v.grad.numpy() for k, v in leafs.items()}


@pytest.mark.parametrize("net", list(R.NETS))
def test_manual_backward_equals_autograd(net, monkeypatch):
    cfg = R.net_cfg(net)
    sd = O.init_weights(cfg, 7)
    pts, dirs = _inputs(300, 8)
    dout = np.random.default_rng(9).standard_normal((300, 4))
    rec = R.truth_forward(cfg, sd, pts, dirs, enc_dtype=torch.float64)      # autograd's float64 encodings
    ref = _autograd(cfg, sd, pts, dirs, dout, monkeypatch)
    got, scale = R.mlp_backward_ref(rec, dout)
    assert set(got) == set(ref) == set(scale)
    for k in ref:
        e = np.abs(got[k] - ref[k]).max() / max(np.abs(ref[k]).max(), 1e-300)
        assert e <= 1e-12, (k, e)
        # the random-walk scale bounds each term: s >= |sum| / sqrt(number of points)
        assert scale[k].shape == ref[k].shape and np.all(scale[k] * np.sqrt(300) * (1 + 1e-12) >= np.abs(got[k]))


# ----------------------------------------------------------------------------------------------------- sensitivity
TAU_B = max(R.TAU_BWD_EXACT, R.TAU_BWD_FP32)        # the looser of the two comparators that pin gradients to truth


@pytest.fixture(scope="module")
def case():
    """nerf256 at M = 4097 (the GPU tests' size), gate-unsafe points filtered as on the GPU."""
    cfg = R.net_cfg("nerf256")
    sd = O.init_weights(cfg, 21)
    pts, dirs = _inputs(4097, 22)
    rec = R.truth_forward(cfg, sd, pts, dirs)
    dout, keep = R.filter_dout(np.random.default_rng(23).standard_normal((4097, 4)).astype(np.float32), rec, R.MU_EXACT)
    assert keep.mean() >= 0.5
    dz = {}
    ref, scale = R.mlp_backward_ref(rec, dout, dz)
    return dict(cfg=cfg, rec=rec, dout=dout, ref=ref, scale=scale, dz=dz)


def _part(case, lo, hi):
    """gradients of the points [lo, hi) alone (the gradient is linear in dout's rows)"""
    d = np.zeros_like(case["dout"])
    d[lo:hi] = case["dout"][lo:hi]
    return R.mlp_backward_ref(case["rec"], d)[0]


def _flags(case, fault):
    return R.grad_ratio(fault, case["ref"], case["scale"])


def _linear_names(case):
    return [L.name for L in R.layer_list(case["cfg"])]


def test_flags_a_missing_k_block(case):
    """one 64-point K block of the weight-gradient GEMM lost, in each layer's weight and bias gradient"""
    block = _part(case, 640, 704)
    for name in _linear_names(case):
        for t in (".weight", ".bias"):
            fault = dict(case["ref"])
            fault[name + t] = case["ref"][name + t] - block[name + t]
            r = _flags(case, fault)[name + t]
            assert r > TAU_B, (name + t, r)


def test_flags_one_tensor_scaled(case):
    """any single tensor's gradient scaled by 1 + 3e-3.  (1 + 1e-3 moves the least sensitive tensor, a bias gradient, by
    3.5e-4 of its scale, below TAU_BWD_EXACT = 4e-4, which the tensor-core backward's measured 9.9e-5 sets.)"""
    for k, v in case["ref"].items():
        r = _flags(case, {**case["ref"], k: v * (1 + 3e-3)})[k]
        assert r > TAU_B, (k, r)


def test_flags_a_tile_counted_twice(case):
    """the rows of one 128-row tile (the last full one below M) added a second time"""
    tile = _part(case, 3968, 4096)
    fault = {k: case["ref"][k] + tile[k] for k in case["ref"]}
    assert max(_flags(case, fault).values()) > TAU_B


def test_flags_a_missing_hi_lo_pass(case):
    """the weight-gradient GEMM of one layer without its a_hi * b_lo pass: dZ^T times the bf16 hi half of X only"""
    rec = case["rec"]
    for li, name in enumerate(_linear_names(case)):
        fault = dict(case["ref"])
        fault[name + ".weight"] = case["dz"][name].T @ R.bf16_rn(rec.X[li])
        r = _flags(case, fault)[name + ".weight"]
        assert r > TAU_B, (name, r)


def test_flags_a_missing_fast_k_step():
    """forward, NM_PREC_FAST: one K-step (16 columns) of one 64x64 weight block missing"""
    cfg = R.net_cfg("nerf256")
    sd = O.init_weights(cfg, 24)
    pts, dirs = _inputs(1000, 25)
    good = R.emulate_forward(cfg, sd, pts, dirs, fast=True)
    for name, rows, cols in (("layers_xyz.2", slice(64, 128), slice(144, 160)), ("layer1", slice(0, 64), slice(48, 63)),
                             ("layers_dir.0", slice(0, 64), slice(256, 272))):
        bad = {k: v.clone() for k, v in sd.items()}
        bad[name + ".weight"][rows, cols] = 0.0
        r = R.forward_ratio(R.emulate_forward(cfg, bad, pts, dirs, fast=True).out, good.out, good.A_out)
        assert r > R.TAU_FWD_FAST, (name, r)


def test_backward_bound_is_tighter_than_the_ray_level_tests(case):
    """The entrywise bound tau_b * s alone allows less relative L2 error per tensor than the ray-level tests' 6e-3; the
    GPU test adds REL_L2_EXACT = 3e-4 (20x below it) per tensor on top."""
    eff = R.effective_rel_l2(case["ref"], case["scale"], R.TAU_BWD_EXACT)
    assert max(eff.values()) <= 6e-3, sorted(eff.items(), key=lambda kv: -kv[1])[:4]
    assert R.REL_L2_EXACT <= 6e-3 / 20
