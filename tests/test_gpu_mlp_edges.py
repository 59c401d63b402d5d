"""The fused MLP forward, the network backward and the weight-gradient GEMM against the float64 references of
tests/_mlp_ref.py, at tile, round and precision edges.

Sizes come from the device: one round of the persistent forward kernel is 2 * SMs * 64 points (two workers per CTA, one
64-point tile each).  Besides the ragged tails around a tile (M = 1 .. 129, 4097), one size makes every worker walk at
least three rounds, so that ring slots shift across tiles whenever the block count is not a multiple of the stage count,
and one leaves an odd number of tiles in the last round (a ghost iteration of the second warpgroup after full rounds).
For those two sizes only a subset of rows is checked (the forward) or carries a gradient (the backward): the first and
last row of every tile, every row of the last round, and every row of the eight tiles before it.

Forward (`point_mlp`): |kernel - emulation| <= tau * A per output, A = |X| |W|^T + |b| of the producing head (a quarter of
it for the sigmoid outputs), against `emulate_forward` of the same precision and act_scale_log2, full and sigma-only;
with a block of far-out-of-domain points at s = 0 whose saturated outputs must match the saturating emulation.  Fast mode
must also sit >= 2.5x further from the float64 truth than from its own emulation (measured 3.5x - 6x: an activation that
lies within the kernel's fp32 accumulation error of an fp16 rounding boundary rounds its single hi half differently from
the emulation, by 2^-11 of it, so the fast kernel cannot be pinned to its emulation more tightly than that).  tau: _mlp_ref.TAU_FWD_EXACT / _FAST.

Backward (`debug_mlp_backward`, dout random normal with the rows of gate-unsafe points zeroed, see _mlp_ref.filter_dout):
every state-dict tensor within tau_b * s of `mlp_backward_ref`, s the random-walk scale.  Exact tensor cores and the fp32
path against the float64 truth (gate margin MU_EXACT); fast mode on the two 128-wide nets against the backward at the
fast emulation's activations (margin MU_FAST), at least 30x worse than exact mode.  At least half the points must survive
the margin filter (fast mode: 2 %, its gates being only as reproducible as its rounding-boundary flips).  Exact mode is
also held to REL_L2_EXACT relative L2 per tensor.  A second call accumulates (2x), nm_zero_grad clears.

GEMM (`debug_gemm`): bf16x3 within TAU_GEMM * s of the float64 product at K < 64, N = 15 / 27, ragged K splits, N > 128
with a partial second B block, M = N = 1 at long K and a D offset by one float (the scalar-atomic epilogue).

The tolerances are >= 4x the worst ratio measured on an H100 and below the smallest synthetic fault that
tests/test_mlp_reference.py shows they flag.
"""
import numpy as np
import pytest
import torch

import _mlp_ref as R
from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu

PREC = dict(exact=0, fast=1, fp32=2)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _round():
    return 2 * _sms() * 64


def _sizes():
    V = 2 * _sms()
    return [1, 63, 64, 65, 127, 128, 129, 4097,
            3 * V * 64 + 7 * 64 + 13,          # every worker walks >= 3 rounds, ragged last tile
            2 * V * 64 + 21 * 64 - 5]          # 21 tiles in the last round: a ghost iteration after two full rounds


def _rows(M):
    """rows of an M-point launch that are checked: all of them up to 4097, else a subset (module docstring)."""
    if M <= 4097:
        return np.arange(M)
    V = 2 * _sms()
    n_tiles = (M + 63) // 64
    last_round = (n_tiles - 1) // V * V
    first = max(0, last_round - 8)
    edges = np.concatenate([np.arange(0, M, 64), np.minimum(np.arange(63, M + 63, 64), M - 1)])
    return np.unique(np.concatenate([edges, np.arange(first * 64, M)]))


def _points(M, seed):
    g = torch.Generator().manual_seed(seed)
    pts = (torch.rand(M, 3, generator=g) * 2 - 1) * 2.5
    dirs = torch.randn(M, 3, generator=g)
    return pts, dirs


def _engine(cfg, prec, s=0):
    import nerfmeshes_b200 as nm
    return nm.Engine(cfg.__dict__, None, nm.RenderSettings(num_coarse=8, num_fine=0, precision=PREC[prec], act_scale_log2=s))


def _report(test, key, value):
    print(f"RATIO {test} {key} {value:.3e}")


# ----------------------------------------------------------------------------------------------------- forward
@pytest.mark.parametrize("net", list(R.NETS))
def test_point_mlp_matches_emulation(net):
    cfg = R.net_cfg(net)
    sd = O.init_weights(cfg, 11)
    sizes = _sizes()
    pool_p, pool_d = _points(max(sizes), 5)
    rows = {M: _rows(M) for M in sizes}
    U = np.unique(np.concatenate(list(rows.values())))
    pos = np.full(max(sizes), -1)
    pos[U] = np.arange(U.size)
    far_p = (pool_p[:256] * 1.2e5)
    far_d = pool_d[:256]
    truth = R.truth_forward(cfg, sd, pool_p[U], pool_d[U])
    eng = _engine(cfg, "exact")
    eng.load_weights(0, sd)
    worst = {}
    for prec in ("exact", "fast"):
        for s in (0, 3):
            emul = R.emulate_forward(cfg, sd, pool_p[U], pool_d[U], fast=prec == "fast", act_scale_log2=s)
            tau = R.TAU_FWD_EXACT if prec == "exact" else R.TAU_FWD_FAST
            eng.configure(precision=PREC[prec], act_scale_log2=s)
            r_emul = r_truth = 0.0
            for M in sizes:
                ix = pos[rows[M]]
                out = eng.point_mlp(0, pool_p[:M].cuda(), pool_d[:M].cuda()).cpu().double().numpy()[rows[M]]
                sg = eng.point_mlp(0, pool_p[:M].cuda(), pool_d[:M].cuda(), sigma_only=True).cpu().double().numpy()[rows[M]]
                r = max(R.forward_ratio(out, emul.out[ix], emul.A_out[ix]),
                        R.forward_ratio(sg, emul.out[ix, 3], emul.A_out[ix, 3]))
                assert np.isfinite(out).all() and r <= tau, (net, prec, s, M, r)
                r_emul = max(r_emul, r)
                r_truth = max(r_truth, R.forward_ratio(out, truth.out[ix], emul.A_out[ix]))
            worst[(prec, s)] = r_emul
            _report("forward", f"{net} {prec} s={s}", r_emul)
            if prec == "fast":
                assert r_truth >= 2.5 * r_emul, (net, s, r_truth, r_emul)  # the emulation models the kernel, not the truth
                _report("forward-fast-vs-truth", f"{net} s={s}", r_truth)
    # far outside the domain at s = 0: operands saturate (satfinite) and the kernel must saturate exactly like the emulation
    for prec in ("exact", "fast"):
        eng.configure(precision=PREC[prec], act_scale_log2=0)
        emul = R.emulate_forward(cfg, sd, far_p, far_d, fast=prec == "fast")
        out = eng.point_mlp(0, far_p.cuda(), far_d.cuda()).cpu().double().numpy()
        r = R.forward_ratio(out, emul.out, emul.A_out)
        _report("forward-saturated", f"{net} {prec}", r)
        assert r <= (R.TAU_FWD_EXACT if prec == "exact" else R.TAU_FWD_FAST), (net, prec, r)
    eng.close()


# ----------------------------------------------------------------------------------------------------- backward
def _grads(eng, cfg, sd):
    return {k: eng.get_grad(0, k, torch.as_tensor(v)).cpu().double().numpy() for k, v in sd.items()}


def _backward_case(net, prec, sizes, seed):
    cfg = R.net_cfg(net)
    sd = O.init_weights(cfg, seed)
    eng = _engine(cfg, prec)
    eng.load_weights(0, sd)
    pool_p, pool_d = _points(max(sizes), seed + 1)
    rng = np.random.default_rng(seed)
    worst = {}
    for M in sizes:
        rows = _rows(M)
        p, d = pool_p[rows], pool_d[rows]
        if prec == "fast":
            rec = R.emulate_forward(cfg, sd, p, d, fast=True)
            mu, tau = R.MU_FAST, R.TAU_BWD_FAST
        else:
            rec = R.truth_forward(cfg, sd, p, d)
            mu, tau = R.MU_EXACT, (R.TAU_BWD_EXACT if prec == "exact" else R.TAU_BWD_FP32)
        # float32 values: the kernel reads what the reference gets
        dout_rows, keep = R.filter_dout(rng.standard_normal((rows.size, 4)).astype(np.float32), rec, mu)
        # fast mode's gates are only as reproducible as its rounding-boundary flips: few points survive its margin
        assert keep.mean() >= (0.02 if prec == "fast" else 0.5) or M == 1, (net, M, keep.mean())
        dout = np.zeros((M, 4))
        dout[rows] = dout_rows
        eng.zero_grad()
        eng.debug_mlp_backward(0, pool_p[:M].cuda(), pool_d[:M].cuda() if cfg.use_viewdirs else None,
                               torch.as_tensor(dout, dtype=torch.float32).cuda())
        got = _grads(eng, cfg, sd)
        ref, scale = R.mlp_backward_ref(rec, dout_rows)
        ratios = R.grad_ratio(got, ref, scale)
        worst[M] = max(ratios.values())
        bad = {k: v for k, v in ratios.items() if not v <= tau}
        assert not bad, (net, prec, M, bad)
        if prec == "exact" and M > 1:
            l2 = {k: float(np.linalg.norm(got[k] - ref[k]) / max(np.linalg.norm(ref[k]), 1e-300)) for k in ref}
            _report("backward-exact-relL2", f"{net} M={M}", max(l2.values()))
            assert max(l2.values()) <= R.REL_L2_EXACT, (net, M, sorted(l2.items(), key=lambda kv: -kv[1])[:3])
    return eng, cfg, sd, worst


@pytest.mark.parametrize("prec", ["exact", "fp32"])
@pytest.mark.parametrize("net", list(R.NETS))
def test_backward_matches_float64(net, prec):
    V = 2 * _sms()
    sizes = [1, 127, 129, 4097, 3 * V * 64 + 7 * 64 + 13]
    eng, cfg, sd, worst = _backward_case(net, prec, sizes, 21)
    for M, r in worst.items():
        _report(f"backward-{prec}", f"{net} M={M}", r)
    eng.close()


@pytest.mark.parametrize("net", ["tiny", "ldir2"])
def test_backward_fast_mode_matches_its_emulation(net):
    """NM_PREC_FAST's backward (one MMA pass everywhere) against the backward at the fast forward's activations: pinned to
    tau_fast, and at least 30x further off than exact mode on the same inputs — its lo passes really contribute."""
    V = 2 * _sms()
    sizes = [4097, 3 * V * 64 + 7 * 64 + 13]
    eng, _, _, fast = _backward_case(net, "fast", sizes, 33)
    eng.close()
    eng, _, _, exact = _backward_case(net, "exact", sizes, 33)
    eng.close()
    for M in sizes:
        _report("backward-fast", f"{net} M={M}", fast[M])
        assert fast[M] >= 30 * exact[M], (net, M, fast[M], exact[M])


def test_backward_accumulates_and_zero_grad_clears():
    cfg = R.net_cfg("nerf256")
    sd = O.init_weights(cfg, 41)
    eng = _engine(cfg, "exact")
    eng.load_weights(0, sd)
    p, d = _points(4097, 42)
    dout = torch.randn(4097, 4, generator=torch.Generator().manual_seed(43))
    eng.zero_grad()
    eng.debug_mlp_backward(0, p.cuda(), d.cuda(), dout.cuda())
    once = _grads(eng, cfg, sd)
    eng.debug_mlp_backward(0, p.cuda(), d.cuda(), dout.cuda())
    twice = _grads(eng, cfg, sd)
    worst = 0.0
    for k in once:
        sc = np.abs(once[k]).max()
        worst = max(worst, np.abs(twice[k] - 2 * once[k]).max() / max(sc, 1e-30))
    _report("accumulate", "nerf256", worst)
    assert worst <= 1e-4, worst                               # fp32 atomic-order noise only
    eng.zero_grad()
    assert all(not np.any(v) for v in _grads(eng, cfg, sd).values())
    eng.close()


# ----------------------------------------------------------------------------------------------------- weight-gradient GEMM
GEMM_SHAPES = [
    (128, 15, 64), (128, 27, 1), (256, 63, 63),                      # K < 64 and the direction-encoding widths
    (256, 256, 511), (256, 256, 512), (256, 256, 513),               # around the 8-blocks-per-split limit
    (128, 128, 64 * 29 - 7),                                         # 4 splits per tile, the last one ragged
    (256, 255, 3000), (200, 300, 2000), (1, 1, 70001),               # partial B blocks, N > 128, long K
]


GEMM_CASES = [(s, 0) for s in GEMM_SHAPES] + [((256, 256, 511), 1), ((200, 300, 2000), 1), ((128, 27, 1), 1)]


@pytest.mark.parametrize("shape,offset", GEMM_CASES, ids=[f"{m}x{n}x{k}-off{o}" for (m, n, k), o in GEMM_CASES])
def test_gemm_edges(shape, offset):
    """D += a^T b through nm_debug_gemm against float64; offset 1 puts D one float past a 16-byte boundary, which forces
    the scalar-atomic epilogue."""
    import nerfmeshes_b200 as nm
    M, N, K = shape
    eng = nm.Engine(O.NetCfg().__dict__, None, nm.RenderSettings())
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(K, M, generator=g) * torch.logspace(-2, 1, K)[:, None]
    b = torch.randn(K, N, generator=g)
    ref = a.double().T @ b.double()
    scale = ((a.double() ** 2).T @ (b.double() ** 2)).sqrt()
    buf = torch.zeros(M * N + 4, dtype=torch.float32, device="cuda")
    d = buf[offset:offset + M * N].view(M, N)
    eng.debug_gemm(a.cuda(), b.cuda(), n_passes=3, out=d)
    r = R.forward_ratio(d.cpu().double().numpy(), ref.numpy(), scale.numpy())
    assert float(buf[:offset].abs().sum()) == 0.0 and float(buf[offset + M * N:].abs().sum()) == 0.0
    _report("gemm", f"{M}x{N}x{K} off={offset}", r)
    assert r <= R.TAU_GEMM, (shape, offset, r)
    eng.close()
