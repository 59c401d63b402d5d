"""The references of the training compositor adjoint (tests/_composite_ref.py) on the CPU: the fp32 emulation of
composite_backward_kernel stays within TAU * error_scale of the float64 truth over the edge matrix of
tests/test_gpu_composite_adjoint.py, every fault variant of the emulation exceeds it there, and the ray kinds really
reach the edges they are named after."""
import numpy as np
import pytest

import _composite_ref as CR

# every segment length 1..16, with full, partly filled and empty last lanes (shared with the GPU test)
S_EDGES = [1, 2, 31, 32, 33, 63, 64, 65, 192, 255, 256, 257, 481, 511, 512]
S_EXTRA = [32 * k + 1 for k in range(1, 16) if not any(-(-s // 32) == k + 1 for s in S_EDGES)]
S_ALL = S_EDGES + S_EXTRA
NOISE = [(0.0, 0), (0.7, 0x2545F4914F6CDD1D ^ CR.SALT_MAIN), (0.7, 977 ^ CR.SALT_COARSE)]   # (std, salted seed)


def test_matrix_covers_every_segment_length():
    layout = []                                       # (segment length, lanes holding samples, samples in the last one)
    for s in S_ALL:
        seg = -(-s // 32)
        lanes = -(-s // seg)
        layout.append((seg, lanes, s - (lanes - 1) * seg))
    assert sorted({seg for seg, _, _ in layout}) == list(range(1, 17))
    assert any(lanes == 32 and last == seg for seg, lanes, last in layout)          # every lane full
    assert any(1 < seg and last < seg for seg, lanes, last in layout)               # a partly filled last lane
    assert any(lanes < 32 for seg, lanes, last in layout)                           # empty lanes at the end


def _cases(R=21):
    for S in S_ALL:
        for white in (0, 1):
            for std, seed in NOISE:
                yield S, white, std, seed, CR.make_rays(R, S, 1000 * S + 10 * white + int(std > 0), kind_offset=S)


def test_emulation_within_tau_of_truth():
    worst = 0.0
    for S, white, std, seed, (raw, t, d, g, _) in _cases():
        a = CR.composite_adjoint(raw, t, d, g, white, std, seed)
        r = CR.ratio(CR.emulate_kernel(raw, t, d, g, white, std, seed), a.dout(), CR.error_scale(a, S))
        assert r.max() <= CR.EMUL_WORST, (S, white, std, float(r.max()))
        worst = max(worst, float(r.max()))
    print(f"RATIO emulation-vs-truth {worst:.3e}")
    assert CR.EMUL_WORST <= CR.TAU


def test_every_fault_is_flagged_at_tau():
    worst = {f: 0.0 for f in CR.FAULTS}
    for S, white, std, seed, (raw, t, d, g, _) in _cases(R=7):
        a = CR.composite_adjoint(raw, t, d, g, white, std, seed)
        ref, sc = a.dout(), CR.error_scale(a, S)
        for f in CR.FAULTS:
            if worst[f] <= 100 * CR.TAU:
                worst[f] = max(worst[f], float(CR.ratio(CR.emulate_kernel(raw, t, d, g, white, std, seed, fault=f), ref, sc).max()))
    for f, v in worst.items():
        print(f"RATIO fault {f} {v:.3e}")
    missed = {f: v for f, v in worst.items() if not v > 100 * CR.TAU}
    assert not missed, missed


@pytest.mark.parametrize("S", [64, 257])
def test_ray_kinds_reach_their_edges(S):
    raw, t, d, g, kinds = CR.make_rays(7, S, 5, kind_offset=0)
    a = CR.composite_adjoint(raw, t, d, g, 0)
    em = CR.emulate_kernel(raw, t, d, g, 0)
    k = {name: i for i, name in enumerate(CR.KINDS)}
    assert (raw[k["nonpositive"], :, 3] <= 0).all() and (raw[k["nonpositive"], ::3, 3] == 0).all()
    assert a.x[k["saturate_first"], 0] >= 110 and em[k["saturate_first"], 0, 3] == 0
    T32 = np.cumprod(np.concatenate([[1.0], a.keep[k["subnormal_T"], :-1]])).astype(np.float32)
    assert ((T32 > 0) & (T32 < np.finfo(np.float32).tiny)).any() and (T32 == 0).any()     # subnormal, then 0
    band = a.e[k["band"]]
    assert ((band > 2.0 ** -25) & (band < 2.0 ** -10)).sum() >= S // 4
    assert 1e8 < abs(a.dsig[k["tiny_last"], -1]) < 1e30 and np.isfinite(em[k["tiny_last"], -1, 3])
    assert (a.dist[k["duplicate_t"], :-1] == 0).any()
    assert (a.dsig[k["nonpositive"]] == 0).all() and (em[k["nonpositive"], :, 3] == 0).all()


def test_noise_emulation_follows_the_device_stream_layout():
    """sample i of ray r reads randn(seed, r*S + i), i.e. draws (2 idx, 2 idx + 1); the clamp keeps a > 0."""
    n = CR.sigma_noise(123, 3, 5, 1.0)
    idx = np.arange(15, dtype=np.uint64)
    assert np.array_equal(n.reshape(-1), CR.randn(123, idx).astype(np.float32))
    big = CR.randn(7, np.arange(1 << 16, dtype=np.uint64))
    assert np.isfinite(big).all() and abs(big.mean()) < 0.02 and abs(big.std() - 1) < 0.02
