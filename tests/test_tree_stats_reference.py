"""BuFF tree integration and the volume statistics restated against the CPU oracle and float64 truths (tests/_tree_stats_ref.py)
— no GPU.

* Exact case (weights k 2^-12, mask weights in {0, 1} or {0, 0.5, 1}): the fp32 restatement equals
  oracle.nerf_oracle.ray_batch_integration bit for bit, at counters 1, 2, 3 and 1000 and with out-of-range indices dropped.
* General case (uniform weights, BuFF's w > 0.1 mask or positive mask weights): restatement and oracle lie within the float64
  bound, and voxels with no mask weight keep their bits.
* The bound flags every fault: one dropped sample, counter + 1, acc and freq swapped.
* The statistics check accepts a double-accumulated two-pass std in another summation order, and rejects the one-pass
  E[x^2] - E[x]^2 on the 1e4 + 0.05 N(0, 1) volume the GPU suite uses.
"""
import numpy as np
import pytest

import _tree_stats_ref as TR

F32 = np.float32
CASES = [(1, 1), (257, 2), (4097, 6143), (20000, 6145), (50000, 40000), (300000, 6144), (300000, 3)]


def _bits_equal(a, b):
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _memm(V, seed):
    return np.random.default_rng(seed + 99).standard_normal(V).astype(F32)


@pytest.mark.parametrize("kind", ["exact", "exact_half", "one_voxel"])
def test_exact_case_restatement_equals_oracle_bit_for_bit(kind):
    for s, (n, V) in enumerate(CASES):
        idx, w, mw = TR.tree_inputs(n, V, kind, s)
        idx[:: 97] = V                                              # dropped: the kernel's contract, the reference would raise
        idx[5:: 101] = np.iinfo(np.int32).min
        for counter in (1, 2, 3, 1000):
            memm = _memm(V, s)
            got = TR.integrate32(memm, counter, idx, w, mw)
            ref = TR.integrate_oracle(memm, counter, idx, w, mw)
            assert _bits_equal(got, ref), (kind, n, V, counter, int((got != ref).sum()))
            assert TR.tree_violations(got, memm, counter, idx, w, mw) == 0


@pytest.mark.parametrize("kind", ["general", "general_mw", "mask_zero"])
def test_general_case_within_the_float64_bound(kind):
    for s, (n, V) in enumerate(CASES):
        idx, w, mw = TR.tree_inputs(n, V, kind, s)
        for counter in (1, 3, 1000):
            memm = _memm(V, s)
            for m in (TR.integrate32(memm, counter, idx, w, mw), TR.integrate_oracle(memm, counter, idx, w, mw)):
                assert TR.tree_violations(m, memm, counter, idx, w, mw) == 0, (kind, n, V, counter)
        if kind == "mask_zero" and n > V:
            _, _, upd = TR.integrate_truth(memm, 1, idx, w, mw)
            even = np.arange(V) % 2 == 0
            assert not upd[even].any() and upd[~even].any()


@pytest.mark.parametrize("fault", TR.TREE_FAULTS)
@pytest.mark.parametrize("kind", ["exact", "general"])
def test_bound_flags_every_fault(fault, kind):
    """In voxels of up to a few hundred samples; in a voxel of 10^5 samples one dropped sample moves the mean by less than
    the summation term of the bound (there the exact case's bitwise comparison still sees it)."""
    for s, (n, V) in enumerate([(257, 2), (20000, 6145), (300000, 6144)]):
        idx, w, mw = TR.tree_inputs(n, V, kind, s)
        for counter in (1, 3, 1000):
            memm = _memm(V, s)
            bad = TR.integrate32(memm, counter, idx, w, mw, fault=fault)
            assert TR.tree_violations(bad, memm, counter, idx, w, mw) > 0, (fault, kind, n, V, counter)


def test_stats_check_accepts_reordered_double_sums_and_rejects_one_pass():
    g = np.random.default_rng(3)
    for v in (g.standard_normal(100003).astype(F32), (1e4 + 0.05 * g.standard_normal(100003)).astype(F32),
              np.maximum(g.standard_normal(4099) * 30, 0).astype(F32), np.full(1000, 2.5, F32), np.array([7.0], F32)):
        x = v.astype(np.float64)
        n = x.size
        mean = np.cumsum(x[::-1])[-1] / n                             # sequential, reversed: another order than the truth's
        sd = np.sqrt(np.cumsum((x - mean) ** 2)[-1] / n)
        assert TR.stats_ok(v.min(), v.max(), sd, v)
    v = (1e4 + 0.05 * g.standard_normal(257 ** 2)).astype(F32)
    x = v.astype(np.float32)
    one_pass = np.sqrt(max(float(np.mean(x * x, dtype=np.float32) - np.mean(x, dtype=np.float32) ** 2), 0.0))
    assert not TR.stats_ok(v.min(), v.max(), one_pass, v)
    assert not TR.stats_ok(v.min(), v.max(), float(np.nextafter(F32(TR.stats_truth(v)[2]), F32(1), dtype=F32)) * (1 + 3e-7), v)
