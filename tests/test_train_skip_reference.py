"""The training contract of empty-space skipping (NM_FLAG_SKIP_EMPTY_TRAIN, DESIGN 4.15) on the CPU, through the fp32
emulations of the compositor adjoint and forward kernels (tests/_composite_ref.py) over their edge matrices: replacing every
sample whose noisy pre-activation is <= 0 (or NaN) with the skipped raw (0,0,0,-inf) leaves the forward outputs in training
mode bit for bit, makes those samples' adjoint rows exactly zero in the dense step, and leaves every other row's adjoint
equal in value.  Replacing a sample whose pre-activation is > 0 changes the outputs: the condition is tight."""
import numpy as np
import pytest

import _composite_ref as CR

S_CASES = (1, 2, 31, 33, 64, 192, 257, 512)
NOISES = ((0.0, 0), (0.7, 0x2545F4914F6CDD1D ^ CR.SALT_MAIN), (0.7, 977 ^ CR.SALT_COARSE))
SKIPPED = np.array([0.0, 0.0, 0.0, -np.inf], np.float32)


def _skip(raw, std, seed):
    pre, _ = CR.noisy_pre(raw, std, seed)
    with np.errstate(invalid="ignore"):
        gone = ~(pre > 0)
    out = raw.copy()
    out[gone] = SKIPPED
    return out, gone, pre


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("S", S_CASES)
@pytest.mark.parametrize("white", (0, 1))
@pytest.mark.parametrize("noise", range(len(NOISES)))
def test_adjoint_rows_of_skipped_samples_are_zero_and_others_unchanged(S, white, noise):
    std, seed = NOISES[noise]
    raw, t, d, g, _ = CR.make_rays(35, S, 31 * S + noise, kind_offset=S + noise)
    skipped, gone, _ = _skip(raw, std, seed)
    dense = CR.emulate_kernel(raw, t, d, g, white, std, seed)
    skip = CR.emulate_kernel(skipped, t, d, g, white, std, seed)
    assert gone.any() and (~gone).any()
    assert (dense[gone] == 0).all(), "a dense adjoint row of a sample with pre-activation <= 0 is not zero"
    assert (skip[gone] == 0).all()
    kept_dense, kept_skip = dense[~gone], skip[~gone]
    assert ((kept_dense == kept_skip) | (np.isnan(kept_dense) & np.isnan(kept_skip))).all(), \
        "an evaluated sample's adjoint changed when the samples with pre-activation <= 0 were skipped"


@pytest.mark.parametrize("S", S_CASES)
@pytest.mark.parametrize("white", (0, 1))
@pytest.mark.parametrize("noise", range(len(NOISES)))
def test_training_forward_is_bit_identical_and_the_condition_is_tight(S, white, noise):
    std, seed = NOISES[noise]
    raw, t, d, _ = CR.make_forward_rays(42, S, 53 * S + noise, kind_offset=S + 2 * noise)
    skipped, gone, pre = _skip(raw, std, seed)
    dense = CR.emulate_forward(raw, t, d, white, 1, 1e-5, std, seed)
    skip = CR.emulate_forward(skipped, t, d, white, 1, 1e-5, std, seed)
    for k in CR.FWD_OUT:
        assert np.array_equal(_bits(dense[k]), _bits(skip[k])), k
    # tight: on every ray with a sample of pre-activation > 0 and positive weight, skipping its heaviest such sample too
    # changes an output of that ray
    w = np.where(gone, -1.0, np.nan_to_num(dense["weights"], nan=-1.0))
    heavy = np.argmax(w, 1)
    rays = np.nonzero(w[np.arange(len(w)), heavy] > 0)[0]
    assert len(rays) >= 5
    more = skipped.copy()
    more[rays, heavy[rays]] = SKIPPED
    assert (pre[rays, heavy[rays]] > 0).all()
    loose = CR.emulate_forward(more, t, d, white, 1, 1e-5, std, seed)
    changed = np.zeros(len(w), bool)
    for k in CR.FWD_OUT:
        a, b = _bits(dense[k]).reshape(len(w), -1), _bits(loose[k]).reshape(len(w), -1)
        changed |= (a != b).any(1)
    assert changed[rays].all(), "skipping a sample with pre-activation > 0 left its ray's outputs unchanged"
