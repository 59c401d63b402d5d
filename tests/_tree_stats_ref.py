"""References for BuFF tree integration (nm_render.cu tree_scatter_kernel / tree_update_kernel) and the volume statistics
(stats_pass1 / stats_pass2 behind nm_volume_stats and nm_volume_stats_dev) — test infrastructure, no GPU.

Tree integration.  The fp32 oracle is oracle.nerf_oracle.ray_batch_integration; `integrate_oracle` feeds it the samples the
kernel keeps (0 <= idx < V: the kernel drops every other index, where the reference would raise).  `integrate_truth` forms
acc A, freq F and the update m + (A / F - m) / counter in float64 from the same fp32 inputs, applied where F > 0, with the
per-voxel bound

    |m32 - m64| <= 4 u (|m_old| + |A / F|) + (c_v u) (S_w / F + |A| S_m / F^2) / counter,     u = 2^-24,

c_v the voxel's sample count, S_w = sum |w| and S_m = sum |mw| over it.  The second term is recursive summation in any
order (a block's shared-memory partial followed by a global atomic is still a summation tree of c_v terms) carried
through A / F; the first covers the division, the subtraction, the division by counter and the addition.  A voxel with
F == 0 keeps its bits.

Exact case.  Weights k 2^-12 with integer k < 4096 and mask weights in {0, 0.5, 1}, with every voxel's sum k below 2^24:
every partial sum is then exact in any order, so the device, `integrate32` and the oracle agree bit for bit.

`TREE_FAULTS` name variants that each carry one plausible bug; tests/test_tree_stats_reference.py shows that the bound
flags each.

Volume statistics.  The truth is the float64 min, max and population standard deviation of the fp32 values.  The kernel
sums doubles in another order; that error is at most about n 2^-53 relative, below an fp32 ulp even at 512^3, but it can
flip a rounding tie, so std must lie within one fp32 ulp of f32(std64) and min / max must be exact.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import nerf_oracle as O

F32 = np.float32
U = 2.0 ** -24
TREE_FAULTS = ("drop_sample", "counter_plus_one", "swap_acc_freq")
STATS_GRID = 1184 * 256                   # stats_pass1 / stats_pass2: 1184 blocks x 256 threads, grid-stride


def kept(idx, V):
    idx = np.asarray(idx)
    return (idx >= 0) & (idx < V)


def integrate_oracle(memm, counter, idx, w, mw):
    """oracle ray_batch_integration on the samples the kernel keeps; memm (V,) fp32 -> new memm (V,) fp32."""
    memm = np.asarray(memm, F32)
    k = kept(idx, memm.shape[0])
    out, _ = O.ray_batch_integration(torch.from_numpy(memm.copy()), int(counter),
                                     torch.from_numpy(np.asarray(idx)[k].astype(np.int64)),
                                     torch.from_numpy(np.asarray(w, F32)[k]), torch.from_numpy(np.asarray(mw, F32)[k]))
    return out.numpy()


def integrate32(memm, counter, idx, w, mw, fault=None):
    """fp32 restatement: sequential per-voxel sums, then the update kernel's m + (A / F - m) / f32(counter)."""
    memm = np.asarray(memm, F32).copy()
    V = memm.shape[0]
    k = kept(idx, V)
    i, ww, mm = np.asarray(idx)[k], np.asarray(w, F32)[k], np.asarray(mw, F32)[k]
    if fault == "drop_sample":
        j = int(np.argmax(np.where(mm > 0, ww, -1)))           # the heaviest counted sample: it moves its voxel's mean
        i, ww, mm = np.delete(i, j), np.delete(ww, j), np.delete(mm, j)
    A, F = np.zeros(V, F32), np.zeros(V, F32)
    np.add.at(A, i, ww)
    np.add.at(F, i, mm)
    if fault == "swap_acc_freq":
        A, F = F, A
    c = F32(counter + 1 if fault == "counter_plus_one" else counter)
    m = F > 0
    memm[m] = memm[m] + (A[m] / F[m] - memm[m]) / c
    return memm


def integrate_truth(memm, counter, idx, w, mw):
    """(m64 (V,), bound (V,), updated mask (V,)) in float64."""
    memm = np.asarray(memm, F32).astype(np.float64)
    V = memm.shape[0]
    k = kept(idx, V)
    i = np.asarray(idx)[k].astype(np.int64)
    ww, mm = np.asarray(w, F32)[k].astype(np.float64), np.asarray(mw, F32)[k].astype(np.float64)
    A = np.bincount(i, ww, minlength=V)
    F = np.bincount(i, mm, minlength=V)
    cv = np.bincount(i, minlength=V).astype(np.float64)
    Sw = np.bincount(i, np.abs(ww), minlength=V)
    Sm = np.bincount(i, np.abs(mm), minlength=V)
    upd = F > 0
    m64 = memm.copy()
    bound = np.zeros(V)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(upd, A / F, 0.0)
        m64[upd] = memm[upd] + (q[upd] - memm[upd]) / counter
        bound[upd] = (4 * U * (np.abs(memm[upd]) + np.abs(q[upd]))
                      + cv[upd] * U * (Sw[upd] / F[upd] + np.abs(A[upd]) * Sm[upd] / F[upd] ** 2) / counter)
    return m64, bound, upd


def tree_violations(m32, memm_old, counter, idx, w, mw):
    """Number of voxels outside the bound (updated voxels) or not bit-identical to memm_old (the others)."""
    m64, bound, upd = integrate_truth(memm_old, counter, idx, w, mw)
    m32 = np.asarray(m32, F32)
    old = np.asarray(memm_old, F32)
    bad_upd = ~(np.abs(m32[upd].astype(np.float64) - m64[upd]) <= bound[upd])
    bad_keep = m32[~upd].view(np.uint32) != old[~upd].view(np.uint32)
    return int(bad_upd.sum()) + int(bad_keep.sum())


def tree_inputs(n, V, kind, seed, *, hit=0.7):
    """(idx int32, w fp32, mw fp32) for n samples over V voxels.  kind: 'exact' (w = k 2^-12, k < 4096 small enough that
    every voxel's sum k stays below 2^24; mw in {0, 1}), 'exact_half' (mw in {0, 0.5, 1}), 'one_voxel' (every sample in
    voxel V // 2, w = 2^-12, mw 1), 'general' (w uniform [0, 1), mw = w > 0.1 as BuFF forms it), 'general_mw' (positive
    mask weights in (0, 2)), 'mask_zero' (w > 0 and mw 0 on every sample of the even voxels).  About 1 - hit of idx are -1
    (rays without a hit)."""
    g = np.random.default_rng(seed)
    idx = g.integers(0, V, n).astype(np.int32)
    idx[g.random(n) > hit] = -1
    if kind == "one_voxel":
        idx[:] = V // 2
        return idx, np.full(n, 2.0 ** -12, F32), np.ones(n, F32)
    if kind.startswith("exact"):
        per_voxel = max(1, int(np.bincount(idx[idx >= 0], minlength=V).max())) if n else 1
        kmax = min(4095, (2 ** 24 - 1) // per_voxel)
        w = (g.integers(0, kmax + 1, n) * 2.0 ** -12).astype(F32)
        levels = np.array([0.0, 0.5, 1.0] if kind == "exact_half" else [0.0, 1.0], F32)
        mw = levels[g.integers(0, len(levels), n)]
        return idx, w, mw
    w = g.random(n, dtype=np.float32)
    if kind == "general_mw":
        mw = (g.random(n, dtype=np.float32) * F32(2.0) + F32(1e-3)).astype(F32)
    else:
        mw = (w > F32(0.1)).astype(F32)
    if kind == "mask_zero":
        mw[(idx >= 0) & (idx % 2 == 0)] = 0.0
    return idx, w, mw


def stats_truth(v):
    """float64 (min, max, population std) of the fp32 values."""
    v64 = np.asarray(v, F32).astype(np.float64).ravel()
    mean = v64.mean()
    return float(v64.min()), float(v64.max()), float(np.sqrt(np.mean((v64 - mean) ** 2)))


def stats_ok(mn, mx, sd, v):
    """min / max exact; std within one fp32 ulp of f32(std64) (exactly 0 for a constant volume)."""
    tmn, tmx, tsd = stats_truth(v)
    s32 = F32(tsd)
    return (F32(mn) == F32(tmn) and F32(mx) == F32(tmx)
            and abs(float(F32(sd)) - float(s32)) <= float(np.spacing(s32)) and (tsd != 0.0 or sd == 0.0))
