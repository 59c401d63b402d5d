"""BuFF tree integration and the volume statistics on the device against tests/_tree_stats_ref.py.

Tree integration (Engine.tree_integrate -> tree_scatter_kernel / tree_update_kernel):
* exact case (weights k 2^-12, mask weights in {0, 1} / {0, 0.5, 1}): equal to the oracle bit for bit on both histogram
  paths — shared memory for V <= 6144, global atomics above — and through the grid-stride tail (n > 1184 x 4096);
* general case (uniform weights, BuFF's w > 0.1 mask, positive mask weights): within the float64 bound;
* V 1, 2, 6143, 6144, 6145, 40000; n 0, 1, 255, 256, 257, 4095, 4096, 4097, 1184 x 4096, 1184 x 4096 + 1; about 30 % of
  idx = -1, and idx V, V + 7, -2, INT32_MIN dropped without touching other voxels; all samples in one voxel; mask-0 rows;
  counters 1, 2, 3, 1000 over random memm; memm a slice of a larger buffer with NaN sentinels on both sides; two consecutive
  calls (counter, counter + 1); V large, small, large on one engine; the argument checks.

Volume statistics (Engine.volume_stats, and the two-pass sharded entry Engine.volume_stats_pass combined as
parallel._gathered_stats combines it): min / max exact, std within one fp32 ulp of the float64 truth (0 for a constant
volume), over n 1 ... 257^3 around the 1184 x 256 grid, normal, all-negative, 1e4 + 0.05 N(0, 1), sigma-like and lego
volumes, with the extremum at index 0, at n - 1 and in the grid-stride tail; the argument checks.
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import _tree_stats_ref as TR
from conftest import GOLDEN
from oracle import nerf_oracle as O

pytestmark = pytest.mark.gpu
NET = O.NetCfg(num_layers=2, hidden_size=128, num_encoding_fn_xyz=6)
F32 = np.float32
VS = [1, 2, 6143, 6144, 6145, 40000]
NS = [0, 1, 255, 256, 257, 4095, 4096, 4097, 1184 * 4096, 1184 * 4096 + 1]
COUNTERS = [1, 2, 3, 1000]
STAT_NS = [1, 2, 31, 32, 33, 255, 256, 257, 303103, 303104, 303105, 5 * 303104 + 7, 257 ** 3]


def _bits_equal(a, b):
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.fixture(scope="module")
def eng():
    import nerfmeshes_b200 as nm
    e = nm.Engine(NET.__dict__, None, nm.RenderSettings(num_coarse=8, num_fine=0))
    e.load_weights(0, O.init_weights(NET, 1))
    yield e
    e.close()


def _run(eng, memm, counter, idx, w, mw):
    m = torch.from_numpy(np.asarray(memm, F32).copy()).cuda()
    eng.tree_integrate(torch.from_numpy(idx).cuda(), torch.from_numpy(w).cuda(), torch.from_numpy(mw).cuda(), m, counter)
    return m.cpu().numpy()


def _memm(V, seed):
    return (np.random.default_rng(seed + 7).standard_normal(V) * 0.5).astype(F32)


@pytest.mark.parametrize("V", VS)
def test_tree_exact_case_bit_for_bit(eng, V):
    for s, n in enumerate(NS):
        kind = ("exact", "exact_half")[s % 2]
        idx, w, mw = TR.tree_inputs(n, V, kind, 1000 * V + s)
        if n >= 8:                                                 # out-of-range indices: dropped by the kernel
            idx[[1, 3, 5, 7]] = [V, V + 7, -2, np.iinfo(np.int32).min]
        counter = COUNTERS[s % 4]
        memm = _memm(V, s)
        got = _run(eng, memm, counter, idx, w, mw)
        ref = TR.integrate_oracle(memm, counter, idx, w, mw)
        assert _bits_equal(got, ref), (V, n, kind, counter, int((got != ref).sum()))
        assert TR.tree_violations(got, memm, counter, idx, w, mw) == 0


@pytest.mark.parametrize("V", VS)
def test_tree_general_case_within_bound(eng, V):
    for s, n in enumerate(NS):
        kind = ("general", "general_mw", "mask_zero")[s % 3]
        idx, w, mw = TR.tree_inputs(n, V, kind, 2000 * V + s)
        counter = COUNTERS[(s + 1) % 4]
        memm = _memm(V, s)
        got = _run(eng, memm, counter, idx, w, mw)
        assert TR.tree_violations(got, memm, counter, idx, w, mw) == 0, (V, n, kind, counter)


@pytest.mark.parametrize("V", [1, 6144, 6145, 40000])
def test_tree_all_samples_in_one_voxel(eng, V):
    for n in (1, 4097, 1184 * 4096 + 1):
        idx, w, mw = TR.tree_inputs(n, V, "one_voxel", n)
        memm = _memm(V, n)
        got = _run(eng, memm, 3, idx, w, mw)
        ref = TR.integrate_oracle(memm, 3, idx, w, mw)
        assert _bits_equal(got, ref), (V, n)
        keep = np.arange(V) != V // 2
        assert _bits_equal(got[keep], memm[keep])


def test_tree_dropped_indices_and_mask_zero_rows(eng):
    for V in (6144, 6145):
        idx, w, mw = TR.tree_inputs(20000, V, "exact", V)
        memm = _memm(V, 1)
        base = _run(eng, memm, 2, idx, w, mw)
        noisy_idx = np.concatenate([idx, np.array([V, V + 7, -2, np.iinfo(np.int32).min, -1] * 50, np.int32)])
        noisy_w = np.concatenate([w, np.full(250, 0.75, F32)])
        noisy_mw = np.concatenate([mw, np.ones(250, F32)])
        assert _bits_equal(_run(eng, memm, 2, noisy_idx, noisy_w, noisy_mw), base)
        # rows with w > 0 and mask 0 only: acc grows, freq does not, the voxel keeps its bits
        z_idx = np.array([0, 0, V - 1, 3], np.int32)
        got = _run(eng, memm, 2, z_idx, np.array([0.5, 0.25, 1.0, 0.0], F32), np.array([0.0, 0.0, 0.0, 1.0], F32))
        ref = memm.copy()
        ref[3] = memm[3] + (F32(0) - memm[3]) / F32(2)
        assert _bits_equal(got, ref)


def test_tree_memm_slice_with_sentinels_and_consecutive_calls(eng):
    V = 6145
    idx, w, mw = TR.tree_inputs(50000, V, "exact", 5)
    buf = torch.full((V + 64,), float("nan"), device="cuda")
    memm0 = _memm(V, 5)
    buf[32:32 + V] = torch.from_numpy(memm0).cuda()
    view = buf[32:32 + V]
    ti, tw, tm = torch.from_numpy(idx).cuda(), torch.from_numpy(w).cuda(), torch.from_numpy(mw).cuda()
    eng.tree_integrate(ti, tw, tm, view, 3)
    eng.tree_integrate(ti, tw * 0.5, tm, view, 4)                   # the model's next step: counter + 1
    ref = TR.integrate_oracle(TR.integrate_oracle(memm0, 3, idx, w, mw), 4, idx, (w * F32(0.5)).astype(F32), mw)
    out = buf.cpu().numpy()
    assert _bits_equal(out[32:32 + V], ref)
    assert np.isnan(out[:32]).all() and np.isnan(out[32 + V:]).all()


def test_tree_scratch_reuse_large_small_large(eng):
    for s, V in enumerate([40000, 3, 40000, 6145, 2]):
        n = 100003
        idx, w, mw = TR.tree_inputs(n, V, "exact", 40 + s)
        memm = _memm(V, s)
        assert _bits_equal(_run(eng, memm, 2, idx, w, mw), TR.integrate_oracle(memm, 2, idx, w, mw)), V


def test_tree_integrate_argument_checks(eng):
    lib, h, st = eng.lib, eng._h, eng._stream()
    idx = torch.zeros(16, dtype=torch.int32, device="cuda")
    w, memm = torch.ones(16, device="cuda"), torch.zeros(8, device="cuda")
    p = lambda x: C.c_void_p(x.data_ptr())
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    for n, V, counter in [(16, 8, 0), (0, 8, 0), (16, 0, 1), (16, 8, -3), (-1, 8, 1)]:
        assert lib.nm_tree_integrate(h, p(idx), p(w), p(w), n, p(memm), V, counter, st) != 0, (n, V, counter)
        assert lib.nm_last_error()
    assert lib.nm_tree_integrate(h, p(idx), p(w), p(w), 16, None, 8, 1, st) != 0
    torch.cuda.synchronize()
    assert eng.launch_count() == n0
    assert lib.nm_tree_integrate(h, p(idx), p(w), p(w), 0, p(memm), 8, 1, st) == 0
    torch.cuda.synchronize()
    assert eng.launch_count() == n0 and float(memm.abs().sum()) == 0
    assert lib.nm_tree_integrate(h, p(idx), p(w), p(w), 16, p(memm), 8, 1, st) == 0
    torch.cuda.synchronize()
    assert eng.launch_count() == n0 + 2 and float(memm[0]) == 1.0


# ----------------------------------------------------------------------------------------------------- volume statistics
def _volumes(n, g):
    """(name, fp32 volume) pairs of size n."""
    x = g.standard_normal(n).astype(F32)
    sig = np.maximum(g.standard_normal(n).astype(F32) * F32(30), F32(0))
    sig[g.integers(0, n, max(1, n // 50000))] = F32(4.6e3)
    out = [("normal", x), ("negative", (-np.abs(x) - F32(1)).astype(F32)),
           ("offset", (F32(1e4) + F32(0.05) * x).astype(F32)), ("sigma", sig), ("constant", np.full(n, F32(-3.25)))]
    tail = (n // TR.STATS_GRID) * TR.STATS_GRID
    for name, pos in (("max_first", 0), ("max_last", n - 1), ("max_tail", min(tail + (n - tail) // 2, n - 1))):
        v = x.copy()
        v[pos] = F32(9.5)
        v[(pos + 1) % n] = F32(-9.25) if n > 1 else v[0]
        out.append((name, v))
    return out


def _sharded(eng, v, k, seed):
    """min, max, std from volume_stats_pass over k uneven shards (one a single element), combined on the device."""
    n = v.numel()
    g = np.random.default_rng(seed)
    cuts = np.sort(g.choice(np.arange(2, n), size=k - 2, replace=False)) if n > k else np.arange(2, k)
    edges = [0, 1] + [int(c) for c in cuts] + [n]
    shards = [v[a:b] for a, b in zip(edges[:-1], edges[1:]) if b > a]
    accs = []
    for s in shards:
        acc = torch.tensor([-1e308, 1e308, 123.0, 456.0, float(s.numel())], dtype=torch.float64, device="cuda")
        eng.volume_stats_pass(s, 1, acc)
        accs.append(acc)
    allacc = torch.stack(accs)
    mean = (allacc[:, 2].sum() / allacc[:, 4].sum()).reshape(1)
    for s, acc in zip(shards, accs):
        eng.volume_stats_pass(s, 2, acc, mean)
    allsq = torch.stack([a[3] for a in accs])
    st3 = torch.stack([allacc[:, 0].min(), allacc[:, 1].max(), (allsq.sum() / allacc[:, 4].sum()).sqrt()]).cpu()
    return tuple(float(x) for x in st3)


@pytest.mark.parametrize("n", STAT_NS)
def test_volume_stats_against_float64(eng, n):
    g = np.random.default_rng(n)
    for name, v in _volumes(n, g):
        dv = torch.from_numpy(v).cuda()
        mn, mx, sd = eng.volume_stats(dv)
        assert TR.stats_ok(mn, mx, sd, v), (n, name, mn, mx, sd, TR.stats_truth(v))
        if name == "constant":
            assert sd == 0.0 and mn == mx == -3.25
        if n >= 3 and name in ("normal", "offset", "max_tail", "constant"):
            smn, smx, ssd = _sharded(eng, dv, 4 if n < 1000 else 7, n)
            assert TR.stats_ok(smn, smx, ssd, v), (n, name, "sharded", smn, smx, ssd)


def test_volume_stats_lego_grid(eng):
    z = np.load(os.path.join(GOLDEN, "golden_lego_grid.npz"))
    v = np.ascontiguousarray(z["radiance"][..., 3], dtype=F32)
    dv = torch.from_numpy(v).cuda()
    assert TR.stats_ok(*eng.volume_stats(dv), v)
    assert TR.stats_ok(*_sharded(eng, dv.reshape(-1), 5, 0), v)


def test_volume_stats_argument_checks(eng):
    lib, h, st = eng.lib, eng._h, eng._stream()
    v = torch.ones(100, device="cuda")
    acc = torch.zeros(5, dtype=torch.float64, device="cuda")
    mean = torch.zeros(1, dtype=torch.float64, device="cuda")
    p = lambda x: C.c_void_p(x.data_ptr())
    out = (C.c_float * 3)()
    torch.cuda.synchronize()
    n0 = eng.launch_count()
    assert lib.nm_volume_stats(h, p(v), 0, out) != 0
    for n, pass_no, m in [(0, 1, None), (100, 0, None), (100, 3, p(mean)), (100, 2, None), (-5, 2, p(mean))]:
        assert lib.nm_volume_stats_dev(h, p(v), n, pass_no, m, p(acc), st) != 0, (n, pass_no)
        assert lib.nm_last_error()
    torch.cuda.synchronize()
    assert eng.launch_count() == n0
    assert lib.nm_volume_stats_dev(h, p(v), 100, 1, None, p(acc), st) == 0
    assert lib.nm_volume_stats_dev(h, p(v), 100, 2, p(mean), p(acc), st) == 0
    torch.cuda.synchronize()
    assert eng.launch_count() == n0 + 3
    assert acc[:4].tolist() == [1.0, 1.0, 100.0, 100.0]
