"""Restatements of the three ray samplers of nm_render.cu in numpy fp32, in the kernels' evaluation order — test
infrastructure, no GPU.  The kernels are built with -fmad=false and use only IEEE + - * / and comparisons (no
transcendentals, no atomics on values), so these restatements match them bit for bit.

* `stratified`: stratified_kernel (a3).  at(i +- 1) recomputed per sample, jitter u01(seed, ray*Nc + i).
* `sample_pdf`: invcdf_kernel (a8).  bins 0.5 (t[i+1] + t[i]); x = w[1:-1] + 1e-5f; `part` summed the kernel's way (lane l
  adds x[l], x[l+32], ... in order, then the xor butterfly 16, 8, 4, 2, 1); cdf = 0 then the sequential run + x / part;
  lo = searchsorted(cdf, u, right=True) (the kernel's binary search), below = max(lo-1, 0), above = min(ncdf-1, lo),
  denom < 1e-5f -> 1; the perturbed u = u01(seed, ray*Nf + j).  The merge with the coarse depths is emulated with the
  kernel's tie rules (a coarse depth goes before equal samples); `sample_pdf` checks nothing itself, the tests hold the
  emulated merge equal to np.sort(concat(t_c, samples)) bit for bit.
* `aabb`: aabb_kernel (a10).  Slab tests in the kernel's order, hits compacted in voxel-index order and capped at 512
  (overflow flag), the bitonic networks restated exactly (with ties in the keys the voxel id that ends up first depends
  on the network, so np.sort would not do), the sequential interval cumsum, the left bucket search, the first-of-bucket
  search, the ascending check, and the random branch's draws on the stream seed ^ SALT_VOXEL.
* `FAULTS`: variants that each carry one plausible bug; tests/test_ray_samplers_reference.py shows that each changes an
  output of the edge matrix, so the bit-exact GPU comparison would catch it.

Float64 truth of SamplePDF (`pdf_truth`).  From the kernel's fp32 inputs it forms x = w + 1e-5f, the cdf and the bins
in float64 (their own error, ~n 2^-53, is negligible).  With U = 2^-24:
  * x_i carries one rounding; `part` adds ceil(nw/32) terms per lane and 5 butterfly levels, so |dpart| <= (D - 1) U part
    with D = ceil(nw/32) + 5; each quotient one more rounding; cdf_k is a sequential sum of k positive terms (k - 1 more
    roundings).  Hence |cdf32_k - cdf_k| <= E_k = 1.01 (k + D + 2) U cdf_k (1.01 covers the second-order terms).
  * lo32 = #{cdf32 <= u} lies between lo_min = #{cdf_k + E_k <= u} and lo_max = #{cdf_k - E_k <= u}.  The denominator
    is exactly 0 when above == below; otherwise the knots are adjacent, cdf32_a = fl(cdf32_b + q32) with q32 within
    (D + 1) U q of q, so fl(ca - cb) (exact, Sterbenz) is within dden = 1.01 (D + 2) U denom + U ca of its float64
    value.  A sample is *decided* when lo_min == lo_max and |denom - 1e-5f| > dden: then the kernel takes the float64
    branch and
      |s32 - s64| <= B = 2 [ U |bb| + |diff| dtt + |tt| ddiff + U |tt diff| + U |s| ],
    tt = (u - cb) / denom (or u - cb when denom -> 1), diff = ba - bb, ddiff = U (|ba| + |bb|) + U |diff| (the bins' and the
    subtraction's roundings), dtt = (E_b + U |u - cb|) / denom + |tt| dden / denom + U |tt| (numerator,
    denominator and quotient; with denom -> 1: E_b + U |u - cb|), and the factor 2 for the second-order terms.
  * An undecided sample must lie within B of the interval spanned by its candidate values: every lo in [lo_min, lo_max]
    and, where the denominator's side of 1e-5f is undecided, both rules.
"""
from __future__ import annotations

import numpy as np

from _chamfer_ref import u01
from _composite_ref import SALT_COARSE, SALT_MAIN

F32 = np.float32
U = 2.0 ** -24
SALT_INVCDF = 0x9e3779b9                 # nm_api.cu kInvCdfSalt: the inverse-CDF jitter of a render chunk
SALT_VOXEL = 0xd1b54a32d192ed03          # nm_api.cu kVoxelSalt: the random voxel draws (NM_FLAG_RANDOM_VOXELS)
MAX_HITS = 512
THR = F32(1e-5)

FAULTS = (
    "strat_jitter_index",      # stratified jitter drawn at i*R + ray instead of ray*Nc + i
    "pdf_searchsorted_left",   # searchsorted(cdf, u) left instead of right
    "pdf_denom_1e-6",          # denom threshold 1e-6 instead of 1e-5
    "pdf_above_clamp",         # above = min(ncdf - 2, lo): the clamp one short
    "pdf_cdf_inclusive",       # the inclusive scan in the exclusive cdf's slots
    "pdf_part_sequential",     # part summed sequentially instead of by lanes and butterfly
    "pdf_jitter_index",        # perturbed u drawn at j*R + ray
    "pdf_merge_ties",          # the merge places a coarse depth after equal samples (both sides count the tie)
    "aabb_neg_from_d",         # the slab's side taken from d < 0 instead of 1/d < 0 (differs at -0)
    "aabb_tmax_lt_far",        # tmax < far instead of <=
    "aabb_stable_sort",        # a stable sort of the hits in place of the bitonic network
    "aabb_bucket_right",       # the bucket search right instead of left
    "aabb_noise_salt",         # the random voxel draws on the fine compositor's noise stream
)


def linspace(n):
    """torch.linspace(0, 1, n) in fp32: ATen's two-sided formula with its upper half one fused multiply-add (float64 holds
    step * k and 1 - step * k exactly, so one rounding to fp32 is the fma), as nm_api.cu's linspace_host."""
    if n == 1:
        return np.zeros(1, F32)
    step = float(F32(1) / F32(n - 1))
    i = np.arange(n)
    return np.where(i < n // 2, step * i, 1.0 - step * (n - 1 - i)).astype(F32)


def lower_bound(n, go_right, shape):
    """The kernels' binary search `lo = 0, hi = n; while lo < hi: mid = (lo+hi)>>1; if go_right(mid) lo = mid+1 else
    hi = mid`, vectorised: n broadcastable to `shape`, go_right(mid) -> bool array of `shape`."""
    lo = np.zeros(shape, np.int64)
    hi = np.broadcast_to(np.asarray(n, np.int64), shape).copy()
    while True:
        act = lo < hi
        if not act.any():
            return lo
        mid = np.where(act, (lo + hi) >> 1, 0)
        right = act & go_right(mid)
        lo = np.where(right, mid + 1, lo)
        hi = np.where(act & ~right, mid, hi)


def _rows(a, idx):
    return np.take_along_axis(a, idx, axis=-1)


# ----------------------------------------------------------------------------------------------------- a3
def stratified(s_table, near, far, lindisp, perturb, seed=0, R=None, fault=None):
    """(R,Nc) stratified_kernel.  near/far: scalars (then R is required) or (R,) per-ray bounds."""
    s = np.asarray(s_table, F32)
    Nc = s.size
    near, far = np.asarray(near, F32), np.asarray(far, F32)
    if near.ndim:
        R = near.size
    nr = np.broadcast_to(near.reshape(-1, 1), (R, 1))
    fr = np.broadcast_to(far.reshape(-1, 1), (R, 1))
    one = F32(1)

    def at(k):
        sk = s[k][None, :]
        if not lindisp:
            return nr * (one - sk) + fr * sk
        return one / (one / nr * (one - sk) + one / fr * sk)
    i = np.arange(Nc)
    with np.errstate(all="ignore"):
        t = at(i)
        if perturb:
            lower = np.where(i == 0, t, F32(0.5) * (t + at(np.maximum(i - 1, 0))))
            upper = np.where(i == Nc - 1, t, F32(0.5) * (at(np.minimum(i + 1, Nc - 1)) + t))
            ray = np.arange(R)[:, None]
            idx = i[None, :] * R + ray if fault == "strat_jitter_index" else ray * Nc + i[None, :]
            t = lower + (upper - lower) * u01(seed, idx)
    return t.astype(F32)


# ----------------------------------------------------------------------------------------------------- a8
def pdf_cdf(w_c, fault=None):
    """(R, Nc-1) the kernel's fp32 cdf of the coarse weights w_c (R,Nc)."""
    w = np.asarray(w_c, F32)
    R, Nc = w.shape
    nw = Nc - 2
    x = w[:, 1:Nc - 1] + THR
    if fault == "pdf_part_sequential":
        part = np.zeros(R, F32)
        for i in range(nw):
            part = part + x[:, i]
    else:
        p = np.zeros((R, 32), F32)
        for c in range(0, nw, 32):
            blk = x[:, c:c + 32]
            p[:, :blk.shape[1]] = p[:, :blk.shape[1]] + blk
        lanes = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            p = p + p[:, lanes ^ o]
        part = p[:, 0]
    cdf = np.zeros((R, nw + 1), F32)
    run = np.zeros(R, F32)
    for i in range(nw):
        run = run + x[:, i] / part
        cdf[:, i + 1] = run
    if fault == "pdf_cdf_inclusive":
        cdf = np.concatenate([cdf[:, 1:], cdf[:, -1:]], 1)
    return cdf


def pdf_u(u, R, Nf, perturb, seed, fault=None):
    """(R,Nf) the u each sample is placed at."""
    if not perturb:
        return np.broadcast_to(np.asarray(u, F32).reshape(1, Nf), (R, Nf)).copy()
    ray, j = np.arange(R)[:, None], np.arange(Nf)[None, :]
    return u01(seed, j * R + ray if fault == "pdf_jitter_index" else ray * Nf + j)


def sample_pdf(t_c, w_c, u, Nf, perturb, seed=0, fault=None, full=False):
    """invcdf_kernel: (R, Nc+Nf) merged output; with full=True also (samples (R,Nf) before the merge, u (R,Nf))."""
    t = np.asarray(t_c, F32)
    R, Nc = t.shape
    ncdf = Nc - 1
    bins = F32(0.5) * (t[:, 1:] + t[:, :-1])
    cdf = pdf_cdf(w_c, fault)
    uu = pdf_u(u, R, Nf, perturb, seed, fault)
    if fault == "pdf_searchsorted_left":
        lo = lower_bound(ncdf, lambda m: _rows(cdf, m) < uu, (R, Nf))
    else:
        lo = lower_bound(ncdf, lambda m: _rows(cdf, m) <= uu, (R, Nf))
    below = np.maximum(lo - 1, 0)
    above = np.minimum(ncdf - 2 if fault == "pdf_above_clamp" else ncdf - 1, lo)
    cb, ca, bb, ba = _rows(cdf, below), _rows(cdf, above), _rows(bins, below), _rows(bins, above)
    denom = ca - cb
    denom = np.where(denom < (F32(1e-6) if fault == "pdf_denom_1e-6" else THR), F32(1), denom)
    smp = (bb + (uu - cb) / denom * (ba - bb)).astype(F32)
    out = merge(t, smp, fault)
    return (out, smp, uu) if full else out


def merge(t, smp, fault=None):
    """The kernel's merge of the ascending coarse depths t (R,Nc) with the samples (R,Nf): the samples are sorted first when
    they do not ascend (a bitonic network without tags: its result is np.sort's), then a coarse depth goes to i + #{samples
    < it} and sample j to j + #{coarse <= it}.  A slot no element lands in stays NaN."""
    R, Nc = t.shape
    Nf = smp.shape[1]
    asc = ~(smp[:, :-1] > smp[:, 1:]).any(1)
    s = np.where(asc[:, None], smp, np.sort(smp, 1))
    if fault == "pdf_merge_ties":
        pc = lower_bound(Nf, lambda m: _rows(s, m) <= t, (R, Nc))
    else:
        pc = lower_bound(Nf, lambda m: _rows(s, m) < t, (R, Nc))
    ps = lower_bound(Nc, lambda m: _rows(t, m) <= s, (R, Nf))
    out = np.full((R, Nc + Nf), np.nan, F32)
    r = np.arange(R)[:, None]
    out[r, np.arange(Nc)[None, :] + pc] = t
    out[r, np.arange(Nf)[None, :] + ps] = s
    return out


def pdf_truth(t_c, w_c, uu):
    """Float64 truth of the samples at u = uu (R,Nf) (module docstring): (s64, decided, lo_val, hi_val, bound), where
    [lo_val, hi_val] spans the candidate values and `bound` is B (the candidates' largest where undecided)."""
    t = np.asarray(t_c, F32).astype(np.float64)
    w = np.asarray(w_c, F32).astype(np.float64)
    u = np.asarray(uu, F32).astype(np.float64)
    R, Nc = t.shape
    nw, ncdf = Nc - 2, Nc - 1
    thr = float(THR)
    bins = 0.5 * (t[:, 1:] + t[:, :-1])
    x = w[:, 1:Nc - 1] + thr
    cdf = np.concatenate([np.zeros((R, 1)), np.cumsum(x / x.sum(1, keepdims=True), 1)], 1)
    D = -(-nw // 32) + 5
    E = 1.01 * (np.arange(ncdf)[None, :] + D + 2) * U * cdf
    lo_min = (cdf[:, None, :] + E[:, None, :] <= u[..., None]).sum(-1)
    lo_max = (cdf[:, None, :] - E[:, None, :] <= u[..., None]).sum(-1)
    vals, bounds, dec = [], [], lo_min == lo_max
    with np.errstate(all="ignore"):
        for dl in range(int((lo_max - lo_min).max()) + 1):
            lo = np.minimum(lo_min + dl, lo_max)
            below, above = np.maximum(lo - 1, 0), np.minimum(ncdf - 1, lo)
            cb, ca, bb, ba = _rows(cdf, below), _rows(cdf, above), _rows(bins, below), _rows(bins, above)
            Eb, Ea = _rows(E, below), _rows(E, above)
            denom = ca - cb
            dden = np.where(above == below, 0.0, 1.01 * (D + 2) * U * denom + U * ca)
            undec_d = np.abs(denom - thr) <= dden
            if dl == 0:
                dec = dec & ~undec_d
            diff = ba - bb
            ddiff = U * (np.abs(ba) + np.abs(bb)) + U * np.abs(diff)
            num = u - cb
            for other in (False, True):                # the float64 side of the threshold, then (where undecided) the other
                repl = (denom < thr) != other
                d = np.where(repl, 1.0, denom)
                tt = num / d
                dtt = np.where(repl, Eb + U * np.abs(num),
                               (Eb + U * np.abs(num)) / d + np.abs(tt) * dden / d + U * np.abs(tt))
                s = bb + tt * diff
                B = 2 * (U * np.abs(bb) + np.abs(diff) * dtt + np.abs(tt) * ddiff + U * np.abs(tt * diff) + U * np.abs(s))
                use = undec_d if other else np.ones_like(undec_d)
                vals.append(np.where(use, s, np.nan))
                bounds.append(np.where(use, B, 0.0))
        V = np.stack(vals)
        return V[0], dec, np.nanmin(V, 0), np.nanmax(V, 0), np.max(np.stack(bounds), 0)


# ----------------------------------------------------------------------------------------------------- a10
def bitonic(key, *tags):
    """warp_bitonic_sort(_tagged / _triples) over len(key) (a power of two) elements: the same compare-exchange network, one
    stage at a time (the pairs of a stage are disjoint, so the lane order inside a stage does not matter)."""
    key = np.array(key)
    tags = [np.array(t) for t in tags]
    n = key.size
    i = np.arange(n)
    k = 2
    while k <= n:
        j = k >> 1
        while j > 0:
            p = i ^ j
            a = i[p > i]
            b = a ^ j
            x, y = key[a], key[b]
            up = (a & k) == 0
            sw = (x > y) == up
            a, b = a[sw], b[sw]
            for arr in (key, *tags):
                tmp = arr[a].copy()
                arr[a] = arr[b]
                arr[b] = tmp
            j >>= 1
        k <<= 1
    return (key, *tags)


def _pow2(n):
    m = 1
    while m < n:
        m <<= 1
    return m


def slab_hits(voxels, o, d, near, far, fault=None):
    """(hit (V,), tmin (V,), tmax (V,)) of one ray in the kernel's order."""
    v = np.asarray(voxels, F32).reshape(-1, 2, 3)
    o, d = np.asarray(o, F32), np.asarray(d, F32)
    with np.errstate(all="ignore"):
        inv = F32(1) / d
        neg = (d < 0) if fault == "aabb_neg_from_d" else (inv < 0)
        vmin, vmax = v[:, 0, :], v[:, 1, :]
        tlo = (np.where(neg, vmax, vmin) - o) * inv
        thi = (np.where(neg, vmin, vmax) - o) * inv
        tmin, tmax = tlo[:, 0], thi[:, 0]
        hit = (tmin <= thi[:, 1]) & (tlo[:, 1] <= tmax)
        tmin = np.where(tlo[:, 1] > tmin, tlo[:, 1], tmin)
        tmax = np.where(thi[:, 1] < tmax, thi[:, 1], tmax)
        hit = hit & (tmin <= thi[:, 2]) & (tlo[:, 2] <= tmax)
        tmin = np.where(tlo[:, 2] > tmin, tlo[:, 2], tmin)
        tmax = np.where(thi[:, 2] < tmax, thi[:, 2], tmax)
        hit = hit & (tmin >= F32(near)) & ((tmax < F32(far)) if fault == "aabb_tmax_lt_far" else (tmax <= F32(far)))
    return hit, tmin, tmax


def aabb(voxels, origins, dirs, near, far, S, s_table, t_uniform, random=False, seed=0, fault=None):
    """aabb_kernel over R rays: (z (R,S) fp32, idx (R,S) int32, hits (R,) before the cap, overflow).  origins (3,) or
    (R,3); t_uniform (R,S) the fallback of rays without a hit; `seed` the render chunk's seed (salted here)."""
    d = np.asarray(dirs, F32).reshape(-1, 3)
    R = d.shape[0]
    o = np.broadcast_to(np.asarray(origins, F32).reshape(-1, 3), (R, 3))
    st = np.asarray(s_table, F32)
    z = np.zeros((R, S), F32)
    idx = np.full((R, S), -1, np.int32)
    nhits = np.zeros(R, np.int64)
    salt = SALT_MAIN if fault == "aabb_noise_salt" else SALT_VOXEL
    for r in range(R):
        hit, tmin, tmax = slab_hits(voxels, o[r], d[r], near, far, fault)
        ids = np.nonzero(hit)[0][:MAX_HITS]
        nhits[r] = int(hit.sum())
        H = ids.size
        if H == 0:
            z[r] = np.asarray(t_uniform, F32)[r]
            continue
        lo, hi, vox = tmin[ids].astype(F32), tmax[ids].astype(F32), ids.astype(np.int32)
        k = np.arange(S)
        if random:
            c = (r * S + k).astype(np.uint64)
            h = np.minimum((u01(seed ^ salt, 2 * c) * F32(H)).astype(np.int32), H - 1)
            zz = lo[h] + (hi[h] - lo[h]) * u01(seed ^ salt, 2 * c + np.uint64(1))
            m2 = _pow2(S)
            zk, bk = bitonic(np.concatenate([zz, np.full(m2 - S, np.inf, F32)]),
                             np.concatenate([vox[h], np.full(m2 - S, -1, np.int32)]))
            z[r], idx[r] = zk[:S], bk[:S]
            continue
        n2 = _pow2(H)
        pad = n2 - H
        lo_p = np.concatenate([lo, np.full(pad, np.inf, F32)])
        hi_p = np.concatenate([hi, np.full(pad, np.inf, F32)])
        vx_p = np.concatenate([vox, np.full(pad, -1, np.int32)])
        if fault == "aabb_stable_sort":
            order = np.argsort(lo_p, kind="stable")
            lo_p, hi_p, vx_p = lo_p[order], hi_p[order], vx_p[order]
        else:
            lo_p, hi_p, vx_p = bitonic(lo_p, hi_p, vx_p)
        cums = np.zeros(H, F32)
        run = F32(0)
        for i in range(H):
            run = F32(run + (hi_p[i] - lo_p[i]))
            cums[i] = run
        total = cums[H - 1]
        s = st * total
        if fault == "aabb_bucket_right":
            a = lower_bound(H, lambda m: cums[m] <= s, (S,))
        else:
            a = lower_bound(H, lambda m: cums[m] < s, (S,))
        bucket = np.minimum(a, H - 1)
        first = lower_bound(k, lambda m: bucket[m] < bucket, (S,))
        zz = lo_p[bucket] + (st * total - st[first] * total)
        bid = vx_p[bucket]
        if (zz[:-1] > zz[1:]).any():
            m2 = _pow2(S)
            zz, bid = bitonic(np.concatenate([zz, np.full(m2 - S, np.inf, F32)]),
                              np.concatenate([bid, np.full(m2 - S, -1, np.int32)]))
            zz, bid = zz[:S], bid[:S]
        z[r], idx[r] = zz, bid
    return z, idx, nhits, bool((nhits > MAX_HITS).any())


# ----------------------------------------------------------------------------------------------------- random streams
G = 0x9E3779B97F4A7C15
G_INV = pow(G, -1, 2 ** 64)


def stream_distance(seed_a, seed_b):
    """u01(seed_a, i) and u01(seed_b, j) share a splitmix64 state iff j - i == this (mod 2^64), returned signed."""
    d = ((seed_a - seed_b) * G_INV) % 2 ** 64
    return d - 2 ** 64 if d >= 2 ** 63 else d


def render_streams(seed, r0s, buff, voxel_salt=SALT_VOXEL):
    """(name, salted seed) of every random stream one render draws from: per chunk seed s = seed + r0, the stratified
    jitter (s), the inverse-CDF jitter (s ^ SALT_INVCDF), the coarse and the fine / only compositor noise (s ^ SALT_COARSE,
    s ^ SALT_MAIN); a BuFF render draws the stratified fallback, the voxel draws (s ^ voxel_salt) and the noise."""
    out = []
    for r0 in r0s:
        s = (seed + r0) % 2 ** 64
        if buff:
            out += [(f"strat@{r0}", s), (f"voxel@{r0}", s ^ voxel_salt), (f"noise@{r0}", s ^ SALT_MAIN)]
        else:
            out += [(f"strat@{r0}", s), (f"invcdf@{r0}", s ^ SALT_INVCDF), (f"noise_c@{r0}", s ^ SALT_COARSE),
                    (f"noise_f@{r0}", s ^ SALT_MAIN)]
    return out


def closest_streams(streams):
    """(|distance|, name a, name b) of the closest pair of distinct streams."""
    best = None
    for i in range(len(streams)):
        for j in range(i + 1, len(streams)):
            dist = abs(stream_distance(streams[i][1], streams[j][1]))
            if best is None or dist < best[0]:
                best = (dist, streams[i][0], streams[j][0])
    return best
