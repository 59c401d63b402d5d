"""Float64 reference of the training compositor adjoint (`composite_backward_kernel`, nm_train.cu) and of the sigma noise
the compositors add — test infrastructure, no GPU.

* `randn` / `sigma_noise`: nm::randn (nm_composite.cuh) as Box-Muller in float64 on the exact splitmix64 draws
  (2 idx, 2 idx + 1) of `_chamfer_ref.u01`, with the max(a, 1e-7f) clamp; the noise of sample i of ray r is
  fp32(fp32(randn(seed, r*S + i)) * noise_std).  The device's logf / cospif are not bit-exact with float64, so its noise
  differs from this one by a few ulp (bounded by NOISE_REL |n|); a sample whose noisy pre-activation lies within
  GATE_MU |n| of 0 may be gated differently by the two and is `undecided`.
* `composite_adjoint`: the float64 truth.  From the kernel's fp32 inputs (raw, t, dirs, d_rgb, the fp32 noisy
  pre-activation) it forms dist, alpha = 1 - exp(-relu(pre) dist), keep = 1 - alpha + 1e-10f, T = exclusive cumprod(keep),
  w = alpha T, G = g . c (- sum g with a white background), dalpha = G T - (sum_{j>i} G_j w_j) / keep and
  d sigma = [pre > 0] dalpha dist exp(-relu(pre) dist).  The last sample's dist is 1e10f |d|.  alpha and keep follow fp32
  where it matters: once e = exp(-x) <= 2^-25, fp32 rounds 1 - e to 1, so alpha = 1 and keep = 1e-10f exactly (float64
  would keep e + 1e-10, orders of magnitude off).
* `error_scale`: per element a bound of the kernel's fp32 error (module constants below): the transmittance product's
  rounding, relative and growing with the sample index (a log-sum of every factor's uncertainty, so that a factor known
  only to a factor of 2 does not give a negative bound), with an absolute floor for subnormal transmittance; alpha's
  rounding on the 2^-24 grid next to 1 (and the noise mismatch) propagated through T, through the suffix sum
  (`sum |G_j| dw_j` plus its own rounding from sum |G_j w_j|) and through suffix / keep (|suffix| dkeep / keep^2 — without
  it samples just short of saturation dominate every ratio).
* `emulate_kernel`: the kernel's evaluation order in numpy fp32 (lane segments of ceil(S/32) samples, segment products,
  Hillis-Steele scans across 32 lanes, the reverse walk inside a segment), and `FAULTS`, variants of it that each carry
  one plausible bug; tests/test_composite_adjoint.py shows on the CPU that the committed tolerance flags every one.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from _chamfer_ref import u01

F32 = np.float32
U = 2.0 ** -24                      # fp32 unit roundoff
K10 = float(F32(1e-10))             # the kernel's 1e-10f
BIG = float(F32(1e10))              # 1e10f (exactly 1e10)
SAT_E = 2.0 ** -25                  # e <= SAT_E: fp32 1 - e rounds to 1
SUB = 2.0 ** -149                   # smallest fp32 subnormal
SALT_MAIN, SALT_COARSE = 0x5bd1e995, 0x7f4a7c15a3c59ac3   # nm_api.cu: the fine / only pass, the coarse pass
NOISE_REL = 2.0 ** -20              # |device noise - sigma_noise| <= NOISE_REL |n| (logf, cospif: ~1 ulp each)
GATE_MU = 2.0 ** -16                # gate margin: 16x NOISE_REL

# Tolerance of tests/test_gpu_composite_adjoint.py: |kernel - truth| <= TAU * error_scale, >= 4x the worst ratio measured
# on an H100 80GB HBM3 (700 W limit) over the whole edge matrix [bracketed].  tests/test_composite_adjoint.py shows that
# the fp32 emulation stays within it and that every variant of FAULTS exceeds it.
# The scale is close to a rigorous bound: both the kernel and the emulation reach ~0.99 of it, on the rgb adjoint of a
# sample after one in the 2^-25 < e < 2^-10 band, where keep is only known to the 2^-25 rounding of alpha next to 1.
TAU = 4.0                           # [0.994]
EMUL_WORST = 1.0                    # the fp32 emulation against the truth on the CPU edge matrix [0.991]


# ----------------------------------------------------------------------------------------------------- noise
def randn(seed, idx):
    """nm::randn(seed, idx) in float64: sqrt(-2 ln max(a, 1e-7f)) cos(2 pi b), a = u01(seed, 2 idx), b = u01(seed, 2 idx + 1)."""
    idx = np.asarray(idx, np.uint64)
    a = np.maximum(u01(seed, np.uint64(2) * idx), F32(1e-7)).astype(np.float64)
    b = u01(seed, np.uint64(2) * idx + np.uint64(1)).astype(np.float64)
    return np.sqrt(-2.0 * np.log(a)) * np.cos(np.pi * (2.0 * b))


def sigma_noise(seed, R, S, noise_std, index_offset=0):
    """(R,S) fp32 noise of a compositor pass whose stream is `seed` (already salted): fp32(randn(seed, r*S + i) * std)."""
    idx = np.arange(R * S, dtype=np.uint64) + np.uint64(index_offset)
    return (randn(seed, idx).astype(F32) * F32(noise_std)).reshape(R, S)


def noisy_pre(raw, noise_std, seed, index_offset=0):
    """(pre, n): the kernel's noisy pre-activation fp32(sigma + n) and the noise n (zeros when noise_std == 0)."""
    s = np.asarray(raw, F32)[..., 3]
    R, S = s.shape
    if noise_std > 0:
        n = sigma_noise(seed, R, S, noise_std, index_offset)
        return s + n, n
    return s.copy(), np.zeros_like(s)


# ----------------------------------------------------------------------------------------------------- float64 truth
@dataclass
class Adjoint:
    dist: np.ndarray
    pre: np.ndarray
    noise: np.ndarray
    x: np.ndarray          # relu(pre) * dist
    e: np.ndarray
    alpha: np.ndarray
    keep: np.ndarray
    T: np.ndarray
    w: np.ndarray
    G: np.ndarray
    AG: np.ndarray         # |g| . c + |white-background term|: the scale of G's rounding
    suffix: np.ndarray
    dalpha: np.ndarray
    drgb: np.ndarray       # (R,S,3) dL/d c (before the sigmoid)
    dsig: np.ndarray       # (R,S) dL/d raw sigma
    c: np.ndarray
    g: np.ndarray

    def dout(self):
        """(R,S,4) what the kernel writes: [dL/d rgb logits = dL/dc c (1 - c), dL/d raw sigma]."""
        return np.concatenate([self.drgb * self.c * (1.0 - self.c), self.dsig[..., None]], -1)


def _excl_rev_cumsum(a):
    """sum_{j>i} a_j along the last axis."""
    return np.flip(np.cumsum(np.flip(a, -1), -1), -1) - a


def composite_adjoint(raw, t, dirs, g, white_bg, noise_std=0.0, seed=0, pre=None) -> Adjoint:
    """The float64 adjoint of L = sum(g * rgb_map) through VolumeRenderer.forward w.r.t. raw = (c, sigma) (module
    docstring).  `pre` overrides the noisy pre-activation (float64 callers: autograd through a float64 oracle)."""
    raw = np.asarray(raw)
    R, S = raw.shape[:2]
    t = np.asarray(t).astype(np.float64)
    d = np.asarray(dirs).astype(np.float64)
    g = np.asarray(g).astype(np.float64)
    if pre is None:
        p32, n32 = noisy_pre(raw, noise_std, seed)
        pre, noise = p32.astype(np.float64), n32.astype(np.float64)
    else:
        pre, noise = np.asarray(pre, np.float64), np.zeros((R, S))
    nrm = np.sqrt((d * d).sum(-1))[:, None]
    dist = np.concatenate([t[:, 1:] - t[:, :-1], np.full((R, 1), BIG)], 1) * nrm
    x = np.maximum(pre, 0.0) * dist
    e = np.exp(-x)
    sat = e <= SAT_E
    alpha = np.where(sat, 1.0, 1.0 - e)
    keep = np.where(sat, K10, e + K10)                  # (1 - alpha) + 1e-10f
    T = np.cumprod(np.concatenate([np.ones((R, 1)), keep[:, :-1]], 1), 1)
    w = alpha * T
    c = raw[..., :3].astype(np.float64)
    bg = g.sum(-1, keepdims=True) if white_bg else np.zeros((R, 1))
    G = (c * g[:, None, :]).sum(-1) - bg
    AG = (c * np.abs(g)[:, None, :]).sum(-1) + np.abs(bg)
    suffix = _excl_rev_cumsum(G * w)
    dalpha = G * T - suffix / keep
    with np.errstate(all="ignore"):
        dsig = np.where(pre > 0, dalpha * dist * e, 0.0)
    dsig = np.where(np.isfinite(dsig), dsig, 0.0)
    drgb = g[:, None, :] * w[..., None]
    return Adjoint(dist, pre, noise, x, e, alpha, keep, T, w, G, AG, suffix, dalpha, drgb, dsig, c, g)


def undecided(a: Adjoint):
    """(R,S) samples whose relu gate the device's noise may decide differently (only with noise on)."""
    return (a.noise != 0) & (np.abs(a.pre) <= GATE_MU * np.abs(a.noise))


def error_scale(a: Adjoint, S):
    """(R,S,4) bound of the kernel's fp32 error per output element (module docstring); inf where the relu gate is
    undecided (d sigma only)."""
    seg = -(-S // 32)
    R = a.pre.shape[0]
    und = undecided(a)
    with np.errstate(all="ignore"):
        # the device's pre-activation: a few ulp of noise mismatch, one rounding of the sum; an undecided gate may open
        dpre = NOISE_REL * np.abs(a.noise) + 2 * U * np.abs(a.pre)
        dpre = np.where(und, np.abs(a.pre) + dpre, dpre)
        # e: the product's and dist's roundings (relative x u each), expf's ulps, the noise, the subnormal grid
        de = a.e * ((3 * a.x + 3) * U + a.dist * dpre) + 4 * SUB
        da = np.where(a.e + de <= SAT_E, 0.0, de + U / 2)          # alpha on the 2^-24 grid next to 1; 0 when surely 1
        dkeep = da + U * a.keep
        keep_lo = np.maximum(a.keep - dkeep, K10)                   # the kernel's keep is never below 1e-10f
        eps = np.log1p(dkeep / keep_lo) + 2 * U                     # log-uncertainty each factor brings into T
        idx = np.arange(S)[None, :]
        rho = np.concatenate([np.zeros((R, 1)), np.cumsum(eps, 1)[:, :-1]], 1) + (idx + 8) * 2 * U
        dT = a.T * np.expm1(rho) + (idx + 8) * SUB
        dw = a.alpha * dT + (a.T + dT) * da + U * a.w
        dG = 4 * U * a.AG
        aGw = np.abs(a.G * a.w)
        dsuffix = _excl_rev_cumsum(np.abs(a.G) * dw + dG * a.w) + (2 * seg + 8) * U * _excl_rev_cumsum(aGw)
        asuf = np.abs(a.suffix)
        ddalpha = (np.abs(a.G) * dT + dG * (a.T + dT) + dsuffix / keep_lo + asuf * dkeep / (a.keep * keep_lo)
                   + 2 * U * (np.abs(a.G) * a.T + asuf / a.keep))
        # + the subnormal grid of dalpha's terms and of the outputs' own products
        ssig = (a.dist * (a.e + de) * (ddalpha + 2 * SUB) + np.abs(a.dalpha) * a.dist * (de + 3 * U * a.e)
                + 4 * U * np.abs(a.dsig) + 2 * SUB)
        ssig = np.where(a.pre > 0, ssig, 0.0)
        ssig = np.where(und, np.inf, np.where(np.isfinite(ssig), ssig, np.inf))
        cc = a.c * (1.0 - a.c)
        srgb = np.abs(a.g)[:, None, :] * cc * dw[..., None] + 5 * U * np.abs(a.drgb * cc) + 3 * SUB
    return np.concatenate([srgb, ssig[..., None]], -1)


def ratio(got, ref, scale):
    """(R,S,4) |got - ref| / scale (0 where both are 0 or the scale is inf; inf where the scale is 0 and they differ)."""
    err = np.abs(np.asarray(got, np.float64) - ref)
    with np.errstate(all="ignore"):
        r = np.where(scale > 0, err / scale, np.where(err > 0, np.inf, 0.0))
    return np.where(np.isinf(scale), 0.0, r)


# ----------------------------------------------------------------------------------------------------- fp32 emulation
FAULTS = (
    "T_inclusive",          # the transmittance scan inclusive instead of exclusive
    "suffix_skip_next",     # the suffix misses the next lane's partial
    "suffix_own_twice",     # the suffix counts its own lane twice
    "last_dist_unscaled",   # the last sample's dist not scaled by |d|
    "last_dist_1e9",        # ... or 1e9 instead of 1e10
    "gate_ge",              # relu' gate >= 0 instead of > 0
    "no_white_bg",          # the white-background term dropped
    "no_sigmoid",           # the sigmoid factor c (1 - c) dropped
    "keep_no_eps",          # keep = 1 - alpha without + 1e-10
    "noise_index_plus1",    # the noise drawn at index ray*S + i + 1
    "noise_other_salt",     # the noise of the other pass's salt
)


def emulate_kernel(raw, t, dirs, g, white_bg, noise_std=0.0, seed=0, fault=None):
    """composite_backward_kernel's evaluation order in numpy fp32 (one row of 32 lanes per ray); `fault` one of FAULTS.
    Returns dout (R,S,4)."""
    raw, t = np.asarray(raw, F32), np.asarray(t, F32)
    dirs, g = np.asarray(dirs, F32), np.asarray(g, F32)
    R, S = t.shape
    seg = -(-S // 32)
    P = 32 * seg
    one, k10 = F32(1), F32(0.0 if fault == "keep_no_eps" else 1e-10)
    if fault == "noise_other_salt":
        seed = seed ^ SALT_MAIN ^ SALT_COARSE
    with np.errstate(all="ignore"):
        pre, _ = noisy_pre(raw, noise_std, seed, 1 if fault == "noise_index_plus1" else 0)
        nrm = np.sqrt(dirs[:, 0] * dirs[:, 0] + dirs[:, 1] * dirs[:, 1] + dirs[:, 2] * dirs[:, 2])[:, None]
        last = F32(1e9) if fault == "last_dist_1e9" else F32(1e10)
        dist = np.concatenate([t[:, 1:] - t[:, :-1], np.full((R, 1), last, F32)], 1) * nrm
        if fault == "last_dist_unscaled":
            dist[:, -1] = last
        gr, gg, gb = g[:, 0, None], g[:, 1, None], g[:, 2, None]
        gbg = (gr + gg) + gb if (white_bg and fault != "no_white_bg") else np.zeros_like(gr)

        def lanes(a, fill):           # (R,S) -> (R,32,seg), padded past S
            out = np.full((R, P), fill, F32)
            out[:, :S] = a
            return out.reshape(R, 32, seg)
        q = [lanes(raw[..., k], 0) for k in range(3)]
        pre_l, dist_l = lanes(pre, 0), lanes(dist, 0)
        valid = lanes(np.ones((R, S), F32), 0) > 0
        e = np.exp(-np.maximum(pre_l, F32(0)) * dist_l)
        alpha = np.where(valid, one - e, F32(0))
        keep = np.where(valid, (one - alpha) + k10, one)
        G = ((gr[:, :, None] * q[0] + gg[:, :, None] * q[1]) + gb[:, :, None] * q[2]) - gbg[:, :, None]
        lane = np.arange(32)[None, :]
        prod = np.ones((R, 32), F32)
        for u in range(seg):
            prod = prod * keep[..., u]
        incl = prod
        for o in (1, 2, 4, 8, 16):
            v = np.concatenate([incl[:, :o], incl[:, :-o]], 1)           # __shfl_up_sync
            incl = np.where(lane >= o, incl * v, incl)
        T = incl if fault == "T_inclusive" else np.concatenate([np.ones((R, 1), F32), incl[:, :-1]], 1)
        Ti = np.empty((R, 32, seg), F32)
        gsum = np.zeros((R, 32), F32)
        for u in range(seg):
            Ti[..., u] = T
            gsum = gsum + (G[..., u] * alpha[..., u]) * T
            T = T * keep[..., u]
        sincl = gsum
        for o in (1, 2, 4, 8, 16):
            v = np.concatenate([sincl[:, o:], sincl[:, -o:]], 1)          # __shfl_down_sync
            sincl = np.where(lane + o < 32, sincl + v, sincl)
        z = np.zeros((R, 1), F32)
        if fault == "suffix_own_twice":
            suffix = sincl
        elif fault == "suffix_skip_next":
            suffix = np.concatenate([sincl[:, 2:], z, z], 1)
        else:
            suffix = np.concatenate([sincl[:, 1:], z], 1)
        out = np.zeros((R, 32, seg, 4), F32)
        for u in range(seg - 1, -1, -1):
            w = alpha[..., u] * Ti[..., u]
            dalpha = G[..., u] * Ti[..., u] - suffix / ((one - alpha[..., u]) + k10)
            suffix = suffix + G[..., u] * w
            for k, gk in enumerate((gr, gg, gb)):
                ck = q[k][..., u]
                out[..., u, k] = gk * w * ck if fault == "no_sigmoid" else ((gk * w) * ck) * (one - ck)
            p = pre_l[..., u]
            gate = (p >= 0) if fault == "gate_ge" else (p > 0)
            o4 = np.where(gate, (dalpha * dist_l[..., u]) * e[..., u], F32(0))
            out[..., u, 3] = np.where(np.isfinite(o4), o4, F32(0))
    return out.reshape(R, P, 4)[:, :S]


# ----------------------------------------------------------------------------------------------------- inputs
KINDS = ("random", "nonpositive", "saturate_first", "subnormal_T", "band", "tiny_last", "duplicate_t")


def make_rays(R, S, seed, kind_offset=0):
    """fp32 (raw (R,S,4), t (R,S), dirs (R,3), d_rgb (R,3), kinds (R,)) with ray r of kind KINDS[(r + kind_offset) % 7]:
    * random: x = sigma dist ~ 2 N(0,1) (both gates), c in (0.02, 0.98)
    * nonpositive: sigma <= 0, every third exactly 0
    * saturate_first: x_0 in [110, 300], so that e_0 == 0 exactly in fp32
    * subnormal_T: x in [18, 60] (saturated: keep = 1e-10f) on the first four samples, then x in [0.5, 3]: T passes
      through the fp32 subnormals to 0
    * band: every fourth sample with 2^-25 < e < 2^-10 (x in [10 ln2, 25 ln2]), light samples between
    * tiny_last: light samples and a tiny positive sigma on the last one: x_last = sigma 1e10 |d| in [0.2, 3], a large
      finite gradient
    * duplicate_t: random, with a third of the intervals of length 0
    |d| log-uniform in [0.05, 20]; t sorted in [2, 6]."""
    rng = np.random.default_rng(seed)
    nd = np.exp(rng.uniform(np.log(0.05), np.log(20.0), R))
    v = rng.standard_normal((R, 3))
    dirs = (v / np.linalg.norm(v, axis=1, keepdims=True) * nd[:, None]).astype(F32)
    t = np.sort(rng.uniform(2.0, 6.0, (R, S)).astype(F32), 1)
    kinds = (np.arange(R) + kind_offset) % len(KINDS)
    dup = (kinds == KINDS.index("duplicate_t"))[:, None] & (rng.uniform(size=(R, S)) < 1 / 3)
    for i in range(1, S):
        t[:, i] = np.where(dup[:, i], t[:, i - 1], t[:, i])
    nrm = np.sqrt((dirs.astype(np.float64) ** 2).sum(1))[:, None]
    dist = np.concatenate([np.diff(t.astype(np.float64), axis=1), np.full((R, 1), 1e10)], 1) * nrm
    dd = np.maximum(dist, 1e-6)
    x = 2.0 * rng.standard_normal((R, S))
    k = kinds[:, None]
    x = np.where(k == KINDS.index("nonpositive"), -np.abs(x) * (np.arange(S) % 3 != 0), x)
    x[:, 0] = np.where(kinds == KINDS.index("saturate_first"), rng.uniform(110, 300, R), x[:, 0])
    first4 = np.arange(S)[None, :] < 4
    x = np.where((k == KINDS.index("subnormal_T")) & first4, rng.uniform(18, 60, (R, S)), x)
    x = np.where((k == KINDS.index("subnormal_T")) & ~first4, rng.uniform(0.5, 3, (R, S)), x)
    band = np.arange(S)[None, :] % 4 == 1
    light = rng.uniform(0, 0.5 / S, (R, S))
    x = np.where(k == KINDS.index("band"), np.where(band, rng.uniform(10 * np.log(2), 25 * np.log(2), (R, S)), light), x)
    x = np.where(k == KINDS.index("tiny_last"), light, x)
    x[:, -1] = np.where(kinds == KINDS.index("tiny_last"), rng.uniform(0.2, 3, R), x[:, -1])
    sigma = (x / dd).astype(F32)
    c = rng.uniform(0.02, 0.98, (R, S, 3))
    raw = np.concatenate([c, sigma[..., None]], -1).astype(F32)
    d_rgb = rng.standard_normal((R, 3)).astype(F32)
    return raw, t, dirs, d_rgb, kinds


# ===================================================================================================== forward compositor
# The inference compositor (`composite_kernel`, nm_render.cu, and the compositor fused into the MLP kernel, nm_mlp_tc.cu:
# both walk nm_composite.cuh's comp_alpha / comp_step / comp_finish): per ray, in sample order, alpha_i and keep_i as
# above, w_i = alpha_i T_i, mask_i = [T_i > thr], rgb = sum w c (+ 1 - acc with a white background), acc = sum w,
# depth_raw = sum w t, disp = 1 / max(1e-10f, depth_raw / acc) with NaN -> 0, depth = depth_raw but 0 where acc < 1 in eval.
#
# `composite_forward` is its float64 truth from the kernel's fp32 inputs, with the fp32 rules of the adjoint's truth
# (alpha = 1, keep = 1e-10f once e <= 2^-25; the last dist 1e10f |d|), keep = 1 where alpha = 0, and one documented
# deviation from
# oracle.volume_render: a NaN noisy pre-activation gives alpha = 0 (the kernel's fmaxf(sigma, 0) drops the NaN; torch.relu
# propagates it).  Everything else equals the oracle run in float64 (tests/test_composite_forward_reference.py).
#
# `forward_error_scale` bounds the kernel's fp32 error per output; with dpre, de, da, dkeep, rho and dT exactly as in
# `error_scale` (T's relative rounding growing with the sample index as a log-sum of every factor's uncertainty, the
# subnormal floor (idx + 8) 2^-149, alpha's 2^-24 grid next to 1, expf's <= 2 ulp inside (3 x + 3) u, the noise mismatch):
#   dw_i     = alpha dT + (T + dT) da + u w + 2^-149                 (the product's own rounding, normal or subnormal)
#   a sequential fp32 sum of terms a_i (every partial sum rounded once) errs by <= u sum_k |partial_k| <= u sum_k
#   cumsum(|a|)_k, plus the propagated error of its terms:
#   dacc     = sum dw + u sum cumsum(w)
#   drgb_c   = sum (dw + u w) c + u sum cumsum(w c)         (+ dacc + u (|1 - acc| + |rgb|) with a white background)
#   ddepth   = sum (dw + u w) |t| + u sum cumsum(w |t|)
#   ddisp    = |disp| (ddepth / |depth| + dacc / acc + 3 u)         (the division, max's clamp (1-Lipschitz), reciprocal)
# Outputs the truth makes NaN or +-inf must be the same bits' class (NaN / the same infinity), and are not scaled.
# The discrete decisions are exact (scale 0) outside their undecided margins (scale inf): the noise gate (|pre| <= GATE_MU
# |n|, which opens every later bound through dpre), mask_i where |T_i - thr| <= dT_i (+ the T rounding), depth where
# |acc - 1| <= dacc + u, and disp where acc <= dacc (the kernel's acc may round to 0: 0/0 -> 0).  The mask has no margin
# while T is exactly 1 in the kernel: at sample 0 (comp_init) and after samples of decided alpha = 0, whose fp32 keep
# 1 + 1e-10f rounds to 1 (the truth takes keep = 1 there too), so a T == thr = 1 decision pins the strict T > thr.
#
# `emulate_forward` is the kernel's order in numpy fp32 and `FWD_FAULTS` its variants with one plausible bug each.
FLT_MAX = float(np.finfo(np.float32).max)
FWD_OUT = ("rgb", "depth", "depth_raw", "acc", "disp", "weights", "mask_weights")
# Tolerance of tests/test_gpu_composite_forward.py: |kernel - truth| <= TAU_FWD * forward_error_scale, >= 4x the worst ratio
# measured on an H100 80GB HBM3 (700 W limit) over the whole edge matrix [bracketed]; tests/test_composite_forward_reference.py
# shows that the fp32 emulation stays within EMUL_WORST_FWD and that every variant of FWD_FAULTS exceeds TAU_FWD.
TAU_FWD = 4.0                       # [0.994]
EMUL_WORST_FWD = 1.0                # the fp32 emulation against the truth on the CPU edge matrix [0.984]


@dataclass
class Forward:
    dist: np.ndarray
    pre: np.ndarray
    noise: np.ndarray
    x: np.ndarray
    e: np.ndarray
    alpha: np.ndarray
    keep: np.ndarray
    T: np.ndarray
    w: np.ndarray
    thr: float
    out: dict              # FWD_OUT -> float64 arrays (mask_weights 0 / 1)


def composite_forward(raw, t, dirs, white_bg, training, thr, noise_std=0.0, seed=0) -> Forward:
    """The float64 truth of the seven forward outputs (section comment above)."""
    raw = np.asarray(raw, F32)
    R, S = raw.shape[:2]
    t = np.asarray(t, F32).astype(np.float64)
    d = np.asarray(dirs, F32).astype(np.float64)
    p32, n32 = noisy_pre(raw, noise_std, seed)
    pre, noise = p32.astype(np.float64), n32.astype(np.float64)
    with np.errstate(all="ignore"):
        nrm = np.sqrt((d * d).sum(-1))[:, None]
        dist = np.concatenate([t[:, 1:] - t[:, :-1], np.full((R, 1), BIG)], 1) * nrm
        sg = np.where(pre > 0, pre, 0.0)                 # NaN -> 0: the kernel's fmaxf rule, not torch.relu's
        x = sg * dist
        e = np.exp(-x)
        sat = e <= SAT_E
        alpha = np.where(sat, 1.0, 1.0 - e)
        keep = np.where(sat, K10, np.where(alpha == 0, 1.0, e + K10))     # fp32 1 + 1e-10f == 1: T stays exactly 1
        T = np.cumprod(np.concatenate([np.ones((R, 1)), keep[:, :-1]], 1), 1)
        w = alpha * T
        c = raw[..., :3].astype(np.float64)
        rgb = (w[..., None] * c).sum(1)
        acc = w.sum(1)
        depth_raw = (w * t).sum(1)
        ratio = depth_raw / acc
        disp = 1.0 / np.maximum(K10, ratio)
        disp = np.where(np.isnan(ratio) | np.isnan(disp), 0.0, disp)
        depth = depth_raw if training else np.where(acc < 1.0, 0.0, depth_raw)
        if white_bg:
            rgb = rgb + (1.0 - acc)[:, None]
    out = dict(rgb=rgb, depth=depth, depth_raw=depth_raw, acc=acc, disp=disp, weights=w,
               mask_weights=(T > float(F32(thr))).astype(np.float64))
    return Forward(dist, pre, noise, x, e, alpha, keep, T, w, float(F32(thr)), out)


def _seqsum_err(a):
    """u sum_k cumsum(|a|)_k along the last axis (+ the subnormal grid of every term): the rounding bound of a sequential
    fp32 sum of a"""
    return U * np.cumsum(np.abs(a), -1).sum(-1) + a.shape[-1] * SUB


def forward_error_scale(f: Forward, raw, t, white_bg):
    """dict FWD_OUT -> bound of the kernel's fp32 error (inf where undecided or not applicable; see the section comment)."""
    raw = np.asarray(raw, F32)
    R, S = f.pre.shape
    t = np.asarray(t, F32).astype(np.float64)
    c = raw[..., :3].astype(np.float64)
    und = (f.noise != 0) & (np.abs(f.pre) <= GATE_MU * np.abs(f.noise))
    with np.errstate(all="ignore"):
        dpre = NOISE_REL * np.abs(f.noise) + 2 * U * np.abs(f.pre)
        dpre = np.where(und, np.abs(f.pre) + dpre, dpre)
        dpre = np.where(np.isnan(f.pre), 0.0, dpre)                               # NaN: alpha = 0, decided
        de = np.where(f.e > 0, f.e * ((3 * f.x + 3) * U + f.dist * dpre), 0.0) + 4 * SUB
        da = np.where(f.e + de <= SAT_E, 0.0, de + U / 2)
        dkeep = da + U * f.keep
        keep_lo = np.maximum(f.keep - dkeep, K10)
        eps = np.log1p(dkeep / keep_lo) + 2 * U
        idx = np.arange(S)[None, :]
        rho = np.concatenate([np.zeros((R, 1)), np.cumsum(eps, 1)[:, :-1]], 1) + (idx + 8) * 2 * U
        dT = f.T * np.expm1(rho) + (idx + 8) * SUB
        dw = f.alpha * dT + (f.T + dT) * da + U * f.w + SUB
        o = f.out
        dacc = dw.sum(1) + _seqsum_err(f.w)
        drgb = ((dw + U * f.w)[..., None] * c).sum(1) + _seqsum_err(np.moveaxis(f.w[..., None] * c, 1, -1))
        if white_bg:
            drgb = drgb + (dacc + U * np.abs(1.0 - o["acc"]))[:, None] + U * np.abs(o["rgb"])
        ddepth = ((dw + U * f.w) * np.abs(t)).sum(1) + _seqsum_err(f.w * t)
        ddisp = np.abs(o["disp"]) * (ddepth / np.abs(o["depth_raw"]) + dacc / o["acc"] + 3 * U)
        sc = dict(rgb=drgb, depth=ddepth, depth_raw=ddepth, acc=dacc, disp=ddisp, weights=dw, mask_weights=np.zeros_like(f.T))
        # a NaN bound comes from an inf or NaN in the truth: 0 there, so that the value must match exactly
        sc = {k: np.where(np.isnan(v), 0.0, v) for k, v in sc.items()}
        sc["disp"] = np.where(o["acc"] <= dacc, np.inf, sc["disp"])                        # acc may round to 0
        sc["depth"] = np.where(np.abs(o["acc"] - 1.0) <= dacc + U, np.inf, sc["depth"])    # acc < 1 undecided
        # T is exactly 1 in the kernel up to and including the first sample whose alpha may be non-zero (comp_init's
        # T = 1.0f, keep = fl(1 + 1e-10f) = 1 after a decided alpha = 0): the mask is decided there even at T == thr
        z = (f.x == 0) & ~und
        one = np.concatenate([np.ones((R, 1), bool), np.cumprod(z[:, :-1], 1).astype(bool)], 1)
        sc["mask_weights"] = np.where(~one & (np.abs(f.T - f.thr) <= dT + U * f.T), np.inf, 0.0)
    return sc


def forward_ratio(got, ref, scale):
    """|got - ref| / scale elementwise, with the special values exact (0 where both are NaN or the same infinity, inf where
    only one is NaN or an infinity differs); 0 where the scale is inf (undecided)."""
    g = np.asarray(got, np.float64)
    with np.errstate(all="ignore"):
        special = np.isnan(ref) | np.isinf(ref) | np.isnan(g) | np.isinf(g)
        same_special = (np.isnan(ref) & np.isnan(g)) | (np.isinf(ref) & (g == ref))
        err = np.abs(g - ref)
        r = np.where(scale > 0, err / scale, np.where(err > 0, np.inf, 0.0))
        r = np.where(special, np.where(same_special, 0.0, np.inf), r)
    return np.where(np.isinf(scale), 0.0, r)


FWD_FAULTS = (
    "mask_after_multiply",      # mask_i = [T_i keep_i > thr]: the mask taken after the transmittance update
    "mask_ge",                  # mask_i = [T_i >= thr]: the comparison not strict
    "T_inclusive",              # w_i = alpha_i T_{i+1}: an inclusive cumprod
    "depth_zero_training",      # depth zeroed where acc < 1 in training mode too
    "disp_from_zeroed_depth",   # disp computed from the thresholded depth
    "disp_nan_propagates",      # disp = 1 / max(1e-10, ratio) with torch.max's NaN and no zeroing
    "last_dist_unscaled",       # the last interval 1e10 instead of 1e10 |d|
    "white_bg_before_acc",      # the white background from the acc before the last sample's weight
    "keep_no_eps",              # keep = 1 - alpha without + 1e-10
    "noise_index_plus1",        # the noise drawn at index ray*S + i + 1
    "noise_other_salt",         # the noise of the other pass's salt
)


def emulate_forward(raw, t, dirs, white_bg, training, thr, noise_std=0.0, seed=0, fault=None):
    """composite_kernel's order in numpy fp32 (one sequential walk per ray); `fault` one of FWD_FAULTS.  Returns
    dict FWD_OUT -> fp32 arrays."""
    raw, t, dirs = np.asarray(raw, F32), np.asarray(t, F32), np.asarray(dirs, F32)
    R, S = t.shape
    one, k10, thr = F32(1), F32(0.0 if fault == "keep_no_eps" else 1e-10), F32(thr)
    if fault == "noise_other_salt":
        seed = seed ^ SALT_MAIN ^ SALT_COARSE
    with np.errstate(all="ignore"):
        pre, _ = noisy_pre(raw, noise_std, seed, 1 if fault == "noise_index_plus1" else 0)
        nrm = np.sqrt((dirs[:, 0] * dirs[:, 0] + dirs[:, 1] * dirs[:, 1]) + dirs[:, 2] * dirs[:, 2])
        T = np.ones(R, F32)
        acc, depth = np.zeros(R, F32), np.zeros(R, F32)
        rgb = np.zeros((R, 3), F32)
        w_all, m_all = np.zeros((R, S), F32), np.zeros((R, S), F32)
        acc_before_last = acc
        for i in range(S):
            if i + 1 < S:
                dist = (t[:, i + 1] - t[:, i]) * nrm
            else:
                dist = np.full(R, F32(1e10)) if fault == "last_dist_unscaled" else F32(1e10) * nrm
            sg = np.fmax(pre[:, i], F32(0))                   # fmaxf: a NaN operand is dropped
            e = np.exp(-sg * dist)
            alpha = one - e
            keep = (one - alpha) + k10
            Tn = T * keep
            w = alpha * (Tn if fault == "T_inclusive" else T)
            Tm = Tn if fault == "mask_after_multiply" else T
            m_all[:, i] = (Tm >= thr) if fault == "mask_ge" else (Tm > thr)
            w_all[:, i] = w
            for k in range(3):
                rgb[:, k] = rgb[:, k] + w * raw[:, i, k]
            acc_before_last = acc
            acc = acc + w
            depth = depth + w * t[:, i]
            T = Tn
        ratio = depth / acc
        zeroed = np.where(((not training) or fault == "depth_zero_training") & (acc < one), F32(0), depth)
        if fault == "disp_from_zeroed_depth":
            ratio = zeroed / acc
        if fault == "disp_nan_propagates":
            disp = one / np.maximum(F32(1e-10), ratio)               # np.maximum propagates NaN, like torch.max
        else:
            disp = one / np.fmax(F32(1e-10), ratio)
            disp = np.where(np.isnan(disp) | np.isnan(ratio), F32(0), disp)
        if white_bg:
            bg = one - (acc_before_last if fault == "white_bg_before_acc" else acc)
            rgb = rgb + bg[:, None]
    return dict(rgb=rgb, depth=zeroed, depth_raw=depth, acc=acc, disp=disp, weights=w_all, mask_weights=m_all)


FWD_KINDS = KINDS + ("empty", "acc_one", "behind", "tiny_ratio", "overflow", "zero_dir", "nan_sigma")


def make_forward_rays(R, S, seed, kind_offset=0):
    """fp32 (raw, t, dirs, kinds) with ray r of kind FWD_KINDS[(r + kind_offset) % 14]: the seven adjoint kinds of
    `make_rays`, and
    * empty: sigma in [-50, -10] everywhere (no noise of std 0.7 opens a gate): acc = 0 exactly, so disp = depth = rgb = 0
      (1 with a white background)
    * acc_one: total optical depth near 17 (T_end near 2^-24: acc just below 1), or one sample with x in [30, 60]
      (alpha = 1 in fp32: acc 1 + 1e-10 sum T, just above) — acc within a few ulp of 1 on both sides
    * behind: t in [-6, -2], sigma > 0: depth / acc < 0, disp = 1e10f exactly
    * tiny_ratio: t in [1e-12, 5e-11]: 0 < depth / acc < 1e-10, disp = 1e10f
    * overflow: the last t is +inf (the interval before it inf): depth inf, disp 0 where the last weight is > 0, and the
      NaN of 0 * inf where the sigma before it is 0 (every other ray)
    * zero_dir: d = 0: every dist 0, acc = 0
    * nan_sigma: every third sigma NaN (alpha = 0 there: the kernel's rule)"""
    raw, t, dirs, _, kinds = make_rays(R, S, seed, kind_offset)
    kinds = (np.arange(R) + kind_offset) % len(FWD_KINDS)
    rng = np.random.default_rng(seed + 1)
    K = {n: i for i, n in enumerate(FWD_KINDS)}
    nd = np.sqrt((dirs.astype(np.float64) ** 2).sum(1))
    for r in np.flatnonzero(kinds >= len(KINDS)):
        name = FWD_KINDS[kinds[r]]
        dist = np.append(np.diff(t[r].astype(np.float64)), 1e10) * nd[r]
        # start from a `random` ray: x = sigma dist ~ 2 N(0,1), colours in (0.02, 0.98)
        raw[r, :, :3] = rng.uniform(0.02, 0.98, (S, 3))
        raw[r, :, 3] = (2.0 * rng.standard_normal(S) / np.maximum(dist, 1e-6)).astype(F32)
        if name == "empty":
            raw[r, :, 3] = rng.uniform(-50, -10, S)
        elif name == "acc_one":
            if (r // len(FWD_KINDS)) % 2 == 0:
                x = np.full(S, rng.uniform(16.0, 18.5) / max(S - 1, 1))
                x[-1] = 0.0 if S > 1 else rng.uniform(16.0, 18.5)
            else:
                x = rng.uniform(0, 0.5 / S, S)
                x[S // 2] = rng.uniform(30, 60)
            raw[r, :, 3] = (x / np.maximum(dist, 1e-6)).astype(F32)
        elif name == "behind":
            t[r] = np.sort(rng.uniform(-6.0, -2.0, S)).astype(F32)
            raw[r, :, 3] = np.abs(raw[r, :, 3]) + F32(0.05)
        elif name == "tiny_ratio":
            t[r] = np.sort(rng.uniform(1e-12, 5e-11, S)).astype(F32)
            d2 = np.append(np.diff(t[r].astype(np.float64)), 1e10) * nd[r]
            raw[r, :, 3] = (np.abs(rng.standard_normal(S)) / np.maximum(d2, 1e-30)).astype(F32)
        elif name == "overflow":
            t[r, -1] = np.inf
            # light samples before it, so that the last weight (T after the saturated inf interval: ~1e-10) stays normal
            raw[r, :, 3] = (rng.uniform(0, 0.5 / S, S) / np.maximum(dist, 1e-6)).astype(F32) + F32(0.05)
            if S > 1 and (r // len(FWD_KINDS)) % 2 == 0:
                raw[r, -2, 3] = 0.0
        elif name == "zero_dir":
            dirs[r] = 0.0
        elif name == "nan_sigma":
            raw[r, ::3, 3] = np.nan
    return raw, t, dirs, kinds
