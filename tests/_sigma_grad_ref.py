"""Float64 reference of the density gradient g = d raw sigma / d p (nm_sigma_grad, DESIGN 4.8) — test infrastructure, no
GPU.

`sigma_grad_ref` differentiates `_mlp_ref.truth_forward`'s network by hand: the data-gradient chain seeded with
d raw sigma = 1 (d rgb = 0), dPE = sum_l dZ_l W_l[:, PE] over the layers that read the xyz encoding (layer1 and the skips),
then the encoding Jacobian (identity block; d sin(f x) = f cos(f x), d cos(f x) = -f sin(f x)).  Every entry gets an
error scale S built the `_mlp_ref` way: the one-step absolute-value data gradient dZ~_l = relu'(z_l) (|dZ_l+1| |W_l+1|)
(+ |w_alpha| at the fc_alpha layer) pushed through |W_l[:, PE]| and |J_PE|.  `gate_margin` / `MU_*` of `_mlp_ref` select
the points whose relu gates every implementation agrees on.

The knobs of `sigma_grad_ref` (`drop_skip`, `drop_identity`, `flip_cos`, `double_band`, `drop_pass`) build the synthetic
faults tests/test_sigma_grad_reference.py shows the GPU tolerances flag.  `emulate_tail_exact` is the tensor-core tail's
arithmetic: bf16 hi / lo splits of dZ and of W[:, PE], three products hi*hi + lo*hi + hi*lo (or fewer).
"""
from __future__ import annotations

import numpy as np
import torch

import _mlp_ref as R

# Tolerances of tests/test_gpu_sigma_grad.py: |g - g_ref| <= tau * S per entry.  Each is >= 4x the worst ratio measured on
# an H100 80GB HBM3 over that test's cases (all four NETS at every edge size), quoted in brackets.
TAU_EXACT = 2e-6      # tensor cores, NM_PREC_EXACT, against the float64 truth [3.9e-7]
TAU_FP32 = 1e-7       # NM_PREC_FP32 (SIMT chain + sgemm) against the float64 truth [1.9e-8]
TAU_FAST = 6e-4       # NM_PREC_FAST against the float64 truth, on the 128-wide nets (FAST_NETS) [1.3e-4]
# Fast mode is checked where its gate margin leaves points: the 256-wide nets have none at MU_FAST (as in the backward tests)
FAST_NETS = ("tiny", "ldir2")


def bands(cfg):
    L = cfg.num_encoding_fn_xyz
    if cfg.log_sampling_xyz:
        return (2.0 ** torch.linspace(0.0, L - 1, L)).numpy().astype(np.float64)
    return torch.linspace(1.0, 2.0 ** (L - 1), L).numpy().astype(np.float64)


def pe_jacobian(cfg, pts, enc_dtype=torch.float32, flip_cos=False, double_band=None, drop_identity=False):
    """(M, dim_xyz, 3) d enc_j / d x_c in the encoder's column order.  The argument f_k x_c is the encoder's (fp32
    product for enc_dtype float32), its sin / cos in float64."""
    p = np.asarray(pts, np.float64)
    M, L = p.shape[0], cfg.num_encoding_fn_xyz
    f = bands(cfg)
    if enc_dtype == torch.float32:
        arg = (np.asarray(p, np.float32)[:, :, None] * f.astype(np.float32)[None, None, :]).astype(np.float64)
    else:
        arg = p[:, :, None] * f[None, None, :]
    fk = f.copy()
    if double_band is not None:
        fk[double_band] *= 2.0
    J = np.zeros((M, cfg.dim_xyz, 3))
    base = 0
    if cfg.include_input_xyz:
        if not drop_identity:
            for c in range(3):
                J[:, c, c] = 1.0
        base = 3
    for c in range(3):
        for k in range(L):
            J[:, base + c * L + k, c] = fk[k] * np.cos(arg[:, c, k])
            J[:, base + 3 * L + c * L + k, c] = (1.0 if flip_cos else -1.0) * fk[k] * np.sin(arg[:, c, k])
    return J


def bf16_split(x):
    hi = R.bf16_rn(x)
    lo = R.bf16_rn((np.asarray(x, np.float64) - hi).astype(np.float32))
    return hi, lo


def emulate_tail_exact(dz, w_pe, passes=("hh", "lh", "hl")):
    """The tensor-core tail's product dZ W_pe with bf16 hi / lo operands (dZ rounded to fp32 first, as the chain stores
    it), the listed passes summed exactly."""
    ah, al = bf16_split(np.asarray(dz, np.float32))
    wh, wl = bf16_split(np.asarray(w_pe, np.float32))
    out = np.zeros((dz.shape[0], w_pe.shape[1]))
    for p in passes:
        a = ah if p[0] == "h" else al
        w = wh if p[1] == "h" else wl
        out += a @ w
    return out


def sigma_grad_ref(cfg, sd, pts, enc_dtype=torch.float32, rec=None, *, drop_skip=False, drop_identity=False,
                   flip_cos=False, double_band=None, drop_pass=None):
    """float64 (g (M,3), S (M,3), sigma (M,), rec) of truth_forward's network at pts (directions = positions).
    Fault knobs: drop_skip leaves the skip layers' PE contribution out, drop_identity the include_input block, flip_cos
    the sign of the cos-derivative term, double_band = k doubles band k's factor, drop_pass in ("lh", "hl") evaluates the
    PE product with the tensor cores' bf16 operands minus that pass."""
    if rec is None:
        rec = R.truth_forward(cfg, sd, pts, None, enc_dtype)
    W = rec.sd
    layers = R.layer_list(cfg)
    M = pts.shape[0]
    last_trunk = cfg.num_layers - 1
    dzs, adzs = {}, {}
    if cfg.use_viewdirs:
        dx = np.zeros((M, cfg.hidden_size))
        adx = np.zeros_like(dx)
        wa = W["fc_alpha.weight"]
        dx, adx = dx + wa[0][None, :], adx + np.abs(wa[0])[None, :]
    else:
        wo = W["fc_out.weight"]
        dx = np.broadcast_to(wo[3][None, :], (M, wo.shape[1])).copy()
        adx = np.abs(dx)
    for li in range(last_trunk, -1, -1):
        L = layers[li]
        if L.relu:
            m = rec.Z[li] > 0
            dx, adx = dx * m, adx * m
        dzs[li], adzs[li] = dx, adx
        Wl = W[L.name + ".weight"]
        dx, adx = dx @ Wl[:, :L.k_act], np.abs(dx) @ np.abs(Wl[:, :L.k_act])
    dpe = np.zeros((M, cfg.dim_xyz))
    spe = np.zeros_like(dpe)
    for li in range(last_trunk + 1):
        L = layers[li]
        if L.pe != "xyz" or (drop_skip and li > 0):
            continue
        wpe = W[L.name + ".weight"][:, L.k_act:L.k_act + cfg.dim_xyz]
        if drop_pass is not None:
            dpe += emulate_tail_exact(dzs[li], wpe, tuple(p for p in ("hh", "lh", "hl") if p != drop_pass))
        else:
            dpe += dzs[li] @ wpe
        spe += adzs[li] @ np.abs(wpe)
    J = pe_jacobian(cfg, pts, enc_dtype, flip_cos=flip_cos, double_band=double_band, drop_identity=drop_identity)
    Jt = pe_jacobian(cfg, pts, enc_dtype)
    g = np.einsum("mj,mjc->mc", dpe, J)
    S = np.einsum("mj,mjc->mc", spe, np.abs(Jt))
    return g, S, rec.logits[:, 3].copy(), rec


def fd_sigma_grad(cfg, sd, pts, h=2e-6):
    """fourth-order central finite differences of truth_forward's raw sigma on float64 encodings (truncation ~h^4 f^5:
    ~1e-9 of the scale at the top band f = 512), and per point whether every relu gate is the same at all four offsets
    as at the point itself (elsewhere the difference straddles a kink)."""
    p = np.asarray(pts, np.float64)
    g = np.zeros_like(p)
    layers = R.layer_list(cfg)
    gates = lambda rec: np.concatenate([z > 0 for L, z in zip(layers, rec.Z) if L.relu], axis=1)
    g0 = gates(R.truth_forward(cfg, sd, torch.as_tensor(p), None, torch.float64))
    same = np.ones(p.shape[0], bool)
    for c in range(3):
        e = np.zeros(3)
        e[c] = h
        val = {}
        for k in (-2, -1, 1, 2):
            rec = R.truth_forward(cfg, sd, torch.as_tensor(p + k * e), None, torch.float64)
            val[k] = rec.logits[:, 3]
            same &= (gates(rec) == g0).all(axis=1)
        g[:, c] = (-val[2] + 8 * val[1] - 8 * val[-1] + val[-2]) / (12 * h)
    return g, same


def sweep_coordinates_ref(verts, lins):
    """mesh.sweep_coordinates in float64 numpy (the linspace tables interpolated per axis), for comparison."""
    v = np.asarray(verts, np.float64)
    out = np.zeros_like(v)
    for a in range(3):
        lin = np.asarray(lins[a], np.float64)
        i0 = np.clip(np.floor(v[:, a]), 0, lin.size - 1).astype(int)
        i1 = np.minimum(i0 + 1, lin.size - 1)
        fr = v[:, a] - i0
        out[:, a] = lin[i0] + fr * (lin[i1] - lin[i0])
    return out
