"""Float64 references of the fused MLP (`mlp_tc_kernel`, nm_mlp_tc.cu) and of the network backward — test infrastructure,
no GPU.

* `truth_forward`: FlexibleNeRFModel (src/nerf/models.py:60-80) in float64 on the fp32 oracle's encodings.  Alongside the
  pre-activations `z` of every layer (and head) it keeps A_z = |X| |W|^T + |b| (the same layer run on |W|, |b| and its
  absolute input |X|), the per-entry error scale of everything below: a product rounded to p bits moves z by at most
  2^-p * A_z.
* `emulate_forward`: the arithmetic of the inference kernel (mode 0) with every product exact in float64.  A operands are
  fp16 `satfinite` hi / lo halves of x * 2^-s (the `encode` lambda and the epilogue), weights fp16 round-to-nearest hi / lo
  (nm_program.cu).  NM_PREC_EXACT sums a_hi*W_hi + a_lo*W_hi + a_hi*W_lo, NM_PREC_FAST a_hi*W_hi alone (its epilogue writes
  lo = 0).  Epilogue: fp32(acc * 2^s + bias), relu; heads are fp32 dot products of the unsplit activation, then the
  sigmoid.  Skip and view-direction layers are K-block concatenations [activation | encoding], as the layer program builds
  them.  What remains between the kernel and this emulation is its fp32 accumulation order.
* `mlp_backward_ref`: the hand-written float64 backward of L = sum(dout * (rgb logits, raw sigma)) for every state-dict
  tensor, and per entry the random-walk scale s[n,k] = sqrt(sum_p (dZ~[p,n] |X[p,k]|)^2).  dZ~ is the absolute-value
  data gradient of one step, dZ~_l = relu'(z_l) * (|dZ_l+1| |W_l+1|) (+ |d sigma| |w_alpha|), the scale of the rounding in
  dZ_l, like A_z in the forward; biases take X = 1, heads |dout| and their input.  |X| is widened by X_ALLOW * A_X to
  cover the forward's own rounding of X.
* `gate_margin` / `filter_dout`: a point whose smallest relu pre-activation |z| / A_z is below mu may be gated differently
  by two implementations; zeroing its `dout` row removes it from every gradient exactly, whatever gate the kernel picks.

The comparators (`forward_ratio`, `grad_ratio`) return the worst error / scale; the tolerances they are held to live in
tests/test_gpu_mlp_edges.py, and tests/test_mlp_reference.py shows on the CPU that those tolerances flag synthetic faults.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np
import torch

from oracle import nerf_oracle as O

F16_MAX = 65504.0

# The networks of the edge tests: 8x256 skip 4 (the shipped shape), `tiny`, a skip-2 net without view directions (fc_out,
# OUT4 head) and a 3x128 net whose 15-wide direction encoding is one K-step.
NETS = {
    "nerf256": dict(),
    "tiny": dict(num_layers=4, hidden_size=128, num_encoding_fn_xyz=6, num_encoding_fn_dir=4),
    "skip2_noview": dict(num_layers=6, hidden_size=256, skip_step=2, num_encoding_fn_xyz=8, use_viewdirs=False),
    "ldir2": dict(num_layers=3, hidden_size=128, num_encoding_fn_xyz=6, num_encoding_fn_dir=2),
}


def net_cfg(name) -> O.NetCfg:
    return O.NetCfg(**NETS[name])


# Tolerances of tests/test_gpu_mlp_edges.py (error / scale).  Each is >= 4x the worst ratio measured on an H100 80GB HBM3
# (700 W limit) over that test's cases, quoted in brackets, and tests/test_mlp_reference.py checks that it flags the
# synthetic faults listed there.
TAU_FWD_EXACT = 8e-6         # point_mlp, NM_PREC_EXACT, against emulate_forward(fast=False): |err| <= tau * A [1.93e-6]
TAU_FWD_FAST = 3.4e-4        # NM_PREC_FAST against emulate_forward(fast=True) [8.14e-5: fp16 rounding-boundary flips]
EMUL_EXACT_VS_TRUTH = 2.0 ** -19   # emulate_forward(fast=False) against truth_forward (CPU-tested)
# Gate margins: 16x the worst measured forward error, i.e. 4 tau (tau carries 4x headroom over it).  Exact and fp32
# kernels are gated against the truth (their distance from it: kernel - emulation + emulation - truth), fast mode against
# its emulation.
MU_EXACT = 4 * (TAU_FWD_EXACT + EMUL_EXACT_VS_TRUTH)
MU_FAST = 4 * TAU_FWD_FAST
TAU_BWD_EXACT = 4e-4         # nm_debug_mlp_backward, tensor cores exact: |g - g_ref| <= tau * s [9.9e-5]
TAU_BWD_FP32 = 6e-5          # the same, NM_PREC_FP32 [1.37e-5]
TAU_BWD_FAST = 3.5e-2        # NM_PREC_FAST against the backward at the fast emulation's activations [7.2e-3]
REL_L2_EXACT = 3e-4          # tensor cores exact: relative L2 error per tensor (20x below the ray-level tests' 6e-3)
TAU_GEMM = 1e-4              # nm_debug_gemm bf16x3 against the float64 product (random-walk scale) [2.29e-5]


# ----------------------------------------------------------------------------------------------------- number formats
def f16_rn(x):
    """fp16 round-to-nearest-even of float32 values (overflow -> inf, subnormals kept), as float64."""
    return np.asarray(x, np.float32).astype(np.float16).astype(np.float64)


def f16_sat(x):
    """cvt.rn.satfinite.f16.f32: round to nearest, clamp to +-65504 instead of overflowing."""
    return f16_rn(np.clip(np.asarray(x, np.float32), -F16_MAX, F16_MAX))


def f16_split_sat(a):
    """The kernel's A-operand halves of fp32 values a: hi = sat(a), lo = sat(fp32(a - hi))."""
    a = np.asarray(a, np.float32)
    hi = f16_sat(a)
    lo = f16_sat((a.astype(np.float64) - hi).astype(np.float32))
    return hi, lo


def f16_split_weights(w):
    """nm_program.cu pack_stream: hi = __float2half_rn(w), lo = __float2half_rn(w - hi)."""
    w = np.asarray(w, np.float32)
    hi = f16_rn(w)
    lo = f16_rn((w.astype(np.float64) - hi).astype(np.float32))
    return hi, lo


def bf16_rn(x):
    """bf16 round-to-nearest-even of float32 values, as float64."""
    b = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    b = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    return b.astype(np.uint32).view(np.float32).astype(np.float64)


# ----------------------------------------------------------------------------------------------------- network
@dataclass
class Layer:
    name: str
    k_act: int            # activation columns of the input (0 for layer1)
    pe: Optional[str]     # "xyz" / "dir": the encoding appended as a K block
    relu: bool


def layer_list(cfg: O.NetCfg) -> List[Layer]:
    """The linear layers of FlexibleNeRFModel in evaluation order (the layer program of nm_program.cu build_one)."""
    h = cfg.hidden_size
    out = [Layer("layer1", 0, "xyz", False)]
    for i in range(cfg.num_layers - 1):
        out.append(Layer(f"layers_xyz.{i}", h, "xyz" if i in cfg.skip_layers() else None, True))
    if cfg.use_viewdirs:
        out.append(Layer("fc_feat", h, None, True))
        out.append(Layer("layers_dir.0", h, "dir", True))
    return out


@dataclass
class Record:
    """One forward pass: per layer its input X (the values its product reads), pre-activation z and abs chain A_z; the
    head inputs; outputs out (M,4) = [sigmoid rgb, raw sigma] and their scale A_out."""
    cfg: O.NetCfg
    sd: Dict[str, np.ndarray]
    X: List[np.ndarray] = field(default_factory=list)
    Z: List[np.ndarray] = field(default_factory=list)
    AZ: List[np.ndarray] = field(default_factory=list)
    AX: List[np.ndarray] = field(default_factory=list)   # scale of X's own rounding: [A_z of the layer below | |encoding|]
    trunk: Optional[np.ndarray] = None     # input of fc_alpha / fc_out
    feat_dir: Optional[np.ndarray] = None  # input of fc_rgb
    logits: Optional[np.ndarray] = None    # (M,4): rgb logits, raw sigma
    A_logits: Optional[np.ndarray] = None
    out: Optional[np.ndarray] = None
    A_out: Optional[np.ndarray] = None


def state_f64(sd) -> Dict[str, np.ndarray]:
    return {k: np.asarray(torch.as_tensor(v).detach().cpu().numpy(), np.float64) for k, v in sd.items()
            if k.endswith((".weight", ".bias"))}


def encodings(cfg: O.NetCfg, pts, dirs, dtype=torch.float32):
    """The oracle's encodings computed in `dtype` (default: the fp32 oracle's), as float64 arrays."""
    pts = torch.as_tensor(pts, dtype=dtype)
    ex = O.positional_encoding(pts, cfg.num_encoding_fn_xyz, cfg.include_input_xyz, cfg.log_sampling_xyz)
    ed = None
    if cfg.use_viewdirs:
        d = pts if dirs is None else torch.as_tensor(dirs, dtype=dtype)
        ed = O.positional_encoding(d, cfg.num_encoding_fn_dir, cfg.include_input_dir, cfg.log_sampling_dir)
        ed = ed.numpy().astype(np.float64)
    return ex.numpy().astype(np.float64), ed


def _forward(cfg, sd, pts, dirs, linear, enc_dtype=torch.float32):
    """Walk the network; linear(li, layer, inputs) -> (z, X, output) evaluates one layer on its activation / encoding
    inputs."""
    sd = state_f64(sd)
    ex, ed = encodings(cfg, pts, dirs, enc_dtype)
    rec = Record(cfg, sd)
    x, az = None, None
    layers = layer_list(cfg)
    n_trunk = cfg.num_layers
    for li, L in enumerate(layers):
        pe = None if L.pe is None else (ex if L.pe == "xyz" else ed)
        ax = np.concatenate([np.abs(v) for v in (az, pe) if v is not None], axis=1)
        z, X, x = linear(li, L, [v for v in (x, pe) if v is not None])
        W, b = sd[L.name + ".weight"], sd[L.name + ".bias"]
        az = np.abs(X) @ np.abs(W).T + np.abs(b)
        rec.X.append(X); rec.Z.append(z); rec.AZ.append(az); rec.AX.append(ax)
        if li == n_trunk - 1:
            rec.trunk = x
    M = ex.shape[0]
    logits, A = np.zeros((M, 4)), np.zeros((M, 4))
    if cfg.use_viewdirs:
        rec.feat_dir = x
        wr, br = sd["fc_rgb.weight"], sd["fc_rgb.bias"]
        wa, ba = sd["fc_alpha.weight"], sd["fc_alpha.bias"]
        logits[:, :3] = x @ wr.T + br
        A[:, :3] = np.abs(x) @ np.abs(wr).T + np.abs(br)
        logits[:, 3] = (rec.trunk @ wa.T + ba)[:, 0]
        A[:, 3] = (np.abs(rec.trunk) @ np.abs(wa).T + np.abs(ba))[:, 0]
    else:
        wo, bo = sd["fc_out.weight"], sd["fc_out.bias"]
        logits = rec.trunk @ wo.T + bo
        A = np.abs(rec.trunk) @ np.abs(wo).T + np.abs(bo)
    rec.logits, rec.A_logits = logits, A
    rec.out = np.concatenate([1.0 / (1.0 + np.exp(-logits[:, :3])), logits[:, 3:]], axis=1)
    rec.A_out = np.concatenate([0.25 * A[:, :3], A[:, 3:]], axis=1)      # sigmoid' <= 1/4
    return rec


def truth_forward(cfg: O.NetCfg, sd, pts, dirs=None, enc_dtype=torch.float32) -> Record:
    """float64 FlexibleNeRFModel on the fp32 oracle's encodings (enc_dtype=torch.float64: on float64 ones)."""
    sdd = state_f64(sd)

    def linear(li, L, ins):
        X = np.concatenate(ins, axis=1)
        z = X @ sdd[L.name + ".weight"].T + sdd[L.name + ".bias"]
        return z, X, (np.maximum(z, 0.0) if L.relu else z)
    return _forward(cfg, sd, pts, dirs, linear, enc_dtype)


def emulate_forward(cfg: O.NetCfg, sd, pts, dirs=None, *, fast=False, act_scale_log2=0) -> Record:
    """mlp_tc_kernel mode 0 with exact products (see the module docstring).  X of a layer is the value its A operand
    carries, (hi + lo) * 2^s (fast: hi * 2^s)."""
    sdd = state_f64(sd)
    s = float(2.0 ** act_scale_log2)
    wsplit = {L.name: f16_split_weights(sdd[L.name + ".weight"]) for L in layer_list(cfg)}

    def operand(v):
        hi, lo = f16_split_sat(np.asarray(v, np.float32) / np.float32(s))
        return hi, (np.zeros_like(lo) if fast else lo)

    def linear(li, L, ins):
        parts = [operand(v) for v in ins]
        ah = np.concatenate([p[0] for p in parts], axis=1)
        al = np.concatenate([p[1] for p in parts], axis=1)
        wh, wl = wsplit[L.name]
        acc = ah @ wh.T
        if not fast:
            acc = acc + al @ wh.T + ah @ wl.T
        z = (acc * s + sdd[L.name + ".bias"]).astype(np.float32).astype(np.float64)      # fmaf(acc, 2^s, bias)
        return z, (ah + al) * s, (np.maximum(z, 0.0) if L.relu else z)
    return _forward(cfg, sd, pts, dirs, linear)


# ----------------------------------------------------------------------------------------------------- backward
# The weight gradient reads the forward's activations X, which the kernel itself computed: an activation of small |X|
# next to a large A carries a forward rounding error (<= ~2^-19 A in exact mode) that is large relative to |X|.  The
# scale uses |X| + X_ALLOW * A_X so that this error stays <= 2^-11 of it; for typical entries (A_X ~ 16 |X|) the scale
# grows by a few percent.
X_ALLOW = 2.0 ** -8

def _rw(a, x):
    """random-walk scale sqrt(sum_p (a[p,n] x[p,k])^2) = sqrt((a^2)^T (x^2))."""
    return np.sqrt((a * a).T @ (x * x))


def mlp_backward_ref(rec: Record, dout, dz_out: Optional[dict] = None):
    """float64 gradients of L = sum(dout * logits) for every state-dict tensor of rec's network, evaluated at rec's
    activations and relu gates, and their random-walk scales.  dout (M,4) = [d rgb logits, d raw sigma].  dz_out, if
    given, receives every linear layer's dZ (gradient of its pre-activation) by layer name."""
    cfg, sd = rec.cfg, rec.sd
    dout = np.asarray(dout, np.float64)
    adout = np.abs(dout)
    g, s = {}, {}
    layers = layer_list(cfg)

    def head(name, x, ax, gcol, agcol):
        W = sd[name + ".weight"]
        g[name + ".weight"] = gcol.T @ x
        s[name + ".weight"] = _rw(agcol, np.abs(x) + X_ALLOW * ax)
        g[name + ".bias"] = gcol.sum(0)
        s[name + ".bias"] = np.sqrt((agcol * agcol).sum(0))
        return gcol @ W, agcol @ np.abs(W)

    def linear(li, dx, adx):
        """dx: gradient w.r.t. layer li's output; returns the gradient w.r.t. its activation input (k_act columns)."""
        L = layers[li]
        if L.relu:
            m = rec.Z[li] > 0
            dx, adx = dx * m, adx * m
        if dz_out is not None:
            dz_out[L.name] = dx
        W = sd[L.name + ".weight"]
        g[L.name + ".weight"] = dx.T @ rec.X[li]
        s[L.name + ".weight"] = _rw(adx, np.abs(rec.X[li]) + X_ALLOW * rec.AX[li])
        g[L.name + ".bias"] = dx.sum(0)
        s[L.name + ".bias"] = np.sqrt((adx * adx).sum(0))
        return dx @ W[:, :L.k_act], np.abs(dx) @ np.abs(W[:, :L.k_act])

    last_trunk = cfg.num_layers - 1
    if cfg.use_viewdirs:
        dx, adx = head("fc_rgb", rec.feat_dir, rec.AZ[-1], dout[:, :3], adout[:, :3])
        dx, adx = linear(last_trunk + 2, dx, adx)             # layers_dir.0 -> d fc_feat output
        dx, adx = linear(last_trunk + 1, dx, adx)             # fc_feat -> d trunk
        da, ada = head("fc_alpha", rec.trunk, rec.AZ[last_trunk], dout[:, 3:4], adout[:, 3:4])
        dx, adx = dx + da, adx + ada
    else:
        dx, adx = head("fc_out", rec.trunk, rec.AZ[last_trunk], dout, adout)
    for li in range(last_trunk, -1, -1):
        dx, adx = linear(li, dx, adx)
    return g, s


# ----------------------------------------------------------------------------------------------------- gates, comparators
def gate_margin(rec: Record):
    """per point: min over all relu units of |z| / A_z (inf for a network without relu units)."""
    M = rec.Z[0].shape[0]
    m = np.full(M, np.inf)
    for L, z, az in zip(layer_list(rec.cfg), rec.Z, rec.AZ):
        if L.relu:
            m = np.minimum(m, (np.abs(z) / np.maximum(az, 1e-300)).min(axis=1))
    return m


def filter_dout(dout, rec: Record, mu):
    """dout with the rows of gate-unsafe points (margin < mu) zeroed, and the mask of the rows kept."""
    keep = gate_margin(rec) >= mu
    d = np.array(dout, np.float64, copy=True)
    d[~keep] = 0.0
    return d, keep


def forward_ratio(got, ref, scale):
    """worst |got - ref| / scale (got, ref, scale of the same shape); inf where the scale is 0 and they differ."""
    err = np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64))
    sc = np.asarray(scale, np.float64)
    r = np.where(sc > 0, err / np.where(sc > 0, sc, 1.0), np.where(err > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0


def grad_ratio(got: Dict[str, np.ndarray], ref: Dict[str, np.ndarray], scale: Dict[str, np.ndarray]):
    """per tensor: worst |got - ref| / scale."""
    assert set(got) == set(ref), (sorted(got), sorted(ref))
    return {k: forward_ratio(np.asarray(got[k]).reshape(ref[k].shape), ref[k], scale[k]) for k in ref}


def effective_rel_l2(ref: Dict[str, np.ndarray], scale: Dict[str, np.ndarray], tau):
    """per tensor: the relative L2 error the entrywise bound tau * scale allows, ||tau s|| / ||g_ref||."""
    return {k: float(tau * np.linalg.norm(scale[k]) / max(np.linalg.norm(ref[k]), 1e-300)) for k in ref}
