"""The references of the forward compositor (tests/_composite_ref.py) on the CPU: the float64 truth has the semantics of
oracle.volume_render run in float64 on every ray kind but `nan_sigma` (the one documented deviation), the fp32 emulation of
composite_kernel stays within EMUL_WORST_FWD of the truth over the edge matrix of tests/test_gpu_composite_forward.py,
every fault variant exceeds TAU_FWD there, and the ray kinds reach the edges they are named after."""
import numpy as np
import pytest
import torch

import _composite_ref as CR
from oracle import nerf_oracle as O
from test_composite_adjoint import NOISE, S_ALL

THRS = (1e-5, 0.0, 1.0, -1.0)
K = {n: i for i, n in enumerate(CR.FWD_KINDS)}


def _cases(R=28):
    for S in S_ALL:
        for j, (white, training) in enumerate(((0, 0), (1, 0), (0, 1), (1, 1))):
            std, seed = NOISE[(S + j) % 3]
            for thr in THRS:
                yield S, white, training, std, seed, thr, CR.make_forward_rays(R, S, 1000 * S + 10 * j, kind_offset=S + j)


def test_truth_equals_float64_oracle_except_nan_sigma():
    for S in (1, 2, 33, 64, 257):
        raw, t, d, kinds = CR.make_forward_rays(56, S, 17 * S, kind_offset=S)
        for white in (0, 1):
            for training in (0, 1):
                for thr in (1e-5, 0.0):
                    f = CR.composite_forward(raw, t, d, white, training, thr)
                    b = O.volume_render(torch.from_numpy(raw).double(), torch.from_numpy(t).double(), torch.from_numpy(d).double(),
                                        white_background=bool(white), training=bool(training), attenuation_threshold=thr)
                    ref = dict(rgb=b.rgb_map, depth=b.depth_map, depth_raw=b.depth_raw, acc=b.acc_map, disp=b.disp_map,
                               weights=b.weights, mask_weights=b.mask_weights)
                    keep = kinds != K["nan_sigma"]
                    # the truth's fp32 rules (alpha = 1 once e <= 2^-25, 1e-10f) move T after a saturated sample by < 4e-8
                    # of its value before it: differences far below these bars; a different rule is O(1) off somewhere
                    und = np.abs(f.out["acc"] - 1.0) <= 1e-7                 # acc < 1 may go either way between the two
                    for k, v in ref.items():
                        v = v.numpy()
                        a = f.out[k]
                        if k == "depth":
                            a, v = a[~und & keep], v[~und & keep]
                        elif k == "mask_weights":          # float64 T underflows after ~31 saturated samples
                            sel = keep[:, None] & ~(f.T < 1e-290)
                            a, v = a[sel], v[sel]
                        else:
                            a, v = a[keep], v[keep]
                        same_nan = np.isnan(a) == np.isnan(v)
                        assert same_nan.all(), (S, k, white, training)
                        fin = np.isfinite(v) & np.isfinite(a)
                        assert (a[~fin & ~np.isnan(a)] == v[~fin & ~np.isnan(v)]).all(), (S, k)
                        tol = 1e-6 * np.maximum(1.0, np.abs(v[fin])) * (1.0 if k not in ("depth", "depth_raw") else 6.0)
                        assert (np.abs(a[fin] - v[fin]) <= tol).all(), (S, k, white, training, thr, float(np.abs(a[fin] - v[fin]).max()))
    # nan_sigma: the oracle propagates the NaN into every output of the ray; the truth maps it to alpha = 0
    raw, t, d, kinds = CR.make_forward_rays(14, 40, 3)
    r = K["nan_sigma"]
    b = O.volume_render(torch.from_numpy(raw).double(), torch.from_numpy(t).double(), torch.from_numpy(d).double())
    f = CR.composite_forward(raw, t, d, 0, 0, 1e-5)
    assert torch.isnan(b.rgb_map[r]).all() and np.isfinite(f.out["rgb"][r]).all() and (f.w[r, ::3] == 0).all()


def test_emulation_within_tau_of_truth():
    worst, at = 0.0, None
    for S, white, training, std, seed, thr, (raw, t, d, kinds) in _cases():
        f = CR.composite_forward(raw, t, d, white, training, thr, std, seed)
        sc = CR.forward_error_scale(f, raw, t, white)
        em = CR.emulate_forward(raw, t, d, white, training, thr, std, seed)
        for k in CR.FWD_OUT:
            r = CR.forward_ratio(em[k], f.out[k], sc[k])
            assert r.max() <= CR.EMUL_WORST_FWD, (S, white, training, std, thr, k, float(r.max()))
            if r.max() > worst:
                i = np.unravel_index(r.argmax(), r.shape)
                worst, at = float(r.max()), (S, k, CR.FWD_KINDS[kinds[i[0]]])
    print(f"RATIO forward emulation-vs-truth {worst:.3e} at {at}")
    assert CR.EMUL_WORST_FWD <= CR.TAU_FWD


def test_every_fault_is_flagged_at_tau():
    worst = {f: 0.0 for f in CR.FWD_FAULTS}
    for S, white, training, std, seed, thr, (raw, t, d, _) in _cases(R=14):
        f = CR.composite_forward(raw, t, d, white, training, thr, std, seed)
        sc = CR.forward_error_scale(f, raw, t, white)
        for fault in CR.FWD_FAULTS:
            if worst[fault] <= 100 * CR.TAU_FWD:
                em = CR.emulate_forward(raw, t, d, white, training, thr, std, seed, fault=fault)
                worst[fault] = max(worst[fault], max(float(CR.forward_ratio(em[k], f.out[k], sc[k]).max()) for k in CR.FWD_OUT))
    for fault, v in worst.items():
        print(f"RATIO forward fault {fault} {v:.3e}")
    missed = {fault: v for fault, v in worst.items() if not v > 100 * CR.TAU_FWD}
    assert not missed, missed


@pytest.mark.parametrize("S", [1, 64, 257])
def test_forward_ray_kinds_reach_their_edges(S):
    raw, t, d, kinds = CR.make_forward_rays(56, S, 5)
    f = CR.composite_forward(raw, t, d, 0, 0, 1e-5)
    em = CR.emulate_forward(raw, t, d, 0, 0, 1e-5)
    rows = lambda name: kinds == K[name]
    o = f.out
    e = rows("empty")
    assert (o["acc"][e] == 0).all() and (em["acc"][e] == 0).all() and (em["disp"][e] == 0).all() and (em["rgb"][e] == 0).all()
    a1 = em["acc"][rows("acc_one")]
    assert (np.abs(a1.astype(np.float64) - 1.0) <= 16 * 2.0 ** -24).all() and (a1 < 1).any() and (a1 >= 1).any()
    assert (em["disp"][rows("behind")] == np.float32(1e10)).all() and (o["depth_raw"][rows("behind")] < 0).all()
    ratio = o["depth_raw"][rows("tiny_ratio")] / o["acc"][rows("tiny_ratio")]
    assert ((ratio > 0) & (ratio < 1e-10)).all() and (em["disp"][rows("tiny_ratio")] == np.float32(1e10)).all()
    ov = rows("overflow")
    assert np.isinf(o["depth_raw"][ov]).any() and (em["disp"][ov][np.isinf(em["depth_raw"][ov])] == 0).all()
    if S > 1:
        assert np.isnan(o["acc"][ov]).any() and np.isnan(em["acc"][ov]).any()
    z = rows("zero_dir")
    assert (em["acc"][z] == 0).all() and (em["weights"][z] == 0).all()
    n = rows("nan_sigma")
    assert np.isnan(raw[n, ::3, 3]).all() and np.isfinite(em["rgb"][n]).all() and (em["weights"][n][:, ::3] == 0).all()
    if S > 4:
        T32 = np.cumprod(np.concatenate([np.ones((1,)), f.keep[kinds == K["subnormal_T"]][0, :-1]])).astype(np.float32)
        assert ((T32 > 0) & (T32 < np.finfo(np.float32).tiny)).any() and (T32 == 0).any()
        m = o["mask_weights"]
        assert (m == 1).any() and (m == 0).any()
    # T == thr decided: thr = 1 against the exact T = 1 of sample 0 and of the samples after gated ones (empty rays);
    # the strict rule gives 0 there, a `>=` slip 1
    f1 = CR.composite_forward(raw, t, d, 0, 0, 1.0)
    sc = CR.forward_error_scale(f1, raw, t, 0)["mask_weights"]
    tie = (f1.T == 1.0) & (sc == 0)
    assert tie[:, 0].all() and tie[rows("empty")].all() and (f1.out["mask_weights"][tie] == 0).all()
    assert (CR.emulate_forward(raw, t, d, 0, 0, 1.0)["mask_weights"][tie] == 0).all()
    assert (CR.emulate_forward(raw, t, d, 0, 0, 1.0, fault="mask_ge")["mask_weights"][tie] == 1).all()
