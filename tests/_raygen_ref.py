"""Restatements of ray generation and NDC (nm_render.cu raygen_kernel / ndc_warp) in numpy fp32, in the kernels' written
order — test infrastructure, no GPU.  The translation unit is built with -fmad=false and uses only IEEE + - * / and sqrt,
so the restatements match the kernels bit for bit.

* `raygen32`: pixel (r, c) of rows [row0, row1) -> x = (f32(c) - f32(W 0.5)) / f32(focal), y = -((f32(r) - f32(H 0.5)) /
  f32(focal)), z = -1; n = sqrt((x x + y y) + z z); x, y, z each divided by n; d_j = (x P[j,0] + y P[j,1]) + z P[j,2];
  o = P[:, 3].
* `ndc32`: ndc_rays (src/nerf/nerf_helpers.py:280-307).  The scalars sx = -1 / (W / (2 focal)), sy likewise, 2 near and
  -2 near are formed in double from the caller's unrounded focal and near and rounded once to fp32, as torch rounds a
  python-scalar operand.  `2 near / o_z` divides a python scalar by a tensor, which torch evaluates as reciprocal(o_z) *
  scalar (Tensor.__rtruediv__); every other division is tensor / tensor, a true division.  With these two rules the
  restatement equals oracle.nerf_oracle.ndc_rays bit for bit (tests/test_raygen_reference.py).
* `ray_truth`: the float64 pixel ray from the fp32 inputs (pose, f32(focal)), and its per-component scale
  scale_j = sum_k |v_k| |P[j,k]| with v the normalised camera vector.  The fp32 direction in the written order carries
  about 7 u scale_j to first order (u = 2^-24): x, y one rounding each, the three squares and two sums, the sqrt, the
  normalising division, the three products and two sums of the rotation.  TAU_RAY = 8 bounds it; torch's own
  get_ray_bundle (another association of the norm) meets the same bound.

`RAYGEN_FAULTS` / `NDC_FAULTS` name variants that each carry one plausible bug; the CPU tests show that the float64 bound
(raygen) or the bitwise oracle comparison (NDC) flags every one of them.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
U = 2.0 ** -24
TAU_RAY = 8.0
RAYGEN_FAULTS = ("half_pixel", "transpose", "flip_y")
NDC_FAULTS = ("f32_scalars", "true_div")


def pose34(pose) -> np.ndarray:
    """The 3x4 camera-to-world matrix as the engine uploads it: fp32, pose[:3, :4]."""
    return np.ascontiguousarray(np.asarray(pose, dtype=np.float32)[:3, :4])


def raygen32(pose, H, W, focal, row0=0, row1=None, fault=None):
    """raygen_kernel without NDC: (origin (3,), dirs (row1-row0, W, 3)), fp32."""
    P = pose34(pose)
    if fault == "transpose":
        P = P.copy()
        P[:, :3] = P[:, :3].T
    row1 = H if row1 is None else row1
    c = np.arange(W, dtype=np.float64).astype(F32)[None, :]
    r = np.arange(row0, row1, dtype=np.float64).astype(F32)[:, None]
    if fault == "half_pixel":
        c, r = c + F32(0.5), r + F32(0.5)
    f, hw, hh = F32(focal), F32(W * 0.5), F32(H * 0.5)
    x = np.broadcast_to((c - hw) / f, (row1 - row0, W))
    y = np.broadcast_to(-((r - hh) / f), (row1 - row0, W))
    if fault == "flip_y":
        y = -y
    z = F32(-1.0)
    n = np.sqrt((x * x + y * y) + z * z)
    x, y, z = x / n, y / n, z / n
    d = np.empty((row1 - row0, W, 3), F32)
    for j in range(3):
        d[..., j] = (x * P[j, 0] + y * P[j, 1]) + z * P[j, 2]
    return P[:, 3].copy(), d


def ndc_scalars(H, W, focal, near, fault=None):
    if fault == "f32_scalars":
        focal, near = float(F32(focal)), float(F32(near))
    return (F32(near), F32(-1.0 / (W / (2.0 * focal))), F32(-1.0 / (H / (2.0 * focal))), F32(2.0 * near), F32(-2.0 * near))


def ndc32(H, W, focal, near, o, d, fault=None):
    """ndc_warp on rays o (3,) or (..., 3) and d (..., 3): (origins, dirs), both shaped like d, fp32."""
    nf, sx, sy, two, neg_two = ndc_scalars(H, W, focal, near, fault)
    d = np.asarray(d, F32)
    o = np.broadcast_to(np.asarray(o, F32), d.shape)
    with np.errstate(all="ignore"):
        t = -(nf + o[..., 2]) / d[..., 2]
        o = o + t[..., None] * d
        if fault == "true_div":
            o2, d2 = F32(1.0) + two / o[..., 2], neg_two / o[..., 2]
        else:
            rz = F32(1.0) / o[..., 2]
            o2, d2 = F32(1.0) + rz * two, rz * neg_two
        o0 = sx * o[..., 0] / o[..., 2]
        o1 = sy * o[..., 1] / o[..., 2]
        d0 = sx * (d[..., 0] / d[..., 2] - o[..., 0] / o[..., 2])
        d1 = sy * (d[..., 1] / d[..., 2] - o[..., 1] / o[..., 2])
    return np.stack([o0, o1, o2], -1).astype(F32), np.stack([d0, d1, d2], -1).astype(F32)


def ray_truth(pose, H, W, focal, row0=0, row1=None):
    """float64 directions (rows, W, 3) from the fp32 pose and f32(focal), and scale (rows, W, 3)."""
    P = pose34(pose).astype(np.float64)
    row1 = H if row1 is None else row1
    f = float(F32(focal))
    c = np.arange(W, dtype=np.float64)[None, :]
    r = np.arange(row0, row1, dtype=np.float64)[:, None]
    x = np.broadcast_to((c - W * 0.5) / f, (row1 - row0, W))
    y = np.broadcast_to(-(r - H * 0.5) / f, (row1 - row0, W))
    v = np.stack([x, y, -np.ones_like(x)], -1)
    v = v / np.sqrt((v * v).sum(-1, keepdims=True))
    return v @ P[:, :3].T, np.abs(v) @ np.abs(P[:, :3]).T


def ray_error_ratio(d32, pose, H, W, focal, row0=0, row1=None):
    """max over components of |d32 - d64| / (u scale); 0 where both are exactly equal (scale 0 included)."""
    d64, scale = ray_truth(pose, H, W, focal, row0, row1)
    err = np.abs(np.asarray(d32, np.float64) - d64)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(err == 0, 0.0, err / (U * scale))
    return float(q.max()) if q.size else 0.0
