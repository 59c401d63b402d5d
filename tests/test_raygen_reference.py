"""Ray generation and NDC restated in numpy fp32 (tests/_raygen_ref.py) against the CPU oracle and a float64 truth — no GPU.

* ndc32 == oracle.nerf_oracle.ndc_rays bit for bit over image sizes 12x10, 37x53, 756x1008 (the fern benchmark), 800x800
  (the lego benchmark) and 5x1; focal 13.5, 41.3, 815.13, 1111.1111, 815.0, 0.37; near 1.0, 0.5, 0.3, 2.7; two
  pose_spherical poses and the identity.
* raygen32 and the oracle's get_ray_bundle both lie within TAU_RAY u scale of the float64 pixel ray.  They are not compared
  bitwise: torch's CPU norm associates the three squares differently (fused multiply-adds), so a fraction of a percent of
  the components differ by an ulp; the test prints that fraction.
* Every fault variant is flagged: NDC scalars formed from float-rounded focal / near (the fern camera), a true division for
  2 near / o_z (near 0.3), pixel centres moved by half a pixel, the rotation transposed, the sign of y flipped.
"""
import numpy as np
import pytest
import torch

import _raygen_ref as RR
from oracle import nerf_oracle as O

POSES = {"spherical_30": O.pose_spherical(30.0, -30.0, 4.0), "spherical_m150": O.pose_spherical(-150.0, -30.0, 4.0),
         "identity": torch.eye(4)}
SHAPES = [(12, 10), (37, 53), (756, 1008), (800, 800), (5, 1)]
FOCALS = [13.5, 41.3, 815.13, 1111.1111, 815.0, 0.37]
NEARS = [1.0, 0.5, 0.3, 2.7]


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _n_bits_differ(a, b):
    return int((np.asarray(a, np.float32).view(np.uint32) != np.asarray(b, np.float32).view(np.uint32)).sum())


@pytest.mark.parametrize("H,W", SHAPES)
def test_ndc_restatement_equals_oracle_bit_for_bit(H, W):
    for pname, pose in POSES.items():
        for f in FOCALS:
            o, d = O.get_ray_bundle(H, W, f, pose)
            for near in NEARS:
                ro, rd = O.ndc_rays(H, W, f, near, o.expand(d.shape), d)
                eo, ed = RR.ndc32(H, W, f, near, o.numpy(), d.numpy())
                assert _bits_equal(eo, ro.numpy()) and _bits_equal(ed, rd.numpy()), \
                    (pname, H, W, f, near, _n_bits_differ(eo, ro.numpy()), _n_bits_differ(ed, rd.numpy()))


@pytest.mark.parametrize("H,W", SHAPES)
def test_raygen_restatement_and_oracle_within_float64_bound(H, W):
    worst, differ, total = 0.0, 0, 0
    for pname, pose in POSES.items():
        for f in FOCALS:
            o32, d32 = RR.raygen32(pose, H, W, f)
            o, d = O.get_ray_bundle(H, W, f, pose)
            assert _bits_equal(o32, o.numpy())
            q32 = RR.ray_error_ratio(d32, pose, H, W, f)
            qo = RR.ray_error_ratio(d.numpy(), pose, H, W, f)
            assert q32 <= RR.TAU_RAY and qo <= RR.TAU_RAY, (pname, H, W, f, q32, qo)
            worst = max(worst, q32, qo)
            differ += _n_bits_differ(d32, d.numpy())
            total += d32.size
            # a row shard is the same rays as the rows of the whole image
            if H > 2:
                _, ds = RR.raygen32(pose, H, W, f, 1, H - 1)
                assert _bits_equal(ds, d32[1:H - 1])
    print(f"{H}x{W}: worst error {worst:.3f} u scale (TAU_RAY {RR.TAU_RAY}); "
          f"{differ} of {total} direction components differ from get_ray_bundle ({differ / total:.4%})")


def test_ray_truth_is_the_reference_formula_in_float64():
    pose = POSES["spherical_30"].double()
    H, W, f = 12, 10, 13.5
    o, d = O.get_ray_bundle(H, W, f, pose)
    d64, scale = RR.ray_truth(pose, H, W, f)
    assert np.abs(d64 - d.numpy()).max() < 1e-14 and bool((scale > 0).all())


def test_ndc_faults_are_flagged():
    pose = POSES["spherical_30"]
    # the fern benchmark's camera: fp32-rounded focal moves sx by an ulp and a large share of the components with it
    H, W, f = 756, 1008, 815.13
    o, d = O.get_ray_bundle(H, W, f, pose)
    ro, rd = O.ndc_rays(H, W, f, 1.0, o.expand(d.shape), d)
    fo, fd = RR.ndc32(H, W, f, 1.0, o.numpy(), d.numpy(), fault="f32_scalars")
    n = _n_bits_differ(fo, ro.numpy()) + _n_bits_differ(fd, rd.numpy())
    assert n > 0.2 * fo.size * 2, n
    # near 0.3: 2 near is not a power of two, so a true division differs from torch's reciprocal-times-scalar
    for H, W, f in [(37, 53, 41.3), (800, 800, 1111.1111)]:
        o, d = O.get_ray_bundle(H, W, f, pose)
        ro, rd = O.ndc_rays(H, W, f, 0.3, o.expand(d.shape), d)
        to, td = RR.ndc32(H, W, f, 0.3, o.numpy(), d.numpy(), fault="true_div")
        assert _n_bits_differ(to, ro.numpy()) + _n_bits_differ(td, rd.numpy()) > 0


@pytest.mark.parametrize("fault", RR.RAYGEN_FAULTS)
def test_raygen_faults_exceed_the_bound(fault):
    for pname in ("spherical_30", "spherical_m150"):
        pose = POSES[pname]
        for H, W, f in [(12, 10, 13.5), (37, 53, 41.3), (756, 1008, 815.13)]:
            _, d = RR.raygen32(pose, H, W, f, fault=fault)
            q = RR.ray_error_ratio(d, pose, H, W, f)
            assert q > 100 * RR.TAU_RAY, (fault, pname, H, W, f, q)
