"""The closed-form compositor adjoint implemented by composite_backward_kernel (csrc/nm_train.cu), as the float64 truth
of tests/_composite_ref.py states it without autograd, checked against autograd through the oracle's VolumeRenderer
(src/nerf/modules.py:67-121) with sigma noise injected into both:
    G_i      = g . c_i  (- sum(g) with a white background)                   dL/dw_i
    dL/da_i  = G_i T_i - (sum_{j>i} G_j w_j) / (1 - a_i + 1e-10)             reverse-cumsum form of cumprod's backward
    dL/ds_i  = dL/da_i * dist_i * exp(-relu(s_i + n_i) dist_i) * [s_i + n_i > 0]
    dL/dc_i  = g w_i                      (the kernel additionally multiplies by c(1-c): the sigmoid of fc_rgb)
CPU only; guards the formula the GPU tests then hold the kernel to."""
import numpy as np
import torch

import _composite_ref as CR
from oracle import nerf_oracle as O


def test_compositor_adjoint_formula_matches_autograd():
    gen = torch.Generator().manual_seed(0)
    R, S = 64, 48
    for white in (False, True):
        for noise_std in (0.0, 0.7):
            raw = torch.cat((torch.rand(R, S, 3, generator=gen), torch.randn(R, S, 1, generator=gen) * 3), -1).double()
            raw[..., 3][:, ::7] = 0.0                                                 # exact zeros: relu' = 0 like torch
            t = torch.sort(torch.rand(R, S, generator=gen) * 4 + 2, -1).values.double()
            dirs = torch.randn(R, 3, generator=gen).double()
            g = torch.randn(R, 3, generator=gen).double()
            noise = torch.from_numpy(CR.sigma_noise(17, R, S, noise_std)).double() if noise_std else torch.zeros(R, S)
            noise[:, ::7] = 0.0                                                       # keep the exact zeros
            leaf = raw.clone().requires_grad_(True)
            b = O.volume_render(leaf, t, dirs, white_background=white, noise=noise)  # float64: the oracle runs in double
            (b.rgb_map * g).sum().backward()
            a = CR.composite_adjoint(raw.numpy(), t.numpy(), dirs.numpy(), g.numpy(), white,
                                     pre=(raw[..., 3] + noise).numpy())
            # the truth's fp32 rules (alpha = 1 once e <= 2^-25, 1e-10f) only matter at saturated samples with a
            # successor; these inputs have none
            assert not (a.e[:, :-1] <= CR.SAT_E).any()
            ref = leaf.grad.numpy()
            scale = np.abs(ref).max()
            assert np.abs(a.drgb - ref[..., :3]).max() <= 1e-9 * scale, (white, noise_std)
            assert np.abs(a.dsig - ref[..., 3]).max() <= 1e-9 * scale, (white, noise_std)
