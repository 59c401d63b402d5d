"""CPU test of the fused MLP kernel's shared-memory layout (nm_mlp_tc.cu mlp_tc_layout, the function its launches use): on an
H100's 232,448-byte opt-in limit the lego network's full and sigma-only inference programs get four 16 KB weight-ring
slots, with the compositor on or off, and the training modes, which keep the bias and head vectors in shared memory, three;
a slot cap only lowers the depth; every region is in bounds and the ring stays 1024-byte aligned; and a limit that leaves
room for fewer than two slots is an error."""
import ctypes as C

import numpy as np
import pytest

from nerfmeshes_b200 import _lib as L
from oracle import nerf_oracle as O
from test_host_logic import debug_pack

H100_OPTIN = 232448
STAGE = 16384
WG_BYTES = 2 * (4 * 16384 + 16384)          # two warpgroups: activation (4 K-blocks) + encoding buffer, hi | lo


def layout(prog, max_smem, comp_on, cap=0, training=False):
    out = (C.c_int64 * 5)()
    L.check(L.load().nm_debug_mlp_layout(C.byref(prog), C.sizeof(prog), max_smem, int(comp_on), int(training), cap, out))
    return dict(zip(("slots", "off_wg", "off_bars", "off_carry", "bytes"), list(out)))


def _prog(sigma_only, **arch):
    cfg = O.NetCfg(**{**O.NetCfg().__dict__, **arch})
    return debug_pack(cfg, O.init_weights(cfg, 1), sigma_only)[0]


@pytest.mark.parametrize("sigma_only", [False, True])
@pytest.mark.parametrize("comp_on", [False, True])
def test_lego_gets_four_slots(sigma_only, comp_on):
    lay = layout(_prog(sigma_only), H100_OPTIN, comp_on)
    assert lay["slots"] == 4, lay
    assert lay["off_wg"] == 4 * STAGE and lay["off_wg"] % 1024 == 0
    assert lay["off_bars"] == lay["off_wg"] + WG_BYTES and lay["off_bars"] % 8 == 0
    assert lay["off_carry"] >= lay["off_bars"] and lay["off_carry"] % 16 == 0
    assert lay["bytes"] - lay["off_carry"] == (128 if comp_on else 0)
    assert lay["bytes"] <= H100_OPTIN


def test_slot_cap_only_lowers_the_depth():
    prog = _prog(False)
    assert [layout(prog, H100_OPTIN, True, cap)["slots"] for cap in (0, 1, 2, 3, 4, 5, 8)] == [4, 2, 2, 3, 4, 4, 4]
    big = layout(prog, 1 << 20, True)             # a larger limit: the ring stops at its eight barriers
    assert big["slots"] == 8


def test_training_keeps_its_vectors_in_shared_memory():
    lay = layout(_prog(False), H100_OPTIN, False, training=True)
    vectors = lay["off_bars"] - lay["off_wg"] - WG_BYTES        # 9,728 B of bias and ~2.6 KB of head, each 16-byte aligned
    assert lay["slots"] == 3 and 9728 + 2576 <= vectors < 9728 + 2576 + 32, lay
    assert lay["bytes"] <= H100_OPTIN


def test_inference_layout_is_the_same_for_every_network():
    """Inference reads the bias and head vectors from global memory, so its layout does not grow with the network."""
    a = layout(_prog(False), H100_OPTIN, True)
    b = layout(_prog(False, num_layers=4, hidden_size=128, num_encoding_fn_xyz=6), H100_OPTIN, True)
    assert a == b


def test_too_small_a_limit_is_an_error():
    prog = _prog(False)
    lim = WG_BYTES + 2 * STAGE + 192 + 128
    assert layout(prog, lim, True)["slots"] == 2
    with pytest.raises(L.NmError, match="shared-memory budget"):
        layout(prog, lim - 1, True)
    with pytest.raises(L.NmError, match="shared-memory budget"):
        layout(prog, 100000, False)
