"""CPU test of the fused MLP kernel's synchronisation protocol (nm_mlp_tc.cu): the functional model in tools/protocol_sim.py
replays the producer and the two consumer warpgroups on the real layer program, with the hardware's ONE-bit mbarrier parity
semantics: the ring is free of deadlock and of premature stage refills for every ring depth, and the model catches the
refill that a release after only one warpgroup would allow."""
import os
import sys

import pytest

from conftest import ROOT
from oracle import nerf_oracle as O

sys.path.insert(0, os.path.join(ROOT, "tools"))
from protocol_sim import simulate  # noqa: E402
from test_host_logic import debug_pack  # noqa: E402


@pytest.mark.parametrize("arch", [dict(), dict(num_layers=4, hidden_size=128, num_encoding_fn_xyz=6),
                                  dict(num_layers=3, hidden_size=128, use_viewdirs=False),
                                  dict(num_layers=6, hidden_size=256, skip_step=2, num_encoding_fn_xyz=8)])
@pytest.mark.parametrize("sigma_only", [False, True])
def test_protocol_is_deadlock_free(arch, sigma_only):
    cfg = O.NetCfg(**{**O.NetCfg().__dict__, **arch})
    prog, _ = debug_pack(cfg, O.init_weights(cfg, 1), sigma_only)
    for ns in (2, 3, 4, 5, 8):
        ok, info = simulate(prog, tiles=4, NS=ns)
        assert ok, (ns, info)


def test_simulator_catches_parity_aliasing():
    """A stage released as soon as ONE warpgroup is done (empty barrier count 1): the producer refills it, and on the one-bit
    parity the slower warpgroup reads the next round's contents."""
    cfg = O.NetCfg()
    prog, _ = debug_pack(cfg, O.init_weights(cfg, 1))
    ok, _ = simulate(prog, tiles=4, NS=3, seeds=range(8), release_count=1)
    assert not ok


@pytest.mark.parametrize("arch", [dict(), dict(num_layers=4, hidden_size=128, num_encoding_fn_xyz=6)])
def test_cta_pair_sharing_one_weight_stream_is_deadlock_free(arch):
    """The two consumer warpgroups of a CTA share ONE weight stream: every stage is released by both (empty count 2); with and
    without warpgroup 1's ghost round (odd / even tile counts), for every ring depth."""
    cfg = O.NetCfg(**{**O.NetCfg().__dict__, **arch})
    for sigma_only in (False, True):
        prog, _ = debug_pack(cfg, O.init_weights(cfg, 1), sigma_only)
        for ns in (2, 3, 5, 7):
            for tiles in (1, 2, 3, 5):
                ok, info = simulate(prog, tiles=tiles, NS=ns)
                assert ok, (ns, tiles, info)
