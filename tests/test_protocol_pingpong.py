"""CPU test of the fused MLP kernel's ping-pong weight stream (nm_mlp_tc.cu): the two consumer warpgroups take turns on
the ring, each stage filled for one owner that alone waits for it (its own full barrier) and releases it (empty barrier
count 1).  The functional model in tools/protocol_sim.py (run_pingpong) replays the producer and both warpgroups with the
hardware's ONE-bit mbarrier parity on the stage runs the kernel walks: free of deadlock and of early refills for every
ring depth, tile count and tile grouping, and a broken variant (one full barrier for both warpgroups) is rejected.  The
same holds for the CTA-pair variant that shares each stage by multicast (measured slower and not shipped, DESIGN 4.1),
whose model must catch rank 0 refilling a slot after only its own CTA has released it."""
import os
import sys

import pytest

from conftest import ROOT
from oracle import nerf_oracle as O

sys.path.insert(0, os.path.join(ROOT, "tools"))
from protocol_sim import simulate_pingpong  # noqa: E402
from test_host_logic import debug_pack  # noqa: E402
from test_wide_stream import wide_runs  # noqa: E402

ARCHS = [dict(), dict(num_layers=4, hidden_size=128, num_encoding_fn_xyz=6),
         dict(num_layers=3, hidden_size=128, use_viewdirs=False),
         dict(num_layers=6, hidden_size=256, skip_step=2, num_encoding_fn_xyz=8)]


def _runs(arch, sigma_only, fast):
    cfg = O.NetCfg(**{**O.NetCfg().__dict__, **arch})
    prog, _ = debug_pack(cfg, O.init_weights(cfg, 1), sigma_only)
    return wide_runs(prog, fast)


@pytest.mark.parametrize("arch", ARCHS)
@pytest.mark.parametrize("sigma_only", [False, True])
@pytest.mark.parametrize("fast", [False, True])
def test_pingpong_stream_is_deadlock_free(arch, sigma_only, fast):
    """Every ring depth 2-8: 1 tile (warpgroup 1 never runs), odd counts (it sits out the last round) and even ones."""
    runs = _runs(arch, sigma_only, fast)
    for ns in range(2, 9):
        for tiles in (1, 2, 3, 5, 6):
            ok, info = simulate_pingpong(runs, tiles, ns)
            assert ok, (ns, tiles, info)


@pytest.mark.parametrize("tile_group", [1, 3])
def test_pingpong_tile_groups_and_short_layers(tile_group):
    """The fused compositor deals groups of tile_group consecutive tiles (3 at 192 samples per ray), so a warpgroup can
    sit out several final rounds; with partial last groups, layers shorter than the ring and a layer with no stages, for
    the kernel (one CTA) and the CTA-pair variant (unequal tile counts across the pair, ghost rounds in rank 1)."""
    for runs in ([1], [1, 1, 1], [2, 0, 3, 1], [7, 1, 2]):
        for ns in (2, 3, 4, 7):
            for tiles in (1, 2, 4, 5, 7, 10, 13):
                for ctas in (1, 2):
                    ok, info = simulate_pingpong(runs, tiles, ns, seeds=range(3), ctas=ctas, tile_group=tile_group)
                    assert ok, (runs, ns, tiles, ctas, info)


def test_model_catches_one_full_barrier_for_both_warpgroups():
    """With one full barrier per slot, a warpgroup that skips the other's turn waits on a parity that aliases a phase it
    never observed: the model must fail (an early read or a hang)."""
    runs = _runs(dict(), False, False)
    for ns in (2, 3, 5):
        ok, _ = simulate_pingpong(runs, 4, ns, seeds=range(4), shared_full=True)
        assert not ok, ns


def test_model_catches_a_refill_after_one_cta():
    """CTA-pair variant: rank 0 refilling a slot once its own CTA has released it (empty count 1), without waiting for
    the peer CTA: the model must fail."""
    runs = _runs(dict(), False, False)
    for ns in (2, 3, 5):
        ok, _ = simulate_pingpong(runs, 8, ns, seeds=range(4), ctas=2, release_count=1)
        assert not ok, ns
