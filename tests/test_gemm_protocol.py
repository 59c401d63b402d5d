"""Functional model of tc_gemm_kernel's mbarrier protocol (nm_gemm_tc.cu): one producer fills the stage ring full[s] /
empty[s] with the K blocks of the CTA's one tile (its K split); the two consumer warpgroups (rows 0-63 / 64-127 of the tile)
each take every stage in order, release a stage once their wgmmas on it have completed, and run the epilogue from their
registers after the last K block.  Modelled by tools/protocol_sim.run_ring with the hardware's ONE parity bit per wait:
every schedule finishes (no deadlock, no arrival overflow) and each warpgroup reads exactly the K blocks the producer
loaded, in order."""
import itertools
import os
import sys

from conftest import ROOT

sys.path.insert(0, os.path.join(ROOT, "tools"))
from protocol_sim import run_ring  # noqa: E402


def test_split_k_row_sum_readers_share_the_stage_ring():
    """The split-K (weight-gradient) variant with a_rowsum: one tile per CTA; each consumer warpgroup sums the rows of its half
    of the staged A tile before it releases the stage, so a stage is refilled only after both have read it."""
    for NS, nk in itertools.product((2, 3), (1, 2, 3, 4, 7, 9, 16)):
        for seed in range(3):
            ok, info = run_ring(NS, 1, [nk], lambda wg, r: True, seed)
            assert ok, (NS, nk, seed, info)
