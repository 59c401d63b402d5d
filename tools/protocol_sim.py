"""Functional model of the weight / operand stage ring both tensor-core kernels use (nm_mlp_tc.cu, nm_gemm_tc.cu), with the
hardware's ONE parity bit per mbarrier wait.

One producer fills a ring of NS stages in a fixed order (full[s]: one arrival per fill, the bulk copies' transaction bytes
completing it; empty[s]: one arrival per consumer warpgroup).  Two consumer warpgroups each take EVERY stage in that order.
A consumer releases a stage only once the wgmmas reading it have completed: it waits for the next stage, issues on it, and
then (wgmma.wait_group 1) releases the previous one; the last stage of a run of blocks is released after wait_group 0.  In
the MLP kernel each warpgroup has its own tiles; when warpgroup 1 has no tile left in a round that warpgroup 0 still runs,
it walks that round's stages as a "ghost" (wait, release) so that both walk the ring the same number of times.

Agents are generators that yield when they would block; a seeded random scheduler runs them until everyone finishes (ok) or
the step budget is spent (deadlock).  Every stage read is checked against what the producer put there, so a stage refilled
before both consumers released it is caught.  Timing is not modelled, only ordering and phase correctness.

    python tools/protocol_sim.py [--tiles 3] [--stages 5]
"""
import argparse
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


class Bar:
    def __init__(self, name, count):
        self.name, self.count, self.pending, self.phase = name, count, count, 0

    def arrive(self):
        self.pending -= 1
        assert self.pending >= 0, f"{self.name}: too many arrivals in phase {self.phase}"
        if self.pending == 0:
            self.phase += 1
            self.pending = self.count

    def done(self, k):            # hardware semantics: try_wait.parity(k & 1) -- ONE parity bit, so a waiter that is two
        return (self.phase & 1) != (k & 1)   # phases away from the barrier's current phase aliases (this is what is modelled)


def run_ring(NS, rounds, runs, own, seed, release_count=2, max_steps=400000):
    """rounds: how many times the producer walks its stage sequence; runs: lengths of the consecutive runs of stages a consumer
    issues before a wait_group 0 (an MLP layer's blocks / a GEMM tile's K blocks), summing to one round; own(wg, r): whether
    warpgroup wg has its own work in round r (else a ghost round).  Returns (ok, info)."""
    per_round = sum(runs)
    full = [Bar(f"full{s}", 1) for s in range(NS)]
    empty = [Bar(f"empty{s}", release_count) for s in range(NS)]
    stage = [None] * NS
    seen = [[], []]
    errors = []

    def wait(bar, k):
        while not bar.done(k):
            yield

    def producer():
        for it in range(rounds * per_round):
            s, ph = it % NS, (it // NS) & 1
            yield from wait(empty[s], ph ^ 1)
            stage[s] = it
            full[s].arrive()
            yield

    def consumer(wg):
        it = 0
        for r in range(rounds):
            real = own(wg, r)
            for n in runs:
                prev = None
                for _ in range(n):
                    s = it % NS
                    yield from wait(full[s], it // NS)
                    if stage[s] != it:
                        errors.append(f"warpgroup {wg} expected stage content {it}, slot {s} holds {stage[s]}")
                    seen[wg].append(it)
                    yield
                    if not real:                   # ghost: hand the stage straight back
                        empty[s].arrive()
                    else:                          # wait_group 1: the previous stage's wgmmas are complete
                        if prev is not None:
                            empty[prev].arrive()
                        prev = s
                    it += 1
                if real and prev is not None:      # wait_group 0 at the end of the run
                    empty[prev].arrive()
                yield

    agents = [producer(), consumer(0), consumer(1)]
    rng = random.Random(seed)
    alive = list(range(len(agents)))
    try:
        for _ in range(max_steps):
            if not alive:
                break
            a = rng.choice(alive)
            try:
                next(agents[a])
            except StopIteration:
                alive.remove(a)
    except AssertionError as e:
        return False, str(e)
    if alive:
        return False, f"deadlock: agents left {alive}"
    if errors:
        return False, errors[0]
    want = list(range(rounds * per_round))
    if seen[0] != want or seen[1] != want:
        return False, "a consumer skipped or repeated a stage"
    return True, "ok"


def layer_runs(prog):
    """Blocks per layer of an MLP layer program (layers without blocks issue nothing)."""
    return [prog.layers[i].blk_end - prog.layers[i].blk_begin for i in range(prog.n_layers)
            if prog.layers[i].blk_end > prog.layers[i].blk_begin]


def simulate(prog, tiles, NS, seeds=(0, 1, 2), release_count=2, runs=None):
    """The MLP kernel on one CTA processing `tiles` 64-point tiles: warpgroup 0 takes tiles 0, 2, 4, ..., warpgroup 1 tiles
    1, 3, ...; rounds = ceil(tiles / 2), warpgroup 1 ghosts the last round when tiles is odd.  runs: stages per layer (as
    run_ring takes them), by default the layer program's block runs (layer_runs)."""
    rounds = (tiles + 1) // 2
    own = lambda wg, r: 2 * r + wg < tiles
    for seed in seeds:
        ok, info = run_ring(NS, rounds, layer_runs(prog) if runs is None else runs, own, seed, release_count)
        if not ok:
            return False, f"seed {seed}: {info}"
    return True, "ok"


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, default=3)
    ap.add_argument("--stages", type=int, default=5)
    a = ap.parse_args()
    from oracle import nerf_oracle as O
    from test_host_logic import debug_pack
    cfg = O.NetCfg()
    prog, _ = debug_pack(cfg, O.init_weights(cfg, 1))
    print(simulate(prog, a.tiles, a.stages))
