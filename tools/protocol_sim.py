"""Functional model of the weight / operand stage ring both tensor-core kernels use (nm_mlp_tc.cu, nm_gemm_tc.cu), with the
hardware's ONE parity bit per mbarrier wait.

run_ring / simulate: the shared stream of the GEMM kernel (and of the MLP kernel before its ping-pong stream).  One producer
fills a ring of NS stages in a fixed order (full[s]: one arrival per fill, the bulk copies' transaction bytes completing
it; empty[s]: one arrival per consumer warpgroup).  Two consumer warpgroups each take EVERY stage in that order.  A
consumer releases a stage only once the wgmmas reading it have completed: it waits for the next stage, issues on it, and
then (wgmma.wait_group 1) releases the previous one; the last stage of a run of blocks is released after wait_group 0.
With per-warpgroup work (simulate), a warpgroup without work in a round walks its stages as a "ghost" (wait, release).

Agents are generators that yield when they would block; a seeded random scheduler runs them until everyone finishes (ok) or
the step budget is spent (deadlock).  Every stage read is checked against what the producer put there, so a stage refilled
before both consumers released it is caught.  Timing is not modelled, only ordering and phase correctness.

run_pingpong / simulate_pingpong: the MLP kernel's stream, in which the two warpgroups take turns and every stage has one
owner warpgroup; with ctas = 2, the variant in which a cluster of two CTAs shares it by multicast.

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


def run_pingpong(NS, runs, n_tiles, seed, ctas=1, tile_group=1, shared_full=False, release_count=None, max_steps=4000000):
    """The ping-pong stream of the MLP kernel (nm_mlp_tc.cu, ctas = 1) and of its CTA-pair variant that shares each stage by
    TMA multicast (ctas = 2: measured slower and not shipped, DESIGN 4.1), on one cluster of `ctas` CTAs (the grid of the
    model): per
    round and layer the producer streams the layer's stages for warpgroup 0, then the same stages for warpgroup 1, and each
    fill has ONE owner warpgroup per CTA.  Rank 0's producer waits on its empty[s] and multicasts the stage into every CTA's
    slot s; every CTA arms its own full[wg][s] (count 2 here: the arming arrival and the data), rank 1 once that barrier's
    previous phase is complete.  The owner in each CTA waits on full[wg][s] (parity: its own fills of slot s) and releases
    the stage on rank 0's empty[s] (one arrival per CTA).  Tiles are dealt as the kernel deals them: groups of `tile_group`
    consecutive tiles round-robin over the 2 * ctas workers (rank 0's warpgroups first).  A warpgroup's stages are streamed
    in a round when rank 0's warpgroup has a tile; a warpgroup of another CTA without one walks them as a ghost.

    shared_full: both warpgroups wait on one full[s] per slot with parities from the ring position (the design the per-
    warpgroup full barriers replace).  release_count: arrivals rank 0's empty[s] waits for (the protocol: one per CTA).
    Both broken variants must make the model fail (an early read, an early refill or a hang).  Returns (ok, info)."""
    release_count = ctas if release_count is None else release_count
    V = 2 * ctas

    def tile_of(v, i):
        t = (v + (i // tile_group) * V) * tile_group + i % tile_group
        return t if t < n_tiles else -1

    # the stream: (round, layer, owner) blocks in producer order, and the global index of each block's first stage
    blocks, g, r = [], 0, 0
    while tile_of(0, r) >= 0:
        for li, n in enumerate(runs):
            for w in (0, 1):
                if tile_of(w, r) >= 0:
                    blocks.append((r, li, w, g, n))
                    g += n
        r += 1
    total = g
    full = [[[Bar(f"cta{c}.full{w}.{s}", 2) for s in range(NS)] for w in (0, 1)] for c in range(ctas)]
    if shared_full:
        for c in range(ctas):
            full[c][1] = full[c][0]
    empty = [Bar(f"empty{s}", release_count) for s in range(NS)]
    stage = [[None] * NS for _ in range(ctas)]
    seen = {}
    errors = []

    def wait(bar, k):
        while not bar.done(k):
            yield

    owner = {}
    for (_, _, w, g0, n) in blocks:
        for j in range(n):
            owner[g0 + j] = w

    def producer(c):
        armed = {}
        for it in range(total):
            s, w = it % NS, owner[it]
            if c == 0:
                yield from wait(empty[s], ((it // NS) & 1) ^ 1)
            else:                               # the previous phase of full[w][s] is complete
                k = armed.get((w, s), 0)
                yield from wait(full[c][w][s], k ^ 1 if k == 0 else k - 1)
                armed[(w, s)] = k + 1
            full[c][w][s].arrive()              # arm
            yield
            if c == 0:
                for d in range(ctas):           # the multicast lands in every CTA
                    stage[d][s] = it
                    full[d][w][s].arrive()
                yield

    def consumer(c, w):
        v = 2 * c + w
        fills = [0] * NS
        got = seen.setdefault((c, w), [])
        ghost_seen = False
        for (r, li, bw, g0, n) in blocks:
            if bw != w or n == 0:
                continue                        # the other warpgroup's stages: the ring position moves past them
            real = tile_of(v, r) >= 0
            if real and ghost_seen:
                errors.append(f"cta {c} warpgroup {w}: a tile after a ghost round")
            ghost_seen = ghost_seen or not real
            prev = None
            for j in range(n):
                it = g0 + j
                s = it % NS
                k = (it // NS) if shared_full else fills[s]
                yield from wait(full[c][w][s], k)
                fills[s] += 1
                if stage[c][s] != it:
                    errors.append(f"cta {c} warpgroup {w} expected stage content {it}, slot {s} holds {stage[c][s]}")
                got.append(it)
                yield
                if not real:
                    empty[s].arrive()           # ghost: hand the stage straight back
                else:
                    if prev is not None:        # wait_group 1: the previous stage's wgmmas are complete
                        empty[prev].arrive()
                    prev = s
            if real:
                empty[prev].arrive()            # wait_group 0 at the end of the layer
            yield

    agents = [producer(c) for c in range(ctas)] + [consumer(c, w) for c in range(ctas) for w in (0, 1)]
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
    for c in range(ctas):
        for w in (0, 1):
            want = [b[3] + j for b in blocks if b[2] == w for j in range(b[4])]
            if seen.get((c, w), []) != want:
                return False, f"cta {c} warpgroup {w} skipped or repeated a stage"
    return True, "ok"


def simulate_pingpong(runs, n_tiles, NS, seeds=(0, 1, 2), **kw):
    """run_pingpong over several scheduler seeds."""
    for seed in seeds:
        ok, info = run_pingpong(NS, runs, n_tiles, seed, **kw)
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
