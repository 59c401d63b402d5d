"""Cost of super-sampled marching cubes (nm_mc_emit_ss) on the lego fine net: the sigma sweep, the count step, the plain
emit (s = 0) and the super-sampled emit for each s, every stage timed on its own (host clock around the call, ending in a
device synchronise) after a warm-up, median and range over --reps repeats.  Prints one JSON line with the card's name and
power limit read in the same run, the vertex count, the network points each emit evaluated and the point count the
dense route (three volumes refined along one axis, mesh_nerf.py:109-117) would need — computed, not run.

    python tools/mesh_ss_bench.py [--res 512] [--s 1 3 7] [--reps 5] [--out mesh_ss.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                     # the measurement stands without it; say so in the output
        return f"unavailable ({e})"


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return out, dict(median_ms=round(float(np.median(ts)), 3), min_ms=round(min(ts), 3), max_ms=round(max(ts), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--limit", type=float, default=1.2)
    ap.add_argument("--iso", type=float, default=32.0)
    ap.add_argument("--s", type=int, nargs="+", default=[1, 3, 7])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_ss_bench needs a CUDA device")
    import nerfmeshes_b200 as nm
    from bench import load_npz, model_cfg
    model = nm.NeRFModel.from_npz(model_cfg(2.0, 6.0), load_npz("weights_lego_nerf.npz")).eval().cuda()
    eng = model._engine()
    res = a.res
    lins, _ = nm.super_sampling_tables(a.limit, res, 0)
    vol, t_sweep = timed(lambda: eng.grid_sigma(lins), a.reps)

    class Args:
        iso_level = a.iso
    iso = float(nm.extract_iso_level(vol, Args, eng))
    (nv, nt), t_count = timed(lambda: eng.mc_count(vol, iso, 0, res, 0, res), a.reps)
    outs = (torch.empty((nv, 3), device=eng.device), torch.empty((nv, 3), device=eng.device),
            torch.empty((nt, 3), dtype=torch.int32, device=eng.device))
    _, t_emit = timed(lambda: eng.mc_emit(vol, iso, 0, res, 0, res, nv, nt, 0, out=outs), a.reps)
    result = dict(card=card(), res=res, limit=a.limit, iso=iso, vertices=nv, triangles=nt, sweep=t_sweep, count=t_count,
                  emit_s0=t_emit, points_sweep=res ** 3, emit_ss={})
    for s in a.s:
        _, fines = nm.super_sampling_tables(a.limit, res, s)
        eng.set_timing(True)
        eng.mc_emit_ss(vol, iso, 0, res, 0, res, nv, nt, 0, s, lins, fines, out=outs)
        torch.cuda.synchronize()
        _, points, launches = eng.mlp_time_ms()
        eng.set_timing(False)
        _, t = timed(lambda: eng.mc_emit_ss(vol, iso, 0, res, 0, res, nv, nt, 0, s, lins, fines, out=outs), a.reps)
        dense = 3 * res * res * (res + (res - 1) * s)
        result["emit_ss"][str(s)] = dict(t, points=points, mlp_launches=launches, dense_points=dense,
                                         vs_sweep=round(t["median_ms"] / t_sweep["median_ms"], 4))
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
