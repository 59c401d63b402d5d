"""Sparse density sweep (args.sparse_sweep, DESIGN 4.10) against the dense sweep on the shipped checkpoints.

Per network (lego and fern fine nets), resolution and block edge B: lattice points, active / total blocks, evaluated / total
points, rounds; host clock around the synchronised lattice call, the run call (rounds + fill) and both, median and range of
--reps after a warm-up, beside the dense sweep + statistics timed the same way; kernel time of one extra, profiled call
split into network, fill and bookkeeping (torch.profiler, CUDA activities); and the mesh difference against the dense mesh
(marching cubes at the sparse call's iso level on both volumes): components and faces missing, the largest missing
component.  The dense sweep is timed at every --res and run once at every --dense-once-res (no timing statistics there).

Prints one JSON line with the card's name, power limit and SM clocks read in the same run.

    python tools/mesh_sparse_bench.py [--res 256 512] [--sparse-only-res 1024] [--dense-once-res 1024] [--blocks 4 8 16]
                                      [--reps 5] [--out f.json]"""
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
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:                     # the measurement stands without it; say so in the output
        return f"unavailable ({e})"


def stats(ts):
    return dict(median_ms=round(float(np.median(ts)), 3), min_ms=round(min(ts), 3), max_ms=round(max(ts), 3))


def clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def kernel_split(fn):
    """Device time of one call by kernel family, ms."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = dict(network_ms=0.0, fill_ms=0.0, bookkeeping_ms=0.0)
    for e in prof.key_averages():
        us = float(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0) or 0)
        if not us or e.key.lower().startswith("memcpy") or e.key.lower().startswith("memset"):
            key = "bookkeeping_ms"
        elif "sp_fill_kernel" in e.key:
            key = "fill_ms"
        elif "mlp" in e.key:
            key = "network_ms"
        else:
            key = "bookkeeping_ms"
        out[key] += us / 1e3
    return {k: round(v, 3) for k, v in out.items()}


def mesh_difference(dv, df, labels, sv):
    """Dense vertices (V,3) / faces (F,3) with their component labels (V,), sparse vertices (rows of the dense ones): which
    dense components the sparse mesh lacks."""
    rows = lambda a: np.ascontiguousarray(a, np.float32).view(np.dtype((np.void, 12))).reshape(-1)
    kept_v = np.isin(rows(dv), rows(sv))
    sizes = np.bincount(labels[df[:, 0]], minlength=len(dv)) if len(df) else np.zeros(len(dv), np.int64)
    roots = np.flatnonzero(sizes > 0)
    kept_c = kept_v[roots]                       # a component's id is its smallest vertex: kept iff that vertex is
    partial = int(np.count_nonzero(kept_v != kept_v[labels]))
    miss = np.sort(sizes[roots][~kept_c])[::-1]
    return dict(dense_vertices=int(len(dv)), dense_faces=int(len(df)), dense_components=int(len(roots)),
                sparse_vertices=int(len(sv)), missing_components=int(len(miss)), missing_faces=int(miss.sum()),
                largest_missing=int(miss[0]) if len(miss) else 0, largest_dense=int(sizes.max()) if len(df) else 0,
                vertices_of_partly_kept_components=partial)


def mesh_of(eng, vol, iso):
    n0 = vol.shape[0]
    nv, nt = eng.mc_count(vol, iso, 0, n0, 0, n0)
    return eng.mc_emit(vol, iso, 0, n0, 0, n0, nv, nt, 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs="*", default=[256, 512])
    ap.add_argument("--sparse-only-res", type=int, nargs="*", default=[1024])
    ap.add_argument("--dense-once-res", type=int, nargs="*", default=[1024])
    ap.add_argument("--blocks", type=int, nargs="+", default=[4, 8, 16])
    ap.add_argument("--nets", nargs="+", default=["lego", "fern"])
    ap.add_argument("--limit", type=float, default=1.2)
    ap.add_argument("--iso", type=float, default=32.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_sparse_bench needs a CUDA device")
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import mesh
    from bench import load_npz, model_cfg

    result = dict(card=card(), limit=a.limit, iso_level=a.iso, reps=a.reps, chunk_points=os.environ.get("NM_SPARSE_CHUNK_POINTS", "default"),
                  cases=[])
    near_far = dict(lego=(2.0, 6.0), fern=(0.0, 1.0))
    for net in a.nets:
        model = nm.NeRFModel.from_npz(model_cfg(*near_far[net]), load_npz(f"weights_{net}_nerf.npz")).eval().cuda()
        eng = model._engine()
        for res in sorted(set(a.res) | set(a.sparse_only_res)):
            lins = [torch.linspace(-a.limit, a.limit, res) for _ in range(3)]
            vol = torch.empty((res, res, res), dtype=torch.float32, device=eng.device)
            timed_dense, once_dense = res in a.res, res in a.dense_once_res
            dense = None
            if timed_dense or once_dense:
                dvol = torch.empty_like(vol)

                def dense_call():
                    eng.grid_sigma(lins, out=dvol)
                    return eng.volume_stats(dvol)
                if timed_dense:
                    dense_call()
                ts = []
                for _ in range(a.reps if timed_dense else 1):
                    st, ms = clock(dense_call)
                    ts.append(ms)
                dense = dict(stats(ts), runs=len(ts), warmed_up=timed_dense,
                             iso=float(mesh.clamp_iso_level(a.iso, *[np.float32(x) for x in st])))
            for B in a.blocks:
                lat_t, run_t, tot_t = [], [], []
                for rep in range(a.reps + 1):
                    st, t0 = clock(lambda: eng.sparse_lattice(lins, B, vol))
                    iso = float(mesh.clamp_iso_level(a.iso, *[np.float32(x) for x in st]))
                    counts, t1 = clock(lambda: eng.sparse_run(lins, B, iso, vol))
                    if rep:                      # rep 0 is the warm-up
                        lat_t.append(t0); run_t.append(t1); tot_t.append(t0 + t1)
                kernels = kernel_split(lambda: eng.sparse_sweep(lins, a.iso, B, vol))
                case = dict(net=net, res=res, block=B, iso=iso, lattice_points=counts[0], active_blocks=counts[1], blocks=counts[2],
                            evaluated_points=counts[3], points=res ** 3, rounds=counts[4], lattice=stats(lat_t), run=stats(run_t),
                            total=stats(tot_t), kernels_of_one_call=kernels, dense=dense)
                if dense is not None:
                    case["speedup_median"] = round(dense["median_ms"] / case["total"]["median_ms"], 2)
                    dv, df, dn = mesh_of(eng, dvol, iso)
                    sv, sf, _ = mesh_of(eng, vol, iso)
                    if dv.shape[0]:
                        labels = eng.mesh_components(dv, dn, df, 0, want_labels=True)[4]
                        case["mesh"] = mesh_difference(dv.cpu().numpy(), df.cpu().numpy(), labels.cpu().numpy(), sv.cpu().numpy())
                        case["mesh"]["sparse_faces"] = int(sf.shape[0])
                    del dv, df, dn, sv, sf
                result["cases"].append(case)
                print(json.dumps(case), file=sys.stderr, flush=True)
            del vol
            if dense is not None:
                del dvol
            torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
