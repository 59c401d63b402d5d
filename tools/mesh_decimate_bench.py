"""Quadric-error decimation (nm_mesh_decimate, DESIGN 4.11) on the lego fine net's iso-32 meshes: what the pass costs, how
many rounds it takes, what it costs in accuracy, and what it saves downstream.

Per mesh (--res dense sweeps, --sparse-res through the sparse sweep, block 8) and per target fraction --frac of the face
count: nm_mesh_decimate time (host clock around a synchronised call, median and range of --reps after a warm-up), rounds and
the final face count; the chamfer distance of the decimated mesh against the undecimated one (--samples area-weighted
surface points each, nm_mesh_sample + nm_chamfer, the two one-sided means [decimated -> full, full -> decimated] in cells^2
of the sweep's index coordinates), next to the sampling floor (the same between two sample sets of the undecimated mesh).
At --appearance-res: the appearance pass (mesh.mesh_appearance: one 64 + 128-sample ray per vertex, view_disparity 1e-2,
bound 4) and the OBJ writer (mesh.export_obj, to a temporary directory) before and after decimation to each fraction.

Prints one JSON line with the card's name, power limit and SM clocks read in the same run.

    python tools/mesh_decimate_bench.py [--res 256 512] [--sparse-res 1024] [--frac 0.5 0.1 0.02] [--reps 5] [--out f.json]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from types import SimpleNamespace

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


def timed(fn, reps, warmup=True):
    if warmup:
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
    ap.add_argument("--res", type=int, nargs="*", default=[256, 512])
    ap.add_argument("--sparse-res", type=int, nargs="*", default=[1024])
    ap.add_argument("--frac", type=float, nargs="+", default=[0.5, 0.1, 0.02])
    ap.add_argument("--appearance-res", type=int, default=512)
    ap.add_argument("--samples", type=int, default=1 << 20)
    ap.add_argument("--limit", type=float, default=1.2)
    ap.add_argument("--iso", type=float, default=32.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_decimate_bench needs a CUDA device")
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import mesh
    from nerfmeshes_b200 import parallel as par
    from bench import load_npz, model_cfg

    model = nm.NeRFModel.from_npz(model_cfg(2.0, 6.0), load_npz("weights_lego_nerf.npz")).eval().cuda()
    eng = model._engine()
    result = dict(card=card(), net="lego", limit=a.limit, iso_level=a.iso, reps=a.reps, samples=a.samples, cases=[])
    chamfer = lambda x, y: [float(c) for c in eng.chamfer(x, y).cpu()]
    for res, sparse in [(r, False) for r in a.res] + [(r, True) for r in a.sparse_res]:
        A = SimpleNamespace(limit=a.limit, res=res, iso_level=a.iso, sparse_sweep=sparse)
        v, f, n, _ = par.extract_geometry_sharded(model, A, group=par.SINGLE, to_host=False)
        v, f, n = v.clone(), f.clone(), n.clone()
        F = int(f.shape[0])
        full_pts = eng.mesh_sample(v, f, a.samples, 1)
        floor = chamfer(eng.mesh_sample(v, f, a.samples, 2), full_pts)
        case = dict(res=res, sparse_sweep=sparse, vertices=int(v.shape[0]), faces=F, sampling_floor=floor, targets=[])
        appearance = res == a.appearance_res
        if appearance:
            args = SimpleNamespace(view_disparity=1e-2, view_disparity_max_bound=4.0)

            def downstream(vv, ff, nn):
                hv, hf, hn = mesh.rescale_vertices(vv, a.limit, res), ff.cpu(), nn.cpu()
                d, t_app = timed(lambda: mesh.mesh_appearance(model, hv, hn, args), min(a.reps, 3), warmup=False)
                path = os.path.join(tempfile.gettempdir(), f"mesh_decimate_bench_{os.getpid()}.obj")
                _, t_obj = timed(lambda: mesh.export_obj(hv, hf, d, hn, path), min(a.reps, 3), warmup=False)
                os.remove(path)
                return dict(appearance=t_app, obj=t_obj)
            mesh.mesh_appearance(model, mesh.rescale_vertices(v[:4096], a.limit, res), n[:4096].cpu(), args)    # warm-up
            case["undecimated"] = downstream(v, f, n)
        for frac in a.frac:
            T = int(frac * F)
            out, t = timed(lambda: eng.mesh_decimate(v, n, f, T), a.reps)
            dv, dn, df, counts, _ = out
            entry = dict(frac=frac, target=T, faces=counts[1], vertices=counts[0], rounds=counts[2], time=t,
                         chamfer=chamfer(eng.mesh_sample(dv, df, a.samples, 1), full_pts))
            if appearance:
                entry.update(downstream(dv, df, dn))
            case["targets"].append(entry)
            print(f"{res}^3{' sparse' if sparse else ''}: {F} -> {counts[1]} faces, {counts[2]} rounds, {t['median_ms']} ms, "
                  f"chamfer {entry['chamfer']} (floor {floor})", file=sys.stderr)
        result["cases"].append(case)
        del v, f, n, full_pts
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
