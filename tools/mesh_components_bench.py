"""Small-component removal (nm_mesh_components, DESIGN 4.9) on the shipped checkpoints: how many floaters the iso-32 meshes
have, what the pass costs, and what removing them does to the chamfer distance.

Per mesh (lego fine net at each --res, fern fine net at --fern-res): vertices, faces, components (with >= 1 face), the five
largest component sizes, and for each --m the components / faces / vertices below it.  Cost: nm_mesh_components at each --m
beside the sigma sweep, host clock around a synchronised call, median and range of --reps after a warm-up.  Quality: the
--res[0] lego mesh against the --ref-res mesh at super-sampling --ref-s, both filtered at the same m (m = 0: unfiltered),
--samples area-weighted surface points each (nm_mesh_sample), the two one-sided chamfer means of nm_chamfer
[test -> reference, reference -> test].  Floaters of the test mesh show in the first.  All in the sweep's coordinates.

Prints one JSON line with the card's name, power limit and SM clocks read in the same run.

    python tools/mesh_components_bench.py [--res 256 512] [--fern-res 256] [--m 16 256 4096] [--reps 5] [--out f.json]"""
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


def mesh(nm, eng, vol, iso, lins, s):
    """(index-coordinate vertices, faces, grid normals) of the volume's mesh at super-sampling s."""
    n0 = vol.shape[0]
    nv, nt = eng.mc_count(vol, iso, 0, n0, 0, n0)
    if s == 0:
        return eng.mc_emit(vol, iso, 0, n0, 0, n0, nv, nt, 0)
    _, fines = nm.super_sampling_tables(float(lins[0][-1]), n0, s)
    return eng.mc_emit_ss(vol, iso, 0, n0, 0, n0, nv, nt, 0, s, lins, fines)


def census(eng, v, f, n, ms):
    """Component statistics of one mesh from its labels (m = 0: every vertex kept, labels of every vertex)."""
    V = v.shape[0]
    _, _, _, (_, _, comps, _), labels = eng.mesh_components(v, n, f, 0, want_labels=True)
    lab = labels.long()
    faces = torch.bincount(lab[f[:, 0].long()], minlength=V)
    verts = torch.bincount(lab, minlength=V)
    roots = (lab == torch.arange(V, device=lab.device)) & (faces > 0)
    sz, vz = faces[roots], verts[roots]
    out = dict(vertices=V, faces=int(f.shape[0]), components=comps, unreferenced_vertices=int((faces[lab] == 0).sum()),
               largest=torch.sort(sz, descending=True).values[:5].tolist(), below={})
    for m in ms:
        small = sz < m
        out["below"][str(m)] = dict(components=int(small.sum()), faces=int(sz[small].sum()), vertices=int(vz[small].sum()))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--fern-res", type=int, nargs="*", default=[256])
    ap.add_argument("--limit", type=float, default=1.2)
    ap.add_argument("--iso", type=float, default=32.0)
    ap.add_argument("--m", type=int, nargs="+", default=[16, 256, 4096])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-res", type=int, default=512)
    ap.add_argument("--ref-s", type=int, default=7)
    ap.add_argument("--samples", type=int, default=1 << 20)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_components_bench needs a CUDA device")
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200.mesh import sweep_coordinates
    from bench import load_npz, model_cfg

    class Args:
        iso_level = a.iso

    result = dict(card=card(), limit=a.limit, iso=a.iso, meshes={}, chamfer={})
    grids = {}
    for name, weights, near_far, resolutions in (("lego", "weights_lego_nerf.npz", (2.0, 6.0), sorted(set(a.res) | {a.ref_res})),
                                                 ("fern", "weights_fern_nerf.npz", (0.0, 1.0), a.fern_res)):
        if not resolutions:
            continue
        model = nm.NeRFModel.from_npz(model_cfg(*near_far), load_npz(weights)).eval().cuda()
        eng = model._engine()
        for res in resolutions:
            lins, _ = nm.super_sampling_tables(a.limit, res, 0)
            vol, t_sweep = timed(lambda: eng.grid_sigma(lins), a.reps)
            iso = float(nm.extract_iso_level(vol, Args, eng))
            if name == "lego":
                grids[res] = (eng, vol, iso, lins)
            if name == "lego" and res not in a.res:
                continue
            v, f, n = mesh(nm, eng, vol, iso, lins, 0)
            key = f"{name}_{res}"
            if f.shape[0] == 0:
                result["meshes"][key] = dict(vertices=int(v.shape[0]), faces=0, sweep=t_sweep)
                continue
            r = census(eng, v, f, n, a.m)
            r["sweep"] = t_sweep
            r["components_pass"] = {}
            for m in a.m:
                _, t = timed(lambda: eng.mesh_components(v, n, f, m), a.reps)
                t["vs_sweep"] = round(t["median_ms"] / t_sweep["median_ms"], 5)
                r["components_pass"][str(m)] = t
            result["meshes"][key] = r
            del vol

    # chamfer: the res[0] lego mesh against the ref-res s = ref-s mesh, both filtered at the same m
    eng, vol, iso, lins = grids[a.ref_res]
    rv, rf, rn = mesh(nm, eng, vol, iso, lins, a.ref_s)
    eng, vol, iso, tlins = grids[a.res[0]]
    tv, tf, tn = mesh(nm, eng, vol, iso, tlins, 0)
    result["chamfer"].update(res=a.res[0], ref_res=a.ref_res, ref_s=a.ref_s, samples=a.samples, by_m={})
    for m in [0] + a.m:
        fv, _, ff, (_, tkf, _, _), _ = eng.mesh_components(tv, tn, tf, m)
        gv, _, gf, (_, rkf, _, _), _ = eng.mesh_components(rv, rn, rf, m)
        if tkf == 0 or rkf == 0:
            result["chamfer"]["by_m"][str(m)] = dict(test_faces=tkf, ref_faces=rkf)
            continue
        x = eng.mesh_sample(sweep_coordinates(fv, tlins), ff, a.samples, 1234)
        y = eng.mesh_sample(sweep_coordinates(gv, lins), gf, a.samples, 4321)
        d = eng.chamfer(x, y).cpu().tolist()
        result["chamfer"]["by_m"][str(m)] = dict(test_faces=tkf, ref_faces=rkf, test_to_ref=d[0], ref_to_test=d[1],
                                                 chamfer=d[0] + d[1])
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
