"""Network-gradient mesh normals (nm_sigma_grad, DESIGN 4.8) on the lego fine net: cost and quality.

Cost: at each --res, the sigma sweep and the normal pass (mesh.network_normals: the vertices' sweep coordinates, then
the density gradient at every vertex) timed on their own — host clock around the call, ending in a device synchronise —
after a warm-up, median and range over --reps repeats; points/s of the normal pass.

Quality: a reference surface, the --ref-res mesh at super-sampling --ref-s, is sampled area-weighted (nm_mesh_sample,
with face indices); every vertex of the --res[0] mesh finds its nearest sample (nm_nearest) and is compared with that
sample's face normal, oriented towards decreasing sigma (one global sign for the whole reference mesh, see below): the
signed angle between the directions (a flipped normal is 180 deg), median and 90th percentile, and the fraction of vertices
facing against the reference, for the grid normals and the network normals, at each --quality-s; and where the grid and the
network normal of a vertex point to opposite sides, the fraction in which the network normal is the one on the
reference's side.  All meshes are compared in the sweep's coordinates (mesh.sweep_coordinates).

Prints one JSON line with the card's name, power limit and max SM clock read in the same run.

    python tools/mesh_normals_bench.py [--res 256 512] [--reps 5] [--ref-res 512] [--ref-s 7] [--quality-s 0 3] [--out f.json]"""
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


def mesh(nm, eng, vol, iso, lins, s):
    """(index-coordinate vertices, faces, grid normals) of the volume's mesh at super-sampling s."""
    n0 = vol.shape[0]
    nv, nt = eng.mc_count(vol, iso, 0, n0, 0, n0)
    if s == 0:
        return eng.mc_emit(vol, iso, 0, n0, 0, n0, nv, nt, 0)
    _, fines = nm.super_sampling_tables(float(lins[0][-1]), n0, s)
    return eng.mc_emit_ss(vol, iso, 0, n0, 0, n0, nv, nt, 0, s, lins, fines)


def angles(n, ref):
    """Signed comparison with the oriented reference normals: the angle between the directions (180 deg = flipped), its
    median and 90th percentile, and the fraction of vertices facing against the reference (dot < 0)."""
    c = (torch.nn.functional.normalize(n.double(), dim=1) * ref).sum(1).clamp(-1.0, 1.0)
    a = torch.rad2deg(torch.acos(c)).cpu().numpy()
    return dict(median_deg=round(float(np.median(a)), 3), p90_deg=round(float(np.percentile(a, 90)), 3),
                against=round(float((c < 0).double().mean()), 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--limit", type=float, default=1.2)
    ap.add_argument("--iso", type=float, default=32.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ref-res", type=int, default=512)
    ap.add_argument("--ref-s", type=int, default=7)
    ap.add_argument("--quality-s", type=int, nargs="+", default=[0, 3])
    ap.add_argument("--samples", type=int, default=1 << 23)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_normals_bench needs a CUDA device")
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200.mesh import network_normals, sweep_coordinates
    from bench import load_npz, model_cfg
    model = nm.NeRFModel.from_npz(model_cfg(2.0, 6.0), load_npz("weights_lego_nerf.npz")).eval().cuda()
    eng = model._engine()
    which = model.get_model()._owner[1]

    class Args:
        iso_level = a.iso

    result = dict(card=card(), limit=a.limit, cost={}, quality={})
    grids = {}
    for res in sorted(set(a.res) | {a.ref_res}):
        lins, _ = nm.super_sampling_tables(a.limit, res, 0)
        vol, t_sweep = timed(lambda: eng.grid_sigma(lins), a.reps)
        iso = float(nm.extract_iso_level(vol, Args, eng))
        grids[res] = (vol, iso, lins)
        if res not in a.res:
            continue
        v, f, n = mesh(nm, eng, vol, iso, lins, 0)
        (_, fb), t_norm = timed(lambda: network_normals(eng, which, v, lins, n), a.reps)
        _, t_grad = timed(lambda: eng.sigma_grad(which, sweep_coordinates(v, lins), want_sigma=False), a.reps)
        nv = int(v.shape[0])
        result["cost"][str(res)] = dict(vertices=nv, sweep=t_sweep, normal_pass=t_norm, sigma_grad_only=t_grad,
                                        normal_pass_points_per_s=round(nv / (t_norm["median_ms"] * 1e-3)),
                                        vs_sweep=round(t_norm["median_ms"] / t_sweep["median_ms"], 4), fallback=fb)

    # reference surface: the fine mesh's faces in sweep coordinates, sampled with face indices
    vol, iso, lins = grids[a.ref_res]
    rv, rf, rn = mesh(nm, eng, vol, iso, lins, a.ref_s)
    rx = sweep_coordinates(rv, lins)
    pts, fi = eng.mesh_sample(rx, rf, a.samples, 1234, want_faces=True)
    tri = rx[rf.long()].double()
    fn = torch.nn.functional.normalize(torch.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0], dim=1), dim=1)
    # Marching cubes winds every face the same way, so the face normals share one orientation; it is turned to point
    # towards decreasing sigma (the convention of both normals compared) by ONE global sign: the side on which the reference
    # mesh's own grid normals lie for the majority of faces.  No per-face choice, so no bias towards either candidate.
    agree = float(((fn * rn[rf.long()].double().mean(1)).sum(1) > 0).double().mean())
    if agree < 0.5:
        fn = -fn
    result["quality"]["ref_orientation_agreement"] = round(max(agree, 1 - agree), 4)
    res0 = a.res[0]
    vol, iso, lins = grids[res0]
    result["quality"].update(ref_res=a.ref_res, ref_s=a.ref_s, samples=a.samples, res=res0, by_s={})
    for s in a.quality_s:
        v, f, n = mesh(nm, eng, vol, iso, lins, s)
        x = sweep_coordinates(v, lins)
        _, idx = eng.nearest(x, pts)
        ref = fn[fi[idx.long()].long()]
        nn_, fb = network_normals(eng, which, v, lins, n)
        # where the two disagree in direction (dot < 0): which one faces the reference's way
        split = (nn_ * n).sum(1) < 0
        net_right = float(((nn_[split].double() * ref[split]).sum(1) > 0).double().mean()) if bool(split.any()) else float("nan")
        result["quality"]["by_s"][str(s)] = dict(vertices=int(v.shape[0]), grid=angles(n, ref), network=angles(nn_, ref),
                                                 opposed=round(float(split.double().mean()), 4),
                                                 opposed_network_right=round(net_right, 4), fallback=fb)
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
