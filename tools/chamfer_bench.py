"""Chamfer evaluation on the lego fine net: (1) the grid nearest-neighbour search (nm_nearest) against the brute-force
kernel (nm_debug_nearest_brute) at N = M in --sizes, on surface samples of the --ref-res mesh and on a uniform cube, each
timed on its own (host clock around the call, ending in a device synchronise) after a warm-up, median and range over the
repeats, with brute force's pair evaluations per second; (2) mesh accuracy: the chamfer distance in world coordinates, at
--samples points per mesh, of the --res mesh at each super-sampling factor --s against the --ref-res mesh at --ref-s.
Prints one JSON line with the card's name and power limit read in the same run.

    python tools/chamfer_bench.py [--sizes 2400 131072 1048576] [--res 256] [--s 0 1 3] [--ref-res 512] [--ref-s 7]
                                  [--samples 1048576] [--reps 5] [--brute-reps 3] [--out chamfer.json]"""
import argparse
import json
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from mesh_ss_bench import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[2400, 1 << 17, 1 << 20])
    ap.add_argument("--res", type=int, default=256)
    ap.add_argument("--s", type=int, nargs="+", default=[0, 1, 3])
    ap.add_argument("--ref-res", type=int, default=512)
    ap.add_argument("--ref-s", type=int, default=7)
    ap.add_argument("--samples", type=int, default=1 << 20)
    ap.add_argument("--limit", type=float, default=1.2)
    ap.add_argument("--iso", type=float, default=32.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--brute-reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("chamfer_bench needs a CUDA device")
    import nerfmeshes_b200 as nm
    from bench import load_npz, model_cfg
    model = nm.NeRFModel.from_npz(model_cfg(2.0, 6.0), load_npz("weights_lego_nerf.npz")).eval().cuda()
    eng = model._engine()

    def mesh(res, s):
        v, f, _, _ = nm.extract_geometry(model, "cuda", SimpleNamespace(limit=a.limit, res=res, iso_level=a.iso, super_sampling=s))
        return v, f

    ref_v, ref_f = mesh(a.ref_res, a.ref_s)
    result = dict(card=card(), ref=dict(res=a.ref_res, s=a.ref_s, vertices=int(ref_v.shape[0]), faces=int(ref_f.shape[0])),
                  nearest={}, accuracy={})
    gen = torch.Generator(device="cuda").manual_seed(0)
    for n in a.sizes:
        clouds = {"surface": (eng.mesh_sample(ref_v, ref_f, n, 1), eng.mesh_sample(ref_v, ref_f, n, 2)),
                  "uniform": (torch.rand((n, 3), device="cuda", generator=gen), torch.rand((n, 3), device="cuda", generator=gen))}
        for name, (q, p) in clouds.items():
            (d, i), tg = timed(lambda: eng.nearest(q, p), a.reps)
            (db, ib), tb = timed(lambda: eng.debug_nearest_brute(q, p), a.brute_reps)
            same = bool(torch.equal(d.view(torch.int32), db.view(torch.int32)) and torch.equal(i, ib))
            result["nearest"][f"{name}_{n}"] = dict(grid=tg, brute=tb, same_as_brute=same,
                                                     speedup=round(tb["median_ms"] / tg["median_ms"], 2),
                                                     brute_pairs_per_s=float(f"{n * n / (tb['median_ms'] * 1e-3):.4g}"))
    ref_pts = eng.mesh_sample(ref_v, ref_f, a.samples, 100)
    m = eng.chamfer(eng.mesh_sample(ref_v, ref_f, a.samples, 101), ref_pts).cpu().tolist()
    result["accuracy"]["sampling_floor"] = dict(chamfer=m[0] + m[1])     # the reference mesh against itself, other seed
    for s in a.s:
        v, f = mesh(a.res, s)
        pts = eng.mesh_sample(v, f, a.samples, 200 + s)
        m = eng.chamfer(pts, ref_pts).cpu().tolist()
        result["accuracy"][f"res{a.res}_s{s}"] = dict(chamfer=m[0] + m[1], to_ref=m[0], from_ref=m[1], vertices=int(v.shape[0]))
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
