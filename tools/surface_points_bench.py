"""Surface point clouds (nm_surface_points, DESIGN 4.14) on the lego fine net: what the filter costs next to the render, how
many points each depth gate keeps, what the PLY writer costs, and how close the cloud lies to the marching-cubes mesh.

The --poses-y x --poses-x ring of mesh.surface_ray_poses (32 poses at radius 4.0 by default) at --size x --size, focal
1111.1111 (the script's), near 2, far 6.  Per view: the render (render_image: rgb, depth_raw, acc) once, and the filter plus
compaction (Engine.surface_points at the defaults, step 2, dist_threshold 0.002, min_count 15) --reps times after a warm-up;
host clock around synchronised calls.  Kept points at each --min-acc, and how many pixels have acc >= that value and
depth_raw > 0 (the gate's own loss, before the neighbourhood test), with acc > 0.5 as the silhouette for scale.  Text and
binary PLY write times (mesh.export_ply, native writer) of the min_acc = 1.0 cloud.  The distance from each cloud to the
--res^3 super-sampled (--ss) marching-cubes mesh: nearest of 2^--log-samples area-weighted samples of the mesh (nm_mesh_sample,
nm_nearest), median and 95th percentile in world units; the sampling floor is the same statistic for 2^18 independent
samples of the mesh itself.

Prints one JSON line with the card's name, power limit and SM clocks read in the same run.

    python tools/surface_points_bench.py [--size 800] [--res 512] [--ss 7] [--out f.json]"""
import argparse
import json
import os
import sys
import tempfile
import time
from types import SimpleNamespace

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.mesh_render_bench import card  # noqa: E402


def clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3


def dist_stats(eng, pts, samples):
    d = eng.nearest(pts, samples)[0].sqrt().double()
    d = d[torch.randperm(d.numel(), generator=torch.Generator().manual_seed(0))[: 1 << 24].to(d.device)] if d.numel() > 1 << 24 else d
    return dict(median=round(float(torch.quantile(d, 0.5)), 6), p95=round(float(torch.quantile(d, 0.95)), 6))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--poses-y", type=int, default=8)
    ap.add_argument("--poses-x", type=int, default=4)
    ap.add_argument("--min-acc", type=float, nargs="+", default=[1.0, 0.99, 0.5])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--ss", type=int, default=7)
    ap.add_argument("--log-samples", type=int, default=22)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("surface_points_bench needs a CUDA device")
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import mesh
    from bench import load_npz, model_cfg

    model = nm.NeRFModel.from_npz(model_cfg(2.0, 6.0), load_npz("weights_lego_nerf.npz")).eval().cuda()
    eng = model._engine()
    S, focal = a.size, 1111.1111
    poses = mesh.surface_ray_poses(a.poses_y, a.poses_x)
    n = S * S
    scratch = dict(points=torch.empty((n, 3), device="cuda"), normals=torch.empty((n, 3), device="cuda"),
                   colors=torch.empty((n, 3), device="cuda"), pixel=torch.empty((n,), dtype=torch.int32, device="cuda"))
    result = dict(card=card(), net="lego", size=S, focal=focal, poses=len(poses), step=2, dist_threshold=0.002, min_count=15)
    render_ms, filter_ms = [], []
    kept = {m: 0 for m in a.min_acc}
    gated = {m: 0 for m in a.min_acc}
    silhouette = 0
    clouds = {m: [] for m in a.min_acc}
    colors = []
    normals = []
    for i, p in enumerate(poses):
        r, t = clock(lambda: eng.render_image(p, S, S, focal, 2.0, 6.0, want=("rgb", "depth_raw", "acc")))
        render_ms.append(t)
        args = (p, S, S, focal, r["depth_raw"], r["acc"], r["rgb"])
        eng.surface_points(*args, out=scratch)                                   # warm-up
        ts = [clock(lambda: eng.surface_points(*args, out=scratch))[1] for _ in range(a.reps)]
        filter_ms.append(float(np.median(ts)))
        silhouette += int((r["acc"] > 0.5).sum())
        for m in a.min_acc:
            outs, k = eng.surface_points(*args, min_acc=m, out=scratch)
            kept[m] += k
            gated[m] += int(((r["acc"] >= m) & (r["depth_raw"] > 0)).sum())
            clouds[m].append(outs["points"].clone())
            if m == 1.0:
                colors.append(outs["colors"].clone())
                normals.append(outs["normals"].clone())
        print(f"view {i}: render {render_ms[-1]:.1f} ms, filter {filter_ms[-1]:.3f} ms", file=sys.stderr)
    result["render_ms_per_view"] = dict(median=round(float(np.median(render_ms)), 2), min=round(min(render_ms), 2),
                                        max=round(max(render_ms), 2))
    result["filter_ms_per_view"] = dict(median=round(float(np.median(filter_ms)), 4), min=round(min(filter_ms), 4),
                                        max=round(max(filter_ms), 4))
    result["silhouette_pixels_acc_gt_0.5"] = silhouette
    result["kept"] = {str(m): kept[m] for m in a.min_acc}
    result["gate_pixels"] = {str(m): gated[m] for m in a.min_acc}
    if 1.0 in clouds:
        pts = torch.cat(clouds[1.0])
        col, nrm = torch.cat(colors), torch.cat(normals)
        with tempfile.TemporaryDirectory() as d:
            for binary in (False, True):
                path = os.path.join(d, "c.ply")
                _, t = clock(lambda: mesh.export_ply(pts, col, nrm, path, binary=binary))
                result["ply_binary_ms" if binary else "ply_text_ms"] = round(t, 1)
                result["ply_binary_bytes" if binary else "ply_text_bytes"] = os.path.getsize(path)
    v, f, _, _ = nm.extract_geometry(model, "cuda", SimpleNamespace(limit=1.2, res=a.res, iso_level=32.0, super_sampling=a.ss))
    samples = eng.mesh_sample(v, f, 1 << a.log_samples, 1)
    result["mesh"] = dict(res=a.res, ss=a.ss, faces=int(f.shape[0]), samples=1 << a.log_samples,
                          floor=dist_stats(eng, eng.mesh_sample(v, f, 1 << 18, 2), samples))
    result["distance"] = {str(m): dist_stats(eng, torch.cat(c), samples) for m, c in clouds.items() if sum(x.shape[0] for x in c)}
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
