"""Mesh rasterizer (nm_rasterize_mesh, DESIGN 4.13) on the lego fine net's iso-32 mesh: what a mesh image costs, and how close
the mesh's images are to the NeRF's.

The --res^3 mesh, full and decimated to each --frac of its faces (nm_mesh_decimate).  Per mesh: vertex colours
(mesh.mesh_appearance) and textures at each N in --texels (Engine.bake_texture).  Per colouring: the raster time at --size x
--size (host clock around the synchronised call, median and range of --reps, every shape warmed up first) over --poses ring
poses pose_spherical(theta, -30, 4.0), theta evenly spaced, with the lego focal scaled to --size; and mesh.compare_with_nerf
over the same poses at --eval-size (PSNR over the image and over the pixels both cover, silhouette IoU against acc > 0.5, mean
|depth difference|).  For scale, one NeRF image (render_image) at --size.  Close-ups: vertex colours at --size from three
poses at radius 1.5, 1.2 and 0.8, with NM_RASTER_BIG_FACE_PIXELS at its default and at 2^30 (no face on the tile pass).

Prints one JSON line with the card's name, power limit and SM clocks read in the same run.

    python tools/mesh_render_bench.py [--res 512] [--frac 0.1 0.02] [--texels 4 8] [--size 800] [--eval-size 800] [--out f.json]"""
import argparse
import json
import os
import subprocess
import sys
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


def timed(fn, reps):
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return dict(median_ms=round(float(np.median(ts)), 3), min_ms=round(min(ts), 3), max_ms=round(max(ts), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--frac", type=float, nargs="+", default=[0.1, 0.02])
    ap.add_argument("--texels", type=int, nargs="*", default=[4, 8])
    ap.add_argument("--size", type=int, default=800)
    ap.add_argument("--eval-size", type=int, default=800)
    ap.add_argument("--poses", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--limit", type=float, default=1.2)
    ap.add_argument("--iso", type=float, default=32.0)
    ap.add_argument("--out")
    a = ap.parse_args()
    os.environ.pop("NM_RASTER_BIG_FACE_PIXELS", None)
    if not torch.cuda.is_available():
        raise SystemExit("mesh_render_bench needs a CUDA device")
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import mesh
    from nerfmeshes_b200 import parallel as par
    from bench import load_npz, model_cfg

    model = nm.NeRFModel.from_npz(model_cfg(2.0, 6.0), load_npz("weights_lego_nerf.npz")).eval().cuda()
    eng = model._engine()
    args = SimpleNamespace(view_disparity=1e-2, view_disparity_max_bound=4.0)
    focal = float(0.5 * 800 / np.tan(0.5 * 0.6911112))                  # the lego scene's focal at 800 pixels
    S, E = a.size, a.eval_size
    poses = [nm.pose_spherical(float(th), -30.0, 4.0) for th in np.linspace(0.0, 360.0, a.poses, endpoint=False)]
    closeups = [nm.pose_spherical(th, -30.0, r) for th, r in ((30.0, 1.5), (120.0, 1.2), (210.0, 0.8))]
    result = dict(card=card(), net="lego", res=a.res, limit=a.limit, iso_level=a.iso, size=S, eval_size=E, poses=a.poses,
                  reps=a.reps, meshes=[])
    A = SimpleNamespace(limit=a.limit, res=a.res, iso_level=a.iso)
    v, f, n, _ = par.extract_geometry_sharded(model, A, group=par.SINGLE, to_host=False)
    v, f, n = v.clone(), f.clone(), n.clone()
    result["nerf_image"] = timed(lambda: eng.render_image(poses[0], S, S, focal * S / 800, 2.0, 6.0, want=("rgb",)), 1)
    for frac in [1.0] + list(a.frac):
        if frac < 1.0:
            dv, dn, df, _, _ = eng.mesh_decimate(v, n, f, int(frac * f.shape[0]))
        else:
            dv, dn, df = v, n, f
        hv, hf, hn = mesh.rescale_vertices(dv, a.limit, a.res), df.cpu(), dn.cpu()
        diffuse = mesh.mesh_appearance(model, hv, hn, args)
        colourings = [("vertex", dict(diffuse=torch.from_numpy(diffuse).cuda()))]
        for N in a.texels:
            u8, _, _, _, _ = eng.bake_texture(hv, hn, hf, N, view_disparity=1e-2, near_far=(0.0, 4.0))
            colourings.append((f"texture N={N}", dict(texture=(u8, N))))
        entry = dict(frac=frac, faces=int(hf.shape[0]), vertices=int(hv.shape[0]), rows=[])
        gv, gf = hv.cuda(), hf.cuda()
        for name, kw in colourings:
            for p in poses:                                              # warm-up: every pose and shape once
                out = mesh.render_mesh(eng, gv, gf, p, S, S, focal * S / 800, **kw)
            t = [timed(lambda p=p: mesh.render_mesh(eng, gv, gf, p, S, S, focal * S / 800, **kw), a.reps) for p in poses]
            med = float(np.median([x["median_ms"] for x in t]))
            cmp = mesh.compare_with_nerf(model, hv, hf, poses, E, E, focal * E / 800, 2.0, 6.0, **kw)
            row = dict(colour=name, raster_ms_median=round(med, 3), raster_ms_min=min(x["min_ms"] for x in t),
                       raster_ms_max=max(x["max_ms"] for x in t), counts_pose0=list(out["counts"]),
                       **{k: round(v_, 4) for k, v_ in cmp["mean"].items()})
            entry["rows"].append(row)
            print(f"{frac:g} ({entry['faces']} faces), {name}: raster {med:.3f} ms, psnr {row['psnr']}, masked "
                  f"{row['psnr_masked']}, iou {row['iou']}, depth {row['depth_mae']}", file=sys.stderr)
        # close-ups, vertex colours: the tile pass at the default threshold against every face on one thread (2^30)
        kw = colourings[0][1]
        entry["closeup"] = []
        for thr in ("default", str(2 ** 30)):
            if thr == "default":
                os.environ.pop("NM_RASTER_BIG_FACE_PIXELS", None)
            else:
                os.environ["NM_RASTER_BIG_FACE_PIXELS"] = thr
            for p in closeups:
                mesh.render_mesh(eng, gv, gf, p, S, S, focal * S / 800, **kw)
            t = [timed(lambda p=p: mesh.render_mesh(eng, gv, gf, p, S, S, focal * S / 800, **kw), a.reps) for p in closeups]
            entry["closeup"].append(dict(big_face_pixels=thr, raster_ms=[x["median_ms"] for x in t]))
            print(f"{frac:g}: close-ups at NM_RASTER_BIG_FACE_PIXELS={thr}: {[x['median_ms'] for x in t]} ms", file=sys.stderr)
        os.environ.pop("NM_RASTER_BIG_FACE_PIXELS", None)
        result["meshes"].append(entry)
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
