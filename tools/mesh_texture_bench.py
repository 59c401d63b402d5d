"""Texture bake (nm_bake_texture, DESIGN 4.12) of the lego fine net's iso-32 mesh, decimated: what the bake costs, what it
writes, and whether the texture carries more colour than the vertices.

Per target fraction --frac of the --res^3 mesh's faces (nm_mesh_decimate) and per N in --texels: the bake (Engine.bake_texture,
host clock around a synchronised call, median of --reps; every shape warmed up on 64 faces first, and each bake is long) split
into its texel queries (nm_debug_texture_rays over all faces, timed alone), the fused-MLP kernels of its render (CUDA events,
nm_mlp_time_ms) and the remainder (ray sampling and the other render stages, scatter, ring, quantisation, uvs, vertex
colours); the PNG and OBJ writes (mesh.write_png, nm_export_obj_textured through mesh.export_textured_obj minus its PNG, to a
temporary directory); texels rendered and atlas size.  For comparison the per-vertex appearance pass (mesh.mesh_appearance)
of the same mesh.

Quality: --points seeded random surface points (face uniform, barycentrics uniform on the triangle), each with the appearance
ray a texel there would get (surface_errors); the mean absolute colour error against that ray of a bilinear lookup in the
float atlas and of the barycentric interpolation of the vertex colours.

Prints one JSON line with the card's name, power limit and SM clocks read in the same run.

    python tools/mesh_texture_bench.py [--res 512] [--frac 0.1 0.02] [--texels 4 8 16] [--reps 1] [--out f.json]"""
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


def appearance(model, points, dirs, args):
    """mesh_appearance's colour of the query at points (n,3) with directions dirs (n,3) (device tensors), rgb only."""
    eng = model._engine()
    if getattr(args, "no_view_dependence", False):
        return eng.point_mlp(model.get_model()._owner[1], points, dirs)[:, :3]
    origins = points - float(np.float32(args.view_disparity)) * dirs
    return eng.render_rays(origins, dirs, 0.0, float(args.view_disparity_max_bound), training=model.training,
                           buff=hasattr(model, "tree"), want=("rgb",))["rgb"]


def surface_errors(model, verts, faces, normals, atlas, diffuse, N, args, n_points, seed):
    """Mean absolute colour error (over points and channels) of (bilinear atlas lookup, barycentric vertex colours) against
    the appearance ray at n_points seeded random surface points, built as a texel's would be.  verts / normals (V,3) world
    coordinates, faces (F,3), atlas (H,W,3) float, diffuse (V,3)."""
    from nerfmeshes_b200.engine import Engine
    dev = torch.device("cuda")
    v, n = torch.as_tensor(verts).to(dev, torch.float32), torch.as_tensor(normals).to(dev, torch.float32)
    f = torch.as_tensor(faces).to(dev, torch.long)
    atlas, diffuse = torch.as_tensor(atlas).to(dev, torch.float32), torch.as_tensor(diffuse).to(dev, torch.float32)
    g = torch.Generator().manual_seed(seed)
    fi = torch.randint(0, f.shape[0], (n_points,), generator=g).to(dev)
    b = -torch.log(torch.rand((n_points, 3), generator=g, dtype=torch.float64))
    b = (b / b.sum(1, keepdim=True)).to(dev)
    w1, w2 = b[:, 1].float(), b[:, 2].float()
    w0 = (1.0 - w1) - w2
    idx = f[fi]
    bary = lambda a: (w0[:, None] * a[idx[:, 0]] + w1[:, None] * a[idx[:, 1]]) + w2[:, None] * a[idx[:, 2]]
    p, m = bary(v), bary(n)
    nn = m / torch.linalg.norm(m, dim=1, keepdim=True).clamp_min(1e-30)
    ref = appearance(model, p, -nn, args)
    # bilinear lookup at the point's atlas coordinates, texel centres at integers (the layout of DESIGN 4.12)
    Q = Engine.texture_layout(f.shape[0], N)[0]
    C_ = N + 2
    cell = fi // 2
    x0, y0 = (cell % Q) * C_, (cell // Q) * C_
    s, t = b[:, 1] * (N - 1), b[:, 2] * (N - 1)
    h1 = (fi % 2) == 1
    x = x0 + torch.where(h1, C_ - 1 - s, s)
    y = y0 + torch.where(h1, C_ - 1 - t, t)
    xi, yi = torch.floor(x).long(), torch.floor(y).long()
    fx, fy = (x - xi)[:, None], (y - yi)[:, None]
    H, W = atlas.shape[:2]
    at = lambda yy, xx: atlas[yy.clamp(0, H - 1), xx.clamp(0, W - 1)].double()
    tex = ((1 - fx) * (1 - fy) * at(yi, xi) + fx * (1 - fy) * at(yi, xi + 1) + (1 - fx) * fy * at(yi + 1, xi) +
           fx * fy * at(yi + 1, xi + 1))
    vert = bary(diffuse).double()
    ref = ref.double()
    return float((tex - ref).abs().mean()), float((vert - ref).abs().mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", type=int, default=512)
    ap.add_argument("--frac", type=float, nargs="+", default=[0.1, 0.02])
    ap.add_argument("--texels", type=int, nargs="+", default=[4, 8, 16])
    ap.add_argument("--points", type=int, default=1 << 20)
    ap.add_argument("--limit", type=float, default=1.2)
    ap.add_argument("--iso", type=float, default=32.0)
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mesh_texture_bench needs a CUDA device")
    import nerfmeshes_b200 as nm
    from nerfmeshes_b200 import mesh
    from nerfmeshes_b200 import parallel as par
    from bench import load_npz, model_cfg

    model = nm.NeRFModel.from_npz(model_cfg(2.0, 6.0), load_npz("weights_lego_nerf.npz")).eval().cuda()
    eng = model._engine()
    args = SimpleNamespace(view_disparity=1e-2, view_disparity_max_bound=4.0)
    result = dict(card=card(), net="lego", res=a.res, limit=a.limit, iso_level=a.iso, reps=a.reps, points=a.points,
                  view_disparity=args.view_disparity, view_disparity_max_bound=args.view_disparity_max_bound, cases=[])
    A = SimpleNamespace(limit=a.limit, res=a.res, iso_level=a.iso)
    v, f, n, _ = par.extract_geometry_sharded(model, A, group=par.SINGLE, to_host=False)
    v, f, n = v.clone(), f.clone(), n.clone()
    result["faces"] = int(f.shape[0])
    tmp = tempfile.mkdtemp(prefix="mesh_texture_bench_")
    used, wf = torch.unique(f[:64].long(), return_inverse=True)
    wv, wn = mesh.rescale_vertices(v[used], a.limit, a.res), n[used].cpu()
    for N in a.texels:                                        # warm-up: every kernel and render shape once, on 64 faces
        eng.bake_texture(wv, wn, wf.int(), N, view_disparity=1e-2, near_far=(0.0, 4.0))
    for frac in a.frac:
        dv, dn, df, counts, _ = eng.mesh_decimate(v, n, f, int(frac * f.shape[0]))
        hv, hf, hn = mesh.rescale_vertices(dv, a.limit, a.res), df.cpu(), dn.cpu()
        _, t_app = timed(lambda: mesh.mesh_appearance(model, hv, hn, args), a.reps)
        case = dict(frac=frac, faces=counts[1], vertices=counts[0], vertex_appearance=t_app, texels=[])
        for N in a.texels:
            eng.set_timing(True)
            out, t_bake = timed(lambda: eng.bake_texture(hv, hn, hf, N, view_disparity=1e-2, near_far=(0.0, 4.0)), a.reps,
                                warmup=False)
            mlp_ms = eng.mlp_time_ms()[0] / a.reps
            eng.set_timing(False)
            u8, atlas, uv, diffuse, counts_t = out
            u8, uv, diffuse = u8.cpu().numpy(), uv.cpu().numpy(), diffuse.cpu().numpy()
            _, t_rays = timed(lambda: eng.debug_texture_rays(hv, hn, hf, N, 0, hf.shape[0], view_disparity=1e-2), a.reps,
                              warmup=False)
            path = os.path.join(tmp, f"m{N}.obj")
            _, t_png = timed(lambda: mesh.write_png(path[:-4] + ".png", u8), a.reps, warmup=False)
            _, t_all = timed(lambda: mesh.export_textured_obj(hv, hf, diffuse, hn, uv, u8, path), a.reps, warmup=False)
            err_tex, err_vert = surface_errors(model, hv, hf, hn, atlas, diffuse, N, args, a.points, seed=7)
            W, H = counts_t[0], counts_t[1]
            entry = dict(N=N, texels=counts_t[2], atlas=[W, H], bake=t_bake, rays=t_rays, render_mlp_ms=round(mlp_ms, 3),
                         rest_ms=round(t_bake["median_ms"] - t_rays["median_ms"] - mlp_ms, 3), png=t_png,
                         obj_ms=round(t_all["median_ms"] - t_png["median_ms"], 3), png_bytes=os.path.getsize(path[:-4] + ".png"),
                         mean_abs_err_texture=err_tex, mean_abs_err_vertex=err_vert)
            case["texels"].append(entry)
            print(f"{frac:g}: {counts[1]} faces, N = {N}: {entry['texels']} texels, {W} x {H}, bake {t_bake['median_ms']} ms "
                  f"(rays {t_rays['median_ms']}, network {mlp_ms:.1f}), error texture {err_tex:.4f} vs vertex "
                  f"{err_vert:.4f}", file=sys.stderr)
            del atlas
            torch.cuda.empty_cache()
        result["cases"].append(case)
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
