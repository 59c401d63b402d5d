"""Dense-grid density query + iso-surface extraction — mirror of src/mesh_nerf.py:27-92 on the fused path."""
from __future__ import annotations

import numpy as np
import torch

from . import _lib as L


def extract_radiance(model, args, device, nums, sigma_only=False, slab=None):
    """src/mesh_nerf.py:27-53.  Returns the (n0,n1,n2,4) numpy radiance grid like the reference, or — with
    sigma_only — the (n0,n1,n2) raw-density DEVICE tensor (the fast path extract_geometry uses; the reference
    discards the rgb channels anyway, mesh_nerf.py:73)."""
    assert isinstance(nums, (tuple, list, int)), "Nums arg should be either iterable or int."
    if isinstance(nums, int):
        nums = (nums,) * 3
    else:
        assert len(nums) == 3, "Nums arg should be of length 3, number of axes for 3D"
    tiles = [torch.linspace(-args.limit, args.limit, num) for num in nums]
    eng = model._engine()
    x0, x1 = slab if slab is not None else (0, nums[0])
    if sigma_only:
        return eng.grid_sigma(tiles, x0, x1)
    sigma, rgb = eng.grid_sigma(tiles, x0, x1, with_rgb=True)
    return torch.cat((rgb, sigma[..., None]), -1).cpu().numpy()


def clamp_iso_level(iso_level, mn, mx, sd):
    """src/mesh_nerf.py:65, in the arithmetic of the statistics it is given (np.float32 for a float32 grid)."""
    return min(max(iso_level, mn + sd), mx - sd)


def extract_iso_level(density, args, engine=None):
    """src/mesh_nerf.py:56-65: clamp(iso_level, min+std, max-std)."""
    if isinstance(density, torch.Tensor) and density.is_cuda:
        mn, mx, sd = engine.volume_stats(density)
        mn, mx, sd = np.float32(mn), np.float32(mx), np.float32(sd)
    else:
        density = np.asarray(density)
        mn, mx, sd = density.min(), density.max(), density.std()
    return clamp_iso_level(args.iso_level, mn, mx, sd)


def marching_cubes(volume, level, engine=None):
    """skimage.measure.marching_cubes(volume, level) seam (src/mesh_nerf.py:79): (verts, faces, normals, values)."""
    if engine is None:
        from .nerf_api import _engine
        engine = _engine()
    vol = torch.as_tensor(volume)
    verts, faces, normals = engine.marching_cubes(vol, float(level))
    values = torch.zeros(verts.shape[0])
    return verts.cpu().numpy(), faces.cpu().numpy(), normals.cpu().numpy(), values.numpy()


def super_sampling_tables(limit, nums, s):
    """Coordinate tables of super-sampled marching cubes (mesh_nerf.py:37,109): (lins, fines), per axis
    torch.linspace(-limit, limit, n) and torch.linspace(-limit, limit, n + (n-1)*s)."""
    if isinstance(nums, int):
        nums = (nums,) * 3
    lins = [torch.linspace(-limit, limit, n) for n in nums]
    fines = [torch.linspace(-limit, limit, n + (n - 1) * s) for n in nums]
    return lins, fines


def sweep_coordinates(verts, lins):
    """Marching-cubes vertices in index coordinates (V,3) -> the sweep's coordinates: per axis the torch.linspace table
    `lins[a]` interpolated at the index coordinate, so that an integer index gives the table's value bit for bit (the grid
    point the sweep sampled).  Not the exported coordinates, whose limit*(v/(res/2) - 1) scale drifts from linspace."""
    out = []
    for a in range(3):
        lin = lins[a].to(verts.device, torch.float32)
        v = verts[:, a]
        n = lin.shape[0]
        i0 = torch.floor(v).clamp(0, n - 1)
        frac = v - i0
        i0 = i0.long()
        i1 = (i0 + 1).clamp(max=n - 1)
        x0 = lin[i0]
        out.append(torch.where(frac == 0, x0, x0 + frac * (lin[i1] - x0)))
    return torch.stack(out, 1).contiguous()


def network_normals(eng, which, verts, lins, grid_normals):
    """n = -g / |g| with g the network's density gradient (nm_sigma_grad) at each vertex's sweep coordinates — the grid
    normals' convention, pointing towards decreasing sigma.  Where |g| is 0 or not finite the grid normal is kept.
    Returns (normals (V,3), number of vertices that kept their grid normal)."""
    if verts.shape[0] == 0:
        return grid_normals, 0
    _, g = eng.sigma_grad(which, sweep_coordinates(verts, lins), want_sigma=False)
    gn = grid_normals.to(g.device)
    norm = torch.sqrt(g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1] + g[:, 2] * g[:, 2])
    ok = torch.isfinite(norm) & (norm > 0)
    n = torch.where(ok[:, None], -g / torch.where(ok, norm, torch.ones_like(norm))[:, None], gn)
    return n, int((~ok).sum())


def _report_fallback(n_fallback, n_vertices):
    if n_fallback:
        print(f"network normals: {n_fallback} of {n_vertices} vertices have a zero or non-finite density gradient "
              "and keep their grid normal")


def remove_small_components(eng, verts, normals, faces, m):
    """Drop the connected components of the mesh with fewer than m faces (nm_mesh_components, DESIGN 4.9): the floaters of
    a NeRF mesh.  Kept vertices and faces stay in their original order, faces re-indexed; rows are copied unchanged.  m <= 0
    returns the inputs as they are.  Prints one line when something was dropped."""
    if m <= 0:
        return verts, normals, faces
    v, n, f, (kv, kf, comps, kept), _ = eng.mesh_components(verts, normals, faces, m)
    if kv < verts.shape[0] or kf < faces.shape[0]:
        print(f"small components: kept {kept} of {comps} components, {kf} of {faces.shape[0]} faces "
              f"(min_component_faces = {m})")
    return v, n, f


def decimate(eng, verts, normals, faces, target_faces, network=None):
    """Quadric-error decimation to at most target_faces faces (nm_mesh_decimate, DESIGN 4.11), on index-coordinate
    vertices.  Surviving vertices stay in input order; an unmoved vertex keeps its normal row, a moved one gets its faces'
    area-weighted winding normal, or with network = (which, lins) the network's normal at its new position
    (network_normals).  target_faces <= 0 returns the inputs as they are.  Prints one line."""
    if target_faces <= 0:
        return verts, normals, faces
    F = faces.shape[0]
    v, n, f, (_, kf, rounds, _), src = eng.mesh_decimate(verts, normals, faces, target_faces, want_source=network is not None)
    stuck = " (no legal collapse left)" if kf > target_faces else ""
    print(f"decimated {F} → {kf} faces in {rounds} rounds{stuck}")
    if network is not None and v.shape[0]:
        vin = verts.to(v.device)[src.long()]
        moved = torch.nonzero((v.view(torch.int32) != vin.view(torch.int32)).any(1)).reshape(-1)
        if moved.numel():
            nn, fb = network_normals(eng, network[0], v[moved], network[1], n[moved])
            n[moved] = nn
            _report_fallback(fb, int(moved.numel()))
    return v, n, f


def rescale_vertices(verts, limit, res):
    """Index coordinates -> (-limit, limit) with the reference's res/2 scale (src/mesh_nerf.py:82-90), on the host like the
    reference's CPU tensors so the rounding is identical (torch's CUDA division by a python scalar multiplies by the
    reciprocal, which differs in the last bit)."""
    return limit * (verts.cpu() / (res / 2.0) - 1.0)


def extract_geometry(model, device, args):
    """src/mesh_nerf.py:68-92: sigma sweep -> adaptive iso -> marching cubes -> rescale to (-limit, limit).  This is the
    one-slab case of the mesh pipeline (parallel._extract_mesh, which lists the stages and what args.super_sampling,
    args.network_normals, args.min_component_faces and args.decimate_faces do), in buffers that die with the call.
    Everything downstream (cache, appearance, OBJ) sees the filtered and decimated mesh.  `device` is the reference's argument and unused: the model's engine
    device is.  Returns CPU (vertices, triangles, normals) and the (res, res, res) numpy density grid; with
    args.sparse_sweep that grid holds +inf / -inf at the points the sparse sweep did not evaluate."""
    from .parallel import _extract_mesh      # parallel imports this module for the stage helpers above
    fresh = lambda key, numel, dtype, dev: torch.empty(numel, dtype=dtype, device=dev)
    verts, faces, normals, _, density = _extract_mesh(model, args, 0, 1, None, fresh)
    return rescale_vertices(verts, args.limit, args.res), faces.cpu(), normals.cpu(), density.cpu().numpy()


def extract_geometry_with_super_sampling(model, device, args):
    """src/mesh_nerf.py:95-128 (which raises NotImplementedError there): extract_geometry with
    args.super_sampling (>= 1) network samples per crossed grid edge."""
    assert int(getattr(args, "super_sampling", 0) or 0) >= 1, "super_sampling must be >= 1"
    return extract_geometry(model, device, args)


def _export_obj_python(vertices, triangles, diffuse, normals, filename):
    """Pure-python formatter (any dtype); the native writer below must produce the same bytes."""
    def rows(a):
        if isinstance(a, torch.Tensor):
            a = a.detach().cpu()
            if a.dtype.is_floating_point:
                return [[repr(x) for x in r] for r in a.double().tolist()]
            return [[str(x) for x in r] for r in a.tolist()]
        a = np.asarray(a)
        if a.dtype.kind == "f":                      # "{}".format(np.float32) widens to a python float first
            return [[repr(x) for x in r] for r in a.astype(np.float64).tolist()]
        return [[str(x) for x in r] for r in a.tolist()]

    v, n, d = rows(vertices), rows(normals), rows(diffuse) if len(diffuse) else []
    out = []
    for i, r in enumerate(v):
        out.append("v " + " ".join(r) + (" " + " ".join(d[i]) if len(d) > i else "") + "\n")
    out.extend("vn " + " ".join(r) + "\n" for r in n)
    tri = triangles.detach().cpu().numpy() if isinstance(triangles, torch.Tensor) else np.asarray(triangles)
    out.extend("f" + "".join(f" {i + 1}//{i + 1}" for i in r) + "\n" for r in tri.tolist())
    with open(filename, "w") as fh:
        fh.writelines(out)


def export_obj(vertices, triangles, diffuse, normals, filename):
    """src/nerf/nerf_helpers.py:86-111, byte-identical text: `v x y z [r g b]`, `vn x y z`, `f i//i j//j k//k` (1-based).
    The reference formats every float32 (torch or numpy) through python's format(): the value widened to double, shortest
    round-trip repr.  float32 inputs (what the mesh path produces) go through the library's native writer
    (nm_export_obj: ~1 s per million vertices); anything else through the python formatter with the same output."""
    def arr(a):
        return a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    v, n, t = arr(vertices), arr(normals), arr(triangles)
    d = arr(diffuse) if len(diffuse) else np.zeros((0, 3), np.float32)
    native = all(x.dtype == np.float32 and x.ndim == 2 and x.shape[1] == 3 for x in (v, n, d)) and t.dtype.kind in "iu" and \
        t.ndim == 2 and t.shape[1] == 3 and (t.size == 0 or int(t.max()) < 2 ** 31 - 1)
    if not native:
        return _export_obj_python(vertices, triangles, diffuse, normals, filename)
    import ctypes as C
    v, n, d = np.ascontiguousarray(v), np.ascontiguousarray(n), np.ascontiguousarray(d)
    t = np.ascontiguousarray(t, dtype=np.int32)
    ptr = lambda a: C.c_void_p(a.ctypes.data) if a.size else None
    L.check(L.load().nm_export_obj(str(filename).encode(), ptr(v), v.shape[0], ptr(t), t.shape[0], ptr(d), d.shape[0],
                                   ptr(n), n.shape[0]))


def load_obj(path):
    """pytorch3d.io.load_obj's verts / faces.verts_idx for what the commented-out target-mesh loader reads
    (src/data/datasets.py:88-103): `v x y z [extra]` lines (per-vertex colours, as export_obj writes them, are ignored) and
    `f` lines with `a`, `a/b`, `a//c` or `a/b/c` entries, 1-based or negative (relative to the vertices read so far);
    polygons are fan-triangulated.  Returns (float32 (V,3), int32 (F,3)) CPU tensors."""
    verts, faces = [], []
    with open(path) as fh:
        for line in fh:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == "v":
                verts.append([float(x) for x in tok[1:4]])
            elif tok[0] == "f":
                ids = []
                for t in tok[1:]:
                    i = int(t.split("/")[0])
                    ids.append(i - 1 if i > 0 else len(verts) + i)
                if len(ids) < 3:
                    raise ValueError(f"{path}: face with fewer than 3 vertices: {line.strip()}")
                faces.extend([ids[0], ids[k], ids[k + 1]] for k in range(1, len(ids) - 1))
    v = torch.tensor(np.asarray(verts, dtype=np.float32).reshape(-1, 3))
    f = torch.tensor(np.asarray(faces, dtype=np.int32).reshape(-1, 3))
    return v, f


def mesh_appearance(model, vertices, normals, args):
    """The appearance pass of export_marching_cubes (src/mesh_nerf.py:160-192): per-vertex colour, either the raw network
    colour at the vertex (no_view_dependence) or a short ray cast along -normal through model.query — one batched call
    on the device instead of the reference's batchify loop."""
    targets, directions = vertices, -normals
    if getattr(args, "no_view_dependence", False):
        return model.sample_points(targets.cuda(), directions.cuda())[..., :3].cpu().numpy()
    ray_bounds = torch.tensor([0.0, args.view_disparity_max_bound], dtype=directions.dtype)
    ray_origins = targets - args.view_disparity * directions
    return model.query((ray_origins.cuda(), directions.cuda(), ray_bounds)).rgb_map.cpu().numpy()


def bake_texture(model, vertices, triangles, normals, args):
    """mesh_appearance per texel instead of per vertex (nm_bake_texture, DESIGN 4.12): args.texture_texels = N texels along
    each triangle leg, the query of every texel built from its face's barycentric point and normal with mesh_appearance's
    mode, bounds and disparity.  vertices: world coordinates (what extract_geometry returns and the cache stores).  Returns
    numpy (atlas_u8 (H,W,3) uint8, uv (F,3,2) float32, diffuse (V,3) float32); diffuse is the colour of each vertex's corner
    texel, which is mesh_appearance's colour of that vertex bit for bit."""
    from .models import _cfg_get
    eng = model._engine()
    mode = 1 if getattr(args, "no_view_dependence", False) else 0
    buff = hasattr(model, "tree")
    if mode == 0 and buff:                        # what BuFFModel.forward does before it renders
        model._sync_tree(eng)
        eng.voxel_random = bool(_cfg_get(model.cfg, "tree.use_random_sampling", False))
    u8, _, uv, rgb, _ = eng.bake_texture(vertices, normals, triangles, int(args.texture_texels), mode=mode,
                                         which=model.get_model()._owner[1], flags=eng._flags(model.training, buff),
                                         view_disparity=float(args.view_disparity),
                                         near_far=(0.0, float(getattr(args, "view_disparity_max_bound", 0.0))))
    return u8.cpu().numpy(), uv.cpu().numpy(), rgb.cpu().numpy()


def write_png(path, rgb):
    """An 8-bit RGB PNG of rgb (H,W,3) uint8, row 0 on top: every scanline with filter 0, one zlib stream."""
    import struct
    import zlib
    a = np.ascontiguousarray(rgb, dtype=np.uint8)
    H, W, _ = a.shape
    raw = np.concatenate([np.zeros((H, 1), np.uint8), a.reshape(H, W * 3)], 1).tobytes()

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)
    with open(path, "wb") as fh:
        fh.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, 2, 0, 0, 0)) +
                 chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b""))


def export_textured_obj(vertices, triangles, diffuse, normals, uv, atlas_u8, filename):
    """export_obj with a texture: the OBJ through nm_export_obj_textured (its `v` / `vn` lines are export_obj's bytes for
    float32 inputs), `<stem>.mtl` naming `<stem>.png`, and the atlas as that PNG.  Returns the three paths."""
    import ctypes as C
    import os
    stem = os.path.splitext(str(filename))[0]
    base = os.path.basename(stem)
    arr = lambda a, dt: np.ascontiguousarray(a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a), dtype=dt)
    v, n, d, t = arr(vertices, np.float32), arr(normals, np.float32), arr(diffuse, np.float32), arr(triangles, np.int32)
    w = arr(uv, np.float32)
    assert w.shape == (t.shape[0], 3, 2), (w.shape, t.shape)
    ptr = lambda a: C.c_void_p(a.ctypes.data) if a.size else None
    L.check(L.load().nm_export_obj_textured(str(filename).encode(), ptr(v), v.shape[0], ptr(t), t.shape[0], ptr(d),
                                            d.shape[0] if d.size else 0, ptr(n), n.shape[0], ptr(w), (base + ".mtl").encode()))
    with open(stem + ".mtl", "w") as fh:
        fh.write(f"newmtl texture\nKa 1.0 1.0 1.0\nKd 1.0 1.0 1.0\nKs 0.0 0.0 0.0\nillum 1\nmap_Kd {base}.png\n")
    write_png(stem + ".png", atlas_u8)
    return str(filename), stem + ".mtl", stem + ".png"


def _raster_inputs(eng, vertices, triangles, diffuse, texture):
    """The mesh and its colouring on the engine's device, once: vertices fp32, faces int32, colours fp32, and the atlas in fp32
    (a uint8 atlas, as bake_texture returns it, divided by 255 on the device)."""
    if (diffuse is None) == (texture is None):
        raise ValueError("render_mesh needs exactly one of diffuse= and texture=")
    from .engine import raster_faces
    v = torch.as_tensor(vertices).to(eng.device, torch.float32).contiguous()
    f = raster_faces(triangles, eng.device)
    col = None if diffuse is None else torch.as_tensor(diffuse).to(eng.device, torch.float32).contiguous()
    atlas, N = (None, 0) if texture is None else texture
    if atlas is not None:
        atlas = torch.as_tensor(atlas).to(eng.device)
        atlas = atlas.to(torch.float32) / 255.0 if atlas.dtype == torch.uint8 else atlas.to(torch.float32)
    return v, f, col, atlas, int(N)


def render_mesh(model_or_engine, vertices, triangles, pose, H, W, focal, *, diffuse=None, texture=None, background=(0.0, 0.0, 0.0)):
    """An image of the mesh from a camera pose (nm_rasterize_mesh, DESIGN 4.13), through the pinhole camera render_image uses
    without NDC, so that pixel (c, r) lies on the ray NeRF pixel (c, r) renders.  vertices: world coordinates (what
    extract_geometry returns and the cache stores); colours from diffuse (V,3) (mesh_appearance's output) or texture =
    (atlas, N) (bake_texture's atlas of these faces, uint8 or float).  Returns {"rgb": (H,W,3), "depth": (H,W) distance along
    the ray, "face": (H,W) int32, -1 where the mesh is not seen, "counts": (covered pixels, faces drawn, faces culled)}, device
    tensors."""
    from .engine import Engine
    eng = model_or_engine if isinstance(model_or_engine, Engine) else model_or_engine._engine()
    v, f, col, atlas, N = _raster_inputs(eng, vertices, triangles, diffuse, texture)
    outs, counts = eng.rasterize_mesh(v, f, pose, int(H), int(W), float(focal), colors=col, atlas=atlas, N=N, background=background)
    outs["counts"] = counts
    return outs


def _psnr(mse):
    return float("inf") if mse == 0 else -10.0 * float(np.log10(mse))


def compare_with_nerf(model, vertices, triangles, poses, H, W, focal, near, far, *, diffuse=None, texture=None):
    """Score a mesh against the NeRF it came from, view by view: for each pose the NeRF image (render_image) and the mesh image
    (render_mesh) on the same background (white when the model's config asks for it, else black).  Per view: PSNR of the mesh
    image against the NeRF image over all pixels; PSNR over the pixels both cover (mesh face != -1 and NeRF acc > 0.5);
    silhouette IoU of the mesh's coverage against acc > 0.5; mean |depth difference| over the pixels both cover, against the
    NeRF's expected hit distance depth_raw / acc; and the number of pixels both cover.  A view where no pixel is covered by
    both has NaN for the masked values.  Returns {"psnr", "psnr_masked", "iou", "depth_mae", "both": per-view lists, "mean":
    the means over the views where a value exists}.  NDC scenes raise NotImplementedError."""
    from .models import _cfg_get
    if _cfg_get(model.cfg, "dataset.use_ndc", False):
        raise NotImplementedError("compare_with_nerf: the scene uses NDC rays, so its mesh lives in NDC space; mapping it back "
                                  "to world space is not implemented")
    eng = model._engine()
    buff = hasattr(model, "tree")
    if buff:                                           # what BuFFModel.forward does before it renders
        model._sync_tree(eng)
        eng.voxel_random = bool(_cfg_get(model.cfg, "tree.use_random_sampling", False))
    bg = (1.0, 1.0, 1.0) if model.volume_renderer.white_background else (0.0, 0.0, 0.0)
    v, f, col, atlas, N = _raster_inputs(eng, vertices, triangles, diffuse, texture)
    out = dict(psnr=[], psnr_masked=[], iou=[], depth_mae=[], both=[])
    for pose in poses:
        n = eng.render_image(pose, H, W, focal, near, far, buff=buff, want=("rgb", "depth_raw", "acc"))
        m, _ = eng.rasterize_mesh(v, f, pose, int(H), int(W), float(focal), colors=col, atlas=atlas, N=N, background=bg)
        n_rgb, acc = n["rgb"].view(H, W, 3).double(), n["acc"].view(H, W)
        m_rgb = m["rgb"].double()
        mesh_in, nerf_in = m["face"] >= 0, acc > 0.5
        both, union = mesh_in & nerf_in, mesh_in | nerf_in
        err2 = (m_rgb - n_rgb) ** 2
        out["psnr"].append(_psnr(float(err2.mean())))
        nb = int(both.sum())
        out["both"].append(nb)
        out["psnr_masked"].append(_psnr(float(err2[both].mean())) if nb else float("nan"))
        nu = int(union.sum())
        out["iou"].append(nb / nu if nu else float("nan"))
        nerf_depth = n["depth_raw"].view(H, W).double() / acc.double()
        out["depth_mae"].append(float((m["depth"].double() - nerf_depth)[both].abs().mean()) if nb else float("nan"))
    out["mean"] = {k: _mean_defined(v_) for k, v_ in out.items()}
    return out


def _mean_defined(xs):
    """The mean of the values that are not NaN, or NaN when none is."""
    xs = [x for x in xs if not np.isnan(x)]
    return float(np.mean(xs)) if xs else float("nan")


def cached_geometry(args, build):
    """The mesh cache of export_marching_cubes (src/mesh_nerf.py:141-158): a torch.save'd tuple
    (vertices, triangles, normals, density) at save_dir/cache_name, loaded when --use-cached-mesh is set and the file
    exists, (re)written when it was requested but missing or --override-cache-mesh is set.  `build()` produces the tuple.
    With args.sparse_sweep the cached density holds +-inf at the points the sparse sweep did not evaluate."""
    import os
    use = bool(getattr(args, "use_cached_mesh", False))
    name = getattr(args, "cache_name", None)
    path = os.path.join(args.save_dir, name) if name else None
    exists = bool(path) and os.path.exists(path)
    if use and exists:
        return tuple(torch.load(path, weights_only=False))
    out = build()
    if path and ((use and not exists) or getattr(args, "override_cache_mesh", False)):
        torch.save(tuple(out), path)
    return out


def export_marching_cubes(model, args, cfg=None, device="cuda"):
    """src/mesh_nerf.py:131-201: geometry (or its cache) -> appearance -> OBJ.  With args.super_sampling >= 1 the geometry
    comes from super-sampled marching cubes (extract_geometry) and the cache stores the refined vertices.  The reference's
    branch would have written a geometry-only OBJ through PyMCubes but raises before it runs, so there is no behaviour to
    match: the refined mesh goes through the same appearance pass and OBJ writer as s = 0.  With args.texture_texels = N > 0
    the appearance is baked into a texture instead (bake_texture) and the OBJ comes with `<stem>.mtl` and `<stem>.png`; its
    vertex colours are the ones mesh_appearance would give.  A mesh without faces gets the untextured OBJ."""
    import os
    vertices, triangles, normals, density = cached_geometry(args, lambda: extract_geometry(model, device, args))
    path = os.path.join(args.save_dir, args.mesh_name)
    if int(getattr(args, "texture_texels", 0) or 0) > 0:
        if len(triangles):
            atlas, uv, diffuse = bake_texture(model, vertices, triangles, normals, args)
            export_textured_obj(vertices, triangles, diffuse, normals, uv, atlas, path)
            return path
        print("texture bake: the mesh has no faces; writing the untextured OBJ")
    diffuse = mesh_appearance(model, vertices, normals, args)
    export_obj(vertices, triangles, diffuse, normals, path)
    return path


# ---------------------------------------------------------------------------------------------- surface point clouds (DESIGN 4.14)
def surface_ray_poses(samples_y=8, samples_x=4, radius=4.0):
    """The ring of src/mesh_surface_ray.py:80-87: pose_spherical(θ, φ, radius) with θ from linspace(-180, 180, samples_y,
    endpoint=False) on the outer loop and φ from linspace(-90, 90, samples_x) on the inner one.  A list of (4,4) float32."""
    from .nerf_api import pose_spherical
    return [pose_spherical(float(th), float(ph), float(radius)) for th in np.linspace(-180, 180, samples_y, endpoint=False)
            for ph in np.linspace(-90, 90, samples_x)]


def surface_min_count(step, prob_threshold):
    """The neighbour count a pixel needs: the script's `sum > size_samples * prob_threshold` (size_samples = (2s+1)^2 - 1)
    as an integer bound, floor(size_samples * prob_threshold) + 1, in python double arithmetic."""
    if not 0.0 <= prob_threshold <= 1.0:
        raise ValueError(f"prob_threshold {prob_threshold} is outside [0, 1]")
    size = 2 * int(step) + 1
    return int(np.floor((size * size - 1) * float(prob_threshold))) + 1


def surface_points(model, poses, H, W, focal, near, far, *, step=2, dist_threshold=0.002, prob_threshold=0.6, min_acc=1.0,
                   network_normals=False):
    """Depth-consistent surface points of a NeRF seen from `poses` (nm_surface_points, DESIGN 4.14; the algorithm of the
    reference's dead src/mesh_surface_ray.py).  Each pose is rendered in validation mode (render_image: rgb, depth_raw, acc);
    a pixel's point is o + d*t with t = depth_raw where acc >= min_acc, and it is kept when t > 0 and at least
    surface_min_count(step, prob_threshold) of its (2*step+1)^2 clamped pixel neighbours lie within squared distance
    dist_threshold.  normals = -d, or with network_normals -∇σ/|∇σ| of the net density_gradient uses (-d kept, and counted
    in a printed line, where the gradient is zero or not finite).  Views are filtered one at a time, so memory is one view's
    scratch plus the output.  Returns device tensors {"points", "normals", "colors": (N,3), "view", "pixel": (N,) int32, in
    (view, row, column) order}, and "counts": the kept points per view.  NDC scenes raise NotImplementedError."""
    from .models import _cfg_get
    if _cfg_get(model.cfg, "dataset.use_ndc", False):
        raise NotImplementedError("surface_points: the scene uses NDC rays, whose depths are not world distances; mapping them "
                                  "back to world space is not implemented")
    min_count = surface_min_count(step, prob_threshold)
    eng = model._engine()
    buff = hasattr(model, "tree")
    if buff:                                           # what BuFFModel.forward does before it renders
        model._sync_tree(eng)
        eng.voxel_random = bool(_cfg_get(model.cfg, "tree.use_random_sampling", False))
    which = model.get_model()._owner[1]
    n = int(H) * int(W)
    scratch = dict(points=torch.empty((n, 3), dtype=torch.float32, device=eng.device),
                   normals=torch.empty((n, 3), dtype=torch.float32, device=eng.device),
                   colors=torch.empty((n, 3), dtype=torch.float32, device=eng.device),
                   pixel=torch.empty((n,), dtype=torch.int32, device=eng.device))
    parts = {k: [] for k in ("points", "normals", "colors", "view", "pixel")}
    counts, fallback = [], 0
    for i, pose in enumerate(poses):
        r = eng.render_image(pose, H, W, focal, near, far, buff=buff, want=("rgb", "depth_raw", "acc"))
        outs, k = eng.surface_points(pose, H, W, focal, r["depth_raw"], r["acc"], r["rgb"], min_acc=min_acc, step=step,
                                     dist_threshold=dist_threshold, min_count=min_count, out=scratch)
        del r
        nrm = outs["normals"]
        if network_normals and k:
            _, g = eng.sigma_grad(which, outs["points"], want_sigma=False)
            norm = torch.sqrt(g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1] + g[:, 2] * g[:, 2])
            ok = torch.isfinite(norm) & (norm > 0)
            nrm = torch.where(ok[:, None], -g / torch.where(ok, norm, torch.ones_like(norm))[:, None], nrm)
            fallback += int((~ok).sum())
        for key in ("points", "colors", "pixel"):
            parts[key].append(outs[key].clone())
        parts["normals"].append(nrm.clone())
        parts["view"].append(torch.full((k,), i, dtype=torch.int32, device=eng.device))
        counts.append(k)
    if network_normals and fallback:
        print(f"network normals: {fallback} of {sum(counts)} surface points have a zero or non-finite density gradient "
              "and keep -d")
    res = {key: (torch.cat(v, 0) if v else scratch[key][:0].clone()) for key, v in parts.items() if key != "view"}
    res["view"] = torch.cat(parts["view"], 0) if parts["view"] else torch.zeros((0,), dtype=torch.int32, device=eng.device)
    res["counts"] = counts
    return res


def ply_colors(colors):
    """Colours as PLY uchar: trunc(fl32(c*255)) clamped to [0, 255], NaN to 0 (numpy, any float input cast to float32)."""
    v = np.asarray(colors, dtype=np.float32) * np.float32(255.0)
    with np.errstate(invalid="ignore"):
        q = np.where(v > 0, np.minimum(np.trunc(v), 255.0), 0.0)
    return q.astype(np.uint8)


def ply_header(n, binary=False):
    fmt = "binary_little_endian" if binary else "ascii"
    props = "".join(f"property float {p}\n" for p in ("x", "y", "z", "nx", "ny", "nz"))
    props += "".join(f"property uchar {p}\n" for p in ("red", "green", "blue"))
    return f"ply\nformat {fmt} 1.0\nelement vertex {n}\n{props}end_header\n".encode()


def _export_ply_python(points, colors, normals, filename, binary=False):
    """Pure-python formatter (any dtype; values become the format's float32 and uchar); the native writer below must
    produce the same bytes."""
    arr = lambda a: np.asarray(a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a, dtype=np.float32).reshape(-1, 3)
    p, n = arr(points), arr(normals)
    q = ply_colors(arr(colors))
    out = [ply_header(p.shape[0], binary)]
    if binary:
        rec = np.empty(p.shape[0], dtype=[("p", "<f4", (3,)), ("n", "<f4", (3,)), ("c", "u1", (3,))])
        rec["p"], rec["n"], rec["c"] = p, n, q
        out.append(rec.tobytes())
    else:
        out.extend((" ".join("%.18g" % x for x in a.tolist() + b.tolist()) + " " + " ".join(str(x) for x in c.tolist())
                    + "\n").encode() for a, b, c in zip(p.astype(np.float64), n.astype(np.float64), q))
    with open(filename, "wb") as fh:
        fh.writelines(out)


def export_ply(points, colors, normals, filename, binary=False):
    """src/mesh_surface_ray.py:45-57's PLY (plyfile's layout): `element vertex N`, float x y z nx ny nz, uchar red green blue.
    Text rows hold the nine values as %.18g separated by single spaces; binary=True writes binary_little_endian 27-byte
    records.  Colours become trunc(fl32(c*255)) clamped to [0, 255], NaN 0.  float32 (N,3) inputs go through the library's
    native writer (nm_export_ply); anything else through the python formatter with the same output."""
    def arr(a):
        return a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
    p, c, n = arr(points), arr(colors), arr(normals)
    if not all(x.dtype == np.float32 and x.ndim == 2 and x.shape == p.shape and x.shape[1:] == (3,) for x in (p, c, n)):
        return _export_ply_python(points, colors, normals, filename, binary)
    import ctypes as C
    p, c, n = np.ascontiguousarray(p), np.ascontiguousarray(c), np.ascontiguousarray(n)
    ptr = lambda a: C.c_void_p(a.ctypes.data) if a.size else None
    L.check(L.load().nm_export_ply(str(filename).encode(), ptr(p), ptr(c), ptr(n), p.shape[0], int(bool(binary))))


def export_surface_points(model, args):
    """src/mesh_surface_ray.py:66-141 (export_ray_trace) on the fused path: the 32 ring poses of surface_ray_poses at radius
    4.0, args.img_size x args.img_size pixels (800) at args.focal (1111.1111), near / far from the config's dataset.near /
    dataset.far, step args.step_size (2), args.dist_threshold (0.002), args.prob_threshold (0.6), args.min_acc (1.0),
    args.network_normals (False), written by export_ply to save_dir/args.ply_name ('lego-sampling.ply'), binary with
    args.ply_binary.  Returns the path."""
    import os
    from .models import _cfg_get
    g = lambda k, d: d if getattr(args, k, None) is None else getattr(args, k)
    size = int(g("img_size", 800))
    near, far = _cfg_get(model.cfg, "dataset.near"), _cfg_get(model.cfg, "dataset.far")
    if near is None or far is None:
        raise ValueError("export_surface_points: the model's config has no dataset.near / dataset.far")
    r = surface_points(model, surface_ray_poses(), size, size, float(g("focal", 1111.1111)), float(near), float(far),
                       step=int(g("step_size", 2)), dist_threshold=float(g("dist_threshold", 0.002)),
                       prob_threshold=float(g("prob_threshold", 0.6)), min_acc=float(g("min_acc", 1.0)),
                       network_normals=bool(g("network_normals", False)))
    path = os.path.join(args.save_dir, g("ply_name", "lego-sampling.ply"))
    export_ply(r["points"], r["colors"], r["normals"], path, binary=bool(g("ply_binary", False)))
    print(f"surface points: {r['points'].shape[0]} points from {len(r['counts'])} views -> {path}")
    return path
