"""Multi-GPU sharding of the hot path (SURVEY section 8e): one process per GPU, independent units, ONE exchange step.

Render: contiguous image-row shards, every rank generates its own rays from the 12-float pose; results are bit-identical
to the single-GPU image (no cross-shard arithmetic), the exchange is one all_gather of the finished rows.
Mesh: ONE pipeline (_extract_mesh) over x-slabs of the density grid, which single-GPU mesh.extract_geometry runs as its
one-slab case; every grid point (vertex, cell) is owned by exactly one rank; halo planes by send/recv; per-slab marching
cubes in global index coordinates with globally consistent vertex ids; the exchange is an all_gather of the vertex /
triangle counts and ONE all_gather of the per-slab indexed meshes (padded to the largest slab), plus two tiny all_gathers
for the iso-level statistics (extract_iso_level, src/mesh_nerf.py:56-65).  The gathered arrays equal the one-slab arrays
bit for bit.
Training: data parallel over rays — every rank runs forward + backward on its own ray batch (no collective inside), then
ONE all_reduce of the flattened gradients of both networks (595 k - 1.19 M floats, 4.8 MB) before the optimiser step.
The collectives go through torch.distributed (NCCL on GPUs, gloo in the CPU tests); there is no data-path collective
inside a shard's computation.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import torch.distributed as dist

from . import mesh


def row_shard(H: int, rank: int, world: int) -> Tuple[int, int]:
    """Rows [r0, r1) of rank `rank`: H split as evenly as possible, earlier ranks take the remainder."""
    base, rem = divmod(H, world)
    r0 = rank * base + min(rank, rem)
    return r0, r0 + base + (1 if rank < rem else 0)


def slab_shard(n0: int, rank: int, world: int) -> Tuple[int, int]:
    """Planes [x0, x1) of the grid's slowest axis owned by `rank` such that the n0-1 cell layers are split evenly and
    neighbouring slabs share one plane (cells between planes x1-1 and x1 belong to the next rank's first plane)."""
    c0, c1 = row_shard(n0 - 1, rank, world)          # cell layers [c0, c1)
    return c0, c1 + 1                                # planes c0 .. c1 inclusive


def _all_gather_padded(t: torch.Tensor, group=None):
    """all_gather of tensors whose first dimension differs per rank -> list of per-rank tensors."""
    world = dist.get_world_size(group)
    n = torch.tensor([t.shape[0]], dtype=torch.int64, device=t.device)
    counts = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(counts, n, group=group)
    counts = [int(c) for c in counts]
    mx = max(counts)
    pad = torch.zeros((mx,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    pad[: t.shape[0]] = t
    out = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(out, pad, group=group)
    return [o[:c] for o, c in zip(out, counts)]


def gather_rows(local: Dict[str, torch.Tensor], group=None) -> Dict[str, torch.Tensor]:
    """Concatenate per-rank row shards (rank order == row order) of every output map."""
    return {k: torch.cat(_all_gather_padded(v.contiguous(), group), 0) for k, v in local.items()}


def gather_mesh(verts: torch.Tensor, faces: torch.Tensor, normals: Optional[torch.Tensor] = None, group=None):
    """Concatenate per-slab indexed meshes; face indices are shifted by the exclusive scan of the vertex counts.
    Vertices on shared planes appear once per adjacent slab with identical bits (use torch.unique for the set)."""
    vs = _all_gather_padded(verts.contiguous(), group)
    fs = _all_gather_padded(faces.contiguous(), group)
    ns = _all_gather_padded(normals.contiguous(), group) if normals is not None else None
    off, shifted = 0, []
    for v, f in zip(vs, fs):
        shifted.append(f + off)
        off += v.shape[0]
    return torch.cat(vs, 0), torch.cat(shifted, 0), (torch.cat(ns, 0) if ns is not None else None)


def global_stats(local_min: float, local_max: float, local_sum: float, local_sumsq_centered_fn, count: int, device, group=None):
    """min / max / population std of a sharded volume: two rounds (mean first, then centred squares) so the result
    matches the two-pass single-GPU computation."""
    t = torch.tensor([local_min, -local_max], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
    s = torch.tensor([local_sum, float(count)], dtype=torch.float64, device=device)
    dist.all_reduce(s, op=dist.ReduceOp.SUM, group=group)
    mean = float(s[0] / s[1])
    q = torch.tensor([local_sumsq_centered_fn(mean)], dtype=torch.float64, device=device)
    dist.all_reduce(q, op=dist.ReduceOp.SUM, group=group)
    return float(t[0]), float(-t[1]), math.sqrt(float(q[0]) / float(s[1]))


def allreduce_gradients(params, group=None, average=True):
    """Data-parallel training step, exchange part: one all_reduce over the flattened .grad of `params` (the parameters of
    both FlexibleNeRFModels); the mean over ranks is what a single process would get from the concatenated ray batch
    when every rank's loss is a mean over equally many rays (src/models/model_nerf.py:118-126)."""
    grads = [p.grad for p in params if p.grad is not None]
    if not grads or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return 0
    flat = torch.cat([g.reshape(-1) for g in grads])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    if average:
        flat /= dist.get_world_size(group)
    off = 0
    for g in grads:
        g.copy_(flat[off:off + g.numel()].view_as(g))
        off += g.numel()
    return int(flat.numel())


class RowExchange:
    """The exchange step of a row-sharded image (SURVEY 8e): one flat buffer per rank, laid out map after map
    ([rgb | depth | acc | disp], every segment padded to the largest shard), which the render kernels fill through
    `views`, and ONE `all_gather_into_tensor` (NCCL over NVLink) that leaves every full map on every rank."""
    MAPS = ("rgb", "depth", "depth_raw", "acc", "disp", "coarse_rgb", "coarse_acc", "coarse_disp")

    def __init__(self, device, H, W, want=("rgb", "depth", "acc", "disp"), group=None):
        self.group, self.H, self.W, self.want = group, H, W, tuple(want)
        assert all(k in self.MAPS for k in self.want), "only per-ray maps can be exchanged"
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.r0, self.r1 = row_shard(H, self.rank, self.world)
        self.widths = {k: (3 if k.endswith("rgb") else 1) for k in self.want}
        self.rmax = (H + self.world - 1) // self.world * W            # rays of the largest shard
        C = sum(self.widths.values())
        self.local = torch.empty(C * self.rmax, dtype=torch.float32, device=device)
        self.full = torch.empty(self.world * C * self.rmax, dtype=torch.float32, device=device)
        R, off = (self.r1 - self.r0) * W, 0
        self.views = {}
        for k in self.want:
            w = self.widths[k]
            self.views[k] = self.local[off:off + w * R].view((R, 3) if w == 3 else (R,))
            off += w * self.rmax

    def gather(self):
        dist.all_gather_into_tensor(self.full, self.local, group=self.group)
        full = self.full.view(self.world, -1)
        out, off = {}, 0
        n = self.H * self.W
        for k in self.want:
            w = self.widths[k]
            if self.H % self.world == 0:
                seg = full[:, off:off + w * self.rmax].reshape((n, 3) if w == 3 else (n,))
            else:
                spans = [row_shard(self.H, r, self.world) for r in range(self.world)]
                parts = [full[r, off:off + w * (b - a) * self.W] for r, (a, b) in enumerate(spans)]
                seg = torch.cat(parts).view((n, 3) if w == 3 else (n,))
            out[k] = seg
            off += w * self.rmax
        return out


_EXCHANGES = {}


def row_exchange(device, H, W, want, group=None) -> RowExchange:
    key = (str(device), H, W, tuple(want), id(group))
    if key not in _EXCHANGES:
        _EXCHANGES.clear()
        _EXCHANGES[key] = RowExchange(device, H, W, want, group)
    return _EXCHANGES[key]


def render_image_sharded(model, pose, H, W, focal, near, far, *, ndc=False, buff=False, want=("rgb", "depth", "acc", "disp"),
                         group=None, seed=0):
    """eval_nerf.py's image loop on N GPUs (SURVEY 8e): this rank renders image rows [r0, r1) — rays generated on the device
    from the pose, kernels writing straight into this rank's segment of the exchange buffer — then ONE all_gather assembles
    every output map on every rank.  No arithmetic crosses a shard boundary, so the assembled maps are bit-identical to
    the single-GPU image."""
    eng = model._engine()
    if buff:
        model._sync_tree(eng)
    ex = row_exchange(eng.device, H, W, want, group)
    eng.render_image(pose, H, W, focal, near, far, ndc=ndc, rows=(ex.r0, ex.r1), buff=buff, seed=seed, want=list(ex.want),
                     out=ex.views)
    return ex.gather()


_MESH_BUFFERS = {}


def _scratch(key, numel, dtype, device):
    """Grow-only scratch tensors of the mesh path (slab buffer, exchange segment, gathered segments): steady-state calls
    make no allocator traffic.  Tensors returned by extract_geometry_sharded(to_host=False) are views of these buffers
    and stay valid until the next call with as many slabs: the segments are keyed by the slab count, so a one-slab result
    survives the N-slab call it is compared with."""
    t = _MESH_BUFFERS.get((key, str(device)))
    if t is None or t.numel() < numel or t.dtype != dtype:
        t = torch.empty(int(numel * 1.25) + 16, dtype=dtype, device=device)
        _MESH_BUFFERS[(key, str(device))] = t
    return t[:numel]


SINGLE = "single"        # pass as `group` to run the sharded code paths as ONE shard (tests compare it with the N-rank result)


def _rank_world(group=None):
    if group is SINGLE or group == SINGLE:
        return 0, 1
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(group), dist.get_world_size(group)
    return 0, 1


class _StageTimer:
    """CUDA-event stage timing on the current stream (filled into a caller-supplied dict as `<stage>_ms`)."""

    def __init__(self, sink):
        self.sink, self.marks = sink, []

    def mark(self, name=None):
        if self.sink is None:
            return
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        self.marks.append((name, e))

    def finish(self):
        if self.sink is None:
            return
        torch.cuda.current_stream().synchronize()
        for (_, a), (name, b) in zip(self.marks, self.marks[1:]):
            self.sink[name + "_ms"] = self.sink.get(name + "_ms", 0.0) + a.elapsed_time(b)


def slab_layout(n0: int, rank: int, world: int):
    """x-slab of rank `rank` of a grid with n0 planes (SURVEY 8e): returns (own0, own1, buf0, buf1).
    Points (and the cells above them) of planes [own0, own1) are OWNED: the n0-1 cell layers are split evenly and the last
    rank also owns the top plane n0-1.  Marching cubes additionally needs, where they exist, plane own1 (upper corners of
    the last owned cell layer), own1+1 and own0-1 (central-difference normals): the buffer is planes [buf0, buf1)."""
    c0, c1 = row_shard(n0 - 1, rank, world)
    own1 = n0 if rank == world - 1 else c1
    return c0, own1, max(c0 - 1, 0), min(own1 + 2, n0)


def exchange_halo_planes(buf: torch.Tensor, n0: int, rank: int, world: int, group=None):
    """Fill the halo planes of `buf` (planes [buf0,buf1) of slab_layout) from the neighbouring ranks: this rank's first two
    owned planes go down to rank-1, its last owned plane goes up to rank+1 — three 4*n1*n2-byte planes per interior rank
    over NVLink (NCCL send/recv), instead of recomputing 3 planes of MLP per rank.  Needs >= 2 owned planes on every rank."""
    own0, own1, buf0, buf1 = slab_layout(n0, rank, world)
    ops = []
    if rank > 0:
        ops.append(dist.P2POp(dist.isend, buf[own0 - buf0:own0 - buf0 + 2], rank - 1, group))
        ops.append(dist.P2POp(dist.irecv, buf[0:own0 - buf0], rank - 1, group))
    if rank < world - 1:
        ops.append(dist.P2POp(dist.isend, buf[own1 - 1 - buf0:own1 - buf0], rank + 1, group))
        ops.append(dist.P2POp(dist.irecv, buf[own1 - buf0:buf1 - buf0], rank + 1, group))
    if ops:
        for r in dist.batch_isend_irecv(ops):
            r.wait()


def _gathered_stats(eng, own, world, group):
    """Two-pass statistics like the single-GPU nm_volume_stats, shards combined on the device: two tiny all_gathers, and one
    host read at the end (every plane is owned exactly once, so sums are exact partitions)."""
    acc = torch.empty(5, dtype=torch.float64, device=own.device)
    acc[4] = float(own.numel())
    eng.volume_stats_pass(own, 1, acc)
    allacc = torch.empty((world, 5), dtype=torch.float64, device=own.device)
    dist.all_gather_into_tensor(allacc, acc, group=group)
    mean = (allacc[:, 2].sum() / allacc[:, 4].sum()).reshape(1)
    eng.volume_stats_pass(own, 2, acc, mean)
    allsq = torch.empty(world, dtype=torch.float64, device=own.device)
    dist.all_gather_into_tensor(allsq, acc[3:4].contiguous(), group=group)
    st3 = torch.stack([allacc[:, 0].min(), allacc[:, 1].max(), (allsq.sum() / allacc[:, 4].sum()).sqrt()]).cpu()
    return tuple(float(x) for x in st3)


def _extract_mesh(model, args, rank, world, group, alloc, timings=None, halo="exchange"):
    """The mesh pipeline, written once: slab `rank` of `world` x-slabs of the grid (SURVEY 8e), one slab being the whole grid.
      1. sweep: this rank's planes of sigma (fused MLP, grid front-end) into its slab buffer; with args.sparse_sweep (one
         slab only, opt-in; DESIGN 4.10) sigma only in the blocks of args.sparse_block^3 cells (4, 8 or 16; default 8) the
         surface crosses, found from a lattice of every sparse_block-th point and followed from block to block to a
         fixpoint, and +-inf (the block's side of iso) everywhere else: every vertex, normal and face of that mesh is the
         dense mesh's bit for bit, and what is missing are whole components of the dense mesh, those that fit between
         lattice points and touch no block the sweep reached;
      2. halo planes: 3 planes per interior rank by send/recv from the neighbours (`halo="exchange"`), or recomputed;
      3. iso level: min / max / std over the whole grid (every plane is owned exactly once), clamped by mesh.clamp_iso_level;
         with args.sparse_sweep the statistics are those of the lattice points (the dense ones do not exist; on lego at iso 32 the
         clamp does not bind from 256^3 up, but a small lattice can clamp the level differently from the dense grid);
      4. marching cubes, count step; the (n_vertices, n_triangles) pairs of all ranks give every rank's index offset;
      5. marching cubes, emit step, straight into this rank's segment [vertices | normals | faces] of the exchange buffer
         (padded to the largest slab); with args.super_sampling = s >= 1 (mesh_nerf.py:95-128) through nm_mc_emit_ss: same
         topology, faces and normals, each edge vertex placed from s extra network samples along its edge (DESIGN 4.3);
      6. args.network_normals: this rank's own normals become the network's density gradient (mesh.network_normals, DESIGN
         4.8) — before the gather, a vertex's normal depends on that vertex alone.  Measured on lego, they are better than
         grid normals with super_sampling >= 1 (vertices on the network's surface) but not at s = 0;
      7. gather: ONE all_gather of the segments leaves the whole mesh on every rank;
      8. args.min_component_faces = m >= 1: components with fewer than m faces (floaters) are removed AFTER the gather
         (components cross slab boundaries; DESIGN 4.9); every rank filters the identical gathered mesh;
      9. args.decimate_faces = T >= 1: quadric-error decimation to at most T faces (DESIGN 4.11), after the filter so that
         no collapse is spent on a floater; every rank decimates the identical mesh, so the result is the single-GPU one.
         Moved vertices get their faces' winding normal, or with args.network_normals the network's at their new position.
    `world > 1` guards nothing but the collectives (halo exchange, statistics, counts, mesh): with one slab the segment is
    the mesh, the index offset is 0 and the gather is the identity.  A vertex belongs to the rank that owns its grid point,
    and the last owned cell layer addresses the next rank's vertices by the ids that rank assigns (nm_mc_count /
    nm_mc_emit), so the concatenation IS the one-slab mesh — same arrays, bit for bit; there are no duplicates to remove.
    `alloc(key, numel, dtype, device)` supplies the flat device buffers; the results are views of them: device (vertices
    in index coordinates, triangles, normals), the iso level and the slab buffer (the whole grid for one slab)."""
    eng = model._engine()
    res, dev = args.res, eng.device
    tm = _StageTimer(timings)
    tiles = [torch.linspace(-args.limit, args.limit, res) for _ in range(3)]
    own0, own1, buf0, buf1 = slab_layout(res, rank, world)
    tm.mark()
    buf = alloc("slab", (buf1 - buf0) * res * res, torch.float32, dev).view(buf1 - buf0, res, res)
    exchange = world > 1 and halo == "exchange" and all(
        (lambda a: a[1] - a[0] >= 2)(slab_layout(res, r, world)) for r in range(world))
    # without an exchange the halo planes are recomputed (bit-identical to the owner's); one slab has none
    p0, p1 = (own0, own1) if exchange else (buf0, buf1)
    sparse = bool(getattr(args, "sparse_sweep", False))
    if sparse and world > 1:
        raise NotImplementedError("sparse_sweep runs on one slab: the block fixpoint does not cross slab boundaries yet")
    if sparse:
        block = int(getattr(args, "sparse_block", 8) or 8)
        iso, (n_lat, n_act, n_blk, n_eval, rounds) = eng.sparse_sweep(tiles, args.iso_level, block, buf)
        print(f"sparse sweep (block {block}): {n_act} of {n_blk} blocks active, {n_eval} of {buf.numel()} points evaluated "
              f"({n_lat} on the lattice), {rounds} rounds")
    else:
        eng.grid_sigma(tiles, p0, p1, out=buf[p0 - buf0:p1 - buf0])
    tm.mark("sweep")
    if exchange:
        exchange_halo_planes(buf, res, rank, world, group)
    own = buf[own0 - buf0:own1 - buf0]
    tm.mark("halo")
    if not sparse:
        smin, smax, sstd = _gathered_stats(eng, own, world, group) if world > 1 else eng.volume_stats(own)
        iso = float(mesh.clamp_iso_level(args.iso_level, np.float32(smin), np.float32(smax), np.float32(sstd)))
    tm.mark("stats")
    shard = (iso, buf0, res, own0 - buf0, own1 - buf0)
    nv, nt = eng.mc_count(buf, *shard)
    nvs, nts = [nv], [nt]
    if world > 1:
        counts = torch.tensor([nv, nt], dtype=torch.int64, device=dev)
        allc = torch.empty((world, 2), dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(allc, counts, group=group)
        allc = allc.cpu()
        nvs, nts = [int(x) for x in allc[:, 0]], [int(x) for x in allc[:, 1]]
        if sum(nvs) >= 2 ** 31:
            raise OverflowError("mesh too large for int32 indices")
    v_base = sum(nvs[:rank])
    vmax, tmax = max(max(nvs), 1), max(max(nts), 1)
    seg = 3 * (2 * vmax + tmax)                               # floats per rank: vertices | normals | faces (int32 bits)
    local = alloc(("local", world), seg, torch.float32, dev)
    views = (local[:3 * vmax].view(vmax, 3), local[3 * vmax:6 * vmax].view(vmax, 3), local[6 * vmax:].view(torch.int32).view(tmax, 3))
    s = int(getattr(args, "super_sampling", 0) or 0)
    if s:          # super-sampled vertices: the network is evaluated at the edge samples directly, no extra halo planes
        lins, fines = mesh.super_sampling_tables(args.limit, res, s)
        eng.mc_emit_ss(buf, *shard, nv, nt, v_base, s, lins, fines, out=views)
    else:
        eng.mc_emit(buf, *shard, nv, nt, v_base, out=views)
    if getattr(args, "network_normals", False) and nv:
        nn, fb = mesh.network_normals(eng, model.get_model()._owner[1], views[0][:nv], tiles, views[1][:nv])
        views[1][:nv].copy_(nn)
        mesh._report_fallback(fb, nv)
    tm.mark("mc")
    v, n, f = views[0][:nv], views[1][:nv], views[2][:nt]
    if world > 1:
        full = alloc(("full", world), world * seg, torch.float32, dev)
        dist.all_gather_into_tensor(full, local, group=group)
        full = full.view(world, seg)
        v = torch.cat([full[r, :3 * nvs[r]] for r in range(world)]).view(-1, 3)
        n = torch.cat([full[r, 3 * vmax:3 * vmax + 3 * nvs[r]] for r in range(world)]).view(-1, 3)
        f = torch.cat([full[r, 6 * vmax:6 * vmax + 3 * nts[r]] for r in range(world)]).view(torch.int32).view(-1, 3)
    tm.mark("gather")
    m = int(getattr(args, "min_component_faces", 0) or 0)
    if m > 0:
        v, n, f = mesh.remove_small_components(eng, v, n, f, m)
        tm.mark("components")
    T = int(getattr(args, "decimate_faces", 0) or 0)
    if T > 0:
        net = (model.get_model()._owner[1], tiles) if getattr(args, "network_normals", False) else None
        v, n, f = mesh.decimate(eng, v, n, f, T, net)
        tm.mark("decimate")
    tm.finish()
    return v, f, n, iso, buf


def extract_geometry_sharded(model, args, group=None, to_host=True, timings=None, halo="exchange"):
    """mesh_nerf.extract_geometry (src/mesh_nerf.py:68-92) on N GPUs: the mesh pipeline (_extract_mesh) on this rank's
    x-slab of the grid, its buffers the grow-only scratch tensors of this module.  Every rank returns the whole mesh, the
    same arrays as single-GPU mesh.extract_geometry bit for bit: (vertices, triangles, normals, iso), on the host with the
    vertices rescaled to (-limit, limit) when to_host, otherwise device views that stay valid until the next call (vertices
    in index coordinates).  Works without a process group (one slab)."""
    rank, world = _rank_world(group)
    v, f, n, iso, _ = _extract_mesh(model, args, rank, world, group, _scratch, timings, halo)
    if to_host:
        return mesh.rescale_vertices(v, args.limit, args.res), f.cpu(), n.cpu(), iso
    return v, f, n, iso


def surface_points_sharded(model, poses, H, W, focal, near, far, *, group=None, **kw):
    """mesh.surface_points on N GPUs: this rank renders and filters the contiguous block of poses row_shard(len(poses), rank,
    world) gives it, then one padded all_gather per output assembles the blocks in rank order, which is pose order.  Views
    are independent, so every rank returns the single-GPU arrays bit for bit: {"points", "normals", "colors", "view",
    "pixel", "counts"} as mesh.surface_points documents them (view = the index into `poses`).  `kw`: its keyword options.
    Works without a process group (one block)."""
    rank, world = _rank_world(group)
    v0, v1 = row_shard(len(poses), rank, world)
    local = mesh.surface_points(model, list(poses)[v0:v1], H, W, focal, near, far, **kw)
    local["view"] = local["view"] + v0
    if world == 1:
        return local
    dev = local["points"].device
    out = {k: torch.cat(_all_gather_padded(local[k].contiguous(), group), 0)
           for k in ("points", "normals", "colors", "view", "pixel")}
    counts = _all_gather_padded(torch.tensor(local["counts"], dtype=torch.int64, device=dev), group)
    out["counts"] = [int(c) for part in counts for c in part.tolist()]
    return out
