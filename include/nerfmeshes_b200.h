/*
 * nerfmeshes_b200 — C ABI of the H100-native (sm_90a) NeRF render / dense-grid hot path (the name is historical).
 *
 * The reference (qway/nerfmeshes, pure Python) has no FFI layer; its de-facto operator API for this path
 * is the Python surface SURVEY.md section 8(b) lists.  Each entry point below names the reference interface it
 * replaces (paths relative to /root/reference/).  The reference-side binding a maintainer would add is a
 * ctypes stub; it is shown in INTEGRATION.md and shipped as nerfmeshes_b200/_lib.py.
 *
 * Conventions
 *   - plain C: pointers + sizes, no torch / C++ types.  `stream` is a cudaStream_t passed as void* (NULL =
 *     legacy default stream).
 *   - every call returns 0 on success, <0 on error; nm_last_error() returns a thread-local message.
 *   - pointers suffixed _dev are device pointers on the handle's device, _host are host pointers.
 *   - device-pointer calls are stream-ordered and asynchronous w.r.t. the host; *_host calls synchronise
 *     before returning (they copy results back).
 *   - the handle owns packed weights, tables, the voxel list and a grow-only workspace; callers own all
 *     input / output buffers.  One host thread per handle at a time.
 */
#ifndef NERFMESHES_B200_H
#define NERFMESHES_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NM_VERSION 100 /* 0.1.0 */

/* Shape of one FlexibleNeRFModel — constructor arguments of src/nerf/models.py:5-22. */
typedef struct NmNetDesc {
  int32_t num_layers;          /* 8  */
  int32_t hidden_size;         /* 256 (128 or 256 supported by the tensor-core path) */
  int32_t skip_step;           /* 4  */
  int32_t num_encoding_fn_xyz; /* 10 */
  int32_t num_encoding_fn_dir; /* 4  */
  int32_t include_input_xyz;   /* 1  */
  int32_t include_input_dir;   /* 1  */
  int32_t log_sampling_xyz;    /* 1  */
  int32_t log_sampling_dir;    /* 1  */
  int32_t use_viewdirs;        /* 1  */
} NmNetDesc;

/* MLP arithmetic selection (SURVEY 7.3.1). */
enum {
  NM_PREC_EXACT = 0, /* wgmma, fp16 hi/lo split operands, 3 MMAs per product, fp32 accumulate (default) */
  NM_PREC_FAST = 1,  /* wgmma, single fp16 operands (misses the 1e-4 target; for comparison only)      */
  NM_PREC_FP32 = 2   /* CUDA-core fp32 FMA kernel (bit-for-bit fp32 arithmetic; slow; debugging yard-stick) */
};

/* cfg.nerf.{train,validation}.* and cfg.dataset.* knobs read on the path (config/nerf-synthetic-lego.yml). */
typedef struct NmRenderCfg {
  int32_t num_coarse;          /* cfg.nerf.train.num_coarse (the reference sizes its samplers from .train,
                                  src/models/model_nerf.py:31-32)                                        */
  int32_t num_fine;            /* cfg.nerf.train.num_fine; 0 = coarse only (models.use_fine False)          */
  int32_t lindisp;
  int32_t perturb;             /* stratified jitter / random u (distributional parity only)                 */
  int32_t white_background;
  float noise_std;             /* radiance_field_noise_std of the active mode                              */
  float attenuation_threshold; /* 1e-5, src/models/model_base.py:28-33                                     */
  int32_t precision;           /* NM_PREC_*                                                                */
  int32_t act_scale_log2;      /* s >= 0: fp16 A-operands are stored as x * 2^-s (range guard, SURVEY 7.3.1)  */
} NmRenderCfg;

typedef struct NmHandle_t* NmHandle;

enum { NM_NET_COARSE = 0, NM_NET_FINE = 1 };

/* Output block of one render call: the fields of OutputBundle (src/nerf/modules.py:40-47).  Any pointer may be
 * NULL (that output is skipped).  depth is the eval-mode thresholded map (modules.py:108-109) unless flag
 * NM_FLAG_TRAINING is set; depth_raw is sum(w*t) before the threshold (what parity tests compare). */
typedef struct NmRenderOut {
  float* rgb;          /* (R,3) */
  float* depth;        /* (R,)  */
  float* depth_raw;    /* (R,)  */
  float* acc;          /* (R,)  */
  float* disp;         /* (R,)  */
  float* weights;      /* (R,S) S = num_coarse+num_fine (or num_coarse when coarse-only / BuFF) */
  float* mask_weights; /* (R,S) */
  float* t_vals;       /* (R,S) the sample distances actually used (debug / parity) */
  float* coarse_rgb;   /* (R,3) coarse-pass colour (training loss needs it, model_nerf.py:128) */
  float* coarse_acc;   /* (R,)  */
  float* coarse_disp;  /* (R,)  */
  float* coarse_weights; /* (R,num_coarse) */
} NmRenderOut;

enum {
  NM_FLAG_TRAINING = 1,    /* module.training: no depth threshold, train noise_std            */
  NM_FLAG_BUFF = 2,        /* BuFFModel.forward: AABB-clipped sampling, single net (coarse slot) */
  NM_FLAG_TEACHER_T = 4,   /* t_vals is an INPUT: skip sampling, run net `which`=fine-if-present on it */
  NM_FLAG_RANDOM_VOXELS = 8, /* with NM_FLAG_BUFF: cfg.tree.use_random_sampling — multinomial voxel draws + uniform depth inside
                               the voxel (src/nerf/tree.py:280-297) instead of the deterministic placement; uses `seed` */
  NM_FLAG_SKIP_EMPTY = 16,  /* empty-space skipping (nm_build_occupancy): only the samples the pass's occupancy grid marks go
                               through the network; inference only (rejected with NM_FLAG_TRAINING / NM_FLAG_TEACHER_T) */
  NM_FLAG_SKIP_EMPTY_TRAIN = 32 /* empty-space skipping in training (see the occupancy section): only with NM_FLAG_TRAINING, by
                               nm_render_rays, nm_backward_rays and nm_loss_backward; rejected with NM_FLAG_TEACHER_T and
                               NM_FLAG_SKIP_EMPTY; takes a stale grid */
};

/* ---- lifecycle -------------------------------------------------------------------------------------- */
int nm_version(void);
const char* nm_last_error(void);
/* 0 if `device` is a compute-capability-10.x GPU, error otherwise (the library fails loudly elsewhere). */
int nm_device_check(int device);
/* Replaces NeRFModel.__init__/BuFFModel.__init__ (src/models/model_nerf.py:24-32, model_buff.py:13-29). */
int nm_create(int device, const NmNetDesc* coarse, const NmNetDesc* fine_or_null, const NmRenderCfg* cfg,
              NmHandle* out);
int nm_destroy(NmHandle h);
int nm_set_render_cfg(NmHandle h, const NmRenderCfg* cfg);

/* Replaces load_state_dict for one FlexibleNeRFModel (weight ABI: SURVEY Appendix A.1).  names[i] is the
 * reference state-dict key without the model prefix ("layer1.weight", "layers_xyz.4.bias", "fc_alpha.weight",
 * ...); tensors_host[i] points at numel[i] fp32 values in the reference (out,in) row-major layout. */
int nm_load_weights(NmHandle h, int which, int n_tensors, const char* const* names,
                    const float* const* tensors_host, const int64_t* numel);
/* Same, with the tensors already in device memory (fp32, contiguous): transposes / packs on the device, stream-ordered,
 * no host round trip — the per-step weight refresh of a training loop whose optimiser updates CUDA parameters. */
int nm_load_weights_dev(NmHandle h, int which, int n_tensors, const char* const* names,
                        const float* const* tensors_dev, const int64_t* numel, void* stream);
/* Sampler tables: coarse s = torch.linspace(0,1,num_coarse) (src/nerf/modules.py:154) and the SamplePDF buffer
 * u = torch.linspace(0,1,num_fine) (modules.py:193).  Host pointers; NULL = recompute i/(n-1) in fp32. */
int nm_set_tables(NmHandle h, const float* coarse_s_host, const float* fine_u_host);
/* BuFF voxel list, checkpoint['tree']['voxels'] (V,2,3) (src/nerf/tree.py:345-358). */
int nm_set_tree(NmHandle h, const float* voxels_host, int32_t V);

/* ---- hot path, device pointers ---------------------------------------------------------------------- */
/* BaseModel.sample_points (src/models/model_base.py:65-73) == FlexibleNeRFModel.forward (src/nerf/models.py:60-80).
 * pts/dirs (M,3) fp32; out (M,4) = [sigmoid rgb, raw sigma], or (M,) raw sigma when sigma_only. */
int nm_point_mlp(NmHandle h, int which, const float* pts_dev, const float* dirs_dev, int64_t M, float* out_dev,
                 int sigma_only, void* stream);
/* d sigma / d p of network `which` at M points (no reference counterpart: analytic normals for the mesh path).  pts (M,3)
 * fp32; grad (M,3); sigma (M,) raw density or NULL (then bit for bit nm_point_mlp's sigma_only output).  Handle precision
 * selects tensor cores (exact / fast) or fp32.  Deterministic, independent of batch composition; leaves the gradient
 * buffers and every other handle state untouched.  M = 0 launches nothing.  Points are walked in chunks of
 * NM_SIGMA_GRAD_CHUNK_POINTS (default 256 Ki) in a workspace of the handle: it grows to one chunk's size (~22 KB per point
 * for the 8x256 network, ~5.8 GB at the default) and is held until nm_destroy; a smaller chunk bounds it. */
int nm_sigma_grad(NmHandle h, int which, const float* pts_dev, int64_t M, float* sigma_dev_or_null, float* grad_dev,
                  void* stream);
/* NeRFModel.forward / BuFFModel.forward (src/models/model_nerf.py:37-78, model_buff.py:34-69).
 * origins: o_stride = 0 -> one shared (3,) origin, 3 -> per-ray (R,3).  near/far: nf_stride = 0 -> 2 scalars in
 * near_far_host[0..1]; 1 -> per-ray near (R,) and far (R,) device arrays in near_dev / far_dev. */
int nm_render_rays(NmHandle h, const float* origins_dev, int o_stride, const float* dirs_dev, int64_t R,
                   const float* near_far_host, const float* near_dev, const float* far_dev, int flags, uint64_t seed,
                   const NmRenderOut* out_dev, void* stream);
/* get_ray_bundle (+ ndc_rays) fused with the render for image rows [row0,row1) — the eval_nerf.py:50-98 image
 * loop with the pose, not 7.7 MB of directions, crossing PCIe.  pose_host: 12 floats, c2w[:3,:4] row-major.
 * Outputs are (row1-row0)*W rays.  focal (and near below) are the caller's python floats, unrounded: ndc_rays forms its
 * scalars from them in double and rounds each once to fp32; the pixel division uses (float)focal, as torch does. */
int nm_render_image(NmHandle h, const float* pose_host, int H, int W, double focal, int ndc, int row0, int row1,
                    const float* near_far_host, int flags, uint64_t seed, const NmRenderOut* out_dev, void* stream);
/* get_ray_bundle / ndc_rays alone (src/nerf/nerf_helpers.py:226-307): dirs (rows,W,3); origins (rows,W,3) only
 * when ndc (else the origin is pose[:,3]). */
int nm_ray_bundle(NmHandle h, const float* pose_host, int H, int W, double focal, int ndc, double ndc_near, int row0,
                  int row1, float* origins_dev_or_null, float* dirs_dev, void* stream);
/* ndc_rays(H, W, focal, near, rays_o, rays_d) on caller-supplied rays (src/nerf/nerf_helpers.py:280-307, called positionally
 * by DataBundle.ndc, src/data/data_helpers.py:164-167): n rays, origins with o_stride 0 (one shared origin) or 3. */
int nm_ndc_rays(NmHandle h, int H, int W, double focal, double near, const float* origins_dev, int o_stride,
                const float* dirs_dev, int64_t n, float* origins_out_dev, float* dirs_out_dev, void* stream);
/* extract_radiance (src/mesh_nerf.py:27-53) for grid planes [x0,x1): points from the three linspace tables
 * (host, lengths n0,n1,n2; pass torch.linspace values for bit-identical coordinates), dirs := positions.
 * sigma_dev (x1-x0,n1,n2) raw density; rgb_dev (x1-x0,n1,n2,3) or NULL (sigma-only fast path). */
int nm_grid_sigma(NmHandle h, const float* lin0_host, const float* lin1_host, const float* lin2_host, int n0, int n1,
                  int n2, int x0, int x1, float* sigma_dev, float* rgb_dev_or_null, void* stream);
/* numpy min / max / std of a float32 volume (extract_iso_level, src/mesh_nerf.py:56-65): out_host[0..2] =
 * {min, max, std}; synchronises. */
int nm_volume_stats(NmHandle h, const float* vol_dev, int64_t n, float* out_host);

/* The same statistics for a volume sharded over several GPUs, stream-ordered and without host synchronisation: pass 1 writes
 * out_dev[0..2] = {min, max, sum} of this shard (doubles), pass 2 writes out_dev[3] = sum (x - *mean_dev)^2; the caller
 * combines the shards between and after the passes (all_gather / all_reduce on the device values). */
int nm_volume_stats_dev(NmHandle h, const float* vol_dev, int64_t n, int pass, const double* mean_dev, double* out_dev, void* stream);

/* skimage.measure.marching_cubes(volume, level) seam (src/mesh_nerf.py:79) on a device volume (nx,ny,nz) fp32, Lewiner-style
 * topology resolution (face / interior tests, cell-centre vertices): sign bit-volume -> count -> scan -> emit.  Two-call
 * protocol: nm_marching_cubes_count fills counts_host = {n_vertices, n_triangles} (synchronises);
 * nm_marching_cubes_emit (same volume and iso) writes verts (n_vertices,3) fp32 in index coordinates (x_off, an integer,
 * added to axis 0), normals (n_vertices,3), faces (n_triangles,3) int32.  Indexed mesh: one vertex per crossed grid edge
 * plus the centre vertices, ordered by owning grid point. */
int nm_marching_cubes_count(NmHandle h, const float* vol_dev, int nx, int ny, int nz, float iso,
                            int64_t* counts_host, void* stream);
int nm_marching_cubes_emit(NmHandle h, const float* vol_dev, int nx, int ny, int nz, float iso, float x_off,
                           float* verts_dev, float* normals_dev, int32_t* faces_dev, void* stream);
/* The same for ONE SHARD of a grid split along axis 0 (mesh_nerf.py:27-92 on N GPUs, SURVEY 8e): the buffer holds global
 * planes [g_x0, g_x0+nb) of a grid with g_nx planes and the call owns the grid points of buffer planes [p_lo,p_hi): it
 * emits their vertices and the triangles of their cells.  The buffer must also hold, where they exist globally, plane
 * p_hi (cells of the last owned layer), p_hi+1 and p_lo-1 (gradient normals): halo planes, received from the neighbours or
 * recomputed.  Face indices are v_base + local id, and ids of plane-p_hi vertices (owned by the next shard) continue the
 * local numbering; with v_base = the exclusive scan of the shards' n_vertices, the concatenated shard outputs ARE the
 * single-GPU arrays, bit for bit (no duplicate vertices, nothing to de-duplicate). */
int nm_mc_count(NmHandle h, const float* vol_dev, int nb, int ny, int nz, float iso, int g_x0, int g_nx, int p_lo, int p_hi,
                int64_t* counts_host, void* stream);
int nm_mc_emit(NmHandle h, const float* vol_dev, int nb, int ny, int nz, float iso, int g_x0, int g_nx, int p_lo, int p_hi,
               int64_t v_base, float* verts_dev, float* normals_dev, int32_t* faces_dev, void* stream);
/* Super-sampled emit step (the --super-sampling branch of mesh_nerf.py:95-128): called after nm_mc_count with the same
 * shard arguments, like nm_mc_emit, whose faces, normals and centre vertices it reproduces bit for bit.  Each vertex on the
 * axis-a edge from global grid point (I,J,K) to its neighbour along a is re-placed from s >= 0 extra samples along that
 * edge: v_0 = vol(point), v_{s+1} = vol(neighbour), and for m = 1..s v_m = sigma of the finest network (the one
 * nm_grid_sigma sweeps, at the handle's precision, directions = positions) at fine_a[idx_a*(s+1)+m] along a and
 * lin_b[idx_b] along the other axes.  With the smallest m in [0,s] where (v_m > iso) != (v_{m+1} > iso), in double:
 *   w0 = 1/(FLT_EPSILON + |v_m - iso|),  w1 = 1/(FLT_EPSILON + |v_{m+1} - iso|),  pos[a] = base[a] + (m + w1/(w0+w1))/(s+1);
 * s = 0 is nm_mc_emit's formula.  lin0 / fine0 cover the GLOBAL grid (g_nx and (g_nx-1)(s+1)+1 entries), lin1 / lin2 have
 * ny / nz entries, fine1 / fine2 (ny-1)(s+1)+1 / (nz-1)(s+1)+1: torch.linspace(-limit, limit, n) and
 * torch.linspace(-limit, limit, n + (n-1)*s).  Host tables.  0 <= s <= 64.  The network sees s points per owned vertex
 * (centre vertices are padded with their grid point), in launches of at most NM_SS_CHUNK_POINTS points (default 4 Mi). */
int nm_mc_emit_ss(NmHandle h, const float* vol_dev, int nb, int ny, int nz, float iso, int g_x0, int g_nx, int p_lo, int p_hi,
                  int64_t v_base, int s, const float* lin0_host, const float* lin1_host, const float* lin2_host,
                  const float* fine0_host, const float* fine1_host, const float* fine2_host,
                  float* verts_dev, float* normals_dev, int32_t* faces_dev, void* stream);

/* ---- chamfer evaluation: the chamfer branch of validation_epoch_end (src/models/model_base.py:82-102) -------------------
 * Argument errors (null pointers, negative sizes, empty point sets or meshes, sizes >= 2^31) are rejected before anything is
 * launched; N = 0 (n = 0) succeeds and launches nothing.  Definitions: DESIGN §4.7.
 *
 * pytorch3d.ops.sample_points_from_meshes (model_base.py:94-96): n points on the mesh verts (V,3) fp32 / faces (F,3) int32,
 * faces chosen with probability proportional to area (first f with cdf[f] > u * total, cdf the double prefix sum of the
 * fp32 areas), barycentric weights w0 = 1 - sqrt(a), w1 = sqrt(a)(1 - b), w2 = sqrt(a) b; u, a, b = splitmix64 draws
 * 3k, 3k+1, 3k+2 of `seed`.  points (n,3); face_idx (n,) int32 or NULL.  A face index outside [0,V) or a total area that
 * is not positive and finite is reported through the device-side error word (nm_check_flags raises it, once). */
int nm_mesh_sample(NmHandle h, const float* verts_dev, int64_t V, const int32_t* faces_dev, int64_t F, int64_t n, uint64_t seed,
                   float* points_dev, int32_t* face_idx_dev_or_null, void* stream);
/* The nearest-neighbour search inside pytorch3d.loss.chamfer_distance (model_base.py:99): for each of N queries q (N,3) the
 * squared distance to the nearest of M >= 1 points p (M,3), dist2 (N,), and that point's index (N,) int32 or NULL, the
 * lowest index on ties.  Exact (an fp32 distance, fmaf(dz,dz,fmaf(dy,dy,dx*dx))) by a uniform grid search. */
int nm_nearest(NmHandle h, const float* q_dev, int64_t N, const float* p_dev, int64_t M, float* dist2_dev,
               int32_t* idx_dev_or_null, void* stream);
/* pytorch3d.loss.chamfer_distance(x, y) without weights or normals (model_base.py:99): means_dev (2 doubles, device) =
 * {mean_i d2(x_i, Y), mean_j d2(y_j, X)}, reduced in double in a fixed order (the same bits on every run); the chamfer
 * loss is their sum. */
int nm_chamfer(NmHandle h, const float* x_dev, int64_t N, const float* y_dev, int64_t M, double* means_dev, void* stream);
/* Test hook: nm_nearest by tiled brute force (the same distance function, same arguments). */
int nm_debug_nearest_brute(NmHandle h, const float* q_dev, int64_t N, const float* p_dev, int64_t M, float* dist2_dev,
                           int32_t* idx_dev_or_null, void* stream);

/* Small-component removal on an indexed mesh (no reference counterpart; DESIGN §4.9).  Components are the connected
 * components of the vertex graph spanned by the faces; a component's id is its smallest vertex index; its size is its
 * number of faces.  Keeps the vertices and faces of components with >= min_faces faces, in their original order, faces
 * re-indexed.  Outputs are caller-allocated with room for V vertices / F faces; labels_out (V,) int32 (the component id of
 * every INPUT vertex) may be NULL.  counts_host = {kept vertices, kept faces, components with >= 1 face, kept components};
 * synchronises.  Deterministic: the same bits on every run.  Argument errors (null pointers, negative sizes or min_faces,
 * sizes >= 2^31) are rejected before anything is launched; V = F = 0 launches nothing.  A face index outside [0,V) is
 * reported through the device-side error word (nm_check_flags raises it, once) and that face is dropped. */
int nm_mesh_components(NmHandle h, const float* verts_dev, const float* normals_dev, int64_t V, const int32_t* faces_dev,
                       int64_t F, int64_t min_faces, float* verts_out_dev, float* normals_out_dev, int32_t* faces_out_dev,
                       int32_t* labels_out_dev_or_null, int64_t* counts_host, void* stream);

/* Quadric-error decimation of an indexed mesh (no reference counterpart; DESIGN §4.11): rounds of edge collapses chosen as an
 * independent set by Garland–Heckbert cost, until at most target_faces faces remain or no collapse is legal.  verts (V,3)
 * fp32 in index coordinates, normals (V,3), faces (F,3) int32.  Vertices on an open or non-manifold edge, in a face with a
 * repeated index, or with more than 32 faces are never moved or removed; a collapse must keep the link condition, at most
 * 32 faces at the survivor, and every surviving face's orientation.  The round that would cross target_faces collapses only
 * the ceil((F - target)/2) cheapest of its edges, so the result has target or target - 1 faces unless it runs out of legal
 * collapses first; target_faces >= F copies the input bit for bit.  Outputs are caller-allocated with room for V vertices /
 * F faces: the surviving vertices in ascending input order, the surviving faces in input order re-indexed, and
 * source_out (V',) int32 (the input row of every output vertex) unless NULL.  A vertex whose position kept its bits keeps
 * its input normal; a moved one gets the normalised area-weighted sum of its faces' winding normals.  counts_host =
 * {V', F', rounds, collapses}; synchronises once and then once per round.  Deterministic: the same bits on every run.
 * Argument errors (null pointers, negative sizes or target_faces, sizes >= 2^31, 3F >= 2^31) are rejected before anything
 * is launched; V = F = 0 launches nothing.  A face index outside [0,V) is reported through the device-side error word
 * (nm_check_flags raises it, once) and the input is copied unchanged. */
int nm_mesh_decimate(NmHandle h, const float* verts_dev, const float* normals_dev, int64_t V, const int32_t* faces_dev, int64_t F,
                     int64_t target_faces, float* verts_out_dev, float* normals_out_dev, int32_t* faces_out_dev,
                     int32_t* source_out_dev_or_null, int64_t* counts_host, void* stream);

/* Sparse density sweep for mesh extraction (no reference counterpart: the reference sweeps the whole grid; these two calls
 * stand in for the extract_radiance interface, src/mesh_nerf.py:27-53, where resolution should cost in proportion to the
 * surface; DESIGN §4.10).  Grid and tables as nm_grid_sigma's (host tables of n0 / n1 / n2 entries), the finest network at
 * the handle's precision, directions = positions; every sigma written equals nm_grid_sigma's at that point bit for bit.
 * block = B in {4, 8, 16}: block b of an axis covers cells [b*B, min((b+1)*B, n-1)); the lattice is every B-th grid point
 * of an axis and its last.  Two calls, because the iso level is clamped between them on the host (mesh_nerf.py:56-65):
 *   nm_sparse_sweep_lattice  writes sigma at the lattice points into vol_dev (n0,n1,n2); stats_host[0..2] = {min, max, std}
 *                            over the LATTICE points (numpy's, like nm_volume_stats); synchronises.
 *   nm_sparse_sweep_run      on the same grid, block and volume: blocks whose 8 lattice corners do not agree in
 *                            sigma > iso are active; every point of an active block's closed point set, dilated by one
 *                            point and clipped to the grid, is evaluated once; an inactive block with an evaluated point
 *                            on the other side of iso than its corners becomes active; repeated until no block does.
 *                            Every point never evaluated is set to +inf (its block's corners are > iso) or -inf.
 *                            counts_host[0..4] = {lattice points, active blocks, blocks, evaluated points, rounds};
 *                            synchronises once per round.
 * Deterministic: the same volume on every run and for every NM_SPARSE_CHUNK_POINTS (points per network launch, default
 * 4 Mi, read per call).  Argument errors (null pointers, block not in {4, 8, 16}, fewer than 2 points on an axis, 2^31
 * grid points or more, missing weights, run without its lattice call) are rejected before anything is launched. */
int nm_sparse_sweep_lattice(NmHandle h, const float* lin0_host, const float* lin1_host, const float* lin2_host, int n0, int n1,
                            int n2, int block, float* vol_dev, float* stats_host, void* stream);
int nm_sparse_sweep_run(NmHandle h, const float* lin0_host, const float* lin1_host, const float* lin2_host, int n0, int n1, int n2,
                        int block, float iso, float* vol_dev, int64_t* counts_host, void* stream);
/* Test hook: device copies of the last nm_sparse_sweep_run's evaluated mask (n0*n1*ceil(n2/32) words, bit k%32 of word k/32
 * of grid line (i,j): the marching-cubes sign bit-volume's layout) and block states ((b0,b1,b2) row-major int32, bit 0: the
 * corners are > iso, bit 1: active); either may be NULL. */
int nm_debug_sparse_sweep_state(NmHandle h, uint32_t* mask_out_dev_or_null, int32_t* blocks_out_dev_or_null, void* stream);

/* Texture bake of a mesh's appearance (no reference counterpart: the reference colours vertices, src/mesh_nerf.py:160-192;
 * DESIGN §4.12).  N = texels along a triangle leg, 2 <= N <= 64.  Face f owns one right-triangle patch of K = N(N+1)/2 texels in
 * half f % 2 of square cell f / 2 of C = N + 2 texels; P = ceil(F/2) cells, Q = the smallest integer with Q^2 >= P cells per
 * row, a W = Q*C by H = ceil(P/Q)*C atlas (row 0 on top), cell c at pixel ((c % Q)*C, (c / Q)*C).  Half 0 holds texel (i, j),
 * i + j <= N - 1, at in-cell pixel (i, j) with corners 0, 1, 2 of the face at (0,0), (N-1,0), (0,N-1); half 1 the same patch
 * at (C-1-i, C-1-j).  Texels are numbered face-major, then row j, then i.
 * nm_texture_layout: out4 = {Q, rows, W, H}; host only.  Rejects N outside [2, 64], F outside [0, 2^31) and a W or H above
 * 16384 (naming the largest N that fits).
 * nm_bake_texture: one appearance query per texel, as mesh_appearance builds one per vertex: with weights w1 = i/(N-1),
 * w2 = j/(N-1), w0 = (1-w1)-w2 the point p = (w0 v0 + w1 v1) + w2 v2 and normal n = m/|m|, m = (w0 n0 + w1 n1) + w2 n2 (the
 * corner of largest weight, lowest on ties, where |m| is 0 or not finite), fp32 in that order; corner texels take v_k and n_k
 * unchanged.  d = -n.  mode 0: a ray from p - view_disparity*d along d through the render path of nm_render_rays with `flags`,
 * near_far_host and seed 0; mode 1: nm_point_mlp of network `which` at (p, d), rgb columns.  verts / normals (V,3), faces (F,3)
 * int32; outputs caller-allocated: atlas_f32 (H,W,3) with every texel of a triangle its query's colour, every ring texel
 * (i + j = N in half 0's coordinates) the mean of its in-triangle 4-neighbours (i-1,j) and (i,j-1) as (a+b)*0.5f or the one
 * that exists, every other texel 0; atlas_u8 = floorf(clamp(c, 0, 1)*255 + 0.5f); uv (F,3,2) = the centre of each corner
 * texel, ((x+0.5)/W, 1-(y+0.5)/H); vertex_rgb (V,3) = the corner texel of the lowest (face, corner slot) that references the
 * vertex, or for a vertex no face references, a query of its own built the same way.  counts_host = {W, H, queries rendered,
 * vertices without a face}; synchronises once.  Faces are walked in chunks of NM_TEXTURE_CHUNK_TEXELS texels (default 4 Mi,
 * read per call); the result is the same bits for every chunk size and on every run.  Argument errors (null pointers, N or
 * atlas out of range, sizes >= 2^31, an unknown mode, NM_FLAG_TEACHER_T) are rejected before anything is launched; V = F = 0
 * launches nothing.  A face index outside [0,V) is reported through the device-side error word (nm_check_flags raises it,
 * once) and nothing is baked.
 * nm_debug_texture_rays: test hook, the queries of faces [f0, f1) (K per face; origins_out = the ray origins in mode 0, the
 * points in mode 1) and their atlas pixels (x, y) int32 unless pixel_xy_out is NULL. */
int nm_texture_layout(int64_t F, int N, int64_t* out4);
int nm_bake_texture(NmHandle h, const float* verts_dev, const float* normals_dev, int64_t V, const int32_t* faces_dev, int64_t F,
                    int N, int mode, int which, int flags, float view_disparity, const float* near_far_host, float* atlas_f32_dev,
                    uint8_t* atlas_u8_dev, float* uv_dev, float* vertex_rgb_dev, int64_t* counts_host, void* stream);
int nm_debug_texture_rays(NmHandle h, const float* verts_dev, const float* normals_dev, int64_t V, const int32_t* faces_dev, int64_t F,
                          int N, int mode, float view_disparity, int64_t f0, int64_t f1, float* origins_out_dev,
                          float* dirs_out_dev, int32_t* pixel_xy_out_dev, void* stream);

/* Mesh rasterizer (no reference counterpart; DESIGN §4.13): an image of a world-coordinate mesh through the pinhole camera of
 * nm_render_image without NDC (pose_host the 3x4 camera-to-world, H x W pixels, focal), so that mesh pixel (c, r) lies on the
 * ray NeRF pixel (c, r) renders.  verts (V,3) fp32, faces (F,3) int32.  Corner v goes to camera coordinates p = R^T (v - t),
 * depth z = -p2 and the screen point X = W/2 + focal p0/z, Y = H/2 - focal p1/z; pixel (c, r) samples the point (c, r).  A
 * face with a corner at z <= z_near, a non-finite coordinate or |X| or |Y| above 2^20 is culled; both windings are drawn.
 * Coverage is exact (corners snapped to 1/256 pixel, int64 edge functions, a top-left rule): a sample on an edge two faces
 * share is covered once.  The nearest face wins by perspective-correct depth, the lower face id on ties.  mode 0: the
 * perspective-correct interpolation of vertex_rgb (V,3); mode 1: a bilinear lookup in atlas (fp32, the layout of
 * nm_texture_layout for F faces at N texels per leg, as nm_bake_texture writes it: the caller must pass an atlas of exactly
 * that H' x W' x 3 for this F and N, which the library cannot check).  Outputs (any may be NULL): rgb (H,W,3),
 * depth (H,W) = the distance along the pixel's ray (what NeRF's depth map estimates), face (H,W) int32; an uncovered pixel
 * gets background_host (3 floats), depth 0 and face -1.  counts_host = {covered pixels, faces drawn (not culled), faces
 * culled}; synchronises once.  Every step is fixed fp32 / integer arithmetic and the depth test an atomicMin of (depth, face)
 * keys, so the image is the same bits on every run and for every NM_RASTER_BIG_FACE_PIXELS (faces whose bounding box holds at
 * least that many pixel samples, default 256, read per call, are drawn per screen tile instead of per thread).  Argument
 * errors (null pointers, H or W outside [1, 16384], focal or z_near not positive and finite, sizes >= 2^31, an unknown mode,
 * mode 1 with an N nm_texture_layout rejects for F) are rejected before anything is launched; F = 0 launches only the
 * background fill.  A face index outside [0,V) is never read through; it is reported through the device-side error word
 * (nm_check_flags raises it, once), and nothing is drawn: every pixel gets the background and the counts are 0. */
int nm_rasterize_mesh(NmHandle h, const float* verts_dev, int64_t V, const int32_t* faces_dev, int64_t F, const float* pose_host,
                      int H, int W, float focal, float z_near, int mode, const float* vertex_rgb_dev_or_null,
                      const float* atlas_dev_or_null, int N, const float* background_host, float* rgb_out_or_null,
                      float* depth_out_or_null, int32_t* face_out_or_null, int64_t* counts_host, void* stream);

/* Surface points of one rendered view (the algorithm of the reference's dead src/mesh_surface_ray.py:66-141; DESIGN §4.14).
 * depth_raw, acc (H*W) and rgb (H*W,3) are nm_render_image's outputs for pose_host (3x4 camera-to-world), H x W and focal
 * without NDC; d(r,c) is the direction that render used (raygen's bits) and o = pose[:,3].  Per pixel t = depth_raw where
 * acc >= min_acc, else 0, and P = o + d*t per component in fp32 (two roundings).  The count of pixel (r,c) is the number
 * of offsets (a,b) in [-step, step]^2 whose neighbour (clamp(r+a, 0, H-1), clamp(c+b, 0, W-1)) has
 * (dx*dx + dy*dy) + dz*dz < dist_threshold, with d the fp32 difference to P(r,c) (an edge pixel counts itself again; a NaN
 * point counts nothing).  A pixel is kept when count >= min_count and t > 0.  Outputs are caller-allocated with room for
 * H*W rows: per kept pixel in row-major order points (P), normals (-d), colors (rgb), and pixel_out (r*W + c, int32) unless
 * NULL.  count_host = the number of kept pixels; synchronises once.  The same bits on every run.  Argument errors (null
 * pointers, H or W below 1, H*W >= 2^31, step outside [0, 8], min_count below 1, focal not positive and finite, a NaN
 * min_acc or dist_threshold) are rejected before anything is launched. */
int nm_surface_points(NmHandle h, const float* pose_host, int H, int W, float focal, const float* depth_raw_dev,
                      const float* acc_dev, const float* rgb_dev, float min_acc, int step, float dist_threshold, int min_count,
                      float* points_out_dev, float* normals_out_dev, float* colors_out_dev, int32_t* pixel_out_dev_or_null,
                      int64_t* count_host, void* stream);

/* Replaces export_obj (src/nerf/nerf_helpers.py:86-111): `v x y z [r g b]`, `vn x y z`, `f i//i j//j k//k` (1-based) with
 * byte-identical number formatting (python repr of the float32 widened to double).  Host arrays, no GPU involved;
 * diffuse may be NULL or shorter than the vertex list (vertices beyond it get no colour, like the reference's
 * len(diffuse) > idx test). */
int nm_export_obj(const char* path, const float* verts_host, int64_t n_verts, const int32_t* faces_host, int64_t n_faces,
                  const float* diffuse_host, int64_t n_diffuse, const float* normals_host, int64_t n_normals);
/* nm_export_obj with a texture: `mtllib <mtl_name>`, the same `v` lines, `vt u v` for uv_host (n_faces,3,2) face-major, the
 * same `vn` lines, `usemtl texture`, then `f a/t/a b/u/b c/w/c` with t = 3f+k+1. */
int nm_export_obj_textured(const char* path, const float* verts_host, int64_t n_verts, const int32_t* faces_host, int64_t n_faces,
                           const float* diffuse_host, int64_t n_diffuse, const float* normals_host, int64_t n_normals,
                           const float* uv_host, const char* mtl_name);
/* Replaces export_ply (src/mesh_surface_ray.py:45-57): a point cloud with normals and colours as PLY.  Header `ply`,
 * `format ascii 1.0` (binary = 0) or `format binary_little_endian 1.0` (binary = 1), `element vertex n`, `property float`
 * x y z nx ny nz, `property uchar` red green blue, `end_header`.  Colours are quantised as trunc(fl32(c*255)) clamped to
 * [0, 255], NaN to 0.  Text rows are the nine values as %.18g separated by single spaces; binary rows are packed 27-byte
 * little-endian records.  Host arrays (n,3) fp32, no GPU involved. */
int nm_export_ply(const char* path, const float* points_host, const float* colors_host, const float* normals_host, int64_t n,
                  int binary);

/* ---- empty-space skipping (DESIGN §4.15) ------------------------------------------------------------------
 * One occupancy grid per network slot: G x G x G cells over the box [lo, hi) (box = {lo_x, lo_y, lo_z, hi_x, hi_y, hi_z} in
 * network-input coordinates, NDC ones for an NDC render), one bit per cell, bit (i*G + j)*G + k of uint32 words
 * (ceil(G^3 / 32) of them).  A point p is EVALUATED when, for some axis a, c_a = floor((p_a - lo_a) * inv_a) is outside [0, G)
 * or not finite (fp32, a rounded subtract then a rounded multiply; inv_a = G / (hi_a - lo_a) rounded once), or when its cell's
 * bit is set.  With NM_FLAG_SKIP_EMPTY a render sends only evaluated samples through the network; every other sample enters
 * the compositor as raw (0,0,0,-inf), i.e. alpha = 0 whatever the sigma noise.  Guarantee: every output of a ray (rgb, depth,
 * depth_raw, acc, disp, weights, mask_weights, t_vals, coarse_*) is bit-identical to the render without the flag when every
 * sample the grid skipped on that ray has a dense noisy pre-activation (raw sigma + the pass's noise) <= 0 or NaN.  A skipping render reads each pass's sample count back to the host (one
 * small copy and one stream synchronisation per pass per NM_CHUNK_RAYS chunk), so it cannot be captured in a CUDA graph; the
 * network runs on at most NM_SKIP_CHUNK_POINTS points per launch (default 4 Mi).
 *
 * Grid lifetime: loading a network's weights marks its grid STALE.  NM_FLAG_SKIP_EMPTY renders and nm_occupancy_query refuse
 * a stale grid; NM_FLAG_SKIP_EMPTY_TRAIN takes it (keeping it fresh enough is the caller's schedule: BaseModel.
 * enable_training_skip rebuilds every few optimiser steps).  nm_build_occupancy / nm_set_occupancy make a grid fresh.
 *
 * Training (NM_FLAG_SKIP_EMPTY_TRAIN with NM_FLAG_TRAINING): each pass compacts and stages its evaluated samples as above,
 * keeps them until its backward, runs the network over them only (emitting the backward's operands when they fit
 * NM_TRAIN_DIRECT_GB for that pass's evaluated count) and composites the expanded (R,S,4) buffer; the compositor adjoint
 * hands the evaluated rows, compacted, to the network backward.  On every ray whose skipped samples all have a dense
 * noisy pre-activation (raw sigma + the training noise) <= 0 or NaN, rgb / coarse_rgb and the loss terms are bit-identical
 * to the dense training call and so are the evaluated samples' adjoints (a skipped sample's dense adjoint row is zero);
 * the weight gradients differ from the dense ones by the order of fp32 atomic sums only.  A pass with no evaluated sample
 * launches no network work.  nm_skip_stats counts these passes too.
 *
 * nm_build_occupancy: the grid of network `which` from its own density.  Lattice: torch.linspace(lo_a, hi_a, G+1) per axis,
 *   sigma from nm_grid_sigma's sigma-only sweep of that network (directions = positions); a cell is raw-occupied when the max
 *   of its 8 corner sigmas is > threshold or a corner is NaN; the grid is the raw occupancy dilated by `dilate` cells in
 *   Chebyshev distance (clamped at the box faces).  1 <= G <= 1024, 0 <= dilate <= G, threshold not NaN.  bits_out_dev (the
 *   ceil(G^3/32) words) or NULL.  Synchronises `stream` once.
 * nm_set_occupancy: installs caller bits (same layout) for network `which`; bits_dev NULL removes the grid.
 * nm_occupancy_query: evaluated_out_dev[m] = 1 if point m (pts_dev (M,3)) is evaluated under network `which`'s fresh grid,
 *   else 0.
 * nm_skip_stats: out_host = {samples seen, samples evaluated} of the coarse (or only) pass, then of the fine pass, summed
 *   over skipping renders and skipping training passes since the last call; resets them.  Synchronises the device. */
int nm_build_occupancy(NmHandle h, int which, const float* box_host, int G, float threshold, int dilate,
                       uint32_t* bits_out_dev_or_null, void* stream);
int nm_set_occupancy(NmHandle h, int which, const float* box_host, int G, const uint32_t* bits_dev_or_null);
int nm_occupancy_query(NmHandle h, int which, const float* pts_dev, int64_t M, uint8_t* evaluated_out_dev, void* stream);
int nm_skip_stats(NmHandle h, int64_t* out_host);

/* ---- hot path, host buffers (what a reference-side caller holding CPU tensors binds) ------------------ */
/* model.query(ray_batch) with host tensors (src/eval_nerf.py:62-69): copies H2D, renders, copies D2H, syncs. */
int nm_query_host(NmHandle h, const float* origins_host, int o_stride, const float* dirs_host, int64_t R,
                  const float* near_far_host, int flags, uint64_t seed, const NmRenderOut* out_host);
/* one image from a pose, results to host (eval_nerf.py image loop). */
int nm_render_image_host(NmHandle h, const float* pose_host, int H, int W, double focal, int ndc, int row0, int row1,
                         const float* near_far_host, int flags, uint64_t seed, const NmRenderOut* out_host);
/* model.sample_points with host tensors (src/mesh_nerf.py:43-48). */
int nm_point_mlp_host(NmHandle h, int which, const float* pts_host, const float* dirs_host, int64_t M,
                      float* out_host, int sigma_only);

/* ---- training (SURVEY §8f-1) --------------------------------------------------------------------------
 * Replaces `loss.backward()` of NeRFModel.training_step / BuFFModel.training_step (src/models/model_nerf.py:88-151,
 * model_buff.py) for the parameters of both FlexibleNeRFModels: gradients flow from the bundles' rgb_map through
 * VolumeRenderer (src/nerf/modules.py:67-121) and the network (src/nerf/models.py:60-80); SamplePDF is detached
 * (modules.py:201).  The call re-runs the forward for these rays (same flags + seed => same samples and noise) and
 * ACCUMULATES dL/dtheta into the handle's gradient buffers (fp32, atomics: summation order is not reproducible).
 *   nm_backward_rays : d_rgb_dev (R,3) = dL/d rgb_map of the main bundle (fine, or the only one);
 *                      d_coarse_rgb_dev (R,3) or NULL = dL/d coarse rgb_map (two-network NeRF only).
 *   nm_loss_backward : the reference's loss itself, mse(coarse.rgb_map, target) + mse(fine.rgb_map, target)
 *                      (mean over R*3); loss_dev (2 floats, device, or NULL) += {coarse-or-only term, fine term}.
 *   nm_get_grad      : copies the gradient of one state-dict tensor (SURVEY A.1 names, reference (out,in) layout)
 *                      into out_dev.
 * Loss terms other than rgb_map (depth, acc, weights) carry no gradient here; the reference has none. */
int nm_zero_grad(NmHandle h, void* stream);
int nm_backward_rays(NmHandle h, const float* origins_dev, int o_stride, const float* dirs_dev, int64_t R,
                     const float* near_far_host, const float* near_dev, const float* far_dev, int flags, uint64_t seed,
                     const float* d_rgb_dev, const float* d_coarse_rgb_dev, void* stream);
int nm_loss_backward(NmHandle h, const float* origins_dev, int o_stride, const float* dirs_dev, int64_t R,
                     const float* near_far_host, const float* near_dev, const float* far_dev, int flags, uint64_t seed,
                     const float* target_rgb_dev, float* loss_dev, void* stream);
int nm_get_grad(NmHandle h, int which, const char* name, float* out_dev, int64_t numel, void* stream);

/* ---- BuFF tree maintenance (SURVEY §8f rank 4) ----------------------------------------------------------
 * nm_ray_voxel_indices: the `indices` output of TreeSampling.batch_ray_voxel_intersect (src/nerf/tree.py:215-343,
 *   deterministic branch) for cfg.num_coarse samples per ray: the voxel (row of the nm_set_tree list) every sample lies
 *   in, int32 (R,S), -1 on rays that hit no voxel; z_out_dev (R,S) optionally receives the sample distances with the
 *   uniform fallback on those rays (model_buff.py:52-53).  _ex: flags = NM_FLAG_RANDOM_VOXELS selects the random branch
 *   (tree.py:280-297) with `seed` — pass the seed of the render call whose samples are being attributed.
 * nm_tree_integrate: TreeSampling.ray_batch_integration (tree.py:177-206) past its step gate: memm[v] +=
 *   (sum of weights / sum of weight masks of the samples in v - memm[v]) / counter for every voxel that received a sample.
 *   idx/weights/mask: n = R*S entries (whole batch, idx -1 skipped, or only the rows of rays that hit); an idx outside [0, V) is
 *   skipped.  counter >= 1 and V >= 1; n = 0 launches nothing. */
int nm_ray_voxel_indices(NmHandle h, const float* origins_dev, int o_stride, const float* dirs_dev, int64_t R,
                         const float* near_far_host, float* z_out_dev, int32_t* idx_out_dev, void* stream);
int nm_ray_voxel_indices_ex(NmHandle h, const float* origins_dev, int o_stride, const float* dirs_dev, int64_t R,
                            const float* near_far_host, int flags, uint64_t seed, float* z_out_dev, int32_t* idx_out_dev,
                            void* stream);
int nm_tree_integrate(NmHandle h, const int32_t* idx_dev, const float* weights_dev, const float* mask_weights_dev, int64_t n,
                      float* memm_dev, int32_t V, int32_t counter, void* stream);

/* Test hook for the weight-gradient GEMM of the backward pass (nm_gemm_tc.cu): D (M,N) += A B^T, i.e.
 * d[m][n] += sum_k a[k][m] b[k][n], from fp32 row-major device arrays a (K,M) and b (K,N) (K = points), packed into the
 * bf16 hi/lo operand layouts the backward uses and reduced over K splits with atomics.  n_passes: 3 (hi*hi + lo*hi +
 * hi*lo) or 1 (hi*hi). */
int nm_debug_gemm(NmHandle h, const float* a_dev, const float* b_dev, int M, int N, int K, int n_passes, float* d_dev,
                  void* stream);

/* Test hook for the network backward alone (no compositor): runs it on M points built like nm_point_mlp's, with
 * dout_dev (M,4) = [d rgb logits (before the sigmoid), d raw sigma] per point, and ACCUMULATES dL/dtheta of network
 * `which` into the handle's gradient buffers (nm_zero_grad clears them, nm_get_grad reads them).  The handle's precision
 * selects the path: tensor cores (training forward that emits the backward's operands, heads, data-gradient chain,
 * weight-gradient GEMMs) or NM_PREC_FP32.  dout_dev must be 16-byte aligned. */
int nm_debug_mlp_backward(NmHandle h, int which, const float* pts_dev, const float* dirs_dev, int64_t M, const float* dout_dev,
                          void* stream);

/* Test hook for the training compositor adjoint alone (composite_backward_kernel, nm_train.cu): from raw_dev (R,S,4) =
 * (sigmoid rgb, raw sigma), t_dev (R,S), dirs_dev (R,3) and d_rgb_dev (R,3) = dL/d rgb_map it writes dout_dev (R,S,4) =
 * [dL/d rgb logits (through the sigmoid), dL/d raw sigma], the per-point adjoint nm_debug_mlp_backward takes.  noise_std
 * and seed are the sigma noise of the forward: seed is the compositor's stream, already salted (the training backward
 * passes seed ^ salt of the pass).  1 <= S <= 512; raw_dev and dout_dev 16-byte aligned; R = 0 launches nothing. */
int nm_debug_composite_backward(NmHandle h, const float* raw_dev, const float* t_dev, const float* dirs_dev,
                                const float* d_rgb_dev, int64_t R, int S, float noise_std, uint64_t seed, int white_bg,
                                float* dout_dev, void* stream);
/* Test hook for the inference compositor alone (composite_kernel, nm_render.cu), with the arguments a render pass gives it:
 * from raw_dev (R,S,4) = (sigmoid rgb, raw sigma), t_dev (R,S) and dirs_dev (R,3) it writes the non-NULL fields rgb, depth,
 * depth_raw, acc, disp, weights and mask_weights of out_dev (a host struct of device pointers; every other field must be
 * NULL).  noise_std and seed are the pass's sigma noise, seed already salted (a render passes its chunk seed ^ the pass's
 * salt); training = 1 leaves depth unthresholded; thr is the mask_weights threshold.  1 <= S <= 512; raw_dev 16-byte
 * aligned; argument errors are rejected before anything is launched; R = 0 launches nothing. */
int nm_debug_composite(NmHandle h, const float* raw_dev, const float* t_dev, const float* dirs_dev, int64_t R, int S,
                       float noise_std, uint64_t seed, int white_bg, int training, float thr, const NmRenderOut* out_dev,
                       void* stream);
/* Test hook for the inverse-CDF resampler alone (invcdf_kernel, nm_render.cu), the call a two-network render makes: from
 * the coarse depths t_c_dev (R,Nc), ascending per ray, and the coarse weights w_c_dev (R,Nc) it writes t_out_dev (R,Nc+Nf),
 * the coarse depths and Nf new samples merged in ascending order.  perturb = 0 places the samples at u_dev (Nf); otherwise
 * u is drawn from the stream `seed` (already salted: a render passes its chunk seed ^ 0x9e3779b9) and u_dev may be NULL.
 * 3 <= Nc <= 256, 1 <= Nf, Nc + Nf <= 512; argument errors are rejected before anything is launched; R = 0 launches
 * nothing. */
int nm_debug_sample_pdf(NmHandle h, const float* t_c_dev, const float* w_c_dev, const float* u_dev, int64_t R, int Nc, int Nf,
                        int perturb, uint64_t seed, float* t_out_dev, void* stream);

/* ---- host-only debugging aid (no CUDA): the layer program + tensor-core weight blocks (64x64, 128B-swizzled, schedule
 * order), for CPU tests of the schedule / swizzle logic.  program_out receives the internal NetProgram struct
 * (nerfmeshes_b200/csrc/nm_program.h). */
int nm_debug_pack(const NmNetDesc* desc, int n_tensors, const char* const* names, const float* const* tensors_host,
                  const int64_t* numel, int sigma_only, void* program_out, size_t program_cap, uint8_t* pack_out,
                  size_t pack_cap, size_t* pack_need);
/* The same blocks regrouped into the wide stream nm_load_weights uploads and the wgmma kernel reads (layout:
 * nm_program.h wide_offset). */
int nm_debug_pack_wide(const NmNetDesc* desc, int n_tensors, const char* const* names, const float* const* tensors_host,
                       const int64_t* numel, int sigma_only, void* program_out, size_t program_cap, uint8_t* pack_out,
                       size_t pack_cap, size_t* pack_need);

/* Host-only: how the fused compositor deals 64-point tiles to the kernel's workers (two consumer warpgroups per CTA) for
 * `samples_per_ray` samples (nm_mlp_tc.cu).  Returns the group size g = lcm(S,64)/64 (0: the fused compositor is not used
 * for this S); if tiles_out != NULL it receives the tile indices worker `cta` of `grid` workers processes, in order, for a launch of n_tiles tiles (at most cap entries; *n_out = count). */
int nm_debug_tile_schedule(int samples_per_ray, int64_t n_tiles, int grid, int cta, int64_t* tiles_out, int64_t cap, int64_t* n_out);
/* Host-only: the fused MLP kernel's shared-memory layout for a layer program (the NetProgram nm_debug_pack returns), a
 * dynamic shared-memory limit of max_smem bytes, the fused compositor on (comp_on != 0) or off, inference (training == 0)
 * or the training modes (which keep the bias and head vectors in shared memory) and a ring-slot cap (slot_cap <= 0: none;
 * NM_MLP_RING_SLOTS sets it for launches).  out5 = {ring slots, activation buffers' offset, barriers' offset, compositor
 * carry offset, total bytes}.  Fails (<0) when the network leaves room for fewer than two slots. */
int nm_debug_mlp_layout(const void* program, size_t program_size, int max_smem, int comp_on, int training, int slot_cap,
                        int64_t* out5);

/* Device-side error flags, readable even after a kernel trapped: out2[0] = tensor-core pipeline watchdog code (0 = ok),
 * out2[1] = AABB hit-list overflow (a ray through more than 512 voxels; cleared once nm_check_flags or an entry point has
 * reported it). */
int nm_kernel_flags(NmHandle h, int32_t* out2);
/* Synchronises `stream`, then fails (<0, message in nm_last_error) if a kernel of this handle raised a device-side flag.
 * The asynchronous device-pointer entry points report flags raised by EARLIER calls when they are entered; *_host calls
 * check before they return.  The watchdog is reported on every call (the device is no longer trusted); the input
 * conditions, an AABB hit-list overflow and a bad mesh, are reported once and then cleared. */
int nm_check_flags(NmHandle h, void* stream);

/* ---- introspection ---------------------------------------------------------------------------------- */
/* number of kernels launched through this handle since creation (bench.py's gpu_launches). */
int64_t nm_launch_count(NmHandle h);
/* number of points this handle has sent through a network's sigma-only program since creation: sigma-only point queries,
 * the density sweeps, and the coarse pass of a two-network inference render that asks for no coarse colour (when the
 * network has a separate sigma head, i.e. view directions). */
int64_t nm_sigma_only_points(NmHandle h);
/* duration in ms of the last fused-MLP launch sequence, measured with CUDA events on the call's stream when
 * timing is enabled (bench.py's roofline); <0 if disabled. */
int nm_set_timing(NmHandle h, int enable);
double nm_mlp_time_ms(NmHandle h, int64_t* points_out, int64_t* launches_out);

#ifdef __cplusplus
}
#endif
#endif /* NERFMESHES_B200_H */
