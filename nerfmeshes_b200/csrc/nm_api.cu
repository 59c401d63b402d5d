// C ABI of libnerfmeshes_b200.so (include/nerfmeshes_b200.h): handle lifecycle, weight loading, and the orchestration
// of the hot path — the body of NeRFModel.forward / BuFFModel.forward (src/models/model_nerf.py:37-78,
// model_buff.py:34-69) and extract_radiance (src/mesh_nerf.py:27-53) as stream-ordered kernel sequences.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <algorithm>
#include <cstring>
#include <vector>

#include "nm_common.h"
#include "nm_gemm.h"

namespace nm {
const char* last_error();
}

using namespace nm;

namespace {

struct Buf {
  void* p = nullptr;
  size_t cap = 0;
  int ensure(size_t bytes) {
    if (bytes <= cap) return 0;
    if (p) cudaFree(p);
    p = nullptr; cap = 0;
    size_t want = bytes + bytes / 8;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) { set_error("cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e)); return -2; }
    cap = want;
    return 0;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  template <class T> T* as() { return reinterpret_cast<T*>(p); }
};

}  // namespace

struct NmHandle_t {
  int device = 0;
  int num_sms = 0;
  NmRenderCfg cfg{};
  NetDev nets[2];
  bool has_fine = false;
  NmNetDesc desc[2]{};
  Buf s_table, u_table, voxels;
  int V = 0;
  // workspace
  Buf t_c, raw_c, w_c, t_f, raw_f, t_u, dirs, origins, lin[3], small, stage_in[3], stage_out[12];
  int lin_n[3] = {0, 0, 0};
  int* d_err = nullptr;       // [0] tensor-core pipeline watchdog code, [1] aabb hit-list overflow (cleared when reported),
                              // [2] mesh input error
                              // (mesh sampler 1: face index out of range, 2: total area not positive; component filter
                              // 3: face index out of range; decimation 4: face index out of range; texture bake 5:
                              // face index out of range; mesh raster 6: face index out of range; cleared when reported)
                              // (device alias of h_err)
  int* h_err = nullptr;       // mapped pinned host memory: still readable after a device-side trap
  double* d_stats = nullptr;
  cudaStream_t own_stream = nullptr;
  int64_t launches = 0;
  // timing of the fused-MLP launches
  bool timing = false;
  std::vector<cudaEvent_t> ev;
  size_t ev_used = 0;
  int64_t mlp_points = 0, mlp_launches = 0;
  int64_t sigma_points = 0;        // points sent through a network's sigma-only program since creation
  Buf mc_ws, mc_ws2;               // marching cubes: the count step's bit masks and scans, read by the emit step; the emit
                                   // step's vertex / triangle records
  int64_t mc_counts[2] = {0, 0};   // {vertices, triangles} of the last count step: sizes of the emit step
  Buf ss_tab, ss_ws;               // super-sampled emit: the six coordinate tables; chunk points (M,3) + sigma (M,)
  Buf ms_ws, nn_ws;                // chamfer evaluation: surface sampler (areas, cdf); grid nearest-neighbour search
  Buf cc_ws;                       // small-component removal: labels, sizes, masks and scans (~28 B per vertex + 8 B per face)
  Buf dc_ws;                       // decimation: positions, quadrics, vertex-face lists, candidate edges (~150 B per vertex
                                   // + 90 B per face)
  Buf tx_ws;                       // texture bake: first references, unreferenced-vertex list, one chunk's queries and colours
                                   // (~40 B per chunk texel: 160 MB at the default 4 Mi)
  Buf rs_ws;                       // mesh raster: one depth-and-face key per pixel, one record per face (8 B per pixel + 52 B
                                   // per face)
  Buf sf_ws;                       // surface points: one view's ray directions, keep mask and its scan (20 B per pixel)
  Buf sp_ws;                       // sparse sweep (nm_sparse_sweep.cu): block flags, two bit-volumes, scans, one chunk of points
  int sp_grid[4] = {0, 0, 0, 0};   // {n0, n1, n2, block} of the last nm_sparse_sweep_lattice, and the volume it wrote:
  const float* sp_vol = nullptr;   // what nm_sparse_sweep_run must be called with
  struct OccGrid {                 // empty-space skipping (nm_occupancy.cu, DESIGN §4.15): one grid per network slot
    bool valid = false;            // installed (nm_build_occupancy / nm_set_occupancy)
    bool stale = false;            // the slot's weights were loaded after it: inference refuses it, training skipping takes it
    float lo[3], hi[3], inv[3];
    int G = 0;
    Buf bits;
  } occ[2];
  Buf oc_ws;                       // grid build: one plane chunk of the sigma lattice, two G^3 byte volumes
  Buf sk_ws;                       // skipping render: marks, scan, index list (12 B per sample of a chunk pass) + one network
                                   // launch's points, directions and outputs (40 B per point, 160 MB at the default 4 Mi)
  Buf ts_ws[2], ts_pts[2];         // skipping training step, per pass (0: coarse or only, 1: fine), held until the backward:
                                   // marks, scan, index list (12 B per sample); staged points, directions (24 B per evaluated
                                   // sample) and one network launch's outputs
  Buf train_ws_c;                  // skipping training step: the coarse pass's emitted operands (the fine pass's are in train_ws)
  int64_t skip_counts[4] = {0, 0, 0, 0};   // samples seen / evaluated, coarse (or only) pass, fine pass (nm_skip_stats)
  Buf sg_ws;                       // density gradient (nm_sigma_grad): one chunk's forward / chain / tail workspace; grow-only,
                                   // held until nm_destroy (~22 KB per chunk point for the 8x256 network, ~5.8 GB at the default)
  // training (nm_train.cu): gradient accumulators per network + scratch
  Buf g_wt[2], g_bias[2], g_head[2], train_ws, dout, trans, tr_rgb[2], tr_drgb[2];
  bool grads_ready = false;
};

namespace {

constexpr int kOccMaxRes = 1024;     // cells per axis of an occupancy grid (two G^3-byte build volumes: 2 GB at 1024)
OccLookup occ_lookup(NmHandle_t::OccGrid& g) {
  return OccLookup{g.bits.as<uint32_t>(), {g.lo[0], g.lo[1], g.lo[2]}, {g.inv[0], g.inv[1], g.inv[2]}, g.G};
}

// points per network launch of the super-sampled mesh emit (16 B of workspace each: 64 MB at 4 Mi); NM_SS_CHUNK_POINTS
// overrides it, read per call (the tests cross chunk boundaries with small values)
long long ss_chunk_points() {
  const char* e = getenv("NM_SS_CHUNK_POINTS");
  const long long x = e ? atoll(e) : 0;
  return x > 0 ? x : (1ll << 22);
}

// points per network launch of the sparse sweep (20 B of workspace each: 80 MB at 4 Mi); NM_SPARSE_CHUNK_POINTS overrides
// it, read per call (the tests use values below one round's point list)
long long sparse_chunk_points() {
  const char* e = getenv("NM_SPARSE_CHUNK_POINTS");
  const long long x = e ? atoll(e) : 0;
  return x > 0 ? x : (1ll << 22);
}

// faces of the mesh raster whose bounding box holds at least this many pixel samples are drawn one screen tile per CTA
// instead of one face per thread; NM_RASTER_BIG_FACE_PIXELS overrides it, read per call (the tests use 1, every face on the
// tile pass, and 2^30, none)
long long raster_big_face_pixels() {
  const char* e = getenv("NM_RASTER_BIG_FACE_PIXELS");
  const long long x = e ? atoll(e) : 0;
  return x > 0 ? x : 256;
}

// texels per chunk of the texture bake (40 B of workspace each: 160 MB at 4 Mi); NM_TEXTURE_CHUNK_TEXELS overrides it, read
// per call (the tests cross chunk boundaries with small values)
long long texture_chunk_texels() {
  const char* e = getenv("NM_TEXTURE_CHUNK_TEXELS");
  const long long x = e ? atoll(e) : 0;
  return x > 0 ? x : (1ll << 22);
}

// points per chunk of the density gradient (~22 KB of workspace each for the 8x256 network: ~5.8 GB at 256 Ki);
// NM_SIGMA_GRAD_CHUNK_POINTS overrides it, read per call (the tests cross chunk boundaries with small values)
long long sigma_grad_chunk_points() {
  const char* e = getenv("NM_SIGMA_GRAD_CHUNK_POINTS");
  const long long x = e ? atoll(e) : 0;
  return x > 0 ? x : (1ll << 18);
}

// points per network launch of the skipping render (40 B of workspace each: 160 MB at 4 Mi); NM_SKIP_CHUNK_POINTS
// overrides it, read per call (the tests cross launch boundaries with small values)
long long skip_chunk_points() {
  const char* e = getenv("NM_SKIP_CHUNK_POINTS");
  const long long x = e ? atoll(e) : 0;
  return x > 0 ? x : (1ll << 22);
}

// rays per internal chunk (bounds the per-sample workspace: 20 B x 192 samples x 1 Mi rays = 4 GB); NM_CHUNK_RAYS overrides (tests)
long long chunk_rays() {
  static long long v = [] { const char* e = getenv("NM_CHUNK_RAYS"); long long x = e ? atoll(e) : 0; return x > 0 ? x : (1ll << 20); }();
  return v;
}

int check_kernel_flags(NmHandle h);

int bind_device(NmHandle h) {
  NM_CHECK(h != nullptr, "null handle");
  NM_CUDA(cudaSetDevice(h->device));
  return 0;
}

// device-pointer (asynchronous) entry points cannot wait for their own kernels; they report the device-side error flags
// raised by EARLIER work on this handle (mapped host memory, no synchronisation) and callers that need the answer for
// the current call use nm_check_flags(h, stream), which synchronises first.
int bind_checked(NmHandle h) {
  if (int e = bind_device(h)) return e;
  return check_kernel_flags(h);
}

// torch.linspace(0,1,n) fp32: ATen's two-sided formula, whose upper half is one fused multiply-add (torch's values; two
// roundings there differ by an ulp at about a tenth of the points)
void linspace_host(int n, std::vector<float>* out) {
  out->resize(n);
  if (n == 1) { (*out)[0] = 0.f; return; }
  const float step = 1.0f / (float)(n - 1);
  for (int i = 0; i < n; ++i) (*out)[i] = (i < n / 2) ? 0.f + step * (float)i : std::fmaf(-step, (float)(n - 1 - i), 1.0f);
}

int upload(Buf* b, const void* src, size_t bytes) {
  if (int e = b->ensure(bytes)) return e;
  NM_CUDA(cudaMemcpy(b->p, src, bytes, cudaMemcpyHostToDevice));
  return 0;
}

int check_kernel_flags(NmHandle h) {
  const volatile int* flags = h->h_err;
  NM_CHECK(flags[0] == 0, "tensor-core pipeline watchdog fired (code %d)", flags[0]);
  if (flags[1]) {                   // an input condition too (a ray through too many voxels): reported once
    h->h_err[1] = 0;
    NM_CHECK(false, "AABB sampler: more than 512 voxel hits on one ray (samples / voxel indices of that ray are truncated)");
  }
  if (const int c = flags[2]) {     // a bad input mesh, not a broken device: reported once
    h->h_err[2] = 0;
    NM_CHECK(false, c == 1   ? "mesh sampler: a face index lies outside [0, V)"
                    : c == 2 ? "mesh sampler: the total face area is not positive and finite"
                    : c == 3 ? "mesh components: a face index lies outside [0, V) (the face was dropped)"
                    : c == 4 ? "mesh decimate: a face index lies outside [0, V) (the mesh was returned unchanged)"
                    : c == 5 ? "texture bake: a face index lies outside [0, V) (nothing was baked)"
                             : "mesh raster: a face index lies outside [0, V) (nothing was drawn)");
  }
  return 0;
}

// one fused-MLP launch in the configured arithmetic
int run_mlp(NmHandle h, int which, bool sigma_only, const MlpInput& in, float* out, cudaStream_t st, const MlpEmit* emit = nullptr,
            const CompositeArgs* comp = nullptr) {
  const NetDev& net = h->nets[which];
  NM_CHECK(net.loaded, "weights of network %d not loaded", which);
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  if (h->timing) {
    while (h->ev.size() < h->ev_used + 2) {
      cudaEvent_t e;
      NM_CUDA(cudaEventCreate(&e));
      h->ev.push_back(e);
    }
    e0 = h->ev[h->ev_used++]; e1 = h->ev[h->ev_used++];
    NM_CUDA(cudaEventRecord(e0, st));
  }
  int rc;
  if (h->cfg.precision == NM_PREC_FP32) rc = launch_mlp_simt(net, sigma_only, in, out, st, &h->launches);
  else rc = launch_mlp_tc(net, sigma_only, h->cfg.precision == NM_PREC_FAST ? 1 : 3, h->cfg.act_scale_log2, in, out,
                          h->num_sms, h->d_err, st, &h->launches, emit, comp);
  if (rc) return rc;
  if (sigma_only) h->sigma_points += in.M;
  if (h->timing) {
    NM_CUDA(cudaEventRecord(e1, st));
    h->mlp_points += in.M;
    h->mlp_launches += 1;
  }
  return 0;
}

constexpr uint64_t kNoiseSaltMain = 0x5bd1e995ull, kNoiseSaltCoarse = 0x7f4a7c15a3c59ac3ull;
// the random voxel draws (NM_FLAG_RANDOM_VOXELS) and the inverse-CDF jitter of a chunk: streams of their own, so that no
// two consumers of one chunk seed share a splitmix64 state (tests/test_ray_samplers_reference.py checks every pair)
constexpr uint64_t kVoxelSalt = 0xd1b54a32d192ed03ull, kInvCdfSalt = 0x9e3779b9ull;

struct RayBatch {
  const float* origins; int o_stride; const float* dirs; long long R;
  float nf[2]; const float* near_dev; const float* far_dev;
};

float* off(float* p, long long n) { return p ? p + n : nullptr; }

// NM_FLAG_SKIP_EMPTY_TRAIN (DESIGN §4.15): what one pass of a skipping training forward leaves for its backward
struct TrainSkip {
  // in
  bool emit = false;            // the pass carries a gradient and may leave the backward's operands (tensor cores, scale 0)
  double budget = 0;            // bytes the emitted operands of both passes may take (NM_TRAIN_DIRECT_GB)
  double* committed = nullptr;  // bytes already taken by the other pass's
  // out
  long long M = 0;              // evaluated samples
  const int* pos = nullptr;     // exclusive scan of the marks (R*s + 1): sample m's compact slot
  const float* pts = nullptr;   // (M,3) staged points
  const float* dirs = nullptr;  // (M,3) their directions
  float* ws = nullptr;          // the emitted operands (train_emit_setup carving for M points), or NULL: walk with recompute
};

// the flag rules of NM_FLAG_SKIP_EMPTY_TRAIN, checked before anything is launched
int check_train_skip(NmHandle h, int flags) {
  if (!(flags & NM_FLAG_SKIP_EMPTY_TRAIN)) return 0;
  NM_CHECK(flags & NM_FLAG_TRAINING, "NM_FLAG_SKIP_EMPTY_TRAIN is a training path: it needs NM_FLAG_TRAINING "
           "(inference renders skip with NM_FLAG_SKIP_EMPTY)");
  NM_CHECK(!(flags & NM_FLAG_TEACHER_T), "NM_FLAG_SKIP_EMPTY_TRAIN does not take NM_FLAG_TEACHER_T");
  NM_CHECK(!(flags & NM_FLAG_SKIP_EMPTY), "NM_FLAG_SKIP_EMPTY_TRAIN and NM_FLAG_SKIP_EMPTY exclude each other "
           "(training and inference skipping)");
  const int nets = (h->has_fine && !(flags & NM_FLAG_BUFF) && h->cfg.num_fine > 0) ? 2 : 1;
  for (int k = 0; k < nets; ++k)
    NM_CHECK(h->occ[k].valid, "NM_FLAG_SKIP_EMPTY_TRAIN: no occupancy grid for network %d (build one with nm_build_occupancy; "
             "a weight load keeps it, stale, for training)", k);
  return 0;
}

// NeRFModel.forward / BuFFModel.forward for one chunk of rays; `o` already offset to the chunk.
// emit_c / emit_f: training only — the coarse (or only) / fine network's forward also leaves the backward's operands (MlpEmit)
// need_raw: the caller reads h->raw_c / h->raw_f afterwards (the training backward) — otherwise the compositor runs inside the
// MLP kernel and the per-sample network outputs never reach HBM (NM_FUSED_COMPOSITE=0 keeps the two-kernel path for A/B tests).
// tsk: NM_FLAG_SKIP_EMPTY_TRAIN — per pass (0: coarse or only, 1: fine) what the backward needs (TrainSkip); with it the
// passes size their emitted operands themselves and emit_c / emit_f are NULL.
int render_chunk(NmHandle h, const RayBatch& rb, int flags, uint64_t seed, const NmRenderOut& o, cudaStream_t st,
                 const MlpEmit* emit_c = nullptr, const MlpEmit* emit_f = nullptr, bool need_raw = false,
                 TrainSkip* tsk = nullptr) {
  const NmRenderCfg& c = h->cfg;
  const long long R = rb.R;
  const int Nc = c.num_coarse;
  const bool buff = flags & NM_FLAG_BUFF;
  const bool teacher = flags & NM_FLAG_TEACHER_T;
  const bool training = flags & NM_FLAG_TRAINING;
  const int Nf = (h->has_fine && !buff) ? c.num_fine : 0;
  const int S = Nc + Nf;
  // the coarse and the fine compositor draw independent sigma noise (two torch.randn calls in the reference): distinct salts
  auto rays_input = [&](const float* t, int s) {
    MlpInput in{};
    in.mode = IN_RAYS; in.dirs = rb.dirs; in.ray_o = rb.origins; in.o_stride = rb.o_stride; in.t = t; in.S = s;
    in.M = R * s;
    return in;
  };
  const char* fe = getenv("NM_FUSED_COMPOSITE");       // read per call: the tests flip it to compare the two paths
  const bool fused_env = !fe || atoi(fe) != 0;
  const bool skip = flags & NM_FLAG_SKIP_EMPTY;
  if (skip) {
    NM_CHECK(!training && !teacher && !need_raw && !emit_c && !emit_f,
             "NM_FLAG_SKIP_EMPTY is an inference path: it takes neither NM_FLAG_TRAINING nor NM_FLAG_TEACHER_T");
    for (int k = 0; k < ((Nf > 0) ? 2 : 1); ++k)
      NM_CHECK(h->occ[k].valid && !h->occ[k].stale, "NM_FLAG_SKIP_EMPTY: no occupancy grid for network %d (nm_build_occupancy / nm_set_occupancy; "
               "loading that network's weights drops its grid)", k);
  }
  // empty-space skipping (DESIGN §4.15): only the samples network `which`'s grid marks go through it, as explicit points in
  // launches of at most skip_chunk_points(); every other sample enters the compositor as raw (0,0,0,-inf), which the pass's
  // sigma noise cannot lift above 0.  Training (ts != NULL): the index data and ALL staged points stay in the pass's own
  // buffers for the backward, and when the backward's operands for the M evaluated points fit the budget the network runs
  // in one emitting launch over them.
  auto skip_raw = [&](int which, Buf& raw_buf, const float* t, int s, TrainSkip* ts) -> int {
    NmHandle_t::OccGrid& g = h->occ[which];
    const long long n = R * s;
    NM_CHECK(n + 1 < (1ll << 31), "%s: %lld samples in one chunk exceed the int32 index list (lower NM_CHUNK_RAYS)",
             ts ? "NM_FLAG_SKIP_EMPTY_TRAIN" : "NM_FLAG_SKIP_EMPTY", n);
    long long P = skip_chunk_points();
    const size_t nb = (size_t)(n + 1) * 4, nblk = (size_t)((n + 1 + kScanBlockEntries - 1) / kScanBlockEntries) * 4;
    const long long cap = P < n ? P : (n > 0 ? n : 1);
    const size_t o_pos = (nb + 255) & ~(size_t)255, o_blk = 2 * o_pos, o_idx = o_blk + ((nblk + 255) & ~(size_t)255);
    const size_t o_pts = o_idx + o_pos, o_dir = o_pts + (((size_t)cap * 12 + 255) & ~(size_t)255);
    const size_t o_out = o_dir + (((size_t)cap * 12 + 255) & ~(size_t)255), bytes = o_out + (size_t)cap * 16;
    Buf& ws_buf = ts ? h->ts_ws[which] : h->sk_ws;
    if (int e = ws_buf.ensure(ts ? o_pts : bytes)) return e;
    uint8_t* ws = ws_buf.as<uint8_t>();
    int* idx = reinterpret_cast<int*>(ws + o_idx);
    long long M = 0;
    if (int e = raw_buf.ensure((size_t)n * 16)) return e;
    if (int e = occ_compact(occ_lookup(g), rb.origins, rb.o_stride, rb.dirs, t, R, s, reinterpret_cast<int*>(ws), reinterpret_cast<int*>(ws + o_pos),
                            reinterpret_cast<int*>(ws + o_blk), idx, raw_buf.as<float>(), &M, st, &h->launches)) return e;
    h->skip_counts[2 * which] += n;
    h->skip_counts[2 * which + 1] += M;
    float* pts = reinterpret_cast<float*>(ws + o_pts);
    float* dirs = reinterpret_cast<float*>(ws + o_dir);
    float* out = reinterpret_cast<float*>(ws + o_out);
    MlpEmit em{};
    if (ts) {
      *ts = TrainSkip{ts->emit, ts->budget, ts->committed};
      ts->M = M;
      ts->pos = reinterpret_cast<const int*>(ws + o_pos);
      if (M == 0) return 0;                       // no network work; the pass's gradients stay untouched
      const NetProgram& G = h->nets[which].full;
      const size_t wsb = ts->emit ? train_ws_bytes(G, M, true) + 1024 : 0;
      if (wsb && *ts->committed + (double)wsb <= ts->budget) {
        Buf& wb = (which == NM_NET_COARSE && Nf > 0) ? h->train_ws_c : h->train_ws;
        if (int e = wb.ensure(wsb + 1024)) return e;
        ts->ws = reinterpret_cast<float*>(((uintptr_t)wb.p + 1023) & ~(uintptr_t)1023);
        train_emit_setup(G, M, ts->ws, &em);
        *ts->committed += (double)wsb;
        P = M;                                    // the emitting launch covers every evaluated point
      }
      const long long lc = P < M ? P : M;
      const size_t q_dir = (((size_t)M * 12 + 255) & ~(size_t)255), q_out = 2 * q_dir;
      if (int e = h->ts_pts[which].ensure(q_out + (size_t)lc * 16)) return e;
      uint8_t* tp = h->ts_pts[which].as<uint8_t>();
      pts = reinterpret_cast<float*>(tp); dirs = reinterpret_cast<float*>(tp + q_dir); out = reinterpret_cast<float*>(tp + q_out);
      if (int e = launch_occ_stage(idx, M, s, rb.origins, rb.o_stride, rb.dirs, t, pts, dirs, st, &h->launches)) return e;
      ts->pts = pts; ts->dirs = dirs;
    }
    for (long long j0 = 0; j0 < M; j0 += P) {
      const long long m = (M - j0 < P) ? M - j0 : P;
      if (!ts)
        if (int e = launch_occ_stage(idx + j0, m, s, rb.origins, rb.o_stride, rb.dirs, t, pts, dirs, st, &h->launches)) return e;
      MlpInput in{};
      in.mode = IN_POINTS; in.pts = ts ? pts + 3 * j0 : pts; in.dirs = ts ? dirs + 3 * j0 : dirs; in.M = m;
      if (int e = run_mlp(h, which, false, in, out, st, (ts && ts->ws) ? &em : nullptr)) return e;
      if (int e = launch_occ_expand(out, idx + j0, m, raw_buf.as<float>(), st, &h->launches)) return e;
    }
    return 0;
  };
  // network `which` on the samples t (R,s) + VolumeRenderer: one launch when eligible, else raw (R,s,4) through `raw_buf`
  auto mlp_composite = [&](int which, Buf& raw_buf, const MlpEmit* emit, const float* t, int s, float* rgb, float* depth,
                           float* depth_raw, float* acc, float* disp, float* w, float* mw, uint64_t salt = kNoiseSaltMain) -> int {
    CompositeArgs a{};
    a.t = t; a.dirs = rb.dirs; a.R = R; a.S = s; a.noise_std = c.noise_std; a.seed = seed ^ salt;
    a.white_bg = c.white_background; a.training = training ? 1 : 0; a.thr = c.attenuation_threshold;
    a.rgb = rgb; a.depth = depth; a.depth_raw = depth_raw; a.acc = acc; a.disp = disp; a.weights = w; a.mask_weights = mw;
    if (skip || tsk) {
      if (int e = skip_raw(which, raw_buf, t, s, tsk ? &tsk[which] : nullptr)) return e;
      a.raw = raw_buf.as<float>();
      return launch_composite(a, st, &h->launches);
    }
    const bool fuse = fused_env && !need_raw && !emit && c.precision != NM_PREC_FP32 && mlp_tc_composite_group(s) > 0;
    // The coarse pass of a two-network inference render whose caller reads no coarse colour: its weights (and so the fine
    // samples), acc and disp depend on sigma alone, so the sigma-only program runs (bit-identical sigma, without the
    // feature, direction and rgb layers).  A network without view directions has one output layer for rgb and sigma; its
    // sigma-only program is the full one, so it keeps the full path.
    const NetProgram& sp = h->nets[which].sigma;
    const bool sigma_only = fuse && which == NM_NET_COARSE && Nf > 0 && !training && rgb == nullptr &&
                            sp.layers[sp.n_layers - 1].kind == KIND_SIGMA;
    if (fuse) return run_mlp(h, which, sigma_only, rays_input(t, s), nullptr, st, nullptr, &a);
    if (int e = raw_buf.ensure((size_t)R * s * 16)) return e;
    if (int e = run_mlp(h, which, false, rays_input(t, s), raw_buf.as<float>(), st, emit)) return e;
    a.raw = raw_buf.as<float>();
    return launch_composite(a, st, &h->launches);
  };

  if (teacher) {
    NM_CHECK(o.t_vals != nullptr, "NM_FLAG_TEACHER_T needs out.t_vals as input");
    const int which = (h->has_fine && !buff) ? NM_NET_FINE : NM_NET_COARSE;
    return mlp_composite(which, h->raw_f, nullptr, o.t_vals, S, o.rgb, o.depth, o.depth_raw, o.acc, o.disp, o.weights, o.mask_weights);
  }

  // coarse / uniform samples (a3)
  if (int e = h->t_c.ensure((size_t)R * Nc * 4)) return e;
  float* t_c = h->t_c.as<float>();
  if (int e = launch_stratified(h->s_table.as<float>(), Nc, R, rb.nf, rb.near_dev, rb.far_dev, c.lindisp, c.perturb,
                                seed, t_c, st, &h->launches)) return e;
  if (buff) {
    NM_CHECK(h->V > 0, "BuFF render without a voxel list (nm_set_tree)");
    NM_CHECK(rb.near_dev == nullptr, "BuFF path takes scalar near/far");
    if (int e = h->t_u.ensure((size_t)R * Nc * 4)) return e;
    float* z = h->t_u.as<float>();
    if (int e = launch_aabb(h->voxels.as<float>(), h->V, rb.origins, rb.o_stride, rb.dirs, R, rb.nf[0], rb.nf[1], Nc,
                            h->s_table.as<float>(), t_c, z, nullptr, h->d_err + 1, st, &h->launches,
                            (flags & NM_FLAG_RANDOM_VOXELS) ? 1 : 0, seed ^ kVoxelSalt)) return e;
    if (o.t_vals) NM_CUDA(cudaMemcpyAsync(o.t_vals, z, (size_t)R * Nc * 4, cudaMemcpyDeviceToDevice, st));
    return mlp_composite(NM_NET_COARSE, h->raw_c, emit_c, z, Nc, o.rgb, o.depth, o.depth_raw, o.acc, o.disp, o.weights, o.mask_weights);
  }
  if (Nf == 0) {
    if (o.t_vals) NM_CUDA(cudaMemcpyAsync(o.t_vals, t_c, (size_t)R * Nc * 4, cudaMemcpyDeviceToDevice, st));
    return mlp_composite(NM_NET_COARSE, h->raw_c, emit_c, t_c, Nc, o.rgb, o.depth, o.depth_raw, o.acc, o.disp, o.weights, o.mask_weights);
  }
  float* w_c = o.coarse_weights;
  if (!w_c) { if (int e = h->w_c.ensure((size_t)R * Nc * 4)) return e; w_c = h->w_c.as<float>(); }
  if (int e = mlp_composite(NM_NET_COARSE, h->raw_c, emit_c, t_c, Nc, o.coarse_rgb, nullptr, nullptr, o.coarse_acc, o.coarse_disp, w_c,
                            nullptr, kNoiseSaltCoarse)) return e;
  // inverse-CDF resampling + merge (a8)
  float* t_f = o.t_vals;
  if (!t_f) { if (int e = h->t_f.ensure((size_t)R * S * 4)) return e; t_f = h->t_f.as<float>(); }
  if (int e = launch_invcdf(t_c, w_c, h->u_table.as<float>(), Nc, Nf, R, c.perturb, seed ^ kInvCdfSalt, t_f, st, &h->launches)) return e;
  return mlp_composite(NM_NET_FINE, h->raw_f, emit_f, t_f, S, o.rgb, o.depth, o.depth_raw, o.acc, o.disp, o.weights, o.mask_weights);
}

NmRenderOut offset_out(const NmRenderOut& o, long long r0, int S, int Nc) {
  NmRenderOut q = o;
  q.rgb = off(o.rgb, 3 * r0); q.depth = off(o.depth, r0); q.depth_raw = off(o.depth_raw, r0); q.acc = off(o.acc, r0);
  q.disp = off(o.disp, r0); q.weights = off(o.weights, r0 * S); q.mask_weights = off(o.mask_weights, r0 * S);
  q.t_vals = off(o.t_vals, r0 * S); q.coarse_rgb = off(o.coarse_rgb, 3 * r0); q.coarse_acc = off(o.coarse_acc, r0);
  q.coarse_disp = off(o.coarse_disp, r0); q.coarse_weights = off(o.coarse_weights, r0 * Nc);
  return q;
}

int out_samples(NmHandle h, int flags) {
  const bool buff = flags & NM_FLAG_BUFF;
  return h->cfg.num_coarse + ((h->has_fine && !buff) ? h->cfg.num_fine : 0);
}

int render_rays_impl(NmHandle h, const float* origins, int o_stride, const float* dirs, long long R, const float* nf_host,
                     const float* near_dev, const float* far_dev, int flags, uint64_t seed, const NmRenderOut& out,
                     cudaStream_t st) {
  NM_CHECK(o_stride == 0 || o_stride == 3, "o_stride must be 0 or 3");
  NM_CHECK(dirs && origins, "null ray pointers");
  NM_CHECK((near_dev == nullptr) == (far_dev == nullptr), "near_dev / far_dev must be given together");
  NM_CHECK(near_dev || nf_host, "no near/far bounds given");
  NM_CHECK(h->s_table.p != nullptr, "sampler tables missing");
  if (int e = check_train_skip(h, flags)) return e;
  const int S = out_samples(h, flags);
  const long long kChunk = chunk_rays();
  double committed = 0;
  TrainSkip ts[2];                   // a forward-only training render: nothing is kept for a backward
  ts[0].committed = ts[1].committed = &committed;
  TrainSkip* tsk = (flags & NM_FLAG_SKIP_EMPTY_TRAIN) ? ts : nullptr;
  for (long long r0 = 0; r0 < R; r0 += kChunk) {
    RayBatch rb{};
    rb.R = (R - r0 < kChunk) ? R - r0 : kChunk;
    rb.origins = origins + (long long)o_stride * r0; rb.o_stride = o_stride; rb.dirs = dirs + 3 * r0;
    if (nf_host) { rb.nf[0] = nf_host[0]; rb.nf[1] = nf_host[1]; }
    rb.near_dev = near_dev ? near_dev + r0 : nullptr; rb.far_dev = far_dev ? far_dev + r0 : nullptr;
    if (int e = render_chunk(h, rb, flags, seed + (uint64_t)r0, offset_out(out, r0, S, h->cfg.num_coarse), st, nullptr, nullptr,
                             false, tsk)) return e;
  }
  return 0;
}

// host-buffer calls: a device-side NmRenderOut whose non-null fields mirror the caller's host block
int stage_outputs(NmHandle h, const NmRenderOut& host, long long R, int S, int Nc, NmRenderOut* dev, size_t sizes[12]) {
  float* const* hp = reinterpret_cast<float* const*>(&host);
  float** dp = reinterpret_cast<float**>(dev);
  const size_t per[12] = {3, 1, 1, 1, 1, (size_t)S, (size_t)S, (size_t)S, 3, 1, 1, (size_t)Nc};
  for (int i = 0; i < 12; ++i) {
    sizes[i] = (size_t)R * per[i] * sizeof(float);
    if (hp[i]) { if (int e = h->stage_out[i].ensure(sizes[i])) return e; dp[i] = h->stage_out[i].as<float>(); }
    else dp[i] = nullptr;
  }
  return 0;
}

int copy_outputs(const NmRenderOut& host, const NmRenderOut& dev, const size_t sizes[12], cudaStream_t st) {
  float* const* hp = reinterpret_cast<float* const*>(&host);
  float* const* dp = reinterpret_cast<float* const*>(&dev);
  for (int i = 0; i < 12; ++i)
    if (hp[i]) NM_CUDA(cudaMemcpyAsync(hp[i], dp[i], sizes[i], cudaMemcpyDeviceToHost, st));
  return 0;
}

// ---------------------------------------------------------------------------------------------- training backward
int ensure_grads(NmHandle h, cudaStream_t st, bool zero) {
  for (int w = 0; w < 2; ++w) {
    const NetDev& net = h->nets[w];
    if (!net.loaded) continue;
    size_t go[kMaxLayers]; int gl[kMaxLayers];
    const size_t nb[3] = {grad_layout(net.full, go, gl) * 4, (size_t)net.full.n_bias * 4, (size_t)(net.full.n_head > 0 ? net.full.n_head : 1) * 4};
    Buf* bufs[3] = {&h->g_wt[w], &h->g_bias[w], &h->g_head[w]};
    for (int i = 0; i < 3; ++i) {
      const bool fresh = bufs[i]->p == nullptr || bufs[i]->cap < nb[i];
      if (int e = bufs[i]->ensure(nb[i])) return e;
      if (fresh || zero) NM_CUDA(cudaMemsetAsync(bufs[i]->p, 0, bufs[i]->cap, st));
    }
  }
  h->grads_ready = true;
  return 0;
}

// sub-chunks of the network backward's walk: `waves` full waves of 128-point row blocks (one per SM) bound the activation
// workspace (~20 KB per point)
long long train_walk_points(NmHandle h) {
  static const int waves = [] { const char* e = getenv("NM_TRAIN_WAVES"); int v = e ? atoi(e) : 0; return v > 0 ? v : 16; }();
  return (long long)h->num_sms * 128 * waves;
}

// The backward of one skipping training pass (NM_FLAG_SKIP_EMPTY_TRAIN, DESIGN §4.15): the compositor adjoint over the
// whole (R,s) buffer stores the rows of the evaluated samples only, compacted in index-list order, and the network
// backward runs over the staged points and directions — on the operands the forward emitted, or in ranges of the staged
// list with a recompute each.  A pass with no evaluated sample launches nothing: every skipped row is zero (alpha = 0
// and a closed relu gate), so it adds nothing to any gradient.
int train_skip_backward(NmHandle h, const RayBatch& rb, const float* raw, const float* t, int s, const float* d_rgb, uint64_t seed,
                        int which, const TrainSkip& T, cudaStream_t st) {
  const NmRenderCfg& c = h->cfg;
  if (T.M == 0) return 0;
  const bool use_tc = c.precision != NM_PREC_FP32;
  if (int e = h->dout.ensure((size_t)T.M * 16)) return e;
  if (int e = h->trans.ensure((size_t)rb.R * s * 4)) return e;
  if (int e = launch_composite_backward(raw, t, rb.dirs, d_rgb, rb.R, s, c.noise_std, seed, c.white_background,
                                        h->trans.as<float>(), h->dout.as<float>(), st, &h->launches, T.pos)) return e;
  NetGrads g{h->g_wt[which].as<float>(), h->g_bias[which].as<float>(), h->g_head[which].as<float>()};
  TrainMode md{use_tc ? 1 : 0, c.precision == NM_PREC_FAST ? 1 : 3, h->d_err};
  MlpInput in{};
  in.mode = IN_POINTS;
  if (T.ws) {
    in.pts = T.pts; in.dirs = T.dirs; in.M = T.M;
    return mlp_backward(h->nets[which], in, h->dout.as<float>(), T.ws, &g, h->num_sms, md, st, &h->launches, 1);
  }
  long long sub = train_walk_points(h);
  if (sub > T.M) sub = T.M;
  if (int e = h->train_ws.ensure(train_ws_bytes(h->nets[which].full, sub, use_tc) + 1024)) return e;
  float* ws = reinterpret_cast<float*>(((uintptr_t)h->train_ws.p + 1023) & ~(uintptr_t)1023);
  for (long long j0 = 0; j0 < T.M; j0 += sub) {
    in.pts = T.pts + 3 * j0; in.dirs = T.dirs + 3 * j0; in.M = (T.M - j0 < sub) ? T.M - j0 : sub;
    if (int e = mlp_backward(h->nets[which], in, h->dout.as<float>() + 4 * j0, ws, &g, h->num_sms, md, st, &h->launches)) return e;
  }
  return 0;
}

// One chunk of rays: forward (fills the per-sample workspaces), then for each bundle that carries a gradient the
// compositor adjoint and the network backward over sub-chunks of points.
int train_chunk(NmHandle h, const RayBatch& rb, int flags, uint64_t seed, const float* d_rgb, const float* d_rgb_coarse,
                const float* target, long long R_total, float* loss_dev, cudaStream_t st) {
  const NmRenderCfg& c = h->cfg;
  const long long R = rb.R;
  const bool buff = flags & NM_FLAG_BUFF;
  const bool two = h->has_fine && !buff && c.num_fine > 0;
  const int Nc = c.num_coarse, S = Nc + (two ? c.num_fine : 0);
  NmRenderOut o{};
  if (int e = h->tr_rgb[0].ensure((size_t)R * 12)) return e;
  o.rgb = h->tr_rgb[0].as<float>();
  if (two) { if (int e = h->tr_rgb[1].ensure((size_t)R * 12)) return e; o.coarse_rgb = h->tr_rgb[1].as<float>(); }
  // Direct mode: when the backward's workspace for ALL points of the chunk fits the budget (NM_TRAIN_DIRECT_GB, default 48),
  // the training forward itself emits the masks / activation packs and the backward skips its recompute launch; larger
  // chunks are walked in sub-chunks with a recompute each (below).
  const bool use_tc = c.precision != NM_PREC_FP32;
  const char* dg_env = getenv("NM_TRAIN_DIRECT_GB");      // read per call: the tests flip it to cover both walks
  const double direct_gb = dg_env ? atof(dg_env) : 48.0;
  const size_t ws_main = use_tc && c.act_scale_log2 == 0 ? train_ws_bytes(h->nets[two ? NM_NET_FINE : NM_NET_COARSE].full, R * S, true) + 1024 : 0;
  const size_t ws_coarse = (ws_main && two) ? train_ws_bytes(h->nets[NM_NET_COARSE].full, R * Nc, true) + 1024 : 0;
  // Skipping (NM_FLAG_SKIP_EMPTY_TRAIN): each pass decides from its evaluated count M, known only after its compaction,
  // whether its operands are emitted (inside render_chunk, against the same budget); the dense sizing below is not used.
  const bool tskip = flags & NM_FLAG_SKIP_EMPTY_TRAIN;
  const bool direct = !tskip && ws_main > 0 && (double)(ws_main + ws_coarse) <= direct_gb * 1e9 && (d_rgb || target) &&
                      (!two || d_rgb_coarse || target);
  float *ws_m = nullptr, *ws_c = nullptr;
  MlpEmit em_main{}, em_coarse{};
  double committed = 0;
  TrainSkip ts[2];                 // [0] coarse (or only) pass, [1] fine pass
  for (int k = 0; k < 2; ++k) {
    const bool grad = target || ((two && k == 0) ? d_rgb_coarse : d_rgb);
    ts[k].emit = use_tc && c.act_scale_log2 == 0 && grad;
    ts[k].budget = direct_gb * 1e9;
    ts[k].committed = &committed;
  }
  if (tskip) {
    if (int e = render_chunk(h, rb, flags, seed, o, st, nullptr, nullptr, true, ts)) return e;
  } else if (direct) {
    if (int e = h->train_ws.ensure(ws_main + ws_coarse + 2048)) return e;
    ws_m = reinterpret_cast<float*>(((uintptr_t)h->train_ws.p + 1023) & ~(uintptr_t)1023);
    train_emit_setup(h->nets[two ? NM_NET_FINE : NM_NET_COARSE].full, R * S, ws_m, &em_main);
    if (two) {
      ws_c = reinterpret_cast<float*>(((uintptr_t)ws_m + ws_main + 1023) & ~(uintptr_t)1023);
      train_emit_setup(h->nets[NM_NET_COARSE].full, R * Nc, ws_c, &em_coarse);
    }
    if (int e = render_chunk(h, rb, flags, seed, o, st, two ? &em_coarse : &em_main, two ? &em_main : nullptr, true)) return e;
  } else {
    if (int e = render_chunk(h, rb, flags, seed, o, st, nullptr, nullptr, true)) return e;
  }
  if (target) {
    for (int i = 0; i < (two ? 2 : 1); ++i) {
      if (int e = h->tr_drgb[i].ensure((size_t)R * 12)) return e;
      // loss_dev[0] = coarse (or only) bundle, loss_dev[1] = fine bundle — the two terms of model_nerf.py:118-126
      float* slot = loss_dev ? loss_dev + ((two && i == 0) ? 1 : 0) : nullptr;
      if (int e = launch_mse_grad(h->tr_rgb[i].as<float>(), target, 3 * R, 3 * R_total, h->tr_drgb[i].as<float>(), slot, st, &h->launches)) return e;
    }
    d_rgb = h->tr_drgb[0].as<float>();
    d_rgb_coarse = two ? h->tr_drgb[1].as<float>() : nullptr;
  }
  struct Pass { int which; const float* raw; const float* t; int s; const float* g; uint64_t salt; };
  Pass passes[2];
  int np = 0;
  if (two) {
    if (d_rgb) passes[np++] = {NM_NET_FINE, h->raw_f.as<float>(), h->t_f.as<float>(), S, d_rgb, kNoiseSaltMain};
    if (d_rgb_coarse) passes[np++] = {NM_NET_COARSE, h->raw_c.as<float>(), h->t_c.as<float>(), Nc, d_rgb_coarse, kNoiseSaltCoarse};
  } else if (d_rgb) {
    passes[np++] = {NM_NET_COARSE, h->raw_c.as<float>(), buff ? h->t_u.as<float>() : h->t_c.as<float>(), Nc, d_rgb, kNoiseSaltMain};
  }
  for (int pi = 0; pi < np; ++pi) {
    const Pass& P = passes[pi];
    NetDev& net = h->nets[P.which];
    if (tskip) {
      if (int e = train_skip_backward(h, rb, P.raw, P.t, P.s, P.g, seed ^ P.salt, P.which, ts[P.which], st)) return e;
      continue;
    }
    if (int e = h->dout.ensure((size_t)R * P.s * 16)) return e;
    if (int e = h->trans.ensure((size_t)R * P.s * 4)) return e;
    if (int e = launch_composite_backward(P.raw, P.t, rb.dirs, P.g, R, P.s, c.noise_std, seed ^ P.salt,
                                          c.white_background, h->trans.as<float>(), h->dout.as<float>(), st, &h->launches)) return e;
    NetGrads gd{h->g_wt[P.which].as<float>(), h->g_bias[P.which].as<float>(), h->g_head[P.which].as<float>()};
    TrainMode md{use_tc ? 1 : 0, c.precision == NM_PREC_FAST ? 1 : 3, h->d_err};
    if (direct) {
      MlpInput in{};
      in.mode = IN_RAYS; in.dirs = rb.dirs; in.ray_o = rb.origins; in.o_stride = rb.o_stride; in.t = P.t; in.S = P.s; in.M = R * P.s;
      float* wsp = (two && P.which == NM_NET_COARSE) ? ws_c : ws_m;
      if (int e = mlp_backward(h->nets[P.which], in, h->dout.as<float>(), wsp, &gd, h->num_sms, md, st, &h->launches, 1)) return e;
      continue;
    }
    long long rays_sub = train_walk_points(h) / P.s;
    if (rays_sub < 1) rays_sub = 1;
    if (rays_sub > R) rays_sub = R;
    if (int e = h->train_ws.ensure(train_ws_bytes(net.full, rays_sub * P.s, use_tc) + 1024)) return e;
    float* ws = reinterpret_cast<float*>(((uintptr_t)h->train_ws.p + 1023) & ~(uintptr_t)1023);
    NetGrads g{h->g_wt[P.which].as<float>(), h->g_bias[P.which].as<float>(), h->g_head[P.which].as<float>()};
    TrainMode mode{use_tc ? 1 : 0, c.precision == NM_PREC_FAST ? 1 : 3, h->d_err};
    for (long long r0 = 0; r0 < R; r0 += rays_sub) {
      const long long n = (R - r0 < rays_sub) ? R - r0 : rays_sub;
      MlpInput in{};
      in.mode = IN_RAYS; in.dirs = rb.dirs + 3 * r0; in.ray_o = rb.origins + (long long)rb.o_stride * r0;
      in.o_stride = rb.o_stride; in.t = P.t + r0 * P.s; in.S = P.s; in.M = n * P.s;
      if (int e = mlp_backward(h->nets[P.which], in, h->dout.as<float>() + r0 * P.s * 4, ws, &g, h->num_sms, mode, st, &h->launches)) return e;
    }
  }
  return 0;
}

int train_impl(NmHandle h, const float* origins, int o_stride, const float* dirs, long long R, const float* nf_host,
               const float* near_dev, const float* far_dev, int flags, uint64_t seed, const float* d_rgb,
               const float* d_rgb_coarse, const float* target, float* loss_dev, cudaStream_t st) {
  NM_CHECK(o_stride == 0 || o_stride == 3, "o_stride must be 0 or 3");
  NM_CHECK(dirs && origins, "null ray pointers");
  NM_CHECK((near_dev == nullptr) == (far_dev == nullptr), "near_dev / far_dev must be given together");
  NM_CHECK(near_dev || nf_host, "no near/far bounds given");
  if (int e = check_train_skip(h, flags)) return e;
  NM_CHECK(!(flags & NM_FLAG_TEACHER_T), "NM_FLAG_TEACHER_T is not supported by the backward pass");
  NM_CHECK(target || d_rgb || d_rgb_coarse, "no gradient source (target or d_rgb)");
  NM_CHECK(h->s_table.p != nullptr, "sampler tables missing");
  if (!h->grads_ready) if (int e = ensure_grads(h, st, true)) return e;
  if (int e = ensure_grads(h, st, false)) return e;
  const long long kChunk = chunk_rays();
  for (long long r0 = 0; r0 < R; r0 += kChunk) {
    RayBatch rb{};
    rb.R = (R - r0 < kChunk) ? R - r0 : kChunk;
    rb.origins = origins + (long long)o_stride * r0; rb.o_stride = o_stride; rb.dirs = dirs + 3 * r0;
    if (nf_host) { rb.nf[0] = nf_host[0]; rb.nf[1] = nf_host[1]; }
    rb.near_dev = near_dev ? near_dev + r0 : nullptr; rb.far_dev = far_dev ? far_dev + r0 : nullptr;
    if (int e = train_chunk(h, rb, flags, seed + (uint64_t)r0, d_rgb ? d_rgb + 3 * r0 : nullptr,
                            d_rgb_coarse ? d_rgb_coarse + 3 * r0 : nullptr, target ? target + 3 * r0 : nullptr, R,
                            loss_dev, st)) return e;
  }
  return 0;
}

}  // namespace

extern "C" {

int nm_version(void) { return NM_VERSION; }
const char* nm_last_error(void) { return nm::last_error(); }

int nm_device_check(int device) {
  int n = 0;
  NM_CUDA(cudaGetDeviceCount(&n));
  NM_CHECK(device >= 0 && device < n, "device %d out of range (%d visible)", device, n);
  cudaDeviceProp p;
  NM_CUDA(cudaGetDeviceProperties(&p, device));
  NM_CHECK(p.major == 9 && p.minor == 0, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, p.major, p.minor);
  return 0;
}

int nm_create(int device, const NmNetDesc* coarse, const NmNetDesc* fine, const NmRenderCfg* cfg, NmHandle* out) {
  NM_CHECK(coarse && cfg && out, "null argument");
  if (int e = nm_device_check(device)) return e;
  NetProgram a, b;
  if (int e = build_programs(*coarse, &a, &b)) return e;
  if (fine) if (int e = build_programs(*fine, &a, &b)) return e;
  NM_CUDA(cudaSetDevice(device));
  NmHandle h = new NmHandle_t();
  h->device = device;
  h->desc[0] = *coarse;
  h->has_fine = fine != nullptr;
  if (fine) h->desc[1] = *fine;
  auto init = [&]() -> int {
    cudaDeviceProp p;
    NM_CUDA(cudaGetDeviceProperties(&p, device));
    h->num_sms = p.multiProcessorCount;
    NM_CUDA(cudaHostAlloc(&h->h_err, 3 * sizeof(int), cudaHostAllocMapped));
    h->h_err[0] = h->h_err[1] = h->h_err[2] = 0;
    NM_CUDA(cudaHostGetDevicePointer(&h->d_err, h->h_err, 0));
    NM_CUDA(cudaMalloc(&h->d_stats, 4 * sizeof(double)));
    NM_CUDA(cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking));
    if (int e = nm_set_render_cfg(h, cfg)) return e;
    return nm_set_tables(h, nullptr, nullptr);
  };
  if (int e = init()) { nm_destroy(h); *out = nullptr; return e; }
  *out = h;
  return 0;
}

int nm_destroy(NmHandle h) {
  if (!h) return 0;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  free_network(&h->nets[0]); free_network(&h->nets[1]);
  Buf* bufs[] = {&h->s_table, &h->u_table, &h->voxels, &h->t_c, &h->raw_c, &h->w_c, &h->t_f, &h->raw_f, &h->t_u,
                 &h->dirs, &h->origins, &h->lin[0], &h->lin[1], &h->lin[2], &h->small};
  for (Buf* b : bufs) b->release();
  for (Buf& b : h->stage_in) b.release();
  for (Buf& b : h->stage_out) b.release();
  for (int i = 0; i < 2; ++i) { h->g_wt[i].release(); h->g_bias[i].release(); h->g_head[i].release(); h->tr_rgb[i].release(); h->tr_drgb[i].release(); }
  h->train_ws.release(); h->dout.release(); h->trans.release();
  h->ss_tab.release(); h->ss_ws.release(); h->ms_ws.release(); h->nn_ws.release(); h->sg_ws.release();
  h->cc_ws.release(); h->dc_ws.release(); h->sp_ws.release(); h->tx_ws.release(); h->rs_ws.release(); h->sf_ws.release(); h->oc_ws.release(); h->sk_ws.release();
  for (int i = 0; i < 2; ++i) { h->ts_ws[i].release(); h->ts_pts[i].release(); }
  h->train_ws_c.release();
  h->occ[0].bits.release(); h->occ[1].bits.release(); h->mc_ws.release(); h->mc_ws2.release();
  if (h->h_err) cudaFreeHost(h->h_err);
  cudaFree(h->d_stats);
  for (cudaEvent_t e : h->ev) cudaEventDestroy(e);
  if (h->own_stream) cudaStreamDestroy(h->own_stream);
  delete h;
  return 0;
}

int nm_set_render_cfg(NmHandle h, const NmRenderCfg* cfg) {
  NM_CHECK(h && cfg, "null argument");
  NM_CHECK(cfg->num_coarse >= 3 && cfg->num_coarse <= 256, "num_coarse %d outside [3,256]", cfg->num_coarse);
  NM_CHECK(cfg->num_fine >= 0 && cfg->num_coarse + cfg->num_fine <= 512, "num_coarse+num_fine exceeds 512");
  NM_CHECK(cfg->precision >= NM_PREC_EXACT && cfg->precision <= NM_PREC_FP32, "unknown precision %d", cfg->precision);
  NM_CHECK(cfg->act_scale_log2 >= 0 && cfg->act_scale_log2 <= 12, "act_scale_log2 outside [0,12]");
  const bool resize = cfg->num_coarse != h->cfg.num_coarse || cfg->num_fine != h->cfg.num_fine;
  h->cfg = *cfg;
  if (resize && h->s_table.p) return nm_set_tables(h, nullptr, nullptr);
  return 0;
}

int nm_load_weights(NmHandle h, int which, int n_tensors, const char* const* names, const float* const* tensors_host,
                    const int64_t* numel) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(which == NM_NET_COARSE || (which == NM_NET_FINE && h->has_fine), "network slot %d not present", which);
  WeightSource src;
  src.n = n_tensors; src.names = names; src.ptrs = tensors_host; src.numel = numel;
  h->occ[which].stale = true;      // a grid describes the weights it was built from: inference refuses it from now on
  return pack_network(h->desc[which], src, &h->nets[which]);
}

int nm_load_weights_dev(NmHandle h, int which, int n_tensors, const char* const* names, const float* const* tensors_dev,
                        const int64_t* numel, void* stream) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(which == NM_NET_COARSE || (which == NM_NET_FINE && h->has_fine), "network slot %d not present", which);
  WeightSource src;
  src.n = n_tensors; src.names = names; src.ptrs = tensors_dev; src.numel = numel;
  h->occ[which].stale = true;      // a grid describes the weights it was built from: inference refuses it from now on
  return load_network_dev(h->desc[which], src, &h->nets[which], (cudaStream_t)stream, &h->launches);
}

int nm_set_tables(NmHandle h, const float* coarse_s_host, const float* fine_u_host) {
  if (int e = bind_device(h)) return e;
  std::vector<float> tmp;
  if (!coarse_s_host) { linspace_host(h->cfg.num_coarse, &tmp); coarse_s_host = tmp.data(); }
  if (int e = upload(&h->s_table, coarse_s_host, sizeof(float) * h->cfg.num_coarse)) return e;
  if (h->cfg.num_fine > 0) {
    std::vector<float> tmp2;
    if (!fine_u_host) { linspace_host(h->cfg.num_fine, &tmp2); fine_u_host = tmp2.data(); }
    if (int e = upload(&h->u_table, fine_u_host, sizeof(float) * h->cfg.num_fine)) return e;
  }
  return 0;
}

int nm_set_tree(NmHandle h, const float* voxels_host, int32_t V) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(voxels_host && V > 0, "empty voxel list");
  h->V = V;
  return upload(&h->voxels, voxels_host, sizeof(float) * 6 * (size_t)V);
}

int nm_point_mlp(NmHandle h, int which, const float* pts_dev, const float* dirs_dev, int64_t M, float* out_dev,
                 int sigma_only, void* stream) {
  if (int e = bind_checked(h)) return e;
  NM_CHECK(which == NM_NET_COARSE || (which == NM_NET_FINE && h->has_fine), "network slot %d not present", which);
  NM_CHECK(pts_dev && out_dev && M >= 0, "bad arguments");
  MlpInput in{};
  in.mode = IN_POINTS; in.pts = pts_dev; in.dirs = dirs_dev; in.M = M;
  return run_mlp(h, which, sigma_only != 0, in, out_dev, (cudaStream_t)stream);
}

int nm_render_rays(NmHandle h, const float* origins_dev, int o_stride, const float* dirs_dev, int64_t R,
                   const float* near_far_host, const float* near_dev, const float* far_dev, int flags, uint64_t seed,
                   const NmRenderOut* out_dev, void* stream) {
  if (int e = bind_checked(h)) return e;
  NM_CHECK(out_dev, "null output block");
  return render_rays_impl(h, origins_dev, o_stride, dirs_dev, R, near_far_host, near_dev, far_dev, flags, seed, *out_dev,
                          (cudaStream_t)stream);
}

int nm_ray_bundle(NmHandle h, const float* pose_host, int H, int W, double focal, int ndc, double ndc_near, int row0,
                  int row1, float* origins_dev, float* dirs_dev, void* stream) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(pose_host && dirs_dev, "null argument");
  NM_CHECK(0 <= row0 && row0 <= row1 && row1 <= H && W > 0, "bad row range");
  NM_CHECK(!ndc || origins_dev, "ndc rays need an origins buffer");
  RayGenArgs a{};
  memcpy(a.pose, pose_host, sizeof(a.pose));
  a.H = H; a.W = W; a.focal = focal; a.ndc = ndc; a.ndc_near = ndc_near; a.row0 = row0; a.row1 = row1;
  return launch_raygen(a, origins_dev, dirs_dev, (cudaStream_t)stream, &h->launches);
}

int nm_render_image(NmHandle h, const float* pose_host, int H, int W, double focal, int ndc, int row0, int row1,
                    const float* near_far_host, int flags, uint64_t seed, const NmRenderOut* out_dev, void* stream) {
  if (int e = bind_checked(h)) return e;
  NM_CHECK(out_dev && pose_host && near_far_host, "null argument");
  NM_CHECK(0 <= row0 && row0 <= row1 && row1 <= H && W > 0, "bad row range");
  NM_CHECK(!(flags & NM_FLAG_SKIP_EMPTY_TRAIN), "NM_FLAG_SKIP_EMPTY_TRAIN is taken by nm_render_rays, nm_backward_rays and nm_loss_backward");
  const long long R = (long long)(row1 - row0) * W;
  cudaStream_t st = (cudaStream_t)stream;
  if (int e = h->dirs.ensure((size_t)R * 12)) return e;
  float* origins = nullptr;
  int o_stride = 0;
  if (ndc) {
    if (int e = h->origins.ensure((size_t)R * 12)) return e;
    origins = h->origins.as<float>();
    o_stride = 3;
  }
  if (int e = nm_ray_bundle(h, pose_host, H, W, focal, ndc, 1.0, row0, row1, origins, h->dirs.as<float>(), stream)) return e;
  if (!ndc) {
    if (int e = h->small.ensure(64)) return e;
    const float o3[3] = {pose_host[3], pose_host[7], pose_host[11]};
    NM_CUDA(cudaMemcpyAsync(h->small.p, o3, sizeof(o3), cudaMemcpyHostToDevice, st));
    origins = h->small.as<float>();
  }
  return render_rays_impl(h, origins, o_stride, h->dirs.as<float>(), R, near_far_host, nullptr, nullptr, flags, seed,
                          *out_dev, st);
}

// ---------------------------------------------------------------------------------------------- training entry points
int nm_zero_grad(NmHandle h, void* stream) {
  if (int e = bind_device(h)) return e;
  return ensure_grads(h, (cudaStream_t)stream, true);
}

int nm_backward_rays(NmHandle h, const float* origins_dev, int o_stride, const float* dirs_dev, int64_t R,
                     const float* near_far_host, const float* near_dev, const float* far_dev, int flags, uint64_t seed,
                     const float* d_rgb_dev, const float* d_coarse_rgb_dev, void* stream) {
  if (int e = bind_checked(h)) return e;
  return train_impl(h, origins_dev, o_stride, dirs_dev, R, near_far_host, near_dev, far_dev, flags, seed, d_rgb_dev,
                    d_coarse_rgb_dev, nullptr, nullptr, (cudaStream_t)stream);
}

int nm_loss_backward(NmHandle h, const float* origins_dev, int o_stride, const float* dirs_dev, int64_t R,
                     const float* near_far_host, const float* near_dev, const float* far_dev, int flags, uint64_t seed,
                     const float* target_rgb_dev, float* loss_dev, void* stream) {
  if (int e = bind_checked(h)) return e;
  NM_CHECK(target_rgb_dev, "null target");
  return train_impl(h, origins_dev, o_stride, dirs_dev, R, near_far_host, near_dev, far_dev, flags, seed, nullptr, nullptr,
                    target_rgb_dev, loss_dev, (cudaStream_t)stream);
}

int nm_get_grad(NmHandle h, int which, const char* name, float* out_dev, int64_t numel, void* stream) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(which == NM_NET_COARSE || (which == NM_NET_FINE && h->has_fine), "network slot %d not present", which);
  NM_CHECK(name && out_dev, "null argument");
  const NetDev& net = h->nets[which];
  NM_CHECK(net.loaded && h->grads_ready && h->g_wt[which].p, "no gradients accumulated for network %d", which);
  cudaStream_t st = (cudaStream_t)stream;
  for (int l = 0; l < net.full.n_layers; ++l) {
    const LayerProg& L = net.full.layers[l];
    const int K = L.k_act + L.k_pe, N = L.n_out;
    const int heads = L.kind == KIND_SIGMA ? 1 : (L.kind == KIND_RGB ? 3 : (L.kind == KIND_OUT4 ? 4 : 0));
    const std::string* nm4 = &net.names[4 * l];
    if (nm4[0] == name) {
      NM_CHECK(numel == (int64_t)K * N, "'%s' has %lld elements, expected %lld", name, (long long)numel, (long long)K * N);
      size_t go[kMaxLayers]; int gl[kMaxLayers];
      grad_layout(net.full, go, gl);
      NM_CUDA(cudaMemcpy2DAsync(out_dev, (size_t)K * 4, h->g_wt[which].as<float>() + go[l], (size_t)gl[l] * 4, (size_t)K * 4, N,
                                cudaMemcpyDeviceToDevice, st));
      return 0;
    }
    const float* src = nullptr;
    int64_t n = 0;
    if (nm4[1] == name) { src = h->g_bias[which].as<float>() + L.bias_off; n = N; }
    else if (heads && nm4[2] == name) { src = h->g_head[which].as<float>() + L.head_off; n = (int64_t)heads * N; }
    else if (heads && nm4[3] == name) { src = h->g_head[which].as<float>() + L.head_off + heads * N; n = heads; }
    if (src) {
      NM_CHECK(numel == n, "'%s' has %lld elements, expected %lld", name, (long long)numel, (long long)n);
      NM_CUDA(cudaMemcpyAsync(out_dev, src, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
      return 0;
    }
  }
  NM_CHECK(false, "no parameter named '%s'", name);
  return -1;
}

int nm_debug_gemm(NmHandle h, const float* a_dev, const float* b_dev, int M, int N, int K, int n_passes, float* d_dev,
                  void* stream) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(a_dev && b_dev && d_dev && M > 0 && N > 0 && K > 0, "bad arguments");
  NM_CHECK(n_passes == 1 || n_passes == 3, "n_passes must be 1 or 3");
  const size_t need = pack_bytes(M, K) + pack_bytes(N, K);
  if (int e = h->train_ws.ensure(need + 1024)) return e;
  uint8_t* ws = reinterpret_cast<uint8_t*>(((uintptr_t)h->train_ws.p + 1023) & ~(uintptr_t)1023);
  return debug_tc_gemm(a_dev, b_dev, M, N, K, n_passes, d_dev, ws, need, h->num_sms, h->d_err, (cudaStream_t)stream,
                       &h->launches);
}

int nm_debug_mlp_backward(NmHandle h, int which, const float* pts_dev, const float* dirs_dev, int64_t M, const float* dout_dev,
                          void* stream) {
  if (int e = bind_checked(h)) return e;
  NM_CHECK(which == NM_NET_COARSE || (which == NM_NET_FINE && h->has_fine), "network slot %d not present", which);
  NM_CHECK(pts_dev && dout_dev && M > 0 && M <= INT32_MAX, "bad arguments");
  NM_CHECK((reinterpret_cast<uintptr_t>(dout_dev) & 15) == 0, "dout must be 16-byte aligned (M,4) rows");
  NetDev& net = h->nets[which];
  NM_CHECK(net.loaded, "weights of network %d not loaded", which);
  cudaStream_t st = (cudaStream_t)stream;
  if (!h->grads_ready) if (int e = ensure_grads(h, st, true)) return e;
  if (int e = ensure_grads(h, st, false)) return e;
  const bool use_tc = h->cfg.precision != NM_PREC_FP32;
  if (int e = h->train_ws.ensure(train_ws_bytes(net.full, M, use_tc) + 1024)) return e;
  float* ws = reinterpret_cast<float*>(((uintptr_t)h->train_ws.p + 1023) & ~(uintptr_t)1023);
  MlpInput in{};
  in.mode = IN_POINTS; in.pts = pts_dev; in.dirs = dirs_dev; in.M = M;
  NetGrads g{h->g_wt[which].as<float>(), h->g_bias[which].as<float>(), h->g_head[which].as<float>()};
  TrainMode mode{use_tc ? 1 : 0, h->cfg.precision == NM_PREC_FAST ? 1 : 3, h->d_err};
  return mlp_backward(net, in, dout_dev, ws, &g, h->num_sms, mode, st, &h->launches, 0);
}

int nm_debug_composite_backward(NmHandle h, const float* raw_dev, const float* t_dev, const float* dirs_dev,
                                const float* d_rgb_dev, int64_t R, int S, float noise_std, uint64_t seed, int white_bg,
                                float* dout_dev, void* stream) {
  if (int e = bind_checked(h)) return e;
  NM_CHECK(raw_dev && t_dev && dirs_dev && d_rgb_dev && dout_dev, "null pointer argument");
  NM_CHECK(R >= 0, "negative ray count %lld", (long long)R);
  NM_CHECK(S >= 1 && S <= 512, "samples per ray %d outside [1, 512] (the compositor adjoint holds 16 per lane)", S);
  NM_CHECK((reinterpret_cast<uintptr_t>(raw_dev) & 15) == 0 && (reinterpret_cast<uintptr_t>(dout_dev) & 15) == 0,
           "raw and dout must be 16-byte aligned (R,S,4) arrays");
  if (R == 0) return 0;
  // the same call as train_chunk's, with the transmittance scratch it passes
  if (int e = h->trans.ensure((size_t)R * S * 4)) return e;
  return launch_composite_backward(raw_dev, t_dev, dirs_dev, d_rgb_dev, R, S, noise_std, seed, white_bg, h->trans.as<float>(),
                                   dout_dev, (cudaStream_t)stream, &h->launches);
}

int nm_debug_composite(NmHandle h, const float* raw_dev, const float* t_dev, const float* dirs_dev, int64_t R, int S,
                       float noise_std, uint64_t seed, int white_bg, int training, float thr, const NmRenderOut* out_dev,
                       void* stream) {
  if (int e = bind_checked(h)) return e;
  NM_CHECK(raw_dev && t_dev && dirs_dev && out_dev, "null pointer argument");
  NM_CHECK(!out_dev->t_vals && !out_dev->coarse_rgb && !out_dev->coarse_acc && !out_dev->coarse_disp && !out_dev->coarse_weights,
           "the compositor writes rgb, depth, depth_raw, acc, disp, weights and mask_weights only: the other fields must be NULL");
  NM_CHECK(R >= 0, "negative ray count %lld", (long long)R);
  NM_CHECK(S >= 1 && S <= 512, "samples per ray %d outside [1, 512]", S);
  NM_CHECK((reinterpret_cast<uintptr_t>(raw_dev) & 15) == 0, "raw must be a 16-byte aligned (R,S,4) array");
  if (R == 0) return 0;
  // the CompositeArgs render_chunk's mlp_composite builds, on the caller's arrays
  CompositeArgs a{};
  a.raw = raw_dev; a.t = t_dev; a.dirs = dirs_dev; a.R = R; a.S = S; a.noise_std = noise_std; a.seed = seed;
  a.white_bg = white_bg ? 1 : 0; a.training = training ? 1 : 0; a.thr = thr;
  a.rgb = out_dev->rgb; a.depth = out_dev->depth; a.depth_raw = out_dev->depth_raw; a.acc = out_dev->acc; a.disp = out_dev->disp;
  a.weights = out_dev->weights; a.mask_weights = out_dev->mask_weights;
  return launch_composite(a, (cudaStream_t)stream, &h->launches);
}

int nm_debug_sample_pdf(NmHandle h, const float* t_c_dev, const float* w_c_dev, const float* u_dev, int64_t R, int Nc, int Nf,
                        int perturb, uint64_t seed, float* t_out_dev, void* stream) {
  if (int e = bind_checked(h)) return e;
  NM_CHECK(t_c_dev && w_c_dev && t_out_dev, "null pointer argument");
  NM_CHECK(R >= 0, "negative ray count %lld", (long long)R);
  NM_CHECK(Nc >= 3 && Nc <= 256, "coarse samples per ray %d outside [3, 256]", Nc);
  NM_CHECK(Nf >= 1 && Nc + Nf <= 512, "fine samples per ray %d outside [1, 512 - Nc]", Nf);
  NM_CHECK(perturb || u_dev, "a deterministic resample needs the u table");
  if (R == 0) return 0;
  // the same call as render_chunk's, on the caller's arrays
  return launch_invcdf(t_c_dev, w_c_dev, u_dev, Nc, Nf, R, perturb, seed, t_out_dev, (cudaStream_t)stream, &h->launches);
}

// ---------------------------------------------------------------------------------------------- BuFF tree maintenance
int nm_ray_voxel_indices(NmHandle h, const float* origins_dev, int o_stride, const float* dirs_dev, int64_t R,
                         const float* near_far_host, float* z_out_dev, int32_t* idx_out_dev, void* stream) {
  return nm_ray_voxel_indices_ex(h, origins_dev, o_stride, dirs_dev, R, near_far_host, 0, 0, z_out_dev, idx_out_dev, stream);
}

int nm_ray_voxel_indices_ex(NmHandle h, const float* origins_dev, int o_stride, const float* dirs_dev, int64_t R,
                            const float* near_far_host, int flags, uint64_t seed, float* z_out_dev, int32_t* idx_out_dev,
                            void* stream) {
  if (int e = bind_checked(h)) return e;
  NM_CHECK(origins_dev && dirs_dev && near_far_host && idx_out_dev, "null argument");
  NM_CHECK(o_stride == 0 || o_stride == 3, "o_stride must be 0 or 3");
  NM_CHECK(h->V > 0, "no voxel list (nm_set_tree)");
  cudaStream_t st = (cudaStream_t)stream;
  const int S = h->cfg.num_coarse;
  float* t_u = nullptr;
  if (z_out_dev) {     // rays without a hit fall back to the uniform samples (src/models/model_buff.py:53)
    if (int e = h->t_c.ensure((size_t)R * S * 4)) return e;
    t_u = h->t_c.as<float>();
    if (int e = launch_stratified(h->s_table.as<float>(), S, R, near_far_host, nullptr, nullptr, h->cfg.lindisp, 0, 0, t_u, st,
                                  &h->launches)) return e;
  }
  // walked in the render calls' ray chunks with their per-chunk seeds, so that a random draw repeats the render's own
  const long long kChunk = chunk_rays();
  for (long long r0 = 0; r0 < R; r0 += kChunk) {
    const long long n = (R - r0 < kChunk) ? R - r0 : kChunk;
    if (int e = launch_aabb(h->voxels.as<float>(), h->V, origins_dev + (long long)o_stride * r0, o_stride, dirs_dev + 3 * r0, n,
                            near_far_host[0], near_far_host[1], S, h->s_table.as<float>(), t_u ? t_u + r0 * S : nullptr,
                            z_out_dev ? z_out_dev + r0 * S : nullptr, idx_out_dev + r0 * S, h->d_err + 1, st, &h->launches,
                            (flags & NM_FLAG_RANDOM_VOXELS) ? 1 : 0, (seed + (uint64_t)r0) ^ kVoxelSalt)) return e;
  }
  return 0;
}

int nm_tree_integrate(NmHandle h, const int32_t* idx_dev, const float* weights_dev, const float* mask_weights_dev, int64_t n,
                      float* memm_dev, int32_t V, int32_t counter, void* stream) {
  if (int e = bind_checked(h)) return e;
  NM_CHECK(idx_dev && weights_dev && mask_weights_dev && memm_dev && V > 0 && n >= 0 && counter >= 1, "bad arguments");
  if (int e = h->small.ensure(sizeof(float) * 2 * (size_t)V + 64)) return e;
  return launch_tree_integrate(idx_dev, weights_dev, mask_weights_dev, n, memm_dev, V, counter, h->small.as<float>(),
                               (cudaStream_t)stream, &h->launches);
}

int nm_grid_sigma(NmHandle h, const float* lin0_host, const float* lin1_host, const float* lin2_host, int n0, int n1,
                  int n2, int x0, int x1, float* sigma_dev, float* rgb_dev, void* stream) {
  if (int e = bind_checked(h)) return e;
  NM_CHECK(lin0_host && lin1_host && lin2_host && sigma_dev, "null argument");
  NM_CHECK(0 <= x0 && x0 <= x1 && x1 <= n0 && n1 > 0 && n2 > 0, "bad slab range");
  const int which = h->has_fine ? NM_NET_FINE : NM_NET_COARSE;     // BaseModel.get_model(): finest net
  const float* hs[3] = {lin0_host, lin1_host, lin2_host};
  const int ns[3] = {n0, n1, n2};
  for (int i = 0; i < 3; ++i) { if (int e = upload(&h->lin[i], hs[i], sizeof(float) * ns[i])) return e; h->lin_n[i] = ns[i]; }
  cudaStream_t st = (cudaStream_t)stream;
  MlpInput in{};
  in.mode = IN_GRID;
  in.lin0 = h->lin[0].as<float>(); in.lin1 = h->lin[1].as<float>(); in.lin2 = h->lin[2].as<float>();
  in.n1 = n1; in.n2 = n2;
  in.grid_base = (long long)x0 * n1 * n2;
  in.M = (long long)(x1 - x0) * n1 * n2;
  if (!rgb_dev) return run_mlp(h, which, true, in, sigma_dev, st);
  // reference-faithful rgb+sigma: run the full net into a scratch (M,4) and split
  if (int e = h->raw_f.ensure((size_t)in.M * 16)) return e;
  if (int e = run_mlp(h, which, false, in, h->raw_f.as<float>(), st)) return e;
  NM_CUDA(cudaMemcpy2DAsync(sigma_dev, 4, h->raw_f.as<float>() + 3, 16, 4, (size_t)in.M, cudaMemcpyDeviceToDevice, st));
  NM_CUDA(cudaMemcpy2DAsync(rgb_dev, 12, h->raw_f.as<float>(), 16, 12, (size_t)in.M, cudaMemcpyDeviceToDevice, st));
  return 0;
}

int nm_volume_stats(NmHandle h, const float* vol_dev, int64_t n, float* out_host) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(vol_dev && out_host, "null argument");
  return launch_volume_stats(vol_dev, n, h->d_stats, out_host, h->own_stream, &h->launches);
}

int nm_volume_stats_dev(NmHandle h, const float* vol_dev, int64_t n, int pass, const double* mean_dev, double* out_dev, void* stream) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(vol_dev && out_dev, "null argument");
  return launch_volume_stats_pass(vol_dev, n, pass, mean_dev, out_dev, (cudaStream_t)stream, &h->launches);
}

int nm_mc_count(NmHandle h, const float* vol_dev, int nb, int ny, int nz, float iso, int g_x0, int g_nx, int p_lo, int p_hi,
                int64_t* counts_host, void* stream) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(vol_dev && counts_host, "null argument");
  const McShard s{vol_dev, nb, ny, nz, iso, g_x0, g_nx, p_lo, p_hi, 0};
  if (int e = h->mc_ws.ensure(mc_ws_bytes(s))) return e;
  if (int e = mc_count(s, h->mc_ws.p, h->mc_ws.cap, counts_host, h->num_sms, (cudaStream_t)stream, &h->launches)) return e;
  h->mc_counts[0] = counts_host[0]; h->mc_counts[1] = counts_host[1];
  return 0;
}

int nm_mc_emit(NmHandle h, const float* vol_dev, int nb, int ny, int nz, float iso, int g_x0, int g_nx, int p_lo, int p_hi,
               int64_t v_base, float* verts_dev, float* normals_dev, int32_t* faces_dev, void* stream) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(vol_dev && verts_dev && faces_dev && h->mc_ws.p, "bad arguments (call nm_mc_count first)");
  const McShard s{vol_dev, nb, ny, nz, iso, g_x0, g_nx, p_lo, p_hi, 0};
  if (int e = h->mc_ws2.ensure(mc_emit_ws_bytes(h->mc_counts[0], h->mc_counts[1]))) return e;
  return mc_emit(s, h->mc_ws.p, h->mc_ws.cap, h->mc_ws2.p, v_base, h->mc_counts[0], h->mc_counts[1], verts_dev, normals_dev,
                 faces_dev, (cudaStream_t)stream, &h->launches);
}

int nm_mc_emit_ss(NmHandle h, const float* vol_dev, int nb, int ny, int nz, float iso, int g_x0, int g_nx, int p_lo, int p_hi,
                  int64_t v_base, int s, const float* lin0_host, const float* lin1_host, const float* lin2_host,
                  const float* fine0_host, const float* fine1_host, const float* fine2_host, float* verts_dev, float* normals_dev,
                  int32_t* faces_dev, void* stream) {
  if (int e = bind_checked(h)) return e;
  NM_CHECK(s >= 0 && s <= kMcMaxSuperSampling, "super-sampling factor %d outside [0, %d]", s, kMcMaxSuperSampling);
  NM_CHECK(lin0_host && lin1_host && lin2_host && fine0_host && fine1_host && fine2_host, "null coordinate table");
  NM_CHECK(vol_dev && verts_dev && faces_dev && h->mc_ws.p, "bad arguments (call nm_mc_count first)");
  NM_CHECK(ny >= 2 && nz >= 2 && g_nx >= 2, "marching cubes: bad volume shape");
  const int64_t nv = h->mc_counts[0], nt = h->mc_counts[1];
  const McShard sh{vol_dev, nb, ny, nz, iso, g_x0, g_nx, p_lo, p_hi, 0};
  cudaStream_t st = (cudaStream_t)stream;
  McSuperSampling ss;
  ss.s = s;
  if (nv > 0) {
    // the six tables in one buffer: lin0 | lin1 | lin2 | fine0 | fine1 | fine2
    const long long n[3] = {g_nx, ny, nz};
    const float* hs[6] = {lin0_host, lin1_host, lin2_host, fine0_host, fine1_host, fine2_host};
    long long len[6], off[6], tot = 0;
    for (int a = 0; a < 6; ++a) {
      len[a] = a < 3 ? n[a] : (n[a - 3] - 1) * (s + 1) + 1;
      off[a] = tot;
      tot += len[a];
    }
    if (int e = h->ss_tab.ensure((size_t)tot * 4)) return e;
    for (int a = 0; a < 6; ++a)
      NM_CUDA(cudaMemcpyAsync(h->ss_tab.as<float>() + off[a], hs[a], (size_t)len[a] * 4, cudaMemcpyHostToDevice, st));
    NM_CUDA(cudaStreamSynchronize(st));      // pageable sources: the copies must finish before the host arrays may change
    for (int a = 0; a < 3; ++a) { ss.lin[a] = h->ss_tab.as<float>() + off[a]; ss.fine[a] = h->ss_tab.as<float>() + off[a + 3]; }
    if (s > 0) {
      ss.chunk_points = ss_chunk_points();
      ss.chunk_vertices = ss.chunk_points >= s ? ss.chunk_points / s : 1;
      if (ss.chunk_vertices > nv) ss.chunk_vertices = nv;
      const long long m = ss.chunk_vertices * s;
      if (int e = h->ss_ws.ensure((size_t)m * 16 + 256)) return e;
      ss.pts = h->ss_ws.as<float>();
      ss.sig = reinterpret_cast<float*>(reinterpret_cast<char*>(h->ss_ws.p) + ((size_t)m * 12 + 255) / 256 * 256);
      const int which = h->has_fine ? NM_NET_FINE : NM_NET_COARSE;     // the net nm_grid_sigma sweeps
      ss.eval = [h, which, st](const float* pts, long long M, float* sigma) -> int {
        MlpInput in{};
        in.mode = IN_POINTS; in.pts = pts; in.dirs = nullptr; in.M = M;   // directions = positions, as in the grid sweep
        return run_mlp(h, which, true, in, sigma, st);
      };
    }
  }
  if (int e = h->mc_ws2.ensure(mc_emit_ws_bytes(nv, nt))) return e;
  return mc_emit_ss(sh, h->mc_ws.p, h->mc_ws.cap, h->mc_ws2.p, v_base, nv, nt, ss, verts_dev, normals_dev, faces_dev, st,
                    &h->launches);
}

// ---------------------------------------------------------------------------------------------- density gradient
// Argument checks come before the handle is touched, so a bad call is rejected without a device.  The gradient buffers and
// the training workspace are not used: the chain runs in a workspace of its own, chunk by chunk.
int nm_sigma_grad(NmHandle h, int which, const float* pts_dev, int64_t M, float* sigma_dev_or_null, float* grad_dev,
                  void* stream) {
  NM_CHECK(pts_dev && grad_dev, "density gradient: null point or gradient pointer");
  NM_CHECK(M >= 0, "density gradient: negative point count %lld", (long long)M);
  NM_CHECK(h != nullptr, "null handle");
  NM_CHECK(which == NM_NET_COARSE || (which == NM_NET_FINE && h->has_fine), "network slot %d not present", which);
  if (M == 0) return 0;
  if (int e = bind_checked(h)) return e;
  NetDev& net = h->nets[which];
  NM_CHECK(net.loaded, "weights of network %d not loaded", which);
  cudaStream_t st = (cudaStream_t)stream;
  const bool use_tc = h->cfg.precision != NM_PREC_FP32;
  const TrainMode mode{use_tc ? 1 : 0, h->cfg.precision == NM_PREC_FAST ? 1 : 3, h->d_err};
  const long long chunk = sigma_grad_chunk_points();
  const long long P = M < chunk ? M : chunk;
  // the chunk workspace is held by the handle like the training workspace: allocating and freeing it per call (stream-ordered)
  // took the 512^3 normal pass from 82 ms to 169 ms on an H100 (DESIGN 4.8)
  if (int e = h->sg_ws.ensure(sigma_grad_ws_bytes(net.full, P, use_tc) + 1024)) return e;
  float* ws = reinterpret_cast<float*>(((uintptr_t)h->sg_ws.p + 1023) & ~(uintptr_t)1023);
  for (long long m0 = 0; m0 < M; m0 += chunk) {
    const long long n = M - m0 < chunk ? M - m0 : chunk;
    if (int e = sigma_grad(net, pts_dev + 3 * m0, n, ws, grad_dev + 3 * m0, h->num_sms, mode, st, &h->launches)) return e;
  }
  if (!sigma_dev_or_null) return 0;
  // sigma: the sigma-only forward of nm_point_mlp, so that it is that call's value bit for bit
  MlpInput in{};
  in.mode = IN_POINTS; in.pts = pts_dev; in.dirs = nullptr; in.M = M;
  return run_mlp(h, which, true, in, sigma_dev_or_null, st);
}

// ---------------------------------------------------------------------------------------------- chamfer evaluation
// Argument checks come before the handle is touched, so a bad call is rejected without a device.
int nm_mesh_sample(NmHandle h, const float* verts_dev, int64_t V, const int32_t* faces_dev, int64_t F, int64_t n, uint64_t seed,
                   float* points_dev, int32_t* face_idx_dev, void* stream) {
  NM_CHECK(verts_dev && faces_dev, "mesh sampler: null mesh pointer");
  NM_CHECK(V > 0 && F > 0, "mesh sampler: empty mesh (V = %lld, F = %lld)", (long long)V, (long long)F);
  NM_CHECK(n >= 0, "mesh sampler: negative sample count %lld", (long long)n);
  NM_CHECK(V < (1ll << 31) && F < (1ll << 31) && n < (1ll << 31), "mesh sampler: sizes must be below 2^31");
  NM_CHECK(n == 0 || points_dev, "mesh sampler: null output pointer");
  NM_CHECK(h != nullptr, "null handle");
  if (n == 0) return 0;
  if (int e = bind_checked(h)) return e;
  if (int e = h->ms_ws.ensure(mesh_sample_ws_bytes(F))) return e;
  return mesh_sample(verts_dev, V, faces_dev, F, n, seed, points_dev, face_idx_dev, h->d_err + 2, h->ms_ws.p, h->ms_ws.cap,
                     (cudaStream_t)stream, &h->launches);
}

namespace {
int check_nn_args(NmHandle h, const float* q, int64_t N, const float* p, int64_t M, const void* out) {
  NM_CHECK(p, "nearest neighbour: null point pointer");
  NM_CHECK(N >= 0 && M >= 0, "nearest neighbour: negative size (N = %lld, M = %lld)", (long long)N, (long long)M);
  NM_CHECK(M > 0, "nearest neighbour: empty point set (M = 0)");
  NM_CHECK(N < (1ll << 31) && M < (1ll << 31), "nearest neighbour: sizes must be below 2^31");
  NM_CHECK(N == 0 || (q && out), "nearest neighbour: null query or output pointer");
  NM_CHECK(h != nullptr, "null handle");
  return 0;
}
}  // namespace

int nm_nearest(NmHandle h, const float* q_dev, int64_t N, const float* p_dev, int64_t M, float* dist2_dev, int32_t* idx_dev,
               void* stream) {
  if (int e = check_nn_args(h, q_dev, N, p_dev, M, dist2_dev)) return e;
  if (N == 0) return 0;
  if (int e = bind_checked(h)) return e;
  if (int e = h->nn_ws.ensure(nearest_ws_bytes(N, M, false))) return e;
  return nearest(q_dev, N, p_dev, M, dist2_dev, idx_dev, h->nn_ws.p, h->nn_ws.cap, h->num_sms, (cudaStream_t)stream,
                 &h->launches);
}

int nm_debug_nearest_brute(NmHandle h, const float* q_dev, int64_t N, const float* p_dev, int64_t M, float* dist2_dev,
                           int32_t* idx_dev, void* stream) {
  if (int e = check_nn_args(h, q_dev, N, p_dev, M, dist2_dev)) return e;
  if (N == 0) return 0;
  if (int e = bind_checked(h)) return e;
  return nearest_brute(q_dev, N, p_dev, M, dist2_dev, idx_dev, (cudaStream_t)stream, &h->launches);
}

int nm_chamfer(NmHandle h, const float* x_dev, int64_t N, const float* y_dev, int64_t M, double* means_dev, void* stream) {
  NM_CHECK(x_dev && y_dev && means_dev, "chamfer: null pointer");
  NM_CHECK(N > 0 && M > 0, "chamfer: empty point set (N = %lld, M = %lld)", (long long)N, (long long)M);
  NM_CHECK(N < (1ll << 31) && M < (1ll << 31), "chamfer: sizes must be below 2^31");
  NM_CHECK(h != nullptr, "null handle");
  if (int e = bind_checked(h)) return e;
  if (int e = h->nn_ws.ensure(nearest_ws_bytes(N, M, true))) return e;
  return chamfer(x_dev, N, y_dev, M, means_dev, h->nn_ws.p, h->nn_ws.cap, h->num_sms, (cudaStream_t)stream, &h->launches);
}

// ---------------------------------------------------------------------------------------------- small-component removal
// Argument checks come before the handle is touched, so a bad call is rejected without a device.
int nm_mesh_components(NmHandle h, const float* verts_dev, const float* normals_dev, int64_t V, const int32_t* faces_dev,
                       int64_t F, int64_t min_faces, float* verts_out_dev, float* normals_out_dev, int32_t* faces_out_dev,
                       int32_t* labels_out_dev_or_null, int64_t* counts_host, void* stream) {
  NM_CHECK(V >= 0 && F >= 0, "mesh components: negative size (V = %lld, F = %lld)", (long long)V, (long long)F);
  NM_CHECK(min_faces >= 0, "mesh components: negative min_faces %lld", (long long)min_faces);
  NM_CHECK(V < (1ll << 31) && F < (1ll << 31), "mesh components: sizes must be below 2^31");
  NM_CHECK(counts_host, "mesh components: null counts pointer");
  NM_CHECK(V == 0 || (verts_dev && normals_dev && verts_out_dev && normals_out_dev), "mesh components: null vertex pointer");
  NM_CHECK(F == 0 || (faces_dev && faces_out_dev), "mesh components: null face pointer");
  NM_CHECK(h != nullptr, "null handle");
  for (int i = 0; i < 4; ++i) counts_host[i] = 0;
  if (V == 0 && F == 0) return 0;
  if (int e = bind_checked(h)) return e;
  if (int e = h->cc_ws.ensure(components_ws_bytes(V, F))) return e;
  return mesh_components(verts_dev, normals_dev, V, faces_dev, F, min_faces, verts_out_dev, normals_out_dev, faces_out_dev,
                         labels_out_dev_or_null, counts_host, h->cc_ws.p, h->d_err + 2, (cudaStream_t)stream, &h->launches);
}

// ---------------------------------------------------------------------------------------------- quadric-error decimation
// Argument checks come before the handle is touched, so a bad call is rejected without a device.
int nm_mesh_decimate(NmHandle h, const float* verts_dev, const float* normals_dev, int64_t V, const int32_t* faces_dev, int64_t F,
                     int64_t target_faces, float* verts_out_dev, float* normals_out_dev, int32_t* faces_out_dev,
                     int32_t* source_out_dev_or_null, int64_t* counts_host, void* stream) {
  NM_CHECK(V >= 0 && F >= 0, "mesh decimate: negative size (V = %lld, F = %lld)", (long long)V, (long long)F);
  NM_CHECK(target_faces >= 0, "mesh decimate: negative target_faces %lld", (long long)target_faces);
  NM_CHECK(V < (1ll << 31) && F < (1ll << 31), "mesh decimate: sizes must be below 2^31");
  NM_CHECK(3 * F < (1ll << 31), "mesh decimate: 3F = %lld face corners must be below 2^31 (int vertex-face lists)", 3ll * F);
  NM_CHECK(counts_host, "mesh decimate: null counts pointer");
  NM_CHECK(V == 0 || (verts_dev && normals_dev && verts_out_dev && normals_out_dev), "mesh decimate: null vertex pointer");
  NM_CHECK(F == 0 || (faces_dev && faces_out_dev), "mesh decimate: null face pointer");
  NM_CHECK(h != nullptr, "null handle");
  for (int i = 0; i < 4; ++i) counts_host[i] = 0;
  if (V == 0 && F == 0) return 0;
  if (int e = bind_checked(h)) return e;
  if (int e = h->dc_ws.ensure(decimate_ws_bytes(V, F))) return e;
  return mesh_decimate(verts_dev, normals_dev, V, faces_dev, F, target_faces, verts_out_dev, normals_out_dev, faces_out_dev,
                       source_out_dev_or_null, counts_host, h->dc_ws.p, h->d_err + 2, (cudaStream_t)stream, &h->launches);
}

// ---------------------------------------------------------------------------------------------- texture bake
namespace {
// Argument checks come before the handle is touched, so a bad call is rejected without a device.
int texture_setup(NmHandle h, const float* verts, const float* normals, int64_t V, const int32_t* faces, int64_t F, int N, int mode,
                  float view_disparity, TextureBake* b, long long layout[4]) {
  NM_CHECK(V >= 0 && F >= 0, "texture bake: negative size (V = %lld, F = %lld)", (long long)V, (long long)F);
  NM_CHECK(V < (1ll << 31) && F < (1ll << 31), "texture bake: sizes must be below 2^31");
  NM_CHECK(mode == 0 || mode == 1, "texture bake: mode %d is neither 0 (rays) nor 1 (points)", mode);
  if (int e = texture_layout(F, N, layout)) return e;
  NM_CHECK(V == 0 || (verts && normals), "texture bake: null vertex pointer");
  NM_CHECK(F == 0 || faces, "texture bake: null face pointer");
  b->verts = verts; b->normals = normals; b->V = V; b->faces = faces; b->F = F; b->N = N; b->mode = mode;
  b->disparity = view_disparity;
  b->chunk_texels = texture_chunk_texels();
  return 0;
}
}  // namespace

int nm_bake_texture(NmHandle h, const float* verts_dev, const float* normals_dev, int64_t V, const int32_t* faces_dev, int64_t F,
                    int N, int mode, int which, int flags, float view_disparity, const float* near_far_host, float* atlas_f32_dev,
                    uint8_t* atlas_u8_dev, float* uv_dev, float* vertex_rgb_dev, int64_t* counts_host, void* stream) {
  TextureBake b;
  long long lay[4];
  if (int e = texture_setup(h, verts_dev, normals_dev, V, faces_dev, F, N, mode, view_disparity, &b, lay)) return e;
  NM_CHECK(counts_host, "texture bake: null counts pointer");
  NM_CHECK(V == 0 || vertex_rgb_dev, "texture bake: null vertex colour pointer");
  NM_CHECK(F == 0 || (atlas_f32_dev && atlas_u8_dev && uv_dev), "texture bake: null atlas or uv pointer");
  NM_CHECK(mode == 1 || near_far_host, "texture bake: null near/far bounds");
  NM_CHECK(!(flags & NM_FLAG_TEACHER_T), "texture bake: NM_FLAG_TEACHER_T takes caller samples, which a bake does not have");
  NM_CHECK(h != nullptr, "null handle");
  counts_host[0] = lay[2]; counts_host[1] = lay[3]; counts_host[2] = 0; counts_host[3] = 0;
  if (V == 0 && F == 0) return 0;
  if (int e = bind_checked(h)) return e;
  cudaStream_t st = (cudaStream_t)stream;
  if (mode == 0) {
    NM_CHECK(h->s_table.p != nullptr, "sampler tables missing");
    const float nf[2] = {near_far_host[0], near_far_host[1]};
    b.rgb_stride = 3;
    b.render = [h, nf, flags, st](const float* o, const float* d, long long n, float* rgb) -> int {
      NmRenderOut out{};
      out.rgb = rgb;
      return render_rays_impl(h, o, 3, d, n, nf, nullptr, nullptr, flags, 0, out, st);     // seed 0: model.query in eval mode
    };
  } else {
    NM_CHECK(which == NM_NET_COARSE || (which == NM_NET_FINE && h->has_fine), "network slot %d not present", which);
    NM_CHECK(h->nets[which].loaded, "weights of network %d not loaded", which);
    b.rgb_stride = 4;
    b.render = [h, which, st](const float* p, const float* d, long long n, float* rgb) -> int {
      MlpInput in{};
      in.mode = IN_POINTS; in.pts = p; in.dirs = d; in.M = n;
      return run_mlp(h, which, false, in, rgb, st);
    };
  }
  if (int e = h->tx_ws.ensure(texture_ws_bytes(b))) return e;
  return bake_texture(b, atlas_f32_dev, atlas_u8_dev, uv_dev, vertex_rgb_dev, counts_host, h->tx_ws.p, h->d_err + 2, h->h_err + 2,
                      st, &h->launches);
}

int nm_debug_texture_rays(NmHandle h, const float* verts_dev, const float* normals_dev, int64_t V, const int32_t* faces_dev, int64_t F,
                          int N, int mode, float view_disparity, int64_t f0, int64_t f1, float* origins_out_dev,
                          float* dirs_out_dev, int32_t* pixel_xy_out_dev, void* stream) {
  TextureBake b;
  long long lay[4];
  if (int e = texture_setup(h, verts_dev, normals_dev, V, faces_dev, F, N, mode, view_disparity, &b, lay)) return e;
  NM_CHECK(0 <= f0 && f0 <= f1 && f1 <= F, "texture bake: face range [%lld, %lld) outside [0, %lld)", (long long)f0, (long long)f1,
           (long long)F);
  NM_CHECK(f0 == f1 || (origins_out_dev && dirs_out_dev), "texture bake: null ray output pointer");
  NM_CHECK(h != nullptr, "null handle");
  if (f0 == f1) return 0;
  if (int e = bind_checked(h)) return e;
  return texture_rays(b, f0, f1, origins_out_dev, dirs_out_dev, pixel_xy_out_dev, h->d_err + 2, (cudaStream_t)stream, &h->launches);
}

// ---------------------------------------------------------------------------------------------- mesh raster
// Argument checks come before the handle is touched, so a bad call is rejected without a device.
int nm_rasterize_mesh(NmHandle h, const float* verts_dev, int64_t V, const int32_t* faces_dev, int64_t F, const float* pose_host,
                      int H, int W, float focal, float z_near, int mode, const float* vertex_rgb_dev_or_null,
                      const float* atlas_dev_or_null, int N, const float* background_host, float* rgb_out_or_null,
                      float* depth_out_or_null, int32_t* face_out_or_null, int64_t* counts_host, void* stream) {
  NM_CHECK(V >= 0 && F >= 0, "mesh raster: negative size (V = %lld, F = %lld)", (long long)V, (long long)F);
  NM_CHECK(V < (1ll << 31) && F < (1ll << 31), "mesh raster: sizes must be below 2^31");
  NM_CHECK(pose_host && background_host && counts_host, "mesh raster: null pose, background or counts pointer");
  NM_CHECK(H >= 1 && H <= 16384 && W >= 1 && W <= 16384, "mesh raster: image %d x %d outside [1, 16384]", H, W);
  NM_CHECK(focal > 0.f && std::isfinite(focal), "mesh raster: focal length %g is not positive and finite", (double)focal);
  NM_CHECK(z_near > 0.f && std::isfinite(z_near), "mesh raster: z_near %g is not positive and finite", (double)z_near);
  NM_CHECK(mode == 0 || mode == 1, "mesh raster: mode %d is neither 0 (vertex colours) nor 1 (texture atlas)", mode);
  if (mode == 1) {
    long long lay[4];
    if (int e = texture_layout(F, N, lay)) return e;
  }
  NM_CHECK(V == 0 || verts_dev, "mesh raster: null vertex pointer");
  NM_CHECK(F == 0 || faces_dev, "mesh raster: null face pointer");
  NM_CHECK(!rgb_out_or_null || mode == 1 || V == 0 || vertex_rgb_dev_or_null, "mesh raster: null vertex colour pointer");
  NM_CHECK(!rgb_out_or_null || mode == 0 || F == 0 || atlas_dev_or_null, "mesh raster: null atlas pointer");
  NM_CHECK(h != nullptr, "null handle");
  counts_host[0] = counts_host[1] = counts_host[2] = 0;
  if (int e = bind_checked(h)) return e;
  RasterMesh m;
  m.verts = verts_dev; m.V = V; m.faces = faces_dev; m.F = F;
  memcpy(m.pose, pose_host, sizeof(m.pose));
  m.H = H; m.W = W; m.focal = focal; m.z_near = z_near; m.mode = mode; m.N = N;
  m.vertex_rgb = vertex_rgb_dev_or_null; m.atlas = atlas_dev_or_null;
  for (int k = 0; k < 3; ++k) m.bg[k] = background_host[k];
  m.rgb = rgb_out_or_null; m.depth = depth_out_or_null; m.face = face_out_or_null;
  m.big_pixels = raster_big_face_pixels();
  if (int e = h->rs_ws.ensure(raster_ws_bytes(m))) return e;
  return rasterize_mesh(m, counts_host, h->rs_ws.p, h->d_err + 2, (cudaStream_t)stream, &h->launches);
}

// ---------------------------------------------------------------------------------------------- surface points
// Argument checks come before the handle is touched, so a bad call is rejected without a device.
int nm_surface_points(NmHandle h, const float* pose_host, int H, int W, float focal, const float* depth_raw_dev,
                      const float* acc_dev, const float* rgb_dev, float min_acc, int step, float dist_threshold, int min_count,
                      float* points_out_dev, float* normals_out_dev, float* colors_out_dev, int32_t* pixel_out_dev_or_null,
                      int64_t* count_host, void* stream) {
  NM_CHECK(H >= 1 && W >= 1, "surface points: image %d x %d is empty", H, W);
  NM_CHECK((long long)H * W < (1ll << 31), "surface points: %d x %d pixels is 2^31 or more", H, W);
  NM_CHECK(step >= 0 && step <= kSurfaceMaxStep, "surface points: step %d outside [0, %d]", step, kSurfaceMaxStep);
  NM_CHECK(min_count >= 1, "surface points: min_count %d is below 1", min_count);
  NM_CHECK(focal > 0.f && std::isfinite(focal), "surface points: focal length %g is not positive and finite", (double)focal);
  NM_CHECK(!std::isnan(min_acc) && !std::isnan(dist_threshold), "surface points: min_acc or dist_threshold is NaN");
  NM_CHECK(pose_host && count_host, "surface points: null pose or count pointer");
  NM_CHECK(depth_raw_dev && acc_dev && rgb_dev, "surface points: null depth_raw, acc or rgb pointer");
  NM_CHECK(points_out_dev && normals_out_dev && colors_out_dev, "surface points: null output pointer");
  NM_CHECK(h != nullptr, "null handle");
  *count_host = 0;
  if (int e = bind_checked(h)) return e;
  SurfaceView v;
  memcpy(v.pose, pose_host, sizeof(v.pose));
  v.H = H; v.W = W; v.focal = focal;
  v.depth_raw = depth_raw_dev; v.acc = acc_dev; v.rgb = rgb_dev;
  v.min_acc = min_acc; v.dist_threshold = dist_threshold; v.step = step; v.min_count = min_count;
  if (int e = h->sf_ws.ensure(surface_ws_bytes(H, W))) return e;
  return surface_points(v, points_out_dev, normals_out_dev, colors_out_dev, pixel_out_dev_or_null, count_host, h->sf_ws.p,
                        (cudaStream_t)stream, &h->launches);
}

// ---------------------------------------------------------------------------------------------- sparse density sweep
namespace {
// Argument checks come before the handle is touched, so a bad call is rejected without a device.
int sparse_sweep_setup(NmHandle h, const float* lin0, const float* lin1, const float* lin2, int n0, int n1, int n2, int block,
                       float* vol_dev, const void* out_host, cudaStream_t st, SparseSweep* s) {
  NM_CHECK(lin0 && lin1 && lin2 && vol_dev && out_host, "sparse sweep: null pointer");
  NM_CHECK(block == 4 || block == 8 || block == 16, "sparse sweep: block edge %d is not one of 4, 8, 16", block);
  NM_CHECK(n0 >= 2 && n1 >= 2 && n2 >= 2, "sparse sweep: grid %d x %d x %d has fewer than 2 points on an axis", n0, n1, n2);
  NM_CHECK((long long)n0 * n1 * n2 < (1ll << 31), "sparse sweep: grid %d x %d x %d has 2^31 points or more", n0, n1, n2);
  NM_CHECK(h != nullptr, "null handle");
  if (int e = bind_checked(h)) return e;
  const int which = h->has_fine ? NM_NET_FINE : NM_NET_COARSE;     // the net nm_grid_sigma sweeps
  NM_CHECK(h->nets[which].loaded, "sparse sweep: weights of network %d not loaded", which);
  const float* hs[3] = {lin0, lin1, lin2};
  const int ns[3] = {n0, n1, n2};
  for (int i = 0; i < 3; ++i) { if (int e = upload(&h->lin[i], hs[i], sizeof(float) * ns[i])) return e; h->lin_n[i] = ns[i]; }
  s->n0 = n0; s->n1 = n1; s->n2 = n2; s->block = block;
  for (int i = 0; i < 3; ++i) s->lin[i] = h->lin[i].as<float>();
  s->vol = vol_dev;
  s->chunk_points = sparse_chunk_points();
  s->eval = [h, which, st](const float* pts, long long M, float* sigma) -> int {
    MlpInput in{};
    in.mode = IN_POINTS; in.pts = pts; in.dirs = nullptr; in.M = M;     // directions = positions, as in the grid sweep
    return run_mlp(h, which, true, in, sigma, st);
  };
  return h->sp_ws.ensure(sparse_sweep_ws_bytes(*s));
}
}  // namespace

int nm_sparse_sweep_lattice(NmHandle h, const float* lin0_host, const float* lin1_host, const float* lin2_host, int n0, int n1,
                            int n2, int block, float* vol_dev, float* stats_host, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SparseSweep s;
  if (h) h->sp_vol = nullptr;
  if (int e = sparse_sweep_setup(h, lin0_host, lin1_host, lin2_host, n0, n1, n2, block, vol_dev, stats_host, st, &s)) return e;
  if (int e = sparse_sweep_lattice(s, h->sp_ws.p, h->d_stats, stats_host, st, &h->launches)) return e;
  h->sp_grid[0] = n0; h->sp_grid[1] = n1; h->sp_grid[2] = n2; h->sp_grid[3] = block;
  h->sp_vol = vol_dev;
  return 0;
}

int nm_sparse_sweep_run(NmHandle h, const float* lin0_host, const float* lin1_host, const float* lin2_host, int n0, int n1, int n2,
                        int block, float iso, float* vol_dev, int64_t* counts_host, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  SparseSweep s;
  if (int e = sparse_sweep_setup(h, lin0_host, lin1_host, lin2_host, n0, n1, n2, block, vol_dev, counts_host, st, &s)) return e;
  NM_CHECK(h->sp_vol == vol_dev && h->sp_grid[0] == n0 && h->sp_grid[1] == n1 && h->sp_grid[2] == n2 && h->sp_grid[3] == block,
           "sparse sweep: call nm_sparse_sweep_lattice with the same grid, block and volume first");
  return sparse_sweep_run(s, iso, h->sp_ws.p, counts_host, h->num_sms, st, &h->launches);
}

int nm_debug_sparse_sweep_state(NmHandle h, uint32_t* mask_out_dev_or_null, int32_t* blocks_out_dev_or_null, void* stream) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(h->sp_vol && h->sp_ws.p, "sparse sweep: no sweep has run on this handle");
  SparseSweep s;
  s.n0 = h->sp_grid[0]; s.n1 = h->sp_grid[1]; s.n2 = h->sp_grid[2]; s.block = h->sp_grid[3];
  s.chunk_points = sparse_chunk_points();
  return sparse_sweep_state(s, h->sp_ws.p, mask_out_dev_or_null, blocks_out_dev_or_null, (cudaStream_t)stream);
}

int nm_marching_cubes_count(NmHandle h, const float* vol_dev, int nx, int ny, int nz, float iso, int64_t* counts_host,
                            void* stream) {
  return nm_mc_count(h, vol_dev, nx, ny, nz, iso, 0, nx, 0, nx, counts_host, stream);
}

int nm_marching_cubes_emit(NmHandle h, const float* vol_dev, int nx, int ny, int nz, float iso, float x_off,
                           float* verts_dev, float* normals_dev, int32_t* faces_dev, void* stream) {
  NM_CHECK(x_off >= 0.f && x_off == (float)(int)x_off, "x_off must be a non-negative integer number of planes");
  // a stand-alone volume whose axis-0 vertex coordinates start at x_off (a pure coordinate shift)
  if (int e = bind_device(h)) return e;
  NM_CHECK(vol_dev && verts_dev && faces_dev && h->mc_ws.p, "bad arguments (call nm_marching_cubes_count first)");
  const McShard s{vol_dev, nx, ny, nz, iso, 0, nx, 0, nx, (int)x_off};
  if (int e = h->mc_ws2.ensure(mc_emit_ws_bytes(h->mc_counts[0], h->mc_counts[1]))) return e;
  return mc_emit(s, h->mc_ws.p, h->mc_ws.cap, h->mc_ws2.p, 0, h->mc_counts[0], h->mc_counts[1], verts_dev, normals_dev,
                 faces_dev, (cudaStream_t)stream, &h->launches);
}

int nm_query_host(NmHandle h, const float* origins_host, int o_stride, const float* dirs_host, int64_t R,
                  const float* near_far_host, int flags, uint64_t seed, const NmRenderOut* out_host) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(origins_host && dirs_host && near_far_host && out_host && R > 0, "bad arguments");
  NM_CHECK(!(flags & NM_FLAG_TEACHER_T), "NM_FLAG_TEACHER_T is a device-pointer feature");
  NM_CHECK(!(flags & NM_FLAG_SKIP_EMPTY_TRAIN), "NM_FLAG_SKIP_EMPTY_TRAIN is taken by nm_render_rays, nm_backward_rays and nm_loss_backward");
  cudaStream_t st = h->own_stream;
  const size_t ob = o_stride ? (size_t)R * 12 : 12;
  if (int e = h->stage_in[0].ensure(ob)) return e;
  if (int e = h->stage_in[1].ensure((size_t)R * 12)) return e;
  NM_CUDA(cudaMemcpyAsync(h->stage_in[0].p, origins_host, ob, cudaMemcpyHostToDevice, st));
  NM_CUDA(cudaMemcpyAsync(h->stage_in[1].p, dirs_host, (size_t)R * 12, cudaMemcpyHostToDevice, st));
  NmRenderOut dev{};
  size_t sizes[12];
  if (int e = stage_outputs(h, *out_host, R, out_samples(h, flags), h->cfg.num_coarse, &dev, sizes)) return e;
  if (int e = render_rays_impl(h, h->stage_in[0].as<float>(), o_stride, h->stage_in[1].as<float>(), R, near_far_host,
                               nullptr, nullptr, flags, seed, dev, st)) return e;
  if (int e = copy_outputs(*out_host, dev, sizes, st)) return e;
  NM_CUDA(cudaStreamSynchronize(st));
  return check_kernel_flags(h);
}

int nm_render_image_host(NmHandle h, const float* pose_host, int H, int W, double focal, int ndc, int row0, int row1,
                         const float* near_far_host, int flags, uint64_t seed, const NmRenderOut* out_host) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(out_host, "null output block");
  NM_CHECK(0 <= row0 && row0 <= row1 && row1 <= H && W > 0, "bad row range");
  const long long R = (long long)(row1 - row0) * W;
  cudaStream_t st = h->own_stream;
  NmRenderOut dev{};
  size_t sizes[12];
  if (int e = stage_outputs(h, *out_host, R, out_samples(h, flags), h->cfg.num_coarse, &dev, sizes)) return e;
  if (int e = nm_render_image(h, pose_host, H, W, focal, ndc, row0, row1, near_far_host, flags, seed, &dev, st)) return e;
  if (int e = copy_outputs(*out_host, dev, sizes, st)) return e;
  NM_CUDA(cudaStreamSynchronize(st));
  return check_kernel_flags(h);
}

int nm_point_mlp_host(NmHandle h, int which, const float* pts_host, const float* dirs_host, int64_t M, float* out_host,
                      int sigma_only) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(pts_host && out_host && M > 0, "bad arguments");
  cudaStream_t st = h->own_stream;
  const size_t outb = (size_t)M * (sigma_only ? 4 : 16);
  if (int e = h->stage_in[0].ensure((size_t)M * 12)) return e;
  if (int e = h->stage_in[1].ensure((size_t)M * 12)) return e;
  if (int e = h->stage_out[0].ensure(outb)) return e;
  NM_CUDA(cudaMemcpyAsync(h->stage_in[0].p, pts_host, (size_t)M * 12, cudaMemcpyHostToDevice, st));
  if (dirs_host) NM_CUDA(cudaMemcpyAsync(h->stage_in[1].p, dirs_host, (size_t)M * 12, cudaMemcpyHostToDevice, st));
  if (int e = nm_point_mlp(h, which, h->stage_in[0].as<float>(), dirs_host ? h->stage_in[1].as<float>() : nullptr, M,
                           h->stage_out[0].as<float>(), sigma_only, st)) return e;
  NM_CUDA(cudaMemcpyAsync(out_host, h->stage_out[0].p, outb, cudaMemcpyDeviceToHost, st));
  NM_CUDA(cudaStreamSynchronize(st));
  return check_kernel_flags(h);
}

int nm_debug_pack(const NmNetDesc* desc, int n_tensors, const char* const* names, const float* const* tensors_host,
                  const int64_t* numel, int sigma_only, void* program_out, size_t program_cap, uint8_t* pack_out,
                  size_t pack_cap, size_t* pack_need) {
  NM_CHECK(desc && program_out && pack_need, "null argument");
  NM_CHECK(program_cap >= sizeof(NetProgram), "program buffer too small (%zu needed)", sizeof(NetProgram));
  WeightSource src;
  src.n = n_tensors; src.names = names; src.ptrs = tensors_host; src.numel = numel;
  return debug_pack(*desc, src, sigma_only != 0, false, reinterpret_cast<NetProgram*>(program_out), pack_out, pack_cap,
                    pack_need);
}

int nm_debug_pack_wide(const NmNetDesc* desc, int n_tensors, const char* const* names, const float* const* tensors_host,
                       const int64_t* numel, int sigma_only, void* program_out, size_t program_cap, uint8_t* pack_out,
                       size_t pack_cap, size_t* pack_need) {
  NM_CHECK(desc && program_out && pack_need, "null argument");
  NM_CHECK(program_cap >= sizeof(NetProgram), "program buffer too small (%zu needed)", sizeof(NetProgram));
  WeightSource src;
  src.n = n_tensors; src.names = names; src.ptrs = tensors_host; src.numel = numel;
  return debug_pack(*desc, src, sigma_only != 0, true, reinterpret_cast<NetProgram*>(program_out), pack_out, pack_cap,
                    pack_need);
}

int nm_check_flags(NmHandle h, void* stream) {
  if (int e = bind_device(h)) return e;
  NM_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  return check_kernel_flags(h);
}

int nm_ndc_rays(NmHandle h, int H, int W, double focal, double near, const float* origins_dev, int o_stride,
                const float* dirs_dev, int64_t n, float* origins_out_dev, float* dirs_out_dev, void* stream) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(origins_dev && dirs_dev && origins_out_dev && dirs_out_dev && n >= 0, "bad arguments");
  NM_CHECK(o_stride == 0 || o_stride == 3, "o_stride must be 0 or 3");
  return launch_ndc(H, W, focal, near, origins_dev, o_stride, dirs_dev, n, origins_out_dev, dirs_out_dev, (cudaStream_t)stream,
                    &h->launches);
}

int nm_kernel_flags(NmHandle h, int32_t* out2) {
  NM_CHECK(h && out2, "null argument");
  out2[0] = h->h_err[0];
  out2[1] = h->h_err[1];
  return 0;
}

int64_t nm_launch_count(NmHandle h) { return h ? h->launches : -1; }

int64_t nm_sigma_only_points(NmHandle h) { return h ? h->sigma_points : -1; }

int nm_debug_tile_schedule(int samples_per_ray, int64_t n_tiles, int grid, int cta, int64_t* tiles_out, int64_t cap, int64_t* n_out) {
  const int g = mlp_tc_composite_group(samples_per_ray);
  if (tiles_out && n_out) {
    const int64_t gt = g > 0 ? g : 1;       // the kernel's tile_of(): groups of gt consecutive tiles dealt round-robin
    int64_t n = 0;
    for (int64_t i = 0;; ++i) {
      const int64_t grp = cta + (i / gt) * grid, t = grp * gt + (i % gt);
      if (t >= n_tiles) break;
      if (n < cap) tiles_out[n] = t;
      ++n;
    }
    *n_out = n;
  }
  return g;
}

int nm_debug_mlp_layout(const void* program, size_t program_size, int max_smem, int comp_on, int training, int slot_cap,
                        int64_t* out5) {
  NM_CHECK(program && out5, "null argument");
  NM_CHECK(program_size >= sizeof(NetProgram), "program buffer too small (%zu needed)", sizeof(NetProgram));
  MlpTcLayout l;
  if (int e = mlp_tc_layout(*reinterpret_cast<const NetProgram*>(program), max_smem, comp_on != 0, training != 0, slot_cap, &l)) return e;
  const int64_t v[5] = {l.num_stages, l.off_wg, l.off_bars, l.off_carry, l.bytes};
  for (int i = 0; i < 5; ++i) out5[i] = v[i];
  return 0;
}

int nm_set_timing(NmHandle h, int enable) {
  NM_CHECK(h, "null handle");
  h->timing = enable != 0;
  h->ev_used = 0; h->mlp_points = 0; h->mlp_launches = 0;
  return 0;
}

double nm_mlp_time_ms(NmHandle h, int64_t* points_out, int64_t* launches_out) {
  if (!h || !h->timing) return -1.0;
  cudaSetDevice(h->device);
  double total = 0.0;
  for (size_t i = 0; i + 1 < h->ev_used; i += 2) {
    if (cudaEventSynchronize(h->ev[i + 1]) != cudaSuccess) return -1.0;
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, h->ev[i], h->ev[i + 1]) != cudaSuccess) return -1.0;
    total += ms;
  }
  if (points_out) *points_out = h->mlp_points;
  if (launches_out) *launches_out = h->mlp_launches;
  h->ev_used = 0; h->mlp_points = 0; h->mlp_launches = 0;
  return total;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------- empty-space skipping
namespace {
int occ_params(NmHandle h, int which, const float* box, int G, NmHandle_t::OccGrid* g) {
  NM_CHECK(which == NM_NET_COARSE || (which == NM_NET_FINE && h->has_fine), "network slot %d not present", which);
  NM_CHECK(box, "null box");
  NM_CHECK(G >= 1 && G <= kOccMaxRes, "occupancy resolution %d outside [1, %d]", G, kOccMaxRes);
  for (int a = 0; a < 3; ++a) {
    const float lo = box[a], hi = box[3 + a];
    NM_CHECK(std::isfinite(lo) && std::isfinite(hi) && lo < hi, "occupancy box axis %d: [%g, %g] is not a finite interval", a, lo, hi);
    const float inv = (float)((double)G / ((double)hi - (double)lo));
    NM_CHECK(std::isfinite(inv) && inv > 0.f, "occupancy box axis %d: G / (hi - lo) is not finite", a);
    g->lo[a] = lo; g->hi[a] = hi; g->inv[a] = inv;
  }
  g->G = G;
  return 0;
}
size_t occ_words(int G) { return (size_t)(((long long)G * G * G + 31) / 32); }
}  // namespace

extern "C" {

int nm_build_occupancy(NmHandle h, int which, const float* box_host, int G, float threshold, int dilate,
                       uint32_t* bits_out_dev_or_null, void* stream) {
  if (int e = bind_checked(h)) return e;
  NmHandle_t::OccGrid p{};
  if (int e = occ_params(h, which, box_host, G, &p)) return e;
  NM_CHECK(!std::isnan(threshold), "occupancy threshold is NaN");
  NM_CHECK(dilate >= 0 && dilate <= G, "occupancy dilation %d outside [0, %d]", dilate, G);
  NmHandle_t::OccGrid& g = h->occ[which];
  g.valid = false;
  cudaStream_t st = (cudaStream_t)stream;
  // torch.linspace(lo, hi, G+1) in fp32: step = (hi - lo) / G, lo + step*i below the midpoint and hi - step*(G-i) from it,
  // each one fused multiply-add (ATen's two-sided formula; the values torch returns on the CPU and the GPU)
  const long long n1 = G + 1, plane = n1 * n1;
  std::vector<float> lins(3 * n1);
  for (int a = 0; a < 3; ++a) {
    const float step = (p.hi[a] - p.lo[a]) / (float)G;
    for (long long i = 0; i < n1; ++i)
      lins[a * n1 + i] = (i < n1 / 2) ? std::fmaf(step, (float)i, p.lo[a]) : std::fmaf(-step, (float)(G - i), p.hi[a]);
  }
  // the lattice is swept in slabs of cells [x0, x1) whose planes [x0, x1] hold at most 4 Mi points (16 MB)
  const long long cells_per = std::max(1ll, std::min((long long)G, (1ll << 22) / plane - 1));
  const size_t cube = (size_t)G * G * G;
  const size_t o_sig = ((size_t)3 * n1 * 4 + 255) & ~(size_t)255;
  const size_t o_a = o_sig + (((size_t)(cells_per + 1) * plane * 4 + 255) & ~(size_t)255), o_b = o_a + ((cube + 255) & ~(size_t)255);
  if (int e = h->oc_ws.ensure(o_b + cube)) return e;
  if (int e = g.bits.ensure(occ_words(G) * 4)) return e;
  uint8_t* ws = h->oc_ws.as<uint8_t>();
  float* lin = reinterpret_cast<float*>(ws);
  NM_CUDA(cudaMemcpyAsync(lin, lins.data(), lins.size() * 4, cudaMemcpyHostToDevice, st));
  float* sigma = reinterpret_cast<float*>(ws + o_sig);
  for (long long x0 = 0; x0 < G; x0 += cells_per) {
    const long long x1 = std::min((long long)G, x0 + cells_per);
    MlpInput in{};
    in.mode = IN_GRID;
    in.lin0 = lin; in.lin1 = lin + n1; in.lin2 = lin + 2 * n1;
    in.n1 = (int)n1; in.n2 = (int)n1;
    in.grid_base = x0 * plane;
    in.M = (x1 - x0 + 1) * plane;
    if (int e = run_mlp(h, which, true, in, sigma, st)) return e;
    if (int e = launch_occ_corners(sigma, G, (int)x0, (int)x1, threshold, ws + o_a, st, &h->launches)) return e;
  }
  if (int e = launch_occ_dilate_pack(ws + o_a, ws + o_b, G, dilate, g.bits.as<uint32_t>(), st, &h->launches)) return e;
  if (bits_out_dev_or_null)
    NM_CUDA(cudaMemcpyAsync(bits_out_dev_or_null, g.bits.p, occ_words(G) * 4, cudaMemcpyDeviceToDevice, st));
  NM_CUDA(cudaStreamSynchronize(st));      // the host copy of `lins` must outlive its transfer
  memcpy(g.lo, p.lo, sizeof(p.lo)); memcpy(g.hi, p.hi, sizeof(p.hi)); memcpy(g.inv, p.inv, sizeof(p.inv));
  g.G = G;
  g.valid = true;
  g.stale = false;
  return 0;
}

int nm_set_occupancy(NmHandle h, int which, const float* box_host, int G, const uint32_t* bits_dev_or_null) {
  if (int e = bind_checked(h)) return e;
  NM_CHECK(which == NM_NET_COARSE || (which == NM_NET_FINE && h->has_fine), "network slot %d not present", which);
  NmHandle_t::OccGrid& g = h->occ[which];
  g.valid = false;
  if (!bits_dev_or_null) return 0;
  NmHandle_t::OccGrid p{};
  if (int e = occ_params(h, which, box_host, G, &p)) return e;
  if (int e = g.bits.ensure(occ_words(G) * 4)) return e;
  NM_CUDA(cudaMemcpy(g.bits.p, bits_dev_or_null, occ_words(G) * 4, cudaMemcpyDeviceToDevice));
  memcpy(g.lo, p.lo, sizeof(p.lo)); memcpy(g.hi, p.hi, sizeof(p.hi)); memcpy(g.inv, p.inv, sizeof(p.inv));
  g.G = G;
  g.valid = true;
  g.stale = false;
  return 0;
}

int nm_occupancy_query(NmHandle h, int which, const float* pts_dev, int64_t M, uint8_t* evaluated_out_dev, void* stream) {
  if (int e = bind_checked(h)) return e;
  NM_CHECK(which == NM_NET_COARSE || (which == NM_NET_FINE && h->has_fine), "network slot %d not present", which);
  NM_CHECK(h->occ[which].valid && !h->occ[which].stale, "no occupancy grid for network %d", which);
  NM_CHECK(M >= 0 && (M == 0 || (pts_dev && evaluated_out_dev)), "bad arguments");
  return launch_occ_query(occ_lookup(h->occ[which]), pts_dev, M, evaluated_out_dev, (cudaStream_t)stream, &h->launches);
}

int nm_skip_stats(NmHandle h, int64_t* out_host) {
  if (int e = bind_device(h)) return e;
  NM_CHECK(out_host, "null argument");
  NM_CUDA(cudaDeviceSynchronize());
  for (int i = 0; i < 4; ++i) { out_host[i] = h->skip_counts[i]; h->skip_counts[i] = 0; }
  return 0;
}

}  // extern "C"
