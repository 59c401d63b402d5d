// Internal declarations shared by the translation units of libnerfmeshes_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <functional>
#include <string>
#include <vector>

#include "../../include/nerfmeshes_b200.h"
#include "nm_program.h"

namespace nm {

void set_error(const char* fmt, ...);
#define NM_CUDA(expr)                                                                             \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      nm::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return -2;                                                                                  \
    }                                                                                             \
  } while (0)
#define NM_CHECK(cond, ...)       \
  do {                            \
    if (!(cond)) {                \
      nm::set_error(__VA_ARGS__); \
      return -1;                  \
    }                             \
  } while (0)

// One network's device-resident data.
struct NetDev {
  bool loaded = false;
  NmNetDesc desc{};
  NetProgram full{};        // rgb + sigma
  NetProgram sigma{};       // trunk + sigma head only (grid fast path)
  // device arrays
  NetProgram* d_full = nullptr;
  NetProgram* d_sigma = nullptr;
  uint8_t* d_wpack_full = nullptr;   // tensor-core weight stages of `full`: the wide stream (nm_program.h)
  uint8_t* d_wpack_sigma = nullptr;
  float* d_bias = nullptr;
  float* d_head = nullptr;
  float* d_wt = nullptr;             // transposed fp32 weights (CUDA-core kernel)
  float* d_w = nullptr;              // the same weights in the reference's (out,in) layout, same per-layer offsets
  size_t n_wt = 0;                   // floats in d_wt
  // fused data-gradient chain (nm_mlp_tc.cu, mode 2): backward program + W^T stages (bf16 hi/lo), rebuilt lazily
  NetProgram bwd{};
  NetProgram* d_bwd = nullptr;
  uint8_t* d_wpack_bwd = nullptr;
  bool bwd_valid = false;
  std::vector<std::string> names;    // per layer of `full`: weight, bias, head weight, head bias ("" if none)
};

// Weight-gradient buffer layout: per layer (n_out, ld) row-major in the reference's (out,in) orientation, ld = in
// features rounded up to 4 floats so that rows stay 16-byte aligned (vector atomics).  Returns the total float count.
inline size_t grad_layout(const NetProgram& G, size_t off[kMaxLayers], int ld[kMaxLayers]) {
  size_t total = 0;
  for (int l = 0; l < G.n_layers; ++l) {
    const int K = G.layers[l].k_act + G.layers[l].k_pe;
    ld[l] = (K + 3) & ~3;
    off[l] = total;
    total += (size_t)G.layers[l].n_out * ld[l];
  }
  return total;
}

// Gradient accumulators of one network: weights per grad_layout(), biases / heads like NetDev.d_bias / d_head.
struct NetGrads {
  float* w = nullptr;
  float* bias = nullptr;
  float* head = nullptr;
};

// Inputs of one fused-MLP launch (three front-end modes).
enum : int { IN_POINTS = 0, IN_RAYS = 1, IN_GRID = 2 };
struct MlpInput {
  int mode = IN_POINTS;
  const float* pts = nullptr;    // IN_POINTS (M,3)
  const float* dirs = nullptr;   // IN_POINTS (M,3);  IN_RAYS (R,3)
  const float* ray_o = nullptr;  // IN_RAYS
  int o_stride = 0;              //   0: shared origin, 3: per ray
  const float* t = nullptr;      // IN_RAYS (R,S)
  int S = 0;
  const float* lin0 = nullptr;   // IN_GRID: device linspace tables
  const float* lin1 = nullptr;
  const float* lin2 = nullptr;
  int n1 = 0, n2 = 0;
  long long grid_base = 0;       //   flat index of the first point
  long long M = 0;               // number of points
};

// Optional by-products of a fused-MLP launch for the training backward (nm_train.cu): per layer (nullptr = not wanted)
//   packT  the layer's output as the point-major bf16 hi/lo operand pack of the weight-gradient GEMM (nm_gemm.h: tiles of
//          128 features x 64 points, [feature block][point block], `kbt` point blocks per feature block; rows >= M zero),
//          K-major from the training forward (mode 1), MN-major from the data-gradient chain (mode 2)
//   bits   its relu mask, one bit per element (halfword [m * n_out/16 + n/16], bit n%16)
//   act    its fp32 value (M, n_out) row-major (the layers the SIMT head kernels read)
struct MlpEmit {
  uint8_t* packT[kMaxLayers];
  uint32_t* bits[kMaxLayers];
  float* act[kMaxLayers];
  int kbt;
};

int build_programs(const NmNetDesc& d, NetProgram* full, NetProgram* sigma);
int build_backward_program(const NetProgram& full, NetProgram* bwd);
int build_backward_stream(NetDev* net, cudaStream_t st, int64_t* launches);
// Packs host fp32 reference tensors into the device layouts.  `get(name, &numel)` returns the host tensor.
struct WeightSource {
  int n = 0;
  const char* const* names = nullptr;
  const float* const* ptrs = nullptr;
  const int64_t* numel = nullptr;
  const float* find(const std::string& name, int64_t expect) const;
};
int pack_network(const NmNetDesc& d, const WeightSource& src, NetDev* net);
int load_network_dev(const NmNetDesc& d, const WeightSource& src_device, NetDev* net, cudaStream_t st, int64_t* launches);
void free_network(NetDev* net);
int debug_pack(const NmNetDesc& d, const WeightSource& src, bool sigma_only, bool wide, NetProgram* prog, uint8_t* out,
               size_t cap, size_t* need);

// kernel launchers (return 0 / <0; count launches via *launches)
struct CompositeArgs;
// comp != nullptr (inference on ray inputs): the compositor runs inside the kernel on the staged outputs of every tile and
// writes the per-ray maps (and weights, if asked); `out` is not written.  mlp_tc_composite_group(S) == 0: not eligible.
// With sigma_only, comp is accepted too: the program's sigma enters the compositor with rgb (0, 0, 0), for a pass whose
// caller reads no colour map (the weights, acc and disp depend on sigma alone).
int mlp_tc_composite_group(int samples_per_ray);
// shared-memory layout of the fused MLP kernel (byte offsets into its dynamic shared memory; the ring is at 0)
struct MlpTcLayout {
  int num_stages;                       // 16 KB weight-ring slots
  uint32_t off_wg, off_bias, off_head, off_bars, off_carry, bytes;
};
int mlp_tc_layout(const NetProgram& prog, int max_smem, bool comp_on, bool training, int slot_cap, MlpTcLayout* out);
int launch_mlp_tc(const NetDev& net, bool sigma_only, int n_passes, int act_scale_log2, const MlpInput& in, float* out,
                  int num_sms, int* d_err, cudaStream_t st, int64_t* launches, const MlpEmit* emit = nullptr,
                  const CompositeArgs* comp = nullptr);
int launch_mlp_tc_bwd(const NetDev& net, long long M, const float* dz_in, int dz_ld, const float* dout,
                      const MlpEmit& io, int n_passes, int num_sms, int* d_err, cudaStream_t st, int64_t* launches);
int launch_mlp_simt(const NetDev& net, bool sigma_only, const MlpInput& in, float* out, cudaStream_t st,
                    int64_t* launches);

// focal and near stay double: ndc_rays forms its scalars from the caller's python floats, so they are rounded to fp32 only
// after that arithmetic (launch_raygen / launch_ndc); the pixel division uses (float)focal, as torch's tensor / scalar does.
struct RayGenArgs {
  float pose[12];
  int H, W;
  double focal;
  int ndc;
  double ndc_near;
  int row0, row1;
};
int launch_raygen(const RayGenArgs& a, float* origins_or_null, float* dirs, cudaStream_t st, int64_t* launches);
int launch_ndc(int H, int W, double focal, double near, const float* origins, int o_stride, const float* dirs, long long n,
               float* out_o, float* out_d, cudaStream_t st, int64_t* launches);
int launch_stratified(const float* s_table, int Nc, long long R, const float* near_far2, const float* near_dev,
                      const float* far_dev, int lindisp, int perturb, uint64_t seed, float* t_out, cudaStream_t st,
                      int64_t* launches);
struct CompositeArgs {
  const float* raw;    // (R,S,4)
  const float* t;      // (R,S)
  const float* dirs;   // (R,3)
  long long R;
  int S;
  float noise_std;
  uint64_t seed;
  int white_bg, training;
  float thr;
  float *rgb, *depth, *depth_raw, *acc, *disp, *weights, *mask_weights;
};
int launch_composite(const CompositeArgs& a, cudaStream_t st, int64_t* launches);
int launch_invcdf(const float* t_c, const float* w_c, const float* u_table, int Nc, int Nf, long long R, int perturb,
                  uint64_t seed, float* t_f, cudaStream_t st, int64_t* launches);
// random != 0: cfg.tree.use_random_sampling, drawn from the stream `seed` (already salted: the callers pass seed ^ kVoxelSalt)
int launch_aabb(const float* voxels, int V, const float* origins, int o_stride, const float* dirs, long long R,
                float near, float far, int S, const float* s_table, const float* t_uniform, float* z_out, int* idx_out,
                int* d_overflow, cudaStream_t st, int64_t* launches, int random = 0, uint64_t seed = 0);
int launch_tree_integrate(const int* idx, const float* w, const float* mw, long long n, float* memm, int V, int counter,
                          float* scratch2v, cudaStream_t st, int64_t* launches);
int launch_volume_stats(const float* vol, long long n, double* d_scratch, float* out_host, cudaStream_t st,
                        int64_t* launches);
int launch_volume_stats_pass(const float* vol, long long n, int pass, const double* mean_dev, double* out_dev, cudaStream_t st,
                             int64_t* launches);
// training backward (nm_train.cu)
size_t train_ws_bytes(const NetProgram& full, long long points, bool use_tc);
struct TrainMode { int use_tc; int n_passes; int* d_err; };
int mlp_backward(NetDev& net, const MlpInput& in, const float* dout, float* ws, NetGrads* g, int num_sms,
                 const TrainMode& mode, cudaStream_t st, int64_t* launches, int have_acts = 0);
void train_emit_setup(const NetProgram& full, long long points, float* ws, MlpEmit* emit);
// pos: NULL, dout (R,S,4); or the exclusive scan of a skipping pass's marks (R*S + 1 entries, nm_occupancy.cu), and dout
// holds only the evaluated samples' rows, sample m's at pos[m] (empty-space skipping in training, DESIGN §4.15)
int launch_composite_backward(const float* raw, const float* t, const float* dirs, const float* d_rgb, long long R, int S,
                              float noise_std, uint64_t seed, int white_bg, float* scratch, float* dout,
                              cudaStream_t st, int64_t* launches, const int* pos = nullptr);
int launch_mse_grad(const float* rgb, const float* target, long long n, long long count, float* d_rgb, float* loss,
                    cudaStream_t st, int64_t* launches);
// density gradient g = d raw sigma / d p (nm_sigma_grad.cu, orchestrated by sigma_grad in nm_train.cu; DESIGN 4.8)
struct PeDesc { int L, inc; float freq[kMaxFreq]; };     // the xyz encoding
constexpr int kSgMaxKb = 64;                             // 64-feature K-blocks of the xyz-reading layers
struct SigmaGradWeights {
  const float* wt[kSgMaxKb];    // per K-block: &Wt[k_act][64 kb'] of its layer; element (column j, feature kk) at wt[j * ld + kk]
  int ld[kSgMaxKb];             // the layer's n_out
  int k_pe;
  uint8_t* out;                 // n_kb x 16 KB of packed B tiles
};
struct SigmaGradTail {
  const uint8_t* a[kSgMaxKb];   // per K-block: the 64-feature group of its layer's dZ pack at point block 0 (point block b: + b ptiles)
  const uint8_t* b;             // SigmaGradWeights.out
  int n_kb, n_passes;
  long long M;
  const float* pts;             // (M,3)
  PeDesc pe;
  float* grad;                  // (M,3)
  int* err;
};
int launch_sigma_grad_tail(const SigmaGradWeights& W, const SigmaGradTail& T, int num_sms, cudaStream_t st, int64_t* launches);
int launch_pe_vjp(const float* pts, long long M, const float* dpe, int ld, const PeDesc& pe, float* grad, cudaStream_t st,
                  int64_t* launches);
// g of network `net` at M points (one chunk); ws: sigma_grad_ws_bytes(full, M, use_tc) bytes, 1 KB aligned.  Writes nothing
// but ws and grad.
size_t sigma_grad_ws_bytes(const NetProgram& full, long long points, bool use_tc);
int sigma_grad(NetDev& net, const float* pts, long long M, float* ws, float* grad, int num_sms, const TrainMode& mode,
               cudaStream_t st, int64_t* launches);
// marching cubes (nm_mc.cu): one shard of a global grid — buffer planes [0,nb) are global planes [g_x0, g_x0+nb) of g_nx;
// the call owns the points (vertices, cells) of buffer planes [p_lo,p_hi)
struct McShard {
  const float* vol;
  int nb, ny, nz;
  float iso;
  int g_x0, g_nx, p_lo, p_hi;
  int x_shift;       // added to the axis-0 vertex coordinates only (stand-alone volumes that are a window of a larger one)
};
// counts_host[2]: {vertices owned, triangles}.  ws: mc_ws_bytes(s) bytes (0 for a shard mc_count rejects) that the count step
// writes and the emit step of the same shard reads; ws2: mc_emit_ws_bytes(nv, nt) bytes (8 per output vertex / triangle)
size_t mc_ws_bytes(const McShard& s);
size_t mc_emit_ws_bytes(int64_t nv, int64_t nt);
int mc_count(const McShard& s, void* ws, size_t ws_bytes, int64_t* counts_host, int num_sms, cudaStream_t st, int64_t* launches);
int mc_emit(const McShard& s, void* ws, size_t ws_bytes, void* ws2, long long v_base, int64_t nv, int64_t nt, float* verts,
            float* normals, int32_t* faces, cudaStream_t st, int64_t* launches);
// super-sampled emit (nm_mc_emit_ss): mc_emit, then every edge vertex is re-placed from s network samples along its edge.
// The vertices are walked in chunks of chunk_vertices; each chunk's chunk_vertices*s points go to `pts` (M,3), are
// evaluated by `eval` (sigma only, at most chunk_points per call) into `sig` (M,), and the chunk's vertices are refined.
constexpr int kMcMaxSuperSampling = 64;
struct McSuperSampling {
  int s = 0;
  const float* lin[3] = {nullptr, nullptr, nullptr};    // device: the coarse tables, g_nx / ny / nz entries
  const float* fine[3] = {nullptr, nullptr, nullptr};   // device: the fine tables, (n-1)(s+1)+1 entries
  float* pts = nullptr;
  float* sig = nullptr;
  long long chunk_vertices = 0, chunk_points = 0;
  std::function<int(const float* pts, long long M, float* sigma)> eval;
};
int mc_emit_ss(const McShard& s, void* ws, size_t ws_bytes, void* ws2, long long v_base, int64_t nv, int64_t nt,
               const McSuperSampling& ss, float* verts, float* normals, int32_t* faces, cudaStream_t st, int64_t* launches);

// exclusive scan of n >= 1 ints (nm_chamfer.cu: the grid search's cell-count scan, also used by the component filter):
// start[i] = cnt[0] + ... + cnt[i-1], exact (integers).  blk: (n + kScanBlockEntries - 1) / kScanBlockEntries ints of scratch.
// Three launches.
constexpr int kScanBlockEntries = 1024;
int exclusive_scan(const int* cnt, long long n, int* blk, int* start, cudaStream_t st);

// chamfer evaluation (nm_chamfer.cu).  ws / ws_bytes: the handle's grow-only workspace, at least *_ws_bytes of the same counts.
size_t mesh_sample_ws_bytes(long long F);
size_t nearest_ws_bytes(long long N, long long M, bool chamfer);      // one search, or chamfer's two with their distances
// mesh_sample: n area-weighted surface points (face index per point if face_idx != nullptr); a face index outside [0,V)
// sets *d_err = 1, a total area that is not positive and finite *d_err = 2 (device-side, mapped memory)
int mesh_sample(const float* verts, long long V, const int32_t* faces, long long F, long long n, uint64_t seed, float* pts,
                int32_t* face_idx, int* d_err, void* ws, size_t ws_bytes, cudaStream_t st, int64_t* launches);
// exact nearest neighbour of each of N queries among M >= 1 points: squared distance (+ index, lowest on ties)
int nearest(const float* q, long long N, const float* p, long long M, float* dist2, int32_t* idx, void* ws, size_t ws_bytes,
            int num_sms, cudaStream_t st, int64_t* launches);
int nearest_brute(const float* q, long long N, const float* p, long long M, float* dist2, int32_t* idx, cudaStream_t st,
                  int64_t* launches);
// means[0] = mean_i d2(x_i, Y), means[1] = mean_j d2(y_j, X) (double, fixed summation order)
int chamfer(const float* x, long long N, const float* y, long long M, double* means, void* ws, size_t ws_bytes, int num_sms,
            cudaStream_t st, int64_t* launches);

// small-component removal (nm_components.cu, DESIGN §4.9).  ws: components_ws_bytes(V, F) bytes of the handle's grow-only
// workspace.  A face index outside [0,V) sets *d_err = 3 (device-side, mapped memory); such a face joins nothing and is
// dropped.  counts_host = {kept vertices, kept faces, components with >= 1 face, kept components}; synchronises.
size_t components_ws_bytes(long long V, long long F);
int mesh_components(const float* verts, const float* normals, long long V, const int32_t* faces, long long F, long long min_faces,
                    float* verts_out, float* normals_out, int32_t* faces_out, int32_t* labels_out, int64_t* counts_host, void* ws,
                    int* d_err, cudaStream_t st, int64_t* launches);

// quadric-error decimation (nm_decimate.cu, DESIGN §4.11).  ws: decimate_ws_bytes(V, F) bytes of the handle's grow-only
// workspace.  A face index outside [0,V) sets *d_err = 4 (device-side, mapped memory) and the input is copied unchanged.
// counts_host = {output vertices, output faces, rounds, collapses}; synchronises once, then once per round.
size_t decimate_ws_bytes(long long V, long long F);
int mesh_decimate(const float* verts, const float* normals, long long V, const int32_t* faces, long long F, long long target,
                  float* verts_out, float* normals_out, int32_t* faces_out, int32_t* source_out, int64_t* counts_host, void* ws,
                  int* d_err, cudaStream_t st, int64_t* launches);

// sparse density sweep (nm_sparse_sweep.cu, DESIGN §4.10): sigma only in the blocks of `block`^3 cells the iso-surface crosses.
// lin: device tables (n0 / n1 / n2 entries); vol: the dense (n0,n1,n2) volume; `eval` is the fused MLP, sigma only, on at
// most chunk_points explicit points per call.  ws: sparse_sweep_ws_bytes(s) bytes of the handle's grow-only workspace.
struct SparseSweep {
  int n0 = 0, n1 = 0, n2 = 0, block = 0;
  const float* lin[3] = {nullptr, nullptr, nullptr};
  float* vol = nullptr;
  long long chunk_points = 0;
  std::function<int(const float* pts, long long M, float* sigma)> eval;
};
size_t sparse_sweep_ws_bytes(const SparseSweep& s);
// sigma at the lattice points into vol; stats_host = {min, max, std} over them (d_stats: 4 doubles of scratch).  Synchronises.
int sparse_sweep_lattice(const SparseSweep& s, void* ws, double* d_stats, float* stats_host, cudaStream_t st, int64_t* launches);
// seeds, rounds to the fixpoint, fill, on a volume that holds the lattice values.  counts_host = {lattice points, active
// blocks, blocks, evaluated points, rounds}.  Synchronises once per round.
int sparse_sweep_run(const SparseSweep& s, float iso, void* ws, int64_t* counts_host, int num_sms, cudaStream_t st, int64_t* launches);
// copies of the last run's evaluated mask (n0*n1*ceil(n2/32) words) and block states (bit 0: sign inside, bit 1: active)
int sparse_sweep_state(const SparseSweep& s, void* ws, uint32_t* mask_out, int32_t* blocks_out, cudaStream_t st);

// texture bake (nm_texture.cu, DESIGN §4.12): N texels per triangle leg, one right-triangle patch per face, two per cell.
// out = {Q cells per row, rows, W, H}; rejects N outside [2, 64], F outside [0, 2^31) and an atlas side above 16384.
constexpr int kTexMinN = 2, kTexMaxN = 64, kTexMaxSide = 16384;
int texture_layout(long long F, int N, long long out[4]);
// mode 0: a = ray origins p - c*d for `render` (the handle's render path), mode 1: a = points p for the point MLP; d = -n.
// `render` writes the colour of ray / point t at rgb[t * rgb_stride + 0..2], for at most chunk_rays(b) of them per call.
struct TextureBake {
  const float* verts = nullptr;
  const float* normals = nullptr;
  long long V = 0;
  const int32_t* faces = nullptr;
  long long F = 0;
  int N = 0, mode = 0, rgb_stride = 3;
  float disparity = 0.f;
  long long chunk_texels = 0;
  std::function<int(const float* a, const float* d, long long n, float* rgb)> render;
};
size_t texture_ws_bytes(const TextureBake& b);
// the texel queries of faces [f0, f1) (texel-major, K = N(N+1)/2 per face) and their atlas pixels (x, y) unless xy_out is null
int texture_rays(const TextureBake& b, long long f0, long long f1, float* a_out, float* d_out, int32_t* xy_out, int* d_err,
                 cudaStream_t st, int64_t* launches);
// the whole bake; ws: texture_ws_bytes(b) bytes.  A face index outside [0, V) sets *d_err = 5 (device-side, mapped memory;
// h_err is its host view) and nothing is baked.  counts_host = {W, H, queries rendered, unreferenced vertices}; synchronises once.
int bake_texture(const TextureBake& b, float* atlas_f32, uint8_t* atlas_u8, float* uv, float* vertex_rgb, int64_t* counts_host,
                 void* ws, int* d_err, const volatile int* h_err, cudaStream_t st, int64_t* launches);

// mesh rasterizer (nm_raster.cu, DESIGN §4.13): world-coordinate triangles through nm_render_image's pinhole camera.  mode 0
// colours by vertex_rgb (V,3), mode 1 by the §4.12 atlas of N texels per leg; any output may be null.  A face whose bounding
// box holds >= big_pixels pixel samples is drawn by the tile pass (the same bits either way).
struct RasterMesh {
  const float* verts = nullptr;
  long long V = 0;
  const int32_t* faces = nullptr;
  long long F = 0;
  float pose[12] = {};
  int H = 0, W = 0;
  float focal = 0.f, z_near = 0.f;
  int mode = 0, N = 0;
  const float* vertex_rgb = nullptr;
  const float* atlas = nullptr;
  float bg[3] = {0.f, 0.f, 0.f};
  float* rgb = nullptr;
  float* depth = nullptr;
  int32_t* face = nullptr;
  long long big_pixels = 0;
};
size_t raster_ws_bytes(const RasterMesh& m);
// ws: raster_ws_bytes(m) bytes.  A face index outside [0, V) sets *d_err = 6 (device-side, mapped memory) and nothing is
// drawn: every pixel gets the background.  counts_host = {covered pixels, faces drawn, faces culled}; synchronises once.
int rasterize_mesh(const RasterMesh& m, int64_t* counts_host, void* ws, int* d_err, cudaStream_t st, int64_t* launches);

// surface points of one rendered view (nm_surface.cu, DESIGN §4.14): depth_raw / acc (H*W), rgb (H*W,3) of nm_render_image
// without NDC for this pose; the kept pixels' points, -directions, colours and pixel indices (pix may be null) in row-major
// order.  ws: surface_ws_bytes(H, W) bytes.  *count_host = kept pixels; synchronises once.
constexpr int kSurfaceMaxStep = 8;
struct SurfaceView {
  float pose[12] = {};
  int H = 0, W = 0;
  float focal = 0.f;
  const float* depth_raw = nullptr;
  const float* acc = nullptr;
  const float* rgb = nullptr;
  float min_acc = 1.f, dist_threshold = 0.f;
  int step = 0, min_count = 1;
};
size_t surface_ws_bytes(long long H, long long W);
int surface_points(const SurfaceView& v, float* pts, float* nrm, float* col, int32_t* pix, int64_t* count_host, void* ws,
                   cudaStream_t st, int64_t* launches);

// occupancy grids for empty-space skipping (nm_occupancy.cu, DESIGN §4.15): G^3 cells over [lo, hi), bit (i*G + j)*G + k of
// uint32 words; inv[a] = G / (hi[a] - lo[a]) rounded once on the host
struct OccLookup {
  const uint32_t* bits;
  float lo[3], inv[3];
  int G;
};
// true when the network must evaluate point p: outside [0, G) on an axis, not finite, or in an occupied cell.  The cell is
// floor((p_a - lo_a) * inv_a) in round-to-nearest fp32, the restatement tests/_occupancy_ref.py makes.
__device__ __forceinline__ bool occ_evaluated(const OccLookup& g, const float p[3]) {
  long long cell = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float f = floorf(__fmul_rn(__fsub_rn(p[a], g.lo[a]), g.inv[a]));
    if (!(f >= 0.f && f < (float)g.G)) return true;
    cell = cell * g.G + (int)f;
  }
  return (__ldg(g.bits + (cell >> 5)) >> (cell & 31)) & 1u;
}
// build: raw occupancy bytes of cells [x0, x1) x G x G from the sigma lattice planes [x0, x1] ((x1-x0+1) x (G+1) x (G+1));
// then the dilation by d cells (ping-pong a / b, G^3 bytes each; a holds the raw bytes) and the bit packing
int launch_occ_corners(const float* sigma, int G, int x0, int x1, float thr, uint8_t* raw, cudaStream_t st, int64_t* launches);
int launch_occ_dilate_pack(uint8_t* a, uint8_t* b, int G, int d, uint32_t* bits, cudaStream_t st, int64_t* launches);
// render: the flat indices of the samples of (R,S) t the network must evaluate, ascending, into idx; *count_host = their
// number; every other sample's row of raw (R,S,4) is set to (0,0,0,-inf), which no sigma noise lifts above 0.  mark / pos:
// R*S + 1 ints, blk: ceil((R*S + 1) / kScanBlockEntries) ints.  Synchronises `st` once (the count).
int occ_compact(const OccLookup& g, const float* origins, int o_stride, const float* dirs, const float* t, long long R, int S,
                int* mark, int* pos, int* blk, int* idx, float* raw, long long* count_host, cudaStream_t st, int64_t* launches);
int launch_occ_stage(const int* idx, long long cnt, int S, const float* origins, int o_stride, const float* dirs, const float* t,
                     float* pts, float* dirs_out, cudaStream_t st, int64_t* launches);
int launch_occ_expand(const float* sub, const int* idx, long long cnt, float* raw, cudaStream_t st, int64_t* launches);
int launch_occ_query(const OccLookup& g, const float* pts, long long M, uint8_t* out, cudaStream_t st, int64_t* launches);

}  // namespace nm
