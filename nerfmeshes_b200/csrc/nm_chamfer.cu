// Chamfer-distance mesh evaluation: the chamfer branch of validation_epoch_end (src/models/model_base.py:82-102), i.e.
// pytorch3d's sample_points_from_meshes and chamfer_distance (DESIGN §4.7).
//   1. surface sampler   ms_area_kernel (areas, index validation) -> ms_range_kernel / ms_chain_kernel (deterministic
//                        two-level double scan) -> ms_sample_kernel (binary search + pytorch3d's barycentric weights)
//   2. nearest neighbour nn_box_kernel (bounding box of both sets) -> nn_params_kernel (cell size) -> count / scan / scatter of
//                        the points (float4, cell order) and of the queries (index, cell order) -> nn_search_kernel
//                        (Chebyshev rings of cells with a rounding-safe stop bound)
//   3. nn_brute_kernel   the tiled brute-force yard-stick (nm_debug_nearest_brute, a test hook)
//   4. chamfer           two searches, then nn_sum_kernel / nn_mean_kernel (double, fixed order)
// Built with -fmad=false: a sampled point is three products and two adds, reproducible on the CPU.
#include <float.h>
#include <math.h>

#include "nm_common.h"
#include "nm_composite.cuh"

namespace nm {
namespace {

constexpr int kBlock = 256;
constexpr int kRange = 256;          // faces per range of the area scan
constexpr int kScanBlock = kScanBlockEntries;   // entries per block of the cell-count scan (shared: exclusive_scan)
constexpr int kSumBlocks = 256;      // blocks per array of the chamfer reduction

size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

// ------------------------------------------------------------------------------------------------ 1. surface sampler
__global__ void __launch_bounds__(kBlock) ms_area_kernel(const float* __restrict__ v, long long V, const int* __restrict__ f,
                                                         long long F, float* __restrict__ area, int* err) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= F) return;
  const int a = f[3 * i], b = f[3 * i + 1], c = f[3 * i + 2];
  if (a < 0 || a >= V || b < 0 || b >= V || c < 0 || c >= V) {
    area[i] = 0.f;
    *(volatile int*)err = 1;
    return;
  }
  const float e1x = __fsub_rn(v[3 * b], v[3 * a]), e1y = __fsub_rn(v[3 * b + 1], v[3 * a + 1]), e1z = __fsub_rn(v[3 * b + 2], v[3 * a + 2]);
  const float e2x = __fsub_rn(v[3 * c], v[3 * a]), e2y = __fsub_rn(v[3 * c + 1], v[3 * a + 1]), e2z = __fsub_rn(v[3 * c + 2], v[3 * a + 2]);
  const float cx = __fsub_rn(__fmul_rn(e1y, e2z), __fmul_rn(e1z, e2y));
  const float cy = __fsub_rn(__fmul_rn(e1z, e2x), __fmul_rn(e1x, e2z));
  const float cz = __fsub_rn(__fmul_rn(e1x, e2y), __fmul_rn(e1y, e2x));
  area[i] = __fmul_rn(0.5f, sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(cx, cx), __fmul_rn(cy, cy)), __fmul_rn(cz, cz))));
}

// one thread per range of kRange faces, each summed sequentially in double.  pass 0: range totals -> base[t];
// pass 1: cdf[f] = base[t] + (running sum of the range up to f), with base[t] the chained prefix of ms_chain_kernel.
// A zero-area face therefore repeats its predecessor's cdf exactly, also across a range boundary (base[t+1] = base[t] + S_t
// is the same rounding as the range's last entry), so the search below never selects it.
__global__ void __launch_bounds__(kBlock) ms_range_kernel(const float* __restrict__ area, long long F, double* __restrict__ base,
                                                          double* __restrict__ cdf, int pass) {
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  const long long f0 = t * kRange;
  if (f0 >= F) return;
  const long long f1 = f0 + kRange < F ? f0 + kRange : F;
  double s = 0.0;
  if (pass == 0) {
    for (long long f = f0; f < f1; ++f) s = __dadd_rn(s, (double)area[f]);
    base[t] = s;
  } else {
    const double b = base[t];
    for (long long f = f0; f < f1; ++f) {
      s = __dadd_rn(s, (double)area[f]);
      cdf[f] = __dadd_rn(b, s);
    }
  }
}

// the range totals -> exclusive prefixes, sequentially (F / kRange entries); base[T] = total.  Total area 0 (or not finite)
// is reported through the error word.
__global__ void ms_chain_kernel(double* base, long long T, int* err) {
  double x = 0.0;
  for (long long t = 0; t < T; ++t) {
    const double s = base[t];
    base[t] = x;
    x = __dadd_rn(x, s);
  }
  base[T] = x;
  if (!(x > 0.0) || !(x <= DBL_MAX)) *(volatile int*)err = 2;
}

__global__ void __launch_bounds__(kBlock) ms_sample_kernel(const float* __restrict__ v, const int* __restrict__ f,
                                                           const double* __restrict__ cdf, long long F,
                                                           const double* __restrict__ total_p, long long n, uint64_t seed,
                                                           float* __restrict__ pts, int* __restrict__ face_idx) {
  const long long k = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (k >= n) return;
  const double total = *total_p;
  if (!(total > 0.0) || !(total <= DBL_MAX)) {          // reported by ms_chain_kernel; nothing is read
    pts[3 * k] = pts[3 * k + 1] = pts[3 * k + 2] = __int_as_float(0x7fc00000);
    if (face_idx) face_idx[k] = -1;
    return;
  }
  const double target = __dmul_rn((double)u01(seed, 3 * (uint64_t)k), total);
  long long lo = 0, hi = F - 1;                          // first face with cdf > target (exists: target < total = cdf[F-1])
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (cdf[mid] > target) hi = mid; else lo = mid + 1;
  }
  const float a = u01(seed, 3 * (uint64_t)k + 1), b = u01(seed, 3 * (uint64_t)k + 2);
  const float r = sqrtf(a);
  const float w0 = __fsub_rn(1.0f, r), w1 = __fmul_rn(r, __fsub_rn(1.0f, b)), w2 = __fmul_rn(r, b);
  const int i0 = f[3 * lo], i1 = f[3 * lo + 1], i2 = f[3 * lo + 2];   // valid: a chosen face has a positive area
#pragma unroll
  for (int c = 0; c < 3; ++c)
    pts[3 * k + c] = __fadd_rn(__fadd_rn(__fmul_rn(w0, v[3 * i0 + c]), __fmul_rn(w1, v[3 * i1 + c])), __fmul_rn(w2, v[3 * i2 + c]));
  if (face_idx) face_idx[k] = (int)lo;
}

// ------------------------------------------------------------------------------------------------ 2. nearest neighbour
// The one squared distance every kernel computes.
__device__ __forceinline__ float nn_dist2(float qx, float qy, float qz, float4 p) {
  const float dx = __fsub_rn(p.x, qx), dy = __fsub_rn(p.y, qy), dz = __fsub_rn(p.z, qz);
  return fmaf(dz, dz, fmaf(dy, dy, __fmul_rn(dx, dx)));
}
__device__ __forceinline__ bool nn_better(float d, int i, float best, int bi) { return d < best || (d == best && i < bi); }

struct NnGrid {
  float lo[3];
  float inv_h;
  int n[3];
  int ncells;
  double hb;                 // 1 / inv_h: the cell edge in coordinates
  int plo[3], phi[3];        // cell box of the indexed points
};

__device__ __forceinline__ int fkey(float x) { const int i = __float_as_int(x); return i >= 0 ? i : i ^ 0x7fffffff; }
__device__ __forceinline__ float fkey_inv(int k) { return __int_as_float(k >= 0 ? k : k ^ 0x7fffffff); }

__device__ __forceinline__ int axis_cell(float x, float lo, float inv_h, int n) {
  const int c = (int)__fmul_rn(__fsub_rn(x, lo), inv_h);    // NaN -> 0, huge -> INT_MAX; clamped below
  return c < 0 ? 0 : (c >= n ? n - 1 : c);
}
__device__ __forceinline__ void cell_of(const NnGrid& g, float x, float y, float z, int c[3]) {
  c[0] = axis_cell(x, g.lo[0], g.inv_h, g.n[0]);
  c[1] = axis_cell(y, g.lo[1], g.inv_h, g.n[1]);
  c[2] = axis_cell(z, g.lo[2], g.inv_h, g.n[2]);
}
__device__ __forceinline__ int cell_id(const NnGrid& g, const int c[3]) { return (c[2] * g.n[1] + c[1]) * g.n[0] + c[0]; }

// bounding box of both sets as order-preserving integer keys (box[0..2] min, box[3..5] max)
__global__ void __launch_bounds__(kBlock) nn_box_kernel(const float* __restrict__ a, long long na, const float* __restrict__ b,
                                                        long long nb, int* box) {
  float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
  for (long long i = (long long)blockIdx.x * kBlock + threadIdx.x; i < na + nb; i += (long long)gridDim.x * kBlock) {
    const float* p = i < na ? a + 3 * i : b + 3 * (i - na);
#pragma unroll
    for (int c = 0; c < 3; ++c) { mn[c] = fminf(mn[c], p[c]); mx[c] = fmaxf(mx[c], p[c]); }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int kmn = __reduce_min_sync(0xffffffffu, fkey(mn[c])), kmx = __reduce_max_sync(0xffffffffu, fkey(mx[c]));
    if ((threadIdx.x & 31) == 0) { atomicMin(box + c, kmn); atomicMax(box + 3 + c, kmx); }
  }
}

// cell size (DESIGN §4.7): h = cbrt(prod_a max(ext_a, L/1024) / T) with L the largest extent and T = target cells
// (about two indexed points per cell), then h >= L/1000 (at most ~1000 cells per axis) and grown by 1.25 until the grid
// has at most `cap` cells.  A box of zero extent is one cell.
__global__ void nn_params_kernel(const int* box, double target, long long cap, NnGrid* g) {
  float lo[3], hi[3];
  double ext[3], L = 0.0;
  for (int a = 0; a < 3; ++a) {
    lo[a] = fkey_inv(box[a]); hi[a] = fkey_inv(box[3 + a]);
    if (!(lo[a] <= hi[a]) || !(fabsf(lo[a]) <= FLT_MAX) || !(fabsf(hi[a]) <= FLT_MAX)) lo[a] = hi[a] = 0.f;   // non-finite input
    ext[a] = (double)hi[a] - (double)lo[a];
    L = fmax(L, ext[a]);
  }
  float inv_h = 1.f;
  int n[3] = {1, 1, 1};
  if (L > 0.0) {
    double e = 1.0;
    for (int a = 0; a < 3; ++a) e *= fmax(ext[a], L / 1024.0);
    double h = fmax(cbrt(e / target), L / 1000.0);
    for (;;) {
      inv_h = (float)(1.0 / h);
      long long tot = 1;
      for (int a = 0; a < 3; ++a) {
        n[a] = (int)__fmul_rn(__fsub_rn(hi[a], lo[a]), inv_h) + 1;     // the cell of `hi` is n-1 (axis_cell's arithmetic)
        tot *= n[a];
      }
      if (tot <= cap) break;
      h *= 1.25;
    }
  }
  for (int a = 0; a < 3; ++a) { g->lo[a] = lo[a]; g->n[a] = n[a]; g->plo[a] = 0x7fffffff; g->phi[a] = -1; }
  g->inv_h = inv_h;
  g->ncells = n[0] * n[1] * n[2];
  g->hb = 1.0 / (double)inv_h;
}

// points per cell (+ the cell box of the indexed set when `track`)
__global__ void __launch_bounds__(kBlock) nn_count_kernel(const float* __restrict__ p, long long n, NnGrid* gp, int* cnt, int track) {
  const NnGrid g = *gp;
  int mn[3] = {0x7fffffff, 0x7fffffff, 0x7fffffff}, mx[3] = {-1, -1, -1};
  for (long long i = (long long)blockIdx.x * kBlock + threadIdx.x; i < n; i += (long long)gridDim.x * kBlock) {
    int c[3];
    cell_of(g, p[3 * i], p[3 * i + 1], p[3 * i + 2], c);
    atomicAdd(cnt + cell_id(g, c), 1);
#pragma unroll
    for (int a = 0; a < 3; ++a) { mn[a] = min(mn[a], c[a]); mx[a] = max(mx[a], c[a]); }
  }
  if (!track) return;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const int kmn = __reduce_min_sync(0xffffffffu, mn[a]), kmx = __reduce_max_sync(0xffffffffu, mx[a]);
    if ((threadIdx.x & 31) == 0) { atomicMin(gp->plo + a, kmn); atomicMax(gp->phi + a, kmx); }
  }
}

// exclusive scan of one value per thread over a block of kScanBlock threads; *total = the block's sum
__device__ __forceinline__ int block_excl_scan(int v, int* s_warp, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_warp[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int w = s_warp[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    s_warp[lane] = w;
  }
  __syncthreads();
  const int r = (wid ? s_warp[wid - 1] : 0) + x - v;
  *total = s_warp[31];
  __syncthreads();
  return r;
}

// three-kernel exclusive scan of cnt[0..n) into start[0..n) (integers: exact in any order)
__global__ void __launch_bounds__(kScanBlock) nn_scan_sums(const int* __restrict__ cnt, long long n, int* __restrict__ blk) {
  __shared__ int s_warp[32];
  const long long i = (long long)blockIdx.x * kScanBlock + threadIdx.x;
  int tot;
  block_excl_scan(i < n ? cnt[i] : 0, s_warp, &tot);
  if (threadIdx.x == 0) blk[blockIdx.x] = tot;
}
__global__ void __launch_bounds__(kScanBlock) nn_scan_blocks(int* blk, int nblk) {
  __shared__ int s_warp[32];
  int carry = 0;
  for (int base = 0; base < nblk; base += kScanBlock) {
    const int l = base + threadIdx.x;
    int tot;
    const int e = block_excl_scan(l < nblk ? blk[l] : 0, s_warp, &tot);
    if (l < nblk) blk[l] = carry + e;
    carry += tot;
  }
}
__global__ void __launch_bounds__(kScanBlock) nn_scan_apply(const int* __restrict__ cnt, long long n, const int* __restrict__ blk,
                                                           int* __restrict__ start) {
  __shared__ int s_warp[32];
  const long long i = (long long)blockIdx.x * kScanBlock + threadIdx.x;
  int tot;
  const int e = block_excl_scan(i < n ? cnt[i] : 0, s_warp, &tot);
  if (i < n) start[i] = blk[blockIdx.x] + e;
}

// into cell order: the points as float4 (w = index bits), or the query indices.  Within a cell the order is the atomics'
// (arbitrary); the search's (distance, index) comparison does not depend on it.
__global__ void __launch_bounds__(kBlock) nn_scatter_kernel(const float* __restrict__ p, long long n, const NnGrid* gp,
                                                            const int* __restrict__ start, int* fill, float4* __restrict__ sp,
                                                            int* __restrict__ order) {
  const NnGrid g = *gp;
  for (long long i = (long long)blockIdx.x * kBlock + threadIdx.x; i < n; i += (long long)gridDim.x * kBlock) {
    const float x = p[3 * i], y = p[3 * i + 1], z = p[3 * i + 2];
    int c[3];
    cell_of(g, x, y, z, c);
    const int id = cell_id(g, c);
    const int pos = start[id] + atomicAdd(fill + id, 1);
    if (sp) sp[pos] = make_float4(x, y, z, __int_as_float((int)i));
    else order[pos] = (int)i;
  }
}

// One thread per query, queries in cell order.  Rings r = r0, r0+1, ... of cells at Chebyshev distance r from the query's
// cell, clipped to the points' cell box (r0: the first ring that meets it).  Stop bound (DESIGN §4.7): a computed cell index
// is within 2^-8 of a cell of the exact one, so a point whose cell is >= r+1 cells from the query's on some axis lies more
// than (r - 2^-7) h from it on that axis, and its computed distance is at least ((r - 2^-7) h)^2 (1 - 2^-20).  When that
// exceeds the best computed distance, no unvisited point can beat or tie it.  Below 2^-100 (float underflow) the walk goes on.
__global__ void __launch_bounds__(kBlock) nn_search_kernel(const float* __restrict__ q, const int* __restrict__ order, long long N,
                                                           const NnGrid* gp, const float4* __restrict__ sp,
                                                           const int* __restrict__ start, float* __restrict__ dist2,
                                                           int* __restrict__ idx) {
  const long long k = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (k >= N) return;
  const NnGrid g = *gp;
  const int qi = order[k];
  const float qx = q[3 * qi], qy = q[3 * qi + 1], qz = q[3 * qi + 2];
  int c[3];
  cell_of(g, qx, qy, qz, c);
  int r0 = 0, r1 = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    r0 = max(r0, max(g.plo[a] - c[a], c[a] - g.phi[a]));
    r1 = max(r1, max(c[a] - g.plo[a], g.phi[a] - c[a]));
  }
  float best = __int_as_float(0x7f800000);
  int bi = 0x7fffffff;
  auto visit = [&](int id0, int id1) {        // the points of cells [id0, id1] (consecutive along x)
    const int e = start[id1 + 1];
    for (int j = start[id0]; j < e; ++j) {
      const float4 p = sp[j];
      const float d = nn_dist2(qx, qy, qz, p);
      const int pi = __float_as_int(p.w);
      if (nn_better(d, pi, best, bi)) { best = d; bi = pi; }
    }
  };
  for (int r = r0; r <= r1; ++r) {
    const int z0 = max(c[2] - r, g.plo[2]), z1 = min(c[2] + r, g.phi[2]);
    const int y0 = max(c[1] - r, g.plo[1]), y1 = min(c[1] + r, g.phi[1]);
    const int x0 = max(c[0] - r, g.plo[0]), x1 = min(c[0] + r, g.phi[0]);
    for (int z = z0; z <= z1; ++z) {
      const bool zr = abs(z - c[2]) == r;
      for (int y = y0; y <= y1; ++y) {
        const int row = (z * g.n[1] + y) * g.n[0];
        if (zr || abs(y - c[1]) == r) {            // a face of the ring's cube: the whole clipped row
          if (x0 <= x1) visit(row + x0, row + x1);
        } else {                                   // inside: the two end cells
          if (c[0] - r >= g.plo[0]) visit(row + c[0] - r, row + c[0] - r);
          if (c[0] + r <= g.phi[0]) visit(row + c[0] + r, row + c[0] + r);
        }
      }
    }
    if (r >= 1 && bi != 0x7fffffff) {
      const double m = ((double)r - 0.0078125) * g.hb;
      const double lb = m * m * (1.0 - 0x1p-20);
      if (lb >= 0x1p-100 && lb > (double)best) break;
    }
  }
  dist2[qi] = best;
  if (idx) idx[qi] = bi;
}

// ------------------------------------------------------------------------------------------------ 3. brute force
__global__ void __launch_bounds__(kBlock) nn_brute_kernel(const float* __restrict__ q, long long N, const float* __restrict__ p,
                                                          long long M, float* __restrict__ dist2, int* __restrict__ idx) {
  __shared__ float4 tile[kBlock];
  const long long k = (long long)blockIdx.x * kBlock + threadIdx.x;
  const bool live = k < N;
  const float qx = live ? q[3 * k] : 0.f, qy = live ? q[3 * k + 1] : 0.f, qz = live ? q[3 * k + 2] : 0.f;
  float best = __int_as_float(0x7f800000);
  int bi = 0x7fffffff;
  for (long long t0 = 0; t0 < M; t0 += kBlock) {
    const long long j = t0 + threadIdx.x;
    tile[threadIdx.x] = j < M ? make_float4(p[3 * j], p[3 * j + 1], p[3 * j + 2], 0.f) : make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    const int m = M - t0 < kBlock ? (int)(M - t0) : kBlock;
    for (int u = 0; u < m; ++u) {
      const float d = nn_dist2(qx, qy, qz, tile[u]);
      if (d < best || (d == best && bi == 0x7fffffff)) { best = d; bi = (int)(t0 + u); }   // index order: the lowest wins ties
    }
    __syncthreads();
  }
  if (live) {
    dist2[k] = best;
    if (idx) idx[k] = bi;
  }
}

// ------------------------------------------------------------------------------------------------ 4. chamfer reduction
// blockIdx.y selects the array; each thread sums a fixed strided subset in double, then a fixed tree: the same bits every run
__global__ void __launch_bounds__(kBlock) nn_sum_kernel(const float* __restrict__ a, long long na, const float* __restrict__ b,
                                                        long long nb, double* __restrict__ partial) {
  __shared__ double s[kBlock];
  const float* x = blockIdx.y ? b : a;
  const long long n = blockIdx.y ? nb : na;
  double acc = 0.0;
  for (long long i = (long long)blockIdx.x * kBlock + threadIdx.x; i < n; i += (long long)kSumBlocks * kBlock)
    acc = __dadd_rn(acc, (double)x[i]);
  s[threadIdx.x] = acc;
  __syncthreads();
  for (int o = kBlock / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) s[threadIdx.x] = __dadd_rn(s[threadIdx.x], s[threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.y * kSumBlocks + blockIdx.x] = s[0];
}
__global__ void __launch_bounds__(kSumBlocks) nn_mean_kernel(const double* __restrict__ partial, long long na, long long nb,
                                                             double* __restrict__ means) {
  __shared__ double s[2][kSumBlocks];
  s[0][threadIdx.x] = partial[threadIdx.x];
  s[1][threadIdx.x] = partial[kSumBlocks + threadIdx.x];
  __syncthreads();
  for (int o = kSumBlocks / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      s[0][threadIdx.x] = __dadd_rn(s[0][threadIdx.x], s[0][threadIdx.x + o]);
      s[1][threadIdx.x] = __dadd_rn(s[1][threadIdx.x], s[1][threadIdx.x + o]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) { means[0] = __ddiv_rn(s[0][0], (double)na); means[1] = __ddiv_rn(s[1][0], (double)nb); }
}

unsigned blocks_for(long long n, int per) { return (unsigned)((n + per - 1) / per); }
unsigned stride_blocks(long long n, int num_sms) {
  const long long b = (n + kBlock - 1) / kBlock, cap = (long long)num_sms * 8;
  return (unsigned)(b < 1 ? 1 : (b > cap ? cap : b));
}

// Workspace of one grid search (all offsets 256-byte aligned)
struct NnWs {
  int* box; NnGrid* grid; int* blk; int* cntP; int* startP; int* cntQ; int* startQ; float4* sp; int* qorder;
  float* d[2]; double* partial;
  long long cells;   // capacity (entries of the cnt / start arrays, one more than the cell cap)
};
long long cell_cap(long long M) {
  const long long T = M / 2 < 1 ? 1 : (M / 2 > (1ll << 20) ? (1ll << 20) : M / 2);
  return 2 * T + 64;
}
// Lays out the workspace of one search of N queries among M points, or (both) of chamfer's two searches with their distance
// arrays, and returns its size; with ws == nullptr only the size is computed.
size_t carve(void* ws, long long N, long long M, bool both, NnWs* w) {
  const long long big = N > M ? N : M, maxM = both ? big : M, maxN = both ? big : N, nd0 = both ? N : 0, nd1 = both ? M : 0;
  const long long cells = cell_cap(maxM) + 1, nblk = (cells + kScanBlock - 1) / kScanBlock;
  const size_t sz[12] = {64, sizeof(NnGrid), (size_t)nblk * 4, (size_t)cells * 4, (size_t)cells * 4, (size_t)cells * 4,
                         (size_t)cells * 4, (size_t)maxM * 16, (size_t)maxN * 4, (size_t)nd0 * 4, (size_t)nd1 * 4,
                         2 * kSumBlocks * sizeof(double)};
  size_t off[12], tot = 0;
  for (int i = 0; i < 12; ++i) { off[i] = tot; tot += align_up(sz[i]); }
  if (!ws) return tot;
  char* b = reinterpret_cast<char*>(ws);
  w->box = reinterpret_cast<int*>(b + off[0]); w->grid = reinterpret_cast<NnGrid*>(b + off[1]);
  w->blk = reinterpret_cast<int*>(b + off[2]); w->cntP = reinterpret_cast<int*>(b + off[3]);
  w->startP = reinterpret_cast<int*>(b + off[4]); w->cntQ = reinterpret_cast<int*>(b + off[5]);
  w->startQ = reinterpret_cast<int*>(b + off[6]); w->sp = reinterpret_cast<float4*>(b + off[7]);
  w->qorder = reinterpret_cast<int*>(b + off[8]); w->d[0] = reinterpret_cast<float*>(b + off[9]);
  w->d[1] = reinterpret_cast<float*>(b + off[10]); w->partial = reinterpret_cast<double*>(b + off[11]);
  w->cells = cells;
  return tot;
}

int scan_cells(const NnWs& w, const int* cnt, int* start, cudaStream_t st) { return exclusive_scan(cnt, w.cells, w.blk, start, st); }

// bounding box of (a, b): the grid every search of one call uses
int box_of(const NnWs& w, const float* a, long long na, const float* b, long long nb, int num_sms, cudaStream_t st,
           int64_t* launches) {
  NM_CUDA(cudaMemsetAsync(w.box, 0x7f, 12, st));
  NM_CUDA(cudaMemsetAsync(w.box + 3, 0x80, 12, st));
  nn_box_kernel<<<stride_blocks(na + nb, num_sms), kBlock, 0, st>>>(a, na, b, nb, w.box);
  NM_CUDA(cudaGetLastError());
  if (launches) *launches += 1;
  return 0;
}

// one search: grid over p (M points, cell size from M), queries q (N), results at the queries' original indices
int search(const NnWs& w, const float* q, long long N, const float* p, long long M, float* dist2, int* idx, int num_sms,
           cudaStream_t st, int64_t* launches) {
  nn_params_kernel<<<1, 1, 0, st>>>(w.box, (double)(M / 2 < 1 ? 1 : M / 2), w.cells - 1, w.grid);
  NM_CUDA(cudaGetLastError());
  NM_CUDA(cudaMemsetAsync(w.cntP, 0, (size_t)w.cells * 4, st));
  NM_CUDA(cudaMemsetAsync(w.cntQ, 0, (size_t)w.cells * 4, st));
  nn_count_kernel<<<stride_blocks(M, num_sms), kBlock, 0, st>>>(p, M, w.grid, w.cntP, 1);
  nn_count_kernel<<<stride_blocks(N, num_sms), kBlock, 0, st>>>(q, N, w.grid, w.cntQ, 0);
  NM_CUDA(cudaGetLastError());
  if (int e = scan_cells(w, w.cntP, w.startP, st)) return e;
  if (int e = scan_cells(w, w.cntQ, w.startQ, st)) return e;
  NM_CUDA(cudaMemsetAsync(w.cntP, 0, (size_t)w.cells * 4, st));
  NM_CUDA(cudaMemsetAsync(w.cntQ, 0, (size_t)w.cells * 4, st));
  nn_scatter_kernel<<<stride_blocks(M, num_sms), kBlock, 0, st>>>(p, M, w.grid, w.startP, w.cntP, w.sp, nullptr);
  nn_scatter_kernel<<<stride_blocks(N, num_sms), kBlock, 0, st>>>(q, N, w.grid, w.startQ, w.cntQ, nullptr, w.qorder);
  nn_search_kernel<<<blocks_for(N, kBlock), kBlock, 0, st>>>(q, w.qorder, N, w.grid, w.sp, w.startP, dist2, idx);
  NM_CUDA(cudaGetLastError());
  if (launches) *launches += 12;
  return 0;
}

}  // namespace

int exclusive_scan(const int* cnt, long long n, int* blk, int* start, cudaStream_t st) {
  const long long nblk = (n + kScanBlock - 1) / kScanBlock;
  nn_scan_sums<<<(unsigned)nblk, kScanBlock, 0, st>>>(cnt, n, blk);
  nn_scan_blocks<<<1, kScanBlock, 0, st>>>(blk, (int)nblk);
  nn_scan_apply<<<(unsigned)nblk, kScanBlock, 0, st>>>(cnt, n, blk, start);
  NM_CUDA(cudaGetLastError());
  return 0;
}

// the surface sampler's workspace: area (F floats) | cdf (F doubles) | base (T+1 doubles), T ranges of kRange faces
struct MsLayout { size_t o_cdf, o_base, bytes; };
static MsLayout ms_layout(long long F) {
  const size_t o_cdf = align_up((size_t)F * 4), o_base = o_cdf + align_up((size_t)F * 8);
  return {o_cdf, o_base, o_base + (size_t)((F + kRange - 1) / kRange + 1) * 8};
}
size_t mesh_sample_ws_bytes(long long F) { return ms_layout(F).bytes; }
size_t nearest_ws_bytes(long long N, long long M, bool chamfer) { return carve(nullptr, N, M, chamfer, nullptr); }

int mesh_sample(const float* verts, long long V, const int32_t* faces, long long F, long long n, uint64_t seed, float* pts,
                int32_t* face_idx, int* d_err, void* ws, size_t ws_bytes, cudaStream_t st, int64_t* launches) {
  const long long T = (F + kRange - 1) / kRange;
  const MsLayout l = ms_layout(F);
  NM_CHECK(ws && ws_bytes >= l.bytes, "mesh sampler: workspace smaller than mesh_sample_ws_bytes");
  char* b = reinterpret_cast<char*>(ws);
  float* area = reinterpret_cast<float*>(b);
  double* cdf = reinterpret_cast<double*>(b + l.o_cdf);
  double* base = reinterpret_cast<double*>(b + l.o_base);
  ms_area_kernel<<<blocks_for(F, kBlock), kBlock, 0, st>>>(verts, V, faces, F, area, d_err);
  ms_range_kernel<<<blocks_for(T, kBlock), kBlock, 0, st>>>(area, F, base, cdf, 0);
  ms_chain_kernel<<<1, 1, 0, st>>>(base, T, d_err);
  ms_range_kernel<<<blocks_for(T, kBlock), kBlock, 0, st>>>(area, F, base, cdf, 1);
  ms_sample_kernel<<<blocks_for(n, kBlock), kBlock, 0, st>>>(verts, faces, cdf, F, base + T, n, seed, pts, face_idx);
  NM_CUDA(cudaGetLastError());
  if (launches) *launches += 5;
  return 0;
}

int nearest(const float* q, long long N, const float* p, long long M, float* dist2, int32_t* idx, void* ws, size_t ws_bytes,
            int num_sms, cudaStream_t st, int64_t* launches) {
  NnWs w{};
  NM_CHECK(ws && ws_bytes >= nearest_ws_bytes(N, M, false), "nearest neighbour: workspace smaller than nearest_ws_bytes");
  carve(ws, N, M, false, &w);
  if (int e = box_of(w, q, N, p, M, num_sms, st, launches)) return e;
  return search(w, q, N, p, M, dist2, idx, num_sms, st, launches);
}

int nearest_brute(const float* q, long long N, const float* p, long long M, float* dist2, int32_t* idx, cudaStream_t st,
                  int64_t* launches) {
  nn_brute_kernel<<<blocks_for(N, kBlock), kBlock, 0, st>>>(q, N, p, M, dist2, idx);
  NM_CUDA(cudaGetLastError());
  if (launches) *launches += 1;
  return 0;
}

int chamfer(const float* x, long long N, const float* y, long long M, double* means, void* ws, size_t ws_bytes, int num_sms,
            cudaStream_t st, int64_t* launches) {
  NnWs w{};
  NM_CHECK(ws && ws_bytes >= nearest_ws_bytes(N, M, true), "chamfer: workspace smaller than nearest_ws_bytes");
  carve(ws, N, M, true, &w);
  if (int e = box_of(w, x, N, y, M, num_sms, st, launches)) return e;
  if (int e = search(w, x, N, y, M, w.d[0], nullptr, num_sms, st, launches)) return e;     // d(x_i, Y)
  if (int e = search(w, y, M, x, N, w.d[1], nullptr, num_sms, st, launches)) return e;     // d(y_j, X)
  nn_sum_kernel<<<dim3(kSumBlocks, 2), kBlock, 0, st>>>(w.d[0], N, w.d[1], M, w.partial);
  nn_mean_kernel<<<1, kSumBlocks, 0, st>>>(w.partial, N, M, means);
  NM_CUDA(cudaGetLastError());
  if (launches) *launches += 2;
  return 0;
}

}  // namespace nm
