// The light stages around the fused MLP: ray generation (a1/a2), stratified sampling (a3), sigma->alpha compositing
// (a7), inverse-CDF resampling (a8), AABB-clipped sampling (a10), volume statistics (a14).  All fp32, written op for
// op like the reference (this TU is compiled with -fmad=false so a*b+c stays two roundings, as torch evaluates it).
// Their traffic is ~20 B per sample against ~3.6 MFLOP of tensor work per sample, so they are deliberately simple:
// correctness and the reference's evaluation order matter here, not bandwidth.
#include <math_constants.h>

#include "nm_common.h"
#include "nm_composite.cuh"

namespace nm {
namespace {

// ------------------------------------------------------------------------------------------------ a1 / a2
// get_ray_bundle (src/nerf/nerf_helpers.py:226-277) and ndc_rays (:280-307).
// The fp32 scalars of ndc_rays: its python-double arithmetic on the caller's unrounded focal and near, each result rounded
// once to fp32, as torch rounds a python-scalar operand of an fp32 tensor op.
struct NdcScalars {
  float near, sx, sy, two_near, neg_two_near;
};
NdcScalars ndc_scalars(int H, int W, double focal, double near) {
  return NdcScalars{(float)near, (float)(-1.0 / ((double)W / (2.0 * focal))), (float)(-1.0 / ((double)H / (2.0 * focal))),
                    (float)(2.0 * near), (float)(-2.0 * near)};
}
struct RayGenDev {
  float pose[12];
  int H, W;
  float focal, half_w, half_h;
  int ndc;
  NdcScalars ndc_s;
  int row0;
  long long n;
};
// ndc_rays body (src/nerf/nerf_helpers.py:283-305), op for op: shift the origin to the near plane, then project.  The two
// `2.0 * near / rays_o[..., 2]` terms divide a python scalar by a tensor, which torch evaluates as reciprocal(t) * scalar
// (Tensor.__rtruediv__); every other division is tensor / tensor, a true division.
__device__ __forceinline__ void ndc_warp(const NdcScalars& s, float o[3], float d[3]) {
  const float t = -(s.near + o[2]) / d[2];
  o[0] = o[0] + t * d[0]; o[1] = o[1] + t * d[1]; o[2] = o[2] + t * d[2];
  const float rz = 1.0f / o[2];
  const float o0 = s.sx * o[0] / o[2], o1 = s.sy * o[1] / o[2], o2 = 1.0f + rz * s.two_near;
  const float d0 = s.sx * (d[0] / d[2] - o[0] / o[2]);
  const float d1 = s.sy * (d[1] / d[2] - o[1] / o[2]);
  const float d2 = rz * s.neg_two_near;
  o[0] = o0; o[1] = o1; o[2] = o2;
  d[0] = d0; d[1] = d1; d[2] = d2;
}
// ndc_rays on caller-supplied rays (the positional call of DataBundle.ndc, src/data/data_helpers.py:164-167).
__global__ void ndc_kernel(const NdcScalars s, const float* __restrict__ origins, int o_stride, const float* __restrict__ dirs,
                           long long n, float* __restrict__ out_o, float* __restrict__ out_d) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float o[3], d[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) { o[j] = origins[(long long)o_stride * i + j]; d[j] = dirs[3 * i + j]; }
  ndc_warp(s, o, d);
#pragma unroll
  for (int j = 0; j < 3; ++j) { out_o[3 * i + j] = o[j]; out_d[3 * i + j] = d[j]; }
}
__global__ void raygen_kernel(const __grid_constant__ RayGenDev a, float* __restrict__ origins, float* __restrict__ dirs) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n) return;
  const int c = (int)(i % a.W), r = a.row0 + (int)(i / a.W);
  float x = ((float)c - a.half_w) / a.focal;
  float y = -((float)r - a.half_h) / a.focal;
  float z = -1.0f;
  const float nrm = sqrtf(x * x + y * y + z * z);
  x = x / nrm; y = y / nrm; z = z / nrm;
  float d[3], o[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    d[j] = (x * a.pose[4 * j + 0] + y * a.pose[4 * j + 1]) + z * a.pose[4 * j + 2];
    o[j] = a.pose[4 * j + 3];
  }
  if (a.ndc) ndc_warp(a.ndc_s, o, d);
  dirs[3 * i + 0] = d[0]; dirs[3 * i + 1] = d[1]; dirs[3 * i + 2] = d[2];
  if (origins) { origins[3 * i + 0] = o[0]; origins[3 * i + 1] = o[1]; origins[3 * i + 2] = o[2]; }
}

// ------------------------------------------------------------------------------------------------ a3
// RaySampleInterval.forward (src/nerf/modules.py:157-186).
__global__ void stratified_kernel(const float* __restrict__ s_table, int Nc, long long R, float near0, float far0,
                                  const float* __restrict__ near_dev, const float* __restrict__ far_dev, int lindisp,
                                  int perturb, uint64_t seed, float* __restrict__ t_out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= R * Nc) return;
  const long long ray = idx / Nc;
  const int i = (int)(idx % Nc);
  const float near = near_dev ? near_dev[ray] : near0, far = far_dev ? far_dev[ray] : far0;
  auto at = [&](int k) -> float {
    const float s = s_table[k];
    if (!lindisp) return near * (1.0f - s) + far * s;
    return 1.0f / (1.0f / near * (1.0f - s) + 1.0f / far * s);
  };
  float t = at(i);
  if (perturb) {
    const float lower = (i == 0) ? t : 0.5f * (t + at(i - 1));
    const float upper = (i == Nc - 1) ? t : 0.5f * (at(i + 1) + t);
    t = lower + (upper - lower) * u01(seed, (uint64_t)idx);
  }
  t_out[idx] = t;
}

// ------------------------------------------------------------------------------------------------ a7
// VolumeRenderer.forward (src/nerf/modules.py:67-121).  One thread per ray, samples visited in order so the
// exclusive cumprod (nerf_helpers.py:199-223) is the same sequential product torch.cumprod forms.
__global__ void composite_kernel(const __grid_constant__ CompositeArgs a) {
  const long long ray = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (ray >= a.R) return;
  const int S = a.S;
  const float4* raw = reinterpret_cast<const float4*>(a.raw) + ray * S;
  const float* t = a.t + ray * S;
  const float nrm = comp_ray_norm(a.dirs, ray);
  CompState cs;
  comp_init(cs);
  float tc = t[0];
  for (int i = 0; i < S; ++i) {        // the arithmetic lives in nm_composite.cuh, shared with the fused compositor (nm_mlp_tc.cu)
    const float tn = (i + 1 < S) ? t[i + 1] : 0.f;
    float mk;
    const float w = comp_step(cs, a, ray, i, tc, tn, nrm, raw[i], &mk);
    if (a.weights) a.weights[ray * S + i] = w;
    if (a.mask_weights) a.mask_weights[ray * S + i] = mk;
    tc = tn;
  }
  comp_finish(cs, a, ray);
}

// ------------------------------------------------------------------------------------------------ a8
// SamplePDF.forward (src/nerf/modules.py:197-248).  One warp per ray; everything in shared memory.
constexpr int kMaxCoarse = 256;
constexpr int kMaxTotal = 512;
constexpr int kInvWarps = 4;

__device__ __forceinline__ void warp_bitonic_sort(float* a, int n_pow2, int lane) {
  for (int k = 2; k <= n_pow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < n_pow2; i += 32) {
        const int p = i ^ j;
        if (p > i) {
          const float x = a[i], y = a[p];
          const bool up = ((i & k) == 0);
          if ((x > y) == up) { a[i] = y; a[p] = x; }
        }
      }
      __syncwarp();
    }
  }
}

__global__ void __launch_bounds__(kInvWarps * 32) invcdf_kernel(const float* __restrict__ t_c, const float* __restrict__ w_c,
                                                              const float* __restrict__ u_table, int Nc, int Nf,
                                                              long long R, int perturb, uint64_t seed,
                                                              float* __restrict__ t_f) {
  __shared__ float s_bins[kInvWarps][kMaxCoarse];
  __shared__ float s_cdf[kInvWarps][kMaxCoarse];
  __shared__ float s_all[kInvWarps][2 * kMaxTotal];      // coarse depths, then the new samples padded to a power of two
  __shared__ float s_out[kInvWarps][kMaxTotal];
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long ray = (long long)blockIdx.x * kInvWarps + wid;
  if (ray >= R) return;
  float* bins = s_bins[wid];
  float* cdf = s_cdf[wid];
  float* all = s_all[wid];
  const float* t = t_c + ray * Nc;
  const float* w = w_c + ray * Nc;
  const int nb = Nc - 1;                       // number of bins (mid points)
  const int nw = Nc - 2;                       // weights[..., 1:-1]
  for (int i = lane; i < nb; i += 32) bins[i] = 0.5f * (t[i + 1] + t[i]);
  for (int i = lane; i < Nc; i += 32) all[i] = t[i];
  // pdf = (w + 1e-5) / sum
  float part = 0.f;
  for (int i = lane; i < nw; i += 32) { const float x = w[i + 1] + 1e-5f; cdf[i + 1] = x; part += x; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
  __syncwarp();
  if (lane == 0) {                             // torch.cumsum: sequential fp32 running sum
    float run = 0.f;
    cdf[0] = 0.f;
    for (int i = 1; i <= nw; ++i) { run = run + cdf[i] / part; cdf[i] = run; }
  }
  __syncwarp();
  const int ncdf = nw + 1;                     // == nb
  const int total = Nc + Nf;
  for (int j = lane; j < Nf; j += 32) {
    const float u = perturb ? u01(seed, (uint64_t)(ray * Nf + j)) : u_table[j];
    int lo = 0, hi = ncdf;                     // searchsorted(cdf, u, right=True) = #{cdf <= u}
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (cdf[mid] <= u) lo = mid + 1; else hi = mid; }
    const int below = max(lo - 1, 0), above = min(ncdf - 1, lo);
    const float cb = cdf[below], ca = cdf[above], bb = bins[below], ba = bins[above];
    float denom = ca - cb;
    if (denom < 1e-5f) denom = 1.0f;
    const float tt = (u - cb) / denom;
    all[Nc + j] = bb + tt * (ba - bb);
  }
  __syncwarp();
  // torch.sort(cat(t, samples)) as a merge.  The coarse depths ascend; the new samples ascend too whenever u does (the
  // shipped validation tables; up to a rounding ulp at bin edges) — checked here, and sorted on their own when they do not
  // (training draws u at random).  An element's place in the merged order is its own index plus the number of elements of
  // the other list that come before it; equal values are interchangeable, so the output equals the full sort's bit for bit.
  float* smp = all + Nc;
  bool ok = true;
  for (int j = lane; j + 1 < Nf; j += 32) ok &= !(smp[j] > smp[j + 1]);
  if (!__all_sync(0xffffffffu, ok)) {
    int n2 = 1;
    while (n2 < Nf) n2 <<= 1;
    for (int i = Nf + lane; i < n2; i += 32) smp[i] = CUDART_INF_F;
    __syncwarp();
    warp_bitonic_sort(smp, n2, lane);
  }
  float* outp = s_out[wid];
  for (int i = lane; i < Nc; i += 32) {         // coarse depth i: samples strictly below it come first
    const float x = all[i];
    int lo = 0, hi = Nf;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (smp[mid] < x) lo = mid + 1; else hi = mid; }
    outp[i + lo] = x;
  }
  for (int j = lane; j < Nf; j += 32) {         // sample j: coarse depths <= it come first
    const float x = smp[j];
    int lo = 0, hi = Nc;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (all[mid] <= x) lo = mid + 1; else hi = mid; }
    outp[j + lo] = x;
  }
  __syncwarp();
  for (int i = lane; i < total; i += 32) t_f[ray * total + i] = outp[i];
}

// ------------------------------------------------------------------------------------------------ a10
// TreeSampling.batch_ray_voxel_intersect, deterministic branch (src/nerf/tree.py:215-343), + the miss fallback of
// BuFFModel.forward (src/models/model_buff.py:53).  One warp per ray, voxel list streamed from global (L1/L2-resident:
// 1533 x 24 B), hit list / prefix sums / samples in shared memory.
constexpr int kMaxHits = 512;
constexpr int kAabbWarps = 4;

__device__ __forceinline__ void warp_bitonic_sort_tagged(float* key, int* tag, int n_pow2, int lane) {
  for (int k = 2; k <= n_pow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < n_pow2; i += 32) {
        const int p = i ^ j;
        if (p > i) {
          const float x = key[i], y = key[p];
          const bool up = ((i & k) == 0);
          if ((x > y) == up) {
            key[i] = y; key[p] = x;
            const int tx = tag[i]; tag[i] = tag[p]; tag[p] = tx;
          }
        }
      }
      __syncwarp();
    }
  }
}

__device__ __forceinline__ void warp_bitonic_sort_triples(float* key, float* val, int* tag, int n_pow2, int lane) {
  for (int k = 2; k <= n_pow2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = lane; i < n_pow2; i += 32) {
        const int p = i ^ j;
        if (p > i) {
          const float x = key[i], y = key[p];
          const bool up = ((i & k) == 0);
          if ((x > y) == up) {
            key[i] = y; key[p] = x;
            const float vx = val[i]; val[i] = val[p]; val[p] = vx;
            const int tx = tag[i]; tag[i] = tag[p]; tag[p] = tx;
          }
        }
      }
      __syncwarp();
    }
  }
}

__global__ void __launch_bounds__(kAabbWarps * 32) aabb_kernel(const float* __restrict__ voxels, int V,
                                                              const float* __restrict__ origins, int o_stride,
                                                              const float* __restrict__ dirs, long long R, float near,
                                                              float far, int S, const float* __restrict__ s_table,
                                                              const float* __restrict__ t_uniform,
                                                              float* __restrict__ z_out, int* __restrict__ idx_out,
                                                              int* __restrict__ overflow, int random, uint64_t seed) {
  __shared__ int s_vox[kAabbWarps][kMaxHits];
  __shared__ float s_lo[kAabbWarps][kMaxHits];
  __shared__ float s_hi[kAabbWarps][kMaxHits];
  __shared__ float s_z[kAabbWarps][kMaxTotal];
  __shared__ int s_bucket[kAabbWarps][kMaxTotal];
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long ray = (long long)blockIdx.x * kAabbWarps + wid;
  if (ray >= R) return;
  float* lo = s_lo[wid];
  float* hi = s_hi[wid];
  float* z = s_z[wid];
  int* bucket = s_bucket[wid];
  int* vox = s_vox[wid];
  float o[3], inv[3];
  bool neg[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    o[c] = origins[(long long)o_stride * ray + c];
    inv[c] = 1.0f / dirs[3 * ray + c];
    neg[c] = inv[c] < 0.f;
  }
  int H = 0;
  for (int v0 = 0; v0 < V; v0 += 32) {
    const int v = v0 + lane;
    bool hit = false;
    float tmin = 0.f, tmax = 0.f;
    if (v < V) {
      float tlo[3], thi[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float vmin = voxels[6 * v + c], vmax = voxels[6 * v + 3 + c];
        tlo[c] = ((neg[c] ? vmax : vmin) - o[c]) * inv[c];
        thi[c] = ((neg[c] ? vmin : vmax) - o[c]) * inv[c];
      }
      tmin = tlo[0]; tmax = thi[0];
      hit = (tmin <= thi[1]) && (tlo[1] <= tmax);
      if (tlo[1] > tmin) tmin = tlo[1];
      if (thi[1] < tmax) tmax = thi[1];
      hit = hit && (tmin <= thi[2]) && (tlo[2] <= tmax);
      if (tlo[2] > tmin) tmin = tlo[2];
      if (thi[2] < tmax) tmax = thi[2];
      hit = hit && (tmin >= near) && (tmax <= far);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, hit);
    if (hit) {
      const int pos = H + __popc(bal & ((1u << lane) - 1));
      if (pos < kMaxHits) { lo[pos] = tmin; hi[pos] = tmax; vox[pos] = v; }
    }
    H += __popc(bal);
  }
  if (H > kMaxHits) { if (lane == 0) atomicExch(overflow, 1); H = kMaxHits; }
  __syncwarp();
  if (H == 0) {                                 // miss: uniform fallback samples, no voxel
    for (int k = lane; k < S; k += 32) {
      if (z_out) z_out[ray * S + k] = t_uniform[ray * S + k];
      if (idx_out) idx_out[ray * S + k] = -1;
    }
    return;
  }
  if (random) {
    // cfg.tree.use_random_sampling (tree.py:280-297): S draws with replacement from a multinomial that weighs every hit voxel 1
    // (and every miss 1e-12: a 1e-9-probability event per draw that would sample a non-intersection's garbage interval —
    // not reproduced), each placed uniformly inside its voxel's [entry, exit]; then the common sort below.  Distributional
    // parity only: torch's generator stream cannot be matched.  `seed` is the draws' own stream (kVoxelSalt, nm_api.cu).
    for (int k = lane; k < S; k += 32) {
      const uint64_t c = (uint64_t)(ray * S + k);
      const int h = min((int)(u01(seed, 2 * c) * (float)H), H - 1);
      z[k] = lo[h] + (hi[h] - lo[h]) * u01(seed, 2 * c + 1);
      bucket[k] = vox[h];
    }
    __syncwarp();
    int m2 = 1;
    while (m2 < S) m2 <<= 1;
    for (int i = S + lane; i < m2; i += 32) { z[i] = CUDART_INF_F; bucket[i] = -1; }
    __syncwarp();
    warp_bitonic_sort_tagged(z, bucket, m2, lane);
    for (int k = lane; k < S; k += 32) {
      if (z_out) z_out[ray * S + k] = z[k];
      if (idx_out) idx_out[ray * S + k] = bucket[k];
    }
    return;
  }
  int n2 = 1;
  while (n2 < H) n2 <<= 1;
  for (int i = H + lane; i < n2; i += 32) { lo[i] = CUDART_INF_F; hi[i] = CUDART_INF_F; vox[i] = -1; }
  __syncwarp();
  warp_bitonic_sort_triples(lo, hi, vox, n2, lane);   // hits by entry distance, voxel ids riding along
  // running sum of the interval lengths (torch.cumsum, sequential), kept in hi[]
  if (lane == 0) {
    float run = 0.f;
    for (int i = 0; i < H; ++i) { run = run + (hi[i] - lo[i]); hi[i] = run; }
  }
  __syncwarp();
  const float total = hi[H - 1];
  for (int k = lane; k < S; k += 32) {
    const float s = s_table[k] * total;
    int a = 0, b = H;                           // searchsorted(cums, s) left = #{cums < s}
    while (a < b) { const int mid = (a + b) >> 1; if (hi[mid] < s) a = mid + 1; else b = mid; }
    bucket[k] = min(a, H - 1);
  }
  __syncwarp();
  for (int k = lane; k < S; k += 32) {
    const int bk = bucket[k];
    int a = 0, b = k;                           // first sample index that falls in the same bucket
    while (a < b) { const int mid = (a + b) >> 1; if (bucket[mid] < bk) a = mid + 1; else b = mid; }
    z[k] = lo[bk] + (s_table[k] * total - s_table[a] * total);
  }
  __syncwarp();
  for (int k = lane; k < S; k += 32) bucket[k] = vox[bucket[k]];      // sample -> voxel id (tree.py:333-335)
  // (:338-341) sort the samples, ids following.  Leaf boxes do not overlap, so the buckets' intervals are disjoint and the
  // samples already ascend (up to a rounding ulp at a bucket edge): the sort network only runs for a ray where they do not.
  bool asc = true;
  for (int k = lane; k + 1 < S; k += 32) asc &= !(z[k] > z[k + 1]);
  if (!__all_sync(0xffffffffu, asc)) {
    int m2 = 1;
    while (m2 < S) m2 <<= 1;
    for (int i = S + lane; i < m2; i += 32) { z[i] = CUDART_INF_F; bucket[i] = -1; }
    __syncwarp();
    warp_bitonic_sort_tagged(z, bucket, m2, lane);
  }
  for (int k = lane; k < S; k += 32) {
    if (z_out) z_out[ray * S + k] = z[k];
    if (idx_out) idx_out[ray * S + k] = bucket[k];
  }
}

// ------------------------------------------------------------------------------------------------ BuFF tree maintenance
// TreeSampling.ray_batch_integration (src/nerf/tree.py:177-206): per-voxel sums of the sample weights / weight masks
// that fell into it (idx < 0: ray without a hit, skipped), then memm[v] += (acc/freq - memm[v]) / counter where freq > 0.
// The reference materialises two dense (R,V) matrices; here a block-level shared-memory histogram feeds fp32 atomics.
__global__ void __launch_bounds__(256) tree_scatter_kernel(const int* __restrict__ idx, const float* __restrict__ w,
                                                           const float* __restrict__ mw, long long n, int V, int use_smem,
                                                           float* __restrict__ acc, float* __restrict__ freq) {
  extern __shared__ float sh[];
  float* a = use_smem ? sh : acc;
  float* f = use_smem ? sh + V : freq;
  if (use_smem) {
    for (int i = threadIdx.x; i < 2 * V; i += blockDim.x) sh[i] = 0.f;
    __syncthreads();
  }
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int v = idx[i];
    if (v >= 0 && v < V) {
      atomicAdd(a + v, w[i]);
      atomicAdd(f + v, mw[i]);
    }
  }
  if (use_smem) {
    __syncthreads();
    for (int i = threadIdx.x; i < V; i += blockDim.x) {
      if (sh[V + i] != 0.f || sh[i] != 0.f) { atomicAdd(acc + i, sh[i]); atomicAdd(freq + i, sh[V + i]); }
    }
  }
}

__global__ void tree_update_kernel(float* __restrict__ memm, const float* __restrict__ acc, const float* __restrict__ freq,
                                   int V, float counter) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const float fr = freq[v];
  if (fr > 0.f) memm[v] = memm[v] + (acc[v] / fr - memm[v]) / counter;
}

// ------------------------------------------------------------------------------------------------ a14
__global__ void stats_pass1(const float* __restrict__ v, long long n, double* __restrict__ acc /*[min,max,sum]*/) {
  float mn = CUDART_INF_F, mx = -CUDART_INF_F;
  double s = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float x = v[i];
    mn = fminf(mn, x); mx = fmaxf(mx, x); s += (double)x;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    s += __shfl_xor_sync(0xffffffffu, s, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(acc + 2, s);
    // float min/max through ordered-int atomics on the double slots' low words would be obscure; use CAS on doubles
    unsigned long long* pmn = reinterpret_cast<unsigned long long*>(acc);
    unsigned long long old = *pmn, assumed;
    do { assumed = old; if (__longlong_as_double(assumed) <= (double)mn) break;
         old = atomicCAS(pmn, assumed, __double_as_longlong((double)mn)); } while (assumed != old);
    unsigned long long* pmx = reinterpret_cast<unsigned long long*>(acc + 1);
    old = *pmx;
    do { assumed = old; if (__longlong_as_double(assumed) >= (double)mx) break;
         old = atomicCAS(pmx, assumed, __double_as_longlong((double)mx)); } while (assumed != old);
  }
}
__global__ void stats_init(double* __restrict__ acc) {
  acc[0] = 1e300; acc[1] = -1e300; acc[2] = 0.0; acc[3] = 0.0;
}
__global__ void stats_pass2(const float* __restrict__ v, long long n, double mean_val, const double* __restrict__ mean_dev,
                            double* __restrict__ acc) {
  const double mean = mean_dev ? *mean_dev : mean_val;
  double s = 0.0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double d = (double)v[i] - mean;
    s += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(acc + 3, s);
}

}  // namespace

int launch_raygen(const RayGenArgs& a, float* origins, float* dirs, cudaStream_t st, int64_t* launches) {
  RayGenDev d{};
  for (int i = 0; i < 12; ++i) d.pose[i] = a.pose[i];
  d.H = a.H; d.W = a.W;
  d.focal = (float)a.focal;                          // (cols - W * 0.5) / focal: torch divides by the scalar rounded to fp32
  d.half_w = (float)(a.W * 0.5); d.half_h = (float)(a.H * 0.5);
  d.ndc = a.ndc;
  d.ndc_s = ndc_scalars(a.H, a.W, a.focal, a.ndc_near);
  d.row0 = a.row0;
  d.n = (long long)(a.row1 - a.row0) * a.W;
  if (d.n <= 0) return 0;
  raygen_kernel<<<(unsigned)((d.n + 255) / 256), 256, 0, st>>>(d, origins, dirs);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

int launch_ndc(int H, int W, double focal, double near, const float* origins, int o_stride, const float* dirs, long long n,
               float* out_o, float* out_d, cudaStream_t st, int64_t* launches) {
  if (n <= 0) return 0;
  ndc_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ndc_scalars(H, W, focal, near), origins, o_stride, dirs, n, out_o,
                                                          out_d);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

int launch_stratified(const float* s_table, int Nc, long long R, const float* near_far2, const float* near_dev,
                      const float* far_dev, int lindisp, int perturb, uint64_t seed, float* t_out, cudaStream_t st,
                      int64_t* launches) {
  const long long n = R * Nc;
  if (n <= 0) return 0;
  stratified_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(s_table, Nc, R, near_far2 ? near_far2[0] : 0.f,
                                                                 near_far2 ? near_far2[1] : 0.f, near_dev, far_dev,
                                                                 lindisp, perturb, seed, t_out);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

int launch_composite(const CompositeArgs& a, cudaStream_t st, int64_t* launches) {
  if (a.R <= 0) return 0;
  composite_kernel<<<(unsigned)((a.R + 127) / 128), 128, 0, st>>>(a);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

int launch_invcdf(const float* t_c, const float* w_c, const float* u_table, int Nc, int Nf, long long R, int perturb,
                  uint64_t seed, float* t_f, cudaStream_t st, int64_t* launches) {
  NM_CHECK(Nc >= 3 && Nc <= kMaxCoarse && Nc + Nf <= kMaxTotal, "sample counts (%d,%d) exceed the resampler limits", Nc, Nf);
  if (R <= 0) return 0;
  invcdf_kernel<<<(unsigned)((R + kInvWarps - 1) / kInvWarps), kInvWarps * 32, 0, st>>>(t_c, w_c, u_table, Nc, Nf, R,
                                                                                       perturb, seed, t_f);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

int launch_aabb(const float* voxels, int V, const float* origins, int o_stride, const float* dirs, long long R,
                     float near, float far, int S, const float* s_table, const float* t_uniform, float* z_out, int* idx_out,
                     int* d_overflow, cudaStream_t st, int64_t* launches, int random, uint64_t seed) {
  NM_CHECK(S <= kMaxTotal, "sample count %d exceeds the AABB sampler limit", S);
  NM_CHECK(z_out == nullptr || t_uniform != nullptr, "z output needs the uniform fallback samples");
  if (R <= 0) return 0;
  aabb_kernel<<<(unsigned)((R + kAabbWarps - 1) / kAabbWarps), kAabbWarps * 32, 0, st>>>(
      voxels, V, origins, o_stride, dirs, R, near, far, S, s_table, t_uniform, z_out, idx_out, d_overflow, random, seed);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

int launch_tree_integrate(const int* idx, const float* w, const float* mw, long long n, float* memm, int V, int counter,
                          float* scratch2v, cudaStream_t st, int64_t* launches) {
  NM_CHECK(counter >= 1, "counter must be >= 1");
  if (n <= 0 || V <= 0) return 0;
  NM_CUDA(cudaMemsetAsync(scratch2v, 0, sizeof(float) * 2 * (size_t)V, st));
  const int use_smem = V <= 6144;
  long long blocks = (n + 256 * 16 - 1) / (256 * 16);
  if (blocks > 1184) blocks = 1184;
  if (blocks < 1) blocks = 1;
  tree_scatter_kernel<<<(unsigned)blocks, 256, use_smem ? sizeof(float) * 2 * (size_t)V : 0, st>>>(idx, w, mw, n, V, use_smem,
                                                                                                  scratch2v, scratch2v + V);
  NM_CUDA(cudaGetLastError());
  tree_update_kernel<<<(V + 255) / 256, 256, 0, st>>>(memm, scratch2v, scratch2v + V, V, (float)counter);
  NM_CUDA(cudaGetLastError());
  if (launches) *launches += 2;
  return 0;
}

int launch_volume_stats(const float* vol, long long n, double* d_scratch, float* out_host, cudaStream_t st,
                        int64_t* launches) {
  NM_CHECK(n > 0, "empty volume");
  const double init[4] = {1e300, -1e300, 0.0, 0.0};
  NM_CUDA(cudaMemcpyAsync(d_scratch, init, sizeof(init), cudaMemcpyHostToDevice, st));
  stats_pass1<<<1184, 256, 0, st>>>(vol, n, d_scratch);
  NM_CUDA(cudaGetLastError());
  double h[4];
  NM_CUDA(cudaMemcpyAsync(h, d_scratch, sizeof(h), cudaMemcpyDeviceToHost, st));
  NM_CUDA(cudaStreamSynchronize(st));
  const double mean = h[2] / (double)n;
  stats_pass2<<<1184, 256, 0, st>>>(vol, n, mean, nullptr, d_scratch);
  NM_CUDA(cudaGetLastError());
  NM_CUDA(cudaMemcpyAsync(h, d_scratch, sizeof(h), cudaMemcpyDeviceToHost, st));
  NM_CUDA(cudaStreamSynchronize(st));
  out_host[0] = (float)h[0];
  out_host[1] = (float)h[1];
  out_host[2] = (float)sqrt(h[3] / (double)n);   // numpy .std(): population std (ddof=0)
  if (launches) *launches += 2;
  return 0;
}

// asynchronous halves of the same statistics for sharded volumes: pass 1 -> out[0..2] = {min, max, sum} (doubles),
// pass 2 -> out[3] = sum (x - *mean_dev)^2; the caller reduces across shards between the passes (device tensors, no sync)
int launch_volume_stats_pass(const float* vol, long long n, int pass, const double* mean_dev, double* out_dev, cudaStream_t st,
                             int64_t* launches) {
  NM_CHECK(n > 0 && (pass == 1 || pass == 2), "bad arguments");
  if (pass == 1) {
    stats_init<<<1, 1, 0, st>>>(out_dev);
    stats_pass1<<<1184, 256, 0, st>>>(vol, n, out_dev);
  } else {
    NM_CHECK(mean_dev != nullptr, "pass 2 needs the mean");
    stats_pass2<<<1184, 256, 0, st>>>(vol, n, 0.0, mean_dev, out_dev);
  }
  NM_CUDA(cudaGetLastError());
  if (launches) *launches += pass == 1 ? 2 : 1;
  return 0;
}

}  // namespace nm
