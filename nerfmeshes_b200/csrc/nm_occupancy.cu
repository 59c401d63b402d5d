// Occupancy grids for empty-space skipping in the render path (DESIGN §4.15).  One grid per network: G^3 cells over an
// axis-aligned box, one bit per cell, set where the network's own density may be positive.
//   build   occ_corner_kernel     raw occupancy of the cells of a slab of planes from the sigma lattice
//                                 (linspace(lo_a, hi_a, G+1) per axis, nm_grid_sigma's sigma-only sweep): the max of the
//                                 8 corner sigmas > threshold, or a NaN corner
//           occ_dilate_kernel     one axis of the Chebyshev dilation by `dilate` cells (three passes, clamped at the faces)
//           occ_pack_kernel       bit (i*G + j)*G + k of uint32 words
//   render  occ_mark_kernel       per sample of one pass: 1 when the network must evaluate it (outside the box, not finite,
//                                 or in an occupied cell); a skipped sample's raw is (0,0,0,-inf) in the compositor's buffer
//           exclusive_scan        of the marks (the grid search's integer scan, nm_chamfer.cu); one extra zero entry
//                                 leaves the total at the end
//           occ_compact_kernel    the evaluated samples' flat indices, ascending
//           occ_stage_kernel      points o + d*t and directions of a range of the index list, for the IN_POINTS network
//           occ_expand_kernel     the network's (M,4) raw into the evaluated slots of the (R,S,4) buffer the compositor reads
// Built with -fmad=false; the point and the cell index are explicit round-to-nearest operations in any case, so the sample
// points equal fetch_point's IN_RAYS ones (nm_frontend.cuh) bit for bit and tests/_occupancy_ref.py restates the lookup.
#include <math_constants.h>

#include "nm_common.h"

namespace nm {
namespace {

constexpr int kBlock = 256;

unsigned blocks_for(long long n) { return (unsigned)((n + kBlock - 1) / kBlock); }

// a13 / a4: p = o + d*t as a rounded multiply and a rounded add, exactly as fetch_point's IN_RAYS branch
__device__ __forceinline__ void ray_point(const float* __restrict__ origins, int o_stride, const float* __restrict__ dirs,
                                          long long ray, float t, float p[3], float d[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    d[c] = __ldg(dirs + 3 * ray + c);
    const float o = __ldg(origins + (long long)o_stride * ray + c);
    p[c] = __fadd_rn(o, __fmul_rn(d[c], t));
  }
}

__global__ void __launch_bounds__(kBlock) occ_corner_kernel(const float* __restrict__ sigma, int G, int x0, int x1,
                                                             float thr, uint8_t* __restrict__ raw) {
  const long long n1 = G + 1;
  const long long cells = (long long)(x1 - x0) * G * G;
  const long long c = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (c >= cells) return;
  const int k = (int)(c % G), j = (int)((c / G) % G), il = (int)(c / ((long long)G * G));
  bool occ = false;
  float m = -CUDART_INF_F;
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float s = __ldg(sigma + ((il + a) * n1 + (j + b)) * n1 + (k + e));
        occ |= isnan(s);
        m = fmaxf(m, s);
      }
  occ |= m > thr;
  raw[((long long)(x0 + il) * G + j) * G + k] = occ ? 1 : 0;
}

// axis 0: i, 1: j, 2: k.  out[c] = max of in over |s| <= d along the axis, inside [0, G)
__global__ void __launch_bounds__(kBlock) occ_dilate_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int G,
                                                             int axis, int d) {
  const long long n = (long long)G * G * G;
  const long long c = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (c >= n) return;
  const long long stride = axis == 0 ? (long long)G * G : (axis == 1 ? G : 1);
  const int x = (int)((c / stride) % G);
  const int lo = x - d < 0 ? 0 : x - d, hi = x + d > G - 1 ? G - 1 : x + d;
  uint8_t v = 0;
  for (int y = lo; y <= hi && !v; ++y) v = in[c + (long long)(y - x) * stride];
  out[c] = v;
}

__global__ void __launch_bounds__(kBlock) occ_pack_kernel(const uint8_t* __restrict__ cells, long long n, uint32_t* __restrict__ bits) {
  const long long w = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (w * 32 >= n) return;
  uint32_t v = 0;
  for (int b = 0; b < 32; ++b) {
    const long long c = w * 32 + b;
    if (c < n && cells[c]) v |= 1u << b;
  }
  bits[w] = v;
}

__global__ void __launch_bounds__(kBlock) occ_mark_kernel(const OccLookup g, const float* __restrict__ origins, int o_stride,
                                                           const float* __restrict__ dirs, const float* __restrict__ t, long long R,
                                                           int S, int* __restrict__ mark, float4* __restrict__ raw) {
  const long long m = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (m >= R * S) return;
  float p[3], d[3];
  ray_point(origins, o_stride, dirs, m / S, __ldg(t + m), p, d);
  const bool ev = occ_evaluated(g, p);
  mark[m] = ev ? 1 : 0;
  if (!ev) raw[m] = make_float4(0.f, 0.f, 0.f, -CUDART_INF_F);    // sigma + noise stays -inf: alpha = 0 whatever the noise
}

__global__ void __launch_bounds__(kBlock) occ_compact_kernel(const int* __restrict__ mark, const int* __restrict__ pos, long long n,
                                                              int* __restrict__ idx) {
  const long long m = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (m < n && mark[m]) idx[pos[m]] = (int)m;
}

__global__ void __launch_bounds__(kBlock) occ_stage_kernel(const int* __restrict__ idx, long long cnt, int S,
                                                            const float* __restrict__ origins, int o_stride,
                                                            const float* __restrict__ dirs, const float* __restrict__ t,
                                                            float* __restrict__ pts, float* __restrict__ dirs_out) {
  const long long j = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (j >= cnt) return;
  const long long m = idx[j];
  float p[3], d[3];
  ray_point(origins, o_stride, dirs, m / S, __ldg(t + m), p, d);
#pragma unroll
  for (int c = 0; c < 3; ++c) { pts[3 * j + c] = p[c]; dirs_out[3 * j + c] = d[c]; }
}

__global__ void __launch_bounds__(kBlock) occ_expand_kernel(const float4* __restrict__ sub, const int* __restrict__ idx, long long cnt,
                                                             float4* __restrict__ raw) {
  const long long j = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (j < cnt) raw[idx[j]] = sub[j];
}

__global__ void __launch_bounds__(kBlock) occ_query_kernel(const OccLookup g, const float* __restrict__ pts, long long M,
                                                            uint8_t* __restrict__ out) {
  const long long m = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (m >= M) return;
  float p[3] = {__ldg(pts + 3 * m), __ldg(pts + 3 * m + 1), __ldg(pts + 3 * m + 2)};
  out[m] = occ_evaluated(g, p) ? 1 : 0;
}

}  // namespace

int launch_occ_corners(const float* sigma, int G, int x0, int x1, float thr, uint8_t* raw, cudaStream_t st, int64_t* launches) {
  const long long cells = (long long)(x1 - x0) * G * G;
  if (cells <= 0) return 0;
  occ_corner_kernel<<<blocks_for(cells), kBlock, 0, st>>>(sigma, G, x0, x1, thr, raw);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

int launch_occ_dilate_pack(uint8_t* a, uint8_t* b, int G, int d, uint32_t* bits, cudaStream_t st, int64_t* launches) {
  const long long n = (long long)G * G * G;
  if (d > 0) {
    occ_dilate_kernel<<<blocks_for(n), kBlock, 0, st>>>(a, b, G, 2, d);
    occ_dilate_kernel<<<blocks_for(n), kBlock, 0, st>>>(b, a, G, 1, d);
    occ_dilate_kernel<<<blocks_for(n), kBlock, 0, st>>>(a, b, G, 0, d);
    NM_CUDA(cudaGetLastError());
    if (launches) *launches += 3;
    a = b;
  }
  occ_pack_kernel<<<blocks_for((n + 31) / 32), kBlock, 0, st>>>(a, n, bits);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

int occ_compact(const OccLookup& g, const float* origins, int o_stride, const float* dirs, const float* t, long long R, int S,
                int* mark, int* pos, int* blk, int* idx, float* raw, long long* count_host, cudaStream_t st, int64_t* launches) {
  const long long n = R * S;
  occ_mark_kernel<<<blocks_for(n), kBlock, 0, st>>>(g, origins, o_stride, dirs, t, R, S, mark, reinterpret_cast<float4*>(raw));
  NM_CUDA(cudaGetLastError());
  NM_CUDA(cudaMemsetAsync(mark + n, 0, sizeof(int), st));
  if (int e = exclusive_scan(mark, n + 1, blk, pos, st)) return e;
  occ_compact_kernel<<<blocks_for(n), kBlock, 0, st>>>(mark, pos, n, idx);
  NM_CUDA(cudaGetLastError());
  if (launches) *launches += 5;       // mark, the scan's three, compact
  int total = 0;
  NM_CUDA(cudaMemcpyAsync(&total, pos + n, sizeof(int), cudaMemcpyDeviceToHost, st));
  NM_CUDA(cudaStreamSynchronize(st));
  *count_host = total;
  return 0;
}

int launch_occ_stage(const int* idx, long long cnt, int S, const float* origins, int o_stride, const float* dirs, const float* t,
                     float* pts, float* dirs_out, cudaStream_t st, int64_t* launches) {
  if (cnt <= 0) return 0;
  occ_stage_kernel<<<blocks_for(cnt), kBlock, 0, st>>>(idx, cnt, S, origins, o_stride, dirs, t, pts, dirs_out);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

int launch_occ_expand(const float* sub, const int* idx, long long cnt, float* raw, cudaStream_t st, int64_t* launches) {
  if (cnt <= 0) return 0;
  occ_expand_kernel<<<blocks_for(cnt), kBlock, 0, st>>>(reinterpret_cast<const float4*>(sub), idx, cnt,
                                                       reinterpret_cast<float4*>(raw));
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

int launch_occ_query(const OccLookup& g, const float* pts, long long M, uint8_t* out, cudaStream_t st, int64_t* launches) {
  if (M <= 0) return 0;
  occ_query_kernel<<<blocks_for(M), kBlock, 0, st>>>(g, pts, M, out);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

}  // namespace nm
