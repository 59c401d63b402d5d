// Texture bake of a mesh's appearance (DESIGN §4.12; no reference counterpart: the reference colours vertices,
// src/mesh_nerf.py:160-192).  One right-triangle patch of N(N+1)/2 texels per face, two faces per square cell of
// C = N + 2 texels; every texel is one appearance query built like a vertex's.
//   1. tex_first_ref_kernel   vfirst[v] = min over the corners (f, k) that reference v of 3f + k (integer atomicMin: exact);
//                             a face index outside [0, V) sets the error word (code 5) and nothing else is launched
//   2. tex_unref_kernel + exclusive_scan + tex_unref_list_kernel   the vertices no face references, in ascending order
//   3. per chunk of faces: tex_rays_kernel (texel -> ray), the caller's render, tex_scatter_kernel (rgb -> atlas pixel, and
//      the corner texel named by vfirst -> vertex colour)
//   4. per chunk of unreferenced vertices: tex_vertex_rays_kernel, render, tex_vertex_scatter_kernel
//   5. tex_ring_kernel (each face's ring: mean of its in-triangle 4-neighbours), tex_quantise_kernel, tex_uv_kernel
// Built with -fmad=false: every position, normal and ray is the fp32 arithmetic in the written order, which
// tests/_texture_ref.py restates bit for bit.  Every texel depends on its face alone, so the chunking changes no bit.
#include <cmath>

#include "nm_common.h"
#include "nm_texture.cuh"

namespace nm {
namespace {

constexpr int kBlock = 256;
constexpr int kErrBadFace = 5;        // codes 1-4 of the same word belong to the sampler, components and decimation
constexpr int kNoRef = 0x7f7f7f7f;    // vfirst of a vertex no face references (memset byte 0x7f; 3F is far below it)

unsigned blocks_for(long long n) { return (unsigned)((n + kBlock - 1) / kBlock); }
size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

// local texel index r in [0, K) -> (i, j): row j holds N - j texels
__device__ __forceinline__ void texel_ij(int r, int N, int* i, int* j) {
  int jj = 0;
  while (r >= N - jj) { r -= N - jj; ++jj; }
  *i = r; *j = jj;
}

// corner k of the patch, or -1: (0,0), (N-1,0), (0,N-1)
__device__ __forceinline__ int texel_corner(int i, int j, int N) {
  return (i == 0 && j == 0) ? 0 : (j == 0 && i == N - 1) ? 1 : (i == 0 && j == N - 1) ? 2 : -1;
}

// the appearance query of mesh_appearance at point p with unit normal n: d = -n; mode 0 the ray origin p - c*d, mode 1 p
__device__ __forceinline__ void store_query(const float p[3], const float n[3], int mode, float c, float* a, float* d) {
  for (int k = 0; k < 3; ++k) {
    const float dk = -n[k];
    d[k] = dk;
    a[k] = mode == 0 ? p[k] - c * dk : p[k];
  }
}

__global__ void __launch_bounds__(kBlock) tex_first_ref_kernel(const int* __restrict__ faces, long long F, long long V,
                                                               int* vfirst, int* err) {
  const long long c = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (c >= 3 * F) return;
  const int v = faces[c];
  if (v < 0 || v >= V) { *err = kErrBadFace; return; }
  atomicMin(vfirst + v, (int)c);
}

__global__ void __launch_bounds__(kBlock) tex_unref_kernel(const int* __restrict__ vfirst, long long V, int* __restrict__ flag) {
  const long long v = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (v <= V) flag[v] = (v < V && vfirst[v] == kNoRef) ? 1 : 0;
}

__global__ void __launch_bounds__(kBlock) tex_unref_list_kernel(const int* __restrict__ flag, const int* __restrict__ start,
                                                                long long V, int* __restrict__ list) {
  const long long v = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (v < V && flag[v]) list[start[v]] = (int)v;
}

// texels [f0*K, f0*K + n) -> (a, d) rows [0, n) and their atlas pixels (x, y)
__global__ void __launch_bounds__(kBlock) tex_rays_kernel(const float* __restrict__ verts, const float* __restrict__ normals,
                                                          long long V, const int* __restrict__ faces, long long f0, long long n,
                                                          TexLayout L, int mode, float c, float* __restrict__ a_out,
                                                          float* __restrict__ d_out, int* __restrict__ xy_out, int* err) {
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (t >= n) return;
  const long long f = f0 + t / L.K;
  int i, j;
  texel_ij((int)(t % L.K), L.N, &i, &j);
  if (xy_out) {
    const long long px = texel_pixel(f, i, j, L);
    xy_out[2 * t] = (int)(px % L.W);
    xy_out[2 * t + 1] = (int)(px / L.W);
  }
  int vi[3];
  for (int k = 0; k < 3; ++k) {
    vi[k] = faces[3 * f + k];
    if (vi[k] < 0 || vi[k] >= V) {
      *err = kErrBadFace;
      for (int q = 0; q < 3; ++q) { a_out[3 * t + q] = 0.f; d_out[3 * t + q] = 0.f; }
      return;
    }
  }
  float p[3], nn[3];
  const int corner = texel_corner(i, j, L.N);
  if (corner >= 0) {                  // corner texels are the vertex's own query, bit for bit
    const long long v = corner == 0 ? vi[0] : corner == 1 ? vi[1] : vi[2];
    for (int q = 0; q < 3; ++q) { p[q] = verts[3 * v + q]; nn[q] = normals[3 * v + q]; }
  } else {
    const float w1 = (float)i / (float)(L.N - 1), w2 = (float)j / (float)(L.N - 1);
    const float w0 = (1.0f - w1) - w2;
    float m[3];
    for (int q = 0; q < 3; ++q) {
      p[q] = (w0 * verts[3 * vi[0] + q] + w1 * verts[3 * vi[1] + q]) + w2 * verts[3 * vi[2] + q];
      m[q] = (w0 * normals[3 * vi[0] + q] + w1 * normals[3 * vi[1] + q]) + w2 * normals[3 * vi[2] + q];
    }
    const float len = sqrtf((m[0] * m[0] + m[1] * m[1]) + m[2] * m[2]);
    if (len > 0.f && isfinite(len)) {
      for (int q = 0; q < 3; ++q) nn[q] = m[q] / len;
    } else {                          // the corner of largest weight, the lowest on ties
      const long long v = (w0 >= w1 && w0 >= w2) ? vi[0] : (w1 >= w2 ? vi[1] : vi[2]);
      for (int q = 0; q < 3; ++q) nn[q] = normals[3 * v + q];
    }
  }
  store_query(p, nn, mode, c, a_out + 3 * t, d_out + 3 * t);
}

__global__ void __launch_bounds__(kBlock) tex_scatter_kernel(const int* __restrict__ faces, const int* __restrict__ vfirst,
                                                             long long f0, long long n, TexLayout L, const float* __restrict__ rgb,
                                                             int stride, float* __restrict__ atlas, float* __restrict__ vertex_rgb) {
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (t >= n) return;
  const long long f = f0 + t / L.K;
  int i, j;
  texel_ij((int)(t % L.K), L.N, &i, &j);
  const long long px = texel_pixel(f, i, j, L);
  const float* c = rgb + (long long)stride * t;
  for (int q = 0; q < 3; ++q) atlas[3 * px + q] = c[q];
  const int corner = texel_corner(i, j, L.N);
  if (corner >= 0) {
    const int v = faces[3 * f + corner];
    if (vfirst[v] == (int)(3 * f + corner))
      for (int q = 0; q < 3; ++q) vertex_rgb[3 * (long long)v + q] = c[q];
  }
}

__global__ void __launch_bounds__(kBlock) tex_vertex_rays_kernel(const float* __restrict__ verts, const float* __restrict__ normals,
                                                                 const int* __restrict__ list, long long n, int mode, float c,
                                                                 float* __restrict__ a_out, float* __restrict__ d_out) {
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (t >= n) return;
  const long long v = list[t];
  float p[3], nn[3];
  for (int q = 0; q < 3; ++q) { p[q] = verts[3 * v + q]; nn[q] = normals[3 * v + q]; }
  store_query(p, nn, mode, c, a_out + 3 * t, d_out + 3 * t);
}

__global__ void __launch_bounds__(kBlock) tex_vertex_scatter_kernel(const int* __restrict__ list, long long n,
                                                                    const float* __restrict__ rgb, int stride,
                                                                    float* __restrict__ vertex_rgb) {
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (t >= n) return;
  const long long v = list[t];
  for (int q = 0; q < 3; ++q) vertex_rgb[3 * v + q] = rgb[(long long)stride * t + q];
}

// ring texel (i, N - i), i in [0, N], of face f: the mean of its in-triangle 4-neighbours (i-1, j) and (i, j-1), where they
// exist.  Reads triangle texels only and writes ring texels only, which no triangle or other ring shares.
__global__ void __launch_bounds__(kBlock) tex_ring_kernel(long long F, TexLayout L, float* __restrict__ atlas) {
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (t >= F * (L.N + 1)) return;
  const long long f = t / (L.N + 1);
  const int i = (int)(t % (L.N + 1)), j = L.N - i;
  const long long px = texel_pixel(f, i, j, L);
  const float* a = i > 0 ? atlas + 3 * texel_pixel(f, i - 1, j, L) : nullptr;
  const float* b = j > 0 ? atlas + 3 * texel_pixel(f, i, j - 1, L) : nullptr;
  for (int q = 0; q < 3; ++q) atlas[3 * px + q] = (a && b) ? (a[q] + b[q]) * 0.5f : (a ? a[q] : b[q]);
}

__global__ void __launch_bounds__(kBlock) tex_quantise_kernel(const float* __restrict__ atlas, long long n, uint8_t* __restrict__ u8) {
  const long long k = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (k < n) u8[k] = (uint8_t)floorf(fminf(fmaxf(atlas[k], 0.f), 1.f) * 255.f + 0.5f);
}

// uv of corner k of face f: the centre of its corner texel, v measured from the bottom row
__global__ void __launch_bounds__(kBlock) tex_uv_kernel(long long F, TexLayout L, long long H, float* __restrict__ uv) {
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (t >= 3 * F) return;
  const int k = (int)(t % 3);
  const long long px = texel_pixel(t / 3, k == 1 ? L.N - 1 : 0, k == 2 ? L.N - 1 : 0, L);
  uv[2 * t] = ((float)(px % L.W) + 0.5f) / (float)L.W;
  uv[2 * t + 1] = 1.0f - ((float)(px / L.W) + 0.5f) / (float)H;
}

TexLayout bake_layout(const TextureBake& b) {
  TexLayout L{};
  nm::tex_layout(b.F, b.N, &L);
  return L;
}

// rays per chunk: whole faces of chunk_texels texels (at least one face), no more than the mesh needs
long long chunk_rays(const TextureBake& b) {
  const long long K = (long long)b.N * (b.N + 1) / 2;
  const long long faces = b.chunk_texels / K > 0 ? b.chunk_texels / K : 1;
  const long long need = b.F * K > b.V ? b.F * K : b.V;
  return faces * K < need ? faces * K : need;
}

struct TexWs {
  int *vfirst, *flag, *start, *blk, *list, *small;
  float *a, *d, *rgb;
};

TexWs carve(const TextureBake& b, void* ws) {
  const long long V = b.V, R = chunk_rays(b);
  char* p = static_cast<char*>(ws);
  TexWs w;
  auto take = [&](size_t bytes) { char* q = p; p += align_up(bytes); return q; };
  w.vfirst = reinterpret_cast<int*>(take((size_t)V * 4));
  w.flag = reinterpret_cast<int*>(take((size_t)(V + 1) * 4));
  w.start = reinterpret_cast<int*>(take((size_t)(V + 1) * 4));
  w.blk = reinterpret_cast<int*>(take((size_t)((V + 1 + kScanBlockEntries - 1) / kScanBlockEntries) * 4));
  w.list = reinterpret_cast<int*>(take((size_t)V * 4));
  w.small = reinterpret_cast<int*>(take(16));
  w.a = reinterpret_cast<float*>(take((size_t)R * 12));
  w.d = reinterpret_cast<float*>(take((size_t)R * 12));
  w.rgb = reinterpret_cast<float*>(take((size_t)R * 16));
  return w;
}

}  // namespace

int texture_layout(long long F, int N, long long out[4]) {
  NM_CHECK(N >= kTexMinN && N <= kTexMaxN, "texture bake: texels per triangle leg N = %d outside [%d, %d]", N, kTexMinN, kTexMaxN);
  NM_CHECK(F >= 0 && F < (1ll << 31), "texture bake: face count %lld outside [0, 2^31)", F);
  const long long C = N + 2, P = (F + 1) / 2;
  long long Q = (long long)sqrt((double)P);
  while (Q * Q < P) ++Q;
  while (Q > 0 && (Q - 1) * (Q - 1) >= P) --Q;
  const long long rows = Q ? (P + Q - 1) / Q : 0;
  const long long W = Q * C, H = rows * C;
  if (W > kTexMaxSide || H > kTexMaxSide) {
    const long long fit = Q ? kTexMaxSide / Q - 2 : kTexMaxN;      // H <= W, so the width decides
    NM_CHECK(fit >= kTexMinN, "texture bake: a %lld x %lld atlas exceeds %d texels per side, and %lld faces need more than %d "
             "texels per side even at N = %d", W, H, kTexMaxSide, F, kTexMaxSide, kTexMinN);
    NM_CHECK(false, "texture bake: a %lld x %lld atlas exceeds %d texels per side; the largest N that fits %lld faces is %lld",
             W, H, kTexMaxSide, F, fit);
  }
  out[0] = Q; out[1] = rows; out[2] = W; out[3] = H;
  return 0;
}

size_t texture_ws_bytes(const TextureBake& b) {
  const long long V = b.V, R = chunk_rays(b);
  return align_up((size_t)V * 4) + 2 * align_up((size_t)(V + 1) * 4) +
         align_up((size_t)((V + 1 + kScanBlockEntries - 1) / kScanBlockEntries) * 4) + align_up((size_t)V * 4) + align_up(16) +
         2 * align_up((size_t)R * 12) + align_up((size_t)R * 16);
}

int texture_rays(const TextureBake& b, long long f0, long long f1, float* a_out, float* d_out, int32_t* xy_out, int* d_err,
                 cudaStream_t st, int64_t* launches) {
  const TexLayout L = bake_layout(b);
  const long long n = (f1 - f0) * L.K;
  if (n == 0) return 0;
  tex_rays_kernel<<<blocks_for(n), kBlock, 0, st>>>(b.verts, b.normals, b.V, b.faces, f0, n, L, b.mode, b.disparity, a_out, d_out,
                                                    xy_out, d_err);
  NM_CUDA(cudaGetLastError());
  ++*launches;
  return 0;
}

int bake_texture(const TextureBake& b, float* atlas_f32, uint8_t* atlas_u8, float* uv, float* vertex_rgb, int64_t* counts_host,
                 void* ws, int* d_err, const volatile int* h_err, cudaStream_t st, int64_t* launches) {
  const TexLayout L = bake_layout(b);
  long long lay[4];
  if (int e = texture_layout(b.F, b.N, lay)) return e;
  const long long V = b.V, F = b.F, R = chunk_rays(b), H = lay[3];
  TexWs w = carve(b, ws);
  // 1-2: first references, bad indices, the unreferenced vertices
  if (V) NM_CUDA(cudaMemsetAsync(w.vfirst, 0x7f, (size_t)V * 4, st));
  if (F) {
    tex_first_ref_kernel<<<blocks_for(3 * F), kBlock, 0, st>>>(b.faces, F, V, w.vfirst, d_err);
    NM_CUDA(cudaGetLastError());
    ++*launches;
  }
  tex_unref_kernel<<<blocks_for(V + 1), kBlock, 0, st>>>(w.vfirst, V, w.flag);
  NM_CUDA(cudaGetLastError());
  ++*launches;
  if (int e = exclusive_scan(w.flag, V + 1, w.blk, w.start, st)) return e;
  if (V) {
    tex_unref_list_kernel<<<blocks_for(V), kBlock, 0, st>>>(w.flag, w.start, V, w.list);
    NM_CUDA(cudaGetLastError());
    ++*launches;
  }
  int U = 0;
  NM_CUDA(cudaMemcpyAsync(&U, w.start + V, 4, cudaMemcpyDeviceToHost, st));
  NM_CUDA(cudaStreamSynchronize(st));
  counts_host[0] = lay[2]; counts_host[1] = H; counts_host[2] = F * L.K + U; counts_host[3] = U;
  if (h_err[0] == kErrBadFace) return 0;                // the error word reports it; nothing is baked
  // 3: the faces, chunk by chunk
  if (F) NM_CUDA(cudaMemsetAsync(atlas_f32, 0, (size_t)lay[2] * H * 12, st));
  const long long faces_per_chunk = R / L.K > 0 ? R / L.K : 1;
  for (long long f0 = 0; f0 < F; f0 += faces_per_chunk) {
    const long long f1 = F - f0 < faces_per_chunk ? F : f0 + faces_per_chunk, n = (f1 - f0) * L.K;
    if (int e = texture_rays(b, f0, f1, w.a, w.d, nullptr, d_err, st, launches)) return e;
    if (int e = b.render(w.a, w.d, n, w.rgb)) return e;
    tex_scatter_kernel<<<blocks_for(n), kBlock, 0, st>>>(b.faces, w.vfirst, f0, n, L, w.rgb, b.rgb_stride, atlas_f32, vertex_rgb);
    NM_CUDA(cudaGetLastError());
    ++*launches;
  }
  // 4: the vertices no face references
  for (long long u0 = 0; u0 < U; u0 += R) {
    const long long n = U - u0 < R ? U - u0 : R;
    tex_vertex_rays_kernel<<<blocks_for(n), kBlock, 0, st>>>(b.verts, b.normals, w.list + u0, n, b.mode, b.disparity, w.a, w.d);
    NM_CUDA(cudaGetLastError());
    ++*launches;
    if (int e = b.render(w.a, w.d, n, w.rgb)) return e;
    tex_vertex_scatter_kernel<<<blocks_for(n), kBlock, 0, st>>>(w.list + u0, n, w.rgb, b.rgb_stride, vertex_rgb);
    NM_CUDA(cudaGetLastError());
    ++*launches;
  }
  if (!F) return 0;
  // 5: rings, quantisation, uv
  tex_ring_kernel<<<blocks_for(F * (L.N + 1)), kBlock, 0, st>>>(F, L, atlas_f32);
  NM_CUDA(cudaGetLastError());
  tex_quantise_kernel<<<blocks_for(lay[2] * H * 3), kBlock, 0, st>>>(atlas_f32, lay[2] * H * 3, atlas_u8);
  NM_CUDA(cudaGetLastError());
  tex_uv_kernel<<<blocks_for(3 * F), kBlock, 0, st>>>(F, L, H, uv);
  NM_CUDA(cudaGetLastError());
  *launches += 3;
  return 0;
}

}  // namespace nm

extern "C" int nm_texture_layout(int64_t F, int N, int64_t* out4) {
  NM_CHECK(out4, "texture bake: null layout pointer");
  long long lay[4];
  if (int e = nm::texture_layout(F, N, lay)) return e;
  for (int k = 0; k < 4; ++k) out4[k] = lay[k];
  return 0;
}
