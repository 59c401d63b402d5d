// Mesh rasterizer (DESIGN §4.13; no reference counterpart: the reference has no way to look at its meshes).  World-coordinate
// triangles seen through the pinhole camera of nm_render_image, so that mesh pixel (c, r) lies on the ray NeRF pixel (c, r)
// renders.
//   1. raster_setup_kernel   per face: project the corners, cull, snap to 1/256 pixel, clip the bounding box of pixel samples
//                            to the frame; a face whose box holds >= NM_RASTER_BIG_FACE_PIXELS samples joins the big list.
//                            A face index outside [0, V) sets the error word (code 6) and nothing is drawn.
//   2. raster_small_kernel   one thread per face walks its box
//      raster_big_kernel     one CTA per 16 x 16 screen tile walks the big list, one thread per pixel
//                            both: exact int64 edge functions with a top-left rule, then one 64-bit atomicMin of
//                            (bits of the perspective-correct depth) << 32 | face per covered sample
//   3. raster_resolve_kernel one thread per pixel: the winning face's weights again, colour (vertex colours or a bilinear
//                            lookup in the §4.12 atlas), ray distance, face id; covered pixels counted
// Built with -fmad=false: every fp32 step is the arithmetic in the written order, which tests/_raster_ref.py restates bit
// for bit.  Coverage is integer arithmetic and the depth test an atomicMin of a total order, so the image does not depend on
// the launch order, the atomic order or which pass drew a face.
#include <cmath>

#include "nm_common.h"
#include "nm_texture.cuh"

namespace nm {
namespace {

constexpr int kBlock = 256;
constexpr int kTile = 16;                       // big-face pass: one CTA of kTile^2 threads per screen tile
constexpr int kErrBadFace = 6;                  // codes 1-5 of the same word belong to the sampler, components, decimation, bake
constexpr float kMaxScreen = 1048576.f;         // 2^20 pixels: snapped coordinates stay below 2^28
constexpr unsigned long long kEmpty = ~0ull;    // key of a pixel no face covers

unsigned blocks_for(long long n) { return (unsigned)((n + kBlock - 1) / kBlock); }
size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

struct alignas(16) FaceRec {
  int x[3], y[3];          // corners in 1/256 pixel
  float z[3];              // depth along the camera axis
  short c0, c1, r0, r1;    // pixel samples of the bounding box inside the frame; c0 > c1: nothing to draw
  int big;                 // drawn by the tile pass
};

struct Counters {
  unsigned long long covered, culled;
  int n_big, bad;
};

struct Cam {
  float R[9], t[3];        // R[3i + k] = pose[4i + k], t[i] = pose[4i + 3]
  float focal, half_w, half_h, z_near;
  int H, W;
  long long big_pixels;
};

__device__ __forceinline__ int floor_div256(int a) { return a >> 8; }
__device__ __forceinline__ int ceil_div256(int a) { return -((-a) >> 8); }

// Edge functions of pixel sample (c, r) (the point (256c, 256r) in snapped units), E[k] opposite corner k, and the face's
// doubled area A = E0 + E1 + E2, both made positive inside.  Covered: every E[k] > 0, or == 0 on a top-left edge (its
// direction in the positive orientation has dy > 0, or dy == 0 and dx > 0: the sample nudged by (-e, +e*d) for tiny d).
__device__ __forceinline__ bool cover(const FaceRec& q, int c, int r, long long E[3], long long* A) {
  const long long px = (long long)c * 256, py = (long long)r * 256;
  long long dx[3], dy[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int a = k == 2 ? 0 : k + 1, b = k == 0 ? 2 : k - 1;
    dx[k] = (long long)q.x[b] - q.x[a];
    dy[k] = (long long)q.y[b] - q.y[a];
    E[k] = dx[k] * (py - q.y[a]) - dy[k] * (px - q.x[a]);
  }
  long long area = E[0] + E[1] + E[2];
  const bool neg = area < 0;
  if (neg) area = -area;
  *A = area;
  bool in = true;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    if (neg) { E[k] = -E[k]; dx[k] = -dx[k]; dy[k] = -dy[k]; }
    in = in && (E[k] > 0 || (E[k] == 0 && (dy[k] > 0 || (dy[k] == 0 && dx[k] > 0))));
  }
  return in;
}

// perspective-correct weights w and depth z_pix = 1/s of a covered sample
__device__ __forceinline__ void weights(const FaceRec& q, const long long E[3], long long A, float w[3], float* zpix) {
  float a[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float l = (float)((double)E[k] / (double)A);
    a[k] = l / q.z[k];
  }
  const float s = (a[0] + a[1]) + a[2];
#pragma unroll
  for (int k = 0; k < 3; ++k) w[k] = a[k] / s;
  *zpix = 1.0f / s;
}

__device__ __forceinline__ unsigned long long sample_key(const FaceRec& q, long long f, int c, int r) {
  long long E[3], A;
  if (!cover(q, c, r, E, &A)) return kEmpty;
  float w[3], z;
  weights(q, E, A, w, &z);
  return ((unsigned long long)__float_as_uint(z) << 32) | (unsigned long long)(unsigned)f;
}

__global__ void __launch_bounds__(kBlock) raster_setup_kernel(const float* __restrict__ verts, long long V,
                                                              const int* __restrict__ faces, long long F, const Cam cam,
                                                              FaceRec* __restrict__ recs, int* __restrict__ big_list,
                                                              Counters* cnt, int* err) {
  const long long f = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (f >= F) return;
  FaceRec q{};
  q.c0 = 1; q.c1 = 0; q.r0 = 1; q.r1 = 0; q.big = 0;
  int vi[3];
  bool bad = false;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    vi[k] = faces[3 * f + k];
    bad = bad || vi[k] < 0 || vi[k] >= V;
  }
  if (bad) {
    *err = kErrBadFace;
    cnt->bad = 1;
    recs[f] = q;
    return;
  }
  bool cull = false;
  float X[3], Y[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float d0 = verts[3ll * vi[k]] - cam.t[0], d1 = verts[3ll * vi[k] + 1] - cam.t[1], d2 = verts[3ll * vi[k] + 2] - cam.t[2];
    float p[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) p[j] = (d0 * cam.R[j] + d1 * cam.R[3 + j]) + d2 * cam.R[6 + j];
    const float z = -p[2];
    X[k] = cam.half_w + cam.focal * (p[0] / z);
    Y[k] = cam.half_h - cam.focal * (p[1] / z);
    q.z[k] = z;
    cull = cull || !(z > cam.z_near) || !isfinite(z) || !isfinite(X[k]) || !isfinite(Y[k]) || fabsf(X[k]) > kMaxScreen ||
           fabsf(Y[k]) > kMaxScreen;
  }
  if (cull) {
    atomicAdd(&cnt->culled, 1ull);
    recs[f] = q;
    return;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) { q.x[k] = (int)rintf(X[k] * 256.f); q.y[k] = (int)rintf(Y[k] * 256.f); }
  const long long area = ((long long)q.x[1] - q.x[0]) * ((long long)q.y[2] - q.y[0]) -
                         ((long long)q.y[1] - q.y[0]) * ((long long)q.x[2] - q.x[0]);
  if (area != 0) {
    const int c0 = max(ceil_div256(min(min(q.x[0], q.x[1]), q.x[2])), 0);
    const int c1 = min(floor_div256(max(max(q.x[0], q.x[1]), q.x[2])), cam.W - 1);
    const int r0 = max(ceil_div256(min(min(q.y[0], q.y[1]), q.y[2])), 0);
    const int r1 = min(floor_div256(max(max(q.y[0], q.y[1]), q.y[2])), cam.H - 1);
    if (c0 <= c1 && r0 <= r1) {
      q.c0 = (short)c0; q.c1 = (short)c1; q.r0 = (short)r0; q.r1 = (short)r1;
      if ((long long)(c1 - c0 + 1) * (r1 - r0 + 1) >= cam.big_pixels) {
        q.big = 1;
        big_list[atomicAdd(&cnt->n_big, 1)] = (int)f;
      }
    }
  }
  recs[f] = q;
}

__global__ void __launch_bounds__(kBlock) raster_small_kernel(const FaceRec* __restrict__ recs, long long F,
                                                              const Counters* __restrict__ cnt, int W,
                                                              unsigned long long* keys) {
  const long long f = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (f >= F || cnt->bad) return;
  const FaceRec q = recs[f];
  if (q.big) return;
  for (int r = q.r0; r <= q.r1; ++r)
    for (int c = q.c0; c <= q.c1; ++c) {
      const unsigned long long key = sample_key(q, f, c, r);
      if (key != kEmpty) atomicMin(keys + (long long)r * W + c, key);
    }
}

__global__ void __launch_bounds__(kTile * kTile) raster_big_kernel(const FaceRec* __restrict__ recs, const int* __restrict__ big_list,
                                                                   const Counters* __restrict__ cnt, int H, int W,
                                                                   unsigned long long* keys) {
  __shared__ int hit[kTile * kTile];
  __shared__ int n_hit;
  if (cnt->bad) return;
  const int n = cnt->n_big;
  const int tx0 = blockIdx.x * kTile, ty0 = blockIdx.y * kTile;
  const int c = tx0 + (int)threadIdx.x % kTile, r = ty0 + (int)threadIdx.x / kTile;
  const bool inside = c < W && r < H;
  unsigned long long best = kEmpty;
  for (int base = 0; base < n; base += kTile * kTile) {
    __syncthreads();
    if (threadIdx.x == 0) n_hit = 0;
    __syncthreads();
    if (base + (int)threadIdx.x < n) {               // the big faces whose box meets this tile, in any order
      const int f = big_list[base + threadIdx.x];
      const FaceRec& q = recs[f];
      if (q.c0 < tx0 + kTile && q.c1 >= tx0 && q.r0 < ty0 + kTile && q.r1 >= ty0) hit[atomicAdd(&n_hit, 1)] = f;
    }
    __syncthreads();
    const int m = n_hit;
    if (!inside) continue;
    for (int k = 0; k < m; ++k) {
      const int f = hit[k];
      const FaceRec q = recs[f];
      if (c < q.c0 || c > q.c1 || r < q.r0 || r > q.r1) continue;
      const unsigned long long key = sample_key(q, f, c, r);
      best = key < best ? key : best;
    }
  }
  if (inside && best != kEmpty) atomicMin(keys + (long long)r * W + c, best);
}

// bilinear lookup of face f's patch at barycentric weights (w1, w2) (DESIGN §4.13): w1, w2 clamped to [0, 1] and scaled by
// 1/(w1 + w2) when their sum exceeds 1; patch coordinates s = min(w1 (N-1), N-1), t = min(w2 (N-1), (N-1) - s), so that
// every tap of nonzero weight lies in the face's patch or ring; taps (i,j), (i+1,j), (i,j+1), (i+1,j+1) summed in that order
__device__ __forceinline__ void texture_lookup(const float* __restrict__ atlas, const TexLayout& L, long long f, float w1, float w2,
                                               float out[3]) {
  w1 = fminf(fmaxf(w1, 0.f), 1.f);
  w2 = fminf(fmaxf(w2, 0.f), 1.f);
  const float sum = w1 + w2;
  if (sum > 1.f) {
    const float k = 1.0f / sum;
    w1 = w1 * k;
    w2 = w2 * k;
  }
  const float S = (float)(L.N - 1);
  const float s = fminf(w1 * S, S);
  const float t = fminf(w2 * S, S - s);
  const float a = floorf(s), b = floorf(t);
  const float fx = s - a, fy = t - b;
  const int i = (int)a, j = (int)b;
  const float tw[4] = {(1.0f - fx) * (1.0f - fy), fx * (1.0f - fy), (1.0f - fx) * fy, fx * fy};
  out[0] = out[1] = out[2] = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (!(tw[k] > 0.f)) continue;                    // a tap of weight 0 may lie outside the patch and ring: never read
    const float* T = atlas + 3 * texel_pixel(f, i + (k & 1), j + (k >> 1), L);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) out[ch] = out[ch] + tw[k] * T[ch];
  }
}

struct ResolveOut {
  float* rgb;
  float* depth;
  int* face;
  float bg[3];
};

__global__ void __launch_bounds__(kBlock) raster_resolve_kernel(const FaceRec* __restrict__ recs, const int* __restrict__ faces,
                                                                const unsigned long long* __restrict__ keys, Counters* cnt,
                                                                const Cam cam, int mode, const float* __restrict__ vrgb,
                                                                const float* __restrict__ atlas, TexLayout L, ResolveOut o) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  const long long n = (long long)cam.H * cam.W;
  const bool valid = i < n;
  const unsigned long long key = (valid && keys && !cnt->bad) ? keys[i] : kEmpty;
  const bool covered = key != kEmpty;
  const unsigned m = __ballot_sync(0xffffffffu, covered);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&cnt->covered, (unsigned long long)__popc(m));
  if (!valid) return;
  if (!covered) {
    if (o.rgb) for (int ch = 0; ch < 3; ++ch) o.rgb[3 * i + ch] = o.bg[ch];
    if (o.depth) o.depth[i] = 0.f;
    if (o.face) o.face[i] = -1;
    return;
  }
  const int c = (int)(i % cam.W), r = (int)(i / cam.W);
  const long long f = (long long)(key & 0xffffffffull);
  const FaceRec q = recs[f];
  long long E[3], A;
  cover(q, c, r, E, &A);
  float w[3], z;
  weights(q, E, A, w, &z);
  if (o.rgb) {
    float col[3];
    if (mode == 0) {
      const float* c0 = vrgb + 3ll * faces[3 * f];
      const float* c1 = vrgb + 3ll * faces[3 * f + 1];
      const float* c2 = vrgb + 3ll * faces[3 * f + 2];
      for (int ch = 0; ch < 3; ++ch) col[ch] = (w[0] * c0[ch] + w[1] * c1[ch]) + w[2] * c2[ch];
    } else {
      texture_lookup(atlas, L, f, w[1], w[2], col);
    }
    for (int ch = 0; ch < 3; ++ch) o.rgb[3 * i + ch] = col[ch];
  }
  if (o.depth) {                                     // the un-normalised direction of raygen_kernel's ray through (c, r)
    const float x = ((float)c - cam.half_w) / cam.focal;
    const float y = -((float)r - cam.half_h) / cam.focal;
    o.depth[i] = z * sqrtf((x * x + y * y) + 1.0f);
  }
  if (o.face) o.face[i] = (int)f;
}

struct RasterWs {
  unsigned long long* keys;
  FaceRec* recs;
  int* big;
  Counters* cnt;
};

RasterWs carve(const RasterMesh& m, void* ws) {
  char* p = static_cast<char*>(ws);
  RasterWs w;
  auto take = [&](size_t bytes) { char* q = p; p += align_up(bytes); return q; };
  w.keys = reinterpret_cast<unsigned long long*>(take((size_t)m.H * m.W * 8));
  w.recs = reinterpret_cast<FaceRec*>(take((size_t)m.F * sizeof(FaceRec)));
  w.big = reinterpret_cast<int*>(take((size_t)m.F * 4));
  w.cnt = reinterpret_cast<Counters*>(take(sizeof(Counters)));
  return w;
}

}  // namespace

size_t raster_ws_bytes(const RasterMesh& m) {
  return align_up((size_t)m.H * m.W * 8) + align_up((size_t)m.F * sizeof(FaceRec)) + align_up((size_t)m.F * 4) +
         align_up(sizeof(Counters));
}

int rasterize_mesh(const RasterMesh& m, int64_t* counts_host, void* ws, int* d_err, cudaStream_t st, int64_t* launches) {
  RasterWs w = carve(m, ws);
  Cam cam{};
  for (int i = 0; i < 3; ++i) {
    for (int k = 0; k < 3; ++k) cam.R[3 * i + k] = m.pose[4 * i + k];
    cam.t[i] = m.pose[4 * i + 3];
  }
  cam.focal = m.focal;
  cam.half_w = (float)(m.W * 0.5);                   // as launch_raygen computes them
  cam.half_h = (float)(m.H * 0.5);
  cam.z_near = m.z_near;
  cam.H = m.H; cam.W = m.W;
  cam.big_pixels = m.big_pixels;
  TexLayout L{};
  if (m.mode == 1 && m.F) {
    if (int e = tex_layout(m.F, m.N, &L)) return e;
  }
  const long long n = (long long)m.H * m.W;
  NM_CUDA(cudaMemsetAsync(w.cnt, 0, sizeof(Counters), st));
  if (m.F) {
    NM_CUDA(cudaMemsetAsync(w.keys, 0xff, (size_t)n * 8, st));
    raster_setup_kernel<<<blocks_for(m.F), kBlock, 0, st>>>(m.verts, m.V, m.faces, m.F, cam, w.recs, w.big, w.cnt, d_err);
    NM_CUDA(cudaGetLastError());
    raster_small_kernel<<<blocks_for(m.F), kBlock, 0, st>>>(w.recs, m.F, w.cnt, m.W, w.keys);
    NM_CUDA(cudaGetLastError());
    const dim3 tiles((unsigned)((m.W + kTile - 1) / kTile), (unsigned)((m.H + kTile - 1) / kTile));
    raster_big_kernel<<<tiles, kTile * kTile, 0, st>>>(w.recs, w.big, w.cnt, m.H, m.W, w.keys);
    NM_CUDA(cudaGetLastError());
    *launches += 3;
  }
  ResolveOut o{m.rgb, m.depth, m.face, {m.bg[0], m.bg[1], m.bg[2]}};
  raster_resolve_kernel<<<blocks_for(n), kBlock, 0, st>>>(w.recs, m.faces, m.F ? w.keys : nullptr, w.cnt, cam, m.mode, m.vertex_rgb,
                                                         m.atlas, L, o);
  NM_CUDA(cudaGetLastError());
  ++*launches;
  Counters h{};
  NM_CUDA(cudaMemcpyAsync(&h, w.cnt, sizeof(Counters), cudaMemcpyDeviceToHost, st));
  NM_CUDA(cudaStreamSynchronize(st));
  if (h.bad) {
    counts_host[0] = counts_host[1] = counts_host[2] = 0;
  } else {
    counts_host[0] = (int64_t)h.covered;
    counts_host[1] = m.F - (int64_t)h.culled;
    counts_host[2] = (int64_t)h.culled;
  }
  return 0;
}

}  // namespace nm
