// Depth-consistent surface points from one rendered view (DESIGN §4.14; the counterpart of the reference's dead
// src/mesh_surface_ray.py, which could not import).  Every pixel's expected hit distance becomes a point on its ray; a
// point is kept when enough of its (2s+1)^2 clamped pixel neighbours lie within a distance of it in 3-D.
//   1. launch_raygen         the render's own ray directions (nm_render.cu's raygen_kernel, without NDC) into the workspace
//   2. sf_mask_kernel        one CTA per kTileW x kTileH pixel tile: t = depth_raw where acc >= min_acc (else 0) and
//                            P = o + d*t for the tile and an s-pixel clamped halo into shared memory, then per pixel the
//                            number of offsets (a, b) in [-s, s]^2 whose neighbour lies within dist2 < thr, and the keep
//                            mask: count >= min_count and t > 0
//   3. exclusive_scan        of the mask (the grid search's integer scan, nm_chamfer.cu): per-block sums, then offsets
//   4. sf_scatter_kernel     the kept pixels in row-major order: P again (the same arithmetic, so the same bits), -d, rgb,
//                            the pixel index
// Built with -fmad=false: o + d*t and (dx*dx + dy*dy) + dz*dz are two roundings per step, which tests/_surface_ref.py
// restates bit for bit.  The mask is a function of the inputs alone and the compaction an integer scan, so the output is
// the same bits on every run and for every tile shape.
#include "nm_common.h"

namespace nm {
namespace {

constexpr int kBlock = 256;
constexpr int kTileW = 32, kTileH = 8;             // one thread per output pixel
constexpr int kHaloW = kTileW + 2 * kSurfaceMaxStep, kHaloH = kTileH + 2 * kSurfaceMaxStep;

unsigned blocks_for(long long n) { return (unsigned)((n + kBlock - 1) / kBlock); }
size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

struct SfArgs {
  const float* depth_raw;
  const float* acc;
  const float* rgb;
  const float* dirs;        // (H*W, 3): the render's directions
  float o[3];
  int H, W, s, min_count;
  float min_acc, thr;
};

// the gated distance t and the surface point of pixel i
__device__ __forceinline__ float sf_point(const SfArgs& a, long long i, float p[3]) {
  const float t = a.acc[i] >= a.min_acc ? a.depth_raw[i] : 0.f;
#pragma unroll
  for (int k = 0; k < 3; ++k) p[k] = a.o[k] + a.dirs[3 * i + k] * t;
  return t;
}

// mask[i] for pixels i in [0, H*W); mask[H*W] = 0 so that the scan's last entry is the kept total
__global__ void __launch_bounds__(kBlock) sf_mask_kernel(const __grid_constant__ SfArgs a, int tiles_x, int* __restrict__ mask) {
  __shared__ float px[kHaloH][kHaloW], py[kHaloH][kHaloW], pz[kHaloH][kHaloW];
  const int r0 = (int)(blockIdx.x / tiles_x) * kTileH, c0 = (int)(blockIdx.x % tiles_x) * kTileW;
  const int s = a.s, hw = kTileW + 2 * s, hh = kTileH + 2 * s;
  for (int j = threadIdx.x; j < hw * hh; j += kBlock) {
    const int ly = j / hw, lx = j % hw;
    const int r = min(max(r0 - s + ly, 0), a.H - 1), c = min(max(c0 - s + lx, 0), a.W - 1);
    float p[3];
    sf_point(a, (long long)r * a.W + c, p);
    px[ly][lx] = p[0]; py[ly][lx] = p[1]; pz[ly][lx] = p[2];
  }
  __syncthreads();
  const int tx = threadIdx.x % kTileW, ty = threadIdx.x / kTileW;
  const int r = r0 + ty, c = c0 + tx;
  const long long n = (long long)a.H * a.W;
  if (r == 0 && c == 0) mask[n] = 0;
  if (r >= a.H || c >= a.W) return;
  const float x = px[ty + s][tx + s], y = py[ty + s][tx + s], z = pz[ty + s][tx + s];
  int count = 0;
  for (int dy = 0; dy <= 2 * s; ++dy)
    for (int dx = 0; dx <= 2 * s; ++dx) {
      const float ex = px[ty + dy][tx + dx] - x, ey = py[ty + dy][tx + dx] - y, ez = pz[ty + dy][tx + dx] - z;
      count += ((ex * ex + ey * ey) + ez * ez) < a.thr;          // NaN compares false
    }
  const long long i = (long long)r * a.W + c;
  const float t = a.acc[i] >= a.min_acc ? a.depth_raw[i] : 0.f;
  mask[i] = count >= a.min_count && t > 0.f;
}

__global__ void __launch_bounds__(kBlock) sf_scatter_kernel(const __grid_constant__ SfArgs a, const int* __restrict__ mask,
                                                            const int* __restrict__ start, float* __restrict__ pts,
                                                            float* __restrict__ nrm, float* __restrict__ col,
                                                            int32_t* __restrict__ pix) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= (long long)a.H * a.W || !mask[i]) return;
  const long long o = start[i];
  float p[3];
  sf_point(a, i, p);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    pts[3 * o + k] = p[k];
    nrm[3 * o + k] = -a.dirs[3 * i + k];
    col[3 * o + k] = a.rgb[3 * i + k];
  }
  if (pix) pix[o] = (int32_t)i;
}

// Workspace (256-byte aligned pieces): dirs (3n floats), mask, start (n+1 ints each), the scan's block sums
struct SfWs {
  float* dirs;
  int *mask, *start, *blk;
};
size_t carve(void* ws, long long n, SfWs* w) {
  const long long nblk = (n + 1 + kScanBlockEntries - 1) / kScanBlockEntries;
  const size_t sz[4] = {(size_t)n * 12, (size_t)(n + 1) * 4, (size_t)(n + 1) * 4, (size_t)nblk * 4};
  void** dst[4] = {(void**)&w->dirs, (void**)&w->mask, (void**)&w->start, (void**)&w->blk};
  size_t tot = 0;
  for (int i = 0; i < 4; ++i) {
    if (ws) *dst[i] = reinterpret_cast<char*>(ws) + tot;
    tot += align_up(sz[i]);
  }
  return tot;
}

}  // namespace

size_t surface_ws_bytes(long long H, long long W) {
  SfWs w{};
  return carve(nullptr, H * W, &w);
}

int surface_points(const SurfaceView& v, float* pts, float* nrm, float* col, int32_t* pix, int64_t* count_host, void* ws,
                   cudaStream_t st, int64_t* launches) {
  const long long n = (long long)v.H * v.W;
  SfWs w{};
  carve(ws, n, &w);
  RayGenArgs g{};
  for (int k = 0; k < 12; ++k) g.pose[k] = v.pose[k];
  g.H = v.H; g.W = v.W; g.focal = v.focal; g.ndc = 0; g.ndc_near = 1.0; g.row0 = 0; g.row1 = v.H;
  if (int e = launch_raygen(g, nullptr, w.dirs, st, launches)) return e;
  SfArgs a{};
  a.depth_raw = v.depth_raw; a.acc = v.acc; a.rgb = v.rgb; a.dirs = w.dirs;
  a.o[0] = v.pose[3]; a.o[1] = v.pose[7]; a.o[2] = v.pose[11];
  a.H = v.H; a.W = v.W; a.s = v.step; a.min_count = v.min_count; a.min_acc = v.min_acc; a.thr = v.dist_threshold;
  const int tiles_x = (v.W + kTileW - 1) / kTileW, tiles_y = (v.H + kTileH - 1) / kTileH;
  sf_mask_kernel<<<(unsigned)((long long)tiles_x * tiles_y), kBlock, 0, st>>>(a, tiles_x, w.mask);
  NM_CUDA(cudaGetLastError());
  if (int e = exclusive_scan(w.mask, n + 1, w.blk, w.start, st)) return e;
  sf_scatter_kernel<<<blocks_for(n), kBlock, 0, st>>>(a, w.mask, w.start, pts, nrm, col, pix);
  NM_CUDA(cudaGetLastError());
  int kept = 0;
  NM_CUDA(cudaMemcpyAsync(&kept, w.start + n, 4, cudaMemcpyDeviceToHost, st));
  NM_CUDA(cudaStreamSynchronize(st));
  *count_host = kept;
  if (launches) *launches += 5;
  return 0;
}

}  // namespace nm
