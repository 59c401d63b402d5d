// Training backward of the fused path (SURVEY §8f-1): dL/dθ of both FlexibleNeRFModels given dL/d rgb_map of the
// coarse and fine bundles — what `loss.backward()` produces for NeRFModel.training_step (src/models/model_nerf.py:88-151)
// through VolumeRenderer (src/nerf/modules.py:67-121), the network (src/nerf/models.py:60-80) and nothing else
// (SamplePDF is detached, modules.py:201; sample positions do not depend on θ).
//
// Tensor cores (default, DESIGN.md 4.4): the training forward is the fused kernel in its emitting mode (nm_mlp_tc.cu mode 1:
// relu masks, head activations, K-major operand packs of every hidden activation) — for the whole chunk when its
// workspace fits (no recompute), else per sub-chunk of points; the data-gradient chain
//     dZ_{l-1} = (dZ_l W_l (+ dsigma w_alpha)) * relu'_{l-1}
// of ALL layers is one more launch of that kernel (mode 2, MN-major operand packs of every dZ); the weight gradients
//     dW_l += dZ_l^T [act_{l-1} | PE]                    (K = points: split over CTAs, fp32 atomics)
// are long-K launches of tc_gemm_kernel (nm_gemm_tc.cu) on the packs, which also take the bias gradients (row sums of the
// staged dZ^T tiles).
// NM_PREC_FP32: the network walked layer by layer in plain fp32 FMAs on the CUDA cores (sgemm_kernel / sgemm_tn_kernel
// below; the reference trains in fp32, TF32 off) — the numerical yard-stick the tensor-core path is tested against.
// Small SIMT kernels around them: encodings, the 3-/4-row heads, the compositor adjoint, the MSE gradient.
// Gradients accumulate in the reference's (out,in) orientation (rows padded to 4 floats, grad_layout()); nm_get_grad
// returns them per state-dict tensor.
#include <math_constants.h>

#include <cuda_bf16.h>

#include "nm_common.h"
#include "nm_composite.cuh"
#include "nm_frontend.cuh"
#include "nm_gemm.h"

namespace nm {
namespace {

constexpr int kPeLd = 64;   // padded row length of the encoding buffers

// ------------------------------------------------------------------------------------------------ encodings
__global__ void encode_kernel(const __grid_constant__ MlpInput in, const NetProgram* __restrict__ prog,
                              float* __restrict__ pe_x, float* __restrict__ pe_d) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= in.M) return;
  const NetProgram& G = *prog;
  float p[3], d[3];
  fetch_point(in, m, p, d);
  float* px = pe_x + m * kPeLd;
  for (int j = G.dim_xyz; j < kPeLd; ++j) px[j] = 0.f;
  positional_encoding(p, G.L_xyz, G.inc_xyz, G.freq_xyz, [&](int j, float v) { px[j] = v; });
  if (G.dim_dir > 0) {
    float* pd = pe_d + m * kPeLd;
    for (int j = G.dim_dir; j < kPeLd; ++j) pd[j] = 0.f;
    positional_encoding(d, G.L_dir, G.inc_dir, G.freq_dir, [&](int j, float v) { pd[j] = v; });
  }
}

// Tensor-core path: the encodings are only ever read as the B operand of the weight-gradient GEMMs, so they go straight
// into the point-major bf16 hi/lo packs (pack_cols_kernel's layout, nm_gemm_tc.cu: tile = [feature block][64-point K
// block], 128 feature rows x 64 points, 128-byte swizzle) without an fp32 round trip.  One CTA per 64 points: threads
// 0..63 encode xyz, 64..127 the direction, all 256 write the two tiles from shared memory.
__global__ void __launch_bounds__(256) encode_pack_kernel(const __grid_constant__ MlpInput in, const NetProgram* __restrict__ prog,
                                                          uint8_t* __restrict__ pkt_x, uint8_t* __restrict__ pkt_d) {
  __shared__ float t[2][64][65];                           // [encoding][feature][point]
  const NetProgram& G = *prog;
  const int kb = blockIdx.x;
  const int which = threadIdx.x >> 6, pt = threadIdx.x & 63;
  if (which < 2) {
    float (*tt)[65] = t[which];
    const long long m = (long long)kb * 64 + pt;
    const int dim = which ? G.dim_dir : G.dim_xyz;
    for (int j = dim; j < 64; ++j) tt[j][pt] = 0.f;
    if (m < in.M && dim > 0) {
      float p[3], d[3];
      fetch_point(in, m, p, d);
      if (which == 0) positional_encoding(p, G.L_xyz, G.inc_xyz, G.freq_xyz, [&](int j, float v) { tt[j][pt] = v; });
      else positional_encoding(d, G.L_dir, G.inc_dir, G.freq_dir, [&](int j, float v) { tt[j][pt] = v; });
    } else {
      for (int j = 0; j < dim; ++j) tt[j][pt] = 0.f;
    }
  }
  __syncthreads();
  const int c8 = threadIdx.x & 7;
  for (int e = 0; e < 2; ++e) {
    if (e == 1 && G.dim_dir <= 0) break;
    uint8_t* tile = (e ? pkt_d : pkt_x) + (size_t)kb * kPtileBytes;        // one feature block: tile index = kb
#pragma unroll
    for (int pass = 0; pass < 4; ++pass) {
      const int r = pass * 32 + (threadIdx.x >> 3);        // feature row of the tile; rows >= 64 are zero padding
      __align__(16) uint16_t hi[8], lo[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float x = r < 64 ? t[e][r][c8 * 8 + i] : 0.f;
        const __nv_bfloat16 h = __float2bfloat16_rn(x);
        const __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
        hi[i] = __bfloat16_as_ushort(h); lo[i] = __bfloat16_as_ushort(l);
      }
      const uint32_t off = (uint32_t)r * 128u + (uint32_t)((c8 ^ (r & 7)) << 4);
      *reinterpret_cast<uint4*>(tile + off) = *reinterpret_cast<const uint4*>(hi);
      *reinterpret_cast<uint4*>(tile + kPtileHalf + off) = *reinterpret_cast<const uint4*>(lo);
    }
  }
}

// ------------------------------------------------------------------------------------------------ SGEMM  C = A * op(B)
// A (M,K) row-major.  BT=false: B (K,N) row-major;  BT=true: B (N,K) row-major (C = A B^T).
// CTA tile 128 x (16*TN), 256 threads, 8 x TN micro-tile, BK = 16, register prefetch of the next K tile.

// fused epilogue: v = acc (+C) (+bias[n]) (+r1_vec[m]*r1_w[n]); relu; relu-mask of another tensor
struct GemmEpi {
  int accumulate;          // C += (else C =)
  const float* bias;       // + bias[n]
  int relu;                // max(.,0)
  const float* r1_vec;     // + r1_vec[m * r1_stride] * r1_w[n]
  int r1_stride;
  const float* r1_w;
  const float* mask;       // * (mask[m*ldmask + n] > 0)
  int ldmask;
};

template <int TN, bool BT>
__global__ void __launch_bounds__(256) sgemm_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B,
                                                    int ldb, float* __restrict__ C, int ldc, int M, int N, int K,
                                                    const GemmEpi epi) {
  constexpr int BM = 128, BN = 16 * TN, BK = 16;
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;

  // global -> register staging
  float4 ra[2];
  float4 rb[BN / 64 > 0 ? BN / 64 : 1];
  constexpr int NB4 = BN / 64;                      // float4 per thread for the B tile (BK*BN/4/256)
  auto load_tiles = [&](int k0) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {                   // A tile: 128 rows x 4 float4
      const int f = tid + i * 256, r = f >> 2, kq = (f & 3) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (m0 + r < M && k0 + kq < K) {
        v = *reinterpret_cast<const float4*>(A + (size_t)(m0 + r) * lda + k0 + kq);
        if (k0 + kq + 1 >= K) v.y = 0.f;
        if (k0 + kq + 2 >= K) v.z = 0.f;
        if (k0 + kq + 3 >= K) v.w = 0.f;
      }
      ra[i] = v;
    }
    if (!BT) {
#pragma unroll
      for (int i = 0; i < NB4; ++i) {               // B tile (K,N): 16 rows x BN/4 float4
        const int f = tid + i * 256, r = f / (BN / 4), c4 = (f % (BN / 4)) * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (k0 + r < K && n0 + c4 < N) v = *reinterpret_cast<const float4*>(B + (size_t)(k0 + r) * ldb + n0 + c4);
        rb[i] = v;
      }
    } else {
#pragma unroll
      for (int i = 0; i < NB4; ++i) {               // B tile (N,K): BN rows x 4 float4
        const int f = tid + i * 256, r = f >> 2, kq = (f & 3) * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (n0 + r < N && k0 + kq < K) {
          v = *reinterpret_cast<const float4*>(B + (size_t)(n0 + r) * ldb + k0 + kq);
          if (k0 + kq + 1 >= K) v.y = 0.f;
          if (k0 + kq + 2 >= K) v.z = 0.f;
          if (k0 + kq + 3 >= K) v.w = 0.f;
        }
        rb[i] = v;
      }
    }
  };
  auto store_tiles = [&]() {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int f = tid + i * 256, r = f >> 2, kq = (f & 3) * 4;
      As[kq + 0][r] = ra[i].x; As[kq + 1][r] = ra[i].y; As[kq + 2][r] = ra[i].z; As[kq + 3][r] = ra[i].w;
    }
    if (!BT) {
#pragma unroll
      for (int i = 0; i < NB4; ++i) {
        const int f = tid + i * 256, r = f / (BN / 4), c4 = (f % (BN / 4)) * 4;
        *reinterpret_cast<float4*>(&Bs[r][c4]) = rb[i];
      }
    } else {
#pragma unroll
      for (int i = 0; i < NB4; ++i) {
        const int f = tid + i * 256, r = f >> 2, kq = (f & 3) * 4;
        Bs[kq + 0][r] = rb[i].x; Bs[kq + 1][r] = rb[i].y; Bs[kq + 2][r] = rb[i].z; Bs[kq + 3][r] = rb[i].w;
      }
    }
  };

  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  load_tiles(0);
  for (int k0 = 0; k0 < K; k0 += BK) {
    store_tiles();
    __syncthreads();
    if (k0 + BK < K) load_tiles(k0 + BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[8], b[TN];
      const float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * 8 + 4]);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][(j >> 2) * 64 + tx * 4]);
        b[j] = bv.x; b[j + 1] = bv.y; b[j + 2] = bv.z; b[j + 3] = bv.w;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + ty * 8 + i;
    if (m >= M) continue;
    const float r1 = epi.r1_vec ? epi.r1_vec[(size_t)m * epi.r1_stride] : 0.f;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
      const int n = n0 + (j >> 2) * 64 + tx * 4 + (j & 3);
      if (n >= N) continue;
      float v = acc[i][j];
      float* c = C + (size_t)m * ldc + n;
      if (epi.accumulate) v += *c;
      if (epi.bias) v += epi.bias[n];
      if (epi.r1_vec) v = fmaf(r1, epi.r1_w[n], v);
      if (epi.relu) v = fmaxf(v, 0.f);
      if (epi.mask && !(epi.mask[(size_t)m * epi.ldmask + n] > 0.f)) v = 0.f;
      *c = v;
    }
  }
}

template <bool BT>
int sgemm(const float* A, int lda, const float* B, int ldb, float* C, int ldc, int M, int N, int K, const GemmEpi& epi,
          cudaStream_t st, int64_t* launches) {
  if (M <= 0 || N <= 0) return 0;
  if (N % 128 == 0) {
    dim3 grid((M + 127) / 128, N / 128);
    sgemm_kernel<8, BT><<<grid, 256, 0, st>>>(A, lda, B, ldb, C, ldc, M, N, K, epi);
  } else {
    dim3 grid((M + 127) / 128, (N + 63) / 64);
    sgemm_kernel<4, BT><<<grid, 256, 0, st>>>(A, lda, B, ldb, C, ldc, M, N, K, epi);
  }
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

// ------------------------------------------------------------------------------------------------ dWt += A^T B
// A (P,K) row-major, B (P,N) row-major, G (K,N) row-major (ldg).  CTA tile 128(k) x 128(n), split over P.
__global__ void __launch_bounds__(256) sgemm_tn_kernel(const float* __restrict__ A, int lda, const float* __restrict__ B,
                                                       int ldb, float* __restrict__ G, int ldg, int P, int K, int N,
                                                       int p_per_split) {
  constexpr int BT_ = 128, BP = 16;
  __shared__ __align__(16) float As[BP][BT_];
  __shared__ __align__(16) float Bs[BP][BT_];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int k0 = blockIdx.x * BT_, n0 = blockIdx.y * BT_;
  const int p_begin = blockIdx.z * p_per_split;
  const int p_end = min(P, p_begin + p_per_split);
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  float4 ra[2], rb[2];
  auto load = [&](int p0) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int f = tid + i * 256, r = f >> 5, c4 = (f & 31) * 4;      // 16 rows x 32 float4
      float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = va;
      if (p0 + r < p_end) {
        if (k0 + c4 < K) {
          va = *reinterpret_cast<const float4*>(A + (size_t)(p0 + r) * lda + k0 + c4);
          if (k0 + c4 + 1 >= K) va.y = 0.f;
          if (k0 + c4 + 2 >= K) va.z = 0.f;
          if (k0 + c4 + 3 >= K) va.w = 0.f;
        }
        if (n0 + c4 < N) vb = *reinterpret_cast<const float4*>(B + (size_t)(p0 + r) * ldb + n0 + c4);
      }
      ra[i] = va; rb[i] = vb;
    }
  };
  load(p_begin);
  for (int p0 = p_begin; p0 < p_end; p0 += BP) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int f = tid + i * 256, r = f >> 5, c4 = (f & 31) * 4;
      *reinterpret_cast<float4*>(&As[r][c4]) = ra[i];
      *reinterpret_cast<float4*>(&Bs[r][c4]) = rb[i];
    }
    __syncthreads();
    if (p0 + BP < p_end) load(p0 + BP);
#pragma unroll
    for (int p = 0; p < BP; ++p) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[p][ty * 8]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[p][ty * 8 + 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[p][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[p][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int k = k0 + ty * 8 + i;
    if (k >= K) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + (j >> 2) * 64 + tx * 4 + (j & 3);
      if (n < N) atomicAdd(G + (size_t)k * ldg + n, acc[i][j]);
    }
  }
}

int sgemm_tn(const float* A, int lda, const float* B, int ldb, float* G, int ldg, int P, int K, int N, int num_sms,
             cudaStream_t st, int64_t* launches) {
  if (P <= 0 || K <= 0 || N <= 0) return 0;
  const int tiles = ((K + 127) / 128) * ((N + 127) / 128);
  int splits = (4 * num_sms + tiles - 1) / tiles;
  const int max_splits = (P + 255) / 256;
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  int per = (P + splits - 1) / splits;
  per = (per + 15) & ~15;
  splits = (P + per - 1) / per;
  dim3 grid((K + 127) / 128, (N + 127) / 128, splits);
  sgemm_tn_kernel<<<grid, 256, 0, st>>>(A, lda, B, ldb, G, ldg, P, K, N, per);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

// bias gradient: g[n] += sum_p Z[p][n]
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ Z, int ldz, int P, int N,
                                                     float* __restrict__ g, int p_per_block) {
  __shared__ float red[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int n = blockIdx.x * 32 + tx;
  const int p0 = blockIdx.y * p_per_block, p1 = min(P, p0 + p_per_block);
  float s = 0.f;
  if (n < N)
    for (int p = p0 + ty; p < p1; p += 8) s += Z[(size_t)p * ldz + n];
  red[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && n < N) {
#pragma unroll
    for (int i = 1; i < 8; ++i) s += red[i][tx];
    atomicAdd(g + n, s);
  }
}

// ------------------------------------------------------------------------------------------------ heads
// The (heads x N) linear heads evaluated in the forward epilogue (fc_alpha / fc_rgb / fc_out, src/nerf/models.py:70-80).
// dout: (P,4) = [d rgb_raw(3), d sigma].  col0: first dout column this head consumes.
// Accumulates g_head (weight rows then bias, the layout of NetDev.d_head) and, if dX != nullptr, writes
// dX[p][k] = relu'(act[p][k]) * sum_h dout[p][col0+h] * W[h][k].
// Thread layout: N/4 column threads (one float4 of the activation row each) x 1024/N row groups; every thread keeps 4 rows
// in flight (16-byte loads: 64 B per thread outstanding), the row groups are folded through shared memory before the
// atomics.  N must be a multiple of 4 and <= 256 (hidden width).
__global__ void __launch_bounds__(256) head_backward_kernel(const float* __restrict__ dout, int col0, int heads,
                                                            const float* __restrict__ act, int N, int P,
                                                            const float* __restrict__ hw, float* __restrict__ g_head,
                                                            float* __restrict__ dX, int relu_mask, int p_per_block,
                                                            float* __restrict__ g_bias) {
  __shared__ float red[256][4 * 4 + 4 + 1];
  const int nct = N >> 2;                                 // column threads per row group
  const int groups = 256 / nct;                           // row groups (N=128: 8, N=256: 4)
  const int ct = threadIdx.x % nct, grp = threadIdx.x / nct;
  const bool live = grp < groups;
  const int k = ct * 4;
  const int p0 = blockIdx.x * p_per_block, p1 = min(P, p0 + p_per_block);
  float w[4][4], gw[4][4], gb[4] = {0.f, 0.f, 0.f, 0.f}, dsum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int h = 0; h < 4; ++h)
#pragma unroll
    for (int c = 0; c < 4; ++c) { w[h][c] = (live && h < heads) ? hw[h * N + k + c] : 0.f; gw[h][c] = 0.f; }
  if (live)
    for (int pb = p0 + grp * 4; pb < p1; pb += groups * 4) {
      float4 a4[4], d4[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int p = min(pb + u, p1 - 1);
        d4[u] = *reinterpret_cast<const float4*>(dout + (size_t)p * 4);
        a4[u] = *reinterpret_cast<const float4*>(act + (size_t)p * N + k);
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int p = pb + u;
        if (p >= p1) break;
        const float dd[4] = {d4[u].x, d4[u].y, d4[u].z, d4[u].w};
        const float a[4] = {a4[u].x, a4[u].y, a4[u].z, a4[u].w};
        float dx[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          if (h >= heads) break;
          const float g = col0 ? dd[3] : dd[h];             // col0 is 0 (colour heads) or 3 (the single sigma head)
#pragma unroll
          for (int c = 0; c < 4; ++c) { gw[h][c] = fmaf(g, a[c], gw[h][c]); dx[c] = fmaf(g, w[h][c], dx[c]); }
          if (ct == 0) gb[h] += g;
        }
        if (dX) {
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            if (relu_mask && !(a[c] > 0.f)) dx[c] = 0.f;
            dsum[c] += dx[c];
          }
          *reinterpret_cast<float4*>(dX + (size_t)p * N + k) = make_float4(dx[0], dx[1], dx[2], dx[3]);
        }
      }
    }
  float* mine = red[threadIdx.x];
#pragma unroll
  for (int h = 0; h < 4; ++h)
#pragma unroll
    for (int c = 0; c < 4; ++c) mine[h * 4 + c] = gw[h][c];
#pragma unroll
  for (int c = 0; c < 4; ++c) mine[16 + c] = dsum[c];
  __syncthreads();
  // fold the row groups: 20 slots (16 head-weight partials, 4 column sums) x nct column threads
  for (int item = threadIdx.x; item < nct * 20; item += 256) {
    const int c_t = item % nct, slot = item / nct;        // slot: 0..15 = gw[h][c], 16..19 = dsum[c]
    float acc = 0.f;
    for (int g2 = 0; g2 < groups; ++g2) acc += red[g2 * nct + c_t][slot];
    if (slot < 16) {
      const int h = slot >> 2, c = slot & 3;
      if (h < heads) atomicAdd(g_head + h * N + c_t * 4 + c, acc);
    } else if (g_bias && dX) {
      atomicAdd(g_bias + c_t * 4 + (slot - 16), acc);
    }
  }
  // head bias gradient (sum of the upstream gradient columns): the ct == 0 thread of every group holds a partial
  __syncthreads();
  if (ct == 0 && live)
#pragma unroll
    for (int h = 0; h < 4; ++h) red[grp][h] = gb[h];
  __syncthreads();
  if (threadIdx.x < heads) {
    float acc = 0.f;
    for (int g2 = 0; g2 < groups; ++g2) acc += red[g2][threadIdx.x];
    atomicAdd(g_head + heads * N + threadIdx.x, acc);
  }
}

// ------------------------------------------------------------------------------------------------ compositor adjoint
// VolumeRenderer.forward (src/nerf/modules.py:67-121) differentiated w.r.t. the raw network outputs, for a loss that
// reads rgb_map only (model_nerf.py:118-126).  raw = (sigmoid rgb, raw sigma) as the forward kernels store it.
// Same arithmetic / noise stream as composite_kernel (nm_render.cu).
struct CompositeBwdArgs {
  const float* raw;   // (R,S,4)
  const float* t;     // (R,S)
  const float* dirs;  // (R,3)
  const float* d_rgb; // (R,3)
  long long R;
  int S;
  float noise_std;
  uint64_t seed;
  int white_bg;
  float* scratch;     // (R,S) transmittance
  float* dout;        // (R,S,4), or (M,4) with pos
  const int* pos;     // compact variant: exclusive scan of the evaluated marks (R*S + 1); sample m is evaluated iff
                      // pos[m+1] > pos[m], and its row goes to dout[pos[m]] (a skipped sample's is dropped: it is zero)
};

// One WARP per ray (a training chunk has a few thousand rays: a thread per ray leaves the GPU idle behind a serial
// 2 x S-step dependency chain).  Lane l owns the contiguous samples [l*seg, (l+1)*seg): transmittance = exclusive product
// scan of the segment products across lanes times the running product inside the segment; the suffix sum the same way
// from the other end.  Association differs from the forward kernel's serial product by rounding only.
// kCompact: the training pass of empty-space skipping — the same arithmetic, only the rows of evaluated samples are
// stored, in index-list order, for the network backward over the staged points.
constexpr int kCbSeg = 16;                  // samples per lane held in registers: S <= 512
template <bool kCompact>
__global__ void __launch_bounds__(128) composite_backward_kernel(const __grid_constant__ CompositeBwdArgs a) {
  const long long ray = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (ray >= a.R) return;
  const int lane = threadIdx.x & 31;
  const int S = a.S;
  const int seg = (S + 31) / 32;
  const int i0 = lane * seg, i1 = min(S, i0 + seg);
  const float4* raw = reinterpret_cast<const float4*>(a.raw) + ray * S;
  const float* t = a.t + ray * S;
  float4* dout = reinterpret_cast<float4*>(a.dout) + ray * S;
  const float dx = a.dirs[3 * ray], dy = a.dirs[3 * ray + 1], dz = a.dirs[3 * ray + 2];
  const float nrm = sqrtf(dx * dx + dy * dy + dz * dz);
  const float gr = a.d_rgb[3 * ray], gg = a.d_rgb[3 * ray + 1], gb = a.d_rgb[3 * ray + 2];
  const float gbg = a.white_bg ? (gr + gg + gb) : 0.f;
  float4 q[kCbSeg];
  float dist[kCbSeg], pre[kCbSeg], keep[kCbSeg];
  float prod = 1.0f;
#pragma unroll
  for (int u = 0; u < kCbSeg; ++u) {
    const int i = i0 + u;
    if (u < seg && i < i1) {
      q[u] = raw[i];
      dist[u] = ((i + 1 < S) ? (t[i + 1] - t[i]) : 1e10f) * nrm;
      float sg = q[u].w;
      if (a.noise_std > 0.f) sg = __fadd_rn(sg, __fmul_rn(randn(a.seed, (uint64_t)(ray * S + i)), a.noise_std));   // as comp_step
      pre[u] = sg;
      const float alpha = 1.0f - expf(-fmaxf(sg, 0.f) * dist[u]);
      keep[u] = 1.0f - alpha + 1e-10f;
      prod *= keep[u];
    }
  }
  // exclusive product scan over lanes
  float incl = prod;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl *= v;
  }
  float T = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) T = 1.0f;
  float Ti[kCbSeg], gsum = 0.f;
#pragma unroll
  for (int u = 0; u < kCbSeg; ++u) {
    const int i = i0 + u;
    if (u < seg && i < i1) {
      Ti[u] = T;
      const float alpha = 1.0f - expf(-fmaxf(pre[u], 0.f) * dist[u]);
      const float G = (gr * q[u].x + gg * q[u].y + gb * q[u].z) - gbg;
      gsum += G * alpha * T;
      T *= keep[u];
    }
  }
  // exclusive suffix sum over lanes: sum of G_j w_j of all samples in higher lanes
  float sincl = gsum;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float v = __shfl_down_sync(0xffffffffu, sincl, o);
    if (lane + o < 32) sincl += v;
  }
  float suffix = __shfl_down_sync(0xffffffffu, sincl, 1);
  if (lane == 31) suffix = 0.f;
#pragma unroll
  for (int u = kCbSeg - 1; u >= 0; --u) {
    const int i = i0 + u;
    if (u < seg && i < i1) {
      const float sg = fmaxf(pre[u], 0.f);
      const float e = expf(-sg * dist[u]);
      const float alpha = 1.0f - e;
      const float w = alpha * Ti[u];
      const float G = (gr * q[u].x + gg * q[u].y + gb * q[u].z) - gbg;        // dL/dw_i
      const float dalpha = G * Ti[u] - suffix / (1.0f - alpha + 1e-10f);
      suffix = suffix + G * w;
      float4 o;
      o.x = gr * w * q[u].x * (1.0f - q[u].x);                               // through the sigmoid
      o.y = gg * w * q[u].y * (1.0f - q[u].y);
      o.z = gb * w * q[u].z * (1.0f - q[u].z);
      o.w = (pre[u] > 0.f) ? dalpha * dist[u] * e : 0.f;                     // relu, alpha = 1 - exp(-sigma dist)
      if (!isfinite(o.w)) o.w = 0.f;                                         // dist = 1e10 on the last sample: 1e10 * 0
      if (kCompact) {
        const int p = a.pos[ray * S + i];
        if (a.pos[ray * S + i + 1] != p) reinterpret_cast<float4*>(a.dout)[p] = o;
      } else {
        dout[i] = o;
      }
    }
  }
}

// MSE loss (torch.nn.functional.mse_loss, mean over R_total*3 elements) and its gradient w.r.t. rgb_map
__global__ void mse_grad_kernel(const float* __restrict__ rgb, const float* __restrict__ target, long long n,
                                float inv_count, float* __restrict__ d_rgb, float* __restrict__ loss) {
  __shared__ float red[256];
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  float sq = 0.f;
  if (i < n) {
    const float d = rgb[i] - target[i];
    d_rgb[i] = 2.0f * d * inv_count;
    sq = d * d * inv_count;
  }
  red[threadIdx.x] = sq;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0 && loss) atomicAdd(loss, red[0]);
}

// Seed of the density-gradient chain (nm_sigma_grad): dout = (0, 0, 0, 1) per point (d raw sigma = 1) and dZ (P,N) of the
// last layer = relu'(act) * w_sigma when that layer's head carries sigma (fc_out row 3, w_sigma != nullptr), else 0 (the
// colour head: d rgb = 0; sigma enters the chain at the fc_alpha layer through dout).
__global__ void sigma_seed_kernel(long long P, int N, const float* __restrict__ act, const float* __restrict__ w_sigma,
                                  int relu, float* __restrict__ dout, float* __restrict__ dZ) {
  const long long n = P * N;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i / N;
    const int k = (int)(i - p * N);
    if (k == 0) reinterpret_cast<float4*>(dout)[p] = make_float4(0.f, 0.f, 0.f, 1.f);
    dZ[i] = (w_sigma && !(relu && !(act[i] > 0.f))) ? w_sigma[k] : 0.f;
  }
}

}  // namespace


// ------------------------------------------------------------------------------------------------ host side
namespace {

constexpr size_t kAlign = 1024;
size_t up(size_t x) { return (x + kAlign - 1) / kAlign * kAlign; }

// workspace carving for one sub-chunk of P points (all regions 1 KB aligned; ptile packs need it)
struct TrainWs {
  float *pe_x, *pe_d, *dbuf[2], *act[kMaxLayers];
  uint8_t *pkt_act[kMaxLayers], *pkt_pex, *pkt_ped;   // K-major bf16 packs of the activations / encodings (B operands of dW)
  uint8_t* pkt_dz[kMaxLayers];    // MN-major bf16 packs of every layer's dZ (A operands of dW)
  uint16_t* bits[kMaxLayers];     // relu masks of the forward's activations, 1 bit per element
  size_t bytes;
};

TrainWs carve(const NetProgram& G, long long P, bool use_tc, uint8_t* base) {
  TrainWs w{};
  size_t off = 0;
  auto take = [&](size_t bytes) { uint8_t* p = base ? base + off : nullptr; off += up(bytes); return p; };
  const int h = G.hidden;
  if (use_tc) {
    // fp32 only where the SIMT head kernels read or write (dZ of the last layer, the activations under a head); the rest
    // lives in the operand packs and relu masks
    w.dbuf[0] = (float*)take((size_t)P * h * 4);
    for (int l = 0; l < G.n_layers; ++l)
      if (G.layers[l].kind != KIND_HIDDEN) w.act[l] = (float*)take((size_t)P * G.layers[l].n_out * 4);
    const int P128 = (int)((P + 127) / 128) * 128;     // K blocks of the point-major packs come in pairs (one per 128-row tile)
    for (int l = 0; l + 1 < G.n_layers; ++l) w.pkt_act[l] = take(pack_bytes(G.layers[l].n_out, P128));
    w.pkt_pex = take(pack_bytes(kPeLd, P128));
    w.pkt_ped = take(pack_bytes(kPeLd, P128));
    for (int l = 0; l < G.n_layers; ++l) w.bits[l] = (uint16_t*)take((size_t)P * (G.layers[l].n_out / 16) * 2);
    for (int l = 0; l < G.n_layers; ++l) w.pkt_dz[l] = take(pack_bytes(G.layers[l].n_out, P128));
  } else {
    w.pe_x = (float*)take((size_t)P * kPeLd * 4);
    w.pe_d = (float*)take((size_t)P * kPeLd * 4);
    w.dbuf[0] = (float*)take((size_t)P * h * 4);
    w.dbuf[1] = (float*)take((size_t)P * h * 4);
    for (int l = 0; l < G.n_layers; ++l) w.act[l] = (float*)take((size_t)P * G.layers[l].n_out * 4);
  }
  w.bytes = off;
  return w;
}

}  // namespace

size_t train_ws_bytes(const NetProgram& G, long long points, bool use_tc) { return carve(G, points, use_tc, nullptr).bytes; }

// The by-products a training forward must leave in `ws` (same carving as mlp_backward) so that the backward can skip its
// recompute launch: see MlpEmit.
void train_emit_setup(const NetProgram& G, long long P, float* ws_base, MlpEmit* E) {
  const TrainWs W = carve(G, P, true, reinterpret_cast<uint8_t*>(ws_base));
  *E = MlpEmit{};
  E->kbt = 2 * (int)((P + 127) / 128);
  for (int l = 0; l < G.n_layers; ++l) {
    const LayerProg& L = G.layers[l];
    if (l + 1 < G.n_layers) E->packT[l] = W.pkt_act[l];
    if (L.relu) E->bits[l] = reinterpret_cast<uint32_t*>(W.bits[l]);
    if (L.kind != KIND_HIDDEN) E->act[l] = W.act[l];
  }
}

int launch_composite_backward(const float* raw, const float* t, const float* dirs, const float* d_rgb, long long R, int S,
                              float noise_std, uint64_t seed, int white_bg, float* scratch, float* dout,
                              cudaStream_t st, int64_t* launches, const int* pos) {
  if (R <= 0) return 0;
  NM_CHECK(S <= 32 * kCbSeg, "sample count %d exceeds the compositor adjoint's limit (%d)", S, 32 * kCbSeg);
  CompositeBwdArgs a{raw, t, dirs, d_rgb, R, S, noise_std, seed, white_bg, scratch, dout, pos};
  if (pos) composite_backward_kernel<true><<<(unsigned)((R + 3) / 4), 128, 0, st>>>(a);
  else composite_backward_kernel<false><<<(unsigned)((R + 3) / 4), 128, 0, st>>>(a);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

int launch_mse_grad(const float* rgb, const float* target, long long n, long long count, float* d_rgb, float* loss,
                    cudaStream_t st, int64_t* launches) {
  if (n <= 0) return 0;
  mse_grad_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(rgb, target, n, 1.0f / (float)count, d_rgb, loss);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

namespace {

// Tensor cores: ONE launch of the fused forward kernel (nm_mlp_tc.cu, mode 1) leaves what the backward needs — relu masks,
// the bf16 packs of every hidden activation and the fp32 activations the head kernels read — unless the training forward
// already did (have_acts); the SIMT heads produce dZ of the last layer; ONE launch of the fused kernel on the backward
// program (mode 2) walks the data gradient down the whole network with dZ in shared memory (W^T streamed through shared
// memory, relu masks from the forward, the rank-1 d sigma term) and leaves every layer's dZ as the pack the long-K
// weight-gradient GEMMs consume — no per-layer round trip of dZ through HBM.
int backward_tc(NetDev& net, const MlpInput& in, const float* dout, float* ws_base, NetGrads* g, int num_sms,
                const TrainMode& mode, cudaStream_t st, int64_t* launches, int have_acts) {
  const NetProgram& G = net.full;
  const int P = (int)in.M;
  const TrainWs W = carve(G, P, true, reinterpret_cast<uint8_t*>(ws_base));
  const int kbtP = 2 * ((P + 127) / 128);      // K blocks of the point-major packs (zero-filled beyond P)
  NM_CHECK(G.dim_xyz <= kPeLd && G.dim_dir <= kPeLd, "encoding wider than %d", kPeLd);
  encode_pack_kernel<<<kbtP, 256, 0, st>>>(in, net.d_full, W.pkt_pex, W.pkt_ped);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  if (!have_acts) {
    MlpEmit E{};
    train_emit_setup(G, P, ws_base, &E);
    if (int e = launch_mlp_tc(net, false, mode.n_passes, 0, in, nullptr, num_sms, mode.d_err, st, launches, &E)) return e;
  }

  size_t gw_off[kMaxLayers];
  int gw_ld[kMaxLayers];
  grad_layout(G, gw_off, gw_ld);
  if (!net.bwd_valid)
    if (int e = build_backward_stream(&net, st, launches)) return e;
  const int last = G.n_layers - 1;
  const LayerProg& Ltop = G.layers[last];
  NM_CHECK(Ltop.kind == KIND_RGB || Ltop.kind == KIND_OUT4, "the last layer must carry the colour head");
  const int p_per_block = (P + 8 * num_sms - 1) / (8 * num_sms);
  const int hb_blocks = (P + p_per_block - 1) / p_per_block;
  NM_CHECK((Ltop.n_out & 3) == 0 && Ltop.n_out <= 1024 && (G.hidden & 3) == 0 && G.hidden <= 1024, "head widths must be multiples of 4, <= 1024");
  float* dZ = W.dbuf[0];
  head_backward_kernel<<<hb_blocks, 256, 0, st>>>(dout, 0, Ltop.kind == KIND_RGB ? 3 : 4, W.act[last], Ltop.n_out, P,
                                                 net.d_head + Ltop.head_off, g->head + Ltop.head_off, dZ, Ltop.relu, p_per_block,
                                                 g->bias + Ltop.bias_off);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  for (int l = 0; l < last; ++l) {
    const LayerProg& L = G.layers[l];
    if (L.kind != KIND_SIGMA) continue;       // weight / bias gradient of fc_alpha (its data-gradient term is in the chain)
    head_backward_kernel<<<hb_blocks, 256, 0, st>>>(dout, 3, 1, W.act[l], L.n_out, P, net.d_head + L.head_off,
                                                   g->head + L.head_off, nullptr, 0, p_per_block, nullptr);
    NM_CUDA(cudaGetLastError());
    if (launches) ++*launches;
  }
  MlpEmit io{};
  io.kbt = kbtP;
  io.packT[0] = W.pkt_dz[last];               // the chain's load stage emits the top dZ's pack too
  for (int li = 1; li < net.bwd.n_layers; ++li) {
    const int l = net.bwd.layers[li].aux;      // this backward layer streams W_l^T and produces dZ of forward layer l-1
    io.packT[li] = W.pkt_dz[l - 1];
    if (G.layers[l - 1].relu) io.bits[li] = reinterpret_cast<uint32_t*>(W.bits[l - 1]);
  }
  if (int e = launch_mlp_tc_bwd(net, P, dZ, Ltop.n_out, dout, io, mode.n_passes, num_sms, mode.d_err, st, launches)) return e;
  for (int l = last; l >= 0; --l) {            // weight gradients dW (N, Kt) += dZ^T [act[l-1] | PE]: long-K GEMMs, fp32 atomics
    const LayerProg& L = G.layers[l];
    TcGemmParams T{};
    T.a = W.pkt_dz[l]; T.kbt = kbtP; T.n_passes = mode.n_passes; T.err = mode.d_err;
    T.ldd = gw_ld[l]; T.M = L.n_out;
    // bias gradient = row sums of dZ^T, taken by the first GEMM that stages this layer's dZ pack (the top layer's comes
    // from head_backward_kernel)
    T.a_rowsum = l < last ? g->bias + L.bias_off : nullptr;
    if (L.k_act > 0) {
      T.b = W.pkt_act[l - 1]; T.D = g->w + gw_off[l]; T.N = L.k_act;
      if (int e = launch_tc_gemm(T, num_sms, st, launches)) return e;
      T.a_rowsum = nullptr;
    }
    if (L.pe_src) {
      T.b = L.pe_src == SRC_PE_XYZ ? W.pkt_pex : W.pkt_ped; T.D = g->w + gw_off[l] + L.k_act; T.N = L.k_pe;
      if (int e = launch_tc_gemm(T, num_sms, st, launches)) return e;
    }
  }
  return 0;
}

// NM_PREC_FP32 forward recompute: the encodings, then act[l] = act_l([act[l-1] | PE] W^T + b) layer by layer in fp32 FMAs
// on the CUDA cores.
int forward_fp32(NetDev& net, const MlpInput& in, const TrainWs& W, cudaStream_t st, int64_t* launches) {
  const NetProgram& G = net.full;
  const int P = (int)in.M;
  encode_kernel<<<(P + 127) / 128, 128, 0, st>>>(in, net.d_full, W.pe_x, W.pe_d);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  auto pe_of = [&](const LayerProg& L) { return L.pe_src == SRC_PE_XYZ ? W.pe_x : W.pe_d; };
  for (int l = 0; l < G.n_layers; ++l) {
    const LayerProg& L = G.layers[l];
    const int N = L.n_out;
    GemmEpi fin{};
    fin.bias = net.d_bias + L.bias_off; fin.relu = L.relu;
    const float* Wt = net.d_wt + L.wt_off;
    if (L.k_act > 0) {
      GemmEpi e0 = L.pe_src ? GemmEpi{} : fin;
      if (int rc = sgemm<false>(W.act[l - 1], G.layers[l - 1].n_out, Wt, N, W.act[l], N, P, N, L.k_act, e0, st, launches)) return rc;
    }
    if (L.pe_src) {
      fin.accumulate = L.k_act > 0 ? 1 : 0;
      if (int rc = sgemm<false>(pe_of(L), kPeLd, Wt + (size_t)L.k_act * N, N, W.act[l], N, P, N, L.k_pe, fin, st, launches)) return rc;
    }
  }
  return 0;
}

// NM_PREC_FP32: forward recompute and the backward layer by layer, every GEMM in fp32 FMAs on the CUDA cores.
int backward_fp32(NetDev& net, const MlpInput& in, const float* dout, float* ws_base, NetGrads* g, int num_sms,
                  cudaStream_t st, int64_t* launches) {
  const NetProgram& G = net.full;
  const int P = (int)in.M;
  const TrainWs W = carve(G, P, false, reinterpret_cast<uint8_t*>(ws_base));
  auto pe_of = [&](const LayerProg& L) { return L.pe_src == SRC_PE_XYZ ? W.pe_x : W.pe_d; };
  if (int rc = forward_fp32(net, in, W, st, launches)) return rc;

  size_t gw_off[kMaxLayers];
  int gw_ld[kMaxLayers];
  grad_layout(G, gw_off, gw_ld);
  int cur = 0;
  bool bias_done = false;      // the kernel that produced dbuf[cur] already accumulated its column sums (bias gradient)
  const int p_per_block = (P + 8 * num_sms - 1) / (8 * num_sms);      // 8 CTAs per SM keep enough loads in flight
  const int hb_blocks = (P + p_per_block - 1) / p_per_block;
  for (int l = 0; l < G.n_layers; ++l)
    NM_CHECK(G.layers[l].kind == KIND_HIDDEN || ((G.layers[l].n_out & 3) == 0 && G.layers[l].n_out <= 1024), "head widths must be multiples of 4, <= 1024");
  for (int l = G.n_layers - 1; l >= 0; --l) {
    const LayerProg& L = G.layers[l];
    const int N = L.n_out;
    float* dZ = W.dbuf[cur];
    if (L.kind == KIND_RGB || L.kind == KIND_OUT4) {
      NM_CHECK(l == G.n_layers - 1, "rgb head must be the last layer");
      const int heads = L.kind == KIND_RGB ? 3 : 4;
      head_backward_kernel<<<hb_blocks, 256, 0, st>>>(dout, 0, heads, W.act[l], N, P, net.d_head + L.head_off,
                                                     g->head + L.head_off, dZ, L.relu, p_per_block, g->bias + L.bias_off);
      bias_done = true;
      NM_CUDA(cudaGetLastError());
      if (launches) ++*launches;
    } else if (L.kind == KIND_SIGMA) {
      // weight/bias gradient of fc_alpha; its contribution to dZ was added by the fc_feat data-grad epilogue
      head_backward_kernel<<<hb_blocks, 256, 0, st>>>(dout, 3, 1, W.act[l], N, P, net.d_head + L.head_off,
                                                     g->head + L.head_off, nullptr, 0, p_per_block, nullptr);
      NM_CUDA(cudaGetLastError());
      if (launches) ++*launches;
    }
    // weight gradient dW (N, Kt) += dZ^T [act[l-1] | PE], bias gradient
    float* gW = g->w + gw_off[l];
    const int ldg = gw_ld[l];
    if (L.k_act > 0)
      if (int rc = sgemm_tn(dZ, N, W.act[l - 1], G.layers[l - 1].n_out, gW, ldg, P, N, L.k_act, num_sms, st, launches)) return rc;
    if (L.pe_src)
      if (int rc = sgemm_tn(dZ, N, pe_of(L), kPeLd, gW + L.k_act, ldg, P, N, L.k_pe, num_sms, st, launches)) return rc;
    if (!bias_done) {
      const int ppb = (P + 63) / 64;
      dim3 grid((N + 31) / 32, (P + ppb - 1) / ppb);
      colsum_kernel<<<grid, 256, 0, st>>>(dZ, N, P, N, g->bias + L.bias_off, ppb);
      NM_CUDA(cudaGetLastError());
      if (launches) ++*launches;
    }
    // data gradient into the previous layer's pre-activation: dX (P,k_act) = dZ (P,N) W[:, :k_act]
    if (l > 0) {
      const LayerProg& Lp = G.layers[l - 1];
      NM_CHECK(L.k_act == Lp.n_out, "layer chain mismatch");
      GemmEpi e{};
      if (Lp.kind == KIND_SIGMA) { e.r1_vec = dout + 3; e.r1_stride = 4; e.r1_w = net.d_head + Lp.head_off; }
      if (Lp.relu) { e.mask = W.act[l - 1]; e.ldmask = Lp.n_out; }
      // W[n][k] = Wt[k][n]  ->  B = Wt rows 0..k_act-1 viewed (k_act, N), read transposed
      if (int rc = sgemm<true>(dZ, N, net.d_wt + L.wt_off, N, W.dbuf[cur ^ 1], L.k_act, P, L.k_act, N, e, st, launches)) return rc;
      bias_done = false;
      cur ^= 1;
    }
  }
  return 0;
}

}  // namespace

// Backward of one network over P = in.M points.  dout (P,4).  ws: train_ws_bytes(full, P, use_tc) bytes, 1 KB aligned.
// Weight gradients accumulate in the reference's (out,in) layout at the offsets of NetDev.d_w.
int mlp_backward(NetDev& net, const MlpInput& in, const float* dout, float* ws_base, NetGrads* g, int num_sms,
                 const TrainMode& mode, cudaStream_t st, int64_t* launches, int have_acts) {
  if (in.M <= 0) return 0;
  if (mode.use_tc) return backward_tc(net, in, dout, ws_base, g, num_sms, mode, st, launches, have_acts);
  return backward_fp32(net, in, dout, ws_base, g, num_sms, st, launches);
}

// ------------------------------------------------------------------------------------------------ density gradient
// g = d raw sigma / d p (DESIGN 4.8): the training backward's data-gradient chain seeded with d raw sigma = 1 and no
// weight- or head-gradient work, then the input tail dPE = sum dZ_l W_l[:, PE] over the xyz-reading layers and the encoding
// Jacobian.  Workspace: the backward's carving for P points, dout (P,4), then the packed B tiles (tensor cores) or the
// fp32 dPE (P, kPeLd).
namespace {

int sigma_xyz_kblocks(const NetProgram& G) {
  int n = 0;
  for (int l = 0; l < G.n_layers; ++l)
    if (G.layers[l].pe_src == SRC_PE_XYZ) n += G.layers[l].n_out / 64;
  return n;
}

int launch_sigma_seed(const NetDev& net, const TrainWs& W, long long P, float* dout, cudaStream_t st, int64_t* launches) {
  const NetProgram& G = net.full;
  const int last = G.n_layers - 1;
  const LayerProg& Ltop = G.layers[last];
  NM_CHECK(Ltop.kind == KIND_RGB || Ltop.kind == KIND_OUT4, "the last layer must carry the colour head");
  const float* w_sigma = Ltop.kind == KIND_OUT4 ? net.d_head + Ltop.head_off + 3 * Ltop.n_out : nullptr;
  const long long n = P * Ltop.n_out;
  const long long blocks = (n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096;
  sigma_seed_kernel<<<(unsigned)blocks, 256, 0, st>>>(P, Ltop.n_out, W.act[last], w_sigma, Ltop.relu, dout, W.dbuf[0]);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

PeDesc pe_desc(const NetProgram& G) {
  PeDesc d{};
  d.L = G.L_xyz; d.inc = G.inc_xyz;
  for (int k = 0; k < kMaxFreq; ++k) d.freq[k] = G.freq_xyz[k];
  return d;
}

// Tensor cores: mode-1 forward (relu masks, activation packs), the mode-2 chain (dZ packs of every layer), the wgmma tail.
int sigma_grad_tc(NetDev& net, const MlpInput& in, uint8_t* ws, float* grad, int num_sms, const TrainMode& mode,
                  cudaStream_t st, int64_t* launches) {
  const NetProgram& G = net.full;
  const int P = (int)in.M;
  const TrainWs W = carve(G, P, true, ws);
  float* dout = reinterpret_cast<float*>(ws + W.bytes);
  uint8_t* bpack = ws + W.bytes + up((size_t)P * 16);
  const int kbtP = 2 * ((P + 127) / 128);
  MlpEmit E{};
  train_emit_setup(G, P, reinterpret_cast<float*>(ws), &E);
  if (int e = launch_mlp_tc(net, false, mode.n_passes, 0, in, nullptr, num_sms, mode.d_err, st, launches, &E)) return e;
  if (!net.bwd_valid)
    if (int e = build_backward_stream(&net, st, launches)) return e;
  if (int e = launch_sigma_seed(net, W, P, dout, st, launches)) return e;
  const int last = G.n_layers - 1;
  MlpEmit io{};
  io.kbt = kbtP;
  io.packT[0] = W.pkt_dz[last];
  for (int li = 1; li < net.bwd.n_layers; ++li) {
    const int l = net.bwd.layers[li].aux;
    io.packT[li] = W.pkt_dz[l - 1];
    if (G.layers[l - 1].relu) io.bits[li] = reinterpret_cast<uint32_t*>(W.bits[l - 1]);
  }
  if (int e = launch_mlp_tc_bwd(net, P, W.dbuf[0], G.layers[last].n_out, dout, io, mode.n_passes, num_sms, mode.d_err, st, launches))
    return e;
  // the tail's K-blocks: every 64-feature group of every xyz-reading layer, layers in forward order
  SigmaGradWeights Wb{};
  SigmaGradTail T{};
  int kb = 0;
  for (int l = 0; l < G.n_layers; ++l) {
    const LayerProg& L = G.layers[l];
    if (L.pe_src != SRC_PE_XYZ) continue;
    NM_CHECK(L.k_pe == G.dim_xyz && L.n_out % 64 == 0, "layer %d: unexpected xyz encoding block", l);
    for (int fg = 0; fg < L.n_out / 64; ++fg, ++kb) {
      NM_CHECK(kb < kSgMaxKb, "density gradient: more than %d K-blocks", kSgMaxKb);
      T.a[kb] = W.pkt_dz[l] + (size_t)(fg >> 1) * kbtP * kPtileBytes + (size_t)(fg & 1) * 8192u;
      Wb.wt[kb] = net.d_wt + L.wt_off + (size_t)L.k_act * L.n_out + fg * 64;
      Wb.ld[kb] = L.n_out;
    }
  }
  Wb.k_pe = G.dim_xyz; Wb.out = bpack;
  T.b = bpack; T.n_kb = kb; T.n_passes = mode.n_passes; T.M = P; T.pts = in.pts; T.pe = pe_desc(G); T.grad = grad;
  T.err = mode.d_err;
  return launch_sigma_grad_tail(Wb, T, num_sms, st, launches);
}

// NM_PREC_FP32: the SIMT recompute, the data-gradient half of backward_fp32's layer loop with dPE taken (sgemm) from the dZ of
// every xyz-reading layer as the walk passes it, then the same Jacobian contraction.
int sigma_grad_fp32(NetDev& net, const MlpInput& in, uint8_t* ws, float* grad, cudaStream_t st, int64_t* launches) {
  const NetProgram& G = net.full;
  const int P = (int)in.M;
  const TrainWs W = carve(G, P, false, ws);
  float* dout = reinterpret_cast<float*>(ws + W.bytes);
  float* dpe = reinterpret_cast<float*>(ws + W.bytes + up((size_t)P * 16));
  if (int rc = forward_fp32(net, in, W, st, launches)) return rc;
  if (int rc = launch_sigma_seed(net, W, P, dout, st, launches)) return rc;
  int cur = 0;
  bool first = true;
  for (int l = G.n_layers - 1; l >= 0; --l) {
    const LayerProg& L = G.layers[l];
    const int N = L.n_out;
    float* dZ = W.dbuf[cur];
    if (L.pe_src == SRC_PE_XYZ) {       // dPE (+)= dZ_l W_l[:, k_act, k_act + k_pe)
      GemmEpi e{};
      e.accumulate = first ? 0 : 1;
      if (int rc = sgemm<true>(dZ, N, net.d_wt + L.wt_off + (size_t)L.k_act * N, N, dpe, kPeLd, P, L.k_pe, N, e, st, launches)) return rc;
      first = false;
    }
    if (l > 0) {                        // dZ of layer l-1, as backward_fp32
      const LayerProg& Lp = G.layers[l - 1];
      NM_CHECK(L.k_act == Lp.n_out, "layer chain mismatch");
      GemmEpi e{};
      if (Lp.kind == KIND_SIGMA) { e.r1_vec = dout + 3; e.r1_stride = 4; e.r1_w = net.d_head + Lp.head_off; }
      if (Lp.relu) { e.mask = W.act[l - 1]; e.ldmask = Lp.n_out; }
      if (int rc = sgemm<true>(dZ, N, net.d_wt + L.wt_off, N, W.dbuf[cur ^ 1], L.k_act, P, L.k_act, N, e, st, launches)) return rc;
      cur ^= 1;
    }
  }
  NM_CHECK(!first, "no layer reads the xyz encoding");
  return launch_pe_vjp(in.pts, P, dpe, kPeLd, pe_desc(G), grad, st, launches);
}

}  // namespace

size_t sigma_grad_ws_bytes(const NetProgram& G, long long points, bool use_tc) {
  const size_t tail = use_tc ? (size_t)sigma_xyz_kblocks(G) * 16384 : (size_t)points * kPeLd * 4;
  return carve(G, points, use_tc, nullptr).bytes + up((size_t)points * 16) + up(tail);
}

int sigma_grad(NetDev& net, const float* pts, long long M, float* ws, float* grad, int num_sms, const TrainMode& mode,
               cudaStream_t st, int64_t* launches) {
  if (M <= 0) return 0;
  NM_CHECK(M <= INT32_MAX, "density gradient: chunk of %lld points", M);
  NM_CHECK(net.full.dim_xyz <= kPeLd, "encoding wider than %d", kPeLd);
  MlpInput in{};
  in.mode = IN_POINTS; in.pts = pts; in.dirs = nullptr; in.M = M;     // directions = positions, as in the grid sweep
  uint8_t* base = reinterpret_cast<uint8_t*>(ws);
  if (mode.use_tc) return sigma_grad_tc(net, in, base, grad, num_sms, mode, st, launches);
  return sigma_grad_fp32(net, in, base, grad, st, launches);
}

}  // namespace nm
