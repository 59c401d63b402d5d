// wgmma GEMM for the weight gradients of the training backward (nm_train.cu): D (M,N) += A (M,K) * B (N,K)^T with K = the
// points of the step, both operands given as pre-packed hi/lo "ptiles" and fp32 accumulation in registers.  fp32 accuracy
// class comes from the same operand split the forward kernel uses (x = hi + lo, three MMAs per product: hi*hi + lo*hi +
// hi*lo).  Halves are bf16: gradients span fp32's exponent range (16 significand bits per operand, ~2^-16 per product).
//
// ptile = one (128 operand rows) x (64 K) block: [hi | lo], each 16 KB, 128-byte swizzled — the shared-memory image wgmma
// reads through a descriptor, so a ptile moves global -> shared with ONE 32 KB cp.async.bulk.  A pack is ptiles ordered
// [row block][K block].  A (dZ^T) comes as MN-major ptiles, written by the data-gradient chain (nm_mlp_tc.cu mode 2);
// B (activations, encodings) as K-major ptiles, written by the training forward (mode 1) and encode_pack_kernel.
//
// Kernel: 12 warps — two consumer warpgroups (rows 0-63 / 64-127 of the 128-row tile; m64n128k16 wgmmas into 64 (NB=1)
// or 128 (NB=2) accumulator registers per thread, then the epilogue from those registers), and a producer warpgroup
// whose first warp issues the bulk copies into a ring of K-block stages (2 x 96 KB for 256-wide tiles, 3 x 64 KB for
// 128-wide).  One tile per CTA: K is split over one wave of CTAs, which reduce into D with vector atomics.  Barriers:
// full[s] (tx bytes), empty[s] (one arrival per consumer warpgroup once its wgmmas on the stage are complete).  With
// a_rowsum the consumers also sum the rows of the staged A tiles (the bias gradient when A = dZ^T).
#include <cuda_bf16.h>

#include <cstdlib>

#include "nm_common.h"
#include "nm_gemm.h"
#include "nm_ptx.cuh"

namespace nm {
namespace {

constexpr int kGemmThreads = 384;   // warps 0-3, 4-7 consumers; 8-11 producer warpgroup (warp 8 issues)
constexpr int kProdWarp = 8;

// x = hi + lo in two bf16 (8+8 significand bits, fp32's exponent range)
__device__ __forceinline__ void split_bf16(float x, uint16_t* hi, uint16_t* lo) {
  const __nv_bfloat16 h = __float2bfloat16_rn(x);
  const __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
  *hi = __bfloat16_as_ushort(h); *lo = __bfloat16_as_ushort(l);
}

constexpr uint32_t kStgOff = 6u * kPtileBytes;                       // epilogue staging: 8 warps x 16 rows x 17 floats
constexpr uint32_t kStgWarp = 16u * 17u * 4u;
constexpr uint32_t kBarOff = kStgOff + 8u * kStgWarp;                // barriers behind the 1024-aligned stages
constexpr uint32_t kGemmSmem = kBarOff + 128u;

// One K block of the tile: every pass of the four K=16 steps into the NB accumulators (MN-major A, K-major B).
template <int NB>
__device__ __forceinline__ void mma_kblock(float (&acc)[2][64], uint32_t a, uint32_t stage, int nbv, int n_passes) {
  const uint64_t a_hi = ptx::make_mnmajor_sw128_desc(a), a_lo = ptx::make_mnmajor_sw128_desc(a + kPtileHalf);
  constexpr uint64_t a_step = 128u, b_step = 2u;   // per k16: 2048 B (MN-major) / 32 B (K-major)
#pragma unroll
  for (int j = 0; j < NB; ++j) {
    if (j >= nbv) break;
    const uint32_t bs = stage + kPtileBytes * (uint32_t)(1 + j);
    const uint64_t b_hi = ptx::make_kmajor_sw128_desc(bs), b_lo = ptx::make_kmajor_sw128_desc(bs + kPtileHalf);
#pragma unroll
    for (int k = 0; k < 4; ++k) ptx::wgmma<128, 1, 0, 1>(acc[j], a_hi + k * a_step, b_hi + k * b_step, 1u);
    if (n_passes == 3) {
#pragma unroll
      for (int k = 0; k < 4; ++k) ptx::wgmma<128, 1, 0, 1>(acc[j], a_lo + k * a_step, b_hi + k * b_step, 1u);
#pragma unroll
      for (int k = 0; k < 4; ++k) ptx::wgmma<128, 1, 0, 1>(acc[j], a_hi + k * a_step, b_lo + k * b_step, 1u);
    }
  }
}

// Epilogue of one 16-row x 16-column block of a warp, staged in stg (pitch 17): lane = (row sub = lane / 4, 4 columns
// q4 = 4 * (lane % 4)), rows sub and sub + 8, added to D.  row0: the block's first global row.
__device__ __noinline__ void epi_block(const TcGemmParams& P, const float* stg, int lane, int row0, int n0) {
  const int sub = lane >> 2, q4 = (lane & 3) * 4;
  const int n = n0 + q4;                 // first of this lane's 4 global columns
  if (n >= P.N) return;
  const bool vec_atomic = (P.ldd & 3) == 0 && (reinterpret_cast<uintptr_t>(P.D) & 15) == 0;
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const int rr = it * 8 + sub, m = row0 + rr;
    const float* sp = &stg[rr * 17 + q4];
    const float4 v = make_float4(sp[0], sp[1], sp[2], sp[3]);
    if (m < P.M) {
      float* dp = P.D + (size_t)m * P.ldd + n;
      if (vec_atomic && n + 3 < P.N) {
        atomicAdd(reinterpret_cast<float4*>(dp), v);      // one 16-byte reduction instead of four
      } else {
        atomicAdd(dp, v.x);
        if (n + 1 < P.N) atomicAdd(dp + 1, v.y);
        if (n + 2 < P.N) atomicAdd(dp + 2, v.z);
        if (n + 3 < P.N) atomicAdd(dp + 3, v.w);
      }
    }
  }
}

// One tile per CTA: (row block, column group of NB B row blocks, K split) = blockIdx.
template <int NB>
__global__ void __launch_bounds__(kGemmThreads, 1) tc_gemm_kernel(const __grid_constant__ TcGemmParams P) {
  extern __shared__ __align__(1024) uint8_t smem[];
  constexpr int NS = (NB == 2) ? 2 : 3;
  constexpr uint32_t STAGE = kPtileBytes * (1 + NB);
  const uint32_t sbase = ptx::smem_u32(smem);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const uint32_t bar0 = sbase + kBarOff;
  auto full = [&](int s) { return bar0 + 8u * s; };
  auto empty = [&](int s) { return bar0 + 8u * (NS + s); };

  const int rb = blockIdx.x, cb0 = blockIdx.y * NB;
  const int nbv = min(NB, P.n_rb_b - cb0);
  const int k0 = blockIdx.z * P.kb_per_split;                 // this split's K blocks: k0 .. k0 + nk - 1
  const int nk = min(P.kbt, k0 + P.kb_per_split) - k0;

  // with a_rowsum the CTAs of the first column group also sum the rows of every A tile they stage (bias gradient)
  const bool sum_rows = P.a_rowsum != nullptr && blockIdx.y == 0;
  if (threadIdx.x == 0) {
    if (sbase & 1023u) { if (P.err) atomicExch(P.err, 90); __trap(); }
    for (int s = 0; s < NS; ++s) { ptx::mbar_init(full(s), 1); ptx::mbar_init(empty(s), 2); }
    ptx::fence_mbar_init();
  }
  __syncthreads();

  if (warp >= kProdWarp) {
    // ------------------------------------------------------------ producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == kProdWarp && lane == 0) {
      for (int kk = 0; kk < nk; ++kk) {
        const int s = kk % NS;
        if (kk >= NS) ptx::mbar_wait(empty(s), (uint32_t)((kk / NS - 1) & 1), P.err, 91);
        const int kb = k0 + kk;
        const uint32_t dst = sbase + (uint32_t)s * STAGE;
        ptx::mbar_expect_tx(full(s), kPtileBytes * (uint32_t)(1 + nbv));
        ptx::bulk_g2s(dst, P.a + ((size_t)rb * P.kbt + kb) * kPtileBytes, kPtileBytes, full(s));
        for (int j = 0; j < nbv; ++j)
          ptx::bulk_g2s(dst + kPtileBytes * (uint32_t)(1 + j), P.b + ((size_t)(cb0 + j) * P.kbt + kb) * kPtileBytes,
                        kPtileBytes, full(s));
      }
    }
    return;
  }
  // ------------------------------------------------------------ consumers: main loop, then the epilogue from the registers
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wg = warp >> 2, wi = warp & 3, t = threadIdx.x & 127;
  float* stg = reinterpret_cast<float*>(smem + kStgOff + (uint32_t)warp * kStgWarp);     // 16 rows, pitch 17 floats
  float rsum = 0.f;                                                                    // sum_rows: this thread's row part
  float acc[2][64];
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[j][i] = 0.f;
  ptx::wgmma_fence();
  int prev = -1;
  for (int kk = 0; kk < nk; ++kk) {
    const int s = kk % NS;
    ptx::mbar_wait(full(s), (uint32_t)((kk / NS) & 1), P.err, 92);
    const uint32_t st = sbase + (uint32_t)s * STAGE;
    if (sum_rows) {
      // Row sums of the A tile (this warpgroup's 64 rows) while the tensor cores consume it; hi + lo halves.
      // MN-major: [feature group of 64][K row (point) 0..63][128 B = 8 chunks of 8 features, chunk ^= row & 7]
      const uint8_t* at = smem + (size_t)s * STAGE;
      const int f = t & 63, kr0 = (t >> 6) * 32;
      for (int k = kr0; k < kr0 + 32; ++k) {
        const uint32_t off = (uint32_t)wg * 8192u + (uint32_t)k * 128u + ((((uint32_t)f >> 3) ^ ((uint32_t)k & 7u)) << 4) + (uint32_t)(f & 7) * 2u;
        const uint32_t h = *reinterpret_cast<const uint16_t*>(at + off), l = *reinterpret_cast<const uint16_t*>(at + kPtileHalf + off);
        rsum += __uint_as_float(h << 16) + __uint_as_float(l << 16);
      }
    }
    const uint32_t a = st + (uint32_t)wg * 8192u;    // rows 64..127: the second MN group of the A tile
    mma_kblock<NB>(acc, a, st, nbv, P.n_passes);
    ptx::wgmma_commit();
    ptx::wgmma_wait<1>();                              // the previous K block's MMAs are complete: release its stage
    if (prev >= 0 && t == 0) ptx::mbar_arrive(empty(prev));
    prev = s;
  }
  ptx::wgmma_wait<0>();
  if (prev >= 0 && t == 0) ptx::mbar_arrive(empty(prev));
#pragma unroll
  for (int j = 0; j < 2; ++j) ptx::fence_regs<64>(acc[j]);

  // epilogue: warp wi of warpgroup wg owns rows 16 wi .. 16 wi + 15 of the warpgroup's 64; each 16 x 16 block goes
  // through the warp's staging tile so that global accesses are contiguous row segments
  const int row0 = rb * 128 + wg * 64 + wi * 16;
  const int lr = lane >> 2, lc = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < NB; ++j) {
    if (j >= nbv) break;
#pragma unroll
    for (int blk = 0; blk < 8; ++blk) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int q = 0; q < 4; ++q)
          stg[(lr + 8 * (q >> 1)) * 17 + h * 8 + lc + (q & 1)] = acc[j][(blk * 2 + h) * 4 + q];
      __syncwarp();
      epi_block(P, stg, lane, row0, (cb0 + j) * 128 + blk * 16);
      __syncwarp();
    }
  }
  if (sum_rows) {
    const int row = rb * 128 + wg * 64 + (t & 63);
    if (row < P.M) atomicAdd(P.a_rowsum + row, rsum);
  }
}

// ------------------------------------------------------------------------------------------------ packers
// The packers of nm_debug_gemm's operands (debug_tc_gemm below).  In training the kernels that produce the operands
// write their packs themselves.
// K-major: operand row r = source column f (f < F valid), K index = source row p (p < P).  grid (K blocks over points,
// row blocks over features); the 64 x 128 fp32 source block goes through shared memory.
__global__ void __launch_bounds__(256) pack_cols_kernel(const float* __restrict__ src, int ld, int P, int F,
                                                        uint8_t* __restrict__ out, int kbt) {
  __shared__ float t[64][129];
  const int kb = blockIdx.x, rb = blockIdx.y;
  uint8_t* tile = out + ((size_t)rb * kbt + kb) * kPtileBytes;
  const bool vec = (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0 && rb * 128 + 128 <= F;
  if (vec) {
    for (int e = threadIdx.x; e < 64 * 32; e += 256) {           // 64 points x 32 float4
      const int p = e >> 5, f4 = (e & 31) * 4;
      const int gp = kb * 64 + p;
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gp < P) x = *reinterpret_cast<const float4*>(src + (size_t)gp * ld + rb * 128 + f4);
      t[p][f4] = x.x; t[p][f4 + 1] = x.y; t[p][f4 + 2] = x.z; t[p][f4 + 3] = x.w;
    }
  } else {
    for (int e = threadIdx.x; e < 64 * 128; e += 256) {
      const int p = e >> 7, f = e & 127;
      const int gp = kb * 64 + p, gf = rb * 128 + f;
      t[p][f] = (gp < P && gf < F) ? src[(size_t)gp * ld + gf] : 0.f;
    }
  }
  __syncthreads();
  const int c8 = threadIdx.x & 7;
#pragma unroll
  for (int pass = 0; pass < 4; ++pass) {
    const int r = pass * 32 + (threadIdx.x >> 3);
    __align__(16) uint16_t hi[8], lo[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) split_bf16(t[c8 * 8 + i][r], &hi[i], &lo[i]);
    const uint32_t off = (uint32_t)r * 128u + (uint32_t)((c8 ^ (r & 7)) << 4);
    *reinterpret_cast<uint4*>(tile + off) = *reinterpret_cast<const uint4*>(hi);
    *reinterpret_cast<uint4*>(tile + kPtileHalf + off) = *reinterpret_cast<const uint4*>(lo);
  }
}

// The same operand as pack_cols_kernel (operand row = source column f, K index = source row p) stored as MN-major tiles (ptx::make_mnmajor_sw128_desc): tile [feature block of 128][64-point K block] = [feature group of 64]
// [point row][128 B = 64 features]; a source row segment is copied as it lies, no transposition.  grid (K blocks over
// points, row blocks over features); 256 threads: 8 lanes cover one 128-byte line, 4 passes of 32 point rows, 2 groups.
__global__ void __launch_bounds__(256) pack_cols_mn_kernel(const float* __restrict__ src, int ld, int P, int F,
                                                           uint8_t* __restrict__ out, int kbt) {
  const int kb = blockIdx.x, rb = blockIdx.y;
  uint8_t* tile = out + ((size_t)rb * kbt + kb) * kPtileBytes;
  const int c8 = threadIdx.x & 7;
  const bool vec = (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0;
#pragma unroll
  for (int g = 0; g < 2; ++g) {
    const int col = rb * 128 + g * 64 + c8 * 8;
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
      const int r = pass * 32 + (threadIdx.x >> 3);            // point row of the K block
      const int gp = kb * 64 + r;
      float v[8];
      if (vec && gp < P && col + 8 <= F) {
        const float4 x0 = *reinterpret_cast<const float4*>(src + (size_t)gp * ld + col);
        const float4 x1 = *reinterpret_cast<const float4*>(src + (size_t)gp * ld + col + 4);
        v[0] = x0.x; v[1] = x0.y; v[2] = x0.z; v[3] = x0.w; v[4] = x1.x; v[5] = x1.y; v[6] = x1.z; v[7] = x1.w;
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = (gp < P && col + i < F) ? src[(size_t)gp * ld + col + i] : 0.f;
      }
      __align__(16) uint16_t hi[8], lo[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) split_bf16(v[i], &hi[i], &lo[i]);
      const uint32_t off = (uint32_t)g * 8192u + (uint32_t)r * 128u + (uint32_t)((c8 ^ (r & 7)) << 4);
      *reinterpret_cast<uint4*>(tile + off) = *reinterpret_cast<const uint4*>(hi);
      *reinterpret_cast<uint4*>(tile + kPtileHalf + off) = *reinterpret_cast<const uint4*>(lo);
    }
  }
}

}  // namespace

size_t pack_bytes(int rows, int k) { return (size_t)((rows + 127) / 128) * ((k + 63) / 64) * kPtileBytes; }

int launch_tc_gemm(TcGemmParams P, int num_sms, cudaStream_t st, int64_t* launches) {
  if (P.M <= 0 || P.N <= 0) return 0;
  NM_CHECK(P.kbt > 0, "empty K range");
  const int n_rb_a = (P.M + 127) / 128;
  P.n_rb_b = (P.N + 127) / 128;
  const int NB = P.n_rb_b >= 2 ? 2 : 1;
  const int col_groups = (P.n_rb_b + NB - 1) / NB;
  int splits = num_sms / (n_rb_a * col_groups);                // one wave: every extra split costs a full atomic epilogue
  const int max_splits = (P.kbt + 7) / 8;                      // at least 8 K blocks (512 points) per split
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  P.kb_per_split = (P.kbt + splits - 1) / splits;
  splits = (P.kbt + P.kb_per_split - 1) / P.kb_per_split;
  static thread_local unsigned configured = 0;
  int dev = 0;
  NM_CUDA(cudaGetDevice(&dev));
  const size_t smem = kGemmSmem;
  if (!(configured & (1u << (dev & 31)))) {
    NM_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    NM_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured |= 1u << (dev & 31);
  }
  const dim3 grid(n_rb_a, col_groups, splits);
  if (NB == 2) tc_gemm_kernel<2><<<grid, kGemmThreads, smem, st>>>(P);
  else tc_gemm_kernel<1><<<grid, kGemmThreads, smem, st>>>(P);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

// A packed MN-major and B K-major, like the weight gradient's operands
int debug_tc_gemm(const float* A, const float* B, int M, int N, int K, int n_passes, float* D, uint8_t* scratch,
                  size_t scratch_bytes, int num_sms, int* d_err, cudaStream_t st, int64_t* launches) {
  NM_CHECK(scratch_bytes >= pack_bytes(M, K) + pack_bytes(N, K), "scratch too small: need %zu bytes",
           pack_bytes(M, K) + pack_bytes(N, K));
  TcGemmParams T{};
  T.a = scratch; T.b = scratch + pack_bytes(M, K); T.kbt = (K + 63) / 64;
  T.n_passes = n_passes; T.D = D; T.ldd = N; T.M = M; T.N = N; T.err = d_err;
  pack_cols_mn_kernel<<<dim3(T.kbt, (M + 127) / 128), 256, 0, st>>>(A, M, K, M, scratch, T.kbt);
  NM_CUDA(cudaGetLastError());
  pack_cols_kernel<<<dim3(T.kbt, (N + 127) / 128), 256, 0, st>>>(B, N, K, N, scratch + pack_bytes(M, K), T.kbt);
  NM_CUDA(cudaGetLastError());
  if (launches) *launches += 2;
  int repeat = 1;
  if (const char* e = getenv("NM_GEMM_REPEAT")) repeat = atoi(e) > 0 ? atoi(e) : 1;     // timing aid (tools/gemm_bench.py)
  for (int i = 0; i < repeat; ++i)
    if (int e = launch_tc_gemm(T, num_sms, st, launches)) return e;
  return 0;
}

}  // namespace nm
