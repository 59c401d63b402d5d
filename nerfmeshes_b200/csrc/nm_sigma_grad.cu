// Input tail of the density gradient g = d sigma / d p (nm_sigma_grad; orchestration in nm_train.cu, DESIGN 4.8).
//
// The data-gradient chain of the training backward (nm_mlp_tc.cu mode 2, seeded with d raw sigma = 1) leaves dZ_l of every
// layer as an MN-major bf16 hi/lo pack in (feature x point).  What it never computes is the last step back to the input:
//     dPE = sum_l dZ_l W_l[:, k_act, k_act + k_pe)        over the layers that read the xyz encoding (layer1, the skips)
//     g   = dPE J_PE(p)                                    (positional_encoding_vjp, nm_frontend.cuh)
// sigma_grad_tail_kernel does both: a wgmma GEMM with M = points whose A operand is the dZ packs themselves — MN-major in
// (feature x point) is K-major once the points are the M rows, so a pack's 64-feature group of a 64-point block is one
// SWIZZLE_128B K-major 64 x 64 tile — and whose B operand is the layers' encoding columns of W (64 encoding columns x 64
// features per K-block, bf16 hi/lo, packed once per call by sigma_grad_pack_w_kernel).  Every K-block of every xyz layer
// accumulates into the same m64n64 registers (hi*hi, then lo*hi and hi*lo in exact mode), and the epilogue contracts a
// point's 64 dPE columns with the encoding Jacobian in fp32.
//
// No atomics, and a point's arithmetic does not depend on its tile or CTA: the K-blocks are summed in one fixed order.
// pe_vjp_kernel is the same epilogue on an fp32 dPE (the NM_PREC_FP32 path: SIMT chain + sgemm).
#include <cuda_bf16.h>

#include "nm_common.h"
#include "nm_frontend.cuh"
#include "nm_gemm.h"
#include "nm_ptx.cuh"

namespace nm {
namespace {

constexpr int kSgThreads = 128;                         // one warpgroup, one 64-point tile at a time
constexpr uint32_t kSgTile = 8192;                      // 64 rows x 128 B: one bf16 half of a 64 x 64 K-major tile
constexpr uint32_t kSgStage = 4 * kSgTile;              // A hi | A lo | B hi | B lo
constexpr uint32_t kSgStgOff = 2 * kSgStage;            // epilogue staging: 64 points x 65 floats
constexpr uint32_t kSgSmem = kSgStgOff + 64u * 65u * 4u;

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// B tiles: K-block kb = rows j (encoding column, zero for j >= k_pe) x 64 features, K-major SWIZZLE_128B, [hi | lo] bf16
__global__ void __launch_bounds__(256) sigma_grad_pack_w_kernel(const __grid_constant__ SigmaGradWeights W) {
  const int kb = blockIdx.x;
  uint8_t* tile = W.out + (size_t)kb * 2 * kSgTile;
  for (int e = threadIdx.x; e < 64 * 64; e += blockDim.x) {
    const int j = e >> 6, kk = e & 63;
    const float w = j < W.k_pe ? W.wt[kb][(size_t)j * W.ld[kb] + kk] : 0.f;
    const __nv_bfloat16 h = __float2bfloat16_rn(w);
    const __nv_bfloat16 l = __float2bfloat16_rn(w - __bfloat162float(h));
    const uint32_t off = (uint32_t)j * 128u + ((((uint32_t)kk >> 3) ^ ((uint32_t)j & 7u)) << 4) + ((uint32_t)kk & 7u) * 2u;
    *reinterpret_cast<uint16_t*>(tile + off) = __bfloat16_as_ushort(h);
    *reinterpret_cast<uint16_t*>(tile + kSgTile + off) = __bfloat16_as_ushort(l);
  }
}

__global__ void __launch_bounds__(kSgThreads) sigma_grad_tail_kernel(const __grid_constant__ SigmaGradTail P) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sbase = ptx::smem_u32(smem);
  const int t = threadIdx.x;
  if (t == 0 && (sbase & 1023u)) { if (P.err) atomicExch(P.err, 95); __trap(); }
  float* stg = reinterpret_cast<float*>(smem + kSgStgOff);
  const bool exact = P.n_passes == 3;
  const long long n_tiles = (P.M + 63) / 64;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    // one K-block into stage s: the A tile of this point block (its hi and lo halves) and the B tile, 16-byte cp.async
    auto issue = [&](int kb, int s) {
      const uint8_t* a = P.a[kb] + (size_t)tile * kPtileBytes;
      const uint8_t* b = P.b + (size_t)kb * 2 * kSgTile;
      const uint32_t dst = sbase + (uint32_t)s * kSgStage;
      for (int i = t; i < 4 * 512; i += kSgThreads) {
        const int part = i >> 9, c = i & 511;               // part: A hi, A lo, B hi, B lo
        if (!exact && (part & 1)) continue;
        const uint8_t* src = part < 2 ? a + (part ? kPtileHalf : 0u) + c * 16 : b + (part - 2) * kSgTile + c * 16;
        cp_async16(dst + (uint32_t)part * kSgTile + (uint32_t)c * 16u, src);
      }
      cp_async_commit();
    };
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    issue(0, 0);
    for (int kb = 0; kb < P.n_kb; ++kb) {
      const int s = kb & 1;
      if (kb + 1 < P.n_kb) { issue(kb + 1, s ^ 1); cp_async_wait<1>(); }
      else cp_async_wait<0>();
      ptx::fence_proxy_async_smem();                       // the wgmmas read what cp.async (generic proxy) wrote
      __syncthreads();
      const uint32_t st = sbase + (uint32_t)s * kSgStage;
      const uint64_t a_hi = ptx::make_kmajor_sw128_desc(st), a_lo = ptx::make_kmajor_sw128_desc(st + kSgTile);
      const uint64_t b_hi = ptx::make_kmajor_sw128_desc(st + 2 * kSgTile), b_lo = ptx::make_kmajor_sw128_desc(st + 3 * kSgTile);
      ptx::wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) ptx::wgmma<64, 0, 0, 1>(acc, a_hi + 2 * k, b_hi + 2 * k, 1u);
      if (exact) {
#pragma unroll
        for (int k = 0; k < 4; ++k) ptx::wgmma<64, 0, 0, 1>(acc, a_lo + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
        for (int k = 0; k < 4; ++k) ptx::wgmma<64, 0, 0, 1>(acc, a_hi + 2 * k, b_lo + 2 * k, 1u);
      }
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
      ptx::fence_regs<32>(acc);
      __syncthreads();                                     // stage s is free for the K-block after next
    }
    // epilogue: fragments -> staging (register i of thread t: row 16 (t/32) + (t%32)/4 + 8 ((i/2)%2), column
    // 8 (i/4) + 2 (t%4) + i%2), then one thread per point contracts its row with the encoding Jacobian
    const int w = t >> 5, lane = t & 31;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int row = 16 * w + (lane >> 2) + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
      stg[row * 65 + col] = acc[i];
    }
    __syncthreads();
    const long long m = tile * 64 + t;
    if (t < 64 && m < P.M) {
      const float x[3] = {__ldg(P.pts + 3 * m), __ldg(P.pts + 3 * m + 1), __ldg(P.pts + 3 * m + 2)};
      float g[3];
      const float* row = stg + t * 65;
      positional_encoding_vjp(x, P.pe.L, P.pe.inc, P.pe.freq, [&](int j) { return row[j]; }, g);
      P.grad[3 * m] = g[0]; P.grad[3 * m + 1] = g[1]; P.grad[3 * m + 2] = g[2];
    }
    __syncthreads();
  }
}

// NM_PREC_FP32: the same contraction on an fp32 dPE (M, ld)
__global__ void pe_vjp_kernel(const float* __restrict__ pts, long long M, const float* __restrict__ dpe, int ld,
                              const __grid_constant__ PeDesc pe, float* __restrict__ grad) {
  const long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  const float x[3] = {pts[3 * m], pts[3 * m + 1], pts[3 * m + 2]};
  const float* row = dpe + (size_t)m * ld;
  float g[3];
  positional_encoding_vjp(x, pe.L, pe.inc, pe.freq, [&](int j) { return row[j]; }, g);
  grad[3 * m] = g[0]; grad[3 * m + 1] = g[1]; grad[3 * m + 2] = g[2];
}

}  // namespace

int launch_sigma_grad_tail(const SigmaGradWeights& W, const SigmaGradTail& T, int num_sms, cudaStream_t st, int64_t* launches) {
  if (T.M <= 0) return 0;
  NM_CHECK(T.n_kb > 0 && T.n_kb <= kSgMaxKb, "density gradient: %d K-blocks of xyz-reading layers (1..%d supported)", T.n_kb, kSgMaxKb);
  NM_CHECK(W.k_pe > 0 && W.k_pe <= 64, "density gradient: xyz encoding width %d outside [1, 64]", W.k_pe);
  sigma_grad_pack_w_kernel<<<T.n_kb, 256, 0, st>>>(W);
  NM_CUDA(cudaGetLastError());
  static thread_local unsigned configured = 0;
  int dev = 0;
  NM_CUDA(cudaGetDevice(&dev));
  if (!(configured & (1u << (dev & 31)))) {
    NM_CUDA(cudaFuncSetAttribute(sigma_grad_tail_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSgSmem));
    configured |= 1u << (dev & 31);
  }
  const long long tiles = (T.M + 63) / 64;
  const long long grid = tiles < 2ll * num_sms ? tiles : 2ll * num_sms;      // two 81 KB CTAs per SM
  sigma_grad_tail_kernel<<<(unsigned)grid, kSgThreads, kSgSmem, st>>>(T);
  NM_CUDA(cudaGetLastError());
  if (launches) *launches += 2;
  return 0;
}

int launch_pe_vjp(const float* pts, long long M, const float* dpe, int ld, const PeDesc& pe, float* grad, cudaStream_t st,
                  int64_t* launches) {
  if (M <= 0) return 0;
  pe_vjp_kernel<<<(unsigned)((M + 127) / 128), 128, 0, st>>>(pts, M, dpe, ld, pe, grad);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

}  // namespace nm
