// Sustained tensor-core rate of the fused MLP's exact-mode MMA pattern at three widths (tools/wgmma_rate.py builds and
// runs this).  One CTA per SM, two warpgroups, every operand resident in shared memory; each warpgroup repeats one K = 64
// slab of a 256-column layer: every K = 16 step issues a_hi*b_hi, a_lo*b_hi, a_hi*b_lo across all 256 output columns as
//   variant 0: 4 x m64n64k16 per pass from 64x64 SW128 K-major blocks (a commit group per 64-column block, 12 wgmmas)
//   variant 1: 2 x m64n128k16 per pass from 128x64 SW128 K-major blocks (a commit group per block, 12 wgmmas)
//   variant 2: 1 x m64n256k16 per pass from 256x16 SW32 K-major steps (a commit group per K step, 3 wgmmas)
// with commit -> wait_group 1 between groups, as the MLP kernel's stage loop does.  Variant 3 is variant 1 issued by ONE
// warpgroup per SM (128 threads): whether a single warpgroup keeps the SM's four tensor cores as busy as two do, which a
// ping-pong of the two consumer warpgroups (one issuing MMAs while the other runs its epilogue) relies on.
//
//     wgmma_rate <iterations>     prints "variant ms" lines for one launch of each variant
#include <cstdio>
#include <cstdlib>

#include "nm_ptx.cuh"

using namespace nm;

constexpr uint32_t kB = 65536;      // B operands: 64 KB (hi and lo of K = 64 x N = 256) in every variant
constexpr uint32_t kA = 16384;      // A operand of one warpgroup: 64 rows x K = 64, hi | lo (SW128)

template <int V>
__global__ void __launch_bounds__(256, 1) rate_kernel(long long iters, float* sink) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t s0 = ptx::smem_u32(smem);
  // finite fp16 values in [0.5, 1) with varied mantissas (all-zero operands would understate the power draw)
  for (uint32_t i = threadIdx.x; i < (kB + 2 * kA) / 2; i += blockDim.x) {
    uint32_t h = i * 2654435761u;
    h ^= h >> 15;
    reinterpret_cast<uint16_t*>(smem)[i] = (uint16_t)(0x3800u | (h & 0x3ffu));
  }
  ptx::fence_proxy_async_smem();
  __syncthreads();
  const int wg = threadIdx.x >> 7;
  const uint32_t a = s0 + kB + (uint32_t)wg * kA;
  const uint64_t a_hi = ptx::make_kmajor_sw128_desc(a), a_lo = ptx::make_kmajor_sw128_desc(a + 8192u);
  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  ptx::wgmma_fence();
  for (long long it = 0; it < iters; ++it) {
    if (V == 0) {
#pragma unroll
      for (int nc = 0; nc < 4; ++nc) {
        const uint64_t b_hi = ptx::make_kmajor_sw128_desc(s0 + nc * 16384u), b_lo = ptx::make_kmajor_sw128_desc(s0 + nc * 16384u + 8192u);
#pragma unroll
        for (int k = 0; k < 4; ++k) ptx::wgmma<64, 0, 0, 0>(acc + 32 * nc, a_hi + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
        for (int k = 0; k < 4; ++k) ptx::wgmma<64, 0, 0, 0>(acc + 32 * nc, a_lo + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
        for (int k = 0; k < 4; ++k) ptx::wgmma<64, 0, 0, 0>(acc + 32 * nc, a_hi + 2 * k, b_lo + 2 * k, 1u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();
      }
    } else if (V == 1 || V == 3) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint64_t b_hi = ptx::make_kmajor_sw128_desc(s0 + h * 32768u), b_lo = ptx::make_kmajor_sw128_desc(s0 + h * 32768u + 16384u);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          ptx::wgmma<128, 0, 0, 0>(acc + 64 * h, a_hi + 2 * k, b_hi + 2 * k, 1u);
          ptx::wgmma<128, 0, 0, 0>(acc + 64 * h, a_lo + 2 * k, b_hi + 2 * k, 1u);
          ptx::wgmma<128, 0, 0, 0>(acc + 64 * h, a_hi + 2 * k, b_lo + 2 * k, 1u);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();
      }
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t b_hi = ptx::make_kmajor_sw32_desc(s0 + k * 16384u), b_lo = ptx::make_kmajor_sw32_desc(s0 + k * 16384u + 8192u);
        ptx::wgmma<256, 0, 0, 0>(acc, a_hi + 2 * k, b_hi, 1u);
        ptx::wgmma<256, 0, 0, 0>(acc, a_lo + 2 * k, b_hi, 1u);
        ptx::wgmma<256, 0, 0, 0>(acc, a_hi + 2 * k, b_lo, 1u);
        ptx::wgmma_commit();
        ptx::wgmma_wait<1>();
      }
    }
  }
  ptx::wgmma_wait<0>();
  ptx::fence_regs<128>(acc);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 128; ++i) s += acc[i];
  if (s == 12345.f) sink[threadIdx.x] = s;      // keeps the MMAs live; never true for these operands in practice
}

#define CK(x)                                                                                    \
  do {                                                                                           \
    cudaError_t e_ = (x);                                                                        \
    if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); return 1; } \
  } while (0)

template <int V>
static int run(int sms, long long iters, float* sink) {
  const int smem = (int)(kB + 2 * kA), threads = V == 3 ? 128 : 256;
  CK(cudaFuncSetAttribute(rate_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  rate_kernel<V><<<sms, threads, smem>>>(iters / 16 + 1, sink);      // warm-up
  CK(cudaGetLastError());
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  CK(cudaEventRecord(e0));
  rate_kernel<V><<<sms, threads, smem>>>(iters, sink);
  CK(cudaEventRecord(e1));
  CK(cudaEventSynchronize(e1));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  printf("%d %.4f\n", V, ms);
  return 0;
}

int main(int argc, char** argv) {
  const long long iters = argc > 1 ? atoll(argv[1]) : 100000;
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, 0));
  float* sink;
  CK(cudaMalloc(&sink, 256 * sizeof(float)));
  printf("sms %d\nname %s\n", prop.multiProcessorCount, prop.name);
  for (int rep = 0; rep < 2; ++rep)
    if (run<0>(prop.multiProcessorCount, iters, sink) || run<1>(prop.multiProcessorCount, iters, sink) ||
        run<2>(prop.multiProcessorCount, iters, sink) || run<3>(prop.multiProcessorCount, iters, sink))
      return 1;
  CK(cudaFree(sink));
  return 0;
}
