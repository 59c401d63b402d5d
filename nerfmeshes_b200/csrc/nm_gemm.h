// The wgmma split-bf16 weight-gradient GEMM of the training backward (nm_gemm_tc.cu, called from nm_train.cu) and the
// layout of its pre-packed operands.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nm {

constexpr uint32_t kPtileBytes = 32768;   // 128 operand rows x 64 K: [hi 16 KB | lo 16 KB] bf16, 128B swizzle
constexpr uint32_t kPtileHalf = 16384;

// D (M,N) += A (M,K) B (N,K)^T with K = points, split over CTAs and reduced with fp32 atomics.  Packs are ptiles ordered
// [row block][K block] with `kbt` K blocks per row block: A (dZ^T) as MN-major ptiles, B (activations / encodings) as
// K-major ones.
struct TcGemmParams {
  const uint8_t* a;
  const uint8_t* b;
  int kbt;                 // K blocks of both packs (the K extent of the product)
  int n_passes;            // 3: hi*hi + lo*hi + hi*lo;  1: hi*hi
  float* D;                // (M,N) fp32 row-major
  int ldd, M, N;
  float* a_rowsum;         // optional: a_rowsum[m] += sum_k A[m][k], taken from the staged A tiles by the consumers —
                           //   with A = dZ^T this is the layer's bias gradient
  int* err;                // watchdog code (mapped host memory) or nullptr
  int n_rb_b, kb_per_split;   // filled by launch_tc_gemm
};

size_t pack_bytes(int rows, int k);
int launch_tc_gemm(TcGemmParams P, int num_sms, cudaStream_t st, int64_t* launches);
// nm_debug_gemm: D (M,N) += A^T B for fp32 row-major device arrays A (K,M), B (K,N), packed into `scratch`
// (pack_bytes(M, K) + pack_bytes(N, K) bytes, 1 KB aligned)
int debug_tc_gemm(const float* A, const float* B, int M, int N, int K, int n_passes, float* D, uint8_t* scratch,
                  size_t scratch_bytes, int num_sms, int* d_err, cudaStream_t st, int64_t* launches);

}  // namespace nm
