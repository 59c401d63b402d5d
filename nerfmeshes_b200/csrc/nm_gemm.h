// GEMM building blocks of the training backward (nm_train.cu): the fp32 CUDA-core SGEMMs (yard-stick, NM_PREC_FP32) and
// the wgmma split-bf16 GEMM on pre-packed operands (nm_gemm_tc.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace nm {

// fused epilogue of a data-path GEMM: v = acc (+C) (+bias[n]) (+r1_vec[m]*r1_w[n]); relu; relu-mask of another tensor
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

constexpr uint32_t kPtileBytes = 32768;   // 128 rows x 64 K: [hi 16 KB | lo 16 KB] bf16 or fp16, K-major, 128B swizzle
constexpr uint32_t kPtileHalf = 16384;

struct TcSeg {             // one K segment: packs ordered [row block][K block], *_kbt = K blocks per row block
  const uint8_t* a;
  int a_kbt;
  const uint8_t* b;
  int b_kbt;
  int nkb;                 // K blocks of this segment
  int mn = 0;              // bit 0 / bit 1: the A / B pack is an MN-major tile (pack_cols with mn=1) instead of a K-major one
};
struct TcGemmParams {
  TcSeg seg[2];
  int nseg;
  int n_passes;            // 3: hi*hi + lo*hi + hi*lo;  1: hi*hi
  int fp16;                // operand packs are fp16 halves (else bf16); both operands must use the same format
  float* D;                // (M,N) fp32 row-major
  int ldd, M, N;
  int atomic;              // D += via atomicAdd, K split over CTAs (weight gradients); the epilogue fields are ignored
  GemmEpi epi;
  float* colsum;           // optional: colsum[n] += sum_m D[m][n] (bias gradient of the layer whose dZ this GEMM produces)
  float* a_rowsum;         // optional (split-K, K-major bf16 A): a_rowsum[m] += sum_k A[m][k], taken from the staged A tiles by the
                           //   otherwise idle epilogue warps — with A = dZ^T this is the layer's bias gradient
  uint8_t* pack_out;       // optional: the epilogue also writes D as the row pack ([row block][K block = column / 64]) the
  int pack_kbt;            //   next GEMM of the chain consumes as its A operand (saves a pack_rows pass over D)
  int pack_fp16;
  uint16_t* bits_out;      // optional: relu mask of the output, one bit per element: halfword [m * bits_ld + n / 16] bit n % 16
  const uint16_t* bits_in; // optional: zero the output where the bit is clear (relu' of the tensor the bits were taken from)
  int bits_ld;             //   halfwords per row (= N / 16)
  uint8_t* packT_out;      // optional: ... and as the bf16 pack with K along the rows (points): the A^T / B^T operand of the
  int packT_kbt;           //   weight-gradient GEMMs ([column block of 128][K block = row / 64]); needs packT_kbt = 2 * row blocks
  int skip_d;              // do not write the fp32 D at all (its only consumers read the packs)
  int* err;                // watchdog code (mapped host memory) or nullptr
  int n_rb_a, n_rb_b, col_groups, kb_per_split;   // filled by launch_tc_gemm
  int dbg;                 // NM_GEMM_DBG experiments: 1 skip MMAs, 2 skip operand loads, 4 skip epilogue stores
};

size_t pack_bytes(int rows, int k);
int launch_pack_rows(const float* src, int ld, int R, int C, uint8_t* out, int fp16, cudaStream_t st, int64_t* launches);
int launch_pack_cols(const float* src, int ld, int P, int F, uint8_t* out, int kbt, int fp16, cudaStream_t st, int64_t* launches, int mn = 0);
int launch_tc_gemm(TcGemmParams P, int num_sms, cudaStream_t st, int64_t* launches);

}  // namespace nm
