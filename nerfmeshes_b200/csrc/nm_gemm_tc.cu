// wgmma GEMM for the training backward (nm_train.cu): D (M,N) = A (M,K) * B (N,K)^T with both operands given as
// pre-packed hi/lo "ptiles" and fp32 accumulation in registers.  fp32 accuracy class comes from the same operand split the
// forward kernel uses (x = hi + lo, three MMAs per product: hi*hi + lo*hi + hi*lo).  Halves are bf16 for the gradient
// GEMMs (gradients span fp32's exponent range; 16 significand bits per operand, ~2^-16 per product) and fp16 for the
// forward recompute (22 bits, the forward kernel's class: its relu masks must agree with the forward's).
//
// ptile = one (128 operand rows) x (64 K) block: [hi | lo], each 16 KB, 128-byte swizzled, K-major or (per segment and
// operand, TcSeg.mn) MN-major — the shared-memory image wgmma reads through a descriptor, so a ptile moves global ->
// shared with ONE 32 KB cp.async.bulk.  A pack is ptiles ordered [row block][K block].  Packs are produced by
// pack_rows_kernel (K along the source's columns), pack_cols_kernel (K along the source's rows: the A^T / B^T operands of
// the weight gradient) and, for everything inside the layer chain, by this kernel's own epilogue.
//
// Kernel: 12 warps — two consumer warpgroups (rows 0-63 / 64-127 of the 128-row tile; m64n128k16 wgmmas into 64 (NB=1)
// or 128 (NB=2) accumulator registers per thread, then the epilogue from those registers), and a producer warpgroup
// whose first warp issues the bulk copies into a ring of K-block stages (2 x 96 KB for 256-wide tiles,
// 3 x 64 KB for 128-wide).  Data-path GEMMs are persistent (grid = min(tiles, SMs)): the producer fills the next tile's
// stages while the consumers run the epilogue of the current one.  The weight gradient (K = points) splits K over one
// wave of CTAs and reduces with vector atomics.  Barriers: full[s] (tx bytes), empty[s] (one arrival per consumer
// warpgroup once its wgmmas on the stage are complete).  In a split-K launch with a_rowsum the consumers also sum the
// rows of the staged A tiles (the bias gradient when A = dZ^T).  The fused epilogue of the layer-wise walk (bias/relu,
// rank-1 term, 1-bit masks in and out, row pack and point-major pack of the output, column sums) is described in
// DESIGN.md section 4.4.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstdlib>

#include "nm_common.h"
#include "nm_gemm.h"
#include "nm_ptx.cuh"

namespace nm {
namespace {

constexpr int kGemmThreads = 384;   // warps 0-3, 4-7 consumers; 8-11 producer warpgroup (warp 8 issues)
constexpr int kProdWarp = 8;

// x = hi + lo in two 16-bit floats: bf16 (8+8 significand bits, fp32's exponent range: gradients) or fp16 (11+11
// bits, |x| < 65504: activations, encodings and weights of the forward recompute, like the forward kernel)
__device__ __forceinline__ void split16(float x, int fp16, uint16_t* hi, uint16_t* lo) {
  if (fp16) {
    const __half h = __float2half_rn(x);
    const __half l = __float2half_rn(x - __half2float(h));
    *hi = __half_as_ushort(h); *lo = __half_as_ushort(l);
  } else {
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    const __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
    *hi = __bfloat16_as_ushort(h); *lo = __bfloat16_as_ushort(l);
  }
}

constexpr uint32_t kStgOff = 6u * kPtileBytes;                       // epilogue staging: 8 warps x 16 rows x 17 floats
constexpr uint32_t kStgWarp = 16u * 17u * 4u;
constexpr uint32_t kBarOff = kStgOff + 8u * kStgWarp;                // barriers behind the 1024-aligned stages
constexpr uint32_t kGemmSmem = kBarOff + 128u;

// One K block of the tile: every pass of the four K=16 steps into the NB accumulators (K-major / MN-major operands).
template <int TA, int TB, int BF16, int NB>
__device__ __forceinline__ void mma_kblock(float (&acc)[2][64], uint32_t a, uint32_t stage, int nbv, int n_passes) {
  const uint64_t a_hi = TA ? ptx::make_mnmajor_sw128_desc(a) : ptx::make_kmajor_sw128_desc(a);
  const uint64_t a_lo = TA ? ptx::make_mnmajor_sw128_desc(a + kPtileHalf) : ptx::make_kmajor_sw128_desc(a + kPtileHalf);
  constexpr uint64_t a_step = TA ? 128u : 2u, b_step = TB ? 128u : 2u;   // per k16: 2048 B (MN-major) / 32 B (K-major)
#pragma unroll
  for (int j = 0; j < NB; ++j) {
    if (j >= nbv) break;
    const uint32_t bs = stage + kPtileBytes * (uint32_t)(1 + j);
    const uint64_t b_hi = TB ? ptx::make_mnmajor_sw128_desc(bs) : ptx::make_kmajor_sw128_desc(bs);
    const uint64_t b_lo = TB ? ptx::make_mnmajor_sw128_desc(bs + kPtileHalf) : ptx::make_kmajor_sw128_desc(bs + kPtileHalf);
#pragma unroll
    for (int k = 0; k < 4; ++k) ptx::wgmma_m64n128<TA, TB, BF16>(acc[j], a_hi + k * a_step, b_hi + k * b_step, 1u);
    if (n_passes == 3) {
#pragma unroll
      for (int k = 0; k < 4; ++k) ptx::wgmma_m64n128<TA, TB, BF16>(acc[j], a_lo + k * a_step, b_hi + k * b_step, 1u);
#pragma unroll
      for (int k = 0; k < 4; ++k) ptx::wgmma_m64n128<TA, TB, BF16>(acc[j], a_hi + k * a_step, b_lo + k * b_step, 1u);
    }
  }
}

// Epilogue of one 16-row x 16-column block of a warp, staged in stg (pitch 17): lane = (row sub = lane / 4, 4 columns
// q4 = 4 * (lane % 4)), rows sub and sub + 8.  row0: the block's first global row; rt0: its row within the 128-row block.
__device__ __noinline__ void epi_block(const TcGemmParams& P, float* stg, int lane, int rb, int row0, int rt0, int n0) {
  const int sub = lane >> 2, q4 = (lane & 3) * 4;
  const GemmEpi& E = P.epi;
  const int n = n0 + q4;                 // first of this lane's 4 global columns
  if (n >= P.N || (P.dbg & 4)) return;
  if (P.atomic) {
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
    return;
  }
  // data-path outputs: N is a multiple of 64, rows are 16-byte aligned
  float4 bias = make_float4(0.f, 0.f, 0.f, 0.f), w1 = bias;
  if (E.bias) bias = *reinterpret_cast<const float4*>(E.bias + n);
  if (E.r1_vec) w1 = *reinterpret_cast<const float4*>(E.r1_w + n);
  float4 v[2], cs = make_float4(0.f, 0.f, 0.f, 0.f);
  uint32_t mw[2];
  float r1[2];
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const int rr = it * 8 + sub, m = min(row0 + rr, P.M - 1);
    const float* sp = &stg[rr * 17 + q4];
    v[it] = make_float4(sp[0], sp[1], sp[2], sp[3]);
    mw[it] = P.bits_in ? ((uint32_t)P.bits_in[(size_t)m * P.bits_ld + (n >> 4)] >> (n & 15)) : 0xfu;   // this lane's 4 mask bits
    r1[it] = E.r1_vec ? E.r1_vec[(size_t)m * E.r1_stride] : 0.f;
    if (E.accumulate) {
      const float4 c = *reinterpret_cast<const float4*>(P.D + (size_t)m * P.ldd + n);
      v[it].x += c.x; v[it].y += c.y; v[it].z += c.z; v[it].w += c.w;
    }
  }
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    const int rr = it * 8 + sub, m = row0 + rr;
    float4 o = v[it];
    o.x = fmaf(r1[it], w1.x, o.x + bias.x); o.y = fmaf(r1[it], w1.y, o.y + bias.y);
    o.z = fmaf(r1[it], w1.z, o.z + bias.z); o.w = fmaf(r1[it], w1.w, o.w + bias.w);
    if (E.relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
    if (!(mw[it] & 1u)) o.x = 0.f;
    if (!(mw[it] & 2u)) o.y = 0.f;
    if (!(mw[it] & 4u)) o.z = 0.f;
    if (!(mw[it] & 8u)) o.w = 0.f;
    if (P.bits_out) {      // relu mask of this output row segment: 4 lanes x 4 bits -> one halfword
      uint32_t bits = ((o.x > 0.f ? 1u : 0u) | (o.y > 0.f ? 2u : 0u) | (o.z > 0.f ? 4u : 0u) | (o.w > 0.f ? 8u : 0u)) << q4;
      bits |= __shfl_xor_sync(0xffffffffu, bits, 1);
      bits |= __shfl_xor_sync(0xffffffffu, bits, 2);
      if (!(lane & 3) && m < P.M) P.bits_out[(size_t)m * P.bits_ld + (n >> 4)] = (uint16_t)bits;
    }
    if (m < P.M) {
      if (!P.skip_d) *reinterpret_cast<float4*>(P.D + (size_t)m * P.ldd + n) = o;
      cs.x += o.x; cs.y += o.y; cs.z += o.z; cs.w += o.w;
    } else {
      o = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (P.packT_out) { float* sp = &stg[rr * 17 + q4]; sp[0] = o.x; sp[1] = o.y; sp[2] = o.z; sp[3] = o.w; }
    if (P.pack_out) {
      // even lanes gather their neighbour's 4 columns: 8 consecutive columns = one 16-byte chunk of the tile row
      const float e0 = __shfl_down_sync(0xffffffffu, o.x, 1), e1 = __shfl_down_sync(0xffffffffu, o.y, 1);
      const float e2 = __shfl_down_sync(0xffffffffu, o.z, 1), e3 = __shfl_down_sync(0xffffffffu, o.w, 1);
      if (!(lane & 1)) {
        const float vals[8] = {o.x, o.y, o.z, o.w, e0, e1, e2, e3};
        __align__(16) uint16_t hi[8], lo[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) split16(vals[e], P.pack_fp16, &hi[e], &lo[e]);
        const int r_t = rt0 + rr, c8 = (n & 63) >> 3;
        uint8_t* tile = P.pack_out + ((size_t)rb * P.pack_kbt + (n >> 6)) * kPtileBytes;
        const uint32_t off = (uint32_t)r_t * 128u + (uint32_t)((c8 ^ (r_t & 7)) << 4);
        *reinterpret_cast<uint4*>(tile + off) = *reinterpret_cast<const uint4*>(hi);
        *reinterpret_cast<uint4*>(tile + kPtileHalf + off) = *reinterpret_cast<const uint4*>(lo);
      }
    }
  }
  if (P.packT_out) {   // the finished 16x16 block, transposed: lane = (column f, 8-row chunk)
    __syncwarp();
    const int f = lane & 15, c = lane >> 4;
    const int nf = n0 + f;
    const int row = nf & 127;
    // points rt0 .. rt0+15 of row block rb: K block rb * 2 + rt0 / 64, 8-point chunk (rt0 % 64) / 8 + c
    uint8_t* tile = P.packT_out + ((size_t)(nf >> 7) * P.packT_kbt + (rb * 2 + (rt0 >> 6))) * kPtileBytes;
    __align__(16) uint16_t hi[8], lo[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) split16(stg[(c * 8 + e) * 17 + f], 0, &hi[e], &lo[e]);
    const int c8 = ((rt0 & 63) >> 3) + c;
    const uint32_t off = (uint32_t)row * 128u + (uint32_t)((c8 ^ (row & 7)) << 4);
    *reinterpret_cast<uint4*>(tile + off) = *reinterpret_cast<const uint4*>(hi);
    *reinterpret_cast<uint4*>(tile + kPtileHalf + off) = *reinterpret_cast<const uint4*>(lo);
  }
  if (P.colsum) {      // lanes with equal lane%4 hold the same 4 columns
#pragma unroll
    for (int d = 4; d <= 16; d <<= 1) {
      cs.x += __shfl_xor_sync(0xffffffffu, cs.x, d); cs.y += __shfl_xor_sync(0xffffffffu, cs.y, d);
      cs.z += __shfl_xor_sync(0xffffffffu, cs.z, d); cs.w += __shfl_xor_sync(0xffffffffu, cs.w, d);
    }
    if (lane < 4) {
      atomicAdd(P.colsum + n, cs.x); atomicAdd(P.colsum + n + 1, cs.y);
      atomicAdd(P.colsum + n + 2, cs.z); atomicAdd(P.colsum + n + 3, cs.w);
    }
  }
}

// Tiles of one CTA.  Data-path GEMMs are persistent: grid = min(tiles, SMs), tile t = blockIdx.x + i * gridDim.x walks
// (row block, column group) pairs.  Split-K (weight gradient) launches one tile per CTA: (row block, column group,
// K split) = blockIdx.
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

  const bool pers = P.atomic == 0;
  const int n_tiles = pers ? P.n_rb_a * P.col_groups : 1;
  const int t_first = pers ? (int)blockIdx.x : 0, t_step = pers ? (int)gridDim.x : 1;
  auto tile_rb = [&](int t) { return pers ? t / P.col_groups : (int)blockIdx.x; };
  auto tile_cb0 = [&](int t) { return (pers ? t % P.col_groups : (int)blockIdx.y) * NB; };
  // K blocks of a tile: segment 0 restricted to the split's range, then segment 1
  int k0 = 0, k1 = P.seg[0].nkb;
  if (P.kb_per_split > 0) { k0 = blockIdx.z * P.kb_per_split; k1 = min(P.seg[0].nkb, k0 + P.kb_per_split); }
  const int n0 = k1 - k0;
  const int nk = n0 + (P.nseg > 1 ? P.seg[1].nkb : 0);

  // split-K with a_rowsum: the CTAs of the first column group also sum the rows of every A tile they stage (bias gradient)
  const bool sum_rows = !pers && P.a_rowsum != nullptr && blockIdx.y == 0;
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
      int it = 0;
      for (int t = t_first; t < n_tiles; t += t_step) {
        const int rb = tile_rb(t), cb0 = tile_cb0(t);
        const int nbv = min(NB, P.n_rb_b - cb0);
        for (int kk = 0; kk < nk; ++kk, ++it) {
          const int s = it % NS;
          if (it >= NS) ptx::mbar_wait(empty(s), (uint32_t)((it / NS - 1) & 1), P.err, 91);
          const int sg = kk < n0 ? 0 : 1;
          const int kb = kk < n0 ? k0 + kk : kk - n0;
          const TcSeg& S = P.seg[sg];
          const uint32_t dst = sbase + (uint32_t)s * STAGE;
          ptx::mbar_expect_tx(full(s), kPtileBytes * (uint32_t)(1 + nbv));
          ptx::bulk_g2s(dst, S.a + ((size_t)rb * S.a_kbt + kb) * kPtileBytes, kPtileBytes, full(s));
          for (int j = 0; j < nbv; ++j)
            ptx::bulk_g2s(dst + kPtileBytes * (uint32_t)(1 + j), S.b + ((size_t)(cb0 + j) * S.b_kbt + kb) * kPtileBytes,
                          kPtileBytes, full(s));
        }
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
  int it = 0;
  for (int tt = t_first; tt < n_tiles; tt += t_step) {
    const int rb = tile_rb(tt), cb0 = tile_cb0(tt);
    const int nbv = min(NB, P.n_rb_b - cb0);
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[j][i] = 0.f;
    ptx::wgmma_fence();
    int prev = -1;
    for (int kk = 0; kk < nk; ++kk, ++it) {
      const int s = it % NS;
      ptx::mbar_wait(full(s), (uint32_t)((it / NS) & 1), P.err, 92);
      const uint32_t st = sbase + (uint32_t)s * STAGE;
      const int mn = P.seg[kk < n0 ? 0 : 1].mn;
      if (sum_rows) {
        // Row sums of the A tile (this warpgroup's 64 rows) while the tensor cores consume it; hi + lo halves.
        const uint8_t* at = smem + (size_t)s * STAGE;
        if (mn & 1) {
          // MN-major: [feature group of 64][K row (point) 0..63][128 B = 8 chunks of 8 features, chunk ^= row & 7]
          const int f = t & 63, kr0 = (t >> 6) * 32;
          for (int k = kr0; k < kr0 + 32; ++k) {
            const uint32_t off = (uint32_t)wg * 8192u + (uint32_t)k * 128u + ((((uint32_t)f >> 3) ^ ((uint32_t)k & 7u)) << 4) + (uint32_t)(f & 7) * 2u;
            const uint32_t h = *reinterpret_cast<const uint16_t*>(at + off), l = *reinterpret_cast<const uint16_t*>(at + kPtileHalf + off);
            rsum += __uint_as_float(h << 16) + __uint_as_float(l << 16);
          }
        } else {
          // K-major: two threads per row, 32 K elements each (the swizzle only permutes chunks within the row)
          const int row = wg * 64 + (t >> 1);
          const uint4* rp = reinterpret_cast<const uint4*>(at + (size_t)row * 128u + (size_t)(t & 1) * 64u);
          float acc_r = 0.f;
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const uint4 h = rp[c], l = rp[c + kPtileHalf / 16];
            const uint32_t w[8] = {h.x, h.y, h.z, h.w, l.x, l.y, l.z, l.w};
#pragma unroll
            for (int e = 0; e < 8; ++e) acc_r += __uint_as_float(w[e] << 16) + __uint_as_float(w[e] & 0xffff0000u);
          }
          rsum += acc_r;
        }
      }
      const uint32_t a = st + (uint32_t)wg * 8192u;    // rows 64.. : +64 rows (K-major) / the second MN group (MN-major)
      if (!(P.dbg & 1)) {
        const bool amn = mn & 1, bmn = mn & 2;
        if (P.fp16) {
          if (amn) { if (bmn) mma_kblock<1, 1, 0, NB>(acc, a, st, nbv, P.n_passes); else mma_kblock<1, 0, 0, NB>(acc, a, st, nbv, P.n_passes); }
          else     { if (bmn) mma_kblock<0, 1, 0, NB>(acc, a, st, nbv, P.n_passes); else mma_kblock<0, 0, 0, NB>(acc, a, st, nbv, P.n_passes); }
        } else {
          if (amn) { if (bmn) mma_kblock<1, 1, 1, NB>(acc, a, st, nbv, P.n_passes); else mma_kblock<1, 0, 1, NB>(acc, a, st, nbv, P.n_passes); }
          else     { if (bmn) mma_kblock<0, 1, 1, NB>(acc, a, st, nbv, P.n_passes); else mma_kblock<0, 0, 1, NB>(acc, a, st, nbv, P.n_passes); }
        }
      }
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
    const int rt0 = wg * 64 + wi * 16, row0 = rb * 128 + rt0;
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
        epi_block(P, stg, lane, rb, row0, rt0, (cb0 + j) * 128 + blk * 16);
        __syncwarp();
      }
    }
  }
  if (sum_rows) {
    if (P.seg[0].mn & 1) {
      const int row = (int)blockIdx.x * 128 + wg * 64 + (t & 63);
      if (row < P.M) atomicAdd(P.a_rowsum + row, rsum);
    } else {
      rsum += __shfl_xor_sync(0xffffffffu, rsum, 1);
      const int row = (int)blockIdx.x * 128 + wg * 64 + (t >> 1);
      if (!(t & 1) && row < P.M) atomicAdd(P.a_rowsum + row, rsum);
    }
  }
}

// ------------------------------------------------------------------------------------------------ packers
// K along the source's columns: operand row r = source row, K index c = source column (c < C valid, zero beyond).
// grid (K blocks, row blocks); 256 threads: 8 lanes cover one 128-byte tile row (8 chunks of 8 columns), a warp 4 rows,
// so every global access is a whole line; 4 passes of 32 rows.
__global__ void __launch_bounds__(256) pack_rows_kernel(const float* __restrict__ src, int ld, int R, int C,
                                                        uint8_t* __restrict__ out, int kbt, int fp16) {
  const int kb = blockIdx.x, rb = blockIdx.y;
  uint8_t* tile = out + ((size_t)rb * kbt + kb) * kPtileBytes;
  const int c8 = threadIdx.x & 7;
  const int col = kb * 64 + c8 * 8;
  const bool vec = (ld & 3) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0;
#pragma unroll
  for (int pass = 0; pass < 4; ++pass) {
    const int r = pass * 32 + (threadIdx.x >> 3);
    const int row = rb * 128 + r;
    float v[8];
    if (vec && row < R && col + 8 <= C) {
      const float4 x0 = *reinterpret_cast<const float4*>(src + (size_t)row * ld + col);
      const float4 x1 = *reinterpret_cast<const float4*>(src + (size_t)row * ld + col + 4);
      v[0] = x0.x; v[1] = x0.y; v[2] = x0.z; v[3] = x0.w; v[4] = x1.x; v[5] = x1.y; v[6] = x1.z; v[7] = x1.w;
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = (row < R && col + i < C) ? src[(size_t)row * ld + col + i] : 0.f;
    }
    __align__(16) uint16_t hi[8], lo[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) split16(v[i], fp16, &hi[i], &lo[i]);
    const uint32_t off = (uint32_t)r * 128u + (uint32_t)((c8 ^ (r & 7)) << 4);
    *reinterpret_cast<uint4*>(tile + off) = *reinterpret_cast<const uint4*>(hi);
    *reinterpret_cast<uint4*>(tile + kPtileHalf + off) = *reinterpret_cast<const uint4*>(lo);
  }
}

// K along the source's rows (points): operand row r = source column f (f < F valid), K index = source row p (p < P).
// grid (K blocks over points, row blocks over features); the 64 x 128 fp32 source block goes through shared memory.
__global__ void __launch_bounds__(256) pack_cols_kernel(const float* __restrict__ src, int ld, int P, int F,
                                                        uint8_t* __restrict__ out, int kbt, int fp16) {
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
    for (int i = 0; i < 8; ++i) split16(t[c8 * 8 + i][r], fp16, &hi[i], &lo[i]);
    const uint32_t off = (uint32_t)r * 128u + (uint32_t)((c8 ^ (r & 7)) << 4);
    *reinterpret_cast<uint4*>(tile + off) = *reinterpret_cast<const uint4*>(hi);
    *reinterpret_cast<uint4*>(tile + kPtileHalf + off) = *reinterpret_cast<const uint4*>(lo);
  }
}

// The same operand as pack_cols_kernel (operand row = source column f, K index = source row p) stored as MN-major tiles (ptx::make_mnmajor_sw128_desc): tile [feature block of 128][64-point K block] = [feature group of 64]
// [point row][128 B = 64 features]; a source row segment is copied as it lies, no transposition.  grid (K blocks over
// points, row blocks over features); 256 threads: 8 lanes cover one 128-byte line, 4 passes of 32 point rows, 2 groups.
__global__ void __launch_bounds__(256) pack_cols_mn_kernel(const float* __restrict__ src, int ld, int P, int F,
                                                        uint8_t* __restrict__ out, int kbt, int fp16) {
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
      for (int i = 0; i < 8; ++i) split16(v[i], fp16, &hi[i], &lo[i]);
      const uint32_t off = (uint32_t)g * 8192u + (uint32_t)r * 128u + (uint32_t)((c8 ^ (r & 7)) << 4);
      *reinterpret_cast<uint4*>(tile + off) = *reinterpret_cast<const uint4*>(hi);
      *reinterpret_cast<uint4*>(tile + kPtileHalf + off) = *reinterpret_cast<const uint4*>(lo);
    }
  }
}

}  // namespace

size_t pack_bytes(int rows, int k) { return (size_t)((rows + 127) / 128) * ((k + 63) / 64) * kPtileBytes; }

int launch_pack_rows(const float* src, int ld, int R, int C, uint8_t* out, int fp16, cudaStream_t st, int64_t* launches) {
  if (R <= 0 || C <= 0) return 0;
  dim3 grid((C + 63) / 64, (R + 127) / 128);
  pack_rows_kernel<<<grid, 256, 0, st>>>(src, ld, R, C, out, (C + 63) / 64, fp16);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

int launch_pack_cols(const float* src, int ld, int P, int F, uint8_t* out, int kbt, int fp16, cudaStream_t st, int64_t* launches, int mn) {
  if (P <= 0 || F <= 0) return 0;
  if (kbt <= 0) kbt = (P + 63) / 64;                  // callers may ask for zero-filled K blocks beyond P
  dim3 grid(kbt, (F + 127) / 128);
  if (mn) pack_cols_mn_kernel<<<grid, 256, 0, st>>>(src, ld, P, F, out, kbt, fp16);
  else pack_cols_kernel<<<grid, 256, 0, st>>>(src, ld, P, F, out, kbt, fp16);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

int launch_tc_gemm(TcGemmParams P, int num_sms, cudaStream_t st, int64_t* launches) {
  if (P.M <= 0 || P.N <= 0) return 0;
  NM_CHECK(P.nseg >= 1 && P.nseg <= 2 && P.seg[0].nkb > 0, "bad K segments");
  const int n_rb_a = (P.M + 127) / 128;
  P.n_rb_b = (P.N + 127) / 128;
  const int NB = P.n_rb_b >= 2 ? 2 : 1;
  const int col_groups = (P.n_rb_b + NB - 1) / NB;
  int splits = 1;
  P.kb_per_split = 0;
  NM_CHECK(!P.a_rowsum || (P.atomic && !P.fp16), "a_rowsum needs split-K with a bf16 A operand");
  if (P.atomic) {
    NM_CHECK(P.nseg == 1, "split-K takes one K segment");
    const int tiles = n_rb_a * col_groups;
    splits = num_sms / tiles;                                  // one wave: every extra split costs a full atomic epilogue
    const int max_splits = (P.seg[0].nkb + 7) / 8;              // at least 8 K blocks (512 points) per split
    if (splits > max_splits) splits = max_splits;
    if (splits < 1) splits = 1;
    P.kb_per_split = (P.seg[0].nkb + splits - 1) / splits;
    splits = (P.seg[0].nkb + P.kb_per_split - 1) / P.kb_per_split;
  }
  static const int dbg_env = [] { const char* e = getenv("NM_GEMM_DBG"); return e ? atoi(e) : 0; }();
  P.dbg = dbg_env;
  static thread_local unsigned configured = 0;
  int dev = 0;
  NM_CUDA(cudaGetDevice(&dev));
  const size_t smem = kGemmSmem;
  if (!(configured & (1u << (dev & 31)))) {
    NM_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    NM_CUDA(cudaFuncSetAttribute(tc_gemm_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    configured |= 1u << (dev & 31);
  }
  P.n_rb_a = n_rb_a;
  P.col_groups = col_groups;
  const int tiles = n_rb_a * col_groups;
  dim3 grid = P.atomic ? dim3(n_rb_a, col_groups, splits) : dim3(tiles < num_sms ? tiles : num_sms, 1, 1);
  if (NB == 2) tc_gemm_kernel<2><<<grid, kGemmThreads, smem, st>>>(P);
  else tc_gemm_kernel<1><<<grid, kGemmThreads, smem, st>>>(P);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

}  // namespace nm
