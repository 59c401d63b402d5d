// Fused FlexibleNeRFModel forward on the Hopper tensor cores (sm_90a, wgmma): positional encoding -> all linear layers
// -> sigma / rgb heads in ONE persistent kernel.  Activations never leave the SM: the fp32 accumulator of a layer lives
// in the registers of a warpgroup, whose epilogue turns it (bias, ReLU, fp16 hi/lo split) into the next layer's A
// operand in shared memory (128B-swizzled K-major tiles that wgmma reads through a descriptor), and the weights stream
// through a shared-memory ring filled by the bulk-copy (TMA) engine from an L2-resident, pre-swizzled image: the wide
// stream of nm_program.h, whose stages hold 64-deep K-blocks of 128 (64) output rows.
//
// Reference semantics: src/nerf/models.py:60-80 (network), src/nerf/modules.py:26-34 (encoding).
//
// Arithmetic (NM_PREC_EXACT): every product x*W is evaluated as xh*Wh + xl*Wh + xh*Wl with x = xh + xl, W = Wh + Wl
// fp16 splits and fp32 accumulation — three f16 MMAs per K-step (SURVEY 7.3.1: 1.5e-6 max-abs on composited RGB
// against fp32, where plain fp16 gives 3.3e-3).  NM_PREC_FAST issues only xh*Wh.
//
// CTA = 12 warps:
//   warps 0-3, 4-7  two consumer warpgroups.  Each owns a 64-point tile at a time (its own tile sequence), its own
//                   activation buffer (4 K-blocks x hi/lo, 64 KB) and encoding buffer (one K-block x hi/lo, 16 KB), and
//                   walks the layer program: encodings -> for each layer, m64nWk16 wgmmas at W = min(n_out, 128) columns
//                   into the register accumulator (128 fp32 registers per thread) -> epilogue straight from the
//                   accumulator fragments back into the activation buffer.
//   warps 8-11      producer: warp 8 issues cp.async.bulk weight stages (16 KB, hi|lo) into the ring.  The two
//                   warpgroups take turns on it (ping-pong): per round the producer streams layer 0's stages for
//                   warpgroup 0, the same stages again for warpgroup 1, then layer 1 for warpgroup 0, and so on.  Each
//                   fill has one owner, which waits on its own full barrier and alone releases the stage (empty barrier
//                   count 1).  Warpgroup 1's stages of a layer land only as warpgroup 0 releases its own, and warpgroup
//                   0's next layer only after all of them, so one warpgroup's epilogue runs under the other's MMAs.
//                   A warpgroup without a tile in a round gets no stages at all; that is only ever warpgroup 1, after
//                   its own last tile (with tile groups of G tiles, for up to G final rounds).
// The view-direction encoding reuses the encoding buffer: every layer that reads the xyz encoding precedes the one that
// reads the directions (checked at launch).  So does the fused compositor's staging, from the final layer's epilogue to the
// next tile's encoding.  Inference reads the bias and head vectors through the read-only data cache, which leaves shared
// memory to the weight ring (4 slots on an H100).
//
// Three template modes — 0 inference; 1 training forward, whose epilogue also emits the backward's operands (relu bit
// masks, head activations, point-major bf16 hi/lo packs); 2 the whole data-gradient chain of the backward on a backward
// layer program (dZ as the A operand, W^T streamed through the ring, bf16 hi/lo).  Mode 0 on ray inputs composites in
// the kernel: the warpgroup runs VolumeRenderer per ray in sample order (nm_composite.cuh) on its tile's staged outputs;
// tiles are dealt in ray-aligned groups and a carry slot passes the ray cut by a tile edge to the next tile.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstdio>
#include <cstdlib>
#include <vector>

#include "nm_common.h"
#include "nm_composite.cuh"
#include "nm_frontend.cuh"
#include "nm_ptx.cuh"

namespace nm {

namespace {

constexpr int kThreads = 384;
constexpr int kProdWarp = 8;                       // warps 8-11: the producer warpgroup (warp 8 issues, 9-11 only lend registers)
constexpr uint32_t kKBlock = 2 * 8192;             // one K-block of a 64-point tile: [hi 64 rows x 128 B | lo]
constexpr uint32_t kActBytes = 4 * kKBlock;        // activation buffer of one warpgroup (K up to 256)
constexpr uint32_t kWgBytes = kActBytes + kKBlock; // + its encoding buffer
constexpr int kMaxStages = 8;
constexpr uint32_t kCarryBytes = 64;             // per warpgroup: the compositor's two carry slots (its staging lives in the encoding buffer)

struct TcParams {
  NetProgram net;   // by value: lives in the constant bank
  const uint8_t* wpack;
  const float* bias;
  const float* head;
  MlpInput in;
  float* out;
  int out_sigma_only;
  int n_passes;
  float act_scale, act_inv_scale;
  int num_stages;
  long long n_tiles;
  int* err;
  uint32_t off_wg, off_bias, off_head, off_bars, off_carry;   // off_bias / off_head: modes 1 and 2 only
  int has_emit;     // training: the epilogue also writes the backward pass's operands (MlpEmit)
  MlpEmit emit;
  // mode 2: the data-gradient chain of the training backward (a KIND_LOAD / KIND_BWD program, W^T stages in bf16 hi/lo):
  // emit.bits[li] is the INPUT relu mask of that layer, emit.packT[li] receives dZ
  int mode;
  const float* dz_in;     // (M, dz_ld) fp32: dZ of the last forward layer
  int dz_ld;
  const float* dout;      // (M, 4): compositor adjoint, column 3 = d sigma
  // fused compositor (mode 0, ray inputs): the last layer's (rgb, sigma) of a tile are staged in shared memory instead of
  // going to `out`; the warpgroup composites every ray in sample order (nm_composite.cuh) and writes the per-ray maps.
  int comp_on;
  int tile_group;         // tiles per scheduling group = lcm(S, 64) / 64 when compositing (rays never straddle groups), else 1
  CompositeArgs comp;
};
static_assert(sizeof(TcParams) <= 4096, "TcParams must fit the 4 KB kernel-parameter window");

// NM_MLP_STALLS=1 (diagnostic build: NM_NVCC_EXTRA=-DNM_MLP_STALLS=1): thread 0 of each consumer warpgroup splits its
// clock64() time into weight-ring full waits, the MMA main loop (its waits excluded), the encodings, the layer epilogues
// (from the end of the MMA loop, so including the first barrier's wait for the other warps' last MMAs), the compositor and
// the rest, and the first two and the last CTA of a launch printf the totals at exit.  The counters live in shared
// memory after the barriers to keep register pressure down; the instrumented kernel still spills more than the shipped
// one, so its split is approximate.
#ifndef NM_MLP_STALLS
#define NM_MLP_STALLS 0
#endif
#if NM_MLP_STALLS
#define NM_ST(...) __VA_ARGS__
#else
#define NM_ST(...)
#endif

// barrier slots (8 B each) relative to off_bars: full[wg][s] at kBarWFull + 64 wg + 8 s, empty[s] (+ the NM_MLP_STALLS
// counters, 8 per warpgroup: wait, mma, start, encoding, epilogue, compositor)
constexpr uint32_t kBarWFull = 0, kBarWEmpty = 128, kBarStalls = 192, kBarBytes = 192 + (NM_MLP_STALLS ? 128 : 0);

enum : int { ERR_ALIGN = 1, ERR_W_EMPTY = 2, ERR_W_FULL = 3 };

__device__ __forceinline__ uint16_t f16_bits_sat(float a) {
  uint16_t h;
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(h) : "f"(a));
  return h;
}
__device__ __forceinline__ float f16_bits_to_float(uint16_t h) {
  float f;
  asm("cvt.f32.f16 %0, %1;" : "=f"(f) : "h"(h));
  return f;
}
__device__ __forceinline__ uint32_t swz_off(int r, int c) {
  return (uint32_t)r * 128u + (uint32_t)((((c >> 3) ^ (r & 7)) << 4) + ((c & 7) << 1));
}
__device__ __forceinline__ void split_bf16x2(float a0, float a1, uint32_t* hi, uint32_t* lo) {
  const __nv_bfloat162 h2 = __floats2bfloat162_rn(a0, a1);
  const float2 f = __bfloat1622float2(h2);
  const __nv_bfloat162 l2 = __floats2bfloat162_rn(a0 - f.x, a1 - f.y);
  *hi = *reinterpret_cast<const uint32_t*>(&h2);
  *lo = *reinterpret_cast<const uint32_t*>(&l2);
}

// The MMAs of one K-block (four K = 16 steps) into a W-column accumulator d, in the canonical order of every column:
// HH: a_hi*b_hi then (LH) a_lo*b_hi over the four steps; HL: a_hi*b_lo.  Straight-line: no guard between two wgmmas, so
// ptxas issues the group back to back.  A and B steps are 32 B apart in their 128B-swizzled K-major tiles.
template <int W, int HH, int LH, int HL, int BF16>
__device__ __forceinline__ void mma_kblock(float* d, uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (HH) ptx::wgmma<W, 0, 0, BF16>(d, a_hi + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (LH) ptx::wgmma<W, 0, 0, BF16>(d, a_lo + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (HL) ptx::wgmma<W, 0, 0, BF16>(d, a_hi + 2 * k, b_lo + 2 * k, 1u);
}

template <int V>
struct IntC {
  static constexpr int value = V;
};

// MODE 0: inference; 1: training forward (the epilogue also emits the backward's operands); 2: data-gradient chain
template <int MODE>
__global__ void __launch_bounds__(kThreads, 1) mlp_tc_kernel(const __grid_constant__ TcParams P) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t sbase = ptx::smem_u32(smem);
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const uint32_t bars = sbase + P.off_bars;
  const int NS = P.num_stages;
  const int n_layers = P.net.n_layers;
  // Bias and head vectors: inference reads them through the read-only data cache, which leaves its shared memory to the
  // weight ring; the training modes, whose epilogues stream their emitted operands through L1, keep copies in shared memory.
  float* s_bias = reinterpret_cast<float*>(smem + P.off_bias);
  float* s_head = reinterpret_cast<float*>(smem + P.off_head);
  const float* vbias = MODE == 0 ? P.bias : s_bias;
  const float* vhead = MODE == 0 ? P.head : s_head;
  auto ldv = [](const float* p) -> float { if constexpr (MODE == 0) return __ldg(p); else return *p; };

  // ---------------------------------------------------------------- one-time setup
  if (threadIdx.x == 0) {
    if (sbase & 1023u) { atomicExch(P.err, ERR_ALIGN); __trap(); }
    for (int i = 0; i < kMaxStages; ++i) {
      ptx::mbar_init(bars + kBarWFull + 8 * i, 1);
      ptx::mbar_init(bars + kBarWFull + 64 + 8 * i, 1);
      ptx::mbar_init(bars + kBarWEmpty + 8 * i, 1);
    }
    ptx::fence_mbar_init();
  }
  if (MODE != 0) {
    for (int i = threadIdx.x; i < P.net.n_bias; i += kThreads) s_bias[i] = (MODE == 2) ? 0.f : P.bias[i];
    for (int i = threadIdx.x; i < P.net.n_head; i += kThreads) s_head[i] = P.head[i];
  }
  __syncthreads();

  // i-th tile of worker v (two workers per CTA, one per consumer warpgroup): groups of `tile_group` consecutive tiles are
  // dealt round-robin to the workers.  Returns -1 past the end.  Round i exists when worker 2 * blockIdx.x (the lower one)
  // has a tile; for a given i the higher worker's tile is the lower one's + Gt, so it lacks one only after its own last
  // tile (for up to Gt rounds), and both sides evaluate per round whether its stages are in the stream.
  const uint32_t Gt = (uint32_t)P.tile_group, V = 2u * gridDim.x, v0 = 2u * blockIdx.x;
  auto tile_of = [&](uint32_t v, uint32_t i) -> long long {
    const long long g = (long long)v + (long long)(i / Gt) * (long long)V;
    const long long t = g * (long long)Gt + (long long)(i % Gt);
    return t < P.n_tiles ? t : -1;
  };

  // the register file is re-divided per warpgroup: 2 x 232 for the consumers (128 accumulators each), 40 for the producer
  if (warp >= kProdWarp) {
    // =============================================================== weight producer
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == kProdWarp && lane == 0) {
      int slot = 0;
      uint32_t ph = 0;
      const bool exact = P.n_passes == 3;
      for (uint32_t i = 0; tile_of(v0, i) >= 0; ++i) {
        const int n_wg = tile_of(v0 + 1, i) >= 0 ? 2 : 1;
        int b0 = 0;                      // image stage of the layer's first stage
        for (int li = 0; li < n_layers; ++li) {
          const LayerProg& L = P.net.layers[li];
          const bool wide = wide_width(L) == 128;
          // exact: every stage in full; fast: the hi stages of a 128-wide layer, the hi half of a 64-wide layer's blocks
          const uint32_t bytes = (exact || wide) ? (uint32_t)kStageBytes : (uint32_t)kHalfStage;
          const int b1 = b0 + wide_stages(L);
          for (int w = 0; w < n_wg; ++w) {
            const uint32_t full = bars + kBarWFull + 64u * (uint32_t)w;
            for (int b = b0; b < b1; b += (wide && !exact) ? 2 : 1) {
              ptx::mbar_wait(bars + kBarWEmpty + 8 * slot, ph ^ 1, P.err, ERR_W_EMPTY);
              ptx::mbar_expect_tx(full + 8 * slot, bytes);
              ptx::bulk_g2s(sbase + (uint32_t)slot * kStageBytes, P.wpack + (size_t)b * kStageBytes, bytes, full + 8 * slot);
              if (++slot == NS) { slot = 0; ph ^= 1; }
            }
          }
          b0 = b1;
        }
      }
    }
    return;
  }

  // =============================================================== consumer warpgroups
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wg = warp >> 2, t = threadIdx.x & 127, wi = warp & 3;
  const uint32_t v = v0 + (uint32_t)wg;
  const int bar_id = 1 + wg;
  uint8_t* act = smem + P.off_wg + (uint32_t)wg * kWgBytes;       // K-block kb: hi at kb * kKBlock, lo 8 KB further
  uint8_t* pe = act + kActBytes;
  const uint32_t act_s = ptx::smem_u32(act), pe_s = ptx::smem_u32(pe);
  const int r0 = wi * 16 + (lane >> 2);                           // this thread's accumulator rows: r0, r0 + 8
  const int cq = 2 * (lane & 3);                                  // ... and columns 8 j + cq, + 1
  const float so = P.act_scale, si = P.act_inv_scale;
  const int n_passes = P.n_passes;
  const int Lx = P.net.L_xyz, Ld = P.net.L_dir, ix = P.net.inc_xyz, idr = P.net.inc_dir;
  // The ring position walks every fill, the other warpgroup's included; parities are per slot and count own fills only, so
  // a wait on full[wg][s] is never more than one phase from the barrier's.
  const uint32_t full_w = bars + kBarWFull + 64u * (uint32_t)wg;
  int slot = 0;
  uint32_t ph = 0;                 // bit s: parity of this warpgroup's next fill of slot s
  float acc[128];
  NM_ST(volatile long long* const st = reinterpret_cast<volatile long long*>(smem + P.off_bars + kBarStalls) + 8 * wg;
        if (t == 0) { st[0] = 0; st[1] = 0; st[2] = clock64(); st[3] = 0; st[4] = 0; st[5] = 0; })

  // encoding of this tile's points (xyz or view direction) -> the encoding buffer, columns past the width zeroed
  auto encode = [&](long long tile, bool dir) {
    NM_ST(const long long c0 = clock64();)
    ptx::named_bar_sync(bar_id, 128);          // every wgmma of the warpgroup that read the buffer has completed
    if (t < 64) {
      long long m = tile * kTileM + t;
      if (m >= P.in.M) m = P.in.M - 1;
      float p[3], d[3];
      fetch_point(P.in, m, p, d);
      auto emit = [&](int j, float val) {
        const float a = val * si;
        const uint16_t h = f16_bits_sat(a);
        const uint32_t off = swz_off(t, j);
        *reinterpret_cast<uint16_t*>(pe + off) = h;
        *reinterpret_cast<uint16_t*>(pe + 8192 + off) = f16_bits_sat(a - f16_bits_to_float(h));
      };
      const int dim = dir ? P.net.dim_dir : P.net.dim_xyz;
      for (int j = dim; j < 64; ++j) {
        const uint32_t off = swz_off(t, j);
        *reinterpret_cast<uint16_t*>(pe + off) = 0;
        *reinterpret_cast<uint16_t*>(pe + 8192 + off) = 0;
      }
      if (dir) positional_encoding(d, Ld, idr, P.net.freq_dir, emit);
      else positional_encoding(p, Lx, ix, P.net.freq_xyz, emit);
    }
    ptx::fence_proxy_async_smem();
    ptx::named_bar_sync(bar_id, 128);
    NM_ST(if (t == 0) st[3] += clock64() - c0;)
  };

  // Fused compositor on tile `itp` of this warpgroup, whose last layer is staged in shared memory.  Same arithmetic, in the
  // same order, as composite_kernel (nm_composite.cuh):  A  every thread takes ONE sample: alpha, keep (the exp lives
  // here);  B  one thread per ray segment runs the transmittance product chain through shared memory;  C  every thread:
  // weight, mask, the four products;  D  one lane per (segment, accumulator) runs the five ordered sums.  The ray cut by
  // the tile's upper edge leaves T and its partial sums in a carry slot for the next tile (tiles of a group are
  // consecutive for this warpgroup and groups start on ray boundaries).
  // The staging arrays live in the encoding buffer, dead from the final layer's MMAs to the next tile's encoding; the carry
  // slots, which outlive the tile, have their own.
  float* carry = reinterpret_cast<float*>(smem + P.off_carry + (uint32_t)wg * kCarryBytes);
  auto composite_tile = [&](uint32_t itp, long long tp) {
    const CompositeArgs& A = P.comp;
    const int r = t;
    float4* stage = reinterpret_cast<float4*>(pe);                          // q per sample, later (w r, w g, w b, w t)
    float* keepT = reinterpret_cast<float*>(pe + 64 * 16);                  // keep per sample, later T
    float* wv = keepT + 64;                                                 // weight per sample
    const float* carry_in = carry + ((itp & 1) ^ 1) * 8;                    // written by the previous tile
    float* carry_out = carry + (itp & 1) * 8;
    const long long p0 = tp * kTileM, p1 = min(p0 + (long long)kTileM, P.in.M);
    const int S = A.S;
    const long long ray_first = p0 / S;
    const int n_seg = (int)((p1 - 1) / S - ray_first) + 1;
    ptx::named_bar_sync(bar_id, 128);            // the staged outputs are visible
    // ---- A
    const long long p = p0 + r;
    const bool live = r < kTileM && p < p1;
    float tc = 0.f, alpha = 0.f;
    float4 q = make_float4(0.f, 0.f, 0.f, 0.f);
    if (live) {
      const long long ray = p / S;
      const int i = (int)(p - ray * S);
      const float* tr = A.t + ray * S;
      tc = tr[i];
      const float tn = (i + 1 < S) ? tr[i + 1] : 0.f;
      q = stage[r];
      float keep;
      alpha = comp_alpha(A, ray, i, tc, tn, comp_ray_norm(A.dirs, ray), q.w, &keep);
      keepT[r] = keep;
    }
    ptx::named_bar_sync(bar_id, 128);
    // ---- B
    for (int k = r; k < n_seg; k += 128) {
      const long long rayk = ray_first + k;
      const long long s0 = max(rayk * (long long)S, p0), s1 = min((rayk + 1) * (long long)S, p1);
      float T = (s0 > rayk * (long long)S) ? carry_in[0] : 1.0f;
      for (int j = (int)(s0 - p0); j < (int)(s1 - p0); ++j) { const float kp = keepT[j]; keepT[j] = T; T = __fmul_rn(T, kp); }
      if (s1 < (rayk + 1) * (long long)S) carry_out[0] = T;
    }
    ptx::named_bar_sync(bar_id, 128);
    // ---- C
    if (live) {
      const float T = keepT[r];
      const float w = __fmul_rn(alpha, T);
      if (A.weights) A.weights[p] = w;
      if (A.mask_weights) A.mask_weights[p] = (T > A.thr) ? 1.f : 0.f;
      wv[r] = w;
      stage[r] = make_float4(__fmul_rn(w, q.x), __fmul_rn(w, q.y), __fmul_rn(w, q.z), __fmul_rn(w, tc));
    }
    ptx::named_bar_sync(bar_id, 128);
    // ---- D: lane c of an 8-lane group owns accumulator c (r, g, b, acc, depth) of the group's segment
    for (int k0 = 0; k0 < n_seg; k0 += 16) {
      const int k = k0 + (r >> 3), c = r & 7;
      const long long rayk = ray_first + k;
      const long long s0 = max(rayk * (long long)S, p0), s1 = min((rayk + 1) * (long long)S, p1);
      const bool actv = k < n_seg && c < 5;
      float sum = 0.f;
      if (actv) {
        if (s0 > rayk * (long long)S) sum = carry_in[1 + c];
        const float* src = (c == 3) ? wv : reinterpret_cast<const float*>(stage) + (c == 4 ? 3 : c);
        const int stride = (c == 3) ? 1 : 4;
        for (int j = (int)(s0 - p0); j < (int)(s1 - p0); ++j) sum = __fadd_rn(sum, src[j * stride]);
      }
      const float s_g = __shfl_down_sync(0xffffffffu, sum, 1), s_b = __shfl_down_sync(0xffffffffu, sum, 2);
      const float s_a = __shfl_down_sync(0xffffffffu, sum, 3), s_d = __shfl_down_sync(0xffffffffu, sum, 4);
      if (actv && c == 0) {
        if (s1 == (rayk + 1) * (long long)S) {
          CompState cs;
          cs.T = 0.f; cs.r = sum; cs.g = s_g; cs.b = s_b; cs.acc = s_a; cs.depth = s_d;
          comp_finish(cs, A, rayk);
        } else {
          carry_out[1] = sum; carry_out[2] = s_g; carry_out[3] = s_b; carry_out[4] = s_a; carry_out[5] = s_d;
        }
      }
    }
    ptx::named_bar_sync(bar_id, 128);            // staging block consumed, carry visible to the next tile
  };

  // point-major bf16 hi/lo pack of the weight-gradient GEMM: features f, f+1 of point pt (nm_gemm.h ptiles of 128 features
  // x 64 points).  Mode 2 (dZ, the GEMM's A operand) writes MN-major tiles: feature group (f % 128) / 64, point row pt % 64,
  // chunk ((f % 64) / 8) ^ (pt % 8); mode 1 (activations, its B operand) K-major ones: row f % 128, 16-byte chunk
  // ((pt % 64) / 8) ^ (f % 8)
  auto emit_pack = [&](uint8_t* packT, int f, long long pt, uint32_t hi2, uint32_t lo2) {
    uint8_t* tb = packT + ((size_t)(f >> 7) * (size_t)P.emit.kbt + (size_t)(pt >> 6)) * 32768u;
    if (MODE == 2) {
      const uint32_t off = (uint32_t)((f & 127) >> 6) * 8192u + (uint32_t)(pt & 63) * 128u +
                           ((((uint32_t)(f & 63) >> 3) ^ (uint32_t)(pt & 7)) << 4) + (uint32_t)(f & 7) * 2u;
      *reinterpret_cast<uint32_t*>(tb + off) = hi2;
      *reinterpret_cast<uint32_t*>(tb + 16384u + off) = lo2;
    } else {
      const uint32_t c8 = (uint32_t)((pt & 63) >> 3);
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int fe = f + e;
        const uint32_t off = (uint32_t)(fe & 127) * 128u + ((c8 ^ (uint32_t)(fe & 7)) << 4) + (uint32_t)(pt & 7) * 2u;
        *reinterpret_cast<uint16_t*>(tb + off) = (uint16_t)(e ? (hi2 >> 16) : (hi2 & 0xffffu));
        *reinterpret_cast<uint16_t*>(tb + 16384u + off) = (uint16_t)(e ? (lo2 >> 16) : (lo2 & 0xffffu));
      }
    }
  };

  float sigma_val[2] = {0.f, 0.f};
  const int stream = n_passes == 3 ? 1 : 2;
  for (uint32_t it = 0; tile_of(v, it) >= 0; ++it) {
    const long long tile = tile_of(v, it);
    const bool peer = wg == 1 || tile_of(v0 + 1, it) >= 0;     // the other warpgroup's stages are in this round's stream
    if (MODE != 2) encode(tile, false);
    const long long m0 = tile * kTileM + r0, m1 = m0 + 8;
    const bool val0 = m0 < P.in.M, val1 = m1 < P.in.M;
    for (int li = 0; li < n_layers; ++li) {
      const LayerProg& L = P.net.layers[li];
      if (MODE != 2 && L.pe_src == SRC_PE_DIR) encode(tile, true);
      // this layer's stages of the other warpgroup: warpgroup 0's precede ours, warpgroup 1's follow them
      const int skip = peer ? wide_stages(L, stream) : 0;
      if (wg == 1) slot = (slot + skip) % NS;
      // ------------------------------------------------------------ main loop: this layer's stages of the wide stream
      // (per K-block — the encoding source's first, then the activation K-blocks in ascending order — and column half: the
      // hi stage's a_hi*b_hi, a_lo*b_hi group, then the lo stage's a_hi*b_lo group; a 64-wide layer has both in one stage).
      // Width and pass count are fixed per layer, so each instantiation's wgmma groups are straight-line.
      auto main_loop = [&](auto width, auto exact) {
        constexpr int N = decltype(width)::value, W = N > 128 ? 128 : N, EX = decltype(exact)::value;
#pragma unroll
        for (int i = 0; i < 128; ++i) acc[i] = 0.f;
        NM_ST(if (t == 0) st[1] -= clock64() - st[0];)      // + (loop end - loop start) - (waits inside the loop)
        int prev = -1;
        // one stage: wait for it, issue its group, release the previous stage once that group's MMAs are complete
        auto stage = [&](auto issue) {
          NM_ST(const long long c0 = clock64();)
          ptx::mbar_wait_warp(full_w + 8 * slot, (ph >> slot) & 1u, P.err, ERR_W_FULL);
          NM_ST(if (t == 0) st[0] += clock64() - c0;)
          ptx::wgmma_fence();                        // (what ptxas would otherwise inject before the group, C7519)
          issue(sbase + (uint32_t)slot * kStageBytes);
          ptx::wgmma_commit();
          ptx::wgmma_wait<1>();
          if (prev >= 0 && t == 0) ptx::mbar_arrive(bars + kBarWEmpty + 8 * prev);
          prev = slot;
          ph ^= 1u << slot;
          if (++slot == NS) slot = 0;
        };
        const int n_kb = wide_kblocks(L), has_pe = L.pe_src ? 1 : 0;
        for (int kbi = 0; kbi < n_kb; ++kbi) {
          const uint32_t a_t = (kbi < has_pe) ? pe_s : act_s + (uint32_t)(kbi - has_pe) * kKBlock;
          const uint64_t a_hi = ptx::make_kmajor_sw128_desc(a_t), a_lo = ptx::make_kmajor_sw128_desc(a_t + 8192u);
#pragma unroll
          for (int h = 0; h < N / W; ++h) {
            if (W == 64) {
              stage([&](uint32_t w) {
                mma_kblock<W, 1, EX, EX, MODE == 2>(acc, a_hi, a_lo, ptx::make_kmajor_sw128_desc(w),
                                                    ptx::make_kmajor_sw128_desc(w + (uint32_t)kHalfStage));
              });
            } else {
              stage([&](uint32_t w) {
                const uint64_t b = ptx::make_kmajor_sw128_desc(w);
                mma_kblock<W, 1, EX, 0, MODE == 2>(acc + 64 * h, a_hi, a_lo, b, b);
              });
              if (EX)
                stage([&](uint32_t w) {
                  const uint64_t b = ptx::make_kmajor_sw128_desc(w);
                  mma_kblock<W, 0, 0, 1, MODE == 2>(acc + 64 * h, a_hi, a_lo, b, b);
                });
            }
          }
        }
        ptx::wgmma_wait<0>();
        if (prev >= 0 && t == 0) ptx::mbar_arrive(bars + kBarWEmpty + 8 * prev);
        NM_ST(if (t == 0) st[1] += clock64() - st[0];)
        ptx::fence_regs<128>(acc);
      };
      if (L.kind != KIND_LOAD) {
        if (L.n_out == 256) {
          if (n_passes == 3) main_loop(IntC<256>{}, IntC<1>{}); else main_loop(IntC<256>{}, IntC<0>{});
        } else if (L.n_out == 128) {
          if (n_passes == 3) main_loop(IntC<128>{}, IntC<1>{}); else main_loop(IntC<128>{}, IntC<0>{});
        } else {
          if (n_passes == 3) main_loop(IntC<64>{}, IntC<1>{}); else main_loop(IntC<64>{}, IntC<0>{});
        }
      }
      if (wg == 0) slot = (slot + skip) % NS;
      // ------------------------------------------------------------ epilogue, straight from the accumulator fragments
      NM_ST(const long long ce = clock64();)
      const int NC = L.n_out >> 6;
      const bool writes_a = (L.kind == KIND_HIDDEN) || (L.kind == KIND_SIGMA && !L.is_final) || (L.kind == KIND_LOAD) ||
                            (L.kind == KIND_BWD && !L.is_final);
      const int heads = L.kind == KIND_SIGMA ? 1 : (L.kind == KIND_RGB ? 3 : (L.kind == KIND_OUT4 ? 4 : 0));
      uint8_t* packT = (MODE >= 1) ? P.emit.packT[li] : nullptr;
      float part[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
      float dsg[2] = {0.f, 0.f};
      if (MODE == 2 && L.kind == KIND_BWD && L.aux2) {
        dsg[0] = val0 ? P.dout[(size_t)m0 * 4 + 3] : 0.f;
        dsg[1] = val1 ? P.dout[(size_t)m1 * 4 + 3] : 0.f;
      }
      if (writes_a) ptx::named_bar_sync(bar_id, 128);    // every warp of the warpgroup is past this layer's MMAs
      // The layer's 64-column chunks.  PLAIN (mode 0, a layer without a head whose outputs go back to the activation buffer:
      // every hidden layer) is the same code with those two decisions fixed at compile time: each 8-column step is then one
      // basic block, and the scheduler overlaps the shared-memory loads and the fp16 split chains of consecutive steps.
      auto chunks = [&](auto plain) {
        constexpr bool PLAIN = decltype(plain)::value;
        const int heads_c = PLAIN ? 0 : heads;
        const bool writes_c = PLAIN || writes_a;
#pragma unroll
        for (int nc = 0; nc < 4; ++nc) {
          if (nc >= NC) continue;
          uint32_t mk_in[2][2] = {{0xffffffffu, 0xffffffffu}, {0xffffffffu, 0xffffffffu}};   // mode 2: [row][32-column word]
          if (MODE == 2 && L.kind == KIND_BWD && L.relu) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const long long m = e ? m1 : m0;
              if (e ? val1 : val0) {
                const uint2 bw = *reinterpret_cast<const uint2*>(P.emit.bits[li] + (size_t)m * (size_t)(L.n_out >> 5) + (size_t)(nc * 2));
                mk_in[e][0] = bw.x; mk_in[e][1] = bw.y;
              }
            }
          }
          uint32_t mk_out[2][2] = {{0u, 0u}, {0u, 0u}};
#pragma unroll
          for (int j8 = 0; j8 < 8; ++j8) {
            const int col = nc * 64 + j8 * 8 + cq;
            // bias_off is a multiple of 64 (layer widths are): an aligned pair
            float2 bias2 = make_float2(0.f, 0.f);
            if constexpr (MODE == 0) bias2 = __ldg(reinterpret_cast<const float2*>(vbias + L.bias_off + col));
            else if constexpr (MODE == 1) bias2 = *reinterpret_cast<const float2*>(vbias + L.bias_off + col);
            float x[2][2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const bool valid = e ? val1 : val0;
              const long long m = e ? m1 : m0;
              if (MODE == 2 && L.kind == KIND_LOAD) {
                // top of the data-gradient chain: dZ of the last forward layer, from HBM (rows past M are zero)
                const float2 z = valid ? *reinterpret_cast<const float2*>(P.dz_in + (size_t)m * P.dz_ld + col) : make_float2(0.f, 0.f);
                x[e][0] = z.x; x[e][1] = z.y;
              } else if (MODE == 2) {
                // dA = dZ W (+ d sigma * w_alpha), masked by relu' of the forward layer below.  (Its column sums — the bias
                // gradient — are taken by the weight-gradient GEMM from the pack emitted below: nm_gemm_tc.cu a_rowsum.)
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                  float y = acc[nc * 32 + j8 * 4 + 2 * e + u] * so;
                  if (L.aux2) y = fmaf(dsg[e], ldv(vhead + L.head_off + col + u), y);
                  const uint32_t w = valid ? mk_in[e][j8 >> 2] : 0u;
                  x[e][u] = ((w >> ((col + u) & 31)) & 1u) ? y : 0.f;
                }
              } else {
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                  float y = fmaf(acc[nc * 32 + j8 * 4 + 2 * e + u], so, u ? bias2.y : bias2.x);
                  if (L.relu) y = fmaxf(y, 0.f);
                  x[e][u] = y;
                }
              }
            }
#pragma unroll
            for (int hh = 0; hh < 4; ++hh) {
              if (hh >= heads_c) break;
              const float* w = vhead + L.head_off + hh * L.n_out + col;
              const float w0 = ldv(w), w1 = ldv(w + 1);
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                part[e][hh] = fmaf(w0, x[e][0], part[e][hh]);
                part[e][hh] = fmaf(w1, x[e][1], part[e][hh]);
              }
            }
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const bool valid = e ? val1 : val0;
              const long long m = e ? m1 : m0;
              const int row = r0 + 8 * e;
              if (MODE == 1) {
                // by-products for the training backward: relu mask bits and the fp32 copy (layers the head kernels read)
                mk_out[e][j8 >> 2] |= ((x[e][0] > 0.f ? 1u : 0u) | (x[e][1] > 0.f ? 2u : 0u)) << (col & 31);
                if (P.emit.act[li] && valid) *reinterpret_cast<float2*>(P.emit.act[li] + (size_t)m * L.n_out + col) = make_float2(x[e][0], x[e][1]);
              }
              if (writes_c) {
                uint32_t hi, lo;
                const float a0 = x[e][0] * si, a1 = x[e][1] * si;
                if (MODE == 2) {            // gradients: bf16 hi/lo (fp32's exponent range)
                  split_bf16x2(a0, a1, &hi, &lo);
                } else {
                  hi = ptx::pack_f16x2_sat(a0, a1);
                  const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&hi));
                  lo = ptx::pack_f16x2_sat(a0 - f.x, a1 - f.y);
                }
                if (n_passes != 3) lo = 0u;
                const uint32_t off = (uint32_t)nc * kKBlock + swz_off(row, col & 63);
                *reinterpret_cast<uint32_t*>(act + off) = hi;
                *reinterpret_cast<uint32_t*>(act + 8192u + off) = lo;
                if (MODE >= 1 && packT) {
                  // the weight-gradient operand is the A operand's value (hi + lo), as bf16 hi / lo; rows past M as zeros
                  uint32_t ph2 = 0u, pl2 = 0u;
                  if (valid) {
                    if (MODE == 2) {
                      ph2 = hi; pl2 = lo;
                    } else {
                      const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(&hi));
                      const float2 fl = __half22float2(*reinterpret_cast<const __half2*>(&lo));
                      split_bf16x2((fh.x + fl.x) * so, (fh.y + fl.y) * so, &ph2, &pl2);
                    }
                  }
                  emit_pack(packT, col, tile * kTileM + row, ph2, pl2);
                }
              } else if (MODE >= 1 && packT) {
                uint32_t ph2, pl2;
                split_bf16x2(valid ? x[e][0] : 0.f, valid ? x[e][1] : 0.f, &ph2, &pl2);
                emit_pack(packT, col, tile * kTileM + row, ph2, pl2);
              }
            }
          }
          if (MODE == 1 && P.emit.bits[li]) {     // relu mask: the four lanes of a quad hold the 32 bits of a row's word
#pragma unroll
            for (int e = 0; e < 2; ++e)
#pragma unroll
              for (int g = 0; g < 2; ++g) {
                uint32_t w = mk_out[e][g];
                w |= __shfl_xor_sync(0xffffffffu, w, 1);
                w |= __shfl_xor_sync(0xffffffffu, w, 2);
                const long long m = e ? m1 : m0;
                if ((lane & 3) == 0 && (e ? val1 : val0)) P.emit.bits[li][(size_t)m * (size_t)(L.n_out >> 5) + (size_t)(nc * 2 + g)] = w;
              }
          }
        }
      };
      if constexpr (MODE == 0) {
        if (heads == 0 && writes_a) chunks(IntC<1>{}); else chunks(IntC<0>{});
      } else {
        chunks(IntC<0>{});
      }
      if (writes_a) {
        ptx::fence_proxy_async_smem();           // the next layer's wgmmas read what the generic proxy wrote
        ptx::named_bar_sync(bar_id, 128);
      }
      if (heads) {
        // a row's columns are spread over the four lanes of a quad
#pragma unroll
        for (int e = 0; e < 2; ++e)
#pragma unroll
          for (int hh = 0; hh < 4; ++hh) {
            part[e][hh] += __shfl_xor_sync(0xffffffffu, part[e][hh], 1);
            part[e][hh] += __shfl_xor_sync(0xffffffffu, part[e][hh], 2);
          }
        const float* hb = vhead + L.head_off + heads * L.n_out;
        // the compositor stages the final layer's outputs in the encoding buffer: every warp's wgmmas are done reading it
        if (MODE == 0 && P.comp_on && L.is_final) ptx::named_bar_sync(bar_id, 128);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const long long m = e ? m1 : m0;
          const bool valid = e ? val1 : val0;
          if (L.kind == KIND_SIGMA) {
            sigma_val[e] = part[e][0] + ldv(hb);
            if (L.is_final && (lane & 3) == 0) {      // sigma-only program
              if (MODE == 0 && P.comp_on) reinterpret_cast<float4*>(pe)[r0 + 8 * e] = make_float4(0.f, 0.f, 0.f, sigma_val[e]);
              else if (valid && P.out) P.out[m] = sigma_val[e];
            }
          } else if ((lane & 3) == 0 && (P.comp_on || (valid && P.out))) {
            float o[4];
#pragma unroll
            for (int hh = 0; hh < 4; ++hh) o[hh] = (hh < heads) ? part[e][hh] + ldv(hb + hh) : 0.f;
            const float sg = (L.kind == KIND_RGB) ? sigma_val[e] : o[3];
            if (P.out_sigma_only) {
              P.out[m] = sg;
            } else {
              float4 res;
              res.x = 1.f / (1.f + expf(-o[0]));
              res.y = 1.f / (1.f + expf(-o[1]));
              res.z = 1.f / (1.f + expf(-o[2]));
              res.w = sg;
              if (MODE == 0 && P.comp_on) reinterpret_cast<float4*>(pe)[r0 + 8 * e] = res;
              else reinterpret_cast<float4*>(P.out)[m] = res;
            }
          }
        }
      }
      NM_ST(if (t == 0) st[4] += clock64() - ce;)
    }
    if (MODE == 0 && P.comp_on) {
      NM_ST(const long long c0 = clock64();)
      composite_tile(it, tile);
      NM_ST(if (t == 0) st[5] += clock64() - c0;)
    }
  }
  NM_ST(if (t == 0 && (blockIdx.x < 2 || blockIdx.x + 1 == gridDim.x))
          printf("mlp_stalls mode %d cta %d wg %d wait %lld mma %lld encode %lld epilogue %lld composite %lld other %lld\n", MODE,
                 (int)blockIdx.x, wg, st[0], st[1], st[3], st[4], st[5], clock64() - st[2] - st[0] - st[1] - st[3] - st[4] - st[5]);)
}

}  // namespace

// The kernel's shared-memory layout for program `hp`, a dynamic shared-memory limit of `max_smem` bytes, the fused
// compositor on or off and the mode (training: 1 and 2, which keep the bias and head vectors in shared memory): as many
// 16 KB ring slots as fit after the two warpgroups' activation and encoding buffers, the vectors, the barriers and the
// compositor's carry slots, at most kMaxStages and at most `slot_cap` (<= 0: no cap).  Pure host logic, so that the CPU
// tests check the layout the kernel launches with.
int mlp_tc_layout(const NetProgram& hp, int max_smem, bool comp_on, bool training, int slot_cap, MlpTcLayout* out) {
  auto align_up = [](uint32_t x, uint32_t a) { return (x + a - 1) / a * a; };
  const uint32_t vb = training ? align_up(hp.n_bias * 4, 16) : 0u, vh = training ? align_up((hp.n_head > 0 ? hp.n_head : 4) * 4, 16) : 0u;
  const uint32_t fixed = 2 * kWgBytes + vb + vh + kBarBytes + (comp_on ? 2 * kCarryBytes : 0u);
  int ns = ((int)max_smem - (int)fixed) / (int)kStageBytes;
  NM_CHECK(ns >= 2, "network too large for the shared-memory budget (%u B fixed, %d B available)", fixed, max_smem);
  if (ns > kMaxStages) ns = kMaxStages;
  if (slot_cap > 0 && ns > slot_cap) ns = slot_cap < 2 ? 2 : slot_cap;
  for (int i = 0; i < hp.n_layers; ++i)
    NM_CHECK(hp.layers[i].kind == KIND_LOAD || hp.layers[i].n_out == 64 || hp.layers[i].n_out == 128 || hp.layers[i].n_out == 256,
             "layer %d: output width %d not 64, 128 or 256", i, hp.layers[i].n_out);
  MlpTcLayout l{};
  l.num_stages = ns;
  uint32_t off = (uint32_t)ns * kStageBytes;
  l.off_wg = off; off += 2 * kWgBytes;
  l.off_bias = off; off += vb;
  l.off_head = off; off += vh;
  l.off_bars = off; off += kBarBytes;
  l.off_carry = off; off += comp_on ? 2 * kCarryBytes : 0u;
  l.bytes = off;
  NM_CHECK((int)off <= max_smem, "shared-memory layout overflow");
  *out = l;
  return 0;
}

// NM_MLP_RING_SLOTS=n (A/B and tests): at most n ring slots (n >= 2; it can only lower the depth the layout allows).  Read
// per launch, so a test can flip it between calls.
static int ring_slot_cap() {
  const char* e = getenv("NM_MLP_RING_SLOTS");
  return e ? atoi(e) : 0;
}

// shared-memory layout + launch of a prepared parameter block
static int launch_prepared(TcParams& P, int num_sms, cudaStream_t st, int64_t* launches) {
  const NetProgram& hp = P.net;
  {
    bool dir_seen = false;
    for (int i = 0; i < hp.n_layers; ++i) {
      NM_CHECK(!(dir_seen && hp.layers[i].pe_src == SRC_PE_XYZ), "xyz encoding read after the view-direction encoding");
      if (hp.layers[i].pe_src == SRC_PE_DIR) dir_seen = true;
    }
  }
  int dev = 0, max_smem = 0;
  NM_CUDA(cudaGetDevice(&dev));
  NM_CUDA(cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const int mode = P.mode == 2 ? 2 : (P.has_emit ? 1 : 0);
  MlpTcLayout lay;
  if (int e = mlp_tc_layout(hp, max_smem, P.comp_on != 0, mode != 0, ring_slot_cap(), &lay)) return e;
  P.num_stages = lay.num_stages;
  P.off_wg = lay.off_wg; P.off_bias = lay.off_bias; P.off_head = lay.off_head; P.off_bars = lay.off_bars; P.off_carry = lay.off_carry;
  const uint32_t off = lay.bytes;
  if (P.tile_group < 1) P.tile_group = 1;

  auto kern = mode == 2 ? mlp_tc_kernel<2> : (mode == 1 ? mlp_tc_kernel<1> : mlp_tc_kernel<0>);
  static thread_local unsigned configured_devs[3] = {0, 0, 0};   // per-device opt-in to the large dynamic shared memory window
  if (!(configured_devs[mode] & (1u << (dev & 31)))) {
    NM_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    configured_devs[mode] |= 1u << (dev & 31);
  }
  const long long n_groups = (P.n_tiles + P.tile_group - 1) / P.tile_group;
  const long long pairs = (n_groups + 1) / 2;                   // two workers (consumer warpgroups) per CTA
  const long long grid = pairs < num_sms ? pairs : num_sms;
  kern<<<(unsigned)grid, kThreads, off, st>>>(P);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  return 0;
}

// Tiles per scheduling group for a fused compositor over S samples per ray (0: not eligible — fall back to raw + composite_kernel)
int mlp_tc_composite_group(int S) {
  if (S <= 0) return 0;
  int a = S, b = kTileM;
  while (b) { const int t = a % b; a = b; b = t; }
  const long long l = (long long)S / a * kTileM;      // lcm(S, kTileM)
  const long long g = l / kTileM;
  return g <= 16 ? (int)g : 0;                         // long groups would unbalance the workers
}

int launch_mlp_tc(const NetDev& net, bool sigma_only, int n_passes, int act_scale_log2, const MlpInput& in, float* out,
                  int num_sms, int* d_err, cudaStream_t st, int64_t* launches, const MlpEmit* emit, const CompositeArgs* comp) {
  if (in.M <= 0) return 0;
  const NetProgram& hp = sigma_only ? net.sigma : net.full;
  TcParams P{};
  P.net = hp;
  P.wpack = sigma_only ? net.d_wpack_sigma : net.d_wpack_full;
  P.bias = net.d_bias;
  P.head = net.d_head;
  P.in = in;
  P.out = out;
  P.out_sigma_only = sigma_only ? 1 : 0;
  P.n_passes = n_passes;
  P.act_scale = ldexpf(1.f, act_scale_log2);
  P.act_inv_scale = ldexpf(1.f, -act_scale_log2);
  P.n_tiles = (in.M + kTileM - 1) / kTileM;
  P.err = d_err;
  if (emit) {
    P.has_emit = 1; P.emit = *emit;
    P.n_tiles = 2 * ((in.M + 127) / 128);      // the packs hold whole 128-point blocks: their zero rows are written too
  }
  P.tile_group = 1;
  if (comp) {
    NM_CHECK(!emit && in.mode == IN_RAYS && comp->S == in.S && comp->R * (long long)comp->S == in.M && comp->t == in.t,
             "fused compositor: needs the ray front end on the compositor's own samples");
    P.tile_group = mlp_tc_composite_group(comp->S);
    NM_CHECK(P.tile_group > 0, "fused compositor: %d samples per ray not supported", comp->S);
    NM_CHECK(!sigma_only || (!comp->rgb && hp.layers[hp.n_layers - 1].kind == KIND_SIGMA),
             "fused compositor: the sigma-only program must end in a sigma layer and write no colour map");
    P.comp_on = 1; P.comp = *comp; P.out = nullptr;
  }
  return launch_prepared(P, num_sms, st, launches);
}

// The data-gradient chain of the training backward for M points (nm_train.cu): dz_in (M, dz_ld) fp32 = dZ of the last
// forward layer; for every backward layer li (net.bwd): io.bits[li] = relu mask to apply (input), io.packT[li] = where dZ
// goes as the weight-gradient operand (its row sums there are the bias gradients: launch_tc_gemm a_rowsum).
int launch_mlp_tc_bwd(const NetDev& net, long long M, const float* dz_in, int dz_ld, const float* dout,
                      const MlpEmit& io, int n_passes, int num_sms, int* d_err, cudaStream_t st, int64_t* launches) {
  if (M <= 0) return 0;
  NM_CHECK(net.bwd_valid && net.d_wpack_bwd, "backward weight stream not built");
  NM_CHECK((dz_ld & 1) == 0 && (reinterpret_cast<uintptr_t>(dz_in) & 7) == 0, "dz_in must be 8-byte aligned rows");
  TcParams P{};
  P.net = net.bwd;
  P.wpack = net.d_wpack_bwd;
  P.bias = net.d_bias;
  P.head = net.d_head;
  P.in.M = M;
  P.n_passes = n_passes;
  P.act_scale = 1.f; P.act_inv_scale = 1.f;
  P.n_tiles = 2 * ((M + 127) / 128);
  P.err = d_err;
  P.has_emit = 1; P.emit = io;
  P.mode = 2; P.dz_in = dz_in; P.dz_ld = dz_ld; P.dout = dout;
  return launch_prepared(P, num_sms, st, launches);
}

}  // namespace nm
