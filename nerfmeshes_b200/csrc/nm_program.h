// Layer "program" of one FlexibleNeRFModel (reference: src/nerf/models.py:5-80) as the fused kernels consume it.
// Built once on the host at weight-load time (nm_program.cu); read by the wgmma kernel (nm_mlp_tc.cu) and
// the fp32 CUDA-core kernel (nm_mlp_simt.cu).
#pragma once
#include <stdint.h>

namespace nm {

constexpr int kMaxLayers = 16;   // NetProgram travels as a kernel parameter (constant bank): keep it under 4 KB
constexpr int kMaxBlocks = 200;
constexpr int kMaxFreq = 16;

// tensor-core tiling constants
constexpr int kIssuers = 4;           // schedule bookkeeping only (BlockProg.flags >> 4); the wgmma kernel does not read it
constexpr int kTileM = 64;           // points per tile (= rows of one warpgroup MMA)
constexpr int kChunk = 64;           // N-chunk / K-block width
constexpr int kStageBytes = 16384;   // one weight stage / canonical block: [hi 64x64 fp16 | lo 64x64 fp16]
constexpr int kHalfStage = 8192;

enum : int { SRC_ACT = 0, SRC_PE_XYZ = 1, SRC_PE_DIR = 2 };
enum : int {
  KIND_HIDDEN = 0,   // y = act(Wx+b) becomes the next layer's A operand
  KIND_SIGMA = 1,    // hidden + the fc_alpha head (256->1) as a dot product in the epilogue
  KIND_RGB = 2,      // layers_dir.0 + the fc_rgb head (->3, sigmoid) in the epilogue; nothing written back
  KIND_OUT4 = 3,     // use_viewdirs=False: trunk output + fc_out head (->4)
  // backward (data-gradient) program of the training step, nm_train.cu: the same machine walks the layers in reverse
  KIND_LOAD = 4,     // no MMA: the epilogue loads the top gradient dZ (fp32, HBM) into the A operand
  KIND_BWD = 5       // dA = dZ W (+ dsigma w_alpha) masked by relu' of forward layer aux-1 -> next A, its pack, column sums
};

struct LayerProg {
  int32_t n_out;      // true output width (multiple of 64)
  int32_t k_act;      // width of the activation input (0 for layer1)
  int32_t pe_src;     // SRC_PE_XYZ / SRC_PE_DIR / 0: extra input columns appended after the activations
  int32_t k_pe;       // true PE width (63 / 27), 0 if none
  int32_t relu;
  int32_t kind;
  int32_t is_final;   // this layer's epilogue writes the kernel output
  int32_t bias_off;   // float offset into the bias array
  int32_t head_off;   // float offset into the head array: rows of the head weight then its bias
  int32_t blk_begin, blk_end;  // tensor-core block list
  int32_t wt_off;     // float offset into the transposed fp32 weights (CUDA-core kernel): Wt[k][n], k over [act|pe]
  // tensor-core kernel, 4 issuing warps: bit (issuer*4 + i) set when that issuer has
  // no block into accumulator chunk i (none_d) / no block reading activation K-block i (none_k) in this layer
  int32_t none_d, none_k;
  int32_t first_blk;  // byte w = offset from blk_begin of issuer w's first block in this layer, 0xFF = none
  int32_t aux;        // backward program: forward layer l whose W^T this layer streams (it produces dZ of layer l-1)
  int32_t aux2;       // backward program: 1 = add dsigma * w_alpha (forward layer l-1 carries the fc_alpha head)
};

// One (K-block, N-chunk) step of the tensor-core schedule == one 16 KB weight stage.
struct BlockProg {
  uint8_t src;     // SRC_*
  uint8_t kb;      // K-block index within the source (activation K-block kb of the shared-memory A operand)
  uint8_t nc;      // N-chunk: accumulator columns nc*64..
  uint8_t ksteps;  // 1..4 MMAs of K=16
  uint8_t group;   // needs epilogue chunks 0..group of the previous layer done
  uint8_t first;   // first block into this accumulator chunk in schedule order (the first MMA overwrites)
  uint8_t last;    // last block into this accumulator chunk in schedule order (bookkeeping / CPU replay)
  uint8_t flags;   // bit0: its issuer's last block into chunk nc; bit1: its issuer's last block reading K-block kb;
                   // bits 2-3: unused; bits 4-5: issuer warp
  uint8_t next;    // distance (in schedule blocks) to the same issuer's next block in this layer, 0 = none
};

struct NetProgram {
  int32_t n_layers;
  int32_t n_blocks;
  int32_t hidden;
  int32_t dim_xyz, dim_dir;      // true PE widths
  int32_t L_xyz, L_dir, inc_xyz, inc_dir;
  int32_t n_bias, n_head;        // floats
  int32_t uses_dir;              // some layer of THIS program reads the view-direction encoding
  int32_t accumulate_only;       // 1: blocks of a chunk come from several issuers (no order): always accumulate, epilogue re-zeroes
  float freq_xyz[kMaxFreq];
  float freq_dir[kMaxFreq];
  LayerProg layers[kMaxLayers];
  BlockProg blocks[kMaxBlocks];
};

// ---- the wide weight stream: what the wgmma kernel's ring walks (packers: nm_program.cu, reader: nm_mlp_tc.cu)
// The canonical 64x64 blocks above are the unit of scheduling and of the CPU checks; the device streams a layer at an MMA
// width W = min(n_out, 128) (n_out / W column halves).  Inside a layer, for every K-block of 64 (the encoding source first
// if the layer has one, then the activation K-blocks in ascending order) and every column half h:
//   W = 128: two 16 KB stages, the hi then the lo fp16 (bf16) copy of the 128 x 64 tile (rows h*128.., 128B-swizzled
//            K-major: 16-byte chunk c of row r at r * 128 + ((c ^ (r % 8)) << 4)), i.e. the hi (lo) halves of the two
//            canonical blocks nc = 2h, 2h + 1 stacked.  Fast precision streams only the hi stages.
//   W = 64:  one stage, the canonical block itself [hi 8 KB | lo 8 KB] (fast precision: its hi half).
// Each K-block's MMAs thus keep the canonical order of every output column: a_hi*b_hi over its four K = 16 steps, then
// a_lo*b_hi, then a_hi*b_lo, one m64nWk16 wgmma each.
#if defined(__CUDACC__)
#define NM_HD __host__ __device__ __forceinline__
#else
#define NM_HD inline
#endif
NM_HD int wide_width(const LayerProg& L) { return L.n_out > 128 ? 128 : L.n_out; }
NM_HD int wide_kblocks(const LayerProg& L) { return L.kind == KIND_LOAD ? 0 : (L.pe_src ? 1 : 0) + L.k_act / 64; }
// stages of the layer in the image (stream = 0) or streamed at the given precision (stream = 1: exact, 2: fast)
NM_HD int wide_stages(const LayerProg& L, int stream = 0) {
  const int W = wide_width(L), per = (W == 128 && stream != 2) ? 2 : 1;
  return wide_kblocks(L) * (L.n_out / W) * per;
}
// first image stage of layer li (li = n_layers: the image's stage count)
NM_HD int wide_stage_begin(const NetProgram& p, int li) {
  int s = 0;
  for (int i = 0; i < li; ++i) s += wide_stages(p.layers[i]);
  return s;
}
// distance of an element's lo copy from its hi copy
NM_HD uint32_t wide_lo_delta(const LayerProg& L) { return wide_width(L) == 128 ? (uint32_t)kStageBytes : (uint32_t)kHalfStage; }
// byte offset, from the layer's first stage, of the hi copy of element (row n, column k) of source pe (1: the encoding,
// k < 64; 0: the activations, k < k_act)
NM_HD uint32_t wide_offset(const LayerProg& L, int pe, int n, int k) {
  const int W = wide_width(L), kbi = pe ? 0 : (L.pe_src ? 1 : 0) + (k >> 6);
  const int stage = (kbi * (L.n_out / W) + n / W) * (W == 128 ? 2 : 1), r = n % W, c = k & 63;
  return (uint32_t)stage * (uint32_t)kStageBytes + (uint32_t)r * 128u + (uint32_t)((((c >> 3) ^ (r & 7)) << 4) + ((c & 7) << 1));
}
#undef NM_HD

}  // namespace nm
