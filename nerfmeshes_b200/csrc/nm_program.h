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
constexpr int kStageBytes = 16384;   // one weight stage: [hi 64x64 fp16 | lo 64x64 fp16], 128B-swizzled K-major
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

}  // namespace nm
