// Host side of the fused MLP: turns the constructor arguments of FlexibleNeRFModel (src/nerf/models.py:5-58) into
// a layer program + tensor-core block schedule, and packs the reference's (out,in) fp32 weights into
//   (a) 16 KB tensor-core stages [hi | lo] fp16: the canonical 64x64 blocks (K-major, 128B-swizzled, in schedule order;
//       the CPU checks read them), regrouped into the wide stream (nm_program.h) that the kernel's producer warp walks
//       with cp.async.bulk, and
//   (b) transposed fp32 Wt[k][n] for the CUDA-core kernel.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "nm_common.h"

namespace nm {

static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* last_error() { return g_err; }

const float* WeightSource::find(const std::string& name, int64_t expect) const {
  for (int i = 0; i < n; ++i) {
    if (name == names[i]) {
      if (numel[i] != expect) {
        set_error("tensor '%s' has %lld elements, expected %lld", name.c_str(), (long long)numel[i], (long long)expect);
        return nullptr;
      }
      return ptrs[i];
    }
  }
  set_error("tensor '%s' missing from the state dict", name.c_str());
  return nullptr;
}

// torch.linspace(start, end, n) in fp32: step = (end-start)/(n-1); first half start+i*step, second half
// end-(n-1-i)*step (ATen RangeFactories).  Used for the PE frequency bands (src/nerf/modules.py:16-23).
static void linspace_f32(float start, float end, int n, float* out) {
  if (n == 1) { out[0] = start; return; }
  float step = (end - start) / (float)(n - 1);
  int half = n / 2;
  for (int i = 0; i < n; ++i) out[i] = (i < half) ? start + step * (float)i : end - step * (float)(n - 1 - i);
}

static void freq_bands(int L, int log_sampling, float* out) {
  if (log_sampling) {
    float e[kMaxFreq];
    linspace_f32(0.f, (float)(L - 1), L, e);
    for (int i = 0; i < L; ++i) out[i] = powf(2.0f, e[i]);
  } else {
    linspace_f32(1.0f, powf(2.0f, (float)(L - 1)), L, out);
  }
}

struct LayerNames {
  std::string w, b, head_w, head_b;
};

static bool is_skip(const NmNetDesc& d, int i) {  // src/nerf/models.py:36-42,64
  return (i % d.skip_step == 0) && i > 0 && i != d.num_layers - 1;
}

// Tensor-core block schedule of a layer list (forward or backward program): fills blocks[], blk_begin/end, the per-issuer
// bookkeeping and n_blocks from each layer's n_out / k_act / pe_src / k_pe.
static int schedule_blocks(NetProgram* p) {
  const int nl = p->n_layers;
  // tensor-core schedule: the block order within a layer (row part first, then the column part of each j) is the order of
  // the canonical block image, which regroup_wide turns into the wide stream the wgmma kernel (nm_mlp_tc.cu) reads; the
  // kernel itself reads no block.  The rest (group, first / last, the per-issuer flags / next / first_blk / none_d /
  // none_k and accumulate_only) is bookkeeping the kernel does not use; the CPU schedule tests check it.
  const int policy = 1;   // a block's "issuer" owns its accumulator chunk
  p->accumulate_only = policy == 0 ? 1 : 0;
  int nb = 0;
  for (int li = 0; li < nl; ++li) {
    LayerProg& L = p->layers[li];
    NM_CHECK(L.n_out % kChunk == 0 && L.k_act % kChunk == 0, "layer widths must be multiples of 64");
    const int KB = L.k_act / kChunk, NC = L.n_out / kChunk;
    NM_CHECK(KB <= 4 && NC <= 4, "layer wider than 256");
    L.blk_begin = nb;
    if (L.kind == KIND_LOAD) {      // no MMA blocks: every issuer has "nothing to do" on every chunk / K-block
      L.blk_end = nb; L.none_d = 0xFFFF; L.none_k = 0xFFFF; L.first_blk = -1;
      continue;
    }
    int started[4] = {0, 0, 0, 0};
    int lastblk[4] = {-1, -1, -1, -1};
    auto push = [&](int src, int kb, int nc, int ksteps, int group) {
      BlockProg& B = p->blocks[nb];
      B.src = (uint8_t)src; B.kb = (uint8_t)kb; B.nc = (uint8_t)nc; B.ksteps = (uint8_t)ksteps; B.group = (uint8_t)group;
      B.first = started[nc] ? 0 : 1; B.last = 0; B.flags = 0;
      started[nc] = 1; lastblk[nc] = nb; ++nb;
    };
    const int G = KB > NC ? KB : NC;
    for (int j = 0; j < G; ++j) {
      // row part first: blocks (j, n<j) finish accumulator chunks 0..j-1 as early as the ring allows, so their
      // epilogue (and with it the next layer) starts while the column part is still being issued
      if (j < KB)
        for (int n = 0; n < (j < NC ? j : NC); ++n) push(SRC_ACT, j, n, 4, j);
      if (j < NC) {
        if (L.pe_src) push(L.pe_src, 0, j, (L.k_pe + 15) / 16, j);
        for (int k = 0; k < (j < KB ? j : KB); ++k) push(SRC_ACT, k, j, 4, j);
        if (j < KB) push(SRC_ACT, j, j, 4, j);
      }
      NM_CHECK(nb <= kMaxBlocks, "block table overflow");
    }
    for (int n = 0; n < NC; ++n) {
      NM_CHECK(lastblk[n] >= 0, "empty accumulator chunk");
      p->blocks[lastblk[n]].last = 1;
    }
    L.blk_end = nb;
    // per-issuer bookkeeping (nm_mlp_tc.cu): which of an issuer's blocks is its last into each accumulator chunk /
    // its last reader of each activation K-block, and which chunks / K-blocks it never touches in this layer
    L.none_d = 0; L.none_k = 0;
    for (int b = L.blk_begin; b < L.blk_end; ++b) {
      const int issuer = policy == 0 ? (b & (kIssuers - 1)) : p->blocks[b].nc;
      p->blocks[b].flags = (uint8_t)(issuer << 4);
    }
    L.first_blk = -1;   // 0xFFFFFFFF
    for (int w = 0; w < kIssuers; ++w) {
      int prev = -1;
      for (int b = L.blk_begin; b < L.blk_end; ++b) {
        if ((p->blocks[b].flags >> 4) != w) continue;
        if (prev < 0) L.first_blk = (L.first_blk & ~(0xFF << (8 * w))) | ((b - L.blk_begin) << (8 * w));
        else p->blocks[prev].next = (uint8_t)(b - prev);
        p->blocks[b].next = 0;
        prev = b;
      }
    }
    for (int w = 0; w < kIssuers; ++w) {
      int ld[4] = {-1, -1, -1, -1}, lk[4] = {-1, -1, -1, -1};
      for (int b = L.blk_begin; b < L.blk_end; ++b) {
        if ((p->blocks[b].flags >> 4) != w) continue;
        ld[p->blocks[b].nc] = b;
        if (p->blocks[b].src == SRC_ACT) lk[p->blocks[b].kb] = b;
      }
      for (int i = 0; i < 4; ++i) {
        if (ld[i] >= 0) p->blocks[ld[i]].flags |= 1; else L.none_d |= 1 << (w * 4 + i);
        if (lk[i] >= 0) p->blocks[lk[i]].flags |= 2; else L.none_k |= 1 << (w * 4 + i);
      }
    }
  }
  p->n_blocks = nb;
  return 0;
}

static int build_one(const NmNetDesc& d, bool sigma_only, NetProgram* p, std::vector<LayerNames>* names) {
  memset(p, 0, sizeof(*p));
  const int h = d.hidden_size;
  NM_CHECK(h == 128 || h == 256, "hidden_size %d unsupported (128 or 256)", h);
  NM_CHECK(d.num_layers >= 1 && d.num_layers + 2 <= kMaxLayers, "num_layers %d unsupported", d.num_layers);
  NM_CHECK(d.skip_step >= 1, "skip_step must be >= 1");
  NM_CHECK(d.num_encoding_fn_xyz >= 0 && d.num_encoding_fn_xyz <= 10, "num_encoding_fn_xyz must be in [0,10]");
  NM_CHECK(d.num_encoding_fn_dir >= 0 && d.num_encoding_fn_dir <= 10, "num_encoding_fn_dir must be in [0,10]");
  p->hidden = h;
  p->L_xyz = d.num_encoding_fn_xyz;
  p->L_dir = d.num_encoding_fn_dir;
  p->inc_xyz = d.include_input_xyz ? 1 : 0;
  p->inc_dir = d.include_input_dir ? 1 : 0;
  p->dim_xyz = 6 * p->L_xyz + (p->inc_xyz ? 3 : 0);
  p->dim_dir = d.use_viewdirs ? 6 * p->L_dir + (p->inc_dir ? 3 : 0) : 0;
  NM_CHECK(p->dim_xyz >= 1 && p->dim_xyz <= 64, "xyz encoding width %d unsupported", p->dim_xyz);
  NM_CHECK(p->dim_dir <= 64 && (!d.use_viewdirs || p->dim_dir >= 1), "dir encoding width %d unsupported", p->dim_dir);
  freq_bands(p->L_xyz, d.log_sampling_xyz, p->freq_xyz);
  freq_bands(p->L_dir, d.log_sampling_dir, p->freq_dir);

  int nl = 0, bias = 0, head = 0, wt = 0;
  auto add = [&](int n_out, int k_act, int pe_src, int k_pe, int relu, const std::string& base) -> LayerProg& {
    LayerProg& L = p->layers[nl++];
    L.n_out = n_out; L.k_act = k_act; L.pe_src = pe_src; L.k_pe = k_pe; L.relu = relu; L.kind = KIND_HIDDEN;
    L.bias_off = bias; bias += n_out;
    L.wt_off = wt; wt += (k_act + k_pe) * n_out;
    names->push_back({base + ".weight", base + ".bias", "", ""});
    return L;
  };
  add(h, 0, SRC_PE_XYZ, p->dim_xyz, 0, "layer1");
  for (int i = 0; i < d.num_layers - 1; ++i) {
    bool sk = is_skip(d, i);
    add(h, h, sk ? SRC_PE_XYZ : 0, sk ? p->dim_xyz : 0, 1, "layers_xyz." + std::to_string(i));
  }
  {
    LayerProg& T = p->layers[nl - 1];
    T.head_off = head;
    if (d.use_viewdirs) {
      T.kind = KIND_SIGMA; head += h + 1;
      names->back().head_w = "fc_alpha.weight"; names->back().head_b = "fc_alpha.bias";
    } else {
      T.kind = KIND_OUT4; head += 4 * h + 4; T.is_final = 1;
      names->back().head_w = "fc_out.weight"; names->back().head_b = "fc_out.bias";
    }
  }
  if (d.use_viewdirs) {
    if (sigma_only) {
      p->layers[nl - 1].is_final = 1;
    } else {
      add(h, h, 0, 0, 1, "fc_feat");
      LayerProg& D = add(h / 2, h, SRC_PE_DIR, p->dim_dir, 1, "layers_dir.0");
      head = (head + 3) & ~3;                       // the epilogue reads head rows as float4
      D.kind = KIND_RGB; D.is_final = 1; D.head_off = head; head += 3 * (h / 2) + 3;
      names->back().head_w = "fc_rgb.weight"; names->back().head_b = "fc_rgb.bias";
    }
  }
  p->n_layers = nl; p->n_bias = bias; p->n_head = head;
  for (int i = 0; i < nl; ++i) if (p->layers[i].pe_src == SRC_PE_DIR) p->uses_dir = 1;

  return schedule_blocks(p);
}

// Data-gradient program of the training backward (nm_train.cu): layer 0 loads dZ of the last forward layer, then one
// KIND_BWD layer per forward layer l = last..1 computing dZ_{l-1} = (dZ_l W_l[:, :k_act] (+ dsigma w_alpha)) * relu'_{l-1}.
// bias_off / head_off are those of forward layer l-1: the column sums of dZ_{l-1} ARE its bias gradient, and the
// rank-1 term reads fc_alpha's row from the same head array.
int build_backward_program(const NetProgram& F, NetProgram* B) {
  memset(B, 0, sizeof(*B));
  B->hidden = F.hidden; B->n_bias = F.n_bias; B->n_head = F.n_head;
  const int last = F.n_layers - 1;
  NM_CHECK(last >= 1 && last + 1 <= kMaxLayers, "network too shallow / deep for the fused backward");
  int nl = 0;
  {
    LayerProg& L = B->layers[nl++];
    L.kind = KIND_LOAD; L.n_out = F.layers[last].n_out; L.aux = last;
  }
  for (int l = last; l >= 1; --l) {
    const LayerProg& Fl = F.layers[l];
    const LayerProg& Fp = F.layers[l - 1];
    NM_CHECK(Fl.k_act == Fp.n_out, "layer chain mismatch");
    LayerProg& L = B->layers[nl++];
    L.kind = KIND_BWD; L.n_out = Fl.k_act; L.k_act = Fl.n_out; L.relu = Fp.relu; L.is_final = (l == 1);
    L.bias_off = Fp.bias_off; L.head_off = Fp.head_off; L.wt_off = Fl.wt_off;
    L.aux = l; L.aux2 = (Fp.kind == KIND_SIGMA) ? 1 : 0;
  }
  B->n_layers = nl;
  return schedule_blocks(B);
}

int build_programs(const NmNetDesc& d, NetProgram* full, NetProgram* sigma) {
  std::vector<LayerNames> n1, n2;
  if (int e = build_one(d, false, full, &n1)) return e;
  return build_one(d, true, sigma, &n2);
}

static inline size_t swz_off(int r, int c) {  // element (row r, k c) of a 64x64 / 128x64 fp16 K-major SW128 tile
  return (size_t)r * 128 + (size_t)((((c >> 3) ^ (r & 7)) << 4) + ((c & 7) << 1));
}

static int pack_stream(const NetProgram& p, const std::vector<LayerNames>& names, const WeightSource& src,
                       std::vector<uint8_t>* out) {
  out->assign((size_t)p.n_blocks * kStageBytes, 0);
  for (int li = 0; li < p.n_layers; ++li) {
    const LayerProg& L = p.layers[li];
    const int K = L.k_act + L.k_pe;
    const float* W = src.find(names[li].w, (int64_t)L.n_out * K);
    if (!W) return -1;
    for (int b = L.blk_begin; b < L.blk_end; ++b) {
      const BlockProg& B = p.blocks[b];
      uint8_t* st = out->data() + (size_t)b * kStageBytes;
      for (int r = 0; r < kChunk; ++r) {
        const int n = B.nc * kChunk + r;
        for (int c = 0; c < kChunk; ++c) {
          int kcol;
          if (B.src == SRC_ACT) kcol = B.kb * kChunk + c;
          else kcol = (c < L.k_pe) ? L.k_act + c : -1;
          float w = (kcol >= 0) ? W[(size_t)n * K + kcol] : 0.f;
          __half hi = __float2half_rn(w);
          __half lo = __float2half_rn(w - __half2float(hi));
          memcpy(st + swz_off(r, c), &hi, 2);
          memcpy(st + kHalfStage + swz_off(r, c), &lo, 2);
        }
      }
    }
  }
  return 0;
}

// The canonical block image regrouped into the wide stream: every element of a block moves to wide_offset() of its layer.
static void regroup_wide(const NetProgram& p, const std::vector<uint8_t>& canon, std::vector<uint8_t>* wide) {
  wide->assign((size_t)wide_stage_begin(p, p.n_layers) * kStageBytes, 0);
  for (int li = 0; li < p.n_layers; ++li) {
    const LayerProg& L = p.layers[li];
    uint8_t* base = wide->data() + (size_t)wide_stage_begin(p, li) * kStageBytes;
    for (int b = L.blk_begin; b < L.blk_end; ++b) {
      const BlockProg& B = p.blocks[b];
      const int pe = B.src == SRC_ACT ? 0 : 1;
      const uint8_t* st = canon.data() + (size_t)b * kStageBytes;
      for (int r = 0; r < kChunk; ++r)
        for (int c = 0; c < kChunk; ++c) {
          const uint32_t o = wide_offset(L, pe, B.nc * kChunk + r, pe ? c : B.kb * kChunk + c);
          memcpy(base + o, st + swz_off(r, c), 2);
          memcpy(base + wide_lo_delta(L) + o, st + kHalfStage + swz_off(r, c), 2);
        }
    }
  }
}

// Host-only views of the packer for CPU tests of the schedule / swizzle logic (no CUDA calls): the canonical block image
// (wide = false) or the wide stream the kernel reads (wide = true).
int debug_pack(const NmNetDesc& d, const WeightSource& src, bool sigma_only, bool wide, NetProgram* prog, uint8_t* out,
               size_t cap, size_t* need) {
  std::vector<LayerNames> names;
  if (int e = build_one(d, sigma_only, prog, &names)) return e;
  *need = (size_t)(wide ? wide_stage_begin(*prog, prog->n_layers) : prog->n_blocks) * kStageBytes;
  if (!out) return 0;
  NM_CHECK(cap >= *need, "buffer too small");
  std::vector<uint8_t> pk, pw;
  if (int e = pack_stream(*prog, names, src, &pk)) return e;
  if (wide) regroup_wide(*prog, pk, &pw);
  memcpy(out, wide ? pw.data() : pk.data(), *need);
  return 0;
}

void free_network(NetDev* net) {
  cudaFree(net->d_full); cudaFree(net->d_sigma); cudaFree(net->d_wpack_full); cudaFree(net->d_wpack_sigma);
  cudaFree(net->d_bias); cudaFree(net->d_head); cudaFree(net->d_wt); cudaFree(net->d_w);
  cudaFree(net->d_bwd); cudaFree(net->d_wpack_bwd);
  *net = NetDev{};
}

int pack_network(const NmNetDesc& d, const WeightSource& src, NetDev* net) {
  std::vector<LayerNames> nf, ns;
  NetProgram full, sig;
  if (int e = build_one(d, false, &full, &nf)) return e;
  if (int e = build_one(d, true, &sig, &ns)) return e;
  // biases / heads / transposed weights follow the FULL program's offsets; the sigma program is a prefix of it.
  std::vector<float> bias(full.n_bias), head(full.n_head > 0 ? full.n_head : 1);
  size_t wt_total = 0;
  for (int li = 0; li < full.n_layers; ++li) wt_total += (size_t)(full.layers[li].k_act + full.layers[li].k_pe) * full.layers[li].n_out;
  std::vector<float> wt(wt_total), w_rm(wt_total);
  for (int li = 0; li < full.n_layers; ++li) {
    const LayerProg& L = full.layers[li];
    const int K = L.k_act + L.k_pe;
    const float* W = src.find(nf[li].w, (int64_t)L.n_out * K);
    const float* Bv = src.find(nf[li].b, L.n_out);
    if (!W || !Bv) return -1;
    memcpy(&bias[L.bias_off], Bv, sizeof(float) * L.n_out);
    memcpy(&w_rm[L.wt_off], W, sizeof(float) * (size_t)L.n_out * K);
    for (int k = 0; k < K; ++k)
      for (int n = 0; n < L.n_out; ++n) wt[L.wt_off + (size_t)k * L.n_out + n] = W[(size_t)n * K + k];
    if (!nf[li].head_w.empty()) {
      const int rows = L.kind == KIND_SIGMA ? 1 : (L.kind == KIND_RGB ? 3 : 4);
      const float* HW = src.find(nf[li].head_w, (int64_t)rows * L.n_out);
      const float* HB = src.find(nf[li].head_b, rows);
      if (!HW || !HB) return -1;
      memcpy(&head[L.head_off], HW, sizeof(float) * rows * L.n_out);
      memcpy(&head[L.head_off + rows * L.n_out], HB, sizeof(float) * rows);
    }
  }
  std::vector<uint8_t> pk_full, pk_sig, canon;
  if (int e = pack_stream(full, nf, src, &canon)) return e;
  regroup_wide(full, canon, &pk_full);
  if (int e = pack_stream(sig, ns, src, &canon)) return e;
  regroup_wide(sig, canon, &pk_sig);

  free_network(net);
  net->desc = d; net->full = full; net->sigma = sig;
  net->n_wt = wt.size();
  for (const LayerNames& n : nf) { net->names.push_back(n.w); net->names.push_back(n.b); net->names.push_back(n.head_w); net->names.push_back(n.head_b); }
  NM_CUDA(cudaMalloc(&net->d_full, sizeof(NetProgram)));
  NM_CUDA(cudaMalloc(&net->d_sigma, sizeof(NetProgram)));
  NM_CUDA(cudaMalloc(&net->d_wpack_full, pk_full.size()));
  NM_CUDA(cudaMalloc(&net->d_wpack_sigma, pk_sig.size()));
  NM_CUDA(cudaMalloc(&net->d_bias, bias.size() * sizeof(float)));
  NM_CUDA(cudaMalloc(&net->d_head, head.size() * sizeof(float)));
  NM_CUDA(cudaMalloc(&net->d_wt, wt.size() * sizeof(float)));
  NM_CUDA(cudaMalloc(&net->d_w, wt.size() * sizeof(float)));
  NM_CUDA(cudaMemcpy(net->d_w, w_rm.data(), wt.size() * sizeof(float), cudaMemcpyHostToDevice));
  NM_CUDA(cudaMemcpy(net->d_full, &full, sizeof(NetProgram), cudaMemcpyHostToDevice));
  NM_CUDA(cudaMemcpy(net->d_sigma, &sig, sizeof(NetProgram), cudaMemcpyHostToDevice));
  NM_CUDA(cudaMemcpy(net->d_wpack_full, pk_full.data(), pk_full.size(), cudaMemcpyHostToDevice));
  NM_CUDA(cudaMemcpy(net->d_wpack_sigma, pk_sig.data(), pk_sig.size(), cudaMemcpyHostToDevice));
  NM_CUDA(cudaMemcpy(net->d_bias, bias.data(), bias.size() * sizeof(float), cudaMemcpyHostToDevice));
  NM_CUDA(cudaMemcpy(net->d_head, head.data(), head.size() * sizeof(float), cudaMemcpyHostToDevice));
  NM_CUDA(cudaMemcpy(net->d_wt, wt.data(), wt.size() * sizeof(float), cudaMemcpyHostToDevice));
  net->loaded = true;
  return 0;
}

// ------------------------------------------------------------------------------------------------ device-side load
// The same packing with the state dict already in device memory (training: the optimiser updates CUDA parameters
// every step, so the host round trip of pack_network would dominate the step).
namespace {

__global__ void transpose_in_kernel(const float* __restrict__ W, int N, int K, float* __restrict__ Wt) {  // (N,K) -> (K,N)
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * K) return;
  const int k = i / N, n = i % N;
  Wt[i] = W[(size_t)n * K + k];
}

// Element e (of 8192) of stage `blockIdx.x` of the wide stream: its layer *li, source *pe, (row *n, column *k) of that
// source and copy *lo (0: hi, 1: lo); every element of the stage (padding included) is visited once, and wide_offset()
// (+ wide_lo_delta() for a lo copy) of the result is where it goes.
__device__ __forceinline__ void wide_element(const NetProgram& P, int e, int* li, int* pe, int* n, int* k, int* lo) {
  int l = 0, s0 = 0;
  while (l + 1 < P.n_layers && (int)blockIdx.x >= s0 + wide_stages(P.layers[l])) s0 += wide_stages(P.layers[l++]);
  const LayerProg& L = P.layers[l];
  const int s = (int)blockIdx.x - s0, W = wide_width(L);
  int kbi;
  if (W == 128) {                       // stage = (K-block * halves + half) * 2 + lo, 128 rows x 64 columns
    kbi = (s >> 1) / (L.n_out / W);
    *n = ((s >> 1) % (L.n_out / W)) * W + (e >> 6);
    *lo = s & 1;
  } else {                              // stage = K-block, [hi | lo] of 64 rows x 64 columns
    kbi = s;
    *n = (e & 4095) >> 6;
    *lo = e >> 12;
  }
  *li = l;
  *pe = (L.pe_src && kbi == 0) ? 1 : 0;
  *k = (*pe ? 0 : (kbi - (L.pe_src ? 1 : 0)) * 64) + (e & 63);
}

__device__ __forceinline__ uint32_t wide_stage_base(const NetProgram& P, int li) { return (uint32_t)wide_stage_begin(P, li) * kStageBytes; }

// one CTA per 16 KB stage of the wide stream (pack_stream + regroup_wide above, on the device)
__global__ void __launch_bounds__(256) pack_stream_kernel(const NetProgram* __restrict__ prog, const float* __restrict__ w_rm,
                                                          uint8_t* __restrict__ out) {
  const NetProgram& P = *prog;
  for (int e = threadIdx.x; e < kStageBytes / 2; e += blockDim.x) {
    int li, pe, n, k, lo;
    wide_element(P, e, &li, &pe, &n, &k, &lo);
    const LayerProg& L = P.layers[li];
    const int K = L.k_act + L.k_pe;
    const float w = (!pe || k < L.k_pe) ? w_rm[L.wt_off + (size_t)n * K + (pe ? L.k_act + k : k)] : 0.f;
    const __half hi = __float2half_rn(w);
    *reinterpret_cast<__half*>(out + wide_stage_base(P, li) + wide_offset(L, pe, n, k) + (lo ? wide_lo_delta(L) : 0u)) =
        lo ? __float2half_rn(w - __half2float(hi)) : hi;
  }
}

// wide stream of the backward program: layer L's element (n', k') is W^T[n'][k'] — row n' an input feature of forward
// layer L.aux, column k' one of its output features — read from the transposed fp32 weights (ld = the forward layer's
// n_out); bf16 hi/lo split (gradients span fp32's exponent range)
__global__ void __launch_bounds__(256) pack_bwd_stream_kernel(const NetProgram* __restrict__ prog, const float* __restrict__ wt,
                                                              uint8_t* __restrict__ out) {
  const NetProgram& P = *prog;
  for (int e = threadIdx.x; e < kStageBytes / 2; e += blockDim.x) {
    int li, pe, n, k, lo;
    wide_element(P, e, &li, &pe, &n, &k, &lo);
    const LayerProg& L = P.layers[li];
    const float w = wt[L.wt_off + (size_t)n * L.k_act + k];
    const __nv_bfloat16 hi = __float2bfloat16_rn(w);
    *reinterpret_cast<__nv_bfloat16*>(out + wide_stage_base(P, li) + wide_offset(L, pe, n, k) + (lo ? wide_lo_delta(L) : 0u)) =
        lo ? __float2bfloat16_rn(w - __bfloat162float(hi)) : hi;
  }
}

}  // namespace

// (re)build the backward program and its weight stream from the current transposed weights (device, stream-ordered)
int build_backward_stream(NetDev* net, cudaStream_t st, int64_t* launches) {
  if (!net->d_bwd) {
    if (int e = build_backward_program(net->full, &net->bwd)) return e;
    NM_CUDA(cudaMalloc(&net->d_bwd, sizeof(NetProgram)));
    NM_CUDA(cudaMemcpyAsync(net->d_bwd, &net->bwd, sizeof(NetProgram), cudaMemcpyHostToDevice, st));
    NM_CUDA(cudaMalloc(&net->d_wpack_bwd, (size_t)wide_stage_begin(net->bwd, net->bwd.n_layers) * kStageBytes));
  }
  pack_bwd_stream_kernel<<<wide_stage_begin(net->bwd, net->bwd.n_layers), 256, 0, st>>>(net->d_bwd, net->d_wt, net->d_wpack_bwd);
  NM_CUDA(cudaGetLastError());
  if (launches) ++*launches;
  net->bwd_valid = true;
  return 0;
}

int load_network_dev(const NmNetDesc& d, const WeightSource& src, NetDev* net, cudaStream_t st, int64_t* launches) {
  std::vector<LayerNames> nf, ns;
  NetProgram full, sig;
  if (int e = build_one(d, false, &full, &nf)) return e;
  if (int e = build_one(d, true, &sig, &ns)) return e;
  size_t wt_total = 0;
  for (int li = 0; li < full.n_layers; ++li) wt_total += (size_t)(full.layers[li].k_act + full.layers[li].k_pe) * full.layers[li].n_out;
  const bool same = net->loaded && memcmp(&net->desc, &d, sizeof(d)) == 0 && net->n_wt == wt_total;
  if (!same) {
    free_network(net);
    net->desc = d; net->full = full; net->sigma = sig; net->n_wt = wt_total;
    for (const LayerNames& n : nf) { net->names.push_back(n.w); net->names.push_back(n.b); net->names.push_back(n.head_w); net->names.push_back(n.head_b); }
    NM_CUDA(cudaMalloc(&net->d_full, sizeof(NetProgram)));
    NM_CUDA(cudaMalloc(&net->d_sigma, sizeof(NetProgram)));
    NM_CUDA(cudaMalloc(&net->d_wpack_full, (size_t)wide_stage_begin(full, full.n_layers) * kStageBytes));
    NM_CUDA(cudaMalloc(&net->d_wpack_sigma, (size_t)wide_stage_begin(sig, sig.n_layers) * kStageBytes));
    NM_CUDA(cudaMalloc(&net->d_bias, (size_t)full.n_bias * sizeof(float)));
    NM_CUDA(cudaMalloc(&net->d_head, (size_t)(full.n_head > 0 ? full.n_head : 1) * sizeof(float)));
    NM_CUDA(cudaMalloc(&net->d_wt, wt_total * sizeof(float)));
    NM_CUDA(cudaMalloc(&net->d_w, wt_total * sizeof(float)));
    NM_CUDA(cudaMemcpy(net->d_full, &full, sizeof(NetProgram), cudaMemcpyHostToDevice));
    NM_CUDA(cudaMemcpy(net->d_sigma, &sig, sizeof(NetProgram), cudaMemcpyHostToDevice));
    NM_CUDA(cudaMemset(net->d_head, 0, (size_t)(full.n_head > 0 ? full.n_head : 1) * sizeof(float)));
  }
  for (int li = 0; li < full.n_layers; ++li) {
    const LayerProg& L = full.layers[li];
    const int K = L.k_act + L.k_pe, N = L.n_out;
    const float* W = src.find(nf[li].w, (int64_t)N * K);
    const float* Bv = src.find(nf[li].b, N);
    if (!W || !Bv) return -1;
    NM_CUDA(cudaMemcpyAsync(net->d_w + L.wt_off, W, sizeof(float) * (size_t)N * K, cudaMemcpyDeviceToDevice, st));
    NM_CUDA(cudaMemcpyAsync(net->d_bias + L.bias_off, Bv, sizeof(float) * N, cudaMemcpyDeviceToDevice, st));
    transpose_in_kernel<<<(N * K + 255) / 256, 256, 0, st>>>(W, N, K, net->d_wt + L.wt_off);
    NM_CUDA(cudaGetLastError());
    if (launches) ++*launches;
    if (!nf[li].head_w.empty()) {
      const int rows = L.kind == KIND_SIGMA ? 1 : (L.kind == KIND_RGB ? 3 : 4);
      const float* HW = src.find(nf[li].head_w, (int64_t)rows * N);
      const float* HB = src.find(nf[li].head_b, rows);
      if (!HW || !HB) return -1;
      NM_CUDA(cudaMemcpyAsync(net->d_head + L.head_off, HW, sizeof(float) * rows * N, cudaMemcpyDeviceToDevice, st));
      NM_CUDA(cudaMemcpyAsync(net->d_head + L.head_off + rows * N, HB, sizeof(float) * rows, cudaMemcpyDeviceToDevice, st));
    }
  }
  pack_stream_kernel<<<wide_stage_begin(full, full.n_layers), 256, 0, st>>>(net->d_full, net->d_w, net->d_wpack_full);
  NM_CUDA(cudaGetLastError());
  pack_stream_kernel<<<wide_stage_begin(sig, sig.n_layers), 256, 0, st>>>(net->d_sigma, net->d_w, net->d_wpack_sigma);
  NM_CUDA(cudaGetLastError());
  if (launches) *launches += 2;
  net->bwd_valid = false;
  net->loaded = true;
  return 0;
}

}  // namespace nm
