// Sparse density sweep for mesh extraction (DESIGN §4.10; no reference counterpart): sigma is evaluated only in the blocks of
// B^3 cells the iso-surface crosses, found from a coarse lattice and followed from block to block to a fixpoint.
//   lattice  sp_lattice_points_kernel   the lattice points (every B-th grid point per axis, and the last) as an explicit point
//                                       list -> fused MLP, sigma only -> sp_scatter_kernel into the volume + a compact array
//                                       (its min / max / std give the iso level)
//   run   1. sp_lattice_mark_kernel     evaluated mask := the lattice points
//         2. sp_seed_kernel             one thread per block: its 8 lattice corners' signs -> sign, active flag, new-block list
//         per round:
//         3. sp_mark_kernel             one thread per (new block, line of its box dilated by one point): OR the line's bits
//                                       into the `wanted` mask (the sign bit-volume's layout: 32-point words of a grid line)
//         4. sp_diff_count_kernel + exclusive_scan   popcount of wanted ^ evaluated per word -> the new points' positions
//         5. per chunk: sp_gather_kernel (one thread per word writes its new points' flat indices and coordinates in
//            ascending order) -> fused MLP, sigma only -> sp_scatter_kernel
//         6. sp_grow_kernel             one thread per (inactive block, line of its closed point set): a point evaluated in
//                                       this round whose sign differs from the block's activates the block
//         7. evaluated := wanted; the host reads {new blocks, new points} once per round and stops when there are none
//         8. sp_fill_kernel             one streaming pass: +inf / -inf (the block's sign) at every unevaluated point
// Every sigma is a function of its point alone and every mask, count and list position is an integer function of the
// volume: the atomics (OR into mask words, the new-block list's order) do not reach the result, so the same inputs give the
// same volume bit for bit on every run and for every chunk size.  No kernel waits for another.
#include <math_constants.h>

#include "nm_common.h"

namespace nm {
namespace {

constexpr int kBlock = 256;
constexpr int kSignInside = 1, kActive = 2;      // block state bits

unsigned blocks_for(long long n) { return (unsigned)((n + kBlock - 1) / kBlock); }
size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

struct SpGrid {
  int n[3];        // grid points per axis
  int nb[3];       // blocks per axis: ceil((n - 1) / B)
  int B, W;        // block edge in cells; 32-point words per grid line
  __host__ __device__ long long blocks() const { return (long long)nb[0] * nb[1] * nb[2]; }
  __host__ __device__ long long lattice() const { return (long long)(nb[0] + 1) * (nb[1] + 1) * (nb[2] + 1); }
  __host__ __device__ long long words() const { return (long long)n[0] * n[1] * W; }
  __host__ __device__ long long points() const { return (long long)n[0] * n[1] * n[2]; }
  // lattice index a in [0, nb] of an axis -> grid index
  __host__ __device__ int lat(int axis, int a) const { const int i = a * B; return i < n[axis] - 1 ? i : n[axis] - 1; }
};

SpGrid make_grid(const SparseSweep& s) {
  SpGrid g;
  const int n[3] = {s.n0, s.n1, s.n2};
  for (int a = 0; a < 3; ++a) { g.n[a] = n[a]; g.nb[a] = (n[a] - 1 + s.block - 1) / s.block; }
  g.B = s.block;
  g.W = (s.n2 + 31) / 32;
  return g;
}

// bits [a, b] of a word, 0 <= a <= b <= 31
__device__ __forceinline__ unsigned bit_range(int a, int b) {
  return (b - a == 31) ? 0xffffffffu : (((1u << (b - a + 1)) - 1u) << a);
}

// lattice points [p0, p0 + cnt) of the lattice's flat order -> flat grid index and coordinates (the tables' values)
__global__ void __launch_bounds__(kBlock) sp_lattice_points_kernel(SpGrid g, long long p0, long long cnt, const float* __restrict__ lin0,
                                                                   const float* __restrict__ lin1, const float* __restrict__ lin2,
                                                                   int* __restrict__ idx, float* __restrict__ pts) {
  const long long o = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (o >= cnt) return;
  const long long t = p0 + o;
  const int l2 = g.nb[2] + 1, l1 = g.nb[1] + 1;
  const int i = g.lat(0, (int)(t / ((long long)l1 * l2))), j = g.lat(1, (int)((t / l2) % l1)), k = g.lat(2, (int)(t % l2));
  idx[o] = (int)(((long long)i * g.n[1] + j) * g.n[2] + k);
  pts[3 * o] = lin0[i]; pts[3 * o + 1] = lin1[j]; pts[3 * o + 2] = lin2[k];
}

__global__ void __launch_bounds__(kBlock) sp_scatter_kernel(const int* __restrict__ idx, const float* __restrict__ sig, long long cnt,
                                                            float* __restrict__ vol) {
  const long long o = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (o < cnt) vol[idx[o]] = sig[o];
}

__global__ void __launch_bounds__(kBlock) sp_lattice_mark_kernel(SpGrid g, unsigned* evaluated) {
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (t >= g.lattice()) return;
  const int l2 = g.nb[2] + 1, l1 = g.nb[1] + 1;
  const int i = g.lat(0, (int)(t / ((long long)l1 * l2))), j = g.lat(1, (int)((t / l2) % l1)), k = g.lat(2, (int)(t % l2));
  atomicOr(evaluated + ((long long)i * g.n[1] + j) * g.W + (k >> 5), 1u << (k & 31));
}

// one thread per block: sign and active flag from the 8 lattice corners; active blocks go to the new-block list
__global__ void __launch_bounds__(kBlock) sp_seed_kernel(SpGrid g, const float* __restrict__ vol, float iso, int* __restrict__ state,
                                                         int* __restrict__ newlist, int* counters) {
  const long long b = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (b >= g.blocks()) return;
  const int b2 = (int)(b % g.nb[2]), b1 = (int)((b / g.nb[2]) % g.nb[1]), b0 = (int)(b / ((long long)g.nb[2] * g.nb[1]));
  int inside = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    const int i = g.lat(0, b0 + (c >> 2)), j = g.lat(1, b1 + ((c >> 1) & 1)), k = g.lat(2, b2 + (c & 1));
    inside += vol[((long long)i * g.n[1] + j) * g.n[2] + k] > iso ? 1 : 0;
  }
  const bool mixed = inside != 0 && inside != 8;
  state[b] = (inside == 8 ? kSignInside : 0) | (mixed ? kActive : 0);
  if (mixed) newlist[atomicAdd(counters, 1)] = (int)b;
}

// one work item per (new block, line of its closed point set dilated by one point and clipped to the grid)
__global__ void __launch_bounds__(kBlock) sp_mark_kernel(SpGrid g, const int* __restrict__ newlist, const int* __restrict__ counters,
                                                         unsigned* wanted) {
  const int side = g.B + 3;
  const long long items = (long long)counters[0] * side * side;
  for (long long it = (long long)blockIdx.x * kBlock + threadIdx.x; it < items; it += (long long)gridDim.x * kBlock) {
    const int b = newlist[it / (side * side)], l = (int)(it % (side * side));
    const int b2 = b % g.nb[2], b1 = (b / g.nb[2]) % g.nb[1], b0 = b / (g.nb[2] * g.nb[1]);
    const int lo0 = max(b0 * g.B - 1, 0), hi0 = min(g.lat(0, b0 + 1) + 1, g.n[0] - 1);
    const int lo1 = max(b1 * g.B - 1, 0), hi1 = min(g.lat(1, b1 + 1) + 1, g.n[1] - 1);
    const int lo2 = max(b2 * g.B - 1, 0), hi2 = min(g.lat(2, b2 + 1) + 1, g.n[2] - 1);
    const int i = lo0 + l / side, j = lo1 + l % side;
    if (i > hi0 || j > hi1) continue;
    unsigned* line = wanted + ((long long)i * g.n[1] + j) * g.W;
    for (int w = lo2 >> 5; w <= hi2 >> 5; ++w)
      atomicOr(line + w, bit_range(max(lo2, 32 * w) - 32 * w, min(hi2, 32 * w + 31) - 32 * w));
  }
}

// words [0, nw]: cnt[w] = points wanted and not yet evaluated (cnt[nw] = 0, so the scan's entry nw is the total)
__global__ void __launch_bounds__(kBlock) sp_diff_count_kernel(const unsigned* __restrict__ wanted, const unsigned* __restrict__ evaluated,
                                                               long long nw, int* __restrict__ cnt) {
  const long long w = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (w <= nw) cnt[w] = w < nw ? __popc(wanted[w] ^ evaluated[w]) : 0;
}

// one thread per word: its new points whose list positions fall in [p0, p0 + cap) -> flat index and coordinates, ascending
__global__ void __launch_bounds__(kBlock) sp_gather_kernel(SpGrid g, const unsigned* __restrict__ wanted, const unsigned* __restrict__ evaluated,
                                                           const int* __restrict__ start, long long p0, long long cap,
                                                           const float* __restrict__ lin0, const float* __restrict__ lin1,
                                                           const float* __restrict__ lin2, int* __restrict__ idx, float* __restrict__ pts) {
  const long long w = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (w >= g.words()) return;
  unsigned m = wanted[w] ^ evaluated[w];
  if (!m) return;
  long long pos = start[w];
  if (pos >= p0 + cap || pos + __popc(m) <= p0) return;
  const long long line = w / g.W;
  const int k0 = 32 * (int)(w % g.W), i = (int)(line / g.n[1]), j = (int)(line % g.n[1]);
  const float x = lin0[i], y = lin1[j];
  for (; m; m &= m - 1, ++pos) {
    if (pos < p0 || pos >= p0 + cap) continue;
    const int k = k0 + __ffs(m) - 1;
    const long long o = pos - p0;
    idx[o] = (int)(line * g.n[2] + k);
    pts[3 * o] = x; pts[3 * o + 1] = y; pts[3 * o + 2] = lin2[k];
  }
}

// one thread per (block, line of its closed point set): an inactive block with a point evaluated in this round (wanted ^
// evaluated) on the other side of iso than its corners becomes active
__global__ void __launch_bounds__(kBlock) sp_grow_kernel(SpGrid g, const unsigned* __restrict__ wanted, const unsigned* __restrict__ evaluated,
                                                         const float* __restrict__ vol, float iso, int* state, int* __restrict__ newlist,
                                                         int* counters) {
  const int side = g.B + 1;
  const long long it = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (it >= g.blocks() * side * side) return;
  const long long b = it / (side * side);
  const int l = (int)(it % (side * side));
  const int st = state[b];
  if (st & kActive) return;
  const int b2 = (int)(b % g.nb[2]), b1 = (int)((b / g.nb[2]) % g.nb[1]), b0 = (int)(b / ((long long)g.nb[2] * g.nb[1]));
  const int i = b0 * g.B + l / side, j = b1 * g.B + l % side;
  if (i > g.lat(0, b0 + 1) || j > g.lat(1, b1 + 1)) return;
  const int lo2 = b2 * g.B, hi2 = g.lat(2, b2 + 1);
  const long long line = (long long)i * g.n[1] + j;
  const bool inside = st & kSignInside;
  bool other = false;
  for (int w = lo2 >> 5; w <= hi2 >> 5; ++w) {
    unsigned m = (wanted[line * g.W + w] ^ evaluated[line * g.W + w]) & bit_range(max(lo2, 32 * w) - 32 * w, min(hi2, 32 * w + 31) - 32 * w);
    for (; m; m &= m - 1) other |= (vol[line * g.n[2] + 32 * w + __ffs(m) - 1] > iso) != inside;
  }
  if (other && !(atomicOr(state + b, kActive) & kActive)) newlist[atomicAdd(counters, 1)] = (int)b;
}

// unevaluated points take the sign of their (inactive) block as +inf / -inf.  VEC: n2 is a multiple of 128, one thread per 4
// points of a line (inside one word and one block: B is a multiple of 4), a 16-byte store where none of the 4 is evaluated.
template <bool VEC>
__global__ void __launch_bounds__(kBlock) sp_fill_kernel(SpGrid g, const unsigned* __restrict__ evaluated, const int* __restrict__ state,
                                                         float* __restrict__ vol) {
  constexpr int PER = VEC ? 4 : 1;
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (t * PER >= g.points()) return;
  const long long flat = t * PER, line = flat / g.n[2];
  const int k = (int)(flat % g.n[2]), i = (int)(line / g.n[1]), j = (int)(line % g.n[1]);
  const unsigned have = (evaluated[line * g.W + (k >> 5)] >> (k & 31)) & (VEC ? 0xfu : 0x1u);
  if (have == (VEC ? 0xfu : 0x1u)) return;
  const int b0 = min(i / g.B, g.nb[0] - 1), b1 = min(j / g.B, g.nb[1] - 1), b2 = min(k / g.B, g.nb[2] - 1);
  const float f = (state[((long long)b0 * g.nb[1] + b1) * g.nb[2] + b2] & kSignInside) ? CUDART_INF_F : -CUDART_INF_F;
  if (VEC && have == 0) {
    *reinterpret_cast<float4*>(vol + flat) = make_float4(f, f, f, f);
    return;
  }
#pragma unroll
  for (int c = 0; c < PER; ++c)
    if (!((have >> c) & 1)) vol[flat + c] = f;
}

// Workspace (256-byte aligned pieces): block state and new-block list (one int per block), counters (4 ints), the wanted and
// evaluated masks (one word per 32 points of a line), the per-word counts, their scan and its block sums, the compact
// lattice values, and one chunk of points: flat indices, coordinates, sigma
struct SpWs {
  int *state, *newlist, *counters;
  unsigned *wanted, *evaluated;
  int *cnt, *start, *blk, *idx;
  float *lat, *pts, *sig;
};
long long chunk_of(const SpGrid& g, long long chunk_points) { return chunk_points < g.points() ? chunk_points : g.points(); }
size_t carve(void* ws, const SpGrid& g, long long chunk_points, SpWs* w) {
  const size_t nblk = (size_t)g.blocks(), nw = (size_t)g.words(), P = (size_t)chunk_of(g, chunk_points);
  const size_t sz[12] = {nblk * 4, nblk * 4, 16, nw * 4, nw * 4, (nw + 1) * 4, (nw + 1) * 4,
                         ((nw + 1 + kScanBlockEntries - 1) / kScanBlockEntries) * 4, P * 4, (size_t)g.lattice() * 4, P * 12, P * 4};
  void** dst[12] = {(void**)&w->state, (void**)&w->newlist, (void**)&w->counters, (void**)&w->wanted, (void**)&w->evaluated,
                    (void**)&w->cnt, (void**)&w->start, (void**)&w->blk, (void**)&w->idx, (void**)&w->lat, (void**)&w->pts,
                    (void**)&w->sig};
  size_t tot = 0;
  for (int i = 0; i < 12; ++i) {
    if (ws) *dst[i] = reinterpret_cast<char*>(ws) + tot;
    tot += align_up(sz[i]);
  }
  return tot;
}

int eval_scatter(const SparseSweep& s, const SpWs& w, long long cnt, cudaStream_t st, int64_t* launches) {
  if (int e = s.eval(w.pts, cnt, w.sig)) return e;
  sp_scatter_kernel<<<blocks_for(cnt), kBlock, 0, st>>>(w.idx, w.sig, cnt, s.vol);
  NM_CUDA(cudaGetLastError());
  if (launches) *launches += 1;
  return 0;
}

}  // namespace

size_t sparse_sweep_ws_bytes(const SparseSweep& s) {
  SpWs w{};
  return carve(nullptr, make_grid(s), s.chunk_points, &w);
}

int sparse_sweep_lattice(const SparseSweep& s, void* ws, double* d_stats, float* stats_host, cudaStream_t st, int64_t* launches) {
  const SpGrid g = make_grid(s);
  SpWs w{};
  carve(ws, g, s.chunk_points, &w);
  const long long L = g.lattice(), P = chunk_of(g, s.chunk_points);
  for (long long p0 = 0; p0 < L; p0 += P) {
    const long long cnt = L - p0 < P ? L - p0 : P;
    sp_lattice_points_kernel<<<blocks_for(cnt), kBlock, 0, st>>>(g, p0, cnt, s.lin[0], s.lin[1], s.lin[2], w.idx, w.pts);
    NM_CUDA(cudaGetLastError());
    if (launches) *launches += 1;
    if (int e = eval_scatter(s, w, cnt, st, launches)) return e;
    NM_CUDA(cudaMemcpyAsync(w.lat + p0, w.sig, (size_t)cnt * 4, cudaMemcpyDeviceToDevice, st));
  }
  return launch_volume_stats(w.lat, L, d_stats, stats_host, st, launches);
}

int sparse_sweep_run(const SparseSweep& s, float iso, void* ws, int64_t* counts_host, int num_sms, cudaStream_t st, int64_t* launches) {
  const SpGrid g = make_grid(s);
  SpWs w{};
  carve(ws, g, s.chunk_points, &w);
  const long long nw = g.words(), nblk = g.blocks(), L = g.lattice(), P = chunk_of(g, s.chunk_points);
  int64_t n = 0;
  NM_CUDA(cudaMemsetAsync(w.counters, 0, 16, st));
  NM_CUDA(cudaMemsetAsync(w.evaluated, 0, (size_t)nw * 4, st));
  sp_lattice_mark_kernel<<<blocks_for(L), kBlock, 0, st>>>(g, w.evaluated);
  NM_CUDA(cudaMemcpyAsync(w.wanted, w.evaluated, (size_t)nw * 4, cudaMemcpyDeviceToDevice, st));
  sp_seed_kernel<<<blocks_for(nblk), kBlock, 0, st>>>(g, s.vol, iso, w.state, w.newlist, w.counters);
  NM_CUDA(cudaGetLastError());
  n += 2;
  long long active = 0, evaluated = L, rounds = 0;
  for (;;) {
    sp_mark_kernel<<<num_sms * 8, kBlock, 0, st>>>(g, w.newlist, w.counters, w.wanted);
    sp_diff_count_kernel<<<blocks_for(nw + 1), kBlock, 0, st>>>(w.wanted, w.evaluated, nw, w.cnt);
    NM_CUDA(cudaGetLastError());
    if (int e = exclusive_scan(w.cnt, nw + 1, w.blk, w.start, st)) return e;
    n += 5;
    int fresh[2];                    // {blocks activated by the previous step, points they add}: the one host read per round
    NM_CUDA(cudaMemcpyAsync(fresh, w.counters, 4, cudaMemcpyDeviceToHost, st));
    NM_CUDA(cudaMemcpyAsync(fresh + 1, w.start + nw, 4, cudaMemcpyDeviceToHost, st));
    NM_CUDA(cudaStreamSynchronize(st));
    if (fresh[0] == 0) break;
    active += fresh[0]; evaluated += fresh[1]; rounds += 1;
    for (long long p0 = 0; p0 < fresh[1]; p0 += P) {
      const long long cnt = fresh[1] - p0 < P ? fresh[1] - p0 : P;
      sp_gather_kernel<<<blocks_for(nw), kBlock, 0, st>>>(g, w.wanted, w.evaluated, w.start, p0, P, s.lin[0], s.lin[1], s.lin[2],
                                                          w.idx, w.pts);
      NM_CUDA(cudaGetLastError());
      n += 1;
      if (int e = eval_scatter(s, w, cnt, st, launches)) return e;
    }
    NM_CUDA(cudaMemsetAsync(w.counters, 0, 4, st));
    const int side = g.B + 1;
    sp_grow_kernel<<<blocks_for(nblk * side * side), kBlock, 0, st>>>(g, w.wanted, w.evaluated, s.vol, iso, w.state, w.newlist,
                                                                      w.counters);
    NM_CUDA(cudaGetLastError());
    n += 1;
    NM_CUDA(cudaMemcpyAsync(w.evaluated, w.wanted, (size_t)nw * 4, cudaMemcpyDeviceToDevice, st));
  }
  if ((g.n[2] & 127) == 0 && (reinterpret_cast<uintptr_t>(s.vol) & 15) == 0) sp_fill_kernel<true><<<blocks_for(g.points() / 4), kBlock, 0, st>>>(g, w.evaluated, w.state, s.vol);
  else sp_fill_kernel<false><<<blocks_for(g.points()), kBlock, 0, st>>>(g, w.evaluated, w.state, s.vol);
  NM_CUDA(cudaGetLastError());
  n += 1;
  if (launches) *launches += n;
  counts_host[0] = L; counts_host[1] = active; counts_host[2] = nblk; counts_host[3] = evaluated; counts_host[4] = rounds;
  return 0;
}

int sparse_sweep_state(const SparseSweep& s, void* ws, uint32_t* mask_out, int32_t* blocks_out, cudaStream_t st) {
  const SpGrid g = make_grid(s);
  SpWs w{};
  carve(ws, g, s.chunk_points, &w);
  if (mask_out) NM_CUDA(cudaMemcpyAsync(mask_out, w.evaluated, (size_t)g.words() * 4, cudaMemcpyDeviceToDevice, st));
  if (blocks_out) NM_CUDA(cudaMemcpyAsync(blocks_out, w.state, (size_t)g.blocks() * 4, cudaMemcpyDeviceToDevice, st));
  return 0;
}

}  // namespace nm
