// Small-component removal on an indexed triangle mesh (DESIGN §4.9; no reference counterpart).
//   1. cc_init_kernel      parent[i] = i
//   2. cc_hook_kernel      one thread per face: union(a, b), union(a, c).  Lock-free: the larger root is hooked under the
//                          smaller one with atomicCAS, retried until both ends share a root; every find halves its path
//                          (pointer jumping).  A face index outside [0, V) sets the error word (code 3); the face joins nothing.
//   3. cc_flatten_kernel   label[i] = root(i), which is the component's smallest vertex index (a separate array: the
//                          finds of other threads still halve paths in `parent` while the labels are written)
//   4. cc_size_kernel      comp_faces[label[face.v0]] += 1 (integer atomics: exact, so deterministic)
//   5. cc_vmask_kernel / cc_fmask_kernel   keep masks (size >= min_faces) and the component counts
//   6. exclusive_scan of both masks (the grid search's integer scan, nm_chamfer.cu)
//   7. cc_vscatter_kernel / cc_fscatter_kernel   stable compaction; faces re-indexed through the vertex scan
// Every array is a function of the mesh alone (labels, sizes, masks, scans): the same bits whatever order the atomics took.
#include "nm_common.h"

namespace nm {
namespace {

constexpr int kBlock = 256;
constexpr int kErrBadFace = 3;        // the mesh sampler uses codes 1 and 2 of the same word

unsigned blocks_for(long long n) { return (unsigned)((n + kBlock - 1) / kBlock); }
size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

// Invariant (DESIGN §4.9): parent[x] <= x, and parent[x] is in x's tree.  Roots are the x with parent[x] == x; only roots
// are ever hooked (atomicCAS from x), and a path write only replaces parent[x] by an ancestor of it, so a non-root never
// becomes a root again and every tree's root is its smallest member.  volatile: other threads' writes must be re-read.
__device__ __forceinline__ int cc_find(volatile int* parent, int x) {
  for (;;) {
    const int p = parent[x];
    if (p == x) return x;
    const int g = parent[p];
    if (g == p) return p;
    parent[x] = g;                    // path halving: x skips to its grandparent
    x = g;
  }
}

__device__ __forceinline__ void cc_union(volatile int* parent, int a, int b) {
  for (;;) {
    int ra = cc_find(parent, a), rb = cc_find(parent, b);
    if (ra == rb) return;
    if (ra > rb) { const int t = ra; ra = rb; rb = t; }
    const int old = atomicCAS(const_cast<int*>(parent) + rb, rb, ra);     // hook the larger root under the smaller
    if (old == rb) return;
    a = ra; b = old;                  // rb was hooked meanwhile: retry from what it now points to
  }
}

__device__ __forceinline__ bool face_ok(int a, int b, int c, long long V) {
  return a >= 0 && a < V && b >= 0 && b < V && c >= 0 && c < V;
}

__global__ void __launch_bounds__(kBlock) cc_init_kernel(int* __restrict__ parent, long long V) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i < V) parent[i] = (int)i;
}

__global__ void __launch_bounds__(kBlock) cc_hook_kernel(int* parent, long long V, const int* __restrict__ f, long long F, int* err) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= F) return;
  const int a = f[3 * i], b = f[3 * i + 1], c = f[3 * i + 2];
  if (!face_ok(a, b, c, V)) {
    *(volatile int*)err = kErrBadFace;
    return;
  }
  cc_union(parent, a, b);
  cc_union(parent, a, c);
}

__global__ void __launch_bounds__(kBlock) cc_flatten_kernel(int* parent, long long V, int* __restrict__ label) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i < V) label[i] = cc_find(parent, (int)i);
}

__global__ void __launch_bounds__(kBlock) cc_size_kernel(const int* __restrict__ label, long long V, const int* __restrict__ f,
                                                         long long F, int* __restrict__ comp_faces) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= F) return;
  const int a = f[3 * i], b = f[3 * i + 1], c = f[3 * i + 2];
  if (face_ok(a, b, c, V)) atomicAdd(comp_faces + label[a], 1);
}

// vertices [0, V]: vmask[i] = component of i kept (vmask[V] = 0, so the scan's entry V is the total); counts[0] += roots with
// >= 1 face, counts[1] += those kept.  Whole warps reach the reductions (the grid covers V + 1 entries in full blocks).
__global__ void __launch_bounds__(kBlock) cc_vmask_kernel(const int* __restrict__ label, long long V, const int* __restrict__ comp_faces,
                                                          long long min_faces, int* __restrict__ vmask, int* __restrict__ counts) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  int comp = 0, kept = 0;
  if (i < V) {
    const int r = label[i];
    const int n = comp_faces[r];
    const int keep = (long long)n >= min_faces;
    vmask[i] = keep;
    comp = r == i && n > 0;
    kept = comp & keep;
  } else if (i == V) {
    vmask[V] = 0;
  }
  comp = __reduce_add_sync(0xffffffffu, comp);
  kept = __reduce_add_sync(0xffffffffu, kept);
  if ((threadIdx.x & 31) == 0 && comp) {
    atomicAdd(counts, comp);
    atomicAdd(counts + 1, kept);
  }
}

// faces [0, F]: fmask[i] = face valid and its component kept (fmask[F] = 0)
__global__ void __launch_bounds__(kBlock) cc_fmask_kernel(const int* __restrict__ label, long long V, const int* __restrict__ f,
                                                          long long F, const int* __restrict__ comp_faces, long long min_faces,
                                                          int* __restrict__ fmask) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i > F) return;
  int keep = 0;
  if (i < F) {
    const int a = f[3 * i], b = f[3 * i + 1], c = f[3 * i + 2];
    keep = face_ok(a, b, c, V) && (long long)comp_faces[label[a]] >= min_faces;
  }
  fmask[i] = keep;
}

__global__ void __launch_bounds__(kBlock) cc_vscatter_kernel(const float* __restrict__ v, const float* __restrict__ n, long long V,
                                                             const int* __restrict__ vmask, const int* __restrict__ vstart,
                                                             float* __restrict__ v_out, float* __restrict__ n_out) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= V || !vmask[i]) return;
  const long long o = vstart[i];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    v_out[3 * o + c] = v[3 * i + c];
    n_out[3 * o + c] = n[3 * i + c];
  }
}

__global__ void __launch_bounds__(kBlock) cc_fscatter_kernel(const int* __restrict__ f, long long F, const int* __restrict__ fmask,
                                                             const int* __restrict__ fstart, const int* __restrict__ vstart,
                                                             int* __restrict__ f_out) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= F || !fmask[i]) return;       // a kept face is valid and its three vertices are kept
  const long long o = fstart[i];
#pragma unroll
  for (int c = 0; c < 3; ++c) f_out[3 * o + c] = vstart[f[3 * i + c]];
}

// Workspace (256-byte aligned pieces, ints): parent, label, comp_faces (V), vmask, vstart (V+1), fmask, fstart (F+1),
// the scan's block sums, counts (4)
struct CcWs {
  int *parent, *label, *comp_faces, *vmask, *vstart, *fmask, *fstart, *blk, *counts;
};
size_t carve(void* ws, long long V, long long F, CcWs* w) {
  const long long nblk = ((V > F ? V : F) + 1 + kScanBlockEntries - 1) / kScanBlockEntries;
  const size_t sz[9] = {(size_t)V * 4, (size_t)V * 4, (size_t)V * 4, (size_t)(V + 1) * 4, (size_t)(V + 1) * 4, (size_t)(F + 1) * 4,
                        (size_t)(F + 1) * 4, (size_t)nblk * 4, 16};
  int** dst[9] = {&w->parent, &w->label, &w->comp_faces, &w->vmask, &w->vstart, &w->fmask, &w->fstart, &w->blk, &w->counts};
  size_t tot = 0;
  for (int i = 0; i < 9; ++i) {
    if (ws) *dst[i] = reinterpret_cast<int*>(reinterpret_cast<char*>(ws) + tot);
    tot += align_up(sz[i]);
  }
  return tot;
}

}  // namespace

size_t components_ws_bytes(long long V, long long F) {
  CcWs w{};
  return carve(nullptr, V, F, &w);
}

int mesh_components(const float* verts, const float* normals, long long V, const int32_t* faces, long long F, long long min_faces,
                    float* verts_out, float* normals_out, int32_t* faces_out, int32_t* labels_out, int64_t* counts_host, void* ws,
                    int* d_err, cudaStream_t st, int64_t* launches) {
  CcWs w{};
  carve(ws, V, F, &w);
  int64_t n = 0;
  NM_CUDA(cudaMemsetAsync(w.counts, 0, 16, st));
  if (V) {
    NM_CUDA(cudaMemsetAsync(w.comp_faces, 0, (size_t)V * 4, st));
    cc_init_kernel<<<blocks_for(V), kBlock, 0, st>>>(w.parent, V);
    n += 1;
  }
  if (F) {
    cc_hook_kernel<<<blocks_for(F), kBlock, 0, st>>>(w.parent, V, faces, F, d_err);
    n += 1;
  }
  if (V) {
    cc_flatten_kernel<<<blocks_for(V), kBlock, 0, st>>>(w.parent, V, w.label);
    n += 1;
  }
  if (F) {
    cc_size_kernel<<<blocks_for(F), kBlock, 0, st>>>(w.label, V, faces, F, w.comp_faces);
    n += 1;
  }
  cc_vmask_kernel<<<blocks_for(V + 1), kBlock, 0, st>>>(w.label, V, w.comp_faces, min_faces, w.vmask, w.counts);
  cc_fmask_kernel<<<blocks_for(F + 1), kBlock, 0, st>>>(w.label, V, faces, F, w.comp_faces, min_faces, w.fmask);
  NM_CUDA(cudaGetLastError());
  if (int e = exclusive_scan(w.vmask, V + 1, w.blk, w.vstart, st)) return e;
  if (int e = exclusive_scan(w.fmask, F + 1, w.blk, w.fstart, st)) return e;
  n += 8;
  if (V) {
    cc_vscatter_kernel<<<blocks_for(V), kBlock, 0, st>>>(verts, normals, V, w.vmask, w.vstart, verts_out, normals_out);
    n += 1;
  }
  if (F) {
    cc_fscatter_kernel<<<blocks_for(F), kBlock, 0, st>>>(faces, F, w.fmask, w.fstart, w.vstart, faces_out);
    n += 1;
  }
  NM_CUDA(cudaGetLastError());
  if (labels_out && V) NM_CUDA(cudaMemcpyAsync(labels_out, w.label, (size_t)V * 4, cudaMemcpyDeviceToDevice, st));
  int tot[4];
  NM_CUDA(cudaMemcpyAsync(tot, w.vstart + V, 4, cudaMemcpyDeviceToHost, st));
  NM_CUDA(cudaMemcpyAsync(tot + 1, w.fstart + F, 4, cudaMemcpyDeviceToHost, st));
  NM_CUDA(cudaMemcpyAsync(tot + 2, w.counts, 8, cudaMemcpyDeviceToHost, st));
  NM_CUDA(cudaStreamSynchronize(st));
  for (int i = 0; i < 4; ++i) counts_host[i] = tot[i];
  if (launches) *launches += n;
  return 0;
}

}  // namespace nm
