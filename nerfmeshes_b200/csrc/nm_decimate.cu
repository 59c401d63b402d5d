// Quadric-error mesh decimation (DESIGN §4.11; no reference counterpart).  Garland–Heckbert quadrics in double, collapses
// chosen as an independent set per round, so every round's collapses commute and the result is a function of the mesh alone.
//   once   dc_validate_kernel   a face index outside [0, V) sets the error word (code 4): the call then copies its input
//          dc_compact_kernel / exclusive_scan / dc_fill_kernel / dc_sort_kernel   vertex -> face lists (CSR, ascending faces)
//          dc_lock_kernel       vertices never moved or removed (open / non-manifold edges, repeated indices, > kValenceCap faces)
//          dc_quadric_kernel    Q_v = sum of the area-weighted face quadrics, in ascending face index
//   round  dc_count_kernel / exclusive_scan / dc_edges_kernel   candidate edges (a, b), a < b, both unlocked, numbered per a
//          dc_eval_kernel       position, cost, legality (link condition, valence, no fold-over), key; m[v] = min key (atomicMin)
//          dc_select_kernel     edges whose key is the minimum over the closed 1-rings of both ends; host reads the count
//          dc_hist_kernel / dc_pick_kernel / dc_trim_kernel   (the round that would cross T) radix select of the smallest keys
//          dc_apply_kernel      b -> a, a's position and quadric, the edge's two faces die
//          exclusive_scan + dc_compact_kernel + CSR rebuild   stable face compaction
//   end    exclusive_scan + dc_vout_kernel / dc_fout_kernel   surviving vertices in input order, normals, faces re-indexed
// Built with -fmad=false: every floating-point operation below is one IEEE double (or float) operation in the order written,
// which tests/_decimate_ref.py restates bit for bit.  Everything else is integer.
#include "nm_common.h"

namespace nm {
namespace {

constexpr int kBlock = 256;
constexpr int kErrBadFace = 4;            // the mesh sampler uses codes 1 and 2, the component filter 3, of the same word
constexpr int kValenceCap = 32;           // an unlocked vertex has at most this many faces, before and after every collapse
constexpr double kDetMin = 1e-12;         // |det| of the quadric's 3x3 block below which its minimiser is not a candidate
constexpr unsigned long long kNoKey = ~0ull;

unsigned blocks_for(long long n) { return (unsigned)((n + kBlock - 1) / kBlock); }
size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

__device__ __forceinline__ bool face_ok(int a, int b, int c, long long V) {
  return a >= 0 && a < V && b >= 0 && b < V && c >= 0 && c < V;
}

__device__ __forceinline__ double3 ldp(const float* p, int v) {
  return make_double3((double)p[3 * v], (double)p[3 * v + 1], (double)p[3 * v + 2]);
}

// (p1 - p0) x (p2 - p0), twice the face's area vector
__device__ __forceinline__ double3 face_cross(double3 p0, double3 p1, double3 p2) {
  const double e1x = p1.x - p0.x, e1y = p1.y - p0.y, e1z = p1.z - p0.z;
  const double e2x = p2.x - p0.x, e2y = p2.y - p0.y, e2z = p2.z - p0.z;
  return make_double3(e1y * e2z - e1z * e2y, e1z * e2x - e1x * e2z, e1x * e2y - e1y * e2x);
}

__device__ __forceinline__ double dot3(double3 a, double3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }

// x^T Q x for x = (p, 1), Q's 10 unique entries row-major over the upper triangle, clamped at 0
__device__ __forceinline__ double qcost(const double* q, double3 p) {
  const double r0 = ((q[0] * p.x + q[1] * p.y) + q[2] * p.z) + q[3];
  const double r1 = ((q[1] * p.x + q[4] * p.y) + q[5] * p.z) + q[6];
  const double r2 = ((q[2] * p.x + q[5] * p.y) + q[7] * p.z) + q[8];
  const double r3 = ((q[3] * p.x + q[6] * p.y) + q[8] * p.z) + q[9];
  const double c = ((r0 * p.x + r1 * p.y) + r2 * p.z) + r3;
  return c > 0.0 ? c : 0.0;
}

__device__ __forceinline__ bool has(const int* t, int v) { return t[0] == v || t[1] == v || t[2] == v; }

// ------------------------------------------------------------------------------------------------------ mesh structure
__global__ void __launch_bounds__(kBlock) dc_validate_kernel(const int* __restrict__ f, long long F, long long V, int* nbad,
                                                             int* err) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= F) return;
  if (!face_ok(f[3 * i], f[3 * i + 1], f[3 * i + 2], V)) {
    atomicAdd(nbad, 1);
    *(volatile int*)err = kErrBadFace;
  }
}

// faces [0, F) of src that are not dead (dead == nullptr: all) to dst at i - dscan[i], counting every corner into deg
__global__ void __launch_bounds__(kBlock) dc_compact_kernel(const int* __restrict__ src, long long F, const int* __restrict__ dead,
                                                            const int* __restrict__ dscan, int* __restrict__ dst, int* deg) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= F || (dead && dead[i])) return;
  const long long o = dead ? i - dscan[i] : i;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int v = src[3 * i + c];
    dst[3 * o + c] = v;
    atomicAdd(deg + v, 1);
  }
}

__global__ void __launch_bounds__(kBlock) dc_fill_kernel(const int* __restrict__ fw, long long F, const int* __restrict__ vstart,
                                                         int* cursor, int* __restrict__ flist) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= F) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int v = fw[3 * i + c];
    flist[vstart[v] + atomicAdd(cursor + v, 1)] = (int)i;
  }
}

// the atomics above fill each list in any order: sorting makes it a function of the faces
__global__ void __launch_bounds__(kBlock) dc_sort_kernel(const int* __restrict__ vstart, long long V, int* __restrict__ flist) {
  const long long v = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (v >= V) return;
  const int k0 = vstart[v], k1 = vstart[v + 1];
  for (int k = k0 + 1; k < k1; ++k) {
    const int x = flist[k];
    int j = k - 1;
    while (j >= k0 && flist[j] > x) { flist[j + 1] = flist[j]; --j; }
    flist[j + 1] = x;
  }
}

// locked: more than kValenceCap faces, a face with a repeated index, or an edge with other than exactly two faces
__global__ void __launch_bounds__(kBlock) dc_lock_kernel(const int* __restrict__ fw, const int* __restrict__ vstart,
                                                         const int* __restrict__ flist, long long V, int* __restrict__ lock) {
  const long long v = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (v >= V) return;
  const int k0 = vstart[v], k1 = vstart[v + 1];
  int locked = k1 - k0 > kValenceCap;
  for (int k = k0; k < k1 && !locked; ++k) {
    const int* t = fw + 3 * flist[k];
    if (t[0] == t[1] || t[1] == t[2] || t[0] == t[2]) { locked = 1; break; }
    for (int c = 0; c < 3 && !locked; ++c) {
      const int w = t[c];
      if (w == v) continue;
      int n = 0;                                     // faces of v that contain w: the faces of edge (v, w)
      for (int k2 = k0; k2 < k1; ++k2) n += has(fw + 3 * flist[k2], w);
      locked = n != 2;
    }
  }
  lock[v] = locked;
}

// Q_f = area [n n^T, n d; d d^2] of each face with non-zero area, summed per vertex in ascending face index
__global__ void __launch_bounds__(kBlock) dc_quadric_kernel(const float* __restrict__ pos, const int* __restrict__ fw,
                                                            const int* __restrict__ vstart, const int* __restrict__ flist,
                                                            long long V, double* __restrict__ Q) {
  const long long v = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (v >= V) return;
  double q[10];
#pragma unroll
  for (int j = 0; j < 10; ++j) q[j] = 0.0;
  for (int k = vstart[v]; k < vstart[v + 1]; ++k) {
    const int* t = fw + 3 * flist[k];
    const double3 p0 = ldp(pos, t[0]);
    const double3 c = face_cross(p0, ldp(pos, t[1]), ldp(pos, t[2]));
    const double len = sqrt(dot3(c, c));
    if (!(len > 0.0)) continue;
    const double nx = c.x / len, ny = c.y / len, nz = c.z / len;
    const double d = -((nx * p0.x + ny * p0.y) + nz * p0.z);
    const double area = 0.5 * len;
    q[0] += area * (nx * nx); q[1] += area * (nx * ny); q[2] += area * (nx * nz); q[3] += area * (nx * d);
    q[4] += area * (ny * ny); q[5] += area * (ny * nz); q[6] += area * (ny * d);
    q[7] += area * (nz * nz); q[8] += area * (nz * d);
    q[9] += area * (d * d);
  }
#pragma unroll
  for (int j = 0; j < 10; ++j) Q[10 * v + j] = q[j];
}

// ------------------------------------------------------------------------------------------------------ one round
// Every neighbour w of an unlocked vertex a appears exactly twice among the other corners of a's faces (the two faces of
// edge (a, w)), so counts over those corners are twice the neighbour counts.
// ecnt[a] = candidate edges (a, b): b > a, both unlocked.  Entries [0, V]; ecnt[V] = 0 so that the scan's entry V is E.
__global__ void __launch_bounds__(kBlock) dc_count_kernel(const int* __restrict__ fw, const int* __restrict__ vstart,
                                                          const int* __restrict__ flist, const int* __restrict__ lock, long long V,
                                                          int* __restrict__ ecnt) {
  const long long a = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (a > V) return;
  int n = 0;
  if (a < V && !lock[a]) {
    for (int k = vstart[a]; k < vstart[a + 1]; ++k) {
      const int* t = fw + 3 * flist[k];
#pragma unroll
      for (int c = 0; c < 3; ++c) n += t[c] > a && !lock[t[c]];
    }
  }
  ecnt[a] = n / 2;
}

// edge id of (a, b) = estart[a] + the number of a's candidate neighbours in (a, b)
__global__ void __launch_bounds__(kBlock) dc_edges_kernel(const int* __restrict__ fw, const int* __restrict__ vstart,
                                                          const int* __restrict__ flist, const int* __restrict__ lock, long long V,
                                                          const int* __restrict__ estart, int* __restrict__ ea, int* __restrict__ eb) {
  const long long a = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (a >= V || lock[a]) return;
  const int k0 = vstart[a], k1 = vstart[a + 1];
  for (int k = k0; k < k1; ++k) {
    const int* t = fw + 3 * flist[k];
    for (int c = 0; c < 3; ++c) {
      const int b = t[c];
      if (b <= a || lock[b]) continue;
      int r = 0;
      for (int k2 = k0; k2 < k1; ++k2) {
        const int* u = fw + 3 * flist[k2];
#pragma unroll
        for (int c2 = 0; c2 < 3; ++c2) r += u[c2] > a && u[c2] < b && !lock[u[c2]];
      }
      ea[estart[a] + r / 2] = (int)a;            // written once per face of the edge, the same values
      eb[estart[a] + r / 2] = b;
    }
  }
}

// every face of v that does not contain `other` keeps n_old . n_new > 0 with v moved to p
__device__ bool no_fold(const float* pos, const int* fw, const int* vstart, const int* flist, int v, int other, double3 p) {
  for (int k = vstart[v]; k < vstart[v + 1]; ++k) {
    const int* t = fw + 3 * flist[k];
    if (has(t, other)) continue;
    double3 c[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) c[j] = ldp(pos, t[j]);
    const double3 n_old = face_cross(c[0], c[1], c[2]);
#pragma unroll
    for (int j = 0; j < 3; ++j)
      if (t[j] == v) c[j] = p;
    const double3 n_new = face_cross(c[0], c[1], c[2]);
    if (!(dot3(n_old, n_new) > 0.0)) return false;
  }
  return true;
}

__global__ void __launch_bounds__(kBlock) dc_eval_kernel(const float* __restrict__ pos, const double* __restrict__ Q,
                                                         const int* __restrict__ fw, const int* __restrict__ vstart,
                                                         const int* __restrict__ flist, const int* __restrict__ n_edges,
                                                         const int* __restrict__ ea, const int* __restrict__ eb,
                                                         unsigned long long* __restrict__ key, float* __restrict__ newpos,
                                                         unsigned long long* m) {
  const long long e = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (e >= *n_edges) return;
  const int a = ea[e], b = eb[e];
  const int ka0 = vstart[a], ka1 = vstart[a + 1], kb0 = vstart[b], kb1 = vstart[b + 1];
  // the opposite vertices c, d of the edge's two faces
  int c = -1, d = -1;
  for (int k = ka0; k < ka1; ++k) {
    const int* t = fw + 3 * flist[k];
    if (!has(t, b)) continue;
    const int o = (int)((long long)t[0] + t[1] + t[2] - a - b);
    if (c < 0) c = o; else d = o;
  }
  bool legal = c != d && (ka1 - ka0) + (kb1 - kb0) - 4 <= kValenceCap;
  // link condition: the common neighbours of a and b are c and d only (each counted twice over a's corners)
  if (legal) {
    int common = 0;
    for (int k = ka0; k < ka1; ++k) {
      const int* t = fw + 3 * flist[k];
      for (int j = 0; j < 3; ++j) {
        const int w = t[j];
        if (w == a || w == b) continue;
        bool in_b = false;
        for (int k2 = kb0; k2 < kb1 && !in_b; ++k2) in_b = has(fw + 3 * flist[k2], w);
        common += in_b;
      }
    }
    legal = common == 4;
  }
  // position: the cheapest of a, b, the midpoint and (if well-conditioned and within one cell of the midpoint) Q's minimiser
  double q[10];
#pragma unroll
  for (int j = 0; j < 10; ++j) q[j] = Q[10 * a + j] + Q[10 * b + j];
  const double3 pa = ldp(pos, a), pb = ldp(pos, b);
  const double3 mid = make_double3((pa.x + pb.x) * 0.5, (pa.y + pb.y) * 0.5, (pa.z + pb.z) * 0.5);
  double3 best = pa;
  double cost = qcost(q, pa);
  double cc = qcost(q, pb);
  if (cc < cost) { cost = cc; best = pb; }
  cc = qcost(q, mid);
  if (cc < cost) { cost = cc; best = mid; }
  const double c00 = q[4] * q[7] - q[5] * q[5], c01 = q[2] * q[5] - q[1] * q[7], c02 = q[1] * q[5] - q[2] * q[4];
  const double c11 = q[0] * q[7] - q[2] * q[2], c12 = q[1] * q[2] - q[0] * q[5], c22 = q[0] * q[4] - q[1] * q[1];
  const double det = (q[0] * c00 + q[1] * c01) + q[2] * c02;
  if (fabs(det) > kDetMin) {
    const double r0 = -q[3], r1 = -q[6], r2 = -q[8];
    const double3 s = make_double3(((c00 * r0 + c01 * r1) + c02 * r2) / det, ((c01 * r0 + c11 * r1) + c12 * r2) / det,
                                   ((c02 * r0 + c12 * r1) + c22 * r2) / det);
    if (fabs(s.x - mid.x) <= 1.0 && fabs(s.y - mid.y) <= 1.0 && fabs(s.z - mid.z) <= 1.0) {
      cc = qcost(q, s);
      if (cc < cost) { cost = cc; best = s; }
    }
  }
  const float px = (float)best.x, py = (float)best.y, pz = (float)best.z;
  const double3 p = make_double3((double)px, (double)py, (double)pz);
  if (legal) legal = no_fold(pos, fw, vstart, flist, a, b, p) && no_fold(pos, fw, vstart, flist, b, a, p);
  newpos[3 * e] = px; newpos[3 * e + 1] = py; newpos[3 * e + 2] = pz;
  const unsigned long long k = legal ? ((unsigned long long)__float_as_uint((float)cost) << 32) | (unsigned long long)e : kNoKey;
  key[e] = k;
  if (legal) {
    atomicMin(m + a, k);
    atomicMin(m + b, k);
  }
}

// selected iff the key is the minimum of m over the closed 1-rings of a and b
__global__ void __launch_bounds__(kBlock) dc_select_kernel(const int* __restrict__ fw, const int* __restrict__ vstart,
                                                           const int* __restrict__ flist, const int* __restrict__ n_edges,
                                                           const int* __restrict__ ea, const int* __restrict__ eb,
                                                           const unsigned long long* __restrict__ key,
                                                           const unsigned long long* __restrict__ m, int* __restrict__ sel,
                                                           int* n_sel) {
  const long long e = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (e >= *n_edges) return;
  const unsigned long long k = key[e];
  int s = 0;
  if (k != kNoKey) {
    unsigned long long mn = k;
    const int ends[2] = {ea[e], eb[e]};
    for (int i = 0; i < 2; ++i)
      for (int j = vstart[ends[i]]; j < vstart[ends[i] + 1]; ++j) {
        const int* t = fw + 3 * flist[j];
#pragma unroll
        for (int c = 0; c < 3; ++c) mn = min(mn, m[t[c]]);
      }
    s = mn == k;
  }
  sel[e] = s;
  if (s) atomicAdd(n_sel, 1);
}

// radix select of the `need` smallest selected keys, one byte per pass from the top: state = {prefix, rank left}
struct SelectState {
  unsigned long long prefix;
  long long rank;
};

__global__ void __launch_bounds__(kBlock) dc_hist_kernel(const int* __restrict__ n_edges, const unsigned long long* __restrict__ key,
                                                         const int* __restrict__ sel, int pass, const SelectState* st, int* hist) {
  const long long e = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (e >= *n_edges || !sel[e]) return;
  const unsigned long long k = key[e];
  if (pass > 0 && (k >> (64 - 8 * pass)) != st->prefix) return;
  atomicAdd(hist + ((k >> (56 - 8 * pass)) & 255), 1);
}

__global__ void dc_pick_kernel(int* hist, SelectState* st) {
  long long r = st->rank;
  int bin = 0;
  for (; bin < 255 && r > hist[bin]; ++bin) r -= hist[bin];
  st->prefix = (st->prefix << 8) | (unsigned long long)bin;
  st->rank = r;
  for (int i = 0; i < 256; ++i) hist[i] = 0;
}

__global__ void __launch_bounds__(kBlock) dc_trim_kernel(const int* __restrict__ n_edges, const unsigned long long* __restrict__ key,
                                                         const SelectState* st, int* __restrict__ sel) {
  const long long e = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (e >= *n_edges || !sel[e]) return;
  sel[e] = key[e] <= st->prefix;
}

// the selected edges' closed neighbourhoods are disjoint: no two collapses touch the same vertex, face or quadric
__global__ void __launch_bounds__(kBlock) dc_apply_kernel(const int* __restrict__ n_edges, const int* __restrict__ ea,
                                                          const int* __restrict__ eb, const int* __restrict__ sel,
                                                          const float* __restrict__ newpos, const int* __restrict__ vstart,
                                                          const int* __restrict__ flist, float* pos, double* Q, int* fw,
                                                          int* __restrict__ dead, int* __restrict__ removed) {
  const long long e = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (e >= *n_edges || !sel[e]) return;
  const int a = ea[e], b = eb[e];
#pragma unroll
  for (int c = 0; c < 3; ++c) pos[3 * a + c] = newpos[3 * e + c];
#pragma unroll
  for (int j = 0; j < 10; ++j) Q[10 * a + j] = Q[10 * a + j] + Q[10 * b + j];
  removed[b] = 1;
  for (int k = vstart[b]; k < vstart[b + 1]; ++k) {
    const int f = flist[k];
    int* t = fw + 3 * f;
    if (has(t, a)) {
      dead[f] = 1;
    } else {
#pragma unroll
      for (int c = 0; c < 3; ++c)
        if (t[c] == b) t[c] = a;
    }
  }
}

// ------------------------------------------------------------------------------------------------------ output
// surviving vertex v -> row v - rscan[v]: its position; its input normal if the position kept its bits, else the normalised
// sum of its faces' (p1 - p0) x (p2 - p0) in ascending face index (the input normal if that sum is zero)
__global__ void __launch_bounds__(kBlock) dc_vout_kernel(const float* __restrict__ pos, const float* __restrict__ v_in,
                                                         const float* __restrict__ n_in, long long V, const int* __restrict__ removed,
                                                         const int* __restrict__ rscan, const int* __restrict__ fw,
                                                         const int* __restrict__ vstart, const int* __restrict__ flist,
                                                         float* __restrict__ v_out, float* __restrict__ n_out, int* __restrict__ src) {
  const long long v = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (v >= V || removed[v]) return;
  const long long o = v - rscan[v];
  bool moved = false;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    v_out[3 * o + c] = pos[3 * v + c];
    moved |= __float_as_uint(pos[3 * v + c]) != __float_as_uint(v_in[3 * v + c]);
  }
  float n[3] = {n_in[3 * v], n_in[3 * v + 1], n_in[3 * v + 2]};
  if (moved) {
    double3 s = make_double3(0.0, 0.0, 0.0);
    for (int k = vstart[v]; k < vstart[v + 1]; ++k) {
      const int* t = fw + 3 * flist[k];
      const double3 c = face_cross(ldp(pos, t[0]), ldp(pos, t[1]), ldp(pos, t[2]));
      s.x += c.x; s.y += c.y; s.z += c.z;
    }
    const double len = sqrt(dot3(s, s));
    if (len > 0.0) { n[0] = (float)(s.x / len); n[1] = (float)(s.y / len); n[2] = (float)(s.z / len); }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) n_out[3 * o + c] = n[c];
  if (src) src[o] = (int)v;
}

// faces re-indexed through the vertex compaction; an index outside [0, V) (the error path) is copied, never dereferenced
__global__ void __launch_bounds__(kBlock) dc_fout_kernel(const int* __restrict__ fw, long long F, long long V,
                                                         const int* __restrict__ rscan, int* __restrict__ f_out) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= F) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int v = fw[3 * i + c];
    f_out[3 * i + c] = v >= 0 && v < V ? v - rscan[v] : v;
  }
}

// Workspace (256-byte aligned pieces): pos (3V floats), Q (10V doubles), m (V u64), lock, removed, rscan, deg, vstart,
// cursor, ecnt, estart (V+1 ints each), fw, fw2, flist (3F ints each), dead, dscan (F+1), per candidate edge (at most 3F/2:
// each has exactly two faces) ea, eb, sel (ints), key (u64), newpos (3 floats), the scans' block sums, misc (counters,
// radix-select state and histogram)
struct DcWs {
  float* pos;
  double* Q;
  unsigned long long *m, *key;
  int *lock, *removed, *rscan, *deg, *vstart, *cursor, *ecnt, *estart, *fw, *fw2, *flist, *dead, *dscan, *ea, *eb, *sel, *blk;
  float* newpos;
  int* misc;     // [0] bad faces, [1] selected edges, [16..31] SelectState, [64..319] histogram
};
constexpr int kMiscInts = 320;

size_t carve(void* ws, long long V, long long F, DcWs* w) {
  const long long E = 3 * F / 2 + 1;
  const long long nblk = ((V > F ? V : F) + 1 + kScanBlockEntries - 1) / kScanBlockEntries;
  const size_t vi = (size_t)(V + 1) * 4, fi = (size_t)F * 12 + 4;
  void** dst[] = {(void**)&w->pos, (void**)&w->Q, (void**)&w->m, (void**)&w->lock, (void**)&w->removed, (void**)&w->rscan,
                  (void**)&w->deg, (void**)&w->vstart, (void**)&w->cursor, (void**)&w->ecnt, (void**)&w->estart,
                  (void**)&w->fw, (void**)&w->fw2, (void**)&w->flist, (void**)&w->dead, (void**)&w->dscan,
                  (void**)&w->ea, (void**)&w->eb, (void**)&w->sel, (void**)&w->key, (void**)&w->newpos, (void**)&w->blk,
                  (void**)&w->misc};
  const size_t sz[] = {(size_t)V * 12, (size_t)V * 80, (size_t)V * 8, vi, vi, vi, vi, vi, vi, vi, vi, fi, fi, fi,
                       (size_t)(F + 1) * 4, (size_t)(F + 1) * 4, (size_t)E * 4, (size_t)E * 4, (size_t)E * 4, (size_t)E * 8,
                       (size_t)E * 12, (size_t)nblk * 4, kMiscInts * 4};
  constexpr int n = sizeof(sz) / sizeof(sz[0]);
  static_assert(n == sizeof(dst) / sizeof(dst[0]), "one size per workspace piece");
  size_t tot = 0;
  for (int i = 0; i < n; ++i) {
    if (ws) *dst[i] = reinterpret_cast<char*>(ws) + tot;
    tot += align_up(sz[i]);
  }
  return tot;
}

// vertex -> face lists of the F faces in w.fw (deg already counted): scan, fill, sort
int build_lists(const DcWs& w, long long V, long long F, cudaStream_t st, int64_t* n) {
  if (int e = exclusive_scan(w.deg, V + 1, w.blk, w.vstart, st)) return e;
  NM_CUDA(cudaMemsetAsync(w.cursor, 0, (size_t)V * 4, st));
  if (F) dc_fill_kernel<<<blocks_for(F), kBlock, 0, st>>>(w.fw, F, w.vstart, w.cursor, w.flist);
  dc_sort_kernel<<<blocks_for(V), kBlock, 0, st>>>(w.vstart, V, w.flist);
  NM_CUDA(cudaGetLastError());
  *n += 3 + (F ? 1 : 0) + 1;
  return 0;
}

}  // namespace

size_t decimate_ws_bytes(long long V, long long F) {
  DcWs w{};
  return carve(nullptr, V, F, &w);
}

int mesh_decimate(const float* verts, const float* normals, long long V, const int32_t* faces, long long F, long long target,
                  float* verts_out, float* normals_out, int32_t* faces_out, int32_t* source_out, int64_t* counts_host, void* ws,
                  int* d_err, cudaStream_t st, int64_t* launches) {
  DcWs w{};
  carve(ws, V, F, &w);
  int64_t n = 0;
  int* nbad = w.misc;
  int* nsel = w.misc + 1;
  SelectState* sstate = reinterpret_cast<SelectState*>(w.misc + 16);
  int* hist = w.misc + 64;
  NM_CUDA(cudaMemsetAsync(w.misc, 0, kMiscInts * 4, st));
  NM_CUDA(cudaMemsetAsync(w.removed, 0, (size_t)(V + 1) * 4, st));
  if (V) NM_CUDA(cudaMemcpyAsync(w.pos, verts, (size_t)V * 12, cudaMemcpyDeviceToDevice, st));
  int bad = 0;
  if (F) {
    dc_validate_kernel<<<blocks_for(F), kBlock, 0, st>>>(faces, F, V, nbad, d_err);
    NM_CUDA(cudaGetLastError());
    n += 1;
    NM_CUDA(cudaMemcpyAsync(&bad, nbad, 4, cudaMemcpyDeviceToHost, st));
    NM_CUDA(cudaStreamSynchronize(st));
  }
  const int* cur = faces;
  long long Fc = F, rounds = 0, collapses = 0;
  if (!bad && target < F) {
    // the input's lists, locks and quadrics
    NM_CUDA(cudaMemsetAsync(w.deg, 0, (size_t)(V + 1) * 4, st));
    dc_compact_kernel<<<blocks_for(F), kBlock, 0, st>>>(faces, F, nullptr, nullptr, w.fw, w.deg);
    NM_CUDA(cudaGetLastError());
    n += 1;
    if (int e = build_lists(w, V, F, st, &n)) return e;
    dc_lock_kernel<<<blocks_for(V), kBlock, 0, st>>>(w.fw, w.vstart, w.flist, V, w.lock);
    dc_quadric_kernel<<<blocks_for(V), kBlock, 0, st>>>(w.pos, w.fw, w.vstart, w.flist, V, w.Q);
    NM_CUDA(cudaGetLastError());
    n += 2;
    cur = w.fw;
    while (Fc > target) {
      const long long Emax = 3 * Fc / 2 + 1;
      NM_CUDA(cudaMemsetAsync(w.m, 0xff, (size_t)V * 8, st));
      NM_CUDA(cudaMemsetAsync(nsel, 0, 4, st));
      dc_count_kernel<<<blocks_for(V + 1), kBlock, 0, st>>>(w.fw, w.vstart, w.flist, w.lock, V, w.ecnt);
      NM_CUDA(cudaGetLastError());
      if (int e = exclusive_scan(w.ecnt, V + 1, w.blk, w.estart, st)) return e;
      const int* ne = w.estart + V;
      dc_edges_kernel<<<blocks_for(V), kBlock, 0, st>>>(w.fw, w.vstart, w.flist, w.lock, V, w.estart, w.ea, w.eb);
      dc_eval_kernel<<<blocks_for(Emax), kBlock, 0, st>>>(w.pos, w.Q, w.fw, w.vstart, w.flist, ne, w.ea, w.eb, w.key, w.newpos, w.m);
      dc_select_kernel<<<blocks_for(Emax), kBlock, 0, st>>>(w.fw, w.vstart, w.flist, ne, w.ea, w.eb, w.key, w.m, w.sel, nsel);
      NM_CUDA(cudaGetLastError());
      n += 1 + 3 + 3;
      int s = 0;
      NM_CUDA(cudaMemcpyAsync(&s, nsel, 4, cudaMemcpyDeviceToHost, st));
      NM_CUDA(cudaStreamSynchronize(st));
      if (s == 0) break;
      const long long need = (Fc - target + 1) / 2;
      if (s > need) {              // the last round: only the `need` smallest keys collapse
        const SelectState init{0ull, need};
        NM_CUDA(cudaMemcpyAsync(sstate, &init, sizeof(init), cudaMemcpyHostToDevice, st));
        for (int pass = 0; pass < 8; ++pass) {
          dc_hist_kernel<<<blocks_for(Emax), kBlock, 0, st>>>(ne, w.key, w.sel, pass, sstate, hist);
          dc_pick_kernel<<<1, 1, 0, st>>>(hist, sstate);
        }
        dc_trim_kernel<<<blocks_for(Emax), kBlock, 0, st>>>(ne, w.key, sstate, w.sel);
        NM_CUDA(cudaGetLastError());
        n += 17;
        s = (int)need;
      }
      NM_CUDA(cudaMemsetAsync(w.dead, 0, (size_t)(Fc + 1) * 4, st));
      dc_apply_kernel<<<blocks_for(Emax), kBlock, 0, st>>>(ne, w.ea, w.eb, w.sel, w.newpos, w.vstart, w.flist, w.pos, w.Q, w.fw,
                                                           w.dead, w.removed);
      NM_CUDA(cudaGetLastError());
      if (int e = exclusive_scan(w.dead, Fc + 1, w.blk, w.dscan, st)) return e;
      NM_CUDA(cudaMemsetAsync(w.deg, 0, (size_t)(V + 1) * 4, st));
      dc_compact_kernel<<<blocks_for(Fc), kBlock, 0, st>>>(w.fw, Fc, w.dead, w.dscan, w.fw2, w.deg);
      NM_CUDA(cudaGetLastError());
      n += 1 + 3 + 1;
      Fc -= 2ll * s;
      collapses += s;
      rounds += 1;
      int* t = w.fw; w.fw = w.fw2; w.fw2 = t;
      cur = w.fw;
      if (int e = build_lists(w, V, Fc, st, &n)) return e;
    }
  }
  if (V) {
    if (int e = exclusive_scan(w.removed, V + 1, w.blk, w.rscan, st)) return e;
    dc_vout_kernel<<<blocks_for(V), kBlock, 0, st>>>(w.pos, verts, normals, V, w.removed, w.rscan, cur, w.vstart, w.flist,
                                                     verts_out, normals_out, source_out);
    n += 4;
  }
  if (Fc) {
    dc_fout_kernel<<<blocks_for(Fc), kBlock, 0, st>>>(cur, Fc, V, w.rscan, faces_out);
    n += 1;
  }
  NM_CUDA(cudaGetLastError());
  NM_CUDA(cudaStreamSynchronize(st));
  counts_host[0] = V - collapses;
  counts_host[1] = Fc;
  counts_host[2] = rounds;
  counts_host[3] = collapses;
  if (launches) *launches += n;
  return 0;
}

}  // namespace nm
