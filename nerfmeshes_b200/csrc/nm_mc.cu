// Marching cubes on a device-resident fp32 volume — the skimage.measure.marching_cubes(volume, level) seam of
// src/mesh_nerf.py:79 (a15), Lewiner-style (MC33) topology resolution.  HBM-bound byte / bit work:
//
//   1. mc_sign_kernel    ONE streaming pass over the 4*N-byte volume -> a sign BIT-volume (1 bit per grid point, N/8 bytes:
//                        16.7 MB at 512^3, L2-resident).  This is the only pass that reads the whole volume.
//   2. mc_count_kernel   one thread per 32-point word of a grid line: crossed edges (X, Y, Z) and active cells fall out of
//                        XORs / shifts of four neighbouring sign words; only active cells (~1 %) are visited one by one, and
//                        only topologically ambiguous ones read their 8 corner values (face tests, interior test).  Writes
//                        per word: the X/Y/Z/C bit words, vertex + triangle counts; per block: the count sums.
//   3. mc_scan_blocks / mc_scan_words   two-level exclusive scan of the counts (per-word vertex / triangle prefixes).
//   4. mc_expand_kernel  one thread per word: writes, for every vertex id and every triangle id of the word, where it comes
//                        from (word, bit, slot / table entry, triangle) — an 8-byte record per output element.
//   5. mc_emit_vertices / mc_emit_triangles   one thread per OUTPUT vertex / triangle (perfectly balanced, coalesced
//                        stores); a vertex id anywhere in the grid is prefix[word] + popcount(bits below) — no dense
//                        per-point id array.
//   6. mc_ss_points_kernel / mc_ss_refine_kernel   super-sampled emit (nm_mc_emit_ss, DESIGN.md 4.3): after 5., s network
//                        points per vertex, the fused MLP sigma-only on them, then each edge vertex re-placed along its edge.
//
// Output contract (mirrors the Lewiner output the reference consumes at mesh_nerf.py:79-90): an INDEXED mesh, one vertex
// per crossed grid edge plus Lewiner's cell-centre vertices, vertices (V,3) fp32 in index coordinates (axis0, axis1, axis2),
// faces (F,3) int32, normals (V,3) unit vectors pointing towards decreasing values.  Canonical order: vertices by owning
// grid point (flat index (i*ny + j)*nz + k), then slot (axis-0/1/2 edge, centre); triangles by cell, then table order —
// identical to oracle/mc_oracle.c, which derives everything procedurally (no shared table), so the two implementations
// can be compared array for array, bit for bit.
//
// Sharding (SURVEY 8e): the buffer holds global planes [g_x0, g_x0+nb); this call owns the points of buffer planes
// [p_lo, p_hi).  Ids of the next plane's vertices (referenced by the last owned cell layer) continue this shard's
// numbering, which is exactly what the next shard assigns from v_base + nv: concatenated shard outputs equal the
// single-GPU arrays bit for bit, no duplicate vertices, no dedup pass.
//
// Parity status: scikit-image 0.17.2 is not installable here: PARITY UNPINNED (SURVEY 8c).  What follows the published
// algorithm and what cannot: oracle/mc_oracle.c header and DESIGN.md 4.3.  This TU is compiled with -fmad=false: the face /
// interior tests and the vertex interpolation are evaluated in double with separate roundings, like the C oracle.
#include <cfloat>
#include <math_constants.h>

#include "nm_common.h"
#include "nm_mc_tables.h"

namespace nm {
namespace {

struct L1Entry { unsigned short base; unsigned char nf, mu, lew_case; unsigned char faces[6]; };
struct L2Entry { unsigned char itest, tif; unsigned short none, tunnel; };
struct L3Entry { unsigned char ntri, uses_c; unsigned char idx[3 * NM_MC_MAX_TRI]; };

__device__ const L1Entry g_l1[256] = NM_MC_L1;
__device__ const L2Entry g_l2[NM_MC_N_L2] = NM_MC_L2;
__device__ const L3Entry g_l3[NM_MC_N_L3] = NM_MC_L3;
__constant__ unsigned char c_edge_lo[12] = NM_MC_EDGE_LO;
__constant__ unsigned char c_edge_axis[12] = NM_MC_EDGE_AXIS;
__constant__ unsigned char c_face_corners[6][4] = NM_MC_FACE_CORNERS;
__constant__ unsigned char c_lew2my[8] = NM_MC_LEW2MY;
__constant__ unsigned char c_itest_edge[12][8] = NM_MC_ITEST_EDGE;

constexpr int kBlock = 256;
constexpr double kEps = (double)FLT_EPSILON;

struct McGrid {
  const float* vol;
  int nb, ny, nz, W;          // buffer planes, lines per plane, points per line, 32-bit words per line
  int g_x0, g_nx, x_shift;    // global index of buffer plane 0, planes of the global grid, pure coordinate offset
  int p_lo, p_hi, p_end;      // owned planes [p_lo,p_hi); [p_hi,p_end) = the shadow plane (ids only), 0 or 1 plane
  float iso;
  // workspace
  unsigned* sign;             // [nb*ny*W]
  uint4* bits;                // [(p_end-p_lo)*ny*W] X, Y, Z, C
  unsigned* cnt;              // per word: vertices | triangles << 16
  unsigned* vpre;             // per word: exclusive vertex prefix
  unsigned* tpre;             // per word: exclusive triangle prefix
  unsigned* blk;              // per block of kBlock words: {vertex sum, triangle sum} -> exclusive prefixes
  unsigned long long* totals; // [n_vertices incl. shadow plane, n_triangles, n_vertices owned]
  unsigned long long* vmap;   // per owned vertex id: word << 7 | bit << 2 | slot            (second workspace, sized after the count)
  unsigned long long* tmap;   // per triangle id:     word << 32 | L3 entry << 9 | bit << 4 | triangle
  long long nwords;           // words of planes [p_lo,p_end)
  long long nwords_own;       // words of planes [p_lo,p_hi)
};

// ------------------------------------------------------------------------------------------------ 1. sign bit-volume
__global__ void __launch_bounds__(kBlock) mc_sign_kernel(const float* __restrict__ vol, long long nlines, int nz, int W,
                                                         float iso, unsigned* __restrict__ sign) {
  const int lane = threadIdx.x & 31;
  const long long nw = nlines * W;
  const long long warps = (long long)gridDim.x * (kBlock / 32);
  const long long warp0 = (long long)blockIdx.x * (kBlock / 32) + (threadIdx.x >> 5);
  if ((nz & 127) == 0) {
    // lines are whole groups of 4 words: one 16-byte load per lane covers 4 points, a warp covers 4 words; the lane's
    // nibble is OR-reduced over its group of 8 lanes (3 shuffles) and the group leader stores the word
    const long long ngroups = nw >> 2;
    const float4* v4 = reinterpret_cast<const float4*>(vol);
    constexpr int U = 4;
    for (long long grp = warp0; grp < ngroups; grp += warps * U) {
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long gq = grp + warps * u;
        v[u] = make_float4(-CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F, -CUDART_INF_F);
        if (gq < ngroups) v[u] = __ldcs(v4 + gq * 32 + lane);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const long long gq = grp + warps * u;
        unsigned nib = (v[u].x > iso ? 1u : 0u) | (v[u].y > iso ? 2u : 0u) | (v[u].z > iso ? 4u : 0u) | (v[u].w > iso ? 8u : 0u);
        nib <<= 4 * (lane & 7);
        nib |= __shfl_xor_sync(0xffffffffu, nib, 1);
        nib |= __shfl_xor_sync(0xffffffffu, nib, 2);
        nib |= __shfl_xor_sync(0xffffffffu, nib, 4);
        if ((lane & 7) == 0 && gq < ngroups) sign[gq * 4 + (lane >> 3)] = nib;
      }
    }
    return;
  }
  constexpr int U = 8;
  for (long long word = warp0; word < nw; word += warps * U) {
    float v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long wd = word + warps * u;
      v[u] = -CUDART_INF_F;
      if (wd < nw) {
        const unsigned line = (unsigned)((unsigned long long)wd / (unsigned)W);      // nw < 2^32 is checked by the host
        const int k = (int)((unsigned)wd - line * (unsigned)W) * 32 + lane;
        if (k < nz) v[u] = __ldcs(vol + (long long)line * nz + k);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long wd = word + warps * u;
      const unsigned b = __ballot_sync(0xffffffffu, v[u] > iso);
      if (lane == 0 && wd < nw) sign[wd] = b;
    }
  }
}

// ------------------------------------------------------------------------------------------------ cell resolution
// test_face: are the MARKED corners joined across ambiguous face f?   (oracle/mc_oracle.c face_joined)
__device__ __forceinline__ int face_joined(const double* val, int f, int mu_pos) {
  const double A = val[c_face_corners[f][0]], B = val[c_face_corners[f][1]], C = val[c_face_corners[f][2]],
               D = val[c_face_corners[f][3]];
  const double X = A * C - B * D;
  if (X > -kEps && X < kEps) return mu_pos;
  return mu_pos ? (A * X >= 0.0) : (A * X <= 0.0);
}

// test_interior reduced to its indicator (oracle/mc_oracle.c interior_I)
__device__ int interior_I(const double* val, int itest) {
  double At, Bt, Ct, Dt;
  if (itest == 1) {
    const double v0 = val[c_lew2my[0]], v1 = val[c_lew2my[1]], v2 = val[c_lew2my[2]], v3 = val[c_lew2my[3]];
    const double v4 = val[c_lew2my[4]], v5 = val[c_lew2my[5]], v6 = val[c_lew2my[6]], v7 = val[c_lew2my[7]];
    const double a = (v4 - v0) * (v6 - v2) - (v7 - v3) * (v5 - v1);
    const double b = v2 * (v4 - v0) + v0 * (v6 - v2) - v1 * (v7 - v3) - v3 * (v5 - v1);
    const double t = -b / (2 * a + kEps);
    if (t < 0 || t > 1) return 0;
    At = v0 + (v4 - v0) * t; Bt = v3 + (v7 - v3) * t; Ct = v2 + (v6 - v2) * t; Dt = v1 + (v5 - v1) * t;
  } else {
    const unsigned char* r = c_itest_edge[itest - 2];
    const double t = val[r[0]] / (val[r[0]] - val[r[1]]);
    At = 0;
    Bt = val[r[2]] + (val[r[3]] - val[r[2]]) * t;
    Ct = val[r[4]] + (val[r[5]] - val[r[4]]) * t;
    Dt = val[r[6]] + (val[r[7]] - val[r[6]]) * t;
  }
  const int test = (At >= 0 ? 1 : 0) | (Bt >= 0 ? 2 : 0) | (Ct >= 0 ? 4 : 0) | (Dt >= 0 ? 8 : 0);
  switch (test) {
    case 7: case 11: case 13: case 14: case 15: return 1;
    case 5: return !(At * Ct - Bt * Dt < kEps);
    case 10: return !(At * Ct - Bt * Dt >= kEps);
    default: return 0;
  }
}

// level-3 entry (triangulation) of the cell with sign mask m whose low corner is flat point index p
__device__ __forceinline__ int resolve_cell(const McGrid& g, unsigned m, size_t p) {
  const L1Entry e1 = g_l1[m];
  L2Entry e2 = g_l2[e1.base];
  if (e1.nf == 0 && e2.itest == 0) return e2.none;
  double val[8];
  const size_t sx = (size_t)g.ny * g.nz, sy = (size_t)g.nz;
#pragma unroll
  for (int c = 0; c < 8; ++c) val[c] = (double)g.vol[p + (c & 1) * sx + ((c >> 1) & 1) * sy + ((c >> 2) & 1)] - (double)g.iso;
  int J = 0;
  for (int q = 0; q < e1.nf; ++q) J |= face_joined(val, e1.faces[q], e1.mu) << q;
  e2 = g_l2[e1.base + J];
  if (e2.itest == 0) return e2.none;
  return interior_I(val, e2.itest) == e2.tif ? e2.tunnel : e2.none;
}

// the four sign words around word (i,j,w) and their k+1 shifts
struct Nbhd {
  unsigned s[4], sh[4];      // index di + 2*dj
  unsigned X, Y, Z, active;
};
__device__ __forceinline__ Nbhd load_nbhd(const McGrid& g, int i, int j, int w) {
  Nbhd n;
  const bool has_i1 = g.g_x0 + i + 1 < g.g_nx, has_j1 = j + 1 < g.ny;
  const int k0 = w * 32;
  const unsigned validk = (g.nz - k0 >= 32) ? 0xffffffffu : ((1u << (g.nz - k0)) - 1u);
  const unsigned validk1 = (g.nz - 1 - k0 >= 32) ? 0xffffffffu : (g.nz - 1 - k0 <= 0 ? 0u : ((1u << (g.nz - 1 - k0)) - 1u));
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const int di = c & 1, dj = c >> 1;
    const bool ok = (!di || has_i1) && (!dj || has_j1);
    unsigned a = 0, an = 0;
    if (ok) {
      const size_t base = ((size_t)(i + di) * g.ny + (j + dj)) * g.W + w;
      a = g.sign[base];
      if (w + 1 < g.W) an = g.sign[base + 1];
    }
    n.s[c] = a;
    n.sh[c] = (a >> 1) | (an << 31);
  }
  n.X = has_i1 ? ((n.s[0] ^ n.s[1]) & validk) : 0u;
  n.Y = has_j1 ? ((n.s[0] ^ n.s[2]) & validk) : 0u;
  n.Z = (n.s[0] ^ n.sh[0]) & validk1;
  if (has_i1 && has_j1) {
    const unsigned o = n.s[0] | n.s[1] | n.s[2] | n.s[3] | n.sh[0] | n.sh[1] | n.sh[2] | n.sh[3];
    const unsigned a = n.s[0] & n.s[1] & n.s[2] & n.s[3] & n.sh[0] & n.sh[1] & n.sh[2] & n.sh[3];
    n.active = (o & ~a) & validk1;
  } else {
    n.active = 0u;
  }
  return n;
}
__device__ __forceinline__ unsigned cell_mask(const Nbhd& n, int b) {   // corner c = di + 2 dj + 4 dk
  return ((n.s[0] >> b) & 1u) | (((n.s[1] >> b) & 1u) << 1) | (((n.s[2] >> b) & 1u) << 2) | (((n.s[3] >> b) & 1u) << 3) |
         (((n.sh[0] >> b) & 1u) << 4) | (((n.sh[1] >> b) & 1u) << 5) | (((n.sh[2] >> b) & 1u) << 6) | (((n.sh[3] >> b) & 1u) << 7);
}

__device__ __forceinline__ void word_coords(const McGrid& g, long long wl, int* i, int* j, int* w) {
  const unsigned u = (unsigned)wl;                     // word counts stay below 2^32 (make_grid): 32-bit divisions
  const unsigned line = u / (unsigned)g.W;
  *w = (int)(u - line * (unsigned)g.W);
  const unsigned pi = line / (unsigned)g.ny;
  *i = g.p_lo + (int)pi;
  *j = (int)(line - pi * (unsigned)g.ny);
}

__device__ __forceinline__ unsigned block_sum(unsigned v, unsigned* s_warp) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = v;
  __syncthreads();
  unsigned t = 0;
#pragma unroll
  for (int w = 0; w < kBlock / 32; ++w) t += s_warp[w];
  __syncthreads();
  return t;
}

// ------------------------------------------------------------------------------------------------ 2. count
__global__ void __launch_bounds__(kBlock) mc_count_kernel(const McGrid g) {
  __shared__ unsigned s_warp[kBlock / 32];
  const long long wl = (long long)blockIdx.x * kBlock + threadIdx.x;
  unsigned vc = 0, tc = 0;
  if (wl < g.nwords) {
    int i, j, w;
    word_coords(g, wl, &i, &j, &w);
    const Nbhd n = load_nbhd(g, i, j, w);
    unsigned C = 0;
    const bool owned = i < g.p_hi;
    unsigned act = n.active;
    while (act) {
      const int b = __ffs(act) - 1;
      act &= act - 1;
      const size_t p = ((size_t)i * g.ny + j) * g.nz + (size_t)w * 32 + b;
      const L3Entry* e = &g_l3[resolve_cell(g, cell_mask(n, b), p)];
      if (owned) tc += e->ntri;
      C |= (unsigned)e->uses_c << b;
    }
    vc = __popc(n.X) + __popc(n.Y) + __popc(n.Z) + __popc(C);
    g.bits[wl] = make_uint4(n.X, n.Y, n.Z, C);
    g.cnt[wl] = vc | (tc << 16);
  }
  const unsigned sv = block_sum(vc, s_warp), stt = block_sum(tc, s_warp);
  if (threadIdx.x == 0) { g.blk[2 * blockIdx.x] = sv; g.blk[2 * blockIdx.x + 1] = stt; }
}

// ------------------------------------------------------------------------------------------------ 3. scans
// exclusive scan of the per-block sums (a few 1e4 entries): one block, 1024 entries per round, coalesced, running carry
__global__ void __launch_bounds__(1024) mc_scan_blocks(McGrid g, int nblocks) {
  __shared__ unsigned long long s_v[32], s_t[32];
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  unsigned long long carry_v = 0, carry_t = 0;
  uint2* blk = reinterpret_cast<uint2*>(g.blk);
  for (int base = 0; base < nblocks; base += 1024) {
    const int l = base + t;
    const uint2 c = l < nblocks ? blk[l] : make_uint2(0u, 0u);
    unsigned long long xv = c.x, xt = c.y;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long yv = __shfl_up_sync(0xffffffffu, xv, o), yt = __shfl_up_sync(0xffffffffu, xt, o);
      if (lane >= o) { xv += yv; xt += yt; }
    }
    if (lane == 31) { s_v[wid] = xv; s_t[wid] = xt; }
    __syncthreads();
    if (wid == 0) {
      unsigned long long av = s_v[lane], at = s_t[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long yv = __shfl_up_sync(0xffffffffu, av, o), yt = __shfl_up_sync(0xffffffffu, at, o);
        if (lane >= o) { av += yv; at += yt; }
      }
      s_v[lane] = av; s_t[lane] = at;                    // inclusive scan of the warp totals
    }
    __syncthreads();
    const unsigned long long wv = wid ? s_v[wid - 1] : 0, wt = wid ? s_t[wid - 1] : 0;
    if (l < nblocks) blk[l] = make_uint2((unsigned)(carry_v + wv + xv - c.x), (unsigned)(carry_t + wt + xt - c.y));
    carry_v += s_v[31]; carry_t += s_t[31];
    __syncthreads();
  }
  if (t == 0) { g.totals[0] = carry_v; g.totals[1] = carry_t; }
}

__global__ void __launch_bounds__(kBlock) mc_scan_words(const McGrid g) {
  __shared__ unsigned s_v[kBlock / 32], s_t[kBlock / 32];
  const long long wl = (long long)blockIdx.x * kBlock + threadIdx.x;
  const unsigned c = wl < g.nwords ? g.cnt[wl] : 0u;
  const unsigned v = c & 0xffffu, t = c >> 16;
  unsigned xv = v, xt = t;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned yv = __shfl_up_sync(0xffffffffu, xv, o), yt = __shfl_up_sync(0xffffffffu, xt, o);
    if (lane >= o) { xv += yv; xt += yt; }
  }
  if (lane == 31) { s_v[wid] = xv; s_t[wid] = xt; }
  __syncthreads();
  unsigned bv = g.blk[2 * blockIdx.x], bt = g.blk[2 * blockIdx.x + 1];
  for (int q = 0; q < wid; ++q) { bv += s_v[q]; bt += s_t[q]; }
  if (wl < g.nwords) {
    g.vpre[wl] = bv + xv - v;
    g.tpre[wl] = bt + xt - t;
    if (wl == g.nwords_own) g.totals[2] = bv + xv - v;            // first word of the shadow plane: owned vertex count
  }
}

// ------------------------------------------------------------------------------------------------ 4. emission
// central difference inside the GLOBAL grid, one-sided on its boundary (the halo planes are in the buffer)
__device__ __forceinline__ void grid_grad(const McGrid& g, int i, int j, int k, float out[3]) {
  const size_t p = ((size_t)i * g.ny + j) * g.nz + k;
  const size_t st[3] = {(size_t)g.ny * g.nz, (size_t)g.nz, 1};
  const int gl[3] = {g.g_x0 + i, j, k}, n[3] = {g.g_nx, g.ny, g.nz};
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const bool lo = gl[a] > 0, hi = gl[a] + 1 < n[a];
    if (lo && hi) out[a] = 0.5f * (g.vol[p + st[a]] - g.vol[p - st[a]]);
    else if (hi) out[a] = g.vol[p + st[a]] - g.vol[p];
    else if (lo) out[a] = g.vol[p] - g.vol[p - st[a]];
    else out[a] = 0.f;
  }
}

__device__ __forceinline__ void store_vertex(float* verts, float* normals, size_t id, const double pos[3], const double n[3]) {
  const double len = sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
  const double inv = len > 0.0 ? 1.0 / len : 0.0;
#pragma unroll
  for (int b = 0; b < 3; ++b) {
    verts[3 * id + b] = (float)pos[b];
    if (normals) normals[3 * id + b] = (float)(n[b] * inv);
  }
}

// 4. expansion: where every output vertex / triangle comes from
__global__ void __launch_bounds__(kBlock) mc_expand_kernel(const McGrid g) {
  const long long wl = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (wl >= g.nwords_own) return;
  const unsigned c = g.cnt[wl];
  if (c == 0) return;
  if (c & 0xffffu) {
    const uint4 B = g.bits[wl];
    unsigned long long id = g.vpre[wl];
    unsigned any = B.x | B.y | B.z | B.w;
    while (any) {
      const int b = __ffs(any) - 1;
      any &= any - 1;
      const unsigned sel = ((B.x >> b) & 1u) | (((B.y >> b) & 1u) << 1) | (((B.z >> b) & 1u) << 2) | (((B.w >> b) & 1u) << 3);
#pragma unroll
      for (int a = 0; a < 4; ++a)
        if ((sel >> a) & 1u) g.vmap[id++] = ((unsigned long long)wl << 7) | ((unsigned long long)b << 2) | (unsigned long long)a;
    }
  }
  if (c >> 16) {
    int i, j, w;
    word_coords(g, wl, &i, &j, &w);
    const Nbhd n = load_nbhd(g, i, j, w);
    unsigned long long tid = g.tpre[wl];
    unsigned act = n.active;
    while (act) {
      const int b = __ffs(act) - 1;
      act &= act - 1;
      const size_t p = ((size_t)i * g.ny + j) * g.nz + (size_t)w * 32 + b;
      const unsigned e = (unsigned)resolve_cell(g, cell_mask(n, b), p);
      const unsigned nt = g_l3[e].ntri;
      for (unsigned t = 0; t < nt; ++t)
        g.tmap[tid++] = ((unsigned long long)wl << 32) | ((unsigned long long)e << 9) | ((unsigned long long)b << 4) | t;
    }
  }
}

// 5. one thread per output vertex
__global__ void __launch_bounds__(kBlock) mc_emit_vertices(const McGrid g, unsigned nv, float* __restrict__ verts,
                                                           float* __restrict__ normals) {
  const unsigned id = blockIdx.x * kBlock + threadIdx.x;
  if (id >= nv) return;
  const unsigned long long rec = g.vmap[id];
  const long long wl = (long long)(rec >> 7);
  const int b = (int)((rec >> 2) & 31u), slot = (int)(rec & 3u);
  int i, j, w;
  word_coords(g, wl, &i, &j, &w);
  const size_t st[3] = {(size_t)g.ny * g.nz, (size_t)g.nz, 1};
  const double iso = (double)g.iso;
  const int k = w * 32 + b;
  const size_t p = ((size_t)i * g.ny + j) * g.nz + k;
  const double base[3] = {(double)(g.g_x0 + i + g.x_shift), (double)j, (double)k};
  if (slot < 3) {
    const int a = slot;
    float g0[3], g1[3];
    grid_grad(g, i, j, k, g0);
    int c1[3] = {i, j, k};
    c1[a] += 1;
    grid_grad(g, c1[0], c1[1], c1[2], g1);
    const double w0 = 1.0 / (kEps + fabs((double)g.vol[p] - iso));
    const double w1 = 1.0 / (kEps + fabs((double)g.vol[p + st[a]] - iso));
    const double ff = w0 + w1;
    double pos[3] = {base[0], base[1], base[2]};
    pos[a] = base[a] + w1 / ff;                  // x + step * fx / ff with fx = 0*w0 + 1*w1 (scikit-image's form)
    double n[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) n[q] = -((double)g0[q] * w0 + (double)g1[q] * w1);
    store_vertex(verts, normals, id, pos, n);
  } else {                                       // calculate_center_vertex: weighted mean of the 8 corners, Lewiner's order
    double f[3] = {0, 0, 0}, ff = 0, n[3] = {0, 0, 0};
    for (int L = 0; L < 8; ++L) {
      const int c = c_lew2my[L];
      const int ci = i + (c & 1), cj = j + ((c >> 1) & 1), ck = k + ((c >> 2) & 1);
      const double wc = 1.0 / (kEps + fabs((double)g.vol[((size_t)ci * g.ny + cj) * g.nz + ck] - iso));
#pragma unroll
      for (int q = 0; q < 3; ++q) if ((c >> q) & 1) f[q] += wc;
      ff += wc;
      float gc[3];
      grid_grad(g, ci, cj, ck, gc);
#pragma unroll
      for (int q = 0; q < 3; ++q) n[q] -= (double)gc[q] * wc;
    }
    const double pos[3] = {base[0] + f[0] / ff, base[1] + f[1] / ff, base[2] + f[2] / ff};
    store_vertex(verts, normals, id, pos, n);
  }
}

// id of the vertex in slot `a` (0..2 edge along axis a, 3 centre) of grid point (i,j,k) (buffer coordinates)
__device__ __forceinline__ unsigned vertex_id(const McGrid& g, int i, int j, int k, int a) {
  const long long wq = ((long long)(i - g.p_lo) * g.ny + j) * g.W + (k >> 5);
  const int b = k & 31;
  const uint4 B = g.bits[wq];
  const unsigned lt = (1u << b) - 1u;
  const unsigned slots = ((B.x >> b) & 1u) | (((B.y >> b) & 1u) << 1) | (((B.z >> b) & 1u) << 2);
  return g.vpre[wq] + __popc(B.x & lt) + __popc(B.y & lt) + __popc(B.z & lt) + __popc(B.w & lt) + __popc(slots & ((1u << a) - 1u));
}

// one thread per output triangle
__global__ void __launch_bounds__(kBlock) mc_emit_triangles(const McGrid g, unsigned nt, long long v_base, int* __restrict__ faces) {
  const unsigned tid = blockIdx.x * kBlock + threadIdx.x;
  if (tid >= nt) return;
  const unsigned long long rec = g.tmap[tid];
  const long long wl = (long long)(rec >> 32);
  const unsigned e = (unsigned)((rec >> 9) & 0x7fffffu), b = (unsigned)((rec >> 4) & 31u), t = (unsigned)(rec & 15u);
  int i, j, w;
  word_coords(g, wl, &i, &j, &w);
  const int k = w * 32 + (int)b;
  const unsigned char* idx = g_l3[e].idx + 3 * t;
  int out[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int s = idx[c];
    unsigned id;
    if (s == 12) id = vertex_id(g, i, j, k, 3);
    else { const int lo = c_edge_lo[s]; id = vertex_id(g, i + (lo & 1), j + ((lo >> 1) & 1), k + ((lo >> 2) & 1), c_edge_axis[s]); }
    out[c] = (int)(v_base + (long long)id);
  }
  faces[3 * (size_t)tid] = out[0]; faces[3 * (size_t)tid + 1] = out[1]; faces[3 * (size_t)tid + 2] = out[2];
}

// ------------------------------------------------------------------------------------------------ 6. super-sampling
// (nm_mc_emit_ss, DESIGN 4.3)  The vertex on the axis-a edge from global grid point (I,J,K) to its neighbour has the
// samples v_0 = vol(point), v_{s+1} = vol(neighbour) and, for m = 1..s, v_m = sigma at (fine_a[idx_a*(s+1)+m] along a,
// lin_b[idx_b] along the other axes).  Vertices [v0, v0+n) of the chunk give n*s points, s per vertex; centre vertices
// are padded with s copies of their grid point (kept flat: point q belongs to vertex v0 + q/s), their sigma is unused.
struct SsTables {
  const float* lin[3];
  const float* fine[3];
  int s;
};

__global__ void __launch_bounds__(kBlock) mc_ss_points_kernel(const McGrid g, const SsTables t, unsigned v0, unsigned n,
                                                              float* __restrict__ pts) {
  const unsigned long long q = (unsigned long long)blockIdx.x * kBlock + threadIdx.x;
  if (q >= (unsigned long long)n * t.s) return;
  const unsigned vq = (unsigned)(q / (unsigned)t.s);
  const int m = (int)(q - (unsigned long long)vq * t.s) + 1;
  const unsigned long long rec = g.vmap[v0 + vq];
  const long long wl = (long long)(rec >> 7);
  const int b = (int)((rec >> 2) & 31u), slot = (int)(rec & 3u);
  int i, j, w;
  word_coords(g, wl, &i, &j, &w);
  const int idx[3] = {g.g_x0 + i, j, w * 32 + b};
  float p[3] = {t.lin[0][idx[0]], t.lin[1][idx[1]], t.lin[2][idx[2]]};
  if (slot < 3) p[slot] = t.fine[slot][(size_t)idx[slot] * (t.s + 1) + m];
#pragma unroll
  for (int c = 0; c < 3; ++c) pts[3 * q + c] = p[c];
}

// refined position of the chunk's edge vertices: the first sub-interval [m, m+1] whose samples straddle iso, placed with
// the same weights as mc_emit_vertices; only coordinate a of the vertex is rewritten (normals, centre vertices untouched)
__global__ void __launch_bounds__(kBlock) mc_ss_refine_kernel(const McGrid g, int s, unsigned v0, unsigned n,
                                                              const float* __restrict__ sig, float* __restrict__ verts) {
  const unsigned q = blockIdx.x * kBlock + threadIdx.x;
  if (q >= n) return;
  const unsigned id = v0 + q;
  const unsigned long long rec = g.vmap[id];
  const int slot = (int)(rec & 3u);
  if (slot == 3) return;
  const long long wl = (long long)(rec >> 7);
  const int b = (int)((rec >> 2) & 31u), a = slot;
  int i, j, w;
  word_coords(g, wl, &i, &j, &w);
  const int k = w * 32 + b;
  const size_t p = ((size_t)i * g.ny + j) * g.nz + k;
  const size_t st = a == 0 ? (size_t)g.ny * g.nz : (a == 1 ? (size_t)g.nz : 1);
  const float* vs = sig + (size_t)q * s;
  float va = g.vol[p], vb = va;
  const bool in0 = va > g.iso;
  int m = 0;
  for (; m <= s; ++m) {                          // v_{s+1} differs from v_0 in sign: the loop always breaks
    vb = m < s ? vs[m] : g.vol[p + st];
    if ((vb > g.iso) != in0) break;
    va = vb;
  }
  const double iso = (double)g.iso;
  const double w0 = 1.0 / (kEps + fabs((double)va - iso));
  const double w1 = 1.0 / (kEps + fabs((double)vb - iso));
  const double base = a == 0 ? (double)(g.g_x0 + i + g.x_shift) : (double)(a == 1 ? j : k);
  verts[3 * (size_t)id + a] = (float)(base + ((double)m + w1 / (w0 + w1)) / (double)(s + 1));
}

size_t align_up(size_t x) { return (x + 255) / 256 * 256; }

int carve(void* base, size_t bytes, McGrid* g, size_t* need) {
  const size_t nsign = (size_t)g->nb * g->ny * g->W;
  const size_t nw = (size_t)g->nwords, nblk = (nw + kBlock - 1) / kBlock;
  size_t off = 0;
  auto take = [&](size_t b) { size_t o = off; off += align_up(b); return o; };
  const size_t o_sign = take(nsign * 4), o_bits = take(nw * 16), o_cnt = take(nw * 4), o_vp = take((nw + 1) * 4),
               o_tp = take((nw + 1) * 4), o_blk = take((nblk + 1) * 8), o_tot = take(64);
  *need = off;
  if (!base || bytes < off) return 1;
  char* b = reinterpret_cast<char*>(base);
  g->sign = reinterpret_cast<unsigned*>(b + o_sign);
  g->bits = reinterpret_cast<uint4*>(b + o_bits);
  g->cnt = reinterpret_cast<unsigned*>(b + o_cnt);
  g->vpre = reinterpret_cast<unsigned*>(b + o_vp);
  g->tpre = reinterpret_cast<unsigned*>(b + o_tp);
  g->blk = reinterpret_cast<unsigned*>(b + o_blk);
  g->totals = reinterpret_cast<unsigned long long*>(b + o_tot);
  return 0;
}

int make_grid(const McShard& s, McGrid* g) {
  NM_CHECK(s.vol && s.nb >= 1 && s.ny >= 2 && s.nz >= 2, "marching cubes: bad volume shape");
  NM_CHECK(s.g_x0 >= 0 && s.g_x0 + s.nb <= s.g_nx && s.g_nx >= 2, "marching cubes: buffer planes outside the global grid");
  NM_CHECK(0 <= s.p_lo && s.p_lo <= s.p_hi && s.p_hi <= s.nb, "marching cubes: bad owned plane range");
  const bool next_exists = s.g_x0 + s.p_hi < s.g_nx;                    // the plane after the owned ones exists globally
  NM_CHECK(!next_exists || s.p_hi < s.nb, "marching cubes: plane after the owned range is missing from the buffer");
  // gradients at the owned planes and at plane p_hi need one more plane on either side (unless it is the global boundary)
  NM_CHECK(s.p_lo == s.p_hi || s.g_x0 + s.p_lo == 0 || s.p_lo >= 1, "marching cubes: halo plane below the owned range missing");
  NM_CHECK(!next_exists || s.g_x0 + s.p_hi + 1 >= s.g_nx || s.p_hi + 1 < s.nb, "marching cubes: halo plane above the owned range missing");
  g->vol = s.vol; g->nb = s.nb; g->ny = s.ny; g->nz = s.nz; g->W = (s.nz + 31) / 32;
  g->g_x0 = s.g_x0; g->g_nx = s.g_nx; g->x_shift = s.x_shift; g->p_lo = s.p_lo; g->p_hi = s.p_hi; g->p_end = s.p_hi + (next_exists ? 1 : 0);
  g->iso = s.iso;
  g->nwords = (long long)(g->p_end - g->p_lo) * g->ny * g->W;
  g->nwords_own = (long long)(g->p_hi - g->p_lo) * g->ny * g->W;
  NM_CHECK((long long)s.nb * s.ny * g->W < (1ll << 32), "marching cubes: volume too large (more than 2^32 words)");
  return 0;
}

}  // namespace

size_t mc_ws_bytes(const McShard& s) {
  McGrid g{};
  size_t need = 0;
  if (make_grid(s, &g)) return 0;            // a bad shard: mc_count reports it
  carve(nullptr, 0, &g, &need);
  return need;
}

size_t mc_emit_ws_bytes(int64_t nv, int64_t nt) { return align_up((size_t)nv * 8 + 8) + (size_t)nt * 8 + 8; }

int mc_count(const McShard& s, void* ws, size_t ws_bytes, int64_t* counts_host, int num_sms, cudaStream_t st,
             int64_t* launches) {
  McGrid g{};
  if (int e = make_grid(s, &g)) return e;
  size_t need = 0;
  NM_CHECK(carve(ws, ws_bytes, &g, &need) == 0, "marching cubes: workspace smaller than mc_ws_bytes");
  counts_host[0] = counts_host[1] = 0;
  if (g.nwords == 0) return 0;
  const long long nlines = (long long)g.nb * g.ny;
  long long sign_blocks = (nlines * g.W + (kBlock / 32) * 8 - 1) / ((kBlock / 32) * 8);
  if (sign_blocks > (long long)num_sms * 4) sign_blocks = (long long)num_sms * 4;       // one resident wave, grid-stride
  NM_CUDA(cudaMemsetAsync(g.totals, 0, 64, st));
  mc_sign_kernel<<<(unsigned)sign_blocks, kBlock, 0, st>>>(g.vol, nlines, g.nz, g.W, g.iso, g.sign);
  NM_CUDA(cudaGetLastError());
  const long long nblk = (g.nwords + kBlock - 1) / kBlock;
  NM_CHECK(nblk < (1ll << 31), "marching cubes: volume too large");
  mc_count_kernel<<<(unsigned)nblk, kBlock, 0, st>>>(g);
  NM_CUDA(cudaGetLastError());
  mc_scan_blocks<<<1, 1024, 0, st>>>(g, (int)nblk);
  NM_CUDA(cudaGetLastError());
  mc_scan_words<<<(unsigned)nblk, kBlock, 0, st>>>(g);
  NM_CUDA(cudaGetLastError());
  unsigned long long h[3];
  NM_CUDA(cudaMemcpyAsync(h, g.totals, sizeof(h), cudaMemcpyDeviceToHost, st));
  NM_CUDA(cudaStreamSynchronize(st));
  const unsigned long long nv_own = (g.p_end > g.p_hi) ? h[2] : h[0];
  NM_CHECK(h[0] < (1ull << 31) && h[1] < (1ull << 31), "mesh too large for int32 indices");
  counts_host[0] = (int64_t)nv_own;
  counts_host[1] = (int64_t)h[1];
  if (launches) *launches += 4;
  return 0;
}

int mc_emit(const McShard& s, void* ws, size_t ws_bytes, void* ws2, long long v_base, int64_t nv, int64_t nt, float* verts,
            float* normals, int32_t* faces, cudaStream_t st, int64_t* launches) {
  McGrid g{};
  if (int e = make_grid(s, &g)) return e;
  size_t need = 0;
  NM_CHECK(carve(ws, ws_bytes, &g, &need) == 0, "workspace missing (call the count step first, same arguments)");
  if (g.nwords_own == 0 || (nv == 0 && nt == 0)) return 0;
  NM_CHECK(g.nwords_own < (1ll << 32) && nv >= 0 && nt >= 0, "bad counts");
  g.vmap = reinterpret_cast<unsigned long long*>(ws2);
  g.tmap = reinterpret_cast<unsigned long long*>(reinterpret_cast<char*>(ws2) + align_up((size_t)nv * 8 + 8));
  const long long nblk = (g.nwords_own + kBlock - 1) / kBlock;
  mc_expand_kernel<<<(unsigned)nblk, kBlock, 0, st>>>(g);
  NM_CUDA(cudaGetLastError());
  if (nv) {
    mc_emit_vertices<<<(unsigned)((nv + kBlock - 1) / kBlock), kBlock, 0, st>>>(g, (unsigned)nv, verts, normals);
    NM_CUDA(cudaGetLastError());
  }
  if (nt) {
    mc_emit_triangles<<<(unsigned)((nt + kBlock - 1) / kBlock), kBlock, 0, st>>>(g, (unsigned)nt, v_base, faces);
    NM_CUDA(cudaGetLastError());
  }
  if (launches) *launches += 3;
  return 0;
}

int mc_emit_ss(const McShard& s, void* ws, size_t ws_bytes, void* ws2, long long v_base, int64_t nv, int64_t nt,
               const McSuperSampling& ss, float* verts, float* normals, int32_t* faces, cudaStream_t st, int64_t* launches) {
  NM_CHECK(ss.s >= 0 && ss.s <= kMcMaxSuperSampling, "super-sampling factor %d outside [0, %d]", ss.s, kMcMaxSuperSampling);
  // the s = 0 mesh (vertices, normals, faces, and the vertex records in the second workspace) ...
  if (int e = mc_emit(s, ws, ws_bytes, ws2, v_base, nv, nt, verts, normals, faces, st, launches)) return e;
  if (nv == 0) return 0;
  NM_CHECK(ss.lin[0] && ss.lin[1] && ss.lin[2] && ss.fine[0] && ss.fine[1] && ss.fine[2], "super-sampling tables missing");
  NM_CHECK(ss.s == 0 || (ss.pts && ss.sig && ss.chunk_vertices > 0 && ss.chunk_points > 0 && ss.eval),
           "super-sampling workspace missing");
  // ... then the edge vertices are moved, chunk by chunk
  McGrid g{};
  if (int e = make_grid(s, &g)) return e;
  g.vmap = reinterpret_cast<unsigned long long*>(ws2);
  SsTables t{};
  for (int a = 0; a < 3; ++a) { t.lin[a] = ss.lin[a]; t.fine[a] = ss.fine[a]; }
  t.s = ss.s;
  const long long per = ss.s ? ss.chunk_vertices : nv;
  for (long long v0 = 0; v0 < nv; v0 += per) {
    const long long n = nv - v0 < per ? nv - v0 : per;
    if (ss.s) {
      const long long npts = n * ss.s;
      mc_ss_points_kernel<<<(unsigned)((npts + kBlock - 1) / kBlock), kBlock, 0, st>>>(g, t, (unsigned)v0, (unsigned)n, ss.pts);
      NM_CUDA(cudaGetLastError());
      if (launches) *launches += 1;
      for (long long q0 = 0; q0 < npts; q0 += ss.chunk_points) {
        const long long m = npts - q0 < ss.chunk_points ? npts - q0 : ss.chunk_points;
        if (int e = ss.eval(ss.pts + 3 * q0, m, ss.sig + q0)) return e;
      }
    }
    mc_ss_refine_kernel<<<(unsigned)((n + kBlock - 1) / kBlock), kBlock, 0, st>>>(g, ss.s, (unsigned)v0, (unsigned)n, ss.sig, verts);
    NM_CUDA(cudaGetLastError());
    if (launches) *launches += 1;
  }
  return 0;
}

}  // namespace nm
