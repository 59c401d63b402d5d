// Point front-end shared by both fused-MLP kernels: fetch / synthesise one point and its view direction, and
// enumerate its positional encoding in the reference's column order.
#pragma once
#include "nm_common.h"

namespace nm {

// a4 intervals_to_ray_points (src/models/model_helpers.py:32-35): p = o + d*t as a rounded multiply then a rounded
// add (torch evaluates the two ops separately; an fma would differ in the last bit).
// a13 grid points (src/mesh_nerf.py:37-40): (lin0[i], lin1[j], lin2[k]), flat index (i*n1 + j)*n2 + k, and the
// "directions" handed to the net are the positions themselves (mesh_nerf.py:45).
__device__ __forceinline__ void fetch_point(const MlpInput& in, long long m, float p[3], float d[3]) {
  if (in.mode == IN_POINTS) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      p[c] = __ldg(in.pts + 3 * m + c);
      d[c] = in.dirs ? __ldg(in.dirs + 3 * m + c) : p[c];
    }
  } else if (in.mode == IN_RAYS) {
    const long long ray = m / in.S;
    const float t = __ldg(in.t + m);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      d[c] = __ldg(in.dirs + 3 * ray + c);
      const float o = __ldg(in.ray_o + (long long)in.o_stride * ray + c);
      p[c] = __fadd_rn(o, __fmul_rn(d[c], t));
    }
  } else {
    const long long g = in.grid_base + m;
    const int k = (int)(g % in.n2);
    const long long gj = g / in.n2;
    const int j = (int)(gj % in.n1);
    const int i = (int)(gj / in.n1);
    p[0] = __ldg(in.lin0 + i);
    p[1] = __ldg(in.lin1 + j);
    p[2] = __ldg(in.lin2 + k);
    d[0] = p[0]; d[1] = p[1]; d[2] = p[2];
  }
}

// a5 PositionalEncoding (src/nerf/modules.py:26-34): column order [x (if include_input), sin(x_c*f_k) for c in xyz
// for k, cos(same)] (SURVEY A.2).  x_c*f_k is an exact fp32 product; sincosf is the accurate (not the __sinf
// intrinsic) path: arguments reach ~3000 rad.  emit(column, value).
template <class Emit>
__device__ __forceinline__ void positional_encoding(const float x[3], int L, int include_input, const float* freq,
                                                    Emit emit) {
  int base = 0;
  if (include_input) {
    emit(0, x[0]); emit(1, x[1]); emit(2, x[2]);
    base = 3;
  }
  for (int c = 0; c < 3; ++c) {
    for (int k = 0; k < L; ++k) {
      float s, co;
      sincosf(__fmul_rn(x[c], freq[k]), &s, &co);
      emit(base + c * L + k, s);
      emit(base + 3 * L + c * L + k, co);
    }
  }
}

// The encoding's vector-Jacobian product: g_c = sum_j adj(j) d enc_j / d x_c in positional_encoding's column order, at the
// same fp32 argument x_c*f_k and with the same accurate sincosf:  d sin(f x)/dx = f cos(f x),  d cos(f x)/dx = -f sin(f x),
// the identity block when include_input.  adj(column) returns the adjoint of that encoding column.
template <class Adj>
__device__ __forceinline__ void positional_encoding_vjp(const float x[3], int L, int include_input, const float* freq,
                                                        Adj adj, float g[3]) {
  const int base = include_input ? 3 : 0;
  for (int c = 0; c < 3; ++c) {
    float acc = include_input ? adj(c) : 0.f;
    for (int k = 0; k < L; ++k) {
      float s, co;
      sincosf(__fmul_rn(x[c], freq[k]), &s, &co);
      const float t = fmaf(adj(base + c * L + k), co, -adj(base + 3 * L + c * L + k) * s);
      acc = fmaf(freq[k], t, acc);
    }
    g[c] = acc;
  }
}

}  // namespace nm
