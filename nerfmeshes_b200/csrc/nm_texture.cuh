// The texture atlas layout of DESIGN §4.12 on the device: where texel (i, j) of face f lies, for the kernels that write the
// atlas (nm_texture.cu) and the ones that read it (nm_raster.cu).  The host side is texture_layout (nm_common.h).
#pragma once
#include "nm_common.h"

namespace nm {

struct TexLayout {
  int N, C, K;          // texels per leg, cell side N + 2, texels per face N(N+1)/2
  long long Q, W;       // cells per row, atlas width
};

inline int tex_layout(long long F, int N, TexLayout* L) {
  long long lay[4];
  if (int e = texture_layout(F, N, lay)) return e;
  *L = TexLayout{N, N + 2, N * (N + 1) / 2, lay[0], lay[2]};
  return 0;
}

// atlas pixel of texel (i, j) of face f: half 0 at (i, j) in its cell, half 1 point-mirrored through the cell
__device__ __forceinline__ long long texel_pixel(long long f, int i, int j, const TexLayout& L) {
  const long long c = f >> 1;
  const long long x0 = (c % L.Q) * L.C, y0 = (c / L.Q) * L.C;
  const bool h1 = f & 1;
  const long long x = x0 + (h1 ? L.C - 1 - i : i), y = y0 + (h1 ? L.C - 1 - j : j);
  return y * L.W + x;
}

}  // namespace nm
