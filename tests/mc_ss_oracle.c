/* CPU oracle of super-sampled marching cubes (nm_mc_emit_ss, DESIGN.md 4.3) — TEST INFRASTRUCTURE ONLY, compiled at test
 * time by tests/_mc_ss_ref.py.
 *
 * The dense definition of the reference's --super-sampling branch (mesh_nerf.py:109-117): three volumes of the GLOBAL grid,
 * each refined along one axis only to (n_a - 1)(s + 1) + 1 samples, so fine sample idx*(s+1) + m lies m/(s+1) of the way along
 * the edge from grid index idx.  Topology, faces, normals and centre vertices are those of the procedural marching-cubes
 * oracle, which is included below unchanged; the edge vertices are then re-placed here, independently of the CUDA kernels:
 * the edge's samples are the two coarse end values and the s fine samples between them, and the vertex goes into the FIRST
 * sub-interval whose ends straddle iso, with the oracle's centre-of-mass weights. */
#include "../oracle/mc_oracle.c"

typedef struct { int s; const float* fine[3]; } SsVol;

static double ss_position(const Vol* V, const SsVol* S, int i, int j, int k, int a, double base_a) {
  const int s = S->s, r = s + 1, I = V->g_x0 + i;
  const size_t fy = (size_t)(V->ny - 1) * r + 1, fz = (size_t)(V->nz - 1) * r + 1;
  const size_t st[3] = {(size_t)V->ny * V->nz, (size_t)V->nz, 1};
  const size_t p = pidx(V, i, j, k);
  double v[66];
  v[0] = (double)V->vol[p];
  v[s + 1] = (double)V->vol[p + st[a]];
  for (int m = 1; m <= s; ++m) {
    size_t q;
    if (a == 0) q = ((size_t)(I * r + m) * V->ny + j) * V->nz + k;
    else if (a == 1) q = ((size_t)I * fy + (size_t)(j * r + m)) * V->nz + k;
    else q = ((size_t)I * V->ny + j) * fz + (size_t)(k * r + m);
    v[m] = (double)S->fine[a][q];
  }
  int m = 0;
  while (m < s && (v[m] - V->iso > 0.0) == (v[m + 1] - V->iso > 0.0)) ++m;
  const double w0 = 1.0 / (EPS + fabs(v[m] - V->iso));
  const double w1 = 1.0 / (EPS + fabs(v[m + 1] - V->iso));
  return base_a + ((double)m + w1 / (w0 + w1)) / (double)r;
}

/* mc_oracle's arguments plus s and the three fine volumes: xf (g_nx-1)(s+1)+1 x ny x nz, yf g_nx x (ny-1)(s+1)+1 x nz,
 * zf g_nx x ny x (nz-1)(s+1)+1. */
int mc_oracle_ss(const float* vol, int nb, int ny, int nz, float iso, int g_x0, int g_nx, int p_lo, int p_hi, int x_shift,
                 long long v_base, int s, const float* xf, const float* yf, const float* zf, float* verts, float* normals,
                 int32_t* faces, int64_t* nv_out, int64_t* nt_out) {
  if (s < 0 || s > 64 || !xf || !yf || !zf) return -5;
  const int rc = mc_oracle(vol, nb, ny, nz, iso, g_x0, g_nx, p_lo, p_hi, x_shift, v_base, verts, normals, faces, nv_out, nt_out,
                           NULL);
  if (rc || !verts) return rc;
  const Vol V = {vol, nb, ny, nz, (double)iso, g_x0, g_nx};
  const SsVol S = {s, {xf, yf, zf}};
  const size_t st[3] = {(size_t)ny * nz, (size_t)nz, 1};
  const int dims[3] = {nb, ny, nz};
  Tris T;
  int64_t id = 0;
  /* the oracle's canonical vertex order: owned points in flat order, per point its crossed edges (axis order), then the
   * centre vertex of the cell whose low corner it is, if that cell's triangulation uses one */
  for (int i = p_lo; i < p_hi; ++i)
    for (int j = 0; j < ny; ++j)
      for (int k = 0; k < nz; ++k) {
        const size_t p = pidx(&V, i, j, k);
        const int c0[3] = {i, j, k};
        const int in0 = (double)vol[p] - V.iso > 0.0;
        const double base[3] = {(double)(g_x0 + i + x_shift), (double)j, (double)k};
        for (int a = 0; a < 3; ++a) {
          const int exists = a == 0 ? (g_x0 + i + 1 < g_nx) : (c0[a] + 1 < dims[a]);
          if (!exists || ((double)vol[p + st[a]] - V.iso > 0.0) == in0) continue;
          verts[3 * id + a] = (float)ss_position(&V, &S, i, j, k, a, base[a]);
          ++id;
        }
        if (cell_exists(&V, i, j, k)) {
          double val[8];
          cell_values(&V, i, j, k, val);
          int any = 0, all = 1;
          for (int c = 0; c < 8; ++c) { const int sg = val[c] > 0.0; any |= sg; all &= sg; }
          if (any && !all) { resolve_cell(val, &T, NULL); id += T.uses_c; }
        }
      }
  return id == *nv_out ? 0 : -6;
}
