/* ORACLE -- test infrastructure only.  Nothing under 3d-re-gen_b200/ may link or call this file; only tests/ do.
 *
 * CPU restatement of r3g's dual marching cubes (include/r3g.h, R3G_MC_DUAL), the surface extractor behind
 * DMCSurfaceExtractor.run (Hunyuan3D-2/hy3dgen/shapegen/models/autoencoders/surface_extractors.py:79-94).  The reference
 * calls diso.DiffDMC, which is neither vendored nor installed; this is r3g's own specification, not diso's.
 *
 * Sequential and table driven, independent in structure from the scan-based CUDA passes: one loop over the cells in
 * traversal order (z, y, x with x = last array axis) appends the vertices of every crossed cell, one vertex per patch of
 * its Lewiner tiling (r3g_mc_dual_patch / r3g_mc_dual_npatch); a second loop appends the quads, each from the cell
 * whose maximum corner the grid edge touches, looking the four vertices up in per-cell arrays.  The Lewiner decisions
 * (test_face, test_interior) are mc_oracle.c's, included below so that both oracles take the same tiling. */
#include "mc_oracle.c"

/* The tiling of a crossed cell, as r3g_oracle_marching_cubes selects it. */
static int dual_tiling(const double *cv, int ci) {
  int sub = 0, j = 0;
  unsigned amb = r3g_mc_amb_faces[ci];
  for (int f = 0; f < 6; ++f)
    if (amb & (1u << f)) {
      if (face_pos_connected(cv, f)) sub |= 1 << j;
      ++j;
    }
  int til = r3g_mc_tiling_offset[ci] + sub;
  if (r3g_mc_interior[til] && interior_joined(cv, r3g_mc_interior[til])) til = r3g_mc_tunnel[til];
  return til;
}

/* Per array axis a of a grid edge: the four cells around it as (dx, dy, dz) offsets from the owner cell and the cube
 * edge the grid edge is in each, counter-clockwise seen from the edge's upper end (a right-handed turn about +a). */
static const unsigned char QUAD[3][4][4] = {
    {{0, 0, 0, 10}, {0, 1, 0, 9}, {1, 1, 0, 8}, {1, 0, 0, 11}},
    {{0, 0, 0, 5}, {1, 0, 0, 7}, {1, 0, 1, 3}, {0, 0, 1, 1}},
    {{0, 0, 0, 6}, {0, 0, 1, 2}, {0, 1, 1, 0}, {0, 1, 0, 4}},
};

static double dist2(const float *v, int i, int j) {
  double s = 0.0;
  for (int a = 0; a < 3; ++a) {
    const double d = (double)v[3 * i + a] - (double)v[3 * j + a];
    s = s + d * d;
  }
  return s;
}

/* Returns 0 on success, 2 if no cell is crossed.  vol is [n0][n1][n2] C-contiguous float32; a point is above iff
 * v > level.  cells_out (optional) receives the flat cell index (z * (n1-1) + y) * (n2-1) + x of every vertex. */
int r3g_oracle_dual_marching_cubes(const float *vol, int n0, int n1, int n2, float level, float **verts_out,
                                   int64_t *nv_out, int32_t **faces_out, int64_t *nf_out, int64_t **cells_out) {
  const int cx = n2 - 1, cy = n1 - 1, cz = n0 - 1;
  const int64_t ncells = (int64_t)cx * cy * cz;
  int32_t *base = (int32_t *)malloc(sizeof(int32_t) * (size_t)ncells);
  int16_t *tils = (int16_t *)malloc(sizeof(int16_t) * (size_t)ncells);
  unsigned char *cis = (unsigned char *)malloc((size_t)ncells);
  int64_t *cells = NULL, capc = 0;
  mesh_t m;
  memset(&m, 0, sizeof(m));
  *verts_out = NULL;
  *faces_out = NULL;
  *nv_out = *nf_out = 0;
  if (cells_out) *cells_out = NULL;

  for (int z = 0; z < cz; ++z)
    for (int y = 0; y < cy; ++y)
      for (int x = 0; x < cx; ++x) {
        const int64_t cell = ((int64_t)z * cy + y) * cx + x;
        double cv[8];
        int ci = 0;
        for (int i = 0; i < 8; ++i) {
          const unsigned char *o = &r3g_mc_corner_xyz[3 * i];
          cv[i] = (double)vol[((int64_t)(z + o[2]) * n1 + (y + o[1])) * n2 + (x + o[0])] - (double)level;
          if (cv[i] > 0.0) ci |= 1 << i;
        }
        cis[cell] = (unsigned char)ci;
        base[cell] = -1;
        if (ci == 0 || ci == 255) continue;
        const int til = dual_tiling(cv, ci);
        tils[cell] = (int16_t)til;
        base[cell] = (int32_t)m.nv;
        const int org[3] = {z, y, x};    /* array-axis order */
        for (int p = 0; p < r3g_mc_dual_npatch[til]; ++p) {
          double s[3] = {0.0, 0.0, 0.0};
          int n = 0;
          for (int e = 0; e < 12; ++e) {
            if (r3g_mc_dual_patch[12 * til + e] != p) continue;
            const int a = r3g_mc_edge_corner[2 * e], b = r3g_mc_edge_corner[2 * e + 1];
            const unsigned char *oa = &r3g_mc_corner_xyz[3 * a], *ob = &r3g_mc_corner_xyz[3 * b];
            const double t = cv[a] / (cv[a] - cv[b]);
            for (int d = 0; d < 3; ++d) {
              const double pa = org[d] + oa[2 - d], pb = org[d] + ob[2 - d];
              s[d] = s[d] + (pa + t * (pb - pa));
            }
            ++n;
          }
          const int nax[3] = {n0, n1, n2};
          float q[3];
          for (int d = 0; d < 3; ++d) q[d] = (float)(s[d] / (double)n / (double)(nax[d] - 1));
          push_vertex(&m, q[0], q[1], q[2]);
          if (cells_out) {
            if (m.nv > capc) {
              capc = capc ? 2 * capc : 1024;
              cells = (int64_t *)realloc(cells, sizeof(int64_t) * (size_t)capc);
            }
            cells[m.nv - 1] = cell;
          }
        }
      }

  for (int z = 0; z < cz; ++z)
    for (int y = 0; y < cy; ++y)
      for (int x = 0; x < cx; ++x) {
        const int64_t cell = ((int64_t)z * cy + y) * cx + x;
        const int ci = cis[cell];
        if (base[cell] < 0) continue;
        /* the owned edge along axis 0 / 1 / 2 is cube edge 10 / 5 / 6; its upper end is corner 6 in all three */
        const int lower[3] = {2, 5, 7};
        const int inside[3] = {x + 1 < cx && y + 1 < cy, x + 1 < cx && z + 1 < cz, y + 1 < cy && z + 1 < cz};
        const int up = (ci >> 6) & 1;
        for (int a = 0; a < 3; ++a) {
          if (!inside[a] || up == ((ci >> lower[a]) & 1)) continue;
          int q[4];
          for (int j = 0; j < 4; ++j) {
            const unsigned char *c = QUAD[a][j];
            const int64_t nb = ((int64_t)(z + c[2]) * cy + (y + c[1])) * cx + (x + c[0]);
            q[j] = base[nb] + r3g_mc_dual_patch[12 * tils[nb] + c[3]];
          }
          if (!up) {       /* the lower end is above: reverse the turn */
            const int t = q[1];
            q[1] = q[3];
            q[3] = t;
          }
          if (dist2(m.v, q[1], q[3]) < dist2(m.v, q[0], q[2])) {
            push_face(&m, q[0], q[1], q[3]);
            push_face(&m, q[1], q[2], q[3]);
          } else {
            push_face(&m, q[0], q[1], q[2]);
            push_face(&m, q[0], q[2], q[3]);
          }
        }
      }
  free(base);
  free(tils);
  free(cis);
  if (m.nv == 0) {
    free(m.v);
    free(m.f);
    free(cells);
    return 2;
  }
  *verts_out = m.v;
  *faces_out = m.f;
  *nv_out = m.nv;
  *nf_out = m.nf;
  if (cells_out) *cells_out = cells;
  return 0;
}
