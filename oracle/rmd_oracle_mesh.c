/* rmd_oracle_mesh.c -- CPU restatement of the TSDF volume's triangle mesh (csrc/volume.cu volume_mesh_*,
 * DESIGN.md 4.8): marching cubes over the generated case table, with the surface points of rmd_oracle_volume.c as
 * its vertices.
 *
 * TEST INFRASTRUCTURE ONLY (see rmd_oracle.h).  The reference has no such step; tests/test_volume_mesh_oracle.py
 * pins this file by known answers (plane, analytic sphere) and by properties (watertightness on random sign fields,
 * the rules for unknown and truncated voxels).  Built together with rmd_oracle_volume.c into librmd_oracle_mesh.so
 * by tests/mesh_oracle.py, which also binds it.  Nothing here is floating-point arithmetic: the vertices are the
 * surface points, and a triangle is three of their ranks.
 *
 * Grids: tsdf and weight are nx * ny * nz floats each, x fastest; origin = centre of voxel (0, 0, 0).
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

#include "../rpg_open_remode_b200/csrc/mc_table.h"   /* the case table the kernels use (generated) */

size_t rmd_oracle_volume_surface(const float *tsdf, const float *weight, int nx, int ny, int nz, float s,
                                 const float *origin, float *out, size_t capacity);

/* the surface-point rule of rmd_oracle_volume_surface: both ends known and |tsdf| < 1, signs differ */
static int near_surface(float t, float w) { return w > 0.0f && fabsf(t) < 1.0f; }

static int is_point(float ta, float wa, float tb, float wb) {
  return near_surface(ta, wa) && near_surface(tb, wb) && ((ta > 0.0f && tb <= 0.0f) || (ta <= 0.0f && tb > 0.0f));
}

/* Points of voxel (i, j, k) on the axes below `axis` (a voxel's points follow in axis order). */
static int points_before(const float *tsdf, const float *weight, int nx, int ny, int nz, int i, int j, int k,
                         int axis) {
  const size_t plane = (size_t)nx * ny, a = ((size_t)k * ny + j) * nx + i;
  const int inside[3] = {i + 1 < nx, j + 1 < ny, k + 1 < nz};
  const size_t step[3] = {1, (size_t)nx, plane};
  int n = 0;
  for (int b = 0; b < axis; ++b)
    n += inside[b] && is_point(tsdf[a], weight[a], tsdf[a + step[b]], weight[a + step[b]]);
  return n;
}

/* Rank of the first surface point of every voxel of plane k, into rank (nx * ny entries); returns the running
 * count of points after the plane. */
static size_t plane_ranks(const float *tsdf, const float *weight, int nx, int ny, int nz, int k, size_t n,
                          uint64_t *rank) {
  for (int j = 0; j < ny; ++j) {
    for (int i = 0; i < nx; ++i) {
      rank[(size_t)j * nx + i] = n;
      n += (size_t)points_before(tsdf, weight, nx, ny, nz, i, j, k, 3);
    }
  }
  return n;
}

/* Marching-cubes mesh (DESIGN.md 4.8).  Its vertices are the surface points (rmd_oracle_volume_surface, at most
 * vertex_capacity written); *n_vertices is their count.  Triangles: 3 int32 vertex indices each, ordered by cube,
 * then table order; at most tri_capacity written; returns their count (0 with *n_vertices unchanged if the rank map
 * cannot be allocated).  Cube (i, j, k) < (nx - 1, ny - 1, nz - 1) is meshed only when its 8 corners have weight
 * > 0 and every edge whose ends differ in sign (inside = tsdf <= 0) has |tsdf| < 1 at both ends.  A vertex index
 * is the rank of the edge's surface point, read from a rank map of the two planes the cube touches. */
size_t rmd_oracle_volume_mesh(const float *tsdf, const float *weight, int nx, int ny, int nz, float s,
                              const float *origin, float *xyzw, size_t vertex_capacity, int32_t *tri,
                              size_t tri_capacity, size_t *n_vertices) {
  const size_t plane = (size_t)nx * ny;
  uint64_t *rank = (uint64_t *)malloc(sizeof(uint64_t) * 2 * plane);
  if (!rank)
    return 0;
  *n_vertices = rmd_oracle_volume_surface(tsdf, weight, nx, ny, nz, s, origin, xyzw, vertex_capacity);
  size_t n_pts = 0, m = 0;
  if (nz > 1)
    n_pts = plane_ranks(tsdf, weight, nx, ny, nz, 0, n_pts, rank);
  for (int k = 0; k + 1 < nz; ++k) {
    n_pts = plane_ranks(tsdf, weight, nx, ny, nz, k + 1, n_pts, rank + (size_t)((k + 1) & 1) * plane);
    for (int j = 0; j + 1 < ny; ++j) {
      for (int i = 0; i + 1 < nx; ++i) {
        const size_t n = ((size_t)k * ny + j) * nx + i;
        float t[8];
        int known = 1, cube = 0;
        for (int c = 0; c < 8; ++c) {
          const size_t v = n + (c & 1) + ((c >> 1) & 1) * (size_t)nx + ((c >> 2) & 1) * plane;
          t[c] = tsdf[v];
          known = known && weight[v] > 0.0f;
          cube |= (t[c] <= 0.0f) << c;
        }
        if (!known || cube == 0 || cube == 255)
          continue;
        int ok = 1;
        for (int e = 0; e < 12; ++e) {
          const int c0 = RMD_MC_EDGE[e][0], c1 = c0 + (1 << RMD_MC_EDGE[e][1]);
          if (((cube >> c0) ^ (cube >> c1)) & 1)
            ok = ok && fabsf(t[c0]) < 1.0f && fabsf(t[c1]) < 1.0f;
        }
        if (!ok)
          continue;
        for (int q = 0; q < RMD_MC_NTRI[cube]; ++q, ++m) {
          for (int r = 0; r < 3 && m < tri_capacity; ++r) {
            const int e = RMD_MC_TRIS[cube][3 * q + r];
            const int c0 = RMD_MC_EDGE[e][0], axis = RMD_MC_EDGE[e][1];
            const int di = c0 & 1, dj = (c0 >> 1) & 1, dk = (c0 >> 2) & 1;
            const uint64_t *rk = rank + (size_t)((k + dk) & 1) * plane;   /* the plane of the edge's lower voxel */
            const uint64_t idx = rk[(size_t)(j + dj) * nx + (i + di)] +
                                 (uint64_t)points_before(tsdf, weight, nx, ny, nz, i + di, j + dj, k + dk, axis);
            tri[3 * m + r] = (int32_t)idx;
          }
        }
      }
    }
  }
  free(rank);
  return m;
}
