/* rmd_oracle_volume_spill_mesh.c -- CPU restatement of the spill mesh of a moving TSDF volume (csrc/volume.cu:
 * volume_spill_mesh_* and volume_spill_tri_*; csrc/volume_api.cu: rmd_volume_spill_mesh; DESIGN.md 4.8).
 *
 * TEST INFRASTRUCTURE ONLY (see rmd_oracle.h).  The reference has no such step; tests/test_volume_spill_mesh_oracle.py
 * pins this file against an independent numpy evaluation.  It filters the outputs of rmd_oracle_volume_mesh (and of
 * the surface, intensity and normals oracles) the way rmd_oracle_volume_shift.c filters the surface outputs: a flag per
 * surface point for the spill mesh's vertices, a flag per triangle for its cube, then the triangles' indices remapped.
 * Built together with rmd_oracle_volume.c, rmd_oracle_volume_intensity.c, rmd_oracle_volume_normals.c,
 * rmd_oracle_mesh.c and rmd_oracle_volume_shift.c (same flags: IEEE fp32, no contraction) into
 * librmd_oracle_volume_spill_mesh.so by tests/spill_mesh_oracle.py, which also binds it.
 *
 * Grids: nx * ny * nz floats per record half, x fastest; origin = centre of voxel (0, 0, 0).
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

#include "../rpg_open_remode_b200/csrc/mc_table.h"   /* the case table the kernels use (generated) */

size_t rmd_oracle_volume_surface(const float *tsdf, const float *weight, int nx, int ny, int nz, float s,
                                 const float *origin, float *out, size_t capacity);
size_t rmd_oracle_volume_surface_intensity(const float *tsdf, const float *weight, const float *cint, const float *cw,
                                           int nx, int ny, int nz, float *out, size_t capacity);
size_t rmd_oracle_volume_surface_normals(const float *tsdf, const float *weight, int nx, int ny, int nz, float *out,
                                         size_t capacity);
size_t rmd_oracle_volume_mesh(const float *tsdf, const float *weight, int nx, int ny, int nz, float s,
                              const float *origin, float *xyzw, size_t vertex_capacity, int32_t *tri,
                              size_t tri_capacity, size_t *n_vertices);

static int near_surface(float t, float w) { return w > 0.0f && fabsf(t) < 1.0f; }

/* Case of cube (i, j, k) (corner c at + (c & 1, c >> 1 & 1, c >> 2 & 1), bit c = tsdf <= 0) when it is meshed: a
 * valid cube, 8 known corners, not all on one side, and no crossing edge with |tsdf| >= 1 at an end; else 0. */
static int cube_case(const float *tsdf, const float *weight, int nx, int ny, int nz, long long i, long long j,
                     long long k) {
  if (i < 0 || j < 0 || k < 0 || i + 1 >= nx || j + 1 >= ny || k + 1 >= nz)
    return 0;
  const size_t plane = (size_t)nx * ny, n = ((size_t)k * ny + (size_t)j) * nx + (size_t)i;
  float t[8];
  int cube = 0;
  for (int c = 0; c < 8; ++c) {
    const size_t v = n + (c & 1) + ((c >> 1) & 1) * (size_t)nx + ((c >> 2) & 1) * plane;
    if (!(weight[v] > 0.0f))
      return 0;
    t[c] = tsdf[v];
    cube |= (t[c] <= 0.0f) << c;
  }
  if (cube == 0 || cube == 255)
    return 0;
  for (int e = 0; e < 12; ++e) {
    const int c0 = RMD_MC_EDGE[e][0], c1 = c0 + (1 << RMD_MC_EDGE[e][1]);
    if ((((cube >> c0) ^ (cube >> c1)) & 1) && !(fabsf(t[c0]) < 1.0f && fabsf(t[c1]) < 1.0f))
      return 0;
  }
  return cube;
}

/* Whether cube (i, j, k) has a corner outside the kept box [lo, hi). */
static int cube_leaves(const long long *lo, const long long *hi, long long i, long long j, long long k) {
  const long long p[3] = {i, j, k};
  for (int a = 0; a < 3; ++a)
    if (p[a] < lo[a] || p[a] + 1 >= hi[a])
      return 1;
  return 0;
}

/* Per surface point (rmd_oracle_volume_surface's order): 1 when it is a vertex of the spill mesh -- voxel a or
 * b = a + e_axis lies outside K, or one of the <= 4 cubes of edge (a, axis) is meshed and has a corner outside K --
 * and its key 3 * voxel + axis.  Returns the point count. */
static size_t vertex_flags(const float *tsdf, const float *weight, int nx, int ny, int nz, const long long *lo,
                           const long long *hi, unsigned char *flags, int64_t *keys) {
  size_t n = 0;
  const size_t plane = (size_t)nx * ny;
  for (int k = 0; k < nz; ++k)
    for (int j = 0; j < ny; ++j)
      for (int i = 0; i < nx; ++i) {
        const size_t a = ((size_t)k * ny + j) * nx + i;
        const float ta = tsdf[a];
        if (!near_surface(ta, weight[a]))
          continue;
        const int p[3] = {i, j, k};
        const int inside[3] = {i + 1 < nx, j + 1 < ny, k + 1 < nz};
        const size_t step[3] = {1, (size_t)nx, plane};
        for (int axis = 0; axis < 3; ++axis) {
          if (!inside[axis])
            continue;
          const float tb = tsdf[a + step[axis]];
          if (!near_surface(tb, weight[a + step[axis]]) || !((ta > 0.0f && tb <= 0.0f) || (ta <= 0.0f && tb > 0.0f)))
            continue;
          int in = 1;
          for (int c = 0; c < 3; ++c) {
            const long long pa = p[c], pb = p[c] + (c == axis);
            in = in && pa >= lo[c] && pa < hi[c] && pb >= lo[c] && pb < hi[c];
          }
          int vertex = !in;
          const int u = axis == 0 ? 1 : 0, w = axis == 2 ? 1 : 2;
          for (int q = 0; q < 4 && !vertex; ++q) {
            long long c[3] = {i, j, k};
            c[u] -= q & 1;
            c[w] -= q >> 1;
            vertex = cube_leaves(lo, hi, c[0], c[1], c[2]) && cube_case(tsdf, weight, nx, ny, nz, c[0], c[1], c[2]);
          }
          flags[n] = (unsigned char)vertex;
          keys[n] = 3 * (int64_t)a + axis;
          ++n;
        }
      }
  return n;
}

/* The spill mesh of a shift by d.  Vertices: kind 0 = positions (4 floats each), 1 = intensities (1 float; cint / cw
 * needed), 2 = normals (4 floats), as the subsequence of the surface output, at most vertex_capacity of them into out
 * and their keys 3 * voxel + axis into keys (may be NULL); *n_vertices = their count.  Triangles: the mesh's
 * triangles (3 int32 each, its order) of the cubes that have a corner outside K, their indices remapped into the
 * vertices, at most tri_capacity into tri.  Returns the triangle count, or (size_t)-1 when out of memory or when the
 * mesh's triangles do not match the cube rule. */
size_t rmd_oracle_volume_spill_mesh(const float *tsdf, const float *weight, const float *cint, const float *cw, int nx,
                                    int ny, int nz, float s, const float *origin, const int *d, int kind, float *out,
                                    size_t vertex_capacity, int32_t *tri, size_t tri_capacity, int64_t *keys,
                                    size_t *n_vertices) {
  const long long n3[3] = {nx, ny, nz};
  long long lo[3], hi[3];
  for (int a = 0; a < 3; ++a) {
    lo[a] = d[a] > 0 ? d[a] : 0;
    hi[a] = d[a] < 0 ? n3[a] + d[a] : n3[a];
  }
  const size_t per = kind == 1 ? 1 : 4;
  size_t total = 0;
  const size_t n_tri = rmd_oracle_volume_mesh(tsdf, weight, nx, ny, nz, s, origin, NULL, 0, NULL, 0, &total);
  unsigned char *flags = malloc(total ? total : 1);
  int64_t *all_keys = malloc(sizeof(int64_t) * (total ? total : 1));
  int64_t *remap = malloc(sizeof(int64_t) * (total ? total : 1));
  float *all = malloc(sizeof(float) * per * (total ? total : 1));
  int32_t *all_tri = malloc(sizeof(int32_t) * 3 * (n_tri ? n_tri : 1));
  size_t result = (size_t)-1;
  if (!flags || !all_keys || !remap || !all || !all_tri)
    goto done;
  if (vertex_flags(tsdf, weight, nx, ny, nz, lo, hi, flags, all_keys) != total)
    goto done;
  if (kind == 0)
    rmd_oracle_volume_surface(tsdf, weight, nx, ny, nz, s, origin, all, total);
  else if (kind == 1)
    rmd_oracle_volume_surface_intensity(tsdf, weight, cint, cw, nx, ny, nz, all, total);
  else
    rmd_oracle_volume_surface_normals(tsdf, weight, nx, ny, nz, all, total);
  rmd_oracle_volume_mesh(tsdf, weight, nx, ny, nz, s, origin, NULL, 0, all_tri, n_tri, &total);
  size_t m = 0;
  for (size_t q = 0; q < total; ++q) {
    remap[q] = flags[q] ? (int64_t)m : -1;
    if (!flags[q])
      continue;
    if (m < vertex_capacity) {
      for (size_t c = 0; c < per; ++c)
        out[per * m + c] = all[per * q + c];
      if (keys)
        keys[m] = all_keys[q];
    }
    ++m;
  }
  *n_vertices = m;
  /* the mesh's triangles come cube by cube, RMD_MC_NTRI[case] per meshed cube */
  size_t t = 0, mt = 0;
  for (int k = 0; k + 1 < nz; ++k)
    for (int j = 0; j + 1 < ny; ++j)
      for (int i = 0; i + 1 < nx; ++i) {
        const int cube = cube_case(tsdf, weight, nx, ny, nz, i, j, k);
        const int spills = cube_leaves(lo, hi, i, j, k);
        for (int q = 0; q < RMD_MC_NTRI[cube]; ++q, ++t) {
          if (t >= n_tri)
            goto done;
          if (!spills)
            continue;
          if (mt < tri_capacity)
            for (int r = 0; r < 3; ++r) {
              const int64_t v = remap[all_tri[3 * t + r]];
              if (v < 0)   /* a vertex of a spilling cube that is not in the vertex set */
                goto done;
              tri[3 * mt + r] = (int32_t)v;
            }
          ++mt;
        }
      }
  if (t == n_tri)
    result = mt;
done:
  free(flags);
  free(all_keys);
  free(remap);
  free(all);
  free(all_tri);
  return result;
}
