/* rmd_oracle_volume_shift.c -- CPU restatement of the moving TSDF volume (csrc/volume.cu: volume_shift_kernel and
 * the spill instances of the surface passes; csrc/volume_api.cu: rmd_volume_shift's origin; DESIGN.md 4.8).
 *
 * TEST INFRASTRUCTURE ONLY (see rmd_oracle.h).  The reference has no such step; tests/test_volume_shift_oracle.py
 * pins this file against an independent numpy evaluation.  The spill reuses the surface code of
 * rmd_oracle_volume.c, rmd_oracle_volume_intensity.c and rmd_oracle_volume_normals.c (it filters their outputs), so
 * it is built together with them (same flags: IEEE fp32, no contraction) into librmd_oracle_volume_shift.so by
 * tests/volume_shift_oracle.py, which also binds it.
 *
 * Grids: nx * ny * nz floats per record half, x fastest; origin = centre of voxel (0, 0, 0).
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

size_t rmd_oracle_volume_surface(const float *tsdf, const float *weight, int nx, int ny, int nz, float s,
                                 const float *origin, float *out, size_t capacity);
size_t rmd_oracle_volume_surface_intensity(const float *tsdf, const float *weight, const float *cint, const float *cw,
                                           int nx, int ny, int nz, float *out, size_t capacity);
size_t rmd_oracle_volume_surface_normals(const float *tsdf, const float *weight, int nx, int ny, int nz, float *out,
                                         size_t capacity);

/* One record half (a, b) of a shift by d into (a_out, b_out): voxel (i, j, k) takes voxel (i + dx, j + dy, k + dz),
 * or 0 where that lies outside the grid. */
void rmd_oracle_volume_shift(const float *a, const float *b, float *a_out, float *b_out, int nx, int ny, int nz,
                             const int *d) {
  size_t n = 0;
  for (int k = 0; k < nz; ++k)
    for (int j = 0; j < ny; ++j)
      for (int i = 0; i < nx; ++i, ++n) {
        const long long si = (long long)i + d[0], sj = (long long)j + d[1], sk = (long long)k + d[2];
        if (si >= 0 && si < nx && sj >= 0 && sj < ny && sk >= 0 && sk < nz) {
          const size_t src = ((size_t)sk * ny + (size_t)sj) * nx + (size_t)si;
          a_out[n] = a[src];
          b_out[n] = b[src];
        } else {
          a_out[n] = 0.0f;
          b_out[n] = 0.0f;
        }
      }
}

/* The origin after shifts totalling D: o0 + (float)D * s per axis, one rounding per operation. */
void rmd_oracle_volume_shift_origin(const float *o0, const long long *D, float s, float *out) {
  for (int a = 0; a < 3; ++a)
    out[a] = o0[a] + (float)D[a] * s;
}

static int near_surface(float t, float w) { return w > 0.0f && fabsf(t) < 1.0f; }

/* 1 for each surface point (rmd_oracle_volume_surface's order) that a shift by d drops: its voxel a or neighbour
 * b = a + e_axis lies outside the kept box [max(0, d), min(n, n + d)) on some axis.  Returns the point count. */
static size_t spill_flags(const float *tsdf, const float *weight, int nx, int ny, int nz, const int *d,
                          unsigned char *flags) {
  const long long n3[3] = {nx, ny, nz};
  long long lo[3], hi[3];
  for (int a = 0; a < 3; ++a) {
    lo[a] = d[a] > 0 ? d[a] : 0;
    hi[a] = d[a] < 0 ? n3[a] + d[a] : n3[a];
  }
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
          int spills = 0;
          for (int c = 0; c < 3; ++c) {
            const long long pa = p[c], pb = p[c] + (c == axis);
            spills = spills || pa < lo[c] || pa >= hi[c] || pb < lo[c] || pb >= hi[c];
          }
          if (flags)
            flags[n] = (unsigned char)spills;
          ++n;
        }
      }
  return n;
}

/* The spill of a shift by d: kind 0 = points (4 floats each), 1 = intensities (1 float; cint / cw needed),
 * 2 = normals (4 floats), as the subsequence of the current grid's surface output.  Writes at most `capacity`,
 * returns the count (or (size_t)-1 when out of memory). */
size_t rmd_oracle_volume_spill(const float *tsdf, const float *weight, const float *cint, const float *cw, int nx,
                               int ny, int nz, float s, const float *origin, const int *d, int kind, float *out,
                               size_t capacity) {
  const size_t total = spill_flags(tsdf, weight, nx, ny, nz, d, NULL);
  const size_t per = kind == 1 ? 1 : 4;
  unsigned char *flags = malloc(total ? total : 1);
  float *all = malloc(sizeof(float) * per * (total ? total : 1));
  if (!flags || !all) {
    free(flags);
    free(all);
    return (size_t)-1;
  }
  spill_flags(tsdf, weight, nx, ny, nz, d, flags);
  if (kind == 0)
    rmd_oracle_volume_surface(tsdf, weight, nx, ny, nz, s, origin, all, total);
  else if (kind == 1)
    rmd_oracle_volume_surface_intensity(tsdf, weight, cint, cw, nx, ny, nz, all, total);
  else
    rmd_oracle_volume_surface_normals(tsdf, weight, nx, ny, nz, all, total);
  size_t m = 0;
  for (size_t q = 0; q < total; ++q) {
    if (!flags[q])
      continue;
    if (m < capacity)
      for (size_t c = 0; c < per; ++c)
        out[per * m + c] = all[per * q + c];
    ++m;
  }
  free(flags);
  free(all);
  return m;
}
