/* rmd_oracle_volume_normals.c -- CPU restatement of the TSDF volume's normals (csrc/volume.cu: the NORMALS surface
 * write instance and volume_raycast_normals_kernel; DESIGN.md 4.8): the per-voxel tsdf gradient, the surface points'
 * normals and the normal at each raycast hit.
 *
 * TEST INFRASTRUCTURE ONLY (see rmd_oracle.h).  The reference has no such step; tests/test_volume_normals_oracle.py
 * pins this file against an independent numpy float32 evaluation and known answers.  One IEEE float operation per
 * C operator (built with -ffp-contract=off), in the order of the kernels' __f*_rn intrinsics.  Built together with
 * rmd_oracle_volume.c (whose raycast gives the hits) into librmd_oracle_volume_normals.so by
 * tests/volume_normals_oracle.py, which also binds it.
 *
 * Grids: tsdf and weight are nx * ny * nz floats each, x fastest; origin = centre of voxel (0, 0, 0).  Images: dense
 * row-major.  Poses: 3x4 row-major.  Normals: 4 floats (nx, ny, nz, 0) each.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

void rmd_oracle_pose_inverse(const float *d, float *r);
void rmd_oracle_volume_raycast(const float *tsdf, const float *weight, int nx, int ny, int nz, float s,
                               const float *origin, int w, int h, float fx, float fy, float cx, float cy,
                               const float *T_curr_world, float *depth);

static float lerp(float a, float b, float f) { return a + f * (b - a); }

/* One gradient component of voxel n (tsdf t0) along an axis of index step `step`: neighbour n - step exists when
 * dn, n + step when up; a neighbour is usable when it exists and has weight > 0. */
static float gradient_component(const float *tsdf, const float *weight, size_t n, size_t step, int dn, int up,
                                float t0) {
  const int um = dn && weight[n - step] > 0.0f, upk = up && weight[n + step] > 0.0f;
  if (um && upk)
    return (tsdf[n + step] - tsdf[n - step]) * 0.5f;
  if (upk)
    return tsdf[n + step] - t0;
  if (um)
    return t0 - tsdf[n - step];
  return 0.0f;
}

/* The tsdf gradient of voxel (i, j, k) into g[3]. */
static void voxel_gradient(const float *tsdf, const float *weight, int nx, int ny, int nz, int i, int j, int k,
                           float *g) {
  const size_t sy = (size_t)nx, sz = (size_t)nx * ny;
  const size_t n = (size_t)k * sz + (size_t)j * sy + (size_t)i;
  const float t0 = tsdf[n];
  g[0] = gradient_component(tsdf, weight, n, 1, i > 0, i + 1 < nx, t0);
  g[1] = gradient_component(tsdf, weight, n, sy, j > 0, j + 1 < ny, t0);
  g[2] = gradient_component(tsdf, weight, n, sz, k > 0, k + 1 < nz, t0);
}

/* out[4] = (g / len, 0), len = sqrt((gx^2 + gy^2) + gz^2); (0, 0, 0, 0) when len is 0 or not finite. */
static void unit_normal(const float *g, float *out) {
  const float len = sqrtf(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
  out[3] = 0.0f;
  if (!(len > 0.0f) || !isfinite(len)) {
    out[0] = out[1] = out[2] = 0.0f;
    return;
  }
  out[0] = g[0] / len;
  out[1] = g[1] / len;
  out[2] = g[2] / len;
}

/* Every voxel's gradient, 3 floats per voxel in voxel order (a known voxel's gradient; the rule is evaluated for
 * unknown voxels too). */
void rmd_oracle_volume_gradients(const float *tsdf, const float *weight, int nx, int ny, int nz, float *out) {
  size_t n = 0;
  for (int k = 0; k < nz; ++k)
    for (int j = 0; j < ny; ++j)
      for (int i = 0; i < nx; ++i, ++n)
        voxel_gradient(tsdf, weight, nx, ny, nz, i, j, k, out + 3 * n);
}

static int near_surface(float t, float w) { return w > 0.0f && fabsf(t) < 1.0f; }

/* One normal per surface point, in rmd_oracle_volume_surface's order; writes at most `capacity`, returns the
 * count. */
size_t rmd_oracle_volume_surface_normals(const float *tsdf, const float *weight, int nx, int ny, int nz, float *out,
                                         size_t capacity) {
  size_t n = 0;
  const size_t plane = (size_t)nx * ny;
  for (int k = 0; k < nz; ++k) {
    for (int j = 0; j < ny; ++j) {
      for (int i = 0; i < nx; ++i) {
        const size_t a = ((size_t)k * ny + j) * nx + i;
        const float ta = tsdf[a], wa = weight[a];
        if (!near_surface(ta, wa))
          continue;
        const int inside[3] = {i + 1 < nx, j + 1 < ny, k + 1 < nz};
        const size_t step[3] = {1, (size_t)nx, plane};
        for (int axis = 0; axis < 3; ++axis) {
          if (!inside[axis])
            continue;
          const size_t b = a + step[axis];
          const float tb = tsdf[b];
          if (!near_surface(tb, weight[b]) || !((ta > 0.0f && tb <= 0.0f) || (ta <= 0.0f && tb > 0.0f)))
            continue;
          if (n < capacity) {
            float ga[3], gb[3], g[3];
            voxel_gradient(tsdf, weight, nx, ny, nz, i, j, k, ga);
            voxel_gradient(tsdf, weight, nx, ny, nz, i + (axis == 0), j + (axis == 1), k + (axis == 2), gb);
            const float f = ta / (ta - tb);
            for (int c = 0; c < 3; ++c)
              g[c] = lerp(ga[c], gb[c], f);
            unit_normal(g, out + 4 * n);
          }
          ++n;
        }
      }
    }
  }
  return n;
}

/* The normal at grid coordinates (gx, gy, gz) into out[4]: trilinear x, then y, then z of the 8 corner gradients,
 * normalised; (0, 0, 0, 0) if a corner lies outside the grid or has weight 0. */
static void sample_normal(const float *tsdf, const float *weight, int nx, int ny, int nz, float gx, float gy,
                          float gz, float *out) {
  out[0] = out[1] = out[2] = out[3] = 0.0f;
  const float x0 = floorf(gx), y0 = floorf(gy), z0 = floorf(gz);
  const int i0 = (x0 >= 0.0f && x0 < 2.0e9f) ? (int)x0 : -1;
  const int j0 = (y0 >= 0.0f && y0 < 2.0e9f) ? (int)y0 : -1;
  const int k0 = (z0 >= 0.0f && z0 < 2.0e9f) ? (int)z0 : -1;
  if (i0 < 0 || j0 < 0 || k0 < 0 || i0 + 1 >= nx || j0 + 1 >= ny || k0 + 1 >= nz)
    return;
  float c[8][3];
  for (int q = 0; q < 8; ++q) {   /* corner q = dx + 2 dy + 4 dz */
    const int i = i0 + (q & 1), j = j0 + ((q >> 1) & 1), k = k0 + ((q >> 2) & 1);
    if (weight[((size_t)k * ny + j) * nx + i] == 0.0f)
      return;
    voxel_gradient(tsdf, weight, nx, ny, nz, i, j, k, c[q]);
  }
  const float fx = gx - x0, fy = gy - y0, fz = gz - z0;
  float g[3];
  for (int a = 0; a < 3; ++a) {
    const float c00 = lerp(c[0][a], c[1][a], fx), c10 = lerp(c[2][a], c[3][a], fx);
    const float c01 = lerp(c[4][a], c[5][a], fx), c11 = lerp(c[6][a], c[7][a], fx);
    g[a] = lerp(lerp(c00, c10, fy), lerp(c01, c11, fy), fz);
  }
  unit_normal(g, out);
}

/* Raycast with normals: depth (w x h) = rmd_oracle_volume_raycast's, normals (w x h x 4) = the normal at each hit
 * (depth > 0), (0, 0, 0, 0) elsewhere. */
void rmd_oracle_volume_raycast_normals(const float *tsdf, const float *weight, int nx, int ny, int nz, float s,
                                       const float *origin, int w, int h, float fx, float fy, float cx, float cy,
                                       const float *T_curr_world, float *depth, float *normals) {
  rmd_oracle_volume_raycast(tsdf, weight, nx, ny, nz, s, origin, w, h, fx, fy, cx, cy, T_curr_world, depth);
  float T[12];
  rmd_oracle_pose_inverse(T_curr_world, T);
  for (int y = 0; y < h; ++y) {
    for (int x = 0; x < w; ++x) {
      const float t = depth[(size_t)y * w + x];
      float *out = normals + 4 * ((size_t)y * w + x);
      out[0] = out[1] = out[2] = out[3] = 0.0f;
      if (t > 0.0f) {
        /* the ray of rmd_oracle_volume_raycast */
        const float vx = ((float)x - cx) / fx, vy = ((float)y - cy) / fy;
        const float inv_len = 1.0f / sqrtf(vx * vx + vy * vy + 1.0f);
        const float qx = vx * inv_len, qy = vy * inv_len, qz = 1.0f * inv_len;
        const float dir[3] = {T[0] * qx + T[1] * qy + T[2] * qz, T[4] * qx + T[5] * qy + T[6] * qz,
                              T[8] * qx + T[9] * qy + T[10] * qz};
        const float org[3] = {T[3], T[7], T[11]};
        sample_normal(tsdf, weight, nx, ny, nz, (org[0] + t * dir[0] - origin[0]) / s,
                      (org[1] + t * dir[1] - origin[1]) / s, (org[2] + t * dir[2] - origin[2]) / s, out);
      }
    }
  }
}
