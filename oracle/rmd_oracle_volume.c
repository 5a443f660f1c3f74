/* rmd_oracle_volume.c -- CPU restatement of the TSDF volume (csrc/volume.cuh, DESIGN.md 4.8): integration of a
 * depth image, surface-point extraction, raycasting, and the host pose inverse the raycast starts from.
 *
 * TEST INFRASTRUCTURE ONLY (see rmd_oracle.h).  The reference has no such step, so nothing pins this file to it;
 * tests/test_volume_oracle.py pins it against an independent numpy float32 evaluation and known answers instead.
 * One IEEE float operation per C operator (built with -ffp-contract=off), in the order of the kernels'
 * __f*_rn intrinsics.  Built on its own into librmd_oracle_volume.so by tests/volume_oracle.py, which also
 * binds it.
 *
 * Grids: tsdf and weight are nx * ny * nz floats each, x fastest; origin = centre of voxel (0, 0, 0).
 * Images: dense row-major.  Poses: 3x4 row-major.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#define RMDO_CONVERGED 1

static float voxel_coord(float origin, int i, float s) { return origin + (float)i * s; }

/* c_api.cu's pose_inverse (host code, no contraction) */
void rmd_oracle_pose_inverse(const float *d, float *r) {
  r[0] = d[0]; r[1] = d[4]; r[2] = d[8];
  r[4] = d[1]; r[5] = d[5]; r[6] = d[9];
  r[8] = d[2]; r[9] = d[6]; r[10] = d[10];
  r[3] = -d[0] * d[3] - d[4] * d[7] - d[8] * d[11];
  r[7] = -d[1] * d[3] - d[5] * d[7] - d[9] * d[11];
  r[11] = -d[2] * d[3] - d[6] * d[7] - d[10] * d[11];
}

/* Integrate one depth image; conv may be NULL (every pixel counts).  Returns the number of updated voxels. */
size_t rmd_oracle_volume_integrate(float *tsdf, float *weight, int nx, int ny, int nz, float s, const float *origin,
                                   int w, int h, float fx, float fy, float cx, float cy, const float *T,
                                   const float *depth, const int *conv, float trunc, float max_weight) {
  size_t updated = 0;
  for (int k = 0; k < nz; ++k) {
    for (int j = 0; j < ny; ++j) {
      for (int i = 0; i < nx; ++i) {
        const float wx = voxel_coord(origin[0], i, s), wy = voxel_coord(origin[1], j, s),
                    wz = voxel_coord(origin[2], k, s);
        const float px = T[0] * wx + T[1] * wy + T[2] * wz + T[3];
        const float py = T[4] * wx + T[5] * wy + T[6] * wz + T[7];
        const float pz = T[8] * wx + T[9] * wy + T[10] * wz + T[11];
        if (!(pz > 0.0f))
          continue;
        const float u = fx * px / pz + cx, v = fy * py / pz + cy;
        const float tu = floorf(u + 0.5f), tv = floorf(v + 0.5f);
        if (!(tu >= 0.0f && tu < (float)w && tv >= 0.0f && tv < (float)h))
          continue;
        const size_t pix = (size_t)(int)tv * w + (int)tu;
        if (conv && conv[pix] != RMDO_CONVERGED)
          continue;
        const float d = depth[pix];
        if (!(d > 0.0f) || !isfinite(d))
          continue;
        const float r = sqrtf(px * px + py * py + pz * pz);
        const float sdf = d - r;
        if (!(sdf >= -trunc))
          continue;
        const float o = fminf(1.0f, sdf / trunc);
        const size_t lin = ((size_t)k * ny + j) * nx + i;
        const float w1 = weight[lin] + 1.0f;
        tsdf[lin] = (tsdf[lin] * weight[lin] + o) / w1;
        weight[lin] = fminf(w1, max_weight);
        ++updated;
      }
    }
  }
  return updated;
}

static int near_surface(float t, float w) { return w > 0.0f && fabsf(t) < 1.0f; }

/* Surface points (x, y, z, w) in voxel order, then axis x, y, z; writes at most `capacity`, returns the count. */
size_t rmd_oracle_volume_surface(const float *tsdf, const float *weight, int nx, int ny, int nz, float s,
                                 const float *origin, float *out, size_t capacity) {
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
          const float tb = tsdf[a + step[axis]], wb = weight[a + step[axis]];
          if (!near_surface(tb, wb) || !((ta > 0.0f && tb <= 0.0f) || (ta <= 0.0f && tb > 0.0f)))
            continue;
          if (n < capacity) {
            float p[3] = {voxel_coord(origin[0], i, s), voxel_coord(origin[1], j, s), voxel_coord(origin[2], k, s)};
            p[axis] = p[axis] + ta / (ta - tb) * s;
            out[4 * n + 0] = p[0];
            out[4 * n + 1] = p[1];
            out[4 * n + 2] = p[2];
            out[4 * n + 3] = fminf(wa, wb);
          }
          ++n;
        }
      }
    }
  }
  return n;
}

static float lerp(float a, float b, float f) { return a + f * (b - a); }

static int sample_tsdf(const float *tsdf, const float *weight, int nx, int ny, int nz, float gx, float gy, float gz,
                       float *out) {
  const float x0 = floorf(gx), y0 = floorf(gy), z0 = floorf(gz);
  const int i0 = (x0 >= 0.0f && x0 < 2.0e9f) ? (int)x0 : -1;
  const int j0 = (y0 >= 0.0f && y0 < 2.0e9f) ? (int)y0 : -1;
  const int k0 = (z0 >= 0.0f && z0 < 2.0e9f) ? (int)z0 : -1;
  if (i0 < 0 || j0 < 0 || k0 < 0 || i0 + 1 >= nx || j0 + 1 >= ny || k0 + 1 >= nz)
    return 0;
  const size_t plane = (size_t)nx * ny, b = ((size_t)k0 * ny + j0) * nx + i0;
  const size_t c[8] = {b, b + 1, b + nx, b + nx + 1, b + plane, b + plane + 1, b + plane + nx, b + plane + nx + 1};
  for (int q = 0; q < 8; ++q)
    if (weight[c[q]] == 0.0f)
      return 0;
  const float fx = gx - x0, fy = gy - y0, fz = gz - z0;
  const float c00 = lerp(tsdf[c[0]], tsdf[c[1]], fx), c10 = lerp(tsdf[c[2]], tsdf[c[3]], fx);
  const float c01 = lerp(tsdf[c[4]], tsdf[c[5]], fx), c11 = lerp(tsdf[c[6]], tsdf[c[7]], fx);
  *out = lerp(lerp(c00, c10, fy), lerp(c01, c11, fy), fz);
  return 1;
}

/* Raycast: depth (w x h) = distance along each pixel's ray to the first zero crossing, 0 where none. */
void rmd_oracle_volume_raycast(const float *tsdf, const float *weight, int nx, int ny, int nz, float s,
                               const float *origin, int w, int h, float fx, float fy, float cx, float cy,
                               const float *T_curr_world, float *depth) {
  float T[12];
  rmd_oracle_pose_inverse(T_curr_world, T);
  const int n[3] = {nx, ny, nz};
  for (int y = 0; y < h; ++y) {
    for (int x = 0; x < w; ++x) {
      const float vx = ((float)x - cx) / fx, vy = ((float)y - cy) / fy;
      const float inv_len = 1.0f / sqrtf(vx * vx + vy * vy + 1.0f);
      const float qx = vx * inv_len, qy = vy * inv_len, qz = 1.0f * inv_len;
      const float dir[3] = {T[0] * qx + T[1] * qy + T[2] * qz, T[4] * qx + T[5] * qy + T[6] * qz,
                            T[8] * qx + T[9] * qy + T[10] * qz};
      const float org[3] = {T[3], T[7], T[11]};
      float t0 = 0.0f, t1 = INFINITY;
      int inside = 1;
      for (int a = 0; a < 3; ++a) {
        const float hi = voxel_coord(origin[a], n[a] - 1, s);
        if (dir[a] == 0.0f) {
          inside = inside && org[a] >= origin[a] && org[a] <= hi;
          continue;
        }
        const float ta = (origin[a] - org[a]) / dir[a], tb = (hi - org[a]) / dir[a];
        t0 = fmaxf(t0, fminf(ta, tb));
        t1 = fminf(t1, fmaxf(ta, tb));
      }
      float out = 0.0f;
      if (inside && t0 <= t1) {
        const int k_max = nx + ny + nz;
        int prev_known = 0;
        float t_prev = 0.0f, f_prev = 0.0f;
        for (int k = 0; k <= k_max; ++k) {
          const float t = t0 + (float)k * s;
          if (!(t <= t1))
            break;
          const float gx = (org[0] + t * dir[0] - origin[0]) / s;
          const float gy = (org[1] + t * dir[1] - origin[1]) / s;
          const float gz = (org[2] + t * dir[2] - origin[2]) / s;
          float f = 0.0f;
          const int known = sample_tsdf(tsdf, weight, nx, ny, nz, gx, gy, gz, &f);
          if (known && prev_known && f_prev > 0.0f && f <= 0.0f) {
            out = t_prev + s * f_prev / (f_prev - f);
            break;
          }
          prev_known = known;
          t_prev = t;
          f_prev = f;
        }
      }
      depth[(size_t)y * w + x] = out;
    }
  }
}
