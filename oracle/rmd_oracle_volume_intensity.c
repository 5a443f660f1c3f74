/* rmd_oracle_volume_intensity.c -- CPU restatement of the TSDF volume's intensity channel (csrc/volume.cu, the
 * INTENSITY instances; DESIGN.md 4.8): fusion of an intensity image, the surface points' intensities and the
 * raycast's intensity at the hit.
 *
 * TEST INFRASTRUCTURE ONLY (see rmd_oracle.h).  The reference has no such step; tests/test_volume_intensity_oracle.py
 * pins this file against an independent numpy float32 evaluation and known answers.  One IEEE float operation per
 * C operator (built with -ffp-contract=off), in the order of the kernels' __f*_rn intrinsics.  Built together with
 * rmd_oracle_volume.c (whose raycast gives the hits) into librmd_oracle_volume_intensity.so by
 * tests/volume_intensity_oracle.py, which also binds it.
 *
 * Grids: tsdf, weight, intensity and intensity weight are nx * ny * nz floats each, x fastest; origin = centre of
 * voxel (0, 0, 0).  Images: dense row-major.  Poses: 3x4 row-major.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#define RMDO_CONVERGED 1

void rmd_oracle_pose_inverse(const float *d, float *r);
void rmd_oracle_volume_raycast(const float *tsdf, const float *weight, int nx, int ny, int nz, float s,
                               const float *origin, int w, int h, float fx, float fy, float cx, float cy,
                               const float *T_curr_world, float *depth);

static float voxel_coord(float origin, int i, float s) { return origin + (float)i * s; }

static float lerp(float a, float b, float f) { return a + f * (b - a); }

/* The intensity half of one integration (rmd_oracle_volume_integrate does the tsdf half; the voxels it updates are
 * those tested here up to the band): every voxel it updates with sdf < trunc whose pixel has a finite intensity
 * averages that intensity into (cint, cw).  conv may be NULL.  Returns the number of updated colour records. */
size_t rmd_oracle_volume_integrate_intensity(float *cint, float *cw, int nx, int ny, int nz, float s,
                                             const float *origin, int w, int h, float fx, float fy, float cx, float cy,
                                             const float *T, const float *depth, const int *conv,
                                             const float *intensity, float trunc, float max_weight) {
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
        if (!(sdf >= -trunc) || !(sdf < trunc))
          continue;
        const float I = intensity[pix];
        if (!isfinite(I))
          continue;
        const size_t lin = ((size_t)k * ny + j) * nx + i;
        const float w1 = cw[lin] + 1.0f;
        cint[lin] = (cint[lin] * cw[lin] + I) / w1;
        cw[lin] = fminf(w1, max_weight);
        ++updated;
      }
    }
  }
  return updated;
}

static int near_surface(float t, float w) { return w > 0.0f && fabsf(t) < 1.0f; }

/* One intensity per surface point, in rmd_oracle_volume_surface's order; writes at most `capacity`, returns the
 * count. */
size_t rmd_oracle_volume_surface_intensity(const float *tsdf, const float *weight, const float *cint, const float *cw,
                                           int nx, int ny, int nz, float *out, size_t capacity) {
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
            float c = -1.0f;
            if (cw[a] > 0.0f && cw[b] > 0.0f)
              c = lerp(cint[a], cint[b], ta / (ta - tb));
            else if (cw[a] > 0.0f)
              c = cint[a];
            else if (cw[b] > 0.0f)
              c = cint[b];
            out[n] = c;
          }
          ++n;
        }
      }
    }
  }
  return n;
}

/* Trilinear intensity at grid coordinates (gx, gy, gz): x, then y, then z; -1 if a corner lies outside the grid or
 * has intensity weight 0. */
static float sample_intensity(const float *cint, const float *cw, int nx, int ny, int nz, float gx, float gy,
                              float gz) {
  const float x0 = floorf(gx), y0 = floorf(gy), z0 = floorf(gz);
  const int i0 = (x0 >= 0.0f && x0 < 2.0e9f) ? (int)x0 : -1;
  const int j0 = (y0 >= 0.0f && y0 < 2.0e9f) ? (int)y0 : -1;
  const int k0 = (z0 >= 0.0f && z0 < 2.0e9f) ? (int)z0 : -1;
  if (i0 < 0 || j0 < 0 || k0 < 0 || i0 + 1 >= nx || j0 + 1 >= ny || k0 + 1 >= nz)
    return -1.0f;
  const size_t plane = (size_t)nx * ny, b = ((size_t)k0 * ny + j0) * nx + i0;
  const size_t c[8] = {b, b + 1, b + nx, b + nx + 1, b + plane, b + plane + 1, b + plane + nx, b + plane + nx + 1};
  for (int q = 0; q < 8; ++q)
    if (cw[c[q]] == 0.0f)
      return -1.0f;
  const float fx = gx - x0, fy = gy - y0, fz = gz - z0;
  const float c00 = lerp(cint[c[0]], cint[c[1]], fx), c10 = lerp(cint[c[2]], cint[c[3]], fx);
  const float c01 = lerp(cint[c[4]], cint[c[5]], fx), c11 = lerp(cint[c[6]], cint[c[7]], fx);
  return lerp(lerp(c00, c10, fy), lerp(c01, c11, fy), fz);
}

/* Raycast with intensity: depth (w x h) = rmd_oracle_volume_raycast's, intensity = the intensity at each hit
 * (depth > 0: a hit's distance t_prev + s f_prev / (f_prev - f) is positive), -1 elsewhere. */
void rmd_oracle_volume_raycast_intensity(const float *tsdf, const float *weight, const float *cint, const float *cw,
                                         int nx, int ny, int nz, float s, const float *origin, int w, int h, float fx,
                                         float fy, float cx, float cy, const float *T_curr_world, float *depth,
                                         float *intensity) {
  rmd_oracle_volume_raycast(tsdf, weight, nx, ny, nz, s, origin, w, h, fx, fy, cx, cy, T_curr_world, depth);
  float T[12];
  rmd_oracle_pose_inverse(T_curr_world, T);
  for (int y = 0; y < h; ++y) {
    for (int x = 0; x < w; ++x) {
      const float t = depth[(size_t)y * w + x];
      float out = -1.0f;
      if (t > 0.0f) {
        /* the ray of rmd_oracle_volume_raycast */
        const float vx = ((float)x - cx) / fx, vy = ((float)y - cy) / fy;
        const float inv_len = 1.0f / sqrtf(vx * vx + vy * vy + 1.0f);
        const float qx = vx * inv_len, qy = vy * inv_len, qz = 1.0f * inv_len;
        const float dir[3] = {T[0] * qx + T[1] * qy + T[2] * qz, T[4] * qx + T[5] * qy + T[6] * qz,
                              T[8] * qx + T[9] * qy + T[10] * qz};
        const float org[3] = {T[3], T[7], T[11]};
        out = sample_intensity(cint, cw, nx, ny, nz, (org[0] + t * dir[0] - origin[0]) / s,
                               (org[1] + t * dir[1] - origin[1]) / s, (org[2] + t * dir[2] - origin[2]) / s);
      }
      intensity[(size_t)y * w + x] = out;
    }
  }
}
