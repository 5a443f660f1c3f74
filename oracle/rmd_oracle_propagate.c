/* rmd_oracle_propagate.c -- CPU restatement of the keyframe depth prior (csrc/prior.cuh, DESIGN.md 4.7):
 * splat a source keyframe's CONVERGED seeds into a new reference view, initialise the new keyframe, apply
 * the splatted depths as its prior.
 *
 * TEST INFRASTRUCTURE ONLY (see rmd_oracle.h).  The reference has no such step, so nothing pins this file to
 * it; tests/test_prior_propagation.py pins it against an independent numpy float32 evaluation and known
 * answers instead.  One IEEE float operation per C operator (built with -ffp-contract=off), in the order of
 * the kernels' __f*_rn intrinsics; the back-projection is the one of rmd_oracle_pointcloud.c.  Built on
 * its own into librmd_oracle_propagate.so by tests/prior_oracle.py, which also binds it.
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#define RMDO_UPDATE 0
#define RMDO_CONVERGED 1
#define RMDO_BORDER 2

/* Splat: zbuf (dw x dh, row-major) receives min over the accepted points of the bit pattern of their distance
 * to the destination camera; 0xFFFFFFFF where nothing landed.  src_mu, src_conv: dense sw x sh maps;
 * T_world_ref_src and T_curr_world_dst: 3x4 row-major.  Returns the number of accepted points. */
size_t rmd_oracle_prior_splat(const float *src_mu, const int *src_conv, int sw, int sh, float sfx, float sfy,
                              float scx, float scy, const float *T_world_ref_src, int dw, int dh, float dfx,
                              float dfy, float dcx, float dcy, const float *T_curr_world_dst, float min_depth,
                              float max_depth, uint32_t *zbuf) {
  size_t accepted = 0;
  memset(zbuf, 0xFF, sizeof(uint32_t) * (size_t)dw * dh);
  const float *A = T_world_ref_src, *B = T_curr_world_dst;
  for (int y = 0; y < sh; ++y) {
    for (int x = 0; x < sw; ++x) {
      const size_t k = (size_t)y * sw + x;
      if (src_conv[k] != RMDO_CONVERGED)
        continue;
      /* the published point (rmd_oracle_point_cloud) */
      const float vx = (x - scx) / sfx, vy = (y - scy) / sfy, vz = 1.0f;
      const float inv_len = 1.0f / sqrtf(vx * vx + vy * vy + vz * vz);
      const float mu = src_mu[k];
      const float qx = (vx * inv_len) * mu, qy = (vy * inv_len) * mu, qz = (vz * inv_len) * mu;
      const float wx = A[0] * qx + A[1] * qy + A[2] * qz + A[3];
      const float wy = A[4] * qx + A[5] * qy + A[6] * qz + A[7];
      const float wz = A[8] * qx + A[9] * qy + A[10] * qz + A[11];
      /* into the destination camera: rotation, then translation */
      const float px = B[0] * wx + B[1] * wy + B[2] * wz + B[3];
      const float py = B[4] * wx + B[5] * wy + B[6] * wz + B[7];
      const float pz = B[8] * wx + B[9] * wy + B[10] * wz + B[11];
      if (!(pz > 0.0f))
        continue;
      const float d = sqrtf(px * px + py * py + pz * pz);
      if (!(d >= min_depth && d <= max_depth))
        continue;
      const float u = dfx * px / pz + dcx, v = dfy * py / pz + dcy;
      const float tu = floorf(u + 0.5f), tv = floorf(v + 0.5f);
      if (!(tu >= 0.0f && tu < (float)dw && tv >= 0.0f && tv < (float)dh))
        continue;
      uint32_t bits;
      memcpy(&bits, &d, sizeof(bits));
      uint32_t *z = zbuf + (size_t)(int)tv * dw + (int)tu;
      if (bits < *z)
        *z = bits;
      ++accepted;
    }
  }
  return accepted;
}

/* Initialise + apply: the destination's seeds (dense dw x dh) as the library leaves them after the prior.
 * Initialisation: mu = (min + max) / 2, sigma_sq = range^2 / 36, a = b = 10, BORDER on the patch-wide ring,
 * UPDATE inside (src/seed_init.cu:57-60, src/seed_check.cu:37-42).  Apply: non-BORDER pixels with a z-buffer
 * entry get (depth, sigma_sq_frac * sigma_sq_max, 10, 10). */
void rmd_oracle_prior_apply(const uint32_t *zbuf, int dw, int dh, int patch, float min_depth, float max_depth,
                            float sigma_sq_frac, float *mu, float *sigma_sq, float *a, float *b, int *conv) {
  const float avg_depth = (min_depth + max_depth) / 2.0f;
  const float depth_range = max_depth - min_depth;
  const float sigma_sq_max = depth_range * depth_range / 36.0f;
  const float sigma_sq_prop = sigma_sq_frac * sigma_sq_max;
  for (int y = 0; y < dh; ++y) {
    for (int x = 0; x < dw; ++x) {
      const size_t k = (size_t)y * dw + x;
      const int border = x > dw - patch - 1 || y > dh - patch - 1 || x < patch || y < patch;
      conv[k] = border ? RMDO_BORDER : RMDO_UPDATE;
      mu[k] = avg_depth;
      sigma_sq[k] = sigma_sq_max;
      a[k] = 10.0f;
      b[k] = 10.0f;
      if (!border && zbuf[k] != 0xFFFFFFFFu) {
        memcpy(&mu[k], &zbuf[k], sizeof(float));
        sigma_sq[k] = sigma_sq_prop;
      }
    }
  }
}
