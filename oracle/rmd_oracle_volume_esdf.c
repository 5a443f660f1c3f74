/* rmd_oracle_volume_esdf.c -- CPU restatement of the TSDF volume's Euclidean signed distance field (csrc/volume.cu:
 * volume_esdf_kernel and volume_esdf_query_kernel; DESIGN.md 4.8).
 *
 * TEST INFRASTRUCTURE ONLY (see rmd_oracle.h).  The reference has no such step; tests/test_volume_esdf_oracle.py
 * pins this file against brute force and scipy.ndimage.distance_transform_edt.  Built on its own (IEEE fp32, no
 * contraction) into librmd_oracle_volume_esdf.so by tests/volume_esdf_oracle.py, which also binds it.
 *
 * Grids: nx * ny * nz floats per record half, x fastest; origin = centre of voxel (0, 0, 0).
 */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

#define ESDF_INF INT64_MAX

/* The exact lower envelope of the parabolas f[p] + (q - p)^2 over the sites p with f[p] != ESDF_INF, evaluated at
 * every q of the column (Felzenszwalb-Huttenlocher; intersections compared by int64 cross-multiplication).  v: n
 * ints of scratch.  ESDF_INF everywhere when there is no site. */
static void envelope(const int64_t *f, int n, int64_t *out, int *v) {
  int top = -1;
  for (int q = 0; q < n; ++q) {
    if (f[q] == ESDF_INF)
      continue;
    const int64_t Fq = f[q] + (int64_t)q * q;
    while (top >= 1) {
      const int a = v[top - 1], b = v[top];
      const int64_t Fa = f[a] + (int64_t)a * a, Fb = f[b] + (int64_t)b * b;
      /* the intersection of b and q lies at or before that of a and b: b is never the lowest */
      if ((Fq - Fb) * (b - a) > (Fb - Fa) * (int64_t)(q - b))
        break;
      --top;
    }
    v[++top] = q;
  }
  int k = 0;
  for (int q = 0; q < n; ++q) {
    if (top < 0) {
      out[q] = ESDF_INF;
      continue;
    }
    while (k < top) {
      const int a = v[k], b = v[k + 1];
      const int64_t Fa = f[a] + (int64_t)a * a, Fb = f[b] + (int64_t)b * b;
      if (!(Fb - Fa < 2 * (int64_t)q * (b - a)))
        break;
      ++k;
    }
    const int64_t d = q - v[k];
    out[q] = f[v[k]] + d * d;
  }
}

/* d2 (n_vox) <- min over the sites of the squared distance, per axis z, y, x; d2 holds 0 at the sites and INT32_MAX
 * elsewhere on entry, and after (< 2^24 by the size limit, or INT32_MAX when there is no site).  Returns -1 when out of
 * memory. */
static int edt3(int32_t *d2, int nx, int ny, int nz) {
  const int nmax = nx > ny ? (nx > nz ? nx : nz) : (ny > nz ? ny : nz);
  int64_t *f = malloc(sizeof(int64_t) * nmax), *o = malloc(sizeof(int64_t) * nmax);
  int *v = malloc(sizeof(int) * nmax);
  if (!f || !o || !v) {
    free(f); free(o); free(v);
    return -1;
  }
  const size_t plane = (size_t)nx * ny;
  const int n[3] = {nz, ny, nx};
  for (int axis = 0; axis < 3; ++axis) {
    const size_t stride = axis == 0 ? plane : axis == 1 ? (size_t)nx : 1;
    const int len = n[axis];
    for (int k = 0; k < nz; ++k)
      for (int j = 0; j < ny; ++j)
        for (int i = 0; i < nx; ++i) {
          /* visit each column once, from its first voxel */
          if ((axis == 0 && k) || (axis == 1 && j) || (axis == 2 && i))
            continue;
          const size_t base = ((size_t)k * ny + j) * nx + i;
          for (int q = 0; q < len; ++q) {
            const int32_t x = d2[base + q * stride];
            f[q] = x == INT32_MAX ? ESDF_INF : x;
          }
          envelope(f, len, o, v);
          for (int q = 0; q < len; ++q)
            d2[base + q * stride] = o[q] == ESDF_INF ? INT32_MAX : (int32_t)o[q];
        }
  }
  free(f); free(o); free(v);
  return 0;
}

static int occupied(float t, float w) { return w > 0.0f && t <= 0.0f; }

/* The snapshot: dist = s sqrt(d2_O) on F, -s sqrt(d2_F) on O (+-inf when the other set is empty), wout = weight.
 * Returns 0, -1 when out of memory, -2 past the size limit. */
int rmd_oracle_volume_esdf(const float *tsdf, const float *weight, int nx, int ny, int nz, float s, float *dist,
                           float *wout) {
  const long long ex = nx - 1, ey = ny - 1, ez = nz - 1;
  if (ex * ex + ey * ey + ez * ez >= (1ll << 24))
    return -2;
  const size_t n_vox = (size_t)nx * ny * nz;
  int32_t *dO = malloc(sizeof(int32_t) * n_vox), *dF = malloc(sizeof(int32_t) * n_vox);
  if (!dO || !dF) {
    free(dO); free(dF);
    return -1;
  }
  for (size_t q = 0; q < n_vox; ++q) {
    const int occ = occupied(tsdf[q], weight[q]);
    dO[q] = occ ? 0 : INT32_MAX;
    dF[q] = occ ? INT32_MAX : 0;
  }
  if (edt3(dO, nx, ny, nz) || edt3(dF, nx, ny, nz)) {
    free(dO); free(dF);
    return -1;
  }
  for (size_t q = 0; q < n_vox; ++q) {
    const int occ = occupied(tsdf[q], weight[q]);
    const int32_t d2 = occ ? dF[q] : dO[q];
    const float d = d2 == INT32_MAX ? INFINITY : sqrtf((float)d2) * s;
    dist[q] = occ ? -d : d;
    wout[q] = weight[q];
  }
  free(dO); free(dF);
  return 0;
}

static float lerp(float a, float b, float f) { return a + f * (b - a); }

/* the kernels' NaN, 0x7fffffff */
static float esdf_nan(void) {
  union { uint32_t u; float f; } x = {0x7fffffffu};
  return x.f;
}

/* The query at n points (4 floats each, w ignored): dg = (distance, d/dx, d/dy, d/dz), wq = min corner weight (may be
 * NULL). */
void rmd_oracle_volume_esdf_query(const float *dist, const float *weight, int nx, int ny, int nz, float s,
                                  const float *origin, const float *xyzw, size_t n, float *dg, float *wq) {
  const int dims[3] = {nx, ny, nz};
  for (size_t t = 0; t < n; ++t) {
    float u[3], fl[3];
    int c[3], inside = 1;
    for (int a = 0; a < 3; ++a) {
      u[a] = (xyzw[4 * t + a] - origin[a]) / s;
      fl[a] = floorf(u[a]);
      c[a] = (fl[a] >= 0.0f && fl[a] < 2.0e9f) ? (int)fl[a] : -1;
      inside = inside && c[a] >= 0 && c[a] + 1 < dims[a];
    }
    float *o = dg + 4 * t;
    o[0] = esdf_nan(); o[1] = 0.0f; o[2] = 0.0f; o[3] = 0.0f;
    float wmin = 0.0f;
    if (inside) {
      float e[8], w[8];
      for (int q = 0; q < 8; ++q) {
        const size_t idx = ((size_t)(c[2] + (q >> 2)) * ny + (size_t)(c[1] + ((q >> 1) & 1))) * nx + c[0] + (q & 1);
        e[q] = dist[idx];
        w[q] = weight[idx];
      }
      wmin = w[0];
      for (int q = 1; q < 8; ++q)
        wmin = fminf(wmin, w[q]);
      int inf = -1;
      for (int q = 0; q < 8 && inf < 0; ++q)
        if (isinf(e[q]))
          inf = q;
      if (inf >= 0)
        o[0] = e[inf];
      else {
        const float fx = u[0] - fl[0], fy = u[1] - fl[1], fz = u[2] - fl[2];
        /* e[x + 2 y + 4 z] */
        o[0] = lerp(lerp(lerp(e[0], e[1], fx), lerp(e[2], e[3], fx), fy),
                    lerp(lerp(e[4], e[5], fx), lerp(e[6], e[7], fx), fy), fz);
        o[1] = lerp(lerp(e[1] - e[0], e[3] - e[2], fy), lerp(e[5] - e[4], e[7] - e[6], fy), fz) / s;
        o[2] = lerp(lerp(e[2] - e[0], e[3] - e[1], fx), lerp(e[6] - e[4], e[7] - e[5], fx), fz) / s;
        o[3] = lerp(lerp(e[4] - e[0], e[5] - e[1], fx), lerp(e[6] - e[2], e[7] - e[3], fx), fy) / s;
      }
    }
    if (wq)
      wq[t] = wmin;
  }
}
