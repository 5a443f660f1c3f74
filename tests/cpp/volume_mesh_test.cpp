// volume_mesh_test.cpp -- rmd::TsdfVolume::mesh (include/rmd/tsdf_volume.cuh): an uploaded sphere SDF meshes to a
// closed surface whose vertices are surfacePoints() and whose normals point outwards; a reset volume has no mesh.
//
// Build (tests/test_cpp_volume_mesh.py does this):
//   g++ -std=c++14 -DRMD_BUILD_TESTS=1 -Iinclude -I/usr/local/cuda/include tests/cpp/volume_mesh_test.cpp \
//       -Lrpg_open_remode_b200 -lrmd_b200 -L/usr/local/cuda/lib64 -lcudart
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <utility>
#include <vector>

#include <rmd/tsdf_volume.cuh>

static int g_failures = 0;
#define CHECK(cond)                                                                  \
  do {                                                                               \
    if(!(cond)) { std::printf("CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++g_failures; } \
  } while(0)

int main()
{
  const int N = 48;
  const float s = 0.05f, origin[3] = {-1.2f, -1.15f, -1.1f}, c[3] = {0.03f, 0.01f, 0.02f}, R = 0.8f, tau = 3 * s;
  const size_t n = (size_t)N * N * N;
  std::vector<float> tsdf(n), weight(n, 1.0f);
  for(int k = 0; k < N; ++k)
    for(int j = 0; j < N; ++j)
      for(int i = 0; i < N; ++i)
      {
        const double x = origin[0] + i * s - c[0], y = origin[1] + j * s - c[1], z = origin[2] + k * s - c[2];
        const double d = (std::sqrt(x * x + y * y + z * z) - R) / tau;
        tsdf[((size_t)k * N + j) * N + i] = (float)std::max(-1.0, std::min(1.0, d));
      }
  try
  {
    rmd::TsdfVolume vol(N, N, N, s, origin, tau, 64.0f);
    vol.upload(tsdf.data(), weight.data());
    std::vector<float> xyzw;
    std::vector<int32_t> tri;
    vol.mesh(xyzw, tri);
    const std::vector<float> pts = vol.surfacePoints();
    CHECK(xyzw == pts);
    const size_t nv = xyzw.size() / 4, nt = tri.size() / 3;
    CHECK(nt > 1000);
    // closed: every directed edge once, and its reverse once
    std::vector<std::pair<int32_t, int32_t> > e;
    bool valid = true;
    for(size_t t = 0; t < nt; ++t)
      for(int r = 0; r < 3; ++r)
      {
        const int32_t a = tri[3 * t + r], b = tri[3 * t + (r + 1) % 3];
        valid = valid && a >= 0 && (size_t)a < nv;
        e.push_back(std::make_pair(a, b));
      }
    CHECK(valid);
    std::sort(e.begin(), e.end());
    CHECK(std::adjacent_find(e.begin(), e.end()) == e.end());
    size_t open = 0, inward = 0;
    for(size_t q = 0; q < e.size(); ++q)
      open += !std::binary_search(e.begin(), e.end(), std::make_pair(e[q].second, e[q].first));
    CHECK(open == 0);
    double area = 0.0;
    for(size_t t = 0; t < nt && valid; ++t)
    {
      const float *a = &xyzw[4 * tri[3 * t]], *b = &xyzw[4 * tri[3 * t + 1]], *d = &xyzw[4 * tri[3 * t + 2]];
      const double u[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]}, w[3] = {d[0] - a[0], d[1] - a[1], d[2] - a[2]};
      const double m[3] = {u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0]};
      const double out = m[0] * (a[0] - c[0]) + m[1] * (a[1] - c[1]) + m[2] * (a[2] - c[2]);
      const double len = std::sqrt(m[0] * m[0] + m[1] * m[1] + m[2] * m[2]);
      inward += len > 1e-9 && out <= 0.0;
      area += 0.5 * len;
    }
    CHECK(inward == 0);
    const double want = 4.0 * M_PI * R * R;
    CHECK(std::fabs(area / want - 1.0) < 0.01);
    std::printf("%zu vertices, %zu triangles, area %.5f (sphere %.5f)\n", nv, nt, area, want);
    vol.reset();
    vol.mesh(xyzw, tri);
    CHECK(xyzw.empty() && tri.empty());
  }
  catch(const rmd::CudaException &e)
  {
    std::printf("unexpected CudaException: %s\n", e.what());
    ++g_failures;
  }
  std::printf(g_failures ? "FAILED (%d)\n" : "ALL VOLUME MESH TESTS PASSED\n", g_failures);
  return g_failures ? 1 : 0;
}
