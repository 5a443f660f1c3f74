// volume_esdf_test.cpp -- the ESDF of rmd::TsdfVolume (include/rmd/tsdf_volume.cuh): a sphere fused from a camera
// inside it; the facade's snapshot and query equal the C-ABI's, the distance is negative inside the shell and grows
// away from it, its gradient points away from the surface, a point outside the grid is NaN with weight 0, and a query
// before the first compute throws rmd::CudaException.
//
// Build (tests/test_cpp_volume_esdf.py does this):
//   g++ -std=c++14 -DRMD_BUILD_TESTS=1 -Iinclude -I/usr/local/cuda/include tests/cpp/volume_esdf_test.cpp \
//       -Lrpg_open_remode_b200 -lrmd_b200 -L/usr/local/cuda/lib64 -lcudart
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include <rmd/device_image.cuh>
#include <rmd/se3.cuh>
#include <rmd/tsdf_volume.cuh>

static int g_failures = 0;
#define CHECK(cond)                                                                  \
  do {                                                                               \
    if(!(cond)) { std::printf("CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++g_failures; } \
  } while(0)

int main()
{
  const int N = 64, W = 160, H = 120;
  const float s = 0.0625f, origin[3] = {-2.0f, -2.0f, -2.0f}, R = 1.2f, tau = 4 * s;
  const rmd::PinholeCamera cam(100.0f, 100.0f, (W - 1) / 2.0f, (H - 1) / 2.0f);
  float r[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {0.0f, 0.0f, 0.0f};
  const rmd::SE3<float> T_curr_world(r, t);   // a camera at the sphere's centre, looking along +z
  std::vector<float> depth((size_t)W * H, R);
  rmd::DeviceImage<float> d_depth(W, H);
  d_depth.setDevData(depth.data());

  rmd::TsdfVolume vol(N, N, N, s, origin, tau, 16.0f);
  float p0[4] = {0.0f, 0.0f, 0.0f, 0.0f}, dg0[4];
  bool threw = false;
  try { vol.esdfQuery(p0, 1, dg0); }
  catch(const rmd::CudaException &) { threw = true; }
  CHECK(threw);

  vol.integrateDepth(W, H, cam, T_curr_world, d_depth.data, d_depth.pitch);
  vol.computeEsdf();
  const size_t n_vox = (size_t)N * N * N;
  std::vector<float> dist(n_vox), weight(n_vox), dist2(n_vox), weight2(n_vox);
  vol.downloadEsdf(dist.data(), weight.data());
  CHECK(rmd_volume_download_esdf(vol.handle(), dist2.data(), weight2.data()) == 0);
  CHECK(std::memcmp(dist.data(), dist2.data(), n_vox * sizeof(float)) == 0);
  size_t inside = 0, known = 0;
  for(size_t q = 0; q < n_vox; ++q)
  {
    inside += dist[q] < 0.0f;
    known += weight[q] > 0.0f;
  }
  CHECK(inside > 100 && known > inside);

  // along the optical axis (+z) from the camera: free (positive), then the shell, and the distance to the shell
  // shrinks as the point approaches it; the gradient points back towards the camera
  const int M = 4;
  float pts[4 * M] = {0.0f, 0.0f, 0.3f, 0.0f, 0.0f, 0.0f, 0.6f, 0.0f, 0.0f, 0.0f, 0.9f, 0.0f,
                      0.0f, 0.0f, 5.0f, 0.0f};   // the last one lies outside the grid
  float dg[4 * M], wq[M], dg2[4 * M], wq2[M];
  vol.esdfQuery(pts, M, dg, wq);
  CHECK(rmd_volume_esdf_query(vol.handle(), pts, M, dg2, wq2) == 0);
  CHECK(std::memcmp(dg, dg2, sizeof(dg)) == 0 && std::memcmp(wq, wq2, sizeof(wq)) == 0);
  CHECK(dg[0] > dg[4] && dg[4] > dg[8] && dg[8] > 0.0f);
  CHECK(std::fabs(dg[4] - (R - 0.6f)) < 2 * s);
  CHECK(dg[11] < 0.0f);                                  // d distance / dz < 0 towards the shell
  CHECK(std::isnan(dg[12]) && dg[13] == 0.0f && wq[3] == 0.0f);

  if(g_failures)
  {
    std::printf("%d FAILURES\n", g_failures);
    return 1;
  }
  std::printf("ALL VOLUME ESDF TESTS PASSED\n");
  return 0;
}
