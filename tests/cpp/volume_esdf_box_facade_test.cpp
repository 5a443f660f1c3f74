// volume_esdf_box_facade_test.cpp -- the ESDF box of rmd::TsdfVolume (include/rmd/tsdf_volume.cuh): a sphere fused
// from a camera inside it into a 64^3 volume with the brick store, shifted by 20 voxels along x so that part of the
// shell lies in the store; then computeEsdf(lo, dims) over a box that holds the window and the stored part.  Checks
// esdfInfo, that the box sees the stored shell (a point beyond the window is finite and near it), and that the window
// box (0, n) equals computeEsdf() bit for bit.  Writes the box's info, snapshot and queries to argv[1], which
// tests/test_cpp_volume_esdf_box.py compares with the same scene run through the Python API.
//
// Build (tests/test_cpp_volume_esdf_box.py does this):
//   g++ -std=c++14 -DRMD_BUILD_TESTS=1 -Iinclude -I/usr/local/cuda/include tests/cpp/volume_esdf_box_facade_test.cpp \
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

int main(int argc, char **argv)
{
  if(argc < 2)
  {
    std::printf("usage: %s out.bin\n", argv[0]);
    return 2;
  }
  const int N = 64, W = 160, H = 120;
  const float s = 0.0625f, origin[3] = {-2.0f, -2.0f, -2.0f}, R = 1.2f, tau = 4 * s;
  const rmd::PinholeCamera cam(100.0f, 100.0f, (W - 1) / 2.0f, (H - 1) / 2.0f);
  float r[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {0.0f, 0.0f, 0.0f};
  const rmd::SE3<float> T_curr_world(r, t);   // a camera at the sphere's centre, looking along +z
  std::vector<float> depth((size_t)W * H, R);
  rmd::DeviceImage<float> d_depth(W, H);
  d_depth.setDevData(depth.data());

  rmd::TsdfVolume vol(N, N, N, s, origin, tau, 16.0f);
  vol.enableStore();
  int64_t lo_u[3];
  int dims[3];
  float o[3];
  bool threw = false;
  try { vol.esdfInfo(lo_u, dims, o); }
  catch(const rmd::CudaException &) { threw = true; }
  CHECK(threw);

  vol.integrateDepth(W, H, cam, T_curr_world, d_depth.data, d_depth.pitch);
  // the window box equals the window's compute
  const size_t n_vox = (size_t)N * N * N;
  std::vector<float> d0(n_vox), w0(n_vox), d1(n_vox), w1(n_vox);
  vol.computeEsdf();
  vol.downloadEsdf(d0.data(), w0.data());
  const int64_t zero[3] = {0, 0, 0};
  const int n3[3] = {N, N, N};
  vol.computeEsdf(zero, n3);
  vol.downloadEsdf(d1.data(), w1.data());
  CHECK(std::memcmp(d0.data(), d1.data(), n_vox * sizeof(float)) == 0);
  CHECK(std::memcmp(w0.data(), w1.data(), n_vox * sizeof(float)) == 0);
  vol.esdfInfo(lo_u, dims, o);
  CHECK(lo_u[0] == 0 && lo_u[1] == 0 && lo_u[2] == 0 && dims[0] == N && dims[1] == N && dims[2] == N);
  CHECK(o[0] == origin[0] && o[1] == origin[1] && o[2] == origin[2]);

  // the window moves 20 voxels along -z (z <= 0.6875 m then): the whole shell goes to the store, and the window alone
  // has no obstacle left
  vol.shift(0, 0, -20);
  const int M = 3;
  float pts[4 * M] = {0.0f, 0.0f, 1.0f, 0.0f, 0.0f, 0.0f, 0.6f, 0.0f, 0.0f, 0.0f, 5.0f, 0.0f};
  float dg[4 * M], wq[M];
  vol.computeEsdf();
  vol.esdfQuery(pts, M, dg, wq);
  CHECK(std::isnan(dg[0]) && dg[4] == INFINITY);
  const int64_t lo[3] = {-4, -4, -4};
  const int m[3] = {N + 8, N + 8, N + 28};
  vol.computeEsdf(lo, m);
  vol.esdfInfo(lo_u, dims, o);
  CHECK(lo_u[0] == -4 && lo_u[1] == -4 && lo_u[2] == -24);
  CHECK(dims[0] == m[0] && dims[1] == m[1] && dims[2] == m[2]);
  const size_t nb = (size_t)m[0] * m[1] * m[2];
  std::vector<float> dist(nb), weight(nb);
  vol.downloadEsdf(dist.data(), weight.data());
  size_t inside = 0;
  for(size_t q = 0; q < nb; ++q)
    inside += dist[q] < 0.0f;
  CHECK(inside > 100);

  // on the optical axis: z = 1.0 lies beyond the window (NaN above), 0.2 m from the stored shell; z = 0.6 lies in it,
  // 0.6 m from the shell (+inf above); z = 5 lies outside the box
  vol.esdfQuery(pts, M, dg, wq);
  CHECK(std::isfinite(dg[0]) && std::fabs(dg[0] - (R - 1.0f)) < 2 * s && wq[0] > 0.0f);
  CHECK(std::isfinite(dg[4]) && std::fabs(dg[4] - (R - 0.6f)) < 2 * s);
  CHECK(std::isnan(dg[8]) && wq[2] == 0.0f);

  FILE *f = std::fopen(argv[1], "wb");
  CHECK(f != NULL);
  if(f)
  {
    std::fwrite(lo_u, sizeof(int64_t), 3, f);
    std::fwrite(dims, sizeof(int), 3, f);
    std::fwrite(o, sizeof(float), 3, f);
    std::fwrite(dist.data(), sizeof(float), nb, f);
    std::fwrite(weight.data(), sizeof(float), nb, f);
    std::fwrite(dg, sizeof(float), 4 * M, f);
    std::fwrite(wq, sizeof(float), M, f);
    std::fclose(f);
  }

  if(g_failures)
  {
    std::printf("%d FAILURES\n", g_failures);
    return 1;
  }
  std::printf("ALL VOLUME ESDF BOX TESTS PASSED\n");
  return 0;
}
