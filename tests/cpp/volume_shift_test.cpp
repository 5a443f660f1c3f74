// volume_shift_test.cpp -- the moving rmd::TsdfVolume (include/rmd/tsdf_volume.cuh): a sphere fused from a camera
// inside it; the facade's spills equal the C-ABI's, spill + the points after a shift make up the points before, the
// origin moves by whole voxels from the creation origin, a shift by the whole grid empties it, and a null offset
// throws rmd::CudaException.
//
// Build (tests/test_cpp_volume_shift.py does this):
//   g++ -std=c++14 -DRMD_BUILD_TESTS=1 -Iinclude -I/usr/local/cuda/include tests/cpp/volume_shift_test.cpp \
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
  std::vector<float> depth((size_t)W * H, R), inten((size_t)W * H, 0.5f);
  rmd::DeviceImage<float> d_depth(W, H), d_inten(W, H);
  d_depth.setDevData(depth.data());
  d_inten.setDevData(inten.data());

  rmd::TsdfVolume vol(N, N, N, s, origin, tau, 16.0f);
  vol.enableIntensity();
  vol.integrateDepthIntensity(W, H, cam, T_curr_world, d_depth.data, d_depth.pitch, d_inten.data, d_inten.pitch);
  vol.sync();
  const std::vector<float> before = vol.surfacePoints();
  const std::vector<float> before_i = vol.surfaceIntensity();
  CHECK(before.size() > 4 * 100);

  const int d[3] = {26, -7, -14};
  const std::vector<float> spill = vol.spillPoints(d);
  const std::vector<float> spill_i = vol.spillIntensity(d);
  const std::vector<float> spill_n = vol.spillNormals(d);
  CHECK(!spill.empty() && spill.size() < before.size());
  CHECK(spill_i.size() * 4 == spill.size() && spill_n.size() == spill.size());
  // the facade == the C-ABI
  size_t n = 0;
  CHECK(rmd_volume_spill_points(vol.handle(), d, NULL, 0, &n) == 0 && 4 * n == spill.size());
  std::vector<float> raw(4 * n);
  CHECK(rmd_volume_spill_points(vol.handle(), d, raw.data(), n, &n) == 0);
  CHECK(std::memcmp(raw.data(), spill.data(), raw.size() * sizeof(float)) == 0);

  vol.shift(d[0], d[1], d[2]);
  const std::vector<float> after = vol.surfacePoints();
  const std::vector<float> after_i = vol.surfaceIntensity();
  CHECK(after.size() + spill.size() == before.size());
  CHECK(after_i.size() + spill_i.size() == before_i.size());
  // s is a power of two and the origin a multiple of it: positions survive the shift, so spill and the points after
  // it interleave back into the points before, in order
  size_t a = 0, b = 0;
  bool ordered = true;
  for(size_t q = 0; q < before.size() / 4 && ordered; ++q)
  {
    if(b < spill.size() / 4 && std::memcmp(&before[4 * q], &spill[4 * b], 16) == 0) ++b;
    else if(a < after.size() / 4 && std::memcmp(&before[4 * q], &after[4 * a], 16) == 0) ++a;
    else ordered = false;
  }
  CHECK(ordered && a == after.size() / 4 && b == spill.size() / 4);

  int nx = 0;
  float vs = 0.0f, o[3];
  CHECK(rmd_volume_size(vol.handle(), &nx, NULL, NULL, &vs, o) == 0);
  CHECK(nx == N && vs == s);
  CHECK(o[0] == origin[0] + 26 * s && o[1] == origin[1] - 7 * s && o[2] == origin[2] - 14 * s);

  vol.shift(-N, 0, 0);   // everything leaves
  CHECK(vol.surfacePoints().empty());
  std::vector<float> tsdf((size_t)N * N * N), weight((size_t)N * N * N);
  vol.download(tsdf.data(), weight.data());
  bool empty = true;
  for(float w : weight) empty = empty && w == 0.0f;
  CHECK(empty);

  bool threw = false;
  try { vol.spillPoints(NULL); }
  catch(const rmd::CudaException &) { threw = true; }
  CHECK(threw);

  if(g_failures)
  {
    std::printf("%d FAILURES\n", g_failures);
    return 1;
  }
  std::printf("ALL VOLUME SHIFT TESTS PASSED\n");
  return 0;
}
