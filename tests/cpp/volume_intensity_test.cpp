// volume_intensity_test.cpp -- the intensity channel of rmd::TsdfVolume (include/rmd/tsdf_volume.cuh): a sphere SDF
// fused from a camera inside it with a constant dyadic intensity extracts and renders to exactly that value, one
// intensity per surface point; a volume without the channel refuses intensity calls with rmd::CudaException.
//
// Build (tests/test_cpp_volume_intensity.py does this):
//   g++ -std=c++14 -DRMD_BUILD_TESTS=1 -Iinclude -I/usr/local/cuda/include tests/cpp/volume_intensity_test.cpp \
//       -Lrpg_open_remode_b200 -lrmd_b200 -L/usr/local/cuda/lib64 -lcudart
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <vector>

#include <rmd/device_image.cuh>
#include <rmd/se3.cuh>
#include <rmd/tsdf_volume.cuh>

static int g_failures = 0;
#define CHECK(cond)                                                                  \
  do {                                                                               \
    if(!(cond)) { std::printf("CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++g_failures; } \
  } while(0)

template<typename Fn>
static bool throws(Fn fn)
{
  try { fn(); }
  catch(const rmd::CudaException &) { return true; }
  return false;
}

int main()
{
  const int N = 64, W = 160, H = 120;
  const float s = 0.05f, origin[3] = {-1.6f, -1.6f, -1.6f}, R = 1.2f, tau = 4 * s;
  const rmd::PinholeCamera cam(100.0f, 100.0f, (W - 1) / 2.0f, (H - 1) / 2.0f);
  float r[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {0.02f, -0.01f, 0.0f};
  const rmd::SE3<float> T_curr_world(r, t);   // a camera at the sphere's centre, looking along +z
  // the depth image of the sphere's inside: every ray meets it at distance R
  std::vector<float> depth((size_t)W * H), inten((size_t)W * H, 0.375f);
  for(int y = 0; y < H; ++y)
    for(int x = 0; x < W; ++x)
    {
      const double vx = (x - cam.cx) / cam.fx, vy = (y - cam.cy) / cam.fy, n = std::sqrt(vx * vx + vy * vy + 1.0);
      const double o[3] = {-0.02, 0.01, 0.0}, d[3] = {vx / n, vy / n, 1.0 / n};   // camera centre, ray
      const double b = o[0] * d[0] + o[1] * d[1] + o[2] * d[2];
      const double c = o[0] * o[0] + o[1] * o[1] + o[2] * o[2] - (double)R * R;
      depth[(size_t)y * W + x] = (float)(-b + std::sqrt(b * b - c));
    }
  try
  {
    rmd::DeviceImage<float> D(W, H), I(W, H), ray(W, H), ray_i(W, H);
    D.setDevData(depth.data());
    I.setDevData(inten.data());
    rmd::TsdfVolume vol(N, N, N, s, origin, tau, 64.0f);
    rmd::TsdfVolume plain(N, N, N, s, origin, tau, 64.0f);
    vol.enableIntensity();
    vol.enableIntensity();   // idempotent
    for(int k = 0; k < 3; ++k)
    {
      vol.integrateDepthIntensity(W, H, cam, T_curr_world, D.data, D.pitch, I.data, I.pitch);
      plain.integrateDepth(W, H, cam, T_curr_world, D.data, D.pitch);
    }
    const std::vector<float> pts = vol.surfacePoints(), inten_pts = vol.surfaceIntensity();
    CHECK(pts == plain.surfacePoints());
    CHECK(inten_pts.size() * 4 == pts.size());
    CHECK(inten_pts.size() > 1000);
    size_t exact = 0;
    for(float v : inten_pts) exact += v == 0.375f;
    CHECK(exact == inten_pts.size());
    vol.raycastIntensity(W, H, cam, T_curr_world, ray.data, ray.pitch, ray_i.data, ray_i.pitch);
    vol.sync();
    std::vector<float> rd((size_t)W * H), ri((size_t)W * H);
    ray.getDevData(rd.data());
    ray_i.getDevData(ri.data());
    size_t hits = 0, shaded = 0, wrong = 0;
    for(size_t p = 0; p < rd.size(); ++p)
    {
      hits += rd[p] > 0.0f;
      shaded += rd[p] > 0.0f && ri[p] == 0.375f;
      wrong += (rd[p] == 0.0f && ri[p] != -1.0f) || (ri[p] != -1.0f && ri[p] != 0.375f);
    }
    CHECK(hits > (size_t)W * H / 2);
    CHECK(shaded > hits * 9 / 10);
    CHECK(wrong == 0);
    std::printf("%zu surface points, all at intensity 0.375: %zu; %zu of %zu hits shaded\n", inten_pts.size(), exact,
                shaded, hits);
    // round trip and reset
    const size_t n = (size_t)N * N * N;
    std::vector<float> c(n), w(n);
    vol.downloadIntensity(c.data(), w.data());
    size_t coloured = 0;
    for(size_t q = 0; q < n; ++q) coloured += w[q] == 3.0f && c[q] == 0.375f;
    CHECK(coloured > 1000);
    vol.uploadIntensity(c.data(), w.data());
    CHECK(vol.surfaceIntensity() == inten_pts);
    vol.reset();
    vol.downloadIntensity(c.data(), w.data());
    size_t left = 0;
    for(size_t q = 0; q < n; ++q) left += w[q] != 0.0f;
    CHECK(left == 0);
    // refusals: no channel, bad pitch
    CHECK(throws([&] { plain.surfaceIntensity(); }));
    CHECK(throws([&] { plain.downloadIntensity(c.data(), w.data()); }));
    CHECK(throws([&] {
      plain.raycastIntensity(W, H, cam, T_curr_world, ray.data, ray.pitch, ray_i.data, ray_i.pitch);
    }));
    CHECK(throws([&] { vol.integrateDepthIntensity(W, H, cam, T_curr_world, D.data, D.pitch, I.data, 2); }));
  }
  catch(const rmd::CudaException &e)
  {
    std::printf("unexpected CudaException: %s\n", e.what());
    ++g_failures;
  }
  std::printf(g_failures ? "FAILED (%d)\n" : "ALL VOLUME INTENSITY TESTS PASSED\n", g_failures);
  return g_failures ? 1 : 0;
}
