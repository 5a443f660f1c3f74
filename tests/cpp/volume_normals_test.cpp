// volume_normals_test.cpp -- the normals of rmd::TsdfVolume (include/rmd/tsdf_volume.cuh): a sphere fused from a camera
// inside it has one unit normal per surface point, pointing to the centre (the free side); the raycast's depth is
// raycast()'s, its normals face the camera and are (0, 0, 0, 0) where there is no hit; a bad pitch throws
// rmd::CudaException.
//
// Build (tests/test_cpp_volume_normals.py does this):
//   g++ -std=c++14 -DRMD_BUILD_TESTS=1 -Iinclude -I/usr/local/cuda/include tests/cpp/volume_normals_test.cpp \
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
  const rmd::SE3<float> T_curr_world(r, t);   // a camera near the sphere's centre, looking along +z
  const double o[3] = {-0.02, 0.01, 0.0};     // its centre in the world
  std::vector<float> depth((size_t)W * H);
  std::vector<double> dirs(3 * (size_t)W * H);
  for(int y = 0; y < H; ++y)
    for(int x = 0; x < W; ++x)
    {
      const double vx = (x - cam.cx) / cam.fx, vy = (y - cam.cy) / cam.fy, n = std::sqrt(vx * vx + vy * vy + 1.0);
      const double d[3] = {vx / n, vy / n, 1.0 / n};
      const double b = o[0] * d[0] + o[1] * d[1] + o[2] * d[2];
      const double c = o[0] * o[0] + o[1] * o[1] + o[2] * o[2] - (double)R * R;
      depth[(size_t)y * W + x] = (float)(-b + std::sqrt(b * b - c));
      for(int a = 0; a < 3; ++a) dirs[3 * ((size_t)y * W + x) + a] = d[a];
    }
  try
  {
    rmd::DeviceImage<float> D(W, H), ray(W, H), ray_n(4 * W, H), plain(W, H);
    D.setDevData(depth.data());
    rmd::TsdfVolume vol(N, N, N, s, origin, tau, 64.0f);
    for(int k = 0; k < 3; ++k)
      vol.integrateDepth(W, H, cam, T_curr_world, D.data, D.pitch);
    const std::vector<float> pts = vol.surfacePoints(), nrm = vol.surfaceNormals();
    CHECK(nrm.size() == pts.size());
    CHECK(pts.size() / 4 > 1000);
    std::vector<float> xyzw;
    std::vector<int32_t> tri;
    vol.mesh(xyzw, tri);
    CHECK(xyzw.size() == nrm.size());
    // inside the sphere is free space: the normals point to the centre, within a few degrees (all but a few at the
    // edge of the view, where a gradient is one-sided against unknown space); each is a unit vector or none
    size_t inward = 0, unit = 0;
    for(size_t p = 0; p < pts.size() / 4; ++p)
    {
      const double c[3] = {-pts[4 * p], -pts[4 * p + 1], -pts[4 * p + 2]};
      const double cl = std::sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
      const double dot = (c[0] * nrm[4 * p] + c[1] * nrm[4 * p + 1] + c[2] * nrm[4 * p + 2]) / cl;
      const double len = std::sqrt((double)nrm[4 * p] * nrm[4 * p] + (double)nrm[4 * p + 1] * nrm[4 * p + 1] +
                                   (double)nrm[4 * p + 2] * nrm[4 * p + 2]);
      inward += dot > 0.99;
      unit += (std::fabs(len - 1.0) < 1e-6 || len == 0.0) && nrm[4 * p + 3] == 0.0f;
    }
    CHECK(inward > pts.size() / 4 * 95 / 100);
    CHECK(unit == pts.size() / 4);
    vol.raycastNormals(W, H, cam, T_curr_world, ray.data, ray.pitch, ray_n.data, ray_n.pitch);
    vol.raycast(W, H, cam, T_curr_world, plain.data, plain.pitch);
    vol.sync();
    std::vector<float> rd((size_t)W * H), rp((size_t)W * H), rn(4 * (size_t)W * H);
    ray.getDevData(rd.data());
    plain.getDevData(rp.data());
    ray_n.getDevData(rn.data());
    size_t hits = 0, facing = 0, wrong = 0;
    for(size_t p = 0; p < rd.size(); ++p)
    {
      const float *n = &rn[4 * p];
      const bool has = n[0] != 0.0f || n[1] != 0.0f || n[2] != 0.0f;
      hits += rd[p] > 0.0f;
      facing += rd[p] > 0.0f && has && n[0] * dirs[3 * p] + n[1] * dirs[3 * p + 1] + n[2] * dirs[3 * p + 2] < -0.9;
      wrong += (rd[p] == 0.0f && (has || n[3] != 0.0f)) || std::memcmp(&rd[p], &rp[p], sizeof(float)) != 0;
    }
    CHECK(hits > (size_t)W * H / 2);
    CHECK(facing > hits * 9 / 10);
    CHECK(wrong == 0);
    std::printf("%zu surface points, %zu pointing inwards; %zu of %zu hits face the camera\n", pts.size() / 4, inward,
                facing, hits);
    // refusals: normals pitch not a multiple of 16, too small
    CHECK(throws([&] { vol.raycastNormals(W, H, cam, T_curr_world, ray.data, ray.pitch, ray_n.data, 16 * W + 4); }));
    CHECK(throws([&] { vol.raycastNormals(W, H, cam, T_curr_world, ray.data, ray.pitch, ray_n.data, 16 * W - 16); }));
    CHECK(throws([&] { vol.raycastNormals(W, H, cam, T_curr_world, ray.data, ray.pitch, NULL, ray_n.pitch); }));
  }
  catch(const rmd::CudaException &e)
  {
    std::printf("unexpected CudaException: %s\n", e.what());
    ++g_failures;
  }
  std::printf(g_failures ? "FAILED (%d)\n" : "ALL VOLUME NORMALS TESTS PASSED\n", g_failures);
  return g_failures ? 1 : 0;
}
