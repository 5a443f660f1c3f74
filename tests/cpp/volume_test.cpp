// volume_test.cpp -- rmd::TsdfVolume (include/rmd/tsdf_volume.cuh): a keyframe fused through integrate(seeds)
// equals the same keyframe fused through integrateDepth from its exported mu and convergence maps; the surface
// points and a raycast see the fused surface; the C-ABI's refusals surface as rmd::CudaException.
//
// Build (tests/test_cpp_volume.py does this):
//   g++ -std=c++14 -DRMD_BUILD_TESTS=1 -Iinclude -I/usr/local/cuda/include tests/cpp/volume_test.cpp \
//       -Lrpg_open_remode_b200 -lrmd_b200 -Lrpg_open_remode_b200/synth -lrmd_synth -L/usr/local/cuda/lib64 -lcudart
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <vector>

#include <rmd/device_image.cuh>
#include <rmd/se3.cuh>
#include <rmd/seed_matrix.cuh>
#include <rmd/tsdf_volume.cuh>

extern "C"
{
void *rmd_synth_create(int width, int height, float fx, float fy, float cx, float cy, uint32_t seed);
void rmd_synth_destroy(void *p);
void rmd_synth_pose(const void *p, int k, float *T_world_cam);
int rmd_synth_render(const void *p, const float *T_world_cam, uint8_t *img_u8, float *img_f32, float *depth);
}

static int g_failures = 0;
#define CHECK(cond)                                                                  \
  do {                                                                               \
    if(!(cond)) { std::printf("CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++g_failures; } \
  } while(0)

struct Frame
{
  std::vector<float> img;
  rmd::SE3<float> T_curr_world;
};

static Frame render(void *scene, int w, int h, int k)
{
  Frame f;
  f.img.resize((size_t)w * h);
  float T[12];
  rmd_synth_pose(scene, k, T);
  rmd_synth_render(scene, T, NULL, f.img.data(), NULL);
  float r[9] = {T[0], T[1], T[2], T[4], T[5], T[6], T[8], T[9], T[10]};
  float t[3] = {T[3], T[7], T[11]};
  f.T_curr_world = rmd::SE3<float>(r, t).inv();
  return f;
}

template<typename Fn>
static bool throws(Fn fn)
{
  try { fn(); }
  catch(const rmd::CudaException &) { return true; }
  return false;
}

int main()
{
  const int W = 160, H = 120, N = 40, G = 96;
  const rmd::PinholeCamera cam(481.2f * W / 640.0f, -480.0f * H / 480.0f, (W - 1) / 2.0f, (H - 1) / 2.0f);
  void *scene = rmd_synth_create(W, H, cam.fx, cam.fy, cam.cx, cam.cy, 0x5EED0001u);
  const float min_d = 0.4f, max_d = 1.8f;
  try
  {
    rmd::SeedMatrix seeds(W, H, cam);
    const Frame f0 = render(scene, W, H, 0);
    seeds.setReferenceImage(const_cast<float*>(f0.img.data()), f0.T_curr_world, min_d, max_d);
    for(int k = 1; k <= N; ++k)
    {
      const Frame f = render(scene, W, H, k);
      seeds.update(const_cast<float*>(f.img.data()), f.T_curr_world);
    }
    CHECK(seeds.getConvergedCount() > (size_t)W * H / 20);
    // a 96^3 grid of 2 cm voxels in front of the reference camera
    rmd::SE3<float> T_world_ref = f0.T_curr_world.inv();
    const float3 c = T_world_ref * make_float3(0.0f, 0.0f, 1.1f);
    const float s = 0.02f, origin[3] = {c.x - 0.5f * G * s, c.y - 0.5f * G * s, c.z - 0.5f * G * s};
    rmd::TsdfVolume a(G, G, G, s, origin, 4 * s, 64.0f), b(G, G, G, s, origin, 4 * s, 64.0f);
    a.integrate(seeds);
    const rmd::DeviceImage<float> &mu = seeds.getMu();
    const rmd::DeviceImage<int> &conv = seeds.getConvergence();
    b.integrateDepth(W, H, cam, f0.T_curr_world, mu.data, mu.pitch, conv.data, conv.pitch);
    const size_t n = (size_t)G * G * G;
    std::vector<float> ta(n), wa(n), tb(n), wb(n);
    a.download(ta.data(), wa.data());
    b.download(tb.data(), wb.data());
    CHECK(ta == tb);
    CHECK(wa == wb);
    size_t touched = 0;
    for(size_t i = 0; i < n; ++i) touched += wa[i] > 0.0f;
    CHECK(touched > n / 100);
    const std::vector<float> pts = a.surfacePoints();
    CHECK(pts.size() > 4 * 1000);
    rmd::DeviceImage<float> ray(W, H);
    a.raycast(W, H, cam, f0.T_curr_world, ray.data, ray.pitch);
    a.sync();
    std::vector<float> depth((size_t)W * H);
    ray.getDevData(depth.data());
    size_t hits = 0;
    for(float d : depth) hits += d > 0.0f;
    CHECK(hits > (size_t)W * H / 20);
    std::printf("%zu voxels touched, %zu surface points, %zu of %d pixels hit\n", touched, pts.size() / 4, hits, W * H);
    // a reset volume is all unknown
    a.reset();
    CHECK(a.surfacePoints().empty());
    // refusals
    CHECK(throws([&] { rmd::TsdfVolume bad(0, G, G, s, origin, 4 * s, 64.0f); }));
    CHECK(throws([&] { rmd::TsdfVolume bad(G, G, G, -s, origin, 4 * s, 64.0f); }));
    CHECK(throws([&] { rmd::TsdfVolume bad(G, G, G, s, origin, 4 * s, 0.5f); }));
    CHECK(throws([&] { b.integrateDepth(W, H, cam, f0.T_curr_world, mu.data, 2, NULL, 0); }));
    rmd::SeedMatrix no_ref(W, H, cam);
    CHECK(throws([&] { b.integrate(no_ref); }));
  }
  catch(const rmd::CudaException &e)
  {
    std::printf("unexpected CudaException: %s\n", e.what());
    ++g_failures;
  }
  rmd_synth_destroy(scene);
  std::printf(g_failures ? "FAILED (%d)\n" : "ALL VOLUME TESTS PASSED\n", g_failures);
  return g_failures ? 1 : 0;
}
