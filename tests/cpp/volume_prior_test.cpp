// volume_prior_test.cpp -- rmd::TsdfVolume::seedPrior (include/rmd/tsdf_volume.cuh): a new keyframe's depth prior
// taken from the fused model through the facade equals the same prior through the C-ABI (rmd_volume_prior_seeds) on
// a second handle, bit for bit; every seed that took the prior holds the raycast depth of its pixel; the C-ABI's
// refusals surface as rmd::CudaException.
//
// Build (tests/test_cpp_volume_prior.py does this):
//   g++ -std=c++14 -DRMD_BUILD_TESTS=1 -Iinclude -I/usr/local/cuda/include tests/cpp/volume_prior_test.cpp \
//       -Lrpg_open_remode_b200 -lrmd_b200 -Lrpg_open_remode_b200/synth -lrmd_synth -L/usr/local/cuda/lib64 -lcudart
#include <cstdint>
#include <cstdio>
#include <cstring>
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

struct State
{
  std::vector<float> mu, sigma_sq, a, b;
  std::vector<int> conv;
};

static State snapshot(const rmd::SeedMatrix &s, int w, int h)
{
  const size_t n = (size_t)w * h;
  State st;
  st.mu.resize(n); st.sigma_sq.resize(n); st.a.resize(n); st.b.resize(n); st.conv.resize(n);
  s.downloadDepthmap(st.mu.data());
  s.downloadSigmaSq(st.sigma_sq.data());
  s.downloadA(st.a.data());
  s.downloadB(st.b.data());
  s.downloadConvergence(st.conv.data());
  return st;
}

static bool same_bits(const std::vector<float> &x, const std::vector<float> &y)
{
  return x.size() == y.size() && std::memcmp(x.data(), y.data(), sizeof(float) * x.size()) == 0;
}

int main()
{
  const int W = 160, H = 120, N = 40, G = 96;
  const float f = 1.0f / 16.0f;
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
      const Frame fk = render(scene, W, H, k);
      seeds.update(const_cast<float*>(fk.img.data()), fk.T_curr_world);
    }
    CHECK(seeds.getConvergedCount() > (size_t)W * H / 20);
    // a 96^3 grid of 2 cm voxels in front of the first reference camera, fused from the finished keyframe
    rmd::SE3<float> T_world_ref = f0.T_curr_world.inv();
    const float3 c = T_world_ref * make_float3(0.0f, 0.0f, 1.1f);
    const float s = 0.02f, origin[3] = {c.x - 0.5f * G * s, c.y - 0.5f * G * s, c.z - 0.5f * G * s};
    rmd::TsdfVolume vol(G, G, G, s, origin, 4 * s, 64.0f);
    vol.integrate(seeds);
    // the next keyframe, twice: through the facade and through the C-ABI
    const Frame fK = render(scene, W, H, N + 1);
    rmd::SeedMatrix facade(W, H, cam), capi(W, H, cam);
    facade.setReferenceImage(const_cast<float*>(fK.img.data()), fK.T_curr_world, min_d, max_d);
    capi.setReferenceImage(const_cast<float*>(fK.img.data()), fK.T_curr_world, min_d, max_d);
    vol.seedPrior(facade, f);
    CHECK(rmd_volume_prior_seeds(vol.handle(), capi.handle(), f) == 0);
    const State A = snapshot(facade, W, H), B = snapshot(capi, W, H);
    CHECK(same_bits(A.mu, B.mu));
    CHECK(same_bits(A.sigma_sq, B.sigma_sq));
    CHECK(same_bits(A.a, B.a));
    CHECK(same_bits(A.b, B.b));
    CHECK(A.conv == B.conv);
    // a seed that took the prior holds its pixel's raycast depth
    rmd::DeviceImage<float> ray(W, H);
    vol.raycast(W, H, cam, fK.T_curr_world, ray.data, ray.pitch);
    vol.sync();
    std::vector<float> depth((size_t)W * H);
    ray.getDevData(depth.data());
    const float uniform = A.sigma_sq[0];   // pixel (0, 0) is BORDER: the uniform prior's sigma^2
    size_t applied = 0, wrong = 0;
    for(size_t i = 0; i < depth.size(); ++i)
    {
      if(A.sigma_sq[i] == uniform)
        continue;
      ++applied;
      wrong += !(std::memcmp(&A.mu[i], &depth[i], sizeof(float)) == 0 && A.a[i] == 10.0f && A.b[i] == 10.0f &&
                 A.sigma_sq[i] == f * uniform && A.conv[i] == rmd::ConvergenceStates::UPDATE);
    }
    CHECK(applied > (size_t)W * H / 20);
    CHECK(wrong == 0);
    std::printf("%zu of %d seeds took the volume prior, %zu differ from the raycast\n", applied, W * H, wrong);
    // refusals
    CHECK(throws([&] { vol.seedPrior(facade, 0.0f); }));
    CHECK(throws([&] { vol.seedPrior(facade, 1.5f); }));
    rmd::SeedMatrix no_ref(W, H, cam);
    CHECK(throws([&] { vol.seedPrior(no_ref, f); }));
    facade.update(const_cast<float*>(f0.img.data()), fK.T_curr_world);
    CHECK(throws([&] { vol.seedPrior(facade, f); }));
  }
  catch(const rmd::CudaException &e)
  {
    std::printf("unexpected CudaException: %s\n", e.what());
    ++g_failures;
  }
  rmd_synth_destroy(scene);
  std::printf(g_failures ? "FAILED (%d)\n" : "ALL VOLUME PRIOR TESTS PASSED\n", g_failures);
  return g_failures ? 1 : 0;
}
