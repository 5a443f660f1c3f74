// prior_test.cpp -- the keyframe-prior members of rmd::SeedMatrix (include/rmd/seed_matrix.cuh):
// setPriorPropagation (in place) and propagatePriorFrom (cross-handle) give the same seeds, and the
// C-ABI's refusals surface as rmd::CudaException.
//
// Build (tests/test_cpp_prior.py does this):
//   g++ -std=c++14 -DRMD_BUILD_TESTS=1 -Iinclude -I/usr/local/cuda/include tests/cpp/prior_test.cpp \
//       -Lrpg_open_remode_b200 -lrmd_b200 -Lrpg_open_remode_b200/synth -lrmd_synth -L/usr/local/cuda/lib64 -lcudart
#include <cstdint>
#include <cstdio>
#include <vector>

#include <rmd/se3.cuh>
#include <rmd/seed_matrix.cuh>

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
  const int W = 160, H = 120, N = 40;
  const rmd::PinholeCamera cam(481.2f * W / 640.0f, -480.0f * H / 480.0f, (W - 1) / 2.0f, (H - 1) / 2.0f);
  void *scene = rmd_synth_create(W, H, cam.fx, cam.fy, cam.cx, cam.cy, 0x5EED0001u);
  const size_t n = (size_t)W * H;
  const float min_d = 0.4f, max_d = 1.8f, frac = 1.0f / 16.0f;
  try
  {
    rmd::SeedMatrix in_place(W, H, cam), source(W, H, cam), fresh(W, H, cam);
    in_place.setPriorPropagation(frac);
    for(rmd::SeedMatrix *s : {&in_place, &source})
    {
      const Frame f0 = render(scene, W, H, 0);
      s->setReferenceImage(const_cast<float*>(f0.img.data()), f0.T_curr_world, min_d, max_d);
      for(int k = 1; k <= N; ++k)
      {
        const Frame f = render(scene, W, H, k);
        s->update(const_cast<float*>(f.img.data()), f.T_curr_world);
      }
    }
    CHECK(source.getConvergedCount() > n / 20);
    const Frame fk = render(scene, W, H, N + 1);
    in_place.setReferenceImage(const_cast<float*>(fk.img.data()), fk.T_curr_world, min_d, max_d);
    fresh.setReferenceImage(const_cast<float*>(fk.img.data()), fk.T_curr_world, min_d, max_d);
    fresh.propagatePriorFrom(source, frac);
    std::vector<float> mu_a(n), mu_b(n), s2_a(n), s2_b(n);
    in_place.downloadDepthmap(mu_a.data()); fresh.downloadDepthmap(mu_b.data());
    in_place.downloadSigmaSq(s2_a.data()); fresh.downloadSigmaSq(s2_b.data());
    CHECK(mu_a == mu_b);
    CHECK(s2_a == s2_b);
    const float sigma_sq_max = (max_d - min_d) * (max_d - min_d) / 36.0f;
    size_t with_prior = 0;
    for(size_t i = 0; i < n; ++i) with_prior += (s2_b[i] == frac * sigma_sq_max);
    CHECK(with_prior > n / 100);
    std::printf("prior on %zu of %zu pixels\n", with_prior, n);
    // refusals: f out of range, src == dst, dst updated since its reference
    CHECK(throws([&] { fresh.setPriorPropagation(1.5f); }));
    CHECK(throws([&] { fresh.propagatePriorFrom(source, 0.0f); }));
    CHECK(throws([&] { fresh.propagatePriorFrom(fresh, frac); }));
    fresh.update(const_cast<float*>(fk.img.data()), fk.T_curr_world);
    CHECK(throws([&] { fresh.propagatePriorFrom(source, frac); }));
  }
  catch(const rmd::CudaException &e)
  {
    std::printf("unexpected CudaException: %s\n", e.what());
    ++g_failures;
  }
  rmd_synth_destroy(scene);
  std::printf(g_failures ? "FAILED (%d)\n" : "ALL PRIOR TESTS PASSED\n", g_failures);
  return g_failures ? 1 : 0;
}
