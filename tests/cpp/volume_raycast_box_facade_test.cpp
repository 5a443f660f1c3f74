// volume_raycast_box_facade_test.cpp -- the box raycasts and box prior of rmd::TsdfVolume
// (include/rmd/tsdf_volume.cuh): a sphere fused with intensity from a camera inside it into a 64^3 volume with the
// brick store.  Checks that the window box (0, n) gives raycast(), raycastIntensity(), raycastNormals() and
// seedPrior() bit for bit; then shifts the window 20 voxels along -z, so that the shell in front of the camera lies in
// the store only, and checks that the window rays miss it where the box (-4, -4, -4) + (72, 72, 92) sees it.  Writes
// the box's depth, intensity, normals and prior mu to argv[1], which tests/test_cpp_volume_raycast_box.py compares
// with the same scene run through the Python API.
//
// Build (tests/test_cpp_volume_raycast_box.py does this):
//   g++ -std=c++14 -DRMD_BUILD_TESTS=1 -Iinclude -I/usr/local/cuda/include \
//       tests/cpp/volume_raycast_box_facade_test.cpp -Lrpg_open_remode_b200 -lrmd_b200 -L/usr/local/cuda/lib64 -lcudart
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include <rmd/device_image.cuh>
#include <rmd/se3.cuh>
#include <rmd/seed_matrix.cuh>
#include <rmd/tsdf_volume.cuh>

static int g_failures = 0;
#define CHECK(cond)                                                                  \
  do {                                                                               \
    if(!(cond)) { std::printf("CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++g_failures; } \
  } while(0)

struct Views
{
  std::vector<float> depth, inten, normals, mu;
};

static bool same(const std::vector<float> &a, const std::vector<float> &b)
{
  return a.size() == b.size() && std::memcmp(a.data(), b.data(), a.size() * sizeof(float)) == 0;
}

int main(int argc, char **argv)
{
  if(argc < 2)
  {
    std::printf("usage: %s out.bin\n", argv[0]);
    return 2;
  }
  const int N = 64, W = 160, H = 120;
  const float s = 0.0625f, origin[3] = {-2.0f, -2.0f, -2.0f}, R = 1.2f, tau = 4 * s, f = 1.0f / 16.0f;
  const rmd::PinholeCamera cam(100.0f, 100.0f, (W - 1) / 2.0f, (H - 1) / 2.0f);
  float r[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {0.0f, 0.0f, 0.0f};
  const rmd::SE3<float> T_curr_world(r, t);   // a camera at the sphere's centre, looking along +z
  std::vector<float> depth((size_t)W * H, R), image((size_t)W * H, 0.5f);
  rmd::DeviceImage<float> d_depth(W, H), d_image(W, H), ray(W, H), inten(W, H), normals(4 * W, H);
  d_depth.setDevData(depth.data());
  d_image.setDevData(image.data());

  rmd::TsdfVolume vol(N, N, N, s, origin, tau, 16.0f);
  vol.enableIntensity();
  vol.enableStore();
  vol.integrateDepthIntensity(W, H, cam, T_curr_world, d_depth.data, d_depth.pitch, d_image.data, d_image.pitch);

  const size_t n_pix = (size_t)W * H;
  // box: NULL = the window's entry points
  auto views = [&](const int64_t *lo, const int *dims) {
    Views V;
    V.depth.resize(n_pix); V.inten.resize(n_pix); V.normals.resize(4 * n_pix); V.mu.resize(n_pix);
    std::vector<float> d2(n_pix), d3(n_pix);
    if(lo)
    {
      vol.raycast(W, H, cam, T_curr_world, ray.data, ray.pitch, lo, dims);
      vol.sync();
      ray.getDevData(V.depth.data());
      vol.raycastIntensity(W, H, cam, T_curr_world, ray.data, ray.pitch, inten.data, inten.pitch, lo, dims);
      vol.sync();
      ray.getDevData(d2.data());
      vol.raycastNormals(W, H, cam, T_curr_world, ray.data, ray.pitch, normals.data, normals.pitch, lo, dims);
    }
    else
    {
      vol.raycast(W, H, cam, T_curr_world, ray.data, ray.pitch);
      vol.sync();
      ray.getDevData(V.depth.data());
      vol.raycastIntensity(W, H, cam, T_curr_world, ray.data, ray.pitch, inten.data, inten.pitch);
      vol.sync();
      ray.getDevData(d2.data());
      vol.raycastNormals(W, H, cam, T_curr_world, ray.data, ray.pitch, normals.data, normals.pitch);
    }
    vol.sync();
    ray.getDevData(d3.data());
    inten.getDevData(V.inten.data());
    normals.getDevData(V.normals.data());
    CHECK(same(V.depth, d2) && same(V.depth, d3));   // every variant writes the plain rays' depth
    rmd::SeedMatrix seeds(W, H, cam);
    seeds.setReferenceImage(image.data(), T_curr_world, 0.5f, 2.0f);
    if(lo)
      vol.seedPrior(seeds, f, lo, dims);
    else
      vol.seedPrior(seeds, f);
    seeds.downloadDepthmap(V.mu.data());
    return V;
  };

  const int64_t zero[3] = {0, 0, 0};
  const int n3[3] = {N, N, N};
  const Views win = views(NULL, NULL), win_box = views(zero, n3);
  CHECK(same(win.depth, win_box.depth) && same(win.inten, win_box.inten) && same(win.normals, win_box.normals) &&
        same(win.mu, win_box.mu));
  const size_t centre = (size_t)(H / 2) * W + W / 2;
  CHECK(std::fabs(win.depth[centre] - R) < s && std::fabs(win.inten[centre] - 0.5f) < 1e-5f);
  CHECK(win.mu[centre] == win.depth[centre]);

  // the window then covers z <= 0.6875 m: the shell ahead of the camera is in the store only
  vol.shift(0, 0, -20);
  const int64_t lo[3] = {-4, -4, -4};
  const int m[3] = {N + 8, N + 8, N + 28};
  const Views moved = views(NULL, NULL), box = views(lo, m);
  CHECK(moved.depth[centre] == 0.0f && moved.inten[centre] == -1.0f);
  CHECK(std::fabs(box.depth[centre] - R) < s && std::fabs(box.inten[centre] - 0.5f) < 1e-5f);
  CHECK(box.mu[centre] == box.depth[centre] && moved.mu[centre] != box.mu[centre]);
  CHECK(std::fabs(box.normals[4 * centre + 2] + 1.0f) < 0.05f);   // the shell faces the camera at its centre

  bool threw = false;
  const int big[3] = {65536, 1, 1};
  try { vol.raycast(W, H, cam, T_curr_world, ray.data, ray.pitch, lo, big); }
  catch(const rmd::CudaException &) { threw = true; }
  CHECK(threw);

  FILE *out = std::fopen(argv[1], "wb");
  CHECK(out != NULL);
  if(out)
  {
    std::fwrite(box.depth.data(), sizeof(float), n_pix, out);
    std::fwrite(box.inten.data(), sizeof(float), n_pix, out);
    std::fwrite(box.normals.data(), sizeof(float), 4 * n_pix, out);
    std::fwrite(box.mu.data(), sizeof(float), n_pix, out);
    std::fclose(out);
  }

  if(g_failures)
  {
    std::printf("%d FAILURES\n", g_failures);
    return 1;
  }
  std::printf("ALL VOLUME RAYCAST BOX TESTS PASSED\n");
  return 0;
}
