// volume_spill_mesh_test.cpp -- the spill mesh of a moving rmd::TsdfVolume (include/rmd/tsdf_volume.cuh): a sphere
// fused from a camera inside it; the facade's spill mesh equals the C-ABI's, its triangles index its vertices, its
// ids carry the offset, the spill mesh and the mesh after the shift share seam ids, and a null offset throws.  The
// outputs go to the file named by argv[1], which tests/test_cpp_volume_spill_mesh.py compares with the Python path.
//
// Build (tests/test_cpp_volume_spill_mesh.py does this):
//   g++ -std=c++14 -DRMD_BUILD_TESTS=1 -Iinclude -I/usr/local/cuda/include tests/cpp/volume_spill_mesh_test.cpp \
//       -Lrpg_open_remode_b200 -lrmd_b200 -L/usr/local/cuda/lib64 -lcudart
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <set>
#include <vector>

#include <rmd/device_image.cuh>
#include <rmd/se3.cuh>
#include <rmd/tsdf_volume.cuh>

static int g_failures = 0;
#define CHECK(cond)                                                                  \
  do {                                                                               \
    if(!(cond)) { std::printf("CHECK FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); ++g_failures; } \
  } while(0)

template<typename T>
static void dump(std::FILE *f, const std::vector<T> &v)
{
  const uint64_t n = v.size();
  std::fwrite(&n, sizeof(n), 1, f);
  if(n) std::fwrite(v.data(), sizeof(T), v.size(), f);
}

int main(int argc, char **argv)
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
  vol.shift(2, 0, -1);   // a non-zero offset, so that the ids carry it
  vol.sync();

  const int d[3] = {26, -7, -14};
  std::vector<float> xyzw;
  std::vector<int32_t> tri;
  std::vector<int64_t> ids;
  vol.spillMesh(d, xyzw, tri, ids);
  const std::vector<float> inten_s = vol.spillMeshIntensity(d);
  const std::vector<float> normals_s = vol.spillMeshNormals(d);
  const size_t nv = xyzw.size() / 4;
  CHECK(nv > 100 && tri.size() > 3 * 100 && ids.size() == 4 * nv);
  CHECK(inten_s.size() == nv && normals_s.size() == 4 * nv);
  bool in_range = true;
  for(int32_t x : tri) in_range = in_range && x >= 0 && (size_t)x < nv;
  CHECK(in_range);
  // the facade == the C-ABI
  size_t cv = 0, ct = 0;
  CHECK(rmd_volume_spill_mesh(vol.handle(), d, NULL, 0, NULL, 0, NULL, &cv, &ct) == 0);
  CHECK(cv == nv && 3 * ct == tri.size());
  std::vector<float> raw(4 * cv);
  std::vector<int32_t> raw_t(3 * ct);
  CHECK(rmd_volume_spill_mesh(vol.handle(), d, raw.data(), cv, raw_t.data(), ct, NULL, &cv, &ct) == 0);
  CHECK(std::memcmp(raw.data(), xyzw.data(), raw.size() * sizeof(float)) == 0);
  CHECK(std::memcmp(raw_t.data(), tri.data(), raw_t.size() * sizeof(int32_t)) == 0);
  int64_t D[3];
  vol.offset(D);
  CHECK(D[0] == 2 && D[1] == 0 && D[2] == -1);
  bool ids_ok = true;
  for(size_t q = 0; q < nv; ++q)
    ids_ok = ids_ok && ids[4 * q] >= D[0] && ids[4 * q] < D[0] + N && ids[4 * q + 3] >= 0 && ids[4 * q + 3] < 3;
  CHECK(ids_ok);

  const std::vector<int64_t> surf_ids = vol.surfaceIds();
  CHECK(surf_ids.size() == vol.surfacePoints().size());
  vol.shift(d[0], d[1], d[2]);
  const std::vector<int64_t> after_ids = vol.surfaceIds();
  std::set<std::vector<int64_t> > spill_set, after_set, before_set;
  for(size_t q = 0; q < nv; ++q) spill_set.insert(std::vector<int64_t>(&ids[4 * q], &ids[4 * q + 4]));
  for(size_t q = 0; q < after_ids.size() / 4; ++q)
    after_set.insert(std::vector<int64_t>(&after_ids[4 * q], &after_ids[4 * q + 4]));
  for(size_t q = 0; q < surf_ids.size() / 4; ++q)
    before_set.insert(std::vector<int64_t>(&surf_ids[4 * q], &surf_ids[4 * q + 4]));
  size_t seam = 0;
  for(const std::vector<int64_t> &x : spill_set) seam += after_set.count(x);
  CHECK(seam > 0);
  CHECK(spill_set.size() + after_set.size() - seam == before_set.size());   // every vertex once

  bool threw = false;
  try { vol.spillMesh(NULL, xyzw, tri, ids); }
  catch(const rmd::CudaException &) { threw = true; }
  CHECK(threw);

  if(argc > 1)
  {
    std::FILE *f = std::fopen(argv[1], "wb");
    CHECK(f != NULL);
    if(f)
    {
      dump(f, raw);
      dump(f, raw_t);
      dump(f, ids);
      dump(f, inten_s);
      dump(f, normals_s);
      dump(f, after_ids);
      std::fclose(f);
    }
  }
  if(g_failures)
  {
    std::printf("%d FAILURES\n", g_failures);
    return 1;
  }
  std::printf("ALL VOLUME SPILL MESH TESTS PASSED\n");
  return 0;
}
