// rmd/tsdf_volume.cuh -- rmd::TsdfVolume: fusion of finished keyframes into a dense TSDF voxel grid
// (DESIGN.md 4.8).  The reference has no such class; this one is a host-only forwarder to the C-ABI
// (rmd_volume_*, include/rmd_b200.h) that throws rmd::CudaException on failure, like rmd::SeedMatrix.
#ifndef TSDF_VOLUME_CUH
#define TSDF_VOLUME_CUH

#include <cstddef>
#include <cstdint>
#include <vector>

#include <rmd/pinhole_camera.cuh>
#include <rmd/se3.cuh>
#include <rmd/seed_matrix.cuh>

namespace rmd
{

class TsdfVolume
{
public:
  // nx * ny * nz voxels (x fastest) of edge voxel_size; origin = world position of the centre of voxel (0, 0, 0).
  TsdfVolume(int nx, int ny, int nz, float voxel_size, const float origin[3], float truncation, float max_weight,
             int device = -1)
    : handle_(NULL)
  {
    detail::throw_on_error(rmd_volume_create(nx, ny, nz, voxel_size, origin, truncation, max_weight, device, &handle_),
                           "TsdfVolume: unable to create");
  }

  ~TsdfVolume() { rmd_volume_destroy(handle_); }

  // A finished keyframe: the CONVERGED seeds of `seeds` at the pose their reference was set with; depth = their mu
  // (dev_depth NULL) or a pitched device image such as rmd::DepthmapDenoiser's output.
  void integrate(const SeedMatrix &seeds, const float *dev_depth = NULL, size_t depth_pitch = 0)
  {
    detail::throw_on_error(rmd_volume_integrate_seeds(handle_, seeds.handle(), dev_depth, depth_pitch),
                           "TsdfVolume: unable to integrate the keyframe");
  }

  // Any depth image on the device; dev_conv NULL = every finite positive depth counts.
  void integrateDepth(int width, int height, const PinholeCamera &cam, const SE3<float> &T_curr_world,
                      const float *dev_depth, size_t depth_pitch, const int *dev_conv = NULL, size_t conv_pitch = 0)
  {
    detail::throw_on_error(rmd_volume_integrate_depth(handle_, width, height, cam.fx, cam.fy, cam.cx, cam.cy,
                                                      T_curr_world.data.data, dev_depth, depth_pitch, dev_conv,
                                                      conv_pitch),
                           "TsdfVolume: unable to integrate the depth image");
  }

  // (x, y, z, weight) of every surface point, 4 floats per point.
  std::vector<float> surfacePoints()
  {
    size_t n = 0;
    detail::throw_on_error(rmd_volume_surface_points(handle_, NULL, 0, &n), "TsdfVolume: unable to count points");
    std::vector<float> out(4 * n);
    if(n)
      detail::throw_on_error(rmd_volume_surface_points(handle_, out.data(), n, &n),
                             "TsdfVolume: unable to extract points");
    out.resize(4 * n < out.size() ? 4 * n : out.size());
    return out;
  }

  // Triangle mesh of the fused surface: xyzw = surfacePoints() (4 floats per vertex), tri = 3 vertex indices per
  // triangle, (b - a) x (c - a) towards free space.  Throws for 2^31 or more vertices.
  void mesh(std::vector<float> &xyzw, std::vector<int32_t> &tri)
  {
    size_t nv = 0, nt = 0;
    detail::throw_on_error(rmd_volume_mesh(handle_, NULL, 0, NULL, 0, &nv, &nt), "TsdfVolume: unable to count the mesh");
    xyzw.resize(4 * nv);
    tri.resize(3 * nt);
    if(nv || nt)
      detail::throw_on_error(rmd_volume_mesh(handle_, xyzw.data(), nv, tri.data(), nt, &nv, &nt),
                             "TsdfVolume: unable to extract the mesh");
    xyzw.resize(4 * nv < xyzw.size() ? 4 * nv : xyzw.size());
    tri.resize(3 * nt < tri.size() ? 3 * nt : tri.size());
  }

  // Distance along each pixel's ray to the fused surface (0 = none) into a pitched device image; asynchronous on
  // the volume's stream (sync() before another stream reads it).
  void raycast(int width, int height, const PinholeCamera &cam, const SE3<float> &T_curr_world, float *dev_depth,
               size_t depth_pitch)
  {
    detail::throw_on_error(rmd_volume_raycast(handle_, width, height, cam.fx, cam.fy, cam.cx, cam.cy,
                                              T_curr_world.data.data, dev_depth, depth_pitch),
                           "TsdfVolume: unable to raycast");
  }

  // Right after seeds.setReferenceImage (no update since): the new keyframe's depth prior from the fused model --
  // every non-BORDER pixel whose ray hits the surface within the seeds' depth range gets (hit, sigma_sq_frac *
  // range^2 / 36, 10, 10); the other seeds are left as they are.  Asynchronous, ordered after the volume's queued
  // work.
  void seedPrior(SeedMatrix &seeds, float sigma_sq_frac)
  {
    detail::throw_on_error(rmd_volume_prior_seeds(handle_, seeds.handle(), sigma_sq_frac),
                           "TsdfVolume: unable to seed the keyframe prior");
  }

  // Intensity channel (8 B per voxel): from now on integrate() also fuses the keyframe's reference image.
  void enableIntensity()
  {
    detail::throw_on_error(rmd_volume_enable_intensity(handle_), "TsdfVolume: unable to enable the intensity");
  }

  // integrateDepth plus a float intensity image of the same size, fused into the intensity channel.
  void integrateDepthIntensity(int width, int height, const PinholeCamera &cam, const SE3<float> &T_curr_world,
                               const float *dev_depth, size_t depth_pitch, const float *dev_intensity,
                               size_t intensity_pitch, const int *dev_conv = NULL, size_t conv_pitch = 0)
  {
    detail::throw_on_error(rmd_volume_integrate_depth_intensity(handle_, width, height, cam.fx, cam.fy, cam.cx, cam.cy,
                                                                T_curr_world.data.data, dev_depth, depth_pitch,
                                                                dev_conv, conv_pitch, dev_intensity,
                                                                intensity_pitch),
                           "TsdfVolume: unable to integrate the depth and intensity images");
  }

  // One intensity per surface point (= mesh vertex), in surfacePoints() order; -1 = none.
  std::vector<float> surfaceIntensity()
  {
    size_t n = 0;
    detail::throw_on_error(rmd_volume_surface_intensity(handle_, NULL, 0, &n), "TsdfVolume: unable to count points");
    std::vector<float> out(n);
    if(n)
      detail::throw_on_error(rmd_volume_surface_intensity(handle_, out.data(), n, &n),
                             "TsdfVolume: unable to extract the intensities");
    out.resize(n < out.size() ? n : out.size());
    return out;
  }

  // raycast() and the intensity at each hit (-1 = none) into two pitched device images; asynchronous.
  void raycastIntensity(int width, int height, const PinholeCamera &cam, const SE3<float> &T_curr_world,
                        float *dev_depth, size_t depth_pitch, float *dev_intensity, size_t intensity_pitch)
  {
    detail::throw_on_error(rmd_volume_raycast_intensity(handle_, width, height, cam.fx, cam.fy, cam.cx, cam.cy,
                                                        T_curr_world.data.data, dev_depth, depth_pitch,
                                                        dev_intensity, intensity_pitch),
                           "TsdfVolume: unable to raycast the intensity");
  }

  // One unit normal (nx, ny, nz, 0) per surface point (= mesh vertex), in surfacePoints() order, towards free space;
  // (0, 0, 0, 0) where the tsdf gradient vanishes.
  std::vector<float> surfaceNormals()
  {
    size_t n = 0;
    detail::throw_on_error(rmd_volume_surface_normals(handle_, NULL, 0, &n), "TsdfVolume: unable to count points");
    std::vector<float> out(4 * n);
    if(n)
      detail::throw_on_error(rmd_volume_surface_normals(handle_, out.data(), n, &n),
                             "TsdfVolume: unable to extract the normals");
    out.resize(4 * n < out.size() ? 4 * n : out.size());
    return out;
  }

  // raycast() and the world-frame normal at each hit ((0, 0, 0, 0) = none) into a pitched device image of float4
  // (normals_pitch a multiple of 16 bytes); asynchronous.
  void raycastNormals(int width, int height, const PinholeCamera &cam, const SE3<float> &T_curr_world,
                      float *dev_depth, size_t depth_pitch, float *dev_normals, size_t normals_pitch)
  {
    detail::throw_on_error(rmd_volume_raycast_normals(handle_, width, height, cam.fx, cam.fy, cam.cx, cam.cy,
                                                      T_curr_world.data.data, dev_depth, depth_pitch, dev_normals,
                                                      normals_pitch),
                           "TsdfVolume: unable to raycast the normals");
  }

  // Moving volume: voxel (i, j, k) then holds what (i + dx, j + dy, k + dz) held (unknown outside the grid), and the
  // origin moves by d * voxel_size.  Asynchronous on the volume's stream; the first shift that moves records doubles
  // the record memory.  Take the spill (below) first.
  void shift(int dx, int dy, int dz)
  {
    const int d[3] = {dx, dy, dz};
    detail::throw_on_error(rmd_volume_shift(handle_, d), "TsdfVolume: unable to shift");
  }

  // The points a shift by d would drop, as the subsequence of surfacePoints() / surfaceIntensity() / surfaceNormals()
  // in their order; call before shift(d).
  std::vector<float> spillPoints(const int d[3]) { return spill(rmd_volume_spill_points, d, 4); }
  std::vector<float> spillIntensity(const int d[3]) { return spill(rmd_volume_spill_intensity, d, 1); }
  std::vector<float> spillNormals(const int d[3]) { return spill(rmd_volume_spill_normals, d, 4); }

  // The mesh a shift by d would drop (call before shift(d)): the triangles of the meshed cubes with a corner leaving
  // the grid, in mesh() order, indexing xyzw = the subsequence of surfacePoints() they need plus the points that
  // spill (4 floats per vertex); ids = (i + D0, j + D1, k + D2, axis) per vertex (4 int64), the vertex's identity
  // across shifts.  Throws for 2^31 or more vertices.
  void spillMesh(const int d[3], std::vector<float> &xyzw, std::vector<int32_t> &tri, std::vector<int64_t> &ids)
  {
    size_t nv = 0, nt = 0;
    detail::throw_on_error(rmd_volume_spill_mesh(handle_, d, NULL, 0, NULL, 0, NULL, &nv, &nt),
                           "TsdfVolume: unable to count the spill mesh");
    xyzw.resize(4 * nv);
    tri.resize(3 * nt);
    ids.resize(4 * nv);
    if(nv || nt)
      detail::throw_on_error(rmd_volume_spill_mesh(handle_, d, xyzw.data(), nv, tri.data(), nt, ids.data(), &nv, &nt),
                             "TsdfVolume: unable to extract the spill mesh");
    xyzw.resize(4 * nv < xyzw.size() ? 4 * nv : xyzw.size());
    ids.resize(4 * nv < ids.size() ? 4 * nv : ids.size());
    tri.resize(3 * nt < tri.size() ? 3 * nt : tri.size());
  }
  // surfaceIntensity() / surfaceNormals() of the spill mesh's vertices, in their order.
  std::vector<float> spillMeshIntensity(const int d[3]) { return spill(rmd_volume_spill_mesh_intensity, d, 1); }
  std::vector<float> spillMeshNormals(const int d[3]) { return spill(rmd_volume_spill_mesh_normals, d, 4); }

  // The ids of surfacePoints() (= mesh() vertices), 4 int64 per point, as spillMesh's.
  std::vector<int64_t> surfaceIds()
  {
    size_t n = 0;
    detail::throw_on_error(rmd_volume_surface_ids(handle_, NULL, 0, &n), "TsdfVolume: unable to count points");
    std::vector<int64_t> out(4 * n);
    if(n)
      detail::throw_on_error(rmd_volume_surface_ids(handle_, out.data(), n, &n), "TsdfVolume: unable to extract ids");
    out.resize(4 * n < out.size() ? 4 * n : out.size());
    return out;
  }

  // The total offset in voxels, the sum of all shifts.
  void offset(int64_t D[3]) { detail::throw_on_error(rmd_volume_offset(handle_, D), "TsdfVolume: unable to read the offset"); }

  // Brick store: shift() then keeps the 8x8x8 bricks that leave the grid with a known voxel and restores the voxels
  // that re-enter (shift(d) then shift(-d) is lossless); each such shift synchronises the volume's stream once.
  void enableStore() { detail::throw_on_error(rmd_volume_enable_store(handle_), "TsdfVolume: unable to enable the store"); }
  // The number of stored bricks and the device bytes of the store's pool.
  void storeInfo(size_t *bricks, size_t *bytes)
  {
    detail::throw_on_error(rmd_volume_store_info(handle_, bricks, bytes), "TsdfVolume: unable to read the store");
  }
  // The stored bricks in ascending (z, y, x): 3 int64 coordinates and 512 records (x fastest) per brick; voxels inside
  // the grid are (0, 0).  intensity / intensity_weight (NULL: not wanted) need the intensity channel.
  void downloadStore(std::vector<int64_t> &coords, std::vector<float> &tsdf, std::vector<float> &weight,
                     std::vector<float> *intensity = NULL, std::vector<float> *intensity_weight = NULL)
  {
    size_t n = 0;
    detail::throw_on_error(rmd_volume_download_store(handle_, NULL, NULL, NULL, NULL, NULL, 0, &n),
                           "TsdfVolume: unable to count the stored bricks");
    coords.resize(3 * n);
    tsdf.resize(512 * n);
    weight.resize(512 * n);
    if(intensity) intensity->resize(512 * n);
    if(intensity_weight) intensity_weight->resize(512 * n);
    if(n)
      detail::throw_on_error(rmd_volume_download_store(handle_, coords.data(), tsdf.data(), weight.data(),
                                                       intensity ? intensity->data() : NULL,
                                                       intensity_weight ? intensity_weight->data() : NULL, n, &n),
                             "TsdfVolume: unable to download the store");
  }
  // Replaces the store with n bricks laid out as downloadStore's (intensity pair optional).
  void uploadStore(const int64_t *coords, const float *tsdf, const float *weight, size_t n,
                   const float *intensity = NULL, const float *intensity_weight = NULL)
  {
    detail::throw_on_error(rmd_volume_upload_store(handle_, coords, tsdf, weight, intensity, intensity_weight, n),
                           "TsdfVolume: unable to upload the store");
  }

  void downloadIntensity(float *host_intensity, float *host_weight)
  {
    detail::throw_on_error(rmd_volume_download_intensity(handle_, host_intensity, host_weight),
                           "TsdfVolume: unable to download the intensity");
  }
  void uploadIntensity(const float *host_intensity, const float *host_weight)
  {
    detail::throw_on_error(rmd_volume_upload_intensity(handle_, host_intensity, host_weight),
                           "TsdfVolume: unable to upload the intensity");
  }

  void download(float *host_tsdf, float *host_weight)
  {
    detail::throw_on_error(rmd_volume_download(handle_, host_tsdf, host_weight), "TsdfVolume: unable to download");
  }
  void upload(const float *host_tsdf, const float *host_weight)
  {
    detail::throw_on_error(rmd_volume_upload(handle_, host_tsdf, host_weight), "TsdfVolume: unable to upload");
  }
  void reset() { detail::throw_on_error(rmd_volume_reset(handle_), "TsdfVolume: unable to reset"); }
  void setStream(cudaStream_t stream)
  {
    detail::throw_on_error(rmd_volume_set_stream(handle_, stream), "TsdfVolume: unable to set the stream");
  }
  void sync() { detail::throw_on_error(rmd_volume_sync(handle_), "TsdfVolume: unable to synchronise"); }

  rmd_volume_t *handle() const { return handle_; }

private:
  TsdfVolume(const TsdfVolume &);
  TsdfVolume &operator=(const TsdfVolume &);

  typedef int (*SpillFn)(rmd_volume_t *, const int *, float *, size_t, size_t *);
  std::vector<float> spill(SpillFn fn, const int d[3], size_t floats_per_point)
  {
    size_t n = 0;
    detail::throw_on_error(fn(handle_, d, NULL, 0, &n), "TsdfVolume: unable to count the spill");
    std::vector<float> out(floats_per_point * n);
    if(n)
      detail::throw_on_error(fn(handle_, d, out.data(), n, &n), "TsdfVolume: unable to extract the spill");
    out.resize(floats_per_point * n < out.size() ? floats_per_point * n : out.size());
    return out;
  }

  rmd_volume_t *handle_;
};

} // rmd namespace

#endif // TSDF_VOLUME_CUH
