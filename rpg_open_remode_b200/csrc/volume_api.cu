// volume_api.cu -- the C-ABI of the TSDF volume (rmd_volume_*, include/rmd_b200.h; DESIGN.md 4.8): the handle,
// argument checks, scratch and staging buffers, and the host sequencing of the kernels in volume.cu.
// rmd_volume_integrate_seeds and rmd_volume_prior_seeds are in c_api.cu, next to the seeds' internals they read.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <new>
#include <string>
#include <vector>

#include "rmd_common.cuh"
#include "volume.cuh"
#include "volume_store.h"

namespace rmdb
{

static_assert(STORE_BRICK_VOXELS == VOLUME_STORE_VOXELS, "one brick size on host and device");

// The brick store (DESIGN.md 4.8): the host index, the device pool of cap bricks (pool_col with the intensity
// channel) and the per-shift scratch: the bricks the kernels visit and the flag kernel's flags.
struct VolumeStore
{
  BrickIndex index;
  float2 *pool, *pool_col;
  size_t cap;
  VolumeStoreBrick *bricks; size_t bricks_cap;
  int *flags; size_t flags_cap;
};

int volume_integrate(rmd_volume *v, VolumeIntegrateParams &P)
{
  P.g = v->g;
  P.trunc = v->trunc; P.max_weight = v->max_weight;
  P.col = P.intensity ? v->col : NULL;
  RMD_CUDA_TRY(launch_volume_integrate(P, v->stream));
  return 0;
}

} // namespace rmdb

using namespace rmdb;

namespace
{

const size_t kVolumeMaxVoxels = (size_t)1 << 31;
const size_t kVolumeChunk = (size_t)1 << 24;   // voxels per host staging chunk of download / upload

// Argument check of an entry point whose name is `what`.
#define VOLUME_REQUIRE(cond, msg)                                                                  \
  do {                                                                                             \
    if(!(cond))                                                                                    \
      return fail(RMD_ERR_INVALID_ARGUMENT, (std::string(what) + ": " + (msg)).c_str());           \
  } while(0)

int no_intensity(const char *what)
{
  return fail(RMD_ERR_NOT_INITIALISED, (std::string(what) + ": the volume has no intensity channel").c_str());
}

// Device buffer of at least n elements, grown (never shrunk) on demand.
template<typename T>
int volume_grow(T **buf, size_t *cap, size_t n)
{
  if(n <= *cap)
    return 0;
  RMD_CUDA_TRY(cudaFree(*buf));
  *buf = NULL; *cap = 0;
  RMD_CUDA_TRY(cudaMalloc(buf, sizeof(T) * n));
  *cap = n;
  return 0;
}

// The surface points' pass parameters on v's grid, with the per-block offsets and total (allocated on first use).
int volume_surface_params(rmd_volume *v, VolumeSurfaceParams &P)
{
  memset(&P, 0, sizeof(P));
  P.g = v->g;
  P.b.n_blocks = (unsigned int)((v->n_vox + VOLUME_SURF_VOXELS - 1) / VOLUME_SURF_VOXELS);
  if(!v->surf_offsets)
  {
    RMD_CUDA_TRY(cudaMalloc(&v->surf_offsets, sizeof(unsigned long long) * P.b.n_blocks));
    RMD_CUDA_TRY(cudaMalloc(&v->surf_total, sizeof(unsigned long long)));
  }
  P.b.block_offsets = v->surf_offsets;
  P.b.total = v->surf_total;
  return 0;
}

enum SurfaceOutput { SURFACE_POINTS, SURFACE_INTENSITY, SURFACE_NORMALS };

// The surface points' count pass and scan, one host read of the count, then for min(count, capacity) points their
// write pass (same blocks and ranks): positions (float4), intensities (float) or normals (float4).  With a spill box,
// only the points that spill from it, or with spill_mesh the spill mesh's vertices.  host: staged in v->stage and
// copied to out.  Synchronous.
int volume_surface(rmd_volume *v, void *out, size_t capacity, size_t *count, bool host, SurfaceOutput kind,
                   const VolumeSpillBox *spill = NULL, bool spill_mesh = false)
{
  const bool intensity = kind == SURFACE_INTENSITY;
  VolumeSurfaceParams P;
  int rc = volume_surface_params(v, P);
  if(rc) return rc;
  if(spill && spill_mesh)
    RMD_CUDA_TRY(launch_volume_spill_mesh_count(P, *spill, v->stream));
  else if(spill)
    RMD_CUDA_TRY(launch_volume_spill_count(P, *spill, v->stream));
  else
    RMD_CUDA_TRY(launch_volume_surface_count(P, v->stream));
  unsigned long long total = 0;
  RMD_CUDA_TRY(cudaMemcpyAsync(&total, v->surf_total, sizeof(total), cudaMemcpyDeviceToHost, v->stream));
  RMD_CUDA_TRY(cudaStreamSynchronize(v->stream));
  *count = (size_t)total;
  const size_t n = *count < capacity ? *count : capacity;
  if(!n)
    return 0;
  const size_t bytes = n * (intensity ? sizeof(float) : sizeof(float4));
  void *dst = out;
  if(host)
  {
    rc = volume_grow(&v->stage, &v->stage_cap, bytes);
    if(rc) return rc;
    dst = v->stage;
  }
  P.capacity = n;
  if(intensity)
  {
    P.col = v->col;
    P.intensity = static_cast<float*>(dst);
  }
  else if(kind == SURFACE_NORMALS)
    P.normals = static_cast<float4*>(dst);
  else
    P.out = static_cast<float4*>(dst);
  if(spill && spill_mesh)
    RMD_CUDA_TRY(launch_volume_spill_mesh_write(P, *spill, v->stream));
  else if(spill)
    RMD_CUDA_TRY(launch_volume_spill_write(P, *spill, v->stream));
  else
    RMD_CUDA_TRY(launch_volume_surface_write(P, v->stream));
  if(host)
    RMD_CUDA_TRY(cudaMemcpyAsync(out, v->stage, bytes, cudaMemcpyDeviceToHost, v->stream));
  RMD_CUDA_TRY(cudaStreamSynchronize(v->stream));
  return 0;
}

// The mesh: both count passes and scans, one host read of the two totals, then -- for what the capacities ask --
// the surface points (with their keys when triangles are wanted) and the triangles.  host: min(count, capacity)
// of each are staged in the volume's buffers and copied to xyzw / tri.  Synchronous.
// The surface points' and the triangles' pass parameters on v's grid, with the per-block offsets and totals of both
// (allocated on first use).
int volume_mesh_params(rmd_volume *v, VolumeSurfaceParams &S, VolumeMeshParams &M)
{
  int rc = volume_surface_params(v, S);
  if(rc) return rc;
  if(!v->tri_offsets)
  {
    RMD_CUDA_TRY(cudaMalloc(&v->tri_offsets, sizeof(unsigned long long) * S.b.n_blocks));
    RMD_CUDA_TRY(cudaMalloc(&v->tri_total, sizeof(unsigned long long)));
  }
  memset(&M, 0, sizeof(M));
  M.g = v->g;
  M.point_offsets = v->surf_offsets;
  M.point_total = v->surf_total;
  M.b.block_offsets = v->tri_offsets;
  M.b.total = v->tri_total;
  M.b.n_blocks = S.b.n_blocks;
  return 0;
}

int volume_mesh(rmd_volume *v, void *xyzw, size_t vertex_capacity, int32_t *tri, size_t tri_capacity,
                size_t *n_vertices, size_t *n_triangles, bool host, const char *what)
{
  VolumeSurfaceParams S;
  VolumeMeshParams M;
  int rc = volume_mesh_params(v, S, M);
  if(rc) return rc;
  RMD_CUDA_TRY(launch_volume_surface_count(S, v->stream));
  RMD_CUDA_TRY(launch_volume_mesh_count(M, v->stream));
  unsigned long long nv = 0, nt = 0;
  RMD_CUDA_TRY(cudaMemcpyAsync(&nv, v->surf_total, sizeof(nv), cudaMemcpyDeviceToHost, v->stream));
  RMD_CUDA_TRY(cudaMemcpyAsync(&nt, v->tri_total, sizeof(nt), cudaMemcpyDeviceToHost, v->stream));
  RMD_CUDA_TRY(cudaStreamSynchronize(v->stream));
  *n_vertices = (size_t)nv;
  *n_triangles = (size_t)nt;
  if(nv >= (1ull << 31))
    return fail(RMD_ERR_UNSUPPORTED, (std::string(what) + ": 2^31 or more vertices do not fit int32 indices").c_str());
  const size_t mv = nv < vertex_capacity ? (size_t)nv : vertex_capacity;
  const size_t mt = nt < tri_capacity ? (size_t)nt : tri_capacity;
  if(!mv && !mt)
    return 0;
  float4 *vout = reinterpret_cast<float4*>(xyzw);
  int *tout = tri;
  if(host)
  {
    rc = volume_grow(&v->stage, &v->stage_cap, mv * sizeof(float4));
    if(!rc) rc = volume_grow(&v->tri_stage, &v->tri_stage_cap, 3 * mt);
    if(rc) return rc;
    vout = reinterpret_cast<float4*>(v->stage);
    tout = v->tri_stage;
  }
  S.out = vout;
  S.capacity = mv;
  if(mt)
  {
    // every vertex's key, whatever the vertex capacity: triangles may index vertices that are not returned
    rc = volume_grow(&v->keys, &v->keys_cap, (size_t)nv);
    if(rc) return rc;
    S.keys = v->keys;
  }
  RMD_CUDA_TRY(launch_volume_surface_write(S, v->stream));
  if(mt)
  {
    M.keys = v->keys;
    M.tri = tout;
    M.capacity = mt;
    RMD_CUDA_TRY(launch_volume_mesh_write(M, v->stream));
  }
  if(host)
  {
    if(mv)
      RMD_CUDA_TRY(cudaMemcpyAsync(xyzw, v->stage, mv * sizeof(float4), cudaMemcpyDeviceToHost, v->stream));
    if(mt)
      RMD_CUDA_TRY(cudaMemcpyAsync(tri, v->tri_stage, mt * 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, v->stream));
  }
  RMD_CUDA_TRY(cudaStreamSynchronize(v->stream));
  return 0;
}

// rmd_volume_integrate_depth[_intensity]: with_intensity also requires and fuses the image.
int volume_integrate_depth(const char *what, rmd_volume_t *v, int width, int height, float fx, float fy, float cx,
                           float cy, const float *T_curr_world, const float *dev_depth, size_t depth_pitch,
                           const int32_t *dev_conv, size_t conv_pitch, bool with_intensity,
                           const float *dev_intensity, size_t intensity_pitch)
{
  VOLUME_REQUIRE(v && T_curr_world && dev_depth && (!with_intensity || dev_intensity), "null argument");
  VOLUME_REQUIRE(width > 0 && height > 0, "bad image size");
  VOLUME_REQUIRE(depth_pitch_ok(depth_pitch, width), "bad depth pitch");
  VOLUME_REQUIRE(!dev_conv || (conv_pitch >= sizeof(int32_t) * (size_t)width && conv_pitch % sizeof(int32_t) == 0),
                 "bad state pitch");
  if(with_intensity)
  {
    VOLUME_REQUIRE(depth_pitch_ok(intensity_pitch, width), "bad intensity pitch");
    if(!v->col)
      return no_intensity(what);
  }
  DeviceGuard guard(v->device);
  VolumeIntegrateParams P;
  memset(&P, 0, sizeof(P));
  P.width = width; P.height = height;
  P.cam.fx = fx; P.cam.fy = fy; P.cam.cx = cx; P.cam.cy = cy;
  P.T_curr_world = pose_from(T_curr_world);
  P.depth = dev_depth; P.depth_stride = depth_pitch / sizeof(float); P.depth_comps = 1;
  P.conv = dev_conv; P.conv_stride = conv_pitch / sizeof(int32_t);
  if(with_intensity)
  {
    P.intensity = dev_intensity; P.intensity_stride = intensity_pitch / sizeof(float);
  }
  return volume_integrate(v, P);
}

// The rays of a pinhole camera at T_curr_world into the volume, writing their depth to dev_depth.
VolumeRaycastParams raycast_params(rmd_volume *v, int width, int height, float fx, float fy, float cx, float cy,
                                   const float *T_curr_world, float *dev_depth, size_t depth_pitch)
{
  VolumeRaycastParams P;
  memset(&P, 0, sizeof(P));
  P.g = v->g;
  P.width = width; P.height = height;
  P.cam.fx = fx; P.cam.fy = fy; P.cam.cx = cx; P.cam.cy = cy;
  P.T_world_curr = pose_inverse(pose_from(T_curr_world));
  P.depth = dev_depth; P.depth_stride = depth_pitch / sizeof(float);
  return P;
}

// rmd_volume_raycast[_intensity]: with_intensity also requires and writes the intensity image.
int volume_raycast(const char *what, rmd_volume_t *v, int width, int height, float fx, float fy, float cx, float cy,
                   const float *T_curr_world, float *dev_depth, size_t depth_pitch, bool with_intensity,
                   float *dev_intensity, size_t intensity_pitch)
{
  VOLUME_REQUIRE(v && T_curr_world && dev_depth && (!with_intensity || dev_intensity), "null argument");
  VOLUME_REQUIRE(width > 0 && height > 0, "bad image size");
  VOLUME_REQUIRE(depth_pitch_ok(depth_pitch, width), "bad depth pitch");
  if(with_intensity)
  {
    VOLUME_REQUIRE(depth_pitch_ok(intensity_pitch, width), "bad intensity pitch");
    if(!v->col)
      return no_intensity(what);
  }
  DeviceGuard guard(v->device);
  const VolumeRaycastParams P = raycast_params(v, width, height, fx, fy, cx, cy, T_curr_world, dev_depth, depth_pitch);
  VolumeRaycastColour C;
  memset(&C, 0, sizeof(C));
  if(with_intensity)
  {
    C.col = v->col;
    C.intensity = dev_intensity; C.intensity_stride = intensity_pitch / sizeof(float);
  }
  RMD_CUDA_TRY(launch_volume_raycast(P, C, v->stream));
  return 0;
}

// rmd_volume_raycast_normals: the plain rays and a float4 normal per pixel.
int volume_raycast_normals(const char *what, rmd_volume_t *v, int width, int height, float fx, float fy, float cx,
                           float cy, const float *T_curr_world, float *dev_depth, size_t depth_pitch,
                           float *dev_normals, size_t normals_pitch)
{
  VOLUME_REQUIRE(v && T_curr_world && dev_depth && dev_normals, "null argument");
  VOLUME_REQUIRE(width > 0 && height > 0, "bad image size");
  VOLUME_REQUIRE(depth_pitch_ok(depth_pitch, width), "bad depth pitch");
  VOLUME_REQUIRE(normals_pitch >= sizeof(float4) * (size_t)width && normals_pitch % sizeof(float4) == 0,
                 "bad normals pitch");
  VOLUME_REQUIRE(((uintptr_t)dev_normals % 16) == 0, "normals must be 16-byte aligned");
  DeviceGuard guard(v->device);
  const VolumeRaycastParams P = raycast_params(v, width, height, fx, fy, cx, cy, T_curr_world, dev_depth, depth_pitch);
  VolumeRaycastNormals N;
  N.normals = reinterpret_cast<float4*>(dev_normals);
  N.normals_stride = normals_pitch / sizeof(float4);
  RMD_CUDA_TRY(launch_volume_raycast_normals(P, N, v->stream));
  return 0;
}

// A record array (g.vox or col) to two host arrays of n_vox floats (.x to a, .y to b), through host chunks.
int volume_download_records(rmd_volume *v, const float2 *records, float *a, float *b, const char *what)
{
  const size_t chunk = v->n_vox < kVolumeChunk ? v->n_vox : kVolumeChunk;
  float2 *tmp = static_cast<float2*>(malloc(sizeof(float2) * chunk));
  if(!tmp) return fail((int)cudaErrorMemoryAllocation, (std::string(what) + ": host allocation failed").c_str());
  cudaError_t err = cudaSuccess;
  for(size_t c = 0; c < v->n_vox && err == cudaSuccess; c += chunk)
  {
    const size_t m = v->n_vox - c < chunk ? v->n_vox - c : chunk;
    err = cudaMemcpyAsync(tmp, records + c, sizeof(float2) * m, cudaMemcpyDeviceToHost, v->stream);
    if(err == cudaSuccess) err = cudaStreamSynchronize(v->stream);
    for(size_t q = 0; q < m && err == cudaSuccess; ++q)
    {
      a[c + q] = tmp[q].x;
      b[c + q] = tmp[q].y;
    }
  }
  free(tmp);
  RMD_CUDA_TRY(err);
  return 0;
}

// The inverse: two host arrays joined into the record array.
int volume_upload_records(rmd_volume *v, float2 *records, const float *a, const float *b, const char *what)
{
  const size_t chunk = v->n_vox < kVolumeChunk ? v->n_vox : kVolumeChunk;
  float2 *tmp = static_cast<float2*>(malloc(sizeof(float2) * chunk));
  if(!tmp) return fail((int)cudaErrorMemoryAllocation, (std::string(what) + ": host allocation failed").c_str());
  cudaError_t err = cudaSuccess;
  for(size_t c = 0; c < v->n_vox && err == cudaSuccess; c += chunk)
  {
    const size_t m = v->n_vox - c < chunk ? v->n_vox - c : chunk;
    for(size_t q = 0; q < m; ++q)
      tmp[q] = make_float2(a[c + q], b[c + q]);
    err = cudaMemcpyAsync(records + c, tmp, sizeof(float2) * m, cudaMemcpyHostToDevice, v->stream);
    if(err == cudaSuccess) err = cudaStreamSynchronize(v->stream);   // tmp is refilled next
  }
  free(tmp);
  RMD_CUDA_TRY(err);
  return 0;
}

// The box a shift by d keeps (VolumeSpillBox), from d clamped to [-n, n]: the same box, without overflow.
VolumeSpillBox spill_box(const rmd_volume *v, const int d[3])
{
  const int n[3] = {v->g.nx, v->g.ny, v->g.nz};
  VolumeSpillBox K;
  for(int a = 0; a < 3; ++a)
  {
    const int c = d[a] < -n[a] ? -n[a] : d[a] > n[a] ? n[a] : d[a];
    K.lo[a] = c > 0 ? c : 0;
    K.hi[a] = c < 0 ? n[a] + c : n[a];
  }
  return K;
}

// rmd_volume_spill_*: the points of the current grid that a shift by d would drop.
int volume_spill(const char *what, rmd_volume_t *v, const int d[3], void *host_out, size_t capacity, size_t *count,
                 SurfaceOutput kind)
{
  VOLUME_REQUIRE(v && d && count && (host_out || capacity == 0), "null argument");
  if(kind == SURFACE_INTENSITY && !v->col)
    return no_intensity(what);
  DeviceGuard guard(v->device);
  const VolumeSpillBox K = spill_box(v, d);
  return volume_surface(v, host_out, capacity, count, true, kind, &K);
}

// The first m entries of ids hold the keys 3 * voxel + axis of m vertices (as uint64); they become the vertices'
// ids (i + D0, j + D1, k + D2, axis), 4 per vertex, in place -- from the back, so that no key is overwritten before
// it is read.
void keys_to_ids(const rmd_volume *v, int64_t *ids, size_t m)
{
  const uint64_t nx = (uint64_t)v->g.nx, ny = (uint64_t)v->g.ny;
  for(size_t q = m; q-- > 0;)
  {
    const uint64_t key = (uint64_t)ids[q], vox = key / 3, row = vox / nx;
    ids[4 * q + 0] = (int64_t)(vox - row * nx) + v->D[0];
    ids[4 * q + 1] = (int64_t)(row % ny) + v->D[1];
    ids[4 * q + 2] = (int64_t)(row / ny) + v->D[2];
    ids[4 * q + 3] = (int64_t)(key - 3 * vox);
  }
}

// rmd_volume_spill_mesh: both count passes and scans on K, one host read of the two totals, then -- for what the
// capacities ask -- the vertices (with their keys when triangles or ids are wanted) and the triangles, staged in the
// volume's buffers and copied to the host; ids from the keys.  Synchronous.
int volume_spill_mesh(rmd_volume *v, const VolumeSpillBox &K, float *xyzw, size_t vertex_capacity, int32_t *tri,
                      size_t tri_capacity, int64_t *ids, size_t *n_vertices, size_t *n_triangles, const char *what)
{
  VolumeSurfaceParams S;
  VolumeMeshParams M;
  int rc = volume_mesh_params(v, S, M);
  if(rc) return rc;
  RMD_CUDA_TRY(launch_volume_spill_mesh_count(S, K, v->stream));
  RMD_CUDA_TRY(launch_volume_spill_tri_count(M, K, v->stream));
  unsigned long long nv = 0, nt = 0;
  RMD_CUDA_TRY(cudaMemcpyAsync(&nv, v->surf_total, sizeof(nv), cudaMemcpyDeviceToHost, v->stream));
  RMD_CUDA_TRY(cudaMemcpyAsync(&nt, v->tri_total, sizeof(nt), cudaMemcpyDeviceToHost, v->stream));
  RMD_CUDA_TRY(cudaStreamSynchronize(v->stream));
  *n_vertices = (size_t)nv;
  *n_triangles = (size_t)nt;
  if(nv >= (1ull << 31))
    return fail(RMD_ERR_UNSUPPORTED, (std::string(what) + ": 2^31 or more vertices do not fit int32 indices").c_str());
  const size_t mv = nv < vertex_capacity ? (size_t)nv : vertex_capacity;
  const size_t mt = nt < tri_capacity ? (size_t)nt : tri_capacity;
  if(!mv && !mt)
    return 0;
  rc = volume_grow(&v->stage, &v->stage_cap, mv * sizeof(float4));
  if(!rc) rc = volume_grow(&v->tri_stage, &v->tri_stage_cap, 3 * mt);
  if(rc) return rc;
  S.out = reinterpret_cast<float4*>(v->stage);
  S.capacity = mv;
  const bool keys = mt || (ids && mv);
  if(keys)
  {
    // every vertex's key, whatever the vertex capacity: triangles may index vertices that are not returned
    rc = volume_grow(&v->keys, &v->keys_cap, (size_t)nv);
    if(rc) return rc;
    S.keys = v->keys;
  }
  RMD_CUDA_TRY(launch_volume_spill_mesh_write(S, K, v->stream));
  if(mt)
  {
    M.keys = v->keys;
    M.tri = v->tri_stage;
    M.capacity = mt;
    RMD_CUDA_TRY(launch_volume_spill_tri_write(M, K, v->stream));
  }
  if(mv)
    RMD_CUDA_TRY(cudaMemcpyAsync(xyzw, v->stage, mv * sizeof(float4), cudaMemcpyDeviceToHost, v->stream));
  if(mt)
    RMD_CUDA_TRY(cudaMemcpyAsync(tri, v->tri_stage, mt * 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, v->stream));
  if(ids && mv)
    RMD_CUDA_TRY(cudaMemcpyAsync(ids, v->keys, mv * sizeof(uint64_t), cudaMemcpyDeviceToHost, v->stream));
  RMD_CUDA_TRY(cudaStreamSynchronize(v->stream));
  if(ids)
    keys_to_ids(v, ids, mv);
  return 0;
}

int no_store(const char *what)
{
  return fail(RMD_ERR_NOT_INITIALISED, (std::string(what) + ": the volume has no brick store").c_str());
}

// The store's pool grown to hold `need` bricks, by doubling: the new arrays of both channels are allocated before the
// used slots are copied and the old arrays freed, so that a failure leaves the store as it was.
int store_grow(rmd_volume *v, size_t need, const char *what)
{
  VolumeStore *S = v->store;
  const size_t cap = store_pool_capacity(S->cap, need);
  if(cap == S->cap)
    return 0;
  const size_t brick = sizeof(float2) * VOLUME_STORE_VOXELS, used = brick * S->index.slot.size();
  float2 *p = NULL, *pc = NULL;
  cudaError_t err = cudaMalloc(&p, brick * cap);
  if(err == cudaSuccess && v->col) err = cudaMalloc(&pc, brick * cap);
  if(err == cudaSuccess && used) err = cudaMemcpyAsync(p, S->pool, used, cudaMemcpyDeviceToDevice, v->stream);
  if(err == cudaSuccess && used && v->col)
    err = cudaMemcpyAsync(pc, S->pool_col, used, cudaMemcpyDeviceToDevice, v->stream);
  if(err == cudaSuccess) err = cudaStreamSynchronize(v->stream);
  if(err != cudaSuccess)
  {
    cudaFree(p); cudaFree(pc);
    return fail_cuda(err, what);
  }
  cudaFree(S->pool); cudaFree(S->pool_col);
  S->pool = p; S->pool_col = pc; S->cap = cap;
  return 0;
}

// The bricks a store kernel visits, to the device (scratch grown by the caller).  Pageable source: the copy is staged
// before the call returns.
int store_upload_bricks(rmd_volume *v, const std::vector<VolumeStoreBrick> &list)
{
  if(!list.empty())
    RMD_CUDA_TRY(cudaMemcpyAsync(v->store->bricks, list.data(), sizeof(VolumeStoreBrick) * list.size(),
                                 cudaMemcpyHostToDevice, v->stream));
  return 0;
}

VolumeStoreBrick store_brick(const BrickCoord &c, int slot, int fresh)
{
  VolumeStoreBrick B;
  B.b[0] = c.b[0]; B.b[1] = c.b[1]; B.b[2] = c.b[2];
  B.slot = slot; B.fresh = fresh;
  return B;
}

// The store's part of rmd_volume_shift before the gather (DESIGN.md 4.8): the candidates -- bricks with a voxel that
// leaves -- split into stored and fresh; the fresh ones flagged on the device and the flags read back (the shift's one
// host synchronisation); the pool and scratch grown; then, the first write, the index updated and the evict kernel
// launched on the pre-shift records.  The stored bricks with a voxel that enters follow the evicted ones in the
// scratch, from *restore_first on, *n_restore of them, for store_restore after the gather.
int store_evict(rmd_volume *v, const int d[3], const long long Dnew[3], size_t *restore_first, size_t *n_restore)
{
  const char *what = "rmd_volume_shift";
  VolumeStore *S = v->store;
  const int n[3] = {v->g.nx, v->g.ny, v->g.nz};
  const VolumeSpillBox K = spill_box(v, d);
  VolumeSpillBox Kin;   // post-shift indices whose source lay in the grid
  for(int a = 0; a < 3; ++a)
  {
    const int c = d[a] < -n[a] ? -n[a] : d[a] > n[a] ? n[a] : d[a];
    Kin.lo[a] = c < 0 ? -c : 0;
    Kin.hi[a] = c > 0 ? n[a] - c : n[a];
  }
  const int64_t Dold[3] = {v->D[0], v->D[1], v->D[2]}, Dn[3] = {Dnew[0], Dnew[1], Dnew[2]};
  std::vector<BrickCoord> known, fresh;
  S->index.split(store_candidates(Dold, n, K.lo, K.hi), known, fresh);
  const std::vector<BrickCoord> entering = store_candidates(Dn, n, Kin.lo, Kin.hi);

  VolumeStoreParams P;
  memset(&P, 0, sizeof(P));
  P.g = v->g;
  P.col = v->col;
  for(int a = 0; a < 3; ++a)
  {
    P.W[a] = Dold[a];
    P.lo[a] = K.lo[a]; P.hi[a] = K.hi[a];
  }
  int rc = volume_grow(&S->bricks, &S->bricks_cap, known.size() + fresh.size() + entering.size());
  if(!rc) rc = volume_grow(&S->flags, &S->flags_cap, fresh.size());
  if(rc) return rc;
  P.bricks = S->bricks;
  P.flags = S->flags;
  std::vector<int> flags(fresh.size(), 0);
  std::vector<VolumeStoreBrick> list;
  if(!fresh.empty())
  {
    for(size_t q = 0; q < fresh.size(); ++q)
      list.push_back(store_brick(fresh[q], (int)q, 1));
    rc = store_upload_bricks(v, list);
    if(rc) return rc;
    RMD_CUDA_TRY(launch_volume_store_flag(P, (unsigned int)fresh.size(), v->stream));
    RMD_CUDA_TRY(cudaMemcpyAsync(flags.data(), S->flags, sizeof(int) * fresh.size(), cudaMemcpyDeviceToHost,
                                 v->stream));
    RMD_CUDA_TRY(cudaStreamSynchronize(v->stream));
  }
  size_t added = 0;
  for(int f : flags)
    added += f ? 1 : 0;
  if(S->index.slot.size() + added > (size_t)INT32_MAX)
    return fail(RMD_ERR_UNSUPPORTED, "rmd_volume_shift: 2^31 or more stored bricks");
  rc = store_grow(v, S->index.slot.size() + added, what);
  if(rc) return rc;

  // nothing has been written so far; from here on the shift happens
  const std::vector<BrickCoord> added_bricks = S->index.add(fresh, flags);
  list.clear();
  for(const BrickCoord &c : known)
    list.push_back(store_brick(c, S->index.slot.at(c), 0));
  for(const BrickCoord &c : added_bricks)
    list.push_back(store_brick(c, S->index.slot.at(c), 1));
  const size_t n_evict = list.size();
  for(const BrickCoord &c : entering)
  {
    auto it = S->index.slot.find(c);
    if(it != S->index.slot.end())
      list.push_back(store_brick(c, it->second, 0));
  }
  *restore_first = n_evict;
  *n_restore = list.size() - n_evict;
  rc = store_upload_bricks(v, list);
  if(rc) return rc;
  P.pool = S->pool; P.pool_col = S->pool_col;
  RMD_CUDA_TRY(launch_volume_store_evict(P, (unsigned int)n_evict, v->stream));
  return 0;
}

// The store's part of rmd_volume_shift after the gather: the stored bricks' entering voxels into the new records.
int store_restore(rmd_volume *v, const int d[3], size_t first, size_t count)
{
  if(!count)
    return 0;
  VolumeStore *S = v->store;
  const int n[3] = {v->g.nx, v->g.ny, v->g.nz};
  VolumeStoreParams P;
  memset(&P, 0, sizeof(P));
  P.g = v->g;
  P.col = v->col;
  P.pool = S->pool; P.pool_col = S->pool_col;
  P.bricks = S->bricks + first;
  for(int a = 0; a < 3; ++a)
  {
    const int c = d[a] < -n[a] ? -n[a] : d[a] > n[a] ? n[a] : d[a];
    P.W[a] = v->D[a];
    P.lo[a] = c < 0 ? -c : 0;
    P.hi[a] = c > 0 ? n[a] - c : n[a];
  }
  RMD_CUDA_TRY(launch_volume_store_restore(P, (unsigned int)count, v->stream));
  return 0;
}

// origin + (float)D * s, one rounding per operation as the kernels' voxel_coord (volatile: no contraction)
float shifted_origin(float origin, long long D, float s)
{
  volatile float step = (float)D * s;
  return origin + step;
}

} // namespace

extern "C"
{

int rmd_volume_create(int nx, int ny, int nz, float voxel_size, const float origin[3], float truncation,
                      float max_weight, int device, rmd_volume_t **out)
{
  RMD_REQUIRE(out, "rmd_volume_create: out is null");
  *out = NULL;
  RMD_REQUIRE(origin, "rmd_volume_create: origin is null");
  RMD_REQUIRE(nx > 0 && ny > 0 && nz > 0, "rmd_volume_create: grid dimensions must be positive");
  const uint64_t plane = (uint64_t)nx * (uint64_t)ny;   // each factor < 2^31: no overflow in 64 bits
  RMD_REQUIRE(plane <= kVolumeMaxVoxels && plane * (uint64_t)nz <= kVolumeMaxVoxels,
              "rmd_volume_create: at most 2^31 voxels");
  RMD_REQUIRE(voxel_size > 0.0f && isfinite(voxel_size), "rmd_volume_create: voxel_size must be > 0");
  RMD_REQUIRE(truncation > 0.0f && isfinite(truncation), "rmd_volume_create: truncation must be > 0");
  RMD_REQUIRE(max_weight >= 1.0f, "rmd_volume_create: max_weight must be >= 1");
  RMD_REQUIRE(isfinite(origin[0]) && isfinite(origin[1]) && isfinite(origin[2]), "rmd_volume_create: bad origin");
  if(device < 0) RMD_CUDA_TRY(cudaGetDevice(&device));
  DeviceGuard guard(device);
  rmd_volume *v = new(std::nothrow) rmd_volume();
  if(!v) return fail((int)cudaErrorMemoryAllocation, "rmd_volume_create: host allocation failed");
  memset(v, 0, sizeof(*v));
  v->device = device;
  v->g.nx = nx; v->g.ny = ny; v->g.nz = nz;
  v->g.voxel = voxel_size;
  v->g.ox = origin[0]; v->g.oy = origin[1]; v->g.oz = origin[2];
  v->o0[0] = origin[0]; v->o0[1] = origin[1]; v->o0[2] = origin[2];
  v->n_vox = (size_t)(plane * (uint64_t)nz);
  v->trunc = truncation; v->max_weight = max_weight;
  cudaError_t err = cudaStreamCreateWithFlags(&v->own_stream, cudaStreamNonBlocking);
  if(err == cudaSuccess) err = cudaEventCreateWithFlags(&v->seeds_ev, cudaEventDisableTiming);
  if(err == cudaSuccess) err = cudaMalloc(&v->g.vox, sizeof(float2) * v->n_vox);
  if(err == cudaSuccess) err = cudaMemsetAsync(v->g.vox, 0, sizeof(float2) * v->n_vox, v->own_stream);
  if(err == cudaSuccess) err = cudaStreamSynchronize(v->own_stream);
  if(err != cudaSuccess)
  {
    rmd_volume_destroy(v);
    return fail_cuda(err, "rmd_volume_create");
  }
  v->stream = v->own_stream;
  *out = v;
  return 0;
}

int rmd_volume_destroy(rmd_volume_t *v)
{
  if(!v) return 0;
  DeviceGuard guard(v->device);
  cudaDeviceSynchronize();
  if(v->own_stream) cudaStreamDestroy(v->own_stream);
  if(v->seeds_ev) cudaEventDestroy(v->seeds_ev);
  cudaFree(v->g.vox);
  cudaFree(v->surf_offsets); cudaFree(v->surf_total); cudaFree(v->stage);
  cudaFree(v->tri_offsets); cudaFree(v->tri_total); cudaFree(v->keys); cudaFree(v->tri_stage);
  cudaFree(v->col);
  cudaFree(v->vox_alt); cudaFree(v->col_alt);
  if(v->store)
  {
    cudaFree(v->store->pool); cudaFree(v->store->pool_col);
    cudaFree(v->store->bricks); cudaFree(v->store->flags);
    delete v->store;
  }
  cudaGetLastError();
  delete v;
  return 0;
}

int rmd_volume_set_stream(rmd_volume_t *v, void *cuda_stream)
{
  RMD_REQUIRE(v, "rmd_volume_set_stream: null handle");
  DeviceGuard guard(v->device);
  RMD_CUDA_TRY(cudaStreamSynchronize(v->stream));
  v->stream = cuda_stream ? (cudaStream_t)cuda_stream : v->own_stream;
  return 0;
}

int rmd_volume_reset(rmd_volume_t *v)
{
  RMD_REQUIRE(v, "rmd_volume_reset: null handle");
  DeviceGuard guard(v->device);
  RMD_CUDA_TRY(cudaMemsetAsync(v->g.vox, 0, sizeof(float2) * v->n_vox, v->stream));
  if(v->col)
    RMD_CUDA_TRY(cudaMemsetAsync(v->col, 0, sizeof(float2) * v->n_vox, v->stream));
  if(v->store)
    v->store->index.slot.clear();
  return 0;
}

int rmd_volume_sync(rmd_volume_t *v)
{
  RMD_REQUIRE(v, "rmd_volume_sync: null handle");
  DeviceGuard guard(v->device);
  RMD_CUDA_TRY(cudaStreamSynchronize(v->stream));
  return 0;
}

int rmd_volume_size(rmd_volume_t *v, int *nx, int *ny, int *nz, float *voxel_size, float origin[3])
{
  RMD_REQUIRE(v, "rmd_volume_size: null handle");
  if(nx) *nx = v->g.nx;
  if(ny) *ny = v->g.ny;
  if(nz) *nz = v->g.nz;
  if(voxel_size) *voxel_size = v->g.voxel;
  if(origin) { origin[0] = v->g.ox; origin[1] = v->g.oy; origin[2] = v->g.oz; }
  return 0;
}

int rmd_volume_shift(rmd_volume_t *v, const int d[3])
{
  RMD_REQUIRE(v && d, "rmd_volume_shift: null argument");
  if(!d[0] && !d[1] && !d[2])
    return 0;
  const int n[3] = {v->g.nx, v->g.ny, v->g.nz};
  long long D[3];
  float o[3];
  bool gather = true;
  for(int a = 0; a < 3; ++a)
  {
    RMD_REQUIRE(!__builtin_add_overflow(v->D[a], (long long)d[a], &D[a]), "rmd_volume_shift: the total offset overflows");
    o[a] = shifted_origin(v->o0[a], D[a], v->g.voxel);
    RMD_REQUIRE(isfinite(o[a]), "rmd_volume_shift: the origin would not be finite");
    gather = gather && (d[a] < 0 ? -(long long)d[a] : (long long)d[a]) < n[a];
    long long end;
    RMD_REQUIRE(!v->store || !__builtin_add_overflow(D[a], (long long)n[a], &end),
                "rmd_volume_shift: the total offset plus the grid size overflows");
  }
  DeviceGuard guard(v->device);
  if(gather)
  {
    if(!v->vox_alt)
      RMD_CUDA_TRY(cudaMalloc(&v->vox_alt, sizeof(float2) * v->n_vox));
    if(v->col && !v->col_alt)
      RMD_CUDA_TRY(cudaMalloc(&v->col_alt, sizeof(float2) * v->n_vox));
  }
  size_t restore_first = 0, n_restore = 0;
  if(v->store)
  {
    const int rc = store_evict(v, d, D, &restore_first, &n_restore);
    if(rc) return rc;
  }
  if(!gather)   // nothing stays in the grid
  {
    RMD_CUDA_TRY(cudaMemsetAsync(v->g.vox, 0, sizeof(float2) * v->n_vox, v->stream));
    if(v->col)
      RMD_CUDA_TRY(cudaMemsetAsync(v->col, 0, sizeof(float2) * v->n_vox, v->stream));
  }
  else
  {
    VolumeShiftParams P;
    memset(&P, 0, sizeof(P));
    P.g = v->g;
    P.out = v->vox_alt;
    if(v->col)
    {
      P.col = v->col; P.col_out = v->col_alt;
    }
    P.dx = d[0]; P.dy = d[1]; P.dz = d[2];
    RMD_CUDA_TRY(launch_volume_shift(P, v->stream));
    // Later work on the stream reads the new arrays.  The next shift writes the old ones, ordered after everything
    // already on the stream -- including the wait of rmd_volume_prior_seeds for its rays.
    float2 *t = v->g.vox; v->g.vox = v->vox_alt; v->vox_alt = t;
    if(v->col)
    {
      t = v->col; v->col = v->col_alt; v->col_alt = t;
    }
  }
  for(int a = 0; a < 3; ++a)
    v->D[a] = D[a];
  v->g.ox = o[0]; v->g.oy = o[1]; v->g.oz = o[2];
  if(v->store)
    return store_restore(v, d, restore_first, n_restore);
  return 0;
}

int rmd_volume_spill_points(rmd_volume_t *v, const int d[3], float *host_xyzw, size_t capacity, size_t *count)
{
  return volume_spill("rmd_volume_spill_points", v, d, host_xyzw, capacity, count, SURFACE_POINTS);
}

int rmd_volume_spill_intensity(rmd_volume_t *v, const int d[3], float *host_intensity, size_t capacity, size_t *count)
{
  return volume_spill("rmd_volume_spill_intensity", v, d, host_intensity, capacity, count, SURFACE_INTENSITY);
}

int rmd_volume_spill_normals(rmd_volume_t *v, const int d[3], float *host_nxyz0, size_t capacity, size_t *count)
{
  return volume_spill("rmd_volume_spill_normals", v, d, host_nxyz0, capacity, count, SURFACE_NORMALS);
}

int rmd_volume_spill_mesh(rmd_volume_t *v, const int d[3], float *host_xyzw, size_t vertex_capacity, int32_t *host_tri,
                          size_t tri_capacity, int64_t *host_ids, size_t *n_vertices, size_t *n_triangles)
{
  const char *what = "rmd_volume_spill_mesh";
  VOLUME_REQUIRE(v && d && n_vertices && n_triangles && (host_xyzw || vertex_capacity == 0) &&
                 (host_tri || tri_capacity == 0), "null argument");
  DeviceGuard guard(v->device);
  return volume_spill_mesh(v, spill_box(v, d), host_xyzw, vertex_capacity, host_tri, tri_capacity, host_ids,
                           n_vertices, n_triangles, what);
}

int rmd_volume_spill_mesh_intensity(rmd_volume_t *v, const int d[3], float *host_intensity, size_t capacity,
                                    size_t *count)
{
  const char *what = "rmd_volume_spill_mesh_intensity";
  VOLUME_REQUIRE(v && d && count && (host_intensity || capacity == 0), "null argument");
  if(!v->col)
    return no_intensity(what);
  DeviceGuard guard(v->device);
  const VolumeSpillBox K = spill_box(v, d);
  return volume_surface(v, host_intensity, capacity, count, true, SURFACE_INTENSITY, &K, true);
}

int rmd_volume_spill_mesh_normals(rmd_volume_t *v, const int d[3], float *host_nxyz0, size_t capacity, size_t *count)
{
  const char *what = "rmd_volume_spill_mesh_normals";
  VOLUME_REQUIRE(v && d && count && (host_nxyz0 || capacity == 0), "null argument");
  DeviceGuard guard(v->device);
  const VolumeSpillBox K = spill_box(v, d);
  return volume_surface(v, host_nxyz0, capacity, count, true, SURFACE_NORMALS, &K, true);
}

int rmd_volume_surface_ids(rmd_volume_t *v, int64_t *host_ids, size_t capacity, size_t *count)
{
  RMD_REQUIRE(v && count && (host_ids || capacity == 0), "rmd_volume_surface_ids: null argument");
  DeviceGuard guard(v->device);
  VolumeSurfaceParams P;
  int rc = volume_surface_params(v, P);
  if(rc) return rc;
  RMD_CUDA_TRY(launch_volume_surface_count(P, v->stream));
  unsigned long long total = 0;
  RMD_CUDA_TRY(cudaMemcpyAsync(&total, v->surf_total, sizeof(total), cudaMemcpyDeviceToHost, v->stream));
  RMD_CUDA_TRY(cudaStreamSynchronize(v->stream));
  *count = (size_t)total;
  const size_t m = *count < capacity ? *count : capacity;
  if(!m)
    return 0;
  // the mesh path's key pass with no point output: every point's key
  rc = volume_grow(&v->keys, &v->keys_cap, (size_t)total);
  if(rc) return rc;
  P.keys = v->keys;
  RMD_CUDA_TRY(launch_volume_surface_write(P, v->stream));
  RMD_CUDA_TRY(cudaMemcpyAsync(host_ids, v->keys, m * sizeof(uint64_t), cudaMemcpyDeviceToHost, v->stream));
  RMD_CUDA_TRY(cudaStreamSynchronize(v->stream));
  keys_to_ids(v, host_ids, m);
  return 0;
}

int rmd_volume_offset(rmd_volume_t *v, int64_t D[3])
{
  RMD_REQUIRE(v && D, "rmd_volume_offset: null argument");
  for(int a = 0; a < 3; ++a)
    D[a] = v->D[a];
  return 0;
}

int rmd_volume_enable_intensity(rmd_volume_t *v)
{
  RMD_REQUIRE(v, "rmd_volume_enable_intensity: null handle");
  if(v->col)
    return 0;
  DeviceGuard guard(v->device);
  cudaError_t err = cudaMalloc(&v->col, sizeof(float2) * v->n_vox);
  if(err != cudaSuccess)
  {
    v->col = NULL;
    return fail_cuda(err, "rmd_volume_enable_intensity");
  }
  err = cudaMemsetAsync(v->col, 0, sizeof(float2) * v->n_vox, v->stream);
  VolumeStore *S = v->store;
  const size_t pool_bytes = S ? sizeof(float2) * VOLUME_STORE_VOXELS * S->cap : 0;
  if(err == cudaSuccess && pool_bytes)   // the bricks already stored get zeroed colour records
  {
    err = cudaMalloc(&S->pool_col, pool_bytes);
    if(err == cudaSuccess) err = cudaMemsetAsync(S->pool_col, 0, pool_bytes, v->stream);
    if(err != cudaSuccess)
    {
      cudaFree(S->pool_col);
      S->pool_col = NULL;
    }
  }
  if(err != cudaSuccess)
  {
    cudaFree(v->col);
    v->col = NULL;
    return fail_cuda(err, "rmd_volume_enable_intensity");
  }
  return 0;
}

int rmd_volume_integrate_depth(rmd_volume_t *v, int width, int height, float fx, float fy, float cx, float cy,
                               const float *T_curr_world, const float *dev_depth, size_t depth_pitch,
                               const int32_t *dev_conv, size_t conv_pitch)
{
  return volume_integrate_depth("rmd_volume_integrate_depth", v, width, height, fx, fy, cx, cy, T_curr_world,
                                dev_depth, depth_pitch, dev_conv, conv_pitch, false, NULL, 0);
}

int rmd_volume_integrate_depth_intensity(rmd_volume_t *v, int width, int height, float fx, float fy, float cx,
                                         float cy, const float *T_curr_world, const float *dev_depth,
                                         size_t depth_pitch, const int32_t *dev_conv, size_t conv_pitch,
                                         const float *dev_intensity, size_t intensity_pitch)
{
  return volume_integrate_depth("rmd_volume_integrate_depth_intensity", v, width, height, fx, fy, cx, cy,
                                T_curr_world, dev_depth, depth_pitch, dev_conv, conv_pitch, true, dev_intensity,
                                intensity_pitch);
}

int rmd_volume_surface_points(rmd_volume_t *v, float *host_xyzw, size_t capacity, size_t *count)
{
  RMD_REQUIRE(v && count && (host_xyzw || capacity == 0), "rmd_volume_surface_points: null argument");
  DeviceGuard guard(v->device);
  return volume_surface(v, host_xyzw, capacity, count, true, SURFACE_POINTS);
}

int rmd_volume_surface_points_device(rmd_volume_t *v, float *dev_xyzw, size_t capacity, size_t *count)
{
  RMD_REQUIRE(v && count && (dev_xyzw || capacity == 0), "rmd_volume_surface_points_device: null argument");
  RMD_REQUIRE(((uintptr_t)dev_xyzw % 16) == 0, "rmd_volume_surface_points_device: output must be 16-byte aligned");
  DeviceGuard guard(v->device);
  return volume_surface(v, dev_xyzw, capacity, count, false, SURFACE_POINTS);
}

int rmd_volume_surface_intensity(rmd_volume_t *v, float *host_intensity, size_t capacity, size_t *count)
{
  RMD_REQUIRE(v && count && (host_intensity || capacity == 0), "rmd_volume_surface_intensity: null argument");
  if(!v->col)
    return no_intensity("rmd_volume_surface_intensity");
  DeviceGuard guard(v->device);
  return volume_surface(v, host_intensity, capacity, count, true, SURFACE_INTENSITY);
}

int rmd_volume_surface_intensity_device(rmd_volume_t *v, float *dev_intensity, size_t capacity, size_t *count)
{
  RMD_REQUIRE(v && count && (dev_intensity || capacity == 0), "rmd_volume_surface_intensity_device: null argument");
  RMD_REQUIRE(((uintptr_t)dev_intensity % 4) == 0, "rmd_volume_surface_intensity_device: output must be 4-byte aligned");
  if(!v->col)
    return no_intensity("rmd_volume_surface_intensity_device");
  DeviceGuard guard(v->device);
  return volume_surface(v, dev_intensity, capacity, count, false, SURFACE_INTENSITY);
}

int rmd_volume_surface_normals(rmd_volume_t *v, float *host_nxyz0, size_t capacity, size_t *count)
{
  RMD_REQUIRE(v && count && (host_nxyz0 || capacity == 0), "rmd_volume_surface_normals: null argument");
  DeviceGuard guard(v->device);
  return volume_surface(v, host_nxyz0, capacity, count, true, SURFACE_NORMALS);
}

int rmd_volume_surface_normals_device(rmd_volume_t *v, float *dev_nxyz0, size_t capacity, size_t *count)
{
  RMD_REQUIRE(v && count && (dev_nxyz0 || capacity == 0), "rmd_volume_surface_normals_device: null argument");
  RMD_REQUIRE(((uintptr_t)dev_nxyz0 % 16) == 0, "rmd_volume_surface_normals_device: output must be 16-byte aligned");
  DeviceGuard guard(v->device);
  return volume_surface(v, dev_nxyz0, capacity, count, false, SURFACE_NORMALS);
}

int rmd_volume_mesh(rmd_volume_t *v, float *host_xyzw, size_t vertex_capacity, int32_t *host_tri,
                    size_t tri_capacity, size_t *n_vertices, size_t *n_triangles)
{
  RMD_REQUIRE(v && n_vertices && n_triangles && (host_xyzw || vertex_capacity == 0) && (host_tri || tri_capacity == 0),
              "rmd_volume_mesh: null argument");
  DeviceGuard guard(v->device);
  return volume_mesh(v, host_xyzw, vertex_capacity, host_tri, tri_capacity, n_vertices, n_triangles, true,
                     "rmd_volume_mesh");
}

int rmd_volume_mesh_device(rmd_volume_t *v, float *dev_xyzw, size_t vertex_capacity, int32_t *dev_tri,
                           size_t tri_capacity, size_t *n_vertices, size_t *n_triangles)
{
  RMD_REQUIRE(v && n_vertices && n_triangles && (dev_xyzw || vertex_capacity == 0) && (dev_tri || tri_capacity == 0),
              "rmd_volume_mesh_device: null argument");
  RMD_REQUIRE(((uintptr_t)dev_xyzw % 16) == 0, "rmd_volume_mesh_device: vertices must be 16-byte aligned");
  RMD_REQUIRE(((uintptr_t)dev_tri % 4) == 0, "rmd_volume_mesh_device: triangles must be 4-byte aligned");
  DeviceGuard guard(v->device);
  return volume_mesh(v, dev_xyzw, vertex_capacity, dev_tri, tri_capacity, n_vertices, n_triangles, false,
                     "rmd_volume_mesh_device");
}

int rmd_volume_raycast(rmd_volume_t *v, int width, int height, float fx, float fy, float cx, float cy,
                       const float *T_curr_world, float *dev_depth, size_t depth_pitch)
{
  return volume_raycast("rmd_volume_raycast", v, width, height, fx, fy, cx, cy, T_curr_world, dev_depth, depth_pitch,
                        false, NULL, 0);
}

int rmd_volume_raycast_intensity(rmd_volume_t *v, int width, int height, float fx, float fy, float cx, float cy,
                                 const float *T_curr_world, float *dev_depth, size_t depth_pitch,
                                 float *dev_intensity, size_t intensity_pitch)
{
  return volume_raycast("rmd_volume_raycast_intensity", v, width, height, fx, fy, cx, cy, T_curr_world, dev_depth,
                        depth_pitch, true, dev_intensity, intensity_pitch);
}

int rmd_volume_raycast_normals(rmd_volume_t *v, int width, int height, float fx, float fy, float cx, float cy,
                               const float *T_curr_world, float *dev_depth, size_t depth_pitch,
                               float *dev_normals, size_t normals_pitch)
{
  return volume_raycast_normals("rmd_volume_raycast_normals", v, width, height, fx, fy, cx, cy, T_curr_world,
                                dev_depth, depth_pitch, dev_normals, normals_pitch);
}

int rmd_volume_download(rmd_volume_t *v, float *host_tsdf, float *host_weight)
{
  RMD_REQUIRE(v && host_tsdf && host_weight, "rmd_volume_download: null argument");
  DeviceGuard guard(v->device);
  return volume_download_records(v, v->g.vox, host_tsdf, host_weight, "rmd_volume_download");
}

int rmd_volume_upload(rmd_volume_t *v, const float *host_tsdf, const float *host_weight)
{
  RMD_REQUIRE(v && host_tsdf && host_weight, "rmd_volume_upload: null argument");
  DeviceGuard guard(v->device);
  return volume_upload_records(v, v->g.vox, host_tsdf, host_weight, "rmd_volume_upload");
}

int rmd_volume_download_intensity(rmd_volume_t *v, float *host_intensity, float *host_weight)
{
  RMD_REQUIRE(v && host_intensity && host_weight, "rmd_volume_download_intensity: null argument");
  if(!v->col)
    return no_intensity("rmd_volume_download_intensity");
  DeviceGuard guard(v->device);
  return volume_download_records(v, v->col, host_intensity, host_weight, "rmd_volume_download_intensity");
}

int rmd_volume_upload_intensity(rmd_volume_t *v, const float *host_intensity, const float *host_weight)
{
  RMD_REQUIRE(v && host_intensity && host_weight, "rmd_volume_upload_intensity: null argument");
  if(!v->col)
    return no_intensity("rmd_volume_upload_intensity");
  DeviceGuard guard(v->device);
  return volume_upload_records(v, v->col, host_intensity, host_weight, "rmd_volume_upload_intensity");
}

int rmd_volume_enable_store(rmd_volume_t *v)
{
  const char *what = "rmd_volume_enable_store";
  VOLUME_REQUIRE(v, "null handle");
  if(v->store)
    return 0;
  const int n[3] = {v->g.nx, v->g.ny, v->g.nz};
  for(int a = 0; a < 3; ++a)
  {
    long long end;
    VOLUME_REQUIRE(!__builtin_add_overflow(v->D[a], (long long)n[a], &end),
                   "the total offset plus the grid size overflows");
  }
  v->store = new(std::nothrow) VolumeStore();
  if(!v->store)
    return fail((int)cudaErrorMemoryAllocation, "rmd_volume_enable_store: host allocation failed");
  return 0;
}

int rmd_volume_store_info(rmd_volume_t *v, size_t *bricks, size_t *bytes)
{
  const char *what = "rmd_volume_store_info";
  VOLUME_REQUIRE(v, "null handle");
  if(!v->store)
    return no_store(what);
  if(bricks) *bricks = v->store->index.slot.size();
  if(bytes) *bytes = sizeof(float2) * VOLUME_STORE_VOXELS * v->store->cap * (v->store->pool_col ? 2 : 1);
  return 0;
}

int rmd_volume_download_store(rmd_volume_t *v, int64_t *host_coords, float *host_tsdf, float *host_weight,
                              float *host_intensity, float *host_intensity_weight, size_t capacity, size_t *count)
{
  const char *what = "rmd_volume_download_store";
  VOLUME_REQUIRE(v && count && (host_coords || capacity == 0), "null argument");
  if((host_intensity || host_intensity_weight) && !v->col)
    return no_intensity(what);
  if(!v->store)
    return no_store(what);
  DeviceGuard guard(v->device);
  VolumeStore *S = v->store;
  *count = S->index.slot.size();
  const size_t m = *count < capacity ? *count : capacity;
  if(!m)
    return 0;
  const bool records = host_tsdf || host_weight, colour = host_intensity || host_intensity_weight;
  const size_t used = VOLUME_STORE_VOXELS * S->index.slot.size();
  std::vector<float2> rec(records ? used : 0), col(colour ? used : 0);
  // the store's copies of voxels that are in the window are stale: wait for the window's last writes, then read
  if(records)
    RMD_CUDA_TRY(cudaMemcpyAsync(rec.data(), S->pool, sizeof(float2) * used, cudaMemcpyDeviceToHost, v->stream));
  if(colour)
    RMD_CUDA_TRY(cudaMemcpyAsync(col.data(), S->pool_col, sizeof(float2) * used, cudaMemcpyDeviceToHost, v->stream));
  RMD_CUDA_TRY(cudaStreamSynchronize(v->stream));
  const int n[3] = {v->g.nx, v->g.ny, v->g.nz};
  size_t q = 0;
  for(auto it = S->index.slot.begin(); it != S->index.slot.end() && q < m; ++it, ++q)
  {
    const BrickCoord &c = it->first;
    for(int a = 0; a < 3; ++a)
      host_coords[3 * q + a] = c.b[a];
    for(int l = 0; l < VOLUME_STORE_VOXELS; ++l)
    {
      const int loc[3] = {l & 7, (l >> 3) & 7, l >> 6};
      bool in_window = true;
      for(int a = 0; a < 3; ++a)
      {
        const int64_t u = c.b[a] * STORE_BRICK + loc[a];
        in_window = in_window && u >= v->D[a] && (uint64_t)u - (uint64_t)v->D[a] < (uint64_t)n[a];
      }
      const size_t src = (size_t)it->second * VOLUME_STORE_VOXELS + l, dst = q * VOLUME_STORE_VOXELS + l;
      const float2 zero = make_float2(0.0f, 0.0f);
      const float2 r = in_window || !records ? zero : rec[src], k = in_window || !colour ? zero : col[src];
      if(host_tsdf) host_tsdf[dst] = r.x;
      if(host_weight) host_weight[dst] = r.y;
      if(host_intensity) host_intensity[dst] = k.x;
      if(host_intensity_weight) host_intensity_weight[dst] = k.y;
    }
  }
  return 0;
}

int rmd_volume_upload_store(rmd_volume_t *v, const int64_t *host_coords, const float *host_tsdf,
                            const float *host_weight, const float *host_intensity,
                            const float *host_intensity_weight, size_t count)
{
  const char *what = "rmd_volume_upload_store";
  VOLUME_REQUIRE(v && (count == 0 || (host_coords && host_tsdf && host_weight)), "null argument");
  VOLUME_REQUIRE(!host_intensity == !host_intensity_weight, "intensity and its weight come together");
  if(host_intensity && !v->col)
    return no_intensity(what);
  if(!v->store)
    return no_store(what);
  VOLUME_REQUIRE(count <= (size_t)INT32_MAX, "2^31 or more bricks");
  BrickIndex index;
  const int64_t bmin = INT64_MIN / STORE_BRICK, bmax = INT64_MAX / STORE_BRICK;   // 8 b + 7 fits
  for(size_t q = 0; q < count; ++q)
  {
    BrickCoord c;
    for(int a = 0; a < 3; ++a)
    {
      c.b[a] = host_coords[3 * q + a];
      VOLUME_REQUIRE(c.b[a] >= bmin && c.b[a] <= bmax, "brick coordinate out of range");
    }
    VOLUME_REQUIRE(index.slot.emplace(c, (int)q).second, "duplicate brick");
  }
  DeviceGuard guard(v->device);
  int rc = store_grow(v, count, what);
  if(rc) return rc;
  const size_t used = VOLUME_STORE_VOXELS * count;
  std::vector<float2> rec(used);
  for(size_t i = 0; i < used; ++i)
    rec[i] = make_float2(host_tsdf[i], host_weight[i]);
  if(used)
    RMD_CUDA_TRY(cudaMemcpyAsync(v->store->pool, rec.data(), sizeof(float2) * used, cudaMemcpyHostToDevice,
                                 v->stream));
  if(used && v->col)
  {
    for(size_t i = 0; i < used; ++i)
      rec[i] = host_intensity ? make_float2(host_intensity[i], host_intensity_weight[i]) : make_float2(0.0f, 0.0f);
    RMD_CUDA_TRY(cudaMemcpyAsync(v->store->pool_col, rec.data(), sizeof(float2) * used, cudaMemcpyHostToDevice,
                                 v->stream));
  }
  RMD_CUDA_TRY(cudaStreamSynchronize(v->stream));
  v->store->index.slot.swap(index.slot);
  return 0;
}

} // extern "C"
