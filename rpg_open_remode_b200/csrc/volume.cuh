// volume.cuh -- fusion of finished keyframes into a dense TSDF voxel grid (DESIGN.md 4.8).
// The reference publishes every keyframe's point cloud on its own and leaves fusion to the consumer; here the
// depth maps are fused on the device into one truncated signed distance function, from which the surface can be
// extracted as points or raycast into a depth map from any pose.
//
// Layout: voxel (i, j, k) is the float2 record (tsdf, weight) at (k * ny + j) * nx + i (64-bit), x fastest; its
// world position is origin + (i, j, k) * voxel_size (origin = centre of voxel (0, 0, 0)).  Weight 0 = unknown.
// Every per-voxel and per-ray expression uses explicit round-to-nearest intrinsics in a fixed operation order,
// so that a CPU restatement can match the kernels bit for bit.
#pragma once

#include <cuda_runtime.h>

#include "rmd_common.cuh"

namespace rmdb
{

struct VolumeGrid
{
  float2 *vox;
  int nx, ny, nz;
  float voxel;            // edge length
  float ox, oy, oz;       // centre of voxel (0, 0, 0)
};

struct VolumeIntegrateParams
{
  VolumeGrid g;
  int width, height;
  Camera cam;
  Pose T_curr_world;                        // world -> camera of the depth image
  const float *depth; size_t depth_stride;  // floats per row ...
  int depth_comps;                          // ... and per pixel: 4 = mu inside the float4 seed records, 1 = planar
  const int *conv; size_t conv_stride;      // ConvergenceState per pixel, or null: every pixel counts
  float trunc, max_weight;
};

struct VolumeSurfaceParams
{
  VolumeGrid g;
  float4 *out;                              // (x, y, z, min weight) per point
  unsigned long long capacity;              // points that fit in out
  unsigned long long *block_offsets;        // [n_blocks] points per block, then exclusive offsets
  unsigned long long *total;                // [0] number of points
  unsigned int n_blocks;
};

struct VolumeRaycastParams
{
  VolumeGrid g;
  int width, height;
  Camera cam;
  Pose T_world_curr;                        // camera -> world (pose_inverse of the caller's T_curr_world)
  float *depth; size_t depth_stride;        // floats per row: distance along the ray, 0 = no surface
};

constexpr int VOLUME_SURF_BLOCK = 256;                               // threads
constexpr int VOLUME_SURF_ROUNDS = 8;                                // rounds of VOLUME_SURF_BLOCK voxels
constexpr int VOLUME_SURF_VOXELS = VOLUME_SURF_BLOCK * VOLUME_SURF_ROUNDS;   // consecutive voxels per block
constexpr int VOLUME_SCAN_BLOCK = 1024;                              // threads of the block-offset scan

// Every voxel in the depth image's view: running average of the truncated SDF, one observation = weight 1.
cudaError_t launch_volume_integrate(const VolumeIntegrateParams &P, cudaStream_t stream);
// Surface points, pass 1: points per block, then one block turns the block totals into exclusive offsets
// (and *total); pass 2: the points at their rank (voxel order, then axis x, y, z).  Pass 2 may run with a
// capacity set after reading *total.
cudaError_t launch_volume_surface_count(const VolumeSurfaceParams &P, cudaStream_t stream);
cudaError_t launch_volume_surface_write(const VolumeSurfaceParams &P, cudaStream_t stream);
// One ray per pixel: distance to the first zero crossing of the trilinearly interpolated TSDF.
cudaError_t launch_volume_raycast(const VolumeRaycastParams &P, cudaStream_t stream);

} // namespace rmdb
