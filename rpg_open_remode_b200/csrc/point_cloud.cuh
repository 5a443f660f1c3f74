// point_cloud.cuh -- point-cloud extraction behind the depth filter
// (SURVEY.md 8f row 3): rmd::Publisher::publishPointCloud, src/publisher.cpp:54-86,
// whose CPU double loop back-projects every CONVERGED pixel with T_world_ref and
// tags it with the reference image's 8-bit intensity, after downloading the
// whole depth and convergence maps.  Here: ordered stream compaction on the
// device (same row-major point order), only the points leave the GPU.
#pragma once

#include <cuda_runtime.h>

#include "rmd_common.cuh"

namespace rmdb
{

struct PointCloudParams
{
  int width, height;
  const int *conv; int conv_stride;          // ConvergenceState per pixel
  const float *depth; int depth_stride;      // floats per row ...
  int depth_comps;                           // ... and per pixel: 4 = mu inside the float4 seed records, 1 = planar image
  const float *ref; int ref_stride;          // reference image in [0,1] (intensity = rint(255 * ref))
  Camera cam;
  Pose T_world_ref;
  float4 *out;                               // (x, y, z, intensity) per point, row-major pixel order
  unsigned int capacity;                     // points that fit in out
  unsigned int *block_counts;                // [n_blocks] converged pixels per block, then exclusive offsets
  unsigned int *total;                       // [0] number of points, [1] ticket of the counting pass
  int n_blocks;
};

constexpr int POINT_CLOUD_BLOCK = 256;          // threads
constexpr int POINT_CLOUD_PIXELS = 4 * POINT_CLOUD_BLOCK;   // consecutive pixels (row-major) per block

// World point of pixel (x, y) at distance `depth` along its ray.  IEEE arithmetic in the order of the
// reference's host code (gcc -O3, no contraction): f = normalize((x-cx)/fx, (y-cy)/fy, 1) with normalize =
// v * (1 / sqrtf(dot)), xyz = T_world_ref * (f * depth)  (src/publisher.cpp:73-74, helper_math.h:1309-1313,
// se3.cuh:111-124,165-168).  Shared by the point cloud and the keyframe prior (prior.cuh), whose splat must
// start from exactly the published points.
__device__ __forceinline__ float3 back_project(const Camera &cam, const Pose &T_world_ref, int x, int y, float depth)
{
  const float vx = __fdiv_rn(__fsub_rn((float)x, cam.cx), cam.fx);
  const float vy = __fdiv_rn(__fsub_rn((float)y, cam.cy), cam.fy);
  const float dot = __fadd_rn(__fadd_rn(__fmul_rn(vx, vx), __fmul_rn(vy, vy)), 1.0f);   // + 1.0f * 1.0f
  const float inv_len = __fdiv_rn(1.0f, __fsqrt_rn(dot));
  const float px = __fmul_rn(__fmul_rn(vx, inv_len), depth);
  const float py = __fmul_rn(__fmul_rn(vy, inv_len), depth);
  const float pz = __fmul_rn(__fmul_rn(1.0f, inv_len), depth);
  const float *T = T_world_ref.m;
  float3 o;
  o.x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[0], px), __fmul_rn(T[1], py)), __fmul_rn(T[2], pz)), T[3]);
  o.y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4], px), __fmul_rn(T[5], py)), __fmul_rn(T[6], pz)), T[7]);
  o.z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[8], px), __fmul_rn(T[9], py)), __fmul_rn(T[10], pz)), T[11]);
  return o;
}

// Two launches: count (+ scan of the block totals by the last block), write.
cudaError_t launch_point_cloud(const PointCloudParams &P, cudaStream_t stream);

} // namespace rmdb
