// prior.cuh -- depth prior of a new keyframe from another keyframe's converged seeds (DESIGN.md 4.7).
// The reference starts every keyframe from the uniform prior; here, on request, the CONVERGED seeds of a
// source keyframe are forward-splatted into the new reference view (nearest surface per pixel) and become
// the prior (mu = splatted depth, sigma^2 = f * sigma^2_max, a = b = 10) of the pixels they land on.
#pragma once

#include <cuda_runtime.h>

#include "rmd_common.cuh"

namespace rmdb
{

struct PriorSplatParams
{
  // source keyframe: its state as the point cloud reads it
  int src_width, src_height;
  const int *conv; int conv_stride;          // ConvergenceState per pixel
  const float4 *seed; int seed_stride;       // (mu, sigma_sq, a, b)
  Camera src_cam;
  Pose T_world_ref;                          // source reference -> world
  // destination: the new reference view
  int dst_width, dst_height;
  Camera dst_cam;
  Pose T_curr_world;                         // world -> destination reference
  float min_depth, max_depth;
  unsigned int *zbuf;                        // dst_width x dst_height, dense; 0xFFFFFFFF = empty
};

struct PriorApplyParams
{
  int width, height;
  const unsigned int *zbuf;
  const int *conv; int conv_stride;
  float4 *seed; int seed_stride;
  float sigma_sq;                            // f * sigma^2_max of the destination
};

// z-buffer <- atomicMin of the bit pattern of every accepted point's distance (caller fills it with 0xFF first).
cudaError_t launch_prior_splat(const PriorSplatParams &P, cudaStream_t stream);
// Seeds of non-BORDER pixels with a z-buffer entry <- (depth, sigma_sq, 10, 10).
cudaError_t launch_prior_apply(const PriorApplyParams &P, cudaStream_t stream);

} // namespace rmdb
