// rmd_common.cuh -- shared definitions of the sm_90a depth-filter library.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/rmd_b200.h"

namespace rmdb
{

// ---------------------------------------------------------------- errors
void set_last_error(const std::string &msg);
int fail(int code, const char *what);
int fail_cuda(cudaError_t err, const char *what);

#define RMD_CUDA_TRY(expr)                                   \
  do {                                                       \
    const cudaError_t rmd_err_ = (expr);                     \
    if(rmd_err_ != cudaSuccess)                              \
      return ::rmdb::fail_cuda(rmd_err_, #expr);             \
  } while(0)

#define RMD_REQUIRE(cond, what)                              \
  do {                                                       \
    if(!(cond))                                              \
      return ::rmdb::fail(RMD_ERR_INVALID_ARGUMENT, what);   \
  } while(0)

// RAII device switch: handles are pinned to the device they were created on.
struct DeviceGuard
{
  explicit DeviceGuard(int device) : prev_(-1), changed_(false)
  {
    if(cudaGetDevice(&prev_) == cudaSuccess && prev_ != device)
    {
      changed_ = (cudaSetDevice(device) == cudaSuccess);
    }
  }
  ~DeviceGuard()
  {
    if(changed_) cudaSetDevice(prev_);
  }
  int prev_;
  bool changed_;
};

// ------------------------------------------------------------ geometry
// SE3 as 12 floats, row-major 3x4 [R|t] (the reference's layout,
// include/rmd/se3.cuh:142 "Matrix<Type,3,4> data").
struct Pose
{
  float m[12];
};

inline Pose pose_from(const float *v)
{
  Pose p;
  for(int i = 0; i < 12; ++i) p.m[i] = v[i];
  return p;
}
Pose pose_inverse(const Pose &T);                 // se3.cuh:81-97
Pose pose_compose(const Pose &a, const Pose &b);  // se3.cuh:146-162

struct Camera
{
  float fx, fy, cx, cy;
};

// Everything the fused depth-filter kernel needs, passed by value as a
// __grid_constant__ parameter (replaces the reference's mvs::DeviceData block
// that lives in device memory and is pointer-chased by every thread,
// include/rmd/mvs_device_data.cuh:47-106).
struct FilterParams
{
  int width, height;
  // seed state, array-of-structures: one float4 (mu, sigma_sq, a, b) per pixel
  float4 *seed;
  int seed_stride;      // in float4 elements
  // NCC template statistics: float2 (sum_templ, const_templ_denom)
  const float2 *templ;
  int templ_stride;     // in float2 elements
  int *conv;            // ConvergenceState per pixel
  int conv_stride;      // in ints
  const float *ref;     // reference image
  int ref_stride;       // in floats
  const float *curr;    // current image
  int curr_stride;      // in floats
  float2 *matches;      // optional (RMD_OPT_RECORD_MATCHES), may be null
  int match_stride;     // in float2 elements
  Camera cam;
  Pose T_curr_ref;
  Pose T_ref_curr;
  float eta_inlier, eta_outlier, epsilon;
  float depth_range;
  float one_pix_angle;
  float tex_quant;      // 2^frac_bits of the bilinear weights, 0 = exact
  int trust_conv;       // 1: absorbing states recorded in conv are final
  unsigned int *converged_now;   // counter of this frame
  unsigned int *converged_next;  // counter to clear for the next frame
  long long *timeline;           // debug: 8 clock64() stamps per CTA of the staged kernel, or null
  // staged kernel: per-frame work list and busy-tile splitting (depth_filter_staged.cu)
  int split_max;                         // most CTAs sharing one tile; 1 = never split
  int split_min_items, split_items_per_cta, sparse_max_seeds;  // tuning (staged_maps.cuh defaults)
  int heavy_min_items;                   // tiles with at least this many items are dispatched first
  int pdl;                               // host only: launch with programmatic stream serialisation
  int split_avg_pct;                     // ... and split only above this percentage of the average items per CTA slot
  int cta_slots;                         // resident CTAs of the whole GPU (SMs x CTAs per SM)
  unsigned long long *tile_keys;         // [tiles][256] partial arg-max keys of split tiles
  unsigned int *tile_arrivals;           // [tiles] CTAs of a split tile that finished searching
  int n_tiles, tiles_x;                  // tile grid of the image
  // Work list of this frame, written by the lead CTAs of the previous frame.
  // Entry = tile | share << 20 | zeff << 26.  CTA b takes heavy_cur[b], then
  // light_cur[b - n_heavy]; CTAs beyond both lists exit.  Tiles whose seeds
  // are all in absorbing states are not listed again (their converged seeds
  // are counted once in *retired_converged).
  const unsigned int *heavy_cur, *light_cur;
  unsigned int *heavy_next, *light_next;
  // Third class: tiles with a handful of seeds left to update and a few dozen candidates in all.  They are
  // processed by ONE WARP each (eight per CTA), entry = tile; counts[6] entries.
  const unsigned int *sparse_cur;
  unsigned int *sparse_next;
  int warp_tile_max_seeds;               // 0: no warp tiles
  int warp_tile_max_cands;               // a warp tile has at most this many candidates in all
  int ctas_per_sm;                       // 5x5 staged kernel: 2 (128 registers) or 3 (80 registers) resident CTAs per SM (host side only)
  int grid_ctas;                         // 0: one CTA per resident slot; else the persistent grid's size (host side only)
  int run_chunks;                        // chunks per work item of the staged search; 0: chosen per tile
  // {heavy entries, light entries, helper entries reserved, work items of the frame, tiles listed (lead
  //  entries), lead CTAs of the previous frame that have finished listing, sparse entries, -}: 8 uints per frame
  const unsigned int *counts_cur;
  unsigned int *counts_next, *counts_zero;
  unsigned int *retired_converged;
  int helper_cap;                        // most helper entries per frame
  // Frame chaining (several consecutive frames of one keyframe in ONE launch, depth_filter_staged.cu):
  unsigned int frame_no;                 // updates since set_reference, 1, 2, ...
  unsigned int *tile_done;               // [tiles] frame_no of the last frame that finalised the tile
  unsigned int *list_ready;              // highest frame_no whose work list is complete
};

} // namespace rmdb
