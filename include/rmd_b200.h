/*
 * rmd_b200.h -- C-ABI of the Hopper-native (sm_90a) REMODE depth-filter hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++ types, no
 * exceptions, no torch.  Every entry point replaces one member of the
 * reference's device-side classes (paths relative to the reference tree):
 *
 *   rmd_seeds_*      rmd::SeedMatrix        include/rmd/seed_matrix.cuh:45-109
 *                                           src/seed_matrix.cu:28-230
 *   rmd_denoiser_*   rmd::DepthmapDenoiser  include/rmd/depthmap_denoiser.cuh:27-54
 *                                           src/depthmap_denoiser.cu:124-229
 *   rmd_reduce_*     rmd::ImageReducer<T>   include/rmd/reduction.cuh:27-62
 *                                           src/reduction.cu:22-187
 *   rmd_image_*      rmd::DeviceImage<T>    include/rmd/device_image.cuh:34-180
 *
 * include/rmd/ holds header-compatible C++ classes (same names and signatures
 * as the reference's) that forward to these functions and turn non-zero
 * return codes back into rmd::CudaException, so rmd::Depthmap / the ROS node
 * compile against them unchanged (see INTEGRATION.md).
 *
 * Conventions
 *   - every function returns 0 on success, otherwise a cudaError_t value or
 *     one of the RMD_ERR_* codes below; rmd_last_error_string() describes the
 *     last failure of the calling thread;
 *   - host images are densely packed row-major (width*sizeof(T) pitch), gray
 *     value / 255 in [0,1] for float frames, as the reference requires
 *     (device_image.cuh:95-102, src/depthmap.cpp:105);
 *   - poses are SE3 3x4 row-major [R|t] float[12] (include/rmd/se3.cuh:27-142),
 *     world -> camera ("T_curr_world"), exactly what SeedMatrix takes;
 *   - a handle owns its device memory and a CUDA stream on the device it was
 *     created for; handles share no process-global state, so several can run
 *     concurrently on one GPU or one per GPU;
 *   - calls on one handle must come from one thread at a time (as with the
 *     reference: src/main_ros.cpp:43-48).
 */
#ifndef RMD_B200_H
#define RMD_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RMD_B200_ABI_VERSION 1

/* own error codes (cudaError_t values are small positive integers) */
#define RMD_ERR_INVALID_ARGUMENT (-1)
#define RMD_ERR_NOT_INITIALISED  (-2)  /* e.g. update before set_reference */
#define RMD_ERR_UNSUPPORTED      (-3)
#define RMD_ERR_DEVICE_WAIT       (-4)  /* a bounded device-side wait of a chained launch expired (a bug, not a state) */

/* rmd::ConvergenceStates, include/rmd/seed_matrix.cuh:31-43 */
enum rmd_convergence_state {
  RMD_UPDATE = 0,
  RMD_CONVERGED = 1,
  RMD_BORDER = 2,
  RMD_DIVERGED = 3,
  RMD_NO_MATCH = 4,
  RMD_NOT_VISIBLE = 5
};

/* Per-pixel fields of a seed matrix (download / upload / device_ptr). */
enum rmd_field {
  RMD_FIELD_MU = 0,                /* float   SeedMatrix::downloadDepthmap    seed_matrix.cu:160 */
  RMD_FIELD_SIGMA_SQ = 1,          /* float   downloadSigmaSq                 :206 */
  RMD_FIELD_A = 2,                 /* float   downloadA                       :210 */
  RMD_FIELD_B = 3,                 /* float   downloadB                       :214 */
  RMD_FIELD_CONVERGENCE = 4,       /* int32   downloadConvergence             :165 */
  RMD_FIELD_SUM_TEMPL = 5,         /* float   downloadSumTempl                :218 */
  RMD_FIELD_CONST_TEMPL_DENOM = 6, /* float   downloadConstTemplDenom         :222 */
  RMD_FIELD_EPIPOLAR_MATCHES = 7,  /* float2  downloadEpipolarMatches         :226 */
  RMD_FIELD_REF_IMG = 8,           /* float   the reference image as uploaded */
  RMD_FIELD_DEBUG_TIMELINE = 100   /* int64[16] per tile, see RMD_OPT_DEBUG_TIMELINE */
};

enum rmd_seeds_option {
  /* 1: keep the best epipolar match of every pixel (RMD_FIELD_EPIPOLAR_MATCHES);
   * off by default because nothing downstream of update() reads it
   * (it exists in the reference for tests: seed_matrix.cuh:76-83). */
  RMD_OPT_RECORD_MATCHES = 0,
  /* 0 (default): staged kernel (TMA -> shared memory, balanced candidate work
   * list), 1: direct kernel (one thread per pixel, global loads); same
   * arithmetic, bit-identical results. */
  RMD_OPT_KERNEL_VARIANT = 1,
  /* fractional bits of the bilinear weights of the current-image taps
   * (8 = what the texture unit of the reference path uses; 0 = exact fp32). */
  RMD_OPT_TEX_FRAC_BITS = 2,
  /* debug: the staged kernel records 16 x int64 per 32x8 tile (clock64 at its
   * phase boundaries, SM id, work items, strip coverage ...); read them back
   * with rmd_seeds_download(h, RMD_FIELD_DEBUG_TIMELINE, dst) where dst holds
   * 16 * ceil(w/32) * ceil(h/8) int64 values. */
  RMD_OPT_DEBUG_TIMELINE = 3,
  /* 1: a host frame given to rmd_seeds_update* / set_reference* that lies in
   * page-locked memory (cudaHostAlloc / cudaHostRegister, detected with
   * cudaPointerGetAttributes) is DMA'd straight from the caller's buffer:
   * no staging copy into the library's pinned ring.  The caller then must
   * leave the frame untouched until rmd_seeds_sync() (or any download)
   * returns -- the reference's "reusable on return" guarantee
   * (device_image.cuh:93-106) no longer holds for such buffers.  Pageable
   * buffers still take the staged path.  Default 0. */
  RMD_OPT_PINNED_INPUT = 4,
  /* Frames per launch of rmd_seeds_update_device_batch (1..8, default 1): with n > 1, n consecutive frames of
   * the keyframe are chained inside ONE persistent launch -- a tile moves on to frame k+1 as soon as its own
   * frame k is final, so frames overlap on the GPU.  Same results as one launch per frame.  Opt-in: whether it
   * pays depends on the image size and the register budget of the kernel (bench.py --chain-frames). */
  RMD_OPT_CHAIN_FRAMES = 5,
  /* Seed-major mode: once at most this percentage of the pixels is still being updated (0 = never, the default)
   * the handle keeps the live seeds as a compact list and a launch walks every listed seed through its frames
   * warp by warp -- no tiles, no per-frame synchronisation (csrc/depth_filter_seeds.cu).  Same results.  Off by
   * default: on the bench workloads 10-20 % of the seeds stay live (NO_MATCH seeds keep searching) and at that
   * density the tile organisation is expected to be faster; it pays for sparser live sets
   * (bench.py --seed-mode-pct). */
  RMD_OPT_SEED_MODE_PCT = 6,
  /* tuning knobs of the staged kernel's busy-tile splitting and sparse-tile
   * path (defaults in csrc/staged_maps.cuh); results never depend on them */
  RMD_OPT_TUNE_SPLIT_MAX = 10,            /* most CTAs sharing one busy tile (1 = never split; default 16) */
  RMD_OPT_TUNE_SPLIT_MIN_ITEMS = 11,      /* tiles with fewer work items are never split (512) */
  RMD_OPT_TUNE_SPLIT_ITEMS_PER_CTA = 12,  /* least work items a CTA of a split tile gets (384) */
  RMD_OPT_TUNE_SPARSE_MAX_SEEDS = 13,     /* tiles with at most this many seeds to update skip TMA staging (16; 0 = off) */
  RMD_OPT_TUNE_HEAVY_MIN_ITEMS = 14,      /* tiles with at least this many items are dispatched first (128) */
  RMD_OPT_TUNE_SPLIT_AVG_PCT = 15,        /* target items per CTA of a split tile, in % of the frame's items per resident CTA slot (50) */
  RMD_OPT_TUNE_PDL = 16,           /* 1 (default): programmatic dependent launch of consecutive frames */
  RMD_OPT_TUNE_WARP_TILE_SEEDS = 17, /* tiles with at most this many seeds to update (and a few dozen candidates) are processed by one warp, eight tiles per CTA (8 = the most; 0 = off) */
  RMD_OPT_TUNE_GRID_CTAS = 18,      /* size of the persistent grid (0, the default: one CTA per resident slot, SMs x occupancy) */
  RMD_OPT_TUNE_CTAS_PER_SM = 19,    /* 5x5 staged kernel: the 128-register build (2, = 0, the default) or the 80-register build (3; sized for 3 CTAs per SM, of which two fit next to the 60 KB strips) */
  RMD_OPT_TUNE_WARP_TILE_CANDS = 20, /* ... and at most this many candidates in all (64 = the most) */
  RMD_OPT_TUNE_RUN_CHUNKS = 21       /* 4-candidate chunks one work item of the staged search scores (0, the default: chosen per tile; 1..36) */
};

typedef struct rmd_seeds rmd_seeds_t;
typedef struct rmd_denoiser rmd_denoiser_t;
typedef struct rmd_multi rmd_multi_t;
typedef struct rmd_volume rmd_volume_t;

/* ------------------------------------------------------------------ misc */
int rmd_abi_version(void);
const char *rmd_last_error_string(void);
int rmd_device_count(int *count);

/* ----------------------------------------------------------- seed matrix */

/* SeedMatrix::SeedMatrix(width, height, PinholeCamera(fx,fy,cx,cy))
 * seed_matrix.cu:28-80.  patch_side = RMD_CORR_PATCH_SIDE (5 or 7; a compile
 * time macro in the reference, CMakeLists.txt:51).  device < 0: current. */
int rmd_seeds_create(int width, int height, float fx, float fy, float cx,
                     float cy, int patch_side, int device, rmd_seeds_t **out);
int rmd_seeds_destroy(rmd_seeds_t *s);

/* Run this handle's work on a caller-owned cudaStream_t (NULL = back to the
 * handle's own stream).  The reference uses the legacy default stream only. */
int rmd_seeds_set_stream(rmd_seeds_t *s, void *cuda_stream);
int rmd_seeds_get_stream(rmd_seeds_t *s, void **cuda_stream);
int rmd_seeds_set_option(rmd_seeds_t *s, int option, int value);

/* SeedMatrix::setReferenceImage, seed_matrix.cu:87-118.  Host buffer. */
int rmd_seeds_set_reference(rmd_seeds_t *s, const float *host_img,
                            const float *T_curr_world, float min_depth,
                            float max_depth);
/* Same with the image already in device memory (pitch in bytes). */
int rmd_seeds_set_reference_device(rmd_seeds_t *s, const float *dev_img,
                                   size_t pitch_bytes,
                                   const float *T_curr_world, float min_depth,
                                   float max_depth);
/* Same from an 8-bit gray frame; value * (1/255.f) is applied on the GPU
 * (what rmd::Depthmap::inputImage does on the CPU, src/depthmap.cpp:105). */
int rmd_seeds_set_reference_u8(rmd_seeds_t *s, const uint8_t *host_img,
                               const float *T_curr_world, float min_depth,
                               float max_depth);

/* Depth prior of a new keyframe from the converged seeds of another one (the
 * reference starts every keyframe from the uniform prior; DESIGN.md 4.7).
 * Every CONVERGED seed of the source is back-projected exactly as
 * rmd_seeds_point_cloud does, moved into the new reference view, and splatted
 * to the nearest pixel (the nearest surface wins; points behind the camera,
 * outside [min_depth, max_depth] or outside the image are dropped).  After the
 * usual initialisation, every non-BORDER pixel that received a point gets the
 * seed (distance, sigma_sq_frac * range^2 / 36, 10, 10); all others keep the
 * uniform prior.  The state stays UPDATE: new frames still have to confirm it.
 *
 * In place, for the reference's single-Depthmap node: with f > 0, every later
 * set_reference* on s (float, u8 with or without undistortion, device) first
 * splats s's own CONVERGED seeds of the keyframe it is leaving into the new
 * reference view, then initialises, then applies the prior.  f = 0 (the
 * default) switches it off.  f must be in [0, 1]. */
int rmd_seeds_set_prior_propagation(rmd_seeds_t *s, float sigma_sq_frac);

/* Cross-handle, for a set of live keyframes: dst has just had set_reference*
 * and no update since; its seeds receive the prior splatted from src's current
 * state (f in (0, 1]).  Image sizes and cameras may differ; the device must be
 * the same.  Asynchronous, ordered on the device like
 * rmd_denoiser_run_seeds_to_device: a later update of src does not overwrite
 * seeds the splat is still reading.  Returns RMD_ERR_NOT_INITIALISED if dst
 * has no reference or has been updated since it was set, or if src has no
 * reference.  A source without CONVERGED seeds leaves dst's initial state. */
int rmd_seeds_propagate_prior(rmd_seeds_t *dst, const rmd_seeds_t *src, float sigma_sq_frac);

/* SeedMatrix::update, seed_matrix.cu:120-158: convergence check, epipolar NCC
 * search, triangulation and Bayesian update of every seed -- one fused kernel.
 * The host buffer may be reused as soon as the call returns (it is copied to
 * a pinned ring); the GPU work is enqueued on the handle's stream and, like
 * the reference's last kernel, may still be running on return. */
int rmd_seeds_update(rmd_seeds_t *s, const float *host_img,
                     const float *T_curr_world);
int rmd_seeds_update_u8(rmd_seeds_t *s, const uint8_t *host_img,
                        const float *T_curr_world);

/* Several live reference keyframes against one incoming frame (SURVEY.md 8f
 * row 2; the reference node keeps a single rmd::Depthmap and re-keyframes,
 * src/depthmap_node.cpp:125-157).  The frame is staged and uploaded ONCE
 * (through handles[0]) and the keyframes are updated by ONE launch per group
 * of up to 8 (on handles[0]'s stream; the other handles' streams wait for
 * it): the launch's work list is the concatenation of the keyframes' lists,
 * so their dependent chains interleave from the first cycle -- steady frames
 * of one keyframe leave most issue slots idle (DESIGN.md 4.1).  Handles on
 * the direct variant or with another patch size are enqueued one by one.
 * Same result, bit for bit, as calling rmd_seeds_update[_u8] on each handle.
 * All handles must have the same image size and device and a reference
 * frame; at most 64 per call. */
int rmd_seeds_update_many(rmd_seeds_t *const *handles, int n, const float *host_img,
                          const float *T_curr_world);
int rmd_seeds_update_many_u8(rmd_seeds_t *const *handles, int n, const uint8_t *host_img,
                             const float *T_curr_world);

/* Frame ingest with lens undistortion (SURVEY.md 8f row 1).
 * rmd::Depthmap::initUndistortionMap(k1, k2, r1, r2), src/depthmap.cpp:45-61:
 * builds the fixed-point maps of cv::initUndistortRectifyMap(K, D, I, K, size,
 * CV_16SC2) for the handle's camera.  From then on the *_u8 entry points
 * (set_reference_u8, update_u8) run rmd::Depthmap::inputImage
 * (src/depthmap.cpp:95-106) on the GPU, fused in one kernel: cv::remap(...,
 * CV_INTER_LINEAR) of the 8-bit frame, then convertTo(CV_32F, 1/255.f).  Float
 * entry points are not affected (the reference's SeedMatrix takes undistorted
 * float images).  k1 = k2 = r1 = r2 = 0 is still a remap (identity up to the
 * map's rounding); rmd_seeds_clear_undistortion_map() switches it off. */
int rmd_seeds_init_undistortion_map(rmd_seeds_t *s, float k1, float k2, float r1, float r2);
int rmd_seeds_clear_undistortion_map(rmd_seeds_t *s);
/* The maps as OpenCV lays them out: xy = CV_16SC2 (2*w*h int16: x, y of the
 * top-left source pixel), frac = CV_16UC1 (w*h: (fy << 5) | fx, 5-bit
 * fractions).  Either pointer may be NULL. */
int rmd_seeds_get_undistortion_map(rmd_seeds_t *s, int16_t *host_xy, uint16_t *host_frac);
/* img_undistorted_8uc1_ of rmd::Depthmap (src/depthmap.cpp:99): the remapped
 * 8-bit frame itself, host to host (the reference keeps it as the intensity
 * source of the published point cloud).  Synchronous. */
int rmd_seeds_undistort_u8(rmd_seeds_t *s, const uint8_t *host_src, uint8_t *host_dst);
/* Frame already resident in device memory (must stay valid until the stream
 * has consumed it).  pitch_bytes must be a multiple of 16. */
int rmd_seeds_update_device(rmd_seeds_t *s, const float *dev_img,
                            size_t pitch_bytes, const float *T_curr_world);

/* n_frames consecutive updates from frames resident in device memory:
 * frame i starts at dev_frames + i*frame_stride_bytes (pitch_bytes per row),
 * its pose is T_curr_world + 12*i.  One call, n_frames fused launches, no
 * host round trip in between (the sequence is strictly ordered: frame k+1
 * searches around the posterior frame k left, epipolar_match.cu:60-75). */
int rmd_seeds_update_device_batch(rmd_seeds_t *s, const float *dev_frames,
                                  size_t frame_stride_bytes,
                                  size_t pitch_bytes, int n_frames,
                                  const float *T_curr_world);

int rmd_seeds_sync(rmd_seeds_t *s);

/* download* accessors: dst is width*height elements, densely packed. */
int rmd_seeds_download(rmd_seeds_t *s, int field, void *host_dst);
/* Test / checkpoint hook the reference lacks: overwrite one field
 * (MU, SIGMA_SQ, A, B, CONVERGENCE). */
int rmd_seeds_upload_state(rmd_seeds_t *s, int field, const void *host_src);
/* getMu()/getSigmaSq()/getA()/getB()/getConvergence(): a pitched planar
 * device image of the field, valid until the next call on this handle. */
int rmd_seeds_device_ptr(rmd_seeds_t *s, int field, void **dev_ptr,
                         size_t *pitch_bytes);
/* Copy a field into caller-owned device memory, ASYNCHRONOUSLY on the handle's
 * stream: a consumer on any other stream (including the legacy default stream
 * of rmd_reduce_* and the denoiser's own stream) must rmd_seeds_sync() first. */
int rmd_seeds_copy_field_to_device(rmd_seeds_t *s, int field, void *dev_dst,
                                   size_t dst_pitch_bytes);

/* SeedMatrix::getConvergedCount, seed_matrix.cu:195-198: number of pixels the
 * last update() classified CONVERGED (the fused kernel counts them; no extra
 * pass).  Before the first update it is 0. */
int rmd_seeds_converged_count(rmd_seeds_t *s, size_t *count);
/* SeedMatrix::getDistFromRef, seed_matrix.cu:200-203. */
int rmd_seeds_dist_from_ref(rmd_seeds_t *s, float *dist);
int rmd_seeds_size(rmd_seeds_t *s, int *width, int *height, int *patch_side);
/* Number of fused depth-filter kernels / all kernels this handle launched. */
int rmd_seeds_launch_count(rmd_seeds_t *s, uint64_t *fused, uint64_t *total);
/* Device time of the last fused depth-filter kernel in milliseconds, measured
 * with CUDA events on the handle's stream (blocks until it finished). */
int rmd_seeds_last_kernel_ms(rmd_seeds_t *s, float *ms);
int rmd_seeds_enable_kernel_timing(rmd_seeds_t *s, int on);
/* Debug: host-side time of the streaming ingest, accumulated over all handles
 * of the process when the environment variable RMD_HOST_PROFILE is set:
 * out[0] wait for a free ring slot, [1] copy into pinned memory, [2] enqueue
 * the host-to-device copy, [3] encode TMA descriptors, [4] launch,
 * [5] whole rmd_seeds_update* call (all seconds), [6] number of calls.
 * reset != 0 clears the accumulators after reading. */
int rmd_debug_host_profile(double out[8], int reset);

/* Point-cloud extraction (SURVEY.md 8f row 3).
 * rmd::Publisher::publishPointCloud, src/publisher.cpp:54-86: every pixel whose
 * state is CONVERGED becomes a point  T_world_ref * (normalize((x-cx)/fx,
 * (y-cy)/fy, 1) * depth(y, x))  with the 8-bit intensity of the reference image,
 * in row-major pixel order.  The reference downloads the depth and convergence
 * maps and loops on the CPU; here the points are compacted on the device (same
 * order, IEEE arithmetic in the reference's operation order) and only they are
 * copied out.  `dev_depth` is a pitched device image (e.g. the denoised map of
 * rmd_denoiser_run_seeds_to_device) or NULL for the seeds' own depth estimate.
 * Points are 4 floats (x, y, z, intensity).  *count is always the number of
 * CONVERGED pixels; at most `capacity_points` points are written.  Synchronous. */
int rmd_seeds_point_cloud(rmd_seeds_t *s, const float *dev_depth, size_t depth_pitch_bytes,
                          float *host_xyzi, size_t capacity_points, size_t *count);
/* Same into device memory (16-byte aligned). */
int rmd_seeds_point_cloud_device(rmd_seeds_t *s, const float *dev_depth, size_t depth_pitch_bytes,
                                 float *dev_xyzi, size_t capacity_points, size_t *count);

/* -------------------------------------------------------------- denoiser */

/* DepthmapDenoiser(width, height), depthmap_denoiser.cu:143-177 */
int rmd_denoiser_create(int width, int height, int device,
                        rmd_denoiser_t **out);
int rmd_denoiser_destroy(rmd_denoiser_t *d);
int rmd_denoiser_set_stream(rmd_denoiser_t *d, void *cuda_stream);
/* setLargeSigmaSq(depth_range), :226-229 */
int rmd_denoiser_set_large_sigma_sq(rmd_denoiser_t *d, float depth_range);
/* denoise(mu, sigma_sq, a, b, host_denoised, lambda, iterations), :179-224.
 * Inputs are pitched planar float images in device memory (pitch in bytes).
 * Returns RMD_ERR_NOT_INITIALISED if set_large_sigma_sq was never called
 * (the reference prints to stderr and returns, :189-193). */
int rmd_denoiser_run(rmd_denoiser_t *d, const float *mu, size_t mu_pitch,
                     const float *sigma_sq, size_t sigma_sq_pitch,
                     const float *a, size_t a_pitch, const float *b,
                     size_t b_pitch, float *host_denoised, float lambda,
                     int iterations);
/* Same, reading the seed state of `s` directly (no planar export). */
int rmd_denoiser_run_seeds(rmd_denoiser_t *d, rmd_seeds_t *s,
                           float *host_denoised, float lambda, int iterations);
/* Same, leaving the result in caller-owned device memory (no D2H copy).
 * Asynchronous on the denoiser's stream.  The seeds handle is ordered after it:
 * a following rmd_seeds_point_cloud(s, dev_out, ...), update or set_reference
 * on `s` waits (on the device) for the denoised map / for the read of the seed
 * state.  Any OTHER consumer of dev_out must rmd_denoiser_sync() first. */
int rmd_denoiser_run_seeds_to_device(rmd_denoiser_t *d, rmd_seeds_t *s,
                                     float *dev_out, size_t out_pitch_bytes,
                                     float lambda, int iterations);
int rmd_denoiser_sync(rmd_denoiser_t *d);
int rmd_denoiser_launch_count(rmd_denoiser_t *d, uint64_t *total);

/* ------------------------------------------------------------ reductions */

/* ImageReducer<T>::sum / countEqual, reduction.cu:81-184.  Device pointer,
 * stride in ELEMENTS (as the reference), legacy default stream, blocking.
 * Only the width x height elements are read, never a row's padding.  Width
 * or height 0 returns an error.
 * sum_f32 accumulates in double and rounds once to float: |out - exact| <=
 * 1/2 ulp(exact) + n 2^-53 sum|x| for n elements (faithful, not always
 * correctly rounded; with cancellation the second term dominates); an inf
 * entry gives that inf, +inf with -inf or a NaN entry gives NaN.
 * sum_i32 wraps exactly like int32 addition. */
int rmd_reduce_sum_f32(const float *dev_img, size_t stride, size_t width,
                       size_t height, float *out);
int rmd_reduce_sum_i32(const int32_t *dev_img, size_t stride, size_t width,
                       size_t height, int32_t *out);
int rmd_reduce_count_eq_i32(const int32_t *dev_img, size_t stride,
                            size_t width, size_t height, int32_t value,
                            size_t *out);
/* extras the north star asks for (not in the reference).
 * min_max_f32: NaN entries are ignored; an image with no non-NaN entry
 * returns (+inf, -inf).  Infinities are values like any other, and -0 and +0
 * compare equal (either may be returned). */
int rmd_reduce_min_max_f32(const float *dev_img, size_t stride, size_t width,
                           size_t height, float *out_min, float *out_max);

/* -------------------------------------------------------------- multi-GPU */

/* Independent reference keyframes, one rmd_seeds_t per GPU (SURVEY.md 8e).  The
 * depth filter never reads a neighbour's or another keyframe's state
 * (src/seed_check.cu, src/epipolar_match.cu, src/seed_update.cu), so there is
 * no data-path collective: the only exchange is the FINAL GATHER of every
 * keyframe's depth (f32) and convergence (i32) map to one root GPU -- grouped
 * ncclSend / ncclRecv over NVLink.  The reference has no multi-GPU path (one
 * SeedMatrix on the current device, src/check_cuda_device.cu:109).  NCCL
 * (libnccl.so.2) is loaded at run time; without it these functions return
 * RMD_ERR_UNSUPPORTED.
 *
 * One process driving n GPUs (e.g. a node owning several rmd::Depthmap
 * objects): rank i <-> devices[i]; ncclCommInitAll. */
int rmd_multi_create(const int *devices, int n, int width, int height, rmd_multi_t **out);
/* One process per GPU: rank 0 calls rmd_multi_unique_id, ships the 128 bytes to
 * the other ranks by its own means, every rank calls rmd_multi_create_rank
 * (collective: ncclCommInitRank).  device < 0: current. */
int rmd_multi_unique_id(char id[128]);
int rmd_multi_create_rank(const char id[128], int n_ranks, int rank, int device, int width,
                          int height, rmd_multi_t **out);
int rmd_multi_destroy(rmd_multi_t *m);
int rmd_multi_size(rmd_multi_t *m, int *n_ranks, int *n_local, int *first_rank);
/* The final gather.  seeds[i]: keyframe of local member i (n entries after
 * rmd_multi_create, one after rmd_multi_create_rank), whose queued updates are
 * waited for on the device.  dev_depth (may be NULL, entries may be NULL): a
 * pitched device image to send instead of the seeds' own depth estimate, e.g.
 * the denoised map of rmd_denoiser_run_seeds_to_device (complete when this is
 * called: rmd_denoiser_sync).  On the process that holds rank `root`,
 * host_depth / host_conv receive n_ranks * width * height elements each, rank
 * after rank; elsewhere they may be NULL.  Collective over all ranks; returns
 * when the exchange has finished. */
int rmd_multi_gather_maps(rmd_multi_t *m, rmd_seeds_t *const *seeds,
                          const float *const *dev_depth, const size_t *dev_depth_pitch,
                          int root, float *host_depth, int32_t *host_conv);

/* ------------------------------------------------------------ TSDF volume */

/* Fusion of finished keyframes into one dense truncated signed distance
 * function on the device (DESIGN.md 4.8; the reference publishes every
 * keyframe's point cloud on its own and leaves fusion to the consumer).
 * Voxel (i, j, k), 0 <= i < nx (x fastest), holds (tsdf, weight); its world
 * position is origin + (i, j, k) * voxel_size, so origin is the CENTRE of
 * voxel (0, 0, 0).  Weight 0 = unknown.  All arithmetic is IEEE
 * round-to-nearest in a fixed operation order (bit-reproducible).
 *
 * A new volume is all unknown.  truncation tau (metres) > 0; max_weight >= 1
 * caps the weight of a voxel (one observation = 1).  At most 2^31 voxels.
 * device < 0: current.  Returns RMD_ERR_INVALID_ARGUMENT for a null pointer,
 * a dimension <= 0, too many voxels, voxel_size or truncation <= 0, or
 * max_weight < 1. */
int rmd_volume_create(int nx, int ny, int nz, float voxel_size, const float origin[3], float truncation,
                      float max_weight, int device, rmd_volume_t **out);
int rmd_volume_destroy(rmd_volume_t *v);
/* Run this volume's work on a caller-owned cudaStream_t (NULL = its own). */
int rmd_volume_set_stream(rmd_volume_t *v, void *cuda_stream);
/* Every voxel back to (0, 0), asynchronously on the volume's stream. */
int rmd_volume_reset(rmd_volume_t *v);
int rmd_volume_sync(rmd_volume_t *v);
/* Any output pointer may be NULL. */
int rmd_volume_size(rmd_volume_t *v, int *nx, int *ny, int *nz, float *voxel_size, float origin[3]);

/* Integrate one keyframe: every voxel in front of the camera whose projection
 * u = floor(fx x / z + cx + 0.5), v = floor(fy y / z + cy + 0.5) lies in the
 * image, on a CONVERGED pixel with a finite depth d > 0, and not more than tau
 * behind the surface (sdf = d - |p| >= -tau, p in camera coordinates), gets
 * the observation o = min(1, sdf / tau):  w' = w + 1,  t' = (t w + o) / w',
 * stored as (t', min(w', max_weight)).  Voxels in front of the surface get
 * o = 1 (free space carves out earlier outliers); all others are untouched.
 *
 * The keyframe is s: its camera, the pose it was set with and its
 * convergence map.  Depth (distance along the ray) is the seeds' mu when
 * dev_depth is NULL, else a pitched device image of s's size (pitch in bytes,
 * >= width * 4 and a multiple of 4), e.g. the output of
 * rmd_denoiser_run_seeds_to_device.  Asynchronous on the volume's stream,
 * ordered on the device like rmd_seeds_propagate_prior with its source: the
 * integration waits for s's queued work and for a denoised image pending
 * against s, and a later update / set_reference / upload_state of s waits
 * for the integration.  RMD_ERR_INVALID_ARGUMENT: null handle, bad pitch,
 * volume and seeds on different devices.  RMD_ERR_NOT_INITIALISED: s has no
 * reference frame. */
int rmd_volume_integrate_seeds(rmd_volume_t *v, rmd_seeds_t *s, const float *dev_depth, size_t depth_pitch);
/* Same for any depth image already on the device, seen by the pinhole camera
 * (fx, fy, cx, cy) at T_curr_world (world -> camera).  dev_conv: int32
 * states (pitch in bytes), only CONVERGED pixels count; NULL = every pixel
 * with a finite positive depth counts.  Asynchronous on the volume's stream:
 * the images must be complete when it runs (produced on that stream or
 * synchronised).  RMD_ERR_INVALID_ARGUMENT: null pointer, size <= 0, pitch
 * smaller than a row or not a multiple of 4. */
int rmd_volume_integrate_depth(rmd_volume_t *v, int width, int height, float fx, float fy, float cx, float cy,
                               const float *T_curr_world, const float *dev_depth, size_t depth_pitch,
                               const int32_t *dev_conv, size_t conv_pitch);

/* The surface as points.  For each voxel a and each of its +x, +y, +z
 * neighbours b inside the grid: a point when both weights are > 0, both
 * |tsdf| < 1 and the signs differ (t_a > 0 >= t_b or t_a <= 0 < t_b), at
 * p_a + t_a / (t_a - t_b) * voxel_size along that axis, with
 * w = min(w_a, w_b).  4 floats (x, y, z, w) per point, ordered by voxel index,
 * then axis x, y, z.  *count is always the number of points; at most
 * `capacity` are written.  The host variant stages min(count, capacity)
 * points in device memory it keeps (grown on demand).  Synchronous. */
int rmd_volume_surface_points(rmd_volume_t *v, float *host_xyzw, size_t capacity, size_t *count);
/* Same into device memory (16-byte aligned). */
int rmd_volume_surface_points_device(rmd_volume_t *v, float *dev_xyzw, size_t capacity, size_t *count);

/* The surface as an indexed, watertight triangle mesh (marching cubes with a
 * generated case table, DESIGN.md 4.8).  The vertices ARE the surface points:
 * the same array, bit for bit, as rmd_volume_surface_points.  Cube (i, j, k),
 * i < nx-1, j < ny-1, k < nz-1, has corner c = dx + 2 dy + 4 dz at voxel
 * (i+dx, j+dy, k+dz); a corner is inside when tsdf <= 0.  A cube is meshed
 * only when its 8 corners have weight > 0 and every cube edge whose ends differ
 * in sign has |tsdf| < 1 at both ends; its triangles then use exactly the
 * surface points on its crossing edges.  Triangles are 3 int32 vertex indices,
 * ordered by cube index, then by the table; (b - a) x (c - a) points to the
 * tsdf > 0 side (free space, the cameras).  Two cubes sharing a face cut it
 * the same way (on a face with four crossings each inside corner is cut off),
 * so the mesh is closed except at unknown / truncated cubes and the grid's
 * outer faces.
 *
 * *n_vertices and *n_triangles are always written; at most vertex_capacity
 * vertices (4 floats x, y, z, w each) and tri_capacity triangles are written.
 * Triangles may reference vertices beyond vertex_capacity.  NULL buffers with
 * capacity 0 only count.  The host variant stages what it writes in device
 * memory it keeps (grown on demand); the mesh path also keeps 8 B of scratch
 * per vertex.  Synchronous.  RMD_ERR_INVALID_ARGUMENT: null handle or count
 * pointer, null buffer with capacity > 0; for the device variant also a vertex
 * buffer not 16-byte aligned or a triangle buffer not 4-byte aligned.
 * RMD_ERR_UNSUPPORTED: 2^31 or more vertices (int32 indices); both counts are
 * still written and nothing else is. */
int rmd_volume_mesh(rmd_volume_t *v, float *host_xyzw, size_t vertex_capacity, int32_t *host_tri,
                    size_t tri_capacity, size_t *n_vertices, size_t *n_triangles);
int rmd_volume_mesh_device(rmd_volume_t *v, float *dev_xyzw, size_t vertex_capacity, int32_t *dev_tri,
                           size_t tri_capacity, size_t *n_vertices, size_t *n_triangles);

/* Depth map of the fused surface seen by the pinhole camera (fx, fy, cx, cy)
 * at T_curr_world: the ray of pixel (x, y), normalize((x-cx)/fx, (y-cy)/fy,
 * 1) rotated into the world from the camera centre, is clipped to the box of
 * the voxel centres and sampled every voxel_size with trilinear
 * interpolation; a sample with a corner outside the grid or unknown is
 * unknown.  The first pair of consecutive known samples f_prev > 0 >= f gives
 * the distance along the ray  t_prev + s f_prev / (f_prev - f);  0 where there
 * is none.  dev_depth: pitched float image (pitch in bytes).  Asynchronous on
 * the volume's stream (rmd_volume_sync before another stream reads it). */
int rmd_volume_raycast(rmd_volume_t *v, int width, int height, float fx, float fy, float cx, float cy,
                       const float *T_curr_world, float *dev_depth, size_t depth_pitch);

/* Depth prior of a new keyframe from the fused model (DESIGN.md 4.8): s has
 * just had set_reference* and no update since.  Every non-BORDER pixel of s is
 * raycast as rmd_volume_raycast does with s's camera and the pose its
 * reference was set with; a hit d with min_depth <= d <= max_depth (s's)
 * becomes the seed (d, sigma_sq_frac * range^2 / 36, 10, 10), d bit-identical
 * to rmd_volume_raycast's.  Every other seed is left as it is, and the state
 * stays UPDATE: new frames still have to confirm the prior.  So after the
 * in-place propagation (rmd_seeds_set_prior_propagation) or
 * rmd_seeds_propagate_prior, the volume wins where it has a hit and the
 * splatted or uniform prior stays elsewhere.  A volume never integrated leaves
 * s as set_reference left it.
 *
 * Asynchronous, no host synchronisation: the rays run on s's stream after
 * everything already enqueued on the volume's stream (e.g. the
 * rmd_volume_integrate_seeds of the keyframe just left) and after work another
 * handle enqueued against s; a later integrate, reset or upload of the volume
 * waits for the rays.  RMD_ERR_INVALID_ARGUMENT: null handle, volume and seeds
 * on different devices, sigma_sq_frac outside (0, 1].  RMD_ERR_NOT_INITIALISED:
 * s has no reference or has been updated since it was set. */
int rmd_volume_prior_seeds(rmd_volume_t *v, rmd_seeds_t *s, float sigma_sq_frac);

/* Test / checkpoint hooks (like rmd_seeds_upload_state): nx * ny * nz floats
 * each, x fastest.  Synchronous. */
int rmd_volume_download(rmd_volume_t *v, float *host_tsdf, float *host_weight);
int rmd_volume_upload(rmd_volume_t *v, const float *host_tsdf, const float *host_weight);

/* Intensity channel (DESIGN.md 4.8): an opt-in second record per voxel,
 * (intensity, weight), that fuses the images the depth maps were seen in, so
 * that surface points, mesh vertices and raycast views can be shaded.  The
 * (tsdf, weight) records, surface points, mesh and raycast depth of a volume
 * are bit-identical with and without it.  Intensity is in the units of the
 * images fused (for seeds: the reference image, 8-bit * 1/255); -1 = none.
 *
 * rmd_volume_enable_intensity allocates the channel (8 B per voxel) and
 * zeroes it asynchronously on the volume's stream; a second call does
 * nothing.  rmd_volume_reset also clears it.  Returns cudaErrorMemoryAllocation
 * when it does not fit.  From then on rmd_volume_integrate_seeds also fuses
 * s's reference image (ordered like the depth it reads); plain
 * rmd_volume_integrate_depth leaves the channel untouched.
 *
 * Every intensity entry point below returns RMD_ERR_NOT_INITIALISED on a
 * volume without the channel and RMD_ERR_INVALID_ARGUMENT for a null handle or
 * pointer or a bad pitch (pitches in bytes, >= width * 4, a multiple of 4). */
int rmd_volume_enable_intensity(rmd_volume_t *v);
/* rmd_volume_integrate_depth, and then every updated voxel in the band
 * (sdf < tau, so -tau <= sdf < tau) whose pixel (x, y) -- the depth's -- has a
 * finite intensity I in dev_intensity (float, the depth's size) gets
 * wc' = wc + 1,  c' = (c wc + I) / wc',  stored as (c', min(wc', max_weight)).
 * Free space (o = 1) does not take the colour of what lies behind it.
 * Asynchronous on the volume's stream. */
int rmd_volume_integrate_depth_intensity(rmd_volume_t *v, int width, int height, float fx, float fy, float cx,
                                         float cy, const float *T_curr_world, const float *dev_depth,
                                         size_t depth_pitch, const int32_t *dev_conv, size_t conv_pitch,
                                         const float *dev_intensity, size_t intensity_pitch);
/* One float per surface point, in rmd_volume_surface_points' order and count
 * (and so per mesh vertex): with f = t_a / (t_a - t_b), the point's factor,
 * c_a + f (c_b - c_a) when both voxels' intensity weights are > 0, the
 * intensity of the one that is > 0, else -1.  Same count / capacity / staging
 * contract as rmd_volume_surface_points[_device] (device output 4-byte
 * aligned).  Synchronous. */
int rmd_volume_surface_intensity(rmd_volume_t *v, float *host_intensity, size_t capacity, size_t *count);
int rmd_volume_surface_intensity_device(rmd_volume_t *v, float *dev_intensity, size_t capacity, size_t *count);
/* rmd_volume_raycast (dev_depth bit-identical to it) and, per pixel, the
 * intensity at the hit t: grid coordinates of org + t dir as the march
 * computes them, trilinear interpolation in x, then y, then z of the 8
 * intensity records around it; -1 when one of them lies outside the grid or
 * has weight 0, and where there is no hit (depth 0).  Asynchronous on the
 * volume's stream. */
int rmd_volume_raycast_intensity(rmd_volume_t *v, int width, int height, float fx, float fy, float cx, float cy,
                                 const float *T_curr_world, float *dev_depth, size_t depth_pitch,
                                 float *dev_intensity, size_t intensity_pitch);
/* Test / checkpoint hooks of the channel, like rmd_volume_download / upload. */
int rmd_volume_download_intensity(rmd_volume_t *v, float *host_intensity, float *host_weight);
int rmd_volume_upload_intensity(rmd_volume_t *v, const float *host_intensity, const float *host_weight);

/* Surface normals (DESIGN.md 4.8), on volumes with or without the intensity
 * channel.  The gradient of a voxel v with tsdf t0 uses the tsdf records
 * only (unitless, per voxel): along each axis e, a neighbour v +- e is usable
 * when it lies inside the grid and has weight > 0, and the component is
 * (t+ - t-) * 0.5 when both are usable, t+ - t0 or t0 - t- when one is, else
 * 0.  A normal is g / len with len = sqrt((gx^2 + gy^2) + gz^2), (0, 0, 0)
 * when len is 0 or not finite; it points towards tsdf > 0 (free space, the
 * cameras), the side the mesh's (b - a) x (c - a) faces.
 *
 * One normal (nx, ny, nz, 0) per surface point / mesh vertex, in
 * rmd_volume_surface_points' order and count/capacity/staging contract: for
 * the point of voxel a with neighbour b and factor f = t_a / (t_a - t_b), the
 * gradients of a and b interpolated per component, g_a + f (g_b - g_a), then
 * normalised.  Device output 16-byte aligned.  Synchronous. */
int rmd_volume_surface_normals(rmd_volume_t *v, float *host_nxyz0, size_t capacity, size_t *count);
int rmd_volume_surface_normals_device(rmd_volume_t *v, float *dev_nxyz0, size_t capacity, size_t *count);
/* rmd_volume_raycast (dev_depth bit-identical) + a world-frame unit normal
 * per pixel, float4 (nx, ny, nz, 0): at a hit t, the grid coordinates of
 * org + t dir as the march computes them, the gradients of the 8 corners of
 * that cell interpolated trilinearly in x, then y, then z, normalised;
 * (0, 0, 0, 0) when a corner lies outside the grid or has weight 0, and where
 * there is no hit.  Along a cube edge this field is the vertex normals' linear
 * interpolation.  dev_normals 16-byte aligned, normals_pitch (bytes) >= 16 *
 * width and a multiple of 16.  RMD_ERR_INVALID_ARGUMENT: null handle or
 * pointer, bad size, pitch or alignment.  Asynchronous on the volume's
 * stream. */
int rmd_volume_raycast_normals(rmd_volume_t *v, int width, int height, float fx, float fy, float cx, float cy,
                               const float *T_curr_world, float *dev_depth, size_t depth_pitch,
                               float *dev_normals, size_t normals_pitch);

/* Moving volume (DESIGN.md 4.8): the grid keeps its size and follows the
 * camera by whole voxels, handing the surface that leaves it to the caller.
 *
 * rmd_volume_shift: afterwards voxel (i, j, k) holds what voxel
 * (i + dx, j + dy, k + dz) held before, or (0, 0) (unknown) where that voxel
 * lies outside the grid; the intensity channel moves the same way.  The
 * volume keeps the origin o0 it was created with and the total offset D
 * (64-bit): the origin is then o0 + (float)D * voxel_size per axis, rounded
 * once per operation, so it depends only on the total and never accumulates
 * rounding.  rmd_volume_size reports it.  d = (0, 0, 0) does nothing; when
 * |d| >= the dimension on any axis the grid is reset and the origin moves.
 * Otherwise a kernel gathers the records into a second array that is then
 * swapped in: a volume that has shifted keeps 2x its record memory (the
 * second arrays are allocated by the first shift that moves records and
 * freed by rmd_volume_destroy); one never shifted allocates nothing.
 * Asynchronous on the volume's stream: later work on it sees the shifted
 * grid, and work already enqueued keeps reading the records it was launched
 * with (the rays of rmd_volume_prior_seeds included: the volume's stream
 * waits for them, so the next shift cannot overwrite what they read).
 * download, upload and reset act on the current grid.  With the brick store
 * (rmd_volume_enable_store, below) the shift also keeps what leaves and
 * restores what re-enters, and synchronises the volume's stream once when it
 * meets a brick not yet stored.
 * RMD_ERR_INVALID_ARGUMENT: null handle or pointer, a total offset that
 * overflows 64 bits or an origin that would not be finite; the volume is then
 * unchanged. */
int rmd_volume_shift(rmd_volume_t *v, const int d[3]);
/* The spill of a shift by d, called BEFORE rmd_volume_shift(v, d): the shift
 * keeps the box K = [max(0, d), min(n, n + d)) per axis (pre-shift indices),
 * and a surface point of voxel a and its neighbour b = a + e_axis spills when
 * a or b lies outside K.  Every point of the current grid either spills or is
 * a point of the shifted grid.  Each call returns the subsequence of
 * rmd_volume_surface_points / _intensity / _normals of the current grid made
 * of the points that spill, in that order and bit for bit, with the same
 * count / capacity / staging contract (host output).  Synchronous.
 * RMD_ERR_INVALID_ARGUMENT: null handle, d or count, null buffer with
 * capacity > 0.  The intensity variant returns RMD_ERR_NOT_INITIALISED on a
 * volume without the channel. */
int rmd_volume_spill_points(rmd_volume_t *v, const int d[3], float *host_xyzw, size_t capacity, size_t *count);
int rmd_volume_spill_intensity(rmd_volume_t *v, const int d[3], float *host_intensity, size_t capacity,
                               size_t *count);
int rmd_volume_spill_normals(rmd_volume_t *v, const int d[3], float *host_nxyz0, size_t capacity, size_t *count);

/* The spill mesh of a shift by d, called BEFORE rmd_volume_shift(v, d)
 * (DESIGN.md 4.8): the part of rmd_volume_mesh that a shift by d drops, so
 * that the surface leaving a moving volume can be meshed and joined to the
 * mesh of what stays.
 *   A cube (lower corner c < n - 1 per axis) spills when it is meshed (the
 * mesh's rule) and at least one of its 8 corners lies outside K.  Every meshed
 * cube either spills or has all corners in K, and is then a cube of the
 * shifted grid with the same records, case and triangles.
 *   The vertices V_s are the surface points that spill (rmd_volume_spill_points'
 * rule) or lie on an edge of a spilling cube (the "seam" points, which also
 * stay in the grid), as the subsequence of rmd_volume_surface_points in its
 * order, bit for bit.  The triangles are those of the spilling cubes in
 * rmd_volume_mesh's order, as int32 indices into V_s.
 *   host_ids (may be NULL): per vertex 4 int64 (i + D0, j + D1, k + D2, axis),
 * where (i, j, k) is the point's voxel and D the volume's total offset
 * (rmd_volume_offset): an identity of the grid edge that survives shifts, by
 * which the chunks are welded (positions may differ by rounding after a
 * shift).  It has vertex_capacity entries.
 *   The mesh's count / capacity / staging contract: NULL buffers with capacity
 * 0 only count; RMD_ERR_UNSUPPORTED for 2^31 or more vertices.  The intensity
 * and normals variants return one value per vertex of V_s in its order, with
 * the spill's contract; the intensity variant returns RMD_ERR_NOT_INITIALISED
 * without the channel.  Synchronous.  Scratch: the mesh's buffers. */
int rmd_volume_spill_mesh(rmd_volume_t *v, const int d[3], float *host_xyzw, size_t vertex_capacity, int32_t *host_tri,
                          size_t tri_capacity, int64_t *host_ids, size_t *n_vertices, size_t *n_triangles);
int rmd_volume_spill_mesh_intensity(rmd_volume_t *v, const int d[3], float *host_intensity, size_t capacity,
                                    size_t *count);
int rmd_volume_spill_mesh_normals(rmd_volume_t *v, const int d[3], float *host_nxyz0, size_t capacity, size_t *count);
/* The ids (as rmd_volume_spill_mesh's) of rmd_volume_surface_points, and so of
 * rmd_volume_mesh's vertices, in their order: at most capacity, *count = the
 * number of points.  Synchronous. */
int rmd_volume_surface_ids(rmd_volume_t *v, int64_t *host_ids, size_t capacity, size_t *count);
/* The volume's total offset D in voxels: the sum of its shifts. */
int rmd_volume_offset(rmd_volume_t *v, int64_t D[3]);

/* Brick store (DESIGN.md 4.8): an opt-in sparse store in device memory that
 * keeps the voxels a moving volume leaves and gives them back when they
 * re-enter, so that the map -- the store plus the window -- loses nothing.
 *   A brick is 8 x 8 x 8 voxels of the unbounded grid: window voxel (i, j, k)
 * is voxel u = (i, j, k) + D (rmd_volume_offset), in brick floor(u / 8) per
 * axis.  A stored brick holds 512 (tsdf, weight) records, x fastest, and with
 * the intensity channel 512 (intensity, weight) records.
 *   On rmd_volume_shift(v, d), every brick with a voxel in the pre-shift
 * window outside the kept box K (rmd_volume_spill_points; empty when
 * |d| >= n) is visited: a stored brick gets all its leaving voxels written; a
 * brick not stored is stored when one of its leaving voxels has weight > 0 --
 * its leaving voxels written, its other voxels (0, 0) -- and skipped
 * otherwise.  Then every voxel that enters the window (its pre-shift source
 * lay outside the grid) takes its brick's stored records, or (0, 0) when the
 * brick is not stored.  So every voxel of the unbounded grid is in the window,
 * or holds its last value in the store, or is unknown, and shift(d) followed
 * by shift(-d) gives back the window bit for bit.  A stored brick stays stored
 * when its voxels are back in the window; its copies of them are stale and
 * never read.
 *   Integration, extraction, raycasts, the prior and the spills act on the
 * window as without the store.  rmd_volume_reset also empties the store (its
 * memory stays allocated until rmd_volume_destroy); download and upload act on
 * the window; rmd_volume_enable_intensity gives bricks already stored zeroed
 * colour records.
 *
 * rmd_volume_enable_store turns the store on (nothing is allocated until a
 * shift stores a brick); a second call does nothing.  From then on
 * rmd_volume_shift reads one flag per new candidate brick back to the host, so
 * it synchronises the volume's stream once when such a brick exists; the pool
 * grows by doubling.  A shift whose pool cannot grow returns
 * cudaErrorMemoryAllocation, and one whose total offset plus the grid size
 * overflows 64 bits RMD_ERR_INVALID_ARGUMENT; the volume (window, offset and
 * store) is then unchanged.  RMD_ERR_INVALID_ARGUMENT: null handle, or an
 * offset already that large.
 *
 * The other entry points return RMD_ERR_NOT_INITIALISED on a volume without
 * the store, and RMD_ERR_INVALID_ARGUMENT for a null handle or pointer. */
int rmd_volume_enable_store(rmd_volume_t *v);
/* The number of stored bricks and the bytes of device memory the store's
 * pool holds.  Either output may be NULL. */
int rmd_volume_store_info(rmd_volume_t *v, size_t *bricks, size_t *bytes);
/* The stored bricks in ascending (z, y, x) brick coordinate: per brick 3
 * int64 (bx, by, bz) to host_coords and 512 records, x fastest, to the record
 * arrays; a voxel inside the current window is returned as (0, 0), since the
 * window holds it.  *count = the number of bricks, of which min(count,
 * capacity) are written; NULL host_coords with capacity 0 only counts.  Any
 * record array may be NULL (not written); the intensity ones return
 * RMD_ERR_NOT_INITIALISED without the channel.  Synchronous. */
int rmd_volume_download_store(rmd_volume_t *v, int64_t *host_coords, float *host_tsdf, float *host_weight,
                              float *host_intensity, float *host_intensity_weight, size_t capacity, size_t *count);
/* Test / checkpoint hook (like rmd_volume_upload): replaces the store with
 * count bricks laid out as rmd_volume_download_store's.  Voxels inside the
 * window are ignored.  host_intensity and host_intensity_weight come together
 * or are both NULL (zeroed colour records); RMD_ERR_NOT_INITIALISED when given
 * without the channel.  RMD_ERR_INVALID_ARGUMENT: null arrays with count > 0,
 * a duplicate brick, a coordinate outside [-2^60, 2^60).  Synchronous. */
int rmd_volume_upload_store(rmd_volume_t *v, const int64_t *host_coords, const float *host_tsdf,
                            const float *host_weight, const float *host_intensity,
                            const float *host_intensity_weight, size_t count);

/* ---------------------------------------------------------- device image */

/* DeviceImage<T>(width,height) = cudaMallocPitch, device_image.cuh:37-50 */
int rmd_image_alloc(size_t width, size_t height, size_t elem_size,
                    void **dev_ptr, size_t *pitch_bytes);
int rmd_image_free(void *dev_ptr);
/* setDevData / getDevData / zero / operator=, device_image.cuh:93-171 */
int rmd_image_upload(void *dev_ptr, size_t pitch_bytes, const void *host_src,
                     size_t width, size_t height, size_t elem_size);
int rmd_image_download(const void *dev_ptr, size_t pitch_bytes, void *host_dst,
                       size_t width, size_t height, size_t elem_size);
int rmd_image_zero(void *dev_ptr, size_t pitch_bytes, size_t width,
                   size_t height, size_t elem_size);
int rmd_image_copy(void *dst, size_t dst_pitch, const void *src,
                   size_t src_pitch, size_t width, size_t height,
                   size_t elem_size);

#ifdef __cplusplus
}
#endif
#endif /* RMD_B200_H */
