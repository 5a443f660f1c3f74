// c_api.cu -- the C-ABI (include/rmd_b200.h): handles, host sequencing, copies.
//
// Host-side counterpart of rmd::SeedMatrix (src/seed_matrix.cu),
// rmd::DepthmapDenoiser (src/depthmap_denoiser.cu:143-229),
// rmd::ImageReducer (src/reduction.cu) and rmd::DeviceImage
// (include/rmd/device_image.cuh), re-designed: per-handle streams instead of
// the legacy default stream, a pinned upload ring with a copy stream so the
// H2D transfer of frame k+1 overlaps the kernel of frame k, one fused launch
// per frame and no device synchronisation inside update().  The TSDF volume's entry points are in volume_api.cu,
// except rmd_volume_integrate_seeds and rmd_volume_prior_seeds, which read the seeds' internals.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <chrono>
#include <mutex>
#include <new>
#include <string>

#include "denoiser.cuh"
#include "host_copy.h"
#include "ingest.cuh"
#include "point_cloud.cuh"
#include "prior.cuh"
#include "depth_filter.cuh"
#include "reduction.cuh"
#include "rmd_common.cuh"
#include "staged_maps.cuh"
#include "volume.cuh"

namespace rmdb
{

// ------------------------------------------------------------------ errors
static thread_local std::string t_last_error;

void set_last_error(const std::string &msg) { t_last_error = msg; }

int fail(int code, const char *what)
{
  t_last_error = what;
  return code;
}

int fail_cuda(cudaError_t err, const char *what)
{
  t_last_error = std::string(what) + ": " + cudaGetErrorName(err) + " (" +
                 cudaGetErrorString(err) + ")";
  cudaGetLastError();  // clear the sticky-less error state
  return (int)err;
}

// ---------------------------------------------------------------- geometry
Pose pose_inverse(const Pose &T)
{
  Pose r;
  const float *d = T.m;
  r.m[0] = d[0]; r.m[1] = d[4]; r.m[2] = d[8];
  r.m[4] = d[1]; r.m[5] = d[5]; r.m[6] = d[9];
  r.m[8] = d[2]; r.m[9] = d[6]; r.m[10] = d[10];
  r.m[3] = -d[0] * d[3] - d[4] * d[7] - d[8] * d[11];
  r.m[7] = -d[1] * d[3] - d[5] * d[7] - d[9] * d[11];
  r.m[11] = -d[2] * d[3] - d[6] * d[7] - d[10] * d[11];
  return r;
}

Pose pose_compose(const Pose &A, const Pose &B)
{
  Pose r;
  for(int row = 0; row < 3; ++row)
  {
    const float *a = A.m + 4 * row;
    for(int col = 0; col < 3; ++col)
      r.m[4 * row + col] = a[0] * B.m[col] + a[1] * B.m[4 + col] + a[2] * B.m[8 + col];
    r.m[4 * row + 3] = a[3] + a[0] * B.m[3] + a[1] * B.m[7] + a[2] * B.m[11];
  }
  return r;
}

static inline size_t round_up(size_t v, size_t m) { return (v + m - 1) / m * m; }

} // namespace rmdb

using namespace rmdb;

// ------------------------------------------------ host profile (debug)
namespace
{
double g_prof[8] = {0, 0, 0, 0, 0, 0, 0, 0};
const bool g_prof_on = (getenv("RMD_HOST_PROFILE") != NULL);

struct ProfScope
{
  int idx;
  std::chrono::steady_clock::time_point t0;
  explicit ProfScope(int i) : idx(i)
  {
    if(g_prof_on) t0 = std::chrono::steady_clock::now();
  }
  ~ProfScope()
  {
    if(g_prof_on)
      g_prof[idx] += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
  }
};
} // namespace

int rmd_debug_host_profile(double out[8], int reset)
{
  RMD_REQUIRE(out, "rmd_debug_host_profile: null argument");
  for(int i = 0; i < 8; ++i) out[i] = g_prof[i];
  if(reset)
    for(int i = 0; i < 8; ++i) g_prof[i] = 0.0;
  return 0;
}

// =========================================================== seed matrix


static const int kSlots = 3;
static const int kStatsSlots = 4, kStatsEvery = 8, kStatsLag = 16;

struct rmd_seeds
{
  int device;
  int width, height, patch;
  Camera cam;
  float one_pix_angle;

  cudaStream_t own_stream, stream, copy_stream;

  float4 *seed; int seed_stride;
  float2 *templ; int templ_stride;
  int *conv; size_t conv_pitch;
  float *ref; size_t ref_pitch;
  float *curr[kSlots]; size_t curr_pitch;
  uint8_t *curr_u8[kSlots]; size_t curr_u8_pitch;
  void *pinned[kSlots];
  cudaEvent_t copied[kSlots], consumed[kSlots];
  bool slot_used[kSlots];
  int next_slot;

  float2 *matches; size_t matches_pitch;
  float *planar[6]; size_t planar_pitch;   // mu, sigma_sq, a, b, sum_templ, denom
  float *dense_tmp;                        // width*height floats, uploads/downloads
  unsigned int *counters;                  // converged count of frame f in [f % 3] + [3] converged seeds of retired tiles

  // scene / algorithm parameters (src/seed_matrix.cu:96-104)
  float min_depth, max_depth, avg_depth, depth_range, sigma_sq_max;
  float eta_inlier, eta_outlier, epsilon;
  Pose T_world_ref;
  Pose T_ref_world;       // the pose given to set_reference (its inverse in floats would not be bit-exact)
  float dist_from_ref;
  bool has_reference;
  uint64_t frame_index;   // number of updates since set_reference
  bool trust_conv;

  bool record_matches;
  long long *timeline; size_t timeline_bytes;   // RMD_OPT_DEBUG_TIMELINE
  int variant;            // 0 staged, 1 direct
  int tex_frac_bits;

  uint64_t n_fused, n_total;
  bool timing;
  cudaEvent_t t0, t1;
  bool t_valid;

  StagedMaps *maps;
  // busy-tile splitting of the staged kernel (depth_filter_staged.cu)
  int n_tiles, cta_slots[2];    // resident CTAs of the staged kernel at 2 / 3 CTAs per SM
  int ctas_per_sm;             // RMD_OPT_TUNE_CTAS_PER_SM: 0 automatic, 2, 3
  unsigned long long *tile_keys;
  unsigned int *tile_arrivals;
  unsigned int *heavy_list[3], *light_list[3], *sparse_list[3];  // work lists of frame f in [f % 3] (written during frame f - 1)
  unsigned int *work_counts;   // 3 rotating slots of 8: {heavy, light, helpers, items, tiles listed, listers done, -, -}
  unsigned int *cursor;        // STAGED_CURSOR_WORDS: work cursors, CTAs out of work, error flag (staged_maps.cuh)
  unsigned int *chain_state;   // [n_tiles] tile_done + [1] list_ready (frame chaining, depth_filter_staged.cu)
  StagedMaps *chain_maps;      // STAGED_BATCH_MAX descriptor sets of a chained launch (allocated on first use)
  int chain_frames;            // frames per chained launch of rmd_seeds_update_device_batch (1 = one launch per frame)
  // seed-major mode (depth_filter_seeds.cu): entered once few seeds are still updated
  int mode;                    // 0: tile-organised kernel, 1: seed-major kernel
  unsigned int *seed_list[2];  // compact lists of the live seeds (ping-pong between launches)
  unsigned int *seed_ctl;      // 8 uints, see SeedModeBatch
  int seed_cur, seed_est;      // list in use; host-side upper bound of its length
  int seed_mode_pct;           // go seed-major when at most this percentage of the pixels is still updated (0 = never)
  // The host enqueues frames far ahead of the GPU, so the statistics that decide the switch are requested
  // every kStatsEvery frames into a small ring and READ WITH A LAG: the host looks at a request as soon as it
  // has completed, and waits for it once it is kStatsLag frames old (the GPU then still has that many frames
  // queued, so it never idles; the host merely stops running further ahead).
  unsigned int *host_stats;    // pinned, kStatsSlots x 8: a frame's work-list counters
  cudaEvent_t stats_ev[4]; bool stats_used[4]; uint64_t stats_frame[4];
  int stats_next; uint64_t stats_last_req;
  bool worklist_valid;         // false: rebuild (all tiles, image order) before the next staged launch
  bool last_staged;            // the last update ran the staged kernel (retired count applies)
  int tiles_x;
  int tune[12];                // split_max, split_min_items, split_items_per_cta, sparse_max_seeds, heavy_min_items, split_avg_pct, pdl, warp_tile_max_seeds, grid_ctas, (ctas_per_sm: own field), warp_tile_max_cands, run_chunks
  ParallelCopier *copier;   // host frame -> pinned ring (created on first host update)
  // lens undistortion of 8-bit frames (ingest.cuh); maps are null until init_undistortion_map
  short2 *undist_xy; uint16_t *undist_frac;
  int16_t *undist_host_xy; uint16_t *undist_host_frac;
  uint8_t *undist_tmp[2]; size_t undist_tmp_pitch;   // src / dst of rmd_seeds_undistort_u8
  cudaEvent_t fan_ev;   // rmd_seeds_update_many: frame ready (handles[0]) / update enqueued (the others)
  bool pinned_input;    // RMD_OPT_PINNED_INPUT
  uint8_t *ref_u8; size_t ref_u8_pitch;   // scratch of rmd_seeds_set_reference_u8 (not a ring slot)
  // Work another handle (the denoiser) enqueued on ITS stream against this handle's buffers: the
  // next operation on s->stream that touches them waits for ext_ev first.
  cudaEvent_t ext_ev; bool ext_pending;
  // point-cloud extraction (point_cloud.cuh), allocated on first use
  float4 *pc_points; unsigned int *pc_counts, *pc_total;
  // keyframe prior (prior.cuh): sigma^2 fraction of the in-place option (0 = off); z-buffer and event are
  // allocated on first use
  float prior_frac;
  unsigned int *prior_z; cudaEvent_t prior_ev;
};

namespace
{

// Ring slot i: device image, pinned staging buffer, events.
int ensure_slot(rmd_seeds *s, int i)
{
  if(s->curr[i]) return 0;
  const int w = s->width, h = s->height;
  RMD_CUDA_TRY(cudaMallocPitch(&s->curr[i], &s->curr_pitch, sizeof(float) * (size_t)w, h));
  RMD_CUDA_TRY(cudaHostAlloc(&s->pinned[i], sizeof(float) * (size_t)w * h, cudaHostAllocDefault));
  RMD_CUDA_TRY(cudaEventCreateWithFlags(&s->copied[i], cudaEventDisableTiming));
  RMD_CUDA_TRY(cudaEventCreateWithFlags(&s->consumed[i], cudaEventDisableTiming));
  return 0;
}

int seeds_alloc(rmd_seeds *s)
{
  const int w = s->width, h = s->height;
  RMD_CUDA_TRY(cudaStreamCreateWithFlags(&s->own_stream, cudaStreamNonBlocking));
  RMD_CUDA_TRY(cudaStreamCreateWithFlags(&s->copy_stream, cudaStreamNonBlocking));
  s->stream = s->own_stream;
  s->seed_stride = (int)round_up(w, 32);
  s->templ_stride = (int)round_up(w, 32);
  RMD_CUDA_TRY(cudaMalloc(&s->seed, sizeof(float4) * (size_t)s->seed_stride * h));
  RMD_CUDA_TRY(cudaMalloc(&s->templ, sizeof(float2) * (size_t)s->templ_stride * h));
  RMD_CUDA_TRY(cudaMallocPitch(&s->conv, &s->conv_pitch, sizeof(int) * (size_t)w, h));
  RMD_CUDA_TRY(cudaMallocPitch(&s->ref, &s->ref_pitch, sizeof(float) * (size_t)w, h));
  for(int i = 0; i < kSlots; ++i)
  {
    const int rc = ensure_slot(s, i);
    if(rc) return rc;
  }
  RMD_CUDA_TRY(cudaEventCreateWithFlags(&s->ext_ev, cudaEventDisableTiming));
  RMD_CUDA_TRY(cudaMalloc(&s->counters, 4 * sizeof(unsigned int)));
  RMD_CUDA_TRY(cudaMemset(s->counters, 0, 4 * sizeof(unsigned int)));
  RMD_CUDA_TRY(cudaMemset2D(s->conv, s->conv_pitch, 0, sizeof(int) * (size_t)w, h));
  {
    s->n_tiles = ((w + staged::TILE_W - 1) / staged::TILE_W) * ((h + staged::TILE_H - 1) / staged::TILE_H);
    // resident CTAs of the staged kernel = its persistent grid (SMs x occupancy: 3 per SM for 5x5, 2 for 7x7)
    for(int mb = 2; mb <= 3; ++mb)
    {
      s->cta_slots[mb - 2] = staged_cta_slots(s->patch, mb);
      if(s->cta_slots[mb - 2] <= 0)
      {
        int sms = 132;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, s->device);
        s->cta_slots[mb - 2] = sms * (s->patch <= 5 ? mb : 2);
        cudaGetLastError();
      }
    }
    RMD_CUDA_TRY(cudaMalloc(&s->tile_keys, sizeof(unsigned long long) * (size_t)s->n_tiles * staged::NPIX));
    RMD_CUDA_TRY(cudaMalloc(&s->tile_arrivals, sizeof(unsigned int) * (size_t)s->n_tiles));
    s->tiles_x = (w + staged::TILE_W - 1) / staged::TILE_W;
    for(int i = 0; i < 3; ++i)
    {
      RMD_CUDA_TRY(cudaMalloc(&s->heavy_list[i], sizeof(unsigned int) * (size_t)(s->n_tiles + staged::HELPER_CAP)));
      RMD_CUDA_TRY(cudaMalloc(&s->light_list[i], sizeof(unsigned int) * (size_t)s->n_tiles));
      RMD_CUDA_TRY(cudaMalloc(&s->sparse_list[i], sizeof(unsigned int) * (size_t)s->n_tiles));
    }
    RMD_CUDA_TRY(cudaMalloc(&s->work_counts, 24 * sizeof(unsigned int)));
    RMD_CUDA_TRY(cudaMalloc(&s->cursor, STAGED_CURSOR_WORDS * sizeof(unsigned int)));
    RMD_CUDA_TRY(cudaMemset(s->cursor, 0, STAGED_CURSOR_WORDS * sizeof(unsigned int)));
    for(int i = 0; i < 2; ++i)
      RMD_CUDA_TRY(cudaMalloc(&s->seed_list[i], sizeof(unsigned int) * (size_t)w * h));
    RMD_CUDA_TRY(cudaMalloc(&s->seed_ctl, 8 * sizeof(unsigned int)));
    RMD_CUDA_TRY(cudaMemset(s->seed_ctl, 0, 8 * sizeof(unsigned int)));
    RMD_CUDA_TRY(cudaHostAlloc(&s->host_stats, kStatsSlots * 8 * sizeof(unsigned int), cudaHostAllocDefault));
    for(int i = 0; i < kStatsSlots; ++i)
      RMD_CUDA_TRY(cudaEventCreateWithFlags(&s->stats_ev[i], cudaEventDisableTiming));
    RMD_CUDA_TRY(cudaMalloc(&s->chain_state, sizeof(unsigned int) * (size_t)(s->n_tiles + 1)));
    RMD_CUDA_TRY(cudaMemset(s->chain_state, 0, sizeof(unsigned int) * (size_t)(s->n_tiles + 1)));
  }
  RMD_CUDA_TRY(cudaEventCreate(&s->t0));
  RMD_CUDA_TRY(cudaEventCreate(&s->t1));
  return 0;
}

void seeds_free(rmd_seeds *s)
{
  cudaDeviceSynchronize();
  if(s->own_stream) cudaStreamDestroy(s->own_stream);
  if(s->copy_stream) cudaStreamDestroy(s->copy_stream);
  cudaFree(s->seed); cudaFree(s->templ); cudaFree(s->conv); cudaFree(s->ref);
  for(int i = 0; i < kSlots; ++i)
  {
    cudaFree(s->curr[i]);
    cudaFree(s->curr_u8[i]);
    if(s->pinned[i]) cudaFreeHost(s->pinned[i]);
    if(s->copied[i]) cudaEventDestroy(s->copied[i]);
    if(s->consumed[i]) cudaEventDestroy(s->consumed[i]);
  }
  cudaFree(s->matches);
  for(int i = 0; i < 6; ++i) cudaFree(s->planar[i]);
  cudaFree(s->dense_tmp);
  cudaFree(s->counters);
  cudaFree(s->timeline);
  cudaFree(s->tile_keys); cudaFree(s->tile_arrivals);
  for(int i = 0; i < 3; ++i) { cudaFree(s->heavy_list[i]); cudaFree(s->light_list[i]); cudaFree(s->sparse_list[i]); }
  cudaFree(s->work_counts);
  cudaFree(s->cursor);
  cudaFree(s->chain_state);
  delete[] s->chain_maps;
  cudaFree(s->seed_list[0]); cudaFree(s->seed_list[1]); cudaFree(s->seed_ctl);
  if(s->host_stats) cudaFreeHost(s->host_stats);
  for(int i = 0; i < kStatsSlots; ++i)
    if(s->stats_ev[i]) cudaEventDestroy(s->stats_ev[i]);
  if(s->t0) cudaEventDestroy(s->t0);
  if(s->t1) cudaEventDestroy(s->t1);
  delete s->maps;
  delete s->copier;
  cudaFree(s->pc_points); cudaFree(s->pc_counts); cudaFree(s->pc_total);
  cudaFree(s->prior_z);
  if(s->prior_ev) cudaEventDestroy(s->prior_ev);
  if(s->fan_ev) cudaEventDestroy(s->fan_ev);
  if(s->ext_ev) cudaEventDestroy(s->ext_ev);
  cudaFree(s->ref_u8);
  cudaFree(s->undist_xy); cudaFree(s->undist_frac); cudaFree(s->undist_tmp[0]); cudaFree(s->undist_tmp[1]);
  free(s->undist_host_xy); free(s->undist_host_frac);
  cudaGetLastError();
}

int ensure_dense_tmp(rmd_seeds *s)
{
  if(!s->dense_tmp)
    RMD_CUDA_TRY(cudaMalloc(&s->dense_tmp, sizeof(float) * 2 * (size_t)s->width * s->height));
  return 0;
}

int ensure_matches(rmd_seeds *s)
{
  if(!s->matches)
  {
    RMD_CUDA_TRY(cudaMallocPitch(&s->matches, &s->matches_pitch, sizeof(float2) * (size_t)s->width,
                                 s->height));
    RMD_CUDA_TRY(cudaMemset2DAsync(s->matches, s->matches_pitch, 0,
                                   sizeof(float2) * (size_t)s->width, s->height, s->stream));
  }
  return 0;
}

// Orders s->stream after whatever another handle enqueued against this handle's buffers
// (rmd_denoiser_run_seeds*: reads s->seed, writes the depth image rmd_seeds_point_cloud reads).
int wait_external(rmd_seeds *s)
{
  if(s->ext_pending)
  {
    RMD_CUDA_TRY(cudaStreamWaitEvent(s->stream, s->ext_ev, 0));
    s->ext_pending = false;
  }
  return 0;
}

// Keyframe prior, step 1 (prior.cuh), on dst->stream: dst's z-buffer <- src's CONVERGED seeds seen from the
// new reference pose T_curr_world of dst, within [min_depth, max_depth].  src's seeds, convergence map and
// T_world_ref are read as they are now (src == dst: the keyframe being left).
int prior_splat(rmd_seeds *dst, const rmd_seeds *src, const float *T_curr_world, float min_depth, float max_depth)
{
  const size_t n = (size_t)dst->width * dst->height;
  if(!dst->prior_z)
    RMD_CUDA_TRY(cudaMalloc(&dst->prior_z, sizeof(unsigned int) * n));
  RMD_CUDA_TRY(cudaMemsetAsync(dst->prior_z, 0xFF, sizeof(unsigned int) * n, dst->stream));
  PriorSplatParams P;
  memset(&P, 0, sizeof(P));
  P.src_width = src->width; P.src_height = src->height;
  P.conv = src->conv; P.conv_stride = (int)(src->conv_pitch / sizeof(int));
  P.seed = src->seed; P.seed_stride = src->seed_stride;
  P.src_cam = src->cam;
  P.T_world_ref = src->T_world_ref;
  P.dst_width = dst->width; P.dst_height = dst->height;
  P.dst_cam = dst->cam;
  P.T_curr_world = pose_from(T_curr_world);
  P.min_depth = min_depth; P.max_depth = max_depth;
  P.zbuf = dst->prior_z;
  RMD_CUDA_TRY(launch_prior_splat(P, dst->stream));
  dst->n_total += 1;
  return 0;
}

// Keyframe prior, step 2, after dst's seed initialisation: the splatted depths become the prior.
int prior_apply(rmd_seeds *dst, float frac)
{
  PriorApplyParams P;
  memset(&P, 0, sizeof(P));
  P.width = dst->width; P.height = dst->height;
  P.zbuf = dst->prior_z;
  P.conv = dst->conv; P.conv_stride = (int)(dst->conv_pitch / sizeof(int));
  P.seed = dst->seed; P.seed_stride = dst->seed_stride;
  P.sigma_sq = frac * dst->sigma_sq_max;
  RMD_CUDA_TRY(launch_prior_apply(P, dst->stream));
  dst->n_total += 1;
  return 0;
}

// Run the seed-initialisation kernel on the reference image now in s->ref.
int finish_set_reference(rmd_seeds *s, const float *T_curr_world, float min_depth, float max_depth)
{
  {
    const int rc = wait_external(s);
    if(rc) return rc;
  }
  // in-place prior: the keyframe being left is splatted before the initialisation overwrites its seeds and
  // T_world_ref
  const bool propagate = s->prior_frac > 0.0f && s->has_reference;
  if(propagate)
  {
    const int rc = prior_splat(s, s, T_curr_world, min_depth, max_depth);
    if(rc) return rc;
  }
  s->min_depth = min_depth;
  s->max_depth = max_depth;
  s->avg_depth = (min_depth + max_depth) / 2.0f;
  s->depth_range = max_depth - min_depth;
  s->sigma_sq_max = s->depth_range * s->depth_range / 36.0f;
  s->eta_inlier = 0.7f;
  s->eta_outlier = 0.05f;
  s->epsilon = s->depth_range / 1000.0f;
  s->T_world_ref = pose_inverse(pose_from(T_curr_world));
  s->T_ref_world = pose_from(T_curr_world);

  InitParams ip;
  ip.width = s->width; ip.height = s->height;
  ip.ref = s->ref; ip.ref_stride = (int)(s->ref_pitch / sizeof(float));
  ip.seed = s->seed; ip.seed_stride = s->seed_stride;
  ip.templ = s->templ; ip.templ_stride = s->templ_stride;
  ip.conv = s->conv; ip.conv_stride = (int)(s->conv_pitch / sizeof(int));
  ip.avg_depth = s->avg_depth; ip.sigma_sq_max = s->sigma_sq_max;
  RMD_CUDA_TRY(launch_seed_init(ip, s->patch, s->stream));
  if(propagate)
  {
    const int rc = prior_apply(s, s->prior_frac);
    if(rc) return rc;
  }
  RMD_CUDA_TRY(cudaMemsetAsync(s->counters, 0, 4 * sizeof(unsigned int), s->stream));
  // the first staged frame of a keyframe starts from the full work list; keys hold "no match"
  s->worklist_valid = false;
  RMD_CUDA_TRY(cudaMemsetAsync(s->tile_arrivals, 0, sizeof(unsigned int) * (size_t)s->n_tiles, s->stream));
  RMD_CUDA_TRY(cudaMemsetAsync(s->cursor, 0, STAGED_CURSOR_WORDS * sizeof(unsigned int), s->stream));
  RMD_CUDA_TRY(cudaMemsetAsync(s->chain_state, 0, sizeof(unsigned int) * (size_t)(s->n_tiles + 1), s->stream));   // frame numbering restarts
  RMD_CUDA_TRY(launch_fill_u64(s->tile_keys, (size_t)s->n_tiles * staged::NPIX, 0x407FFFFF00000000ull, s->stream));
  s->n_total += 1;
  s->n_total += 1;
  s->has_reference = true;
  s->mode = 0;            // a new keyframe starts tile-organised; pending statistics belong to the old one
  for(int i = 0; i < kStatsSlots; ++i) s->stats_used[i] = false;
  s->stats_last_req = 0;
  s->frame_index = 0;
  s->trust_conv = true;
  s->dist_from_ref = 0.0f;
  return 0;
}

// Resident CTAs per SM of the 5x5 staged kernel for the next launch (RMD_OPT_TUNE_CTAS_PER_SM).  Automatic = the
// 128-register build (2 per SM): no spills, room for the two-candidates-at-once NCC; the 80-register build
// (3 per SM) stays selectable for A/B runs (tools/tune_probe.py).
int staged_ctas_per_sm(const rmd_seeds *s)
{
  if(s->patch > 5) return 2;
  return s->ctas_per_sm == 3 ? 3 : 2;
}

// Host side of one update: pose chain, parameter block, TMA descriptors and -- when the keyframe's work
// list is not valid (first frame, state upload, variant switch) -- its rebuild on the handle's stream.
// Nothing is launched for the frame itself; `P` is ready for launch_depth_filter_*.
int prepare_update(rmd_seeds *s, const float *curr, size_t curr_pitch, const float *T_curr_world, FilterParams &P,
                   StagedMaps *maps = NULL)
{
  const Pose T_curr_ref = pose_compose(pose_from(T_curr_world), s->T_world_ref);  // seed_matrix.cu:124
  const float tx = T_curr_ref.m[3], ty = T_curr_ref.m[7], tz = T_curr_ref.m[11];
  s->dist_from_ref = sqrtf(tx * tx + ty * ty + tz * tz);                          // :125

  {
    const int rc = wait_external(s);
    if(rc) return rc;
  }
  s->frame_index += 1;
  memset(&P, 0, sizeof(P));
  P.width = s->width; P.height = s->height;
  P.seed = s->seed; P.seed_stride = s->seed_stride;
  P.templ = s->templ; P.templ_stride = s->templ_stride;
  P.conv = s->conv; P.conv_stride = (int)(s->conv_pitch / sizeof(int));
  P.ref = s->ref; P.ref_stride = (int)(s->ref_pitch / sizeof(float));
  P.curr = curr; P.curr_stride = (int)(curr_pitch / sizeof(float));
  if(s->record_matches)
  {
    const int rc = ensure_matches(s);
    if(rc) return rc;
    P.matches = s->matches; P.match_stride = (int)(s->matches_pitch / sizeof(float2));
  }
  P.cam = s->cam;
  P.T_curr_ref = T_curr_ref;
  P.T_ref_curr = pose_inverse(T_curr_ref);  // seed_matrix.cu:155
  P.eta_inlier = s->eta_inlier; P.eta_outlier = s->eta_outlier; P.epsilon = s->epsilon;
  P.depth_range = s->depth_range;
  P.one_pix_angle = s->one_pix_angle;
  P.tex_quant = s->tex_frac_bits > 0 ? (float)(1 << s->tex_frac_bits) : 0.0f;
  P.trust_conv = s->trust_conv ? 1 : 0;
  P.converged_now = s->counters + (s->frame_index % 3);
  P.converged_next = s->counters + ((s->frame_index + 1) % 3);
  P.timeline = s->timeline;
  {
    const uint64_t f = s->frame_index;
    P.split_max = s->tune[0]; P.split_min_items = s->tune[1]; P.split_items_per_cta = s->tune[2];
    P.sparse_max_seeds = s->tune[3];
    P.ctas_per_sm = staged_ctas_per_sm(s);
    P.cta_slots = s->cta_slots[P.ctas_per_sm - 2];
    P.tile_keys = s->tile_keys;
    P.tile_arrivals = s->tile_arrivals;
    P.n_tiles = s->n_tiles; P.tiles_x = s->tiles_x; P.helper_cap = staged::HELPER_CAP;
    P.heavy_min_items = s->tune[4]; P.split_avg_pct = s->tune[5]; P.pdl = s->tune[6];
    P.heavy_cur = s->heavy_list[f % 3]; P.heavy_next = s->heavy_list[(f + 1) % 3];
    P.light_cur = s->light_list[f % 3]; P.light_next = s->light_list[(f + 1) % 3];
    P.sparse_cur = s->sparse_list[f % 3]; P.sparse_next = s->sparse_list[(f + 1) % 3];
    P.warp_tile_max_seeds = s->tune[7];
    P.warp_tile_max_cands = s->tune[10];
    P.grid_ctas = s->tune[8];
    P.run_chunks = s->tune[11];
    P.counts_cur = s->work_counts + 8 * (f % 3);
    P.counts_next = s->work_counts + 8 * ((f + 1) % 3);
    P.counts_zero = s->work_counts + 8 * ((f + 2) % 3);
    P.retired_converged = s->counters + 3;
    P.frame_no = (unsigned int)f;
    P.tile_done = s->chain_state;
    P.list_ready = s->chain_state + s->n_tiles;
  }
  if(s->variant == 0 && s->mode == 0)
  {
    if(!s->maps) s->maps = new StagedMaps();
    {
      ProfScope prof(3);
      const int rc = (maps ? maps : s->maps)->encode(P, s->patch);
      if(rc) return rc;
    }
    if(!s->worklist_valid)
    {
      // every tile once, in image order, no helpers; nothing retired yet
      RMD_CUDA_TRY(cudaMemsetAsync(s->work_counts, 0, 24 * sizeof(unsigned int), s->stream));
      RMD_CUDA_TRY(cudaMemsetAsync(s->counters + 3, 0, sizeof(unsigned int), s->stream));
      RMD_CUDA_TRY(launch_worklist_init(const_cast<unsigned int*>(P.light_cur),
                                        const_cast<unsigned int*>(P.counts_cur), s->n_tiles, s->stream));
      s->worklist_valid = true;
    }
    if(s->timeline)
      RMD_CUDA_TRY(cudaMemsetAsync(s->timeline, 0, s->timeline_bytes, s->stream));
  }
  return 0;
}

// Book-keeping after the frame's kernel has been enqueued (by this handle or by a batched launch).
void finish_update(rmd_seeds *s)
{
  s->last_staged = (s->variant == 0);
  if(s->variant != 0)
    s->worklist_valid = false;   // the direct kernel does not maintain the staged kernel's work list
  s->n_fused += 1;
  s->n_total += 1;
  s->trust_conv = true;
}

// Seed-major mode is only for the staged variant without per-tile debugging / per-launch timing.
bool seed_mode_allowed(const rmd_seeds *s)
{
  return s->variant == 0 && s->seed_mode_pct > 0 && !s->timeline && !s->timing;
}

// Tile mode, before a frame: has the share of seeds that are still updated (counted by the kernel two or
// three frames ago and copied back asynchronously -- no stall) dropped below the threshold?  Then build the
// compact list of live seeds from the convergence map and continue seed-major (depth_filter_seeds.cu).
int maybe_enter_seed_mode(rmd_seeds *s)
{
  if(s->mode != 0 || !seed_mode_allowed(s))
    return 0;
  for(int n = 0; n < kStatsSlots; ++n)
  {
    const int slot = (s->stats_next + n) % kStatsSlots;    // oldest request first
    if(!s->stats_used[slot])
      continue;
    bool done = (cudaEventQuery(s->stats_ev[slot]) == cudaSuccess);
    if(!done)
    {
      cudaGetLastError();
      if(s->frame_index - s->stats_frame[slot] < (uint64_t)kStatsLag)
        break;                                              // younger requests are not done either
      RMD_CUDA_TRY(cudaEventSynchronize(s->stats_ev[slot]));
      done = true;
    }
    s->stats_used[slot] = false;
    const unsigned int active = s->host_stats[8 * slot + 7];
    const size_t pixels = (size_t)s->width * s->height;
    if((size_t)active * 100 > pixels * (size_t)s->seed_mode_pct)
      continue;
    for(int i = 0; i < kStatsSlots; ++i) s->stats_used[i] = false;
    RMD_CUDA_TRY(cudaMemsetAsync(s->seed_ctl, 0, 8 * sizeof(unsigned int), s->stream));
    RMD_CUDA_TRY(launch_seed_list_build(s->conv, (int)(s->conv_pitch / sizeof(int)), s->width, s->height,
                                        s->seed_list[0], s->seed_ctl, s->stream));
    s->n_total += 1;
    s->seed_cur = 0;
    s->seed_est = (int)active;    // the live set only shrinks: an upper bound from now on
    s->mode = 1;
    s->worklist_valid = false;    // the tile work list is not maintained while seed-major
    return 0;
  }
  return 0;
}

// Leave seed-major mode (state upload, variant / debugging options): the tile work list is rebuilt.
void leave_seed_mode(rmd_seeds *s)
{
  if(s->mode == 1)
  {
    s->mode = 0;
    s->worklist_valid = false;
  }
  for(int i = 0; i < kStatsSlots; ++i) s->stats_used[i] = false;
  s->stats_last_req = 0;
}

// Tile mode, after a frame's launch: ask for its statistics (asynchronously; one request in flight).
int request_stats(rmd_seeds *s, const FilterParams &P, cudaStream_t stream)
{
  if(s->mode != 0 || !seed_mode_allowed(s))
    return 0;
  if(s->stats_last_req != 0 && s->frame_index - s->stats_last_req < (uint64_t)kStatsEvery)
    return 0;
  const int slot = s->stats_next;      // (an unread request of kStatsSlots requests ago is simply superseded)
  RMD_CUDA_TRY(cudaMemcpyAsync(s->host_stats + 8 * slot, P.counts_next, 8 * sizeof(unsigned int), cudaMemcpyDeviceToHost,
                               stream));
  RMD_CUDA_TRY(cudaEventRecord(s->stats_ev[slot], stream));
  s->stats_used[slot] = true;
  s->stats_frame[slot] = s->frame_index;
  s->stats_next = (slot + 1) % kStatsSlots;
  s->stats_last_req = s->frame_index;
  return 0;
}

// One seed-major launch over n consecutive frames (device-resident: frames[k] / poses 12 * k).
int enqueue_seed_mode(rmd_seeds *s, const float *const *frames, size_t pitch, const float *T_curr_world, int n)
{
  SeedModeBatch B;
  memset(&B, 0, sizeof(B));
  for(int k = 0; k < n; ++k)
  {
    const int rc = prepare_update(s, frames[k], pitch, T_curr_world + 12 * k, B.p[k]);
    if(rc) return rc;
  }
  B.list_cur = s->seed_list[s->seed_cur];
  B.list_next = s->seed_list[s->seed_cur ^ 1];
  B.ctl = s->seed_ctl;
  B.cur = s->seed_cur;
  B.n_frames = n;
  RMD_CUDA_TRY(launch_depth_filter_seeds(B, s->seed_est, s->patch, s->stream));
  s->seed_cur ^= 1;
  for(int k = 0; k < n; ++k)
    finish_update(s);
  s->n_fused -= (uint64_t)(n - 1);
  s->n_total -= (uint64_t)(n - 1);
  return 0;
}

// Enqueue the fused depth-filter kernel for the frame at (curr, pitch).
int enqueue_update(rmd_seeds *s, const float *curr, size_t curr_pitch, const float *T_curr_world)
{
  if(s->mode == 1 && !seed_mode_allowed(s))
    leave_seed_mode(s);
  {
    const int rc = maybe_enter_seed_mode(s);
    if(rc) return rc;
  }
  if(s->mode == 1)
    return enqueue_seed_mode(s, &curr, curr_pitch, T_curr_world, 1);
  FilterParams P;
  const int rc = prepare_update(s, curr, curr_pitch, T_curr_world, P);
  if(rc) return rc;
  if(s->timing) RMD_CUDA_TRY(cudaEventRecord(s->t0, s->stream));
  if(s->variant == 0)
  {
    ProfScope prof_launch(4);
    const FilterParams *pp = &P;
    const StagedMaps *mm = s->maps;
    RMD_CUDA_TRY(launch_depth_filter_staged(&pp, &mm, 1, 0, s->cursor, s->patch, s->stream));
  }
  else
  {
    RMD_CUDA_TRY(launch_depth_filter_direct(P, s->patch, s->stream));
  }
  if(s->timing)
  {
    RMD_CUDA_TRY(cudaEventRecord(s->t1, s->stream));
    s->t_valid = true;
  }
  finish_update(s);
  return request_stats(s, P, s->stream);
}

// Enqueue n consecutive frames (device pointers, one pitch, poses 12 floats apiece).  Frame chaining: up to
// chain_frames (<= STAGED_BATCH_MAX) consecutive frames per launch of the staged kernel.  Every tile walks
// through the frames of a launch on its own (frame k+1 of a tile only needs frame k of that tile), so frames
// overlap on the GPU and the per-frame launch gap disappears; results are those of one launch per frame.
int enqueue_frames(rmd_seeds *s, const float *const *frames, size_t pitch_bytes, const float *T_curr_world, int n_frames)
{
  const int per_launch = (s->variant == 0 && !s->timeline && !s->timing) ? s->chain_frames : 1;
  for(int i = 0; i < n_frames; )
  {
    if(s->mode == 1 && !seed_mode_allowed(s))
      leave_seed_mode(s);
    {
      const int rc = maybe_enter_seed_mode(s);
      if(rc) return rc;
    }
    if(s->mode == 1)
    {
      // seed-major: every listed seed walks through up to SEED_FRAMES_MAX frames inside one launch
      const int m = (n_frames - i < SEED_FRAMES_MAX) ? n_frames - i : SEED_FRAMES_MAX;
      const int rc = enqueue_seed_mode(s, frames + i, pitch_bytes, T_curr_world + 12 * i, m);
      if(rc) return rc;
      i += m;
      continue;
    }
    const int m = (n_frames - i < per_launch) ? n_frames - i : per_launch;
    if(m <= 1)
    {
      const int rc = enqueue_update(s, frames[i], pitch_bytes, T_curr_world + 12 * i);
      if(rc) return rc;
      i += 1;
      continue;
    }
    if(!s->chain_maps) s->chain_maps = new StagedMaps[STAGED_BATCH_MAX];
    FilterParams P[STAGED_BATCH_MAX];
    const FilterParams *pp[STAGED_BATCH_MAX];
    const StagedMaps *mm[STAGED_BATCH_MAX];
    for(int k = 0; k < m; ++k)
    {
      const int rc = prepare_update(s, frames[i + k], pitch_bytes, T_curr_world + 12 * (i + k), P[k], &s->chain_maps[k]);
      if(rc) return rc;
      pp[k] = &P[k];
      mm[k] = &s->chain_maps[k];
    }
    {
      ProfScope prof_launch(4);
      RMD_CUDA_TRY(launch_depth_filter_staged(pp, mm, m, 1, s->cursor, s->patch, s->stream));
    }
    for(int k = 0; k < m; ++k)
      finish_update(s);
    s->n_fused -= (uint64_t)(m - 1);   // launch counters count launches, not frames
    s->n_total -= (uint64_t)(m - 1);
    {
      const int rc = request_stats(s, P[m - 1], s->stream);
      if(rc) return rc;
    }
    i += m;
  }
  return 0;
}

// rmd::Depthmap::inputImage (src/depthmap.cpp:95-106) for a frame already on the
// device: remap through the undistortion maps if the camera has them, then
// 8U -> 32F * (1/255), in one kernel on the compute stream.
cudaError_t u8_frame_to_float(rmd_seeds *s, const uint8_t *src, size_t src_pitch, float *dst, size_t dst_pitch,
                              cudaStream_t stream)
{
  if(s->undist_xy)
    return launch_undistort_u8(src, (int)src_pitch, s->undist_xy, s->undist_frac, dst,
                               (int)(dst_pitch / sizeof(float)), NULL, 0, s->width, s->height, stream);
  return launch_u8_to_float(src, (int)src_pitch, dst, (int)(dst_pitch / sizeof(float)), s->width, s->height,
                            stream);
}

// True when `p` lies in page-locked host memory the copy engine can read directly.
bool is_page_locked(const void *p)
{
  cudaPointerAttributes attr;
  if(cudaPointerGetAttributes(&attr, p) != cudaSuccess)
  {
    cudaGetLastError();
    return false;
  }
  return attr.type == cudaMemoryTypeHost;
}

// Stage a host frame (float or u8) into the next ring slot and make the
// compute stream wait for it.  Returns the slot.
int stage_host_frame(rmd_seeds *s, const void *host_img, size_t elem_size, int *slot_out)
{
  const int slot = s->next_slot;
  s->next_slot = (slot + 1) % kSlots;
  const size_t row_bytes = elem_size * (size_t)s->width;
  // RMD_OPT_PINNED_INPUT: the caller's buffer is page-locked and stays untouched until the next sync,
  // so the DMA reads it in place (no staging copy, no wait for the pinned ring slot)
  const bool direct = s->pinned_input && is_page_locked(host_img);
  const void *dma_src = host_img;
  if(!direct)
  {
    if(s->slot_used[slot])
    {
      ProfScope prof(0);
      RMD_CUDA_TRY(cudaEventSynchronize(s->copied[slot]));  // pinned buffer free again
    }
    if(!s->copier)
    {
      // helper threads for the ingest copy: RMD_COPY_THREADS, else an eighth of the
      // machine (3..15).  One core cannot stage a cold frame at the rate the GPU
      // consumes them; tools/copy_probe.cpp measures the scaling on a given host.
      const char *env = getenv("RMD_COPY_THREADS");
      int helpers = env ? atoi(env) : (int)(std::thread::hardware_concurrency() / 8) - 1;
      if(!env && helpers < 3) helpers = 3;
      if(helpers < 0) helpers = 0;
      if(helpers > 15) helpers = 15;
      s->copier = new ParallelCopier(helpers);
    }
    {
      ProfScope prof(1);
      s->copier->copy(s->pinned[slot], host_img, row_bytes * s->height);
    }
    dma_src = s->pinned[slot];
  }
  ProfScope prof_h2d(2);
  if(s->slot_used[slot])
    RMD_CUDA_TRY(cudaStreamWaitEvent(s->copy_stream, s->consumed[slot], 0));
  if(elem_size == sizeof(float))
  {
    RMD_CUDA_TRY(cudaMemcpy2DAsync(s->curr[slot], s->curr_pitch, dma_src, row_bytes,
                                   row_bytes, s->height, cudaMemcpyHostToDevice, s->copy_stream));
  }
  else
  {
    if(!s->curr_u8[slot])
      RMD_CUDA_TRY(cudaMallocPitch(&s->curr_u8[slot], &s->curr_u8_pitch, (size_t)s->width, s->height));
    RMD_CUDA_TRY(cudaMemcpy2DAsync(s->curr_u8[slot], s->curr_u8_pitch, dma_src, row_bytes,
                                   row_bytes, s->height, cudaMemcpyHostToDevice, s->copy_stream));
  }
  if(elem_size != sizeof(float))
  {
    // the ingest kernel follows the upload on the COPY stream: it overlaps the filter kernel of the frames
    // before it, and consecutive filter launches stay back to back on the compute stream
    RMD_CUDA_TRY(u8_frame_to_float(s, s->curr_u8[slot], s->curr_u8_pitch, s->curr[slot], s->curr_pitch, s->copy_stream));
    s->n_total += 1;
  }
  RMD_CUDA_TRY(cudaEventRecord(s->copied[slot], s->copy_stream));
  RMD_CUDA_TRY(cudaStreamWaitEvent(s->stream, s->copied[slot], 0));
  s->slot_used[slot] = true;
  *slot_out = slot;
  return 0;
}

bool is_seed_field(int f) { return f >= RMD_FIELD_MU && f <= RMD_FIELD_B; }
bool is_templ_field(int f) { return f == RMD_FIELD_SUM_TEMPL || f == RMD_FIELD_CONST_TEMPL_DENOM; }

// Export a float field into a dense or pitched planar device image.
int export_field(rmd_seeds *s, int field, float *dst, int dst_stride)
{
  if(is_seed_field(field))
  {
    RMD_CUDA_TRY(launch_export_plane(reinterpret_cast<const float*>(s->seed), s->seed_stride * 4, 4,
                                     field - RMD_FIELD_MU, dst, dst_stride, s->width, s->height,
                                     s->stream));
  }
  else if(is_templ_field(field))
  {
    RMD_CUDA_TRY(launch_export_plane(reinterpret_cast<const float*>(s->templ), s->templ_stride * 2, 2,
                                     field - RMD_FIELD_SUM_TEMPL, dst, dst_stride, s->width,
                                     s->height, s->stream));
  }
  else
  {
    return fail(RMD_ERR_INVALID_ARGUMENT, "export_field: not a float plane");
  }
  s->n_total += 1;
  return 0;
}

} // namespace

extern "C"
{

int rmd_abi_version(void) { return RMD_B200_ABI_VERSION; }

const char *rmd_last_error_string(void) { return t_last_error.c_str(); }

int rmd_device_count(int *count)
{
  RMD_REQUIRE(count, "rmd_device_count: null");
  *count = 0;
  RMD_CUDA_TRY(cudaGetDeviceCount(count));
  return 0;
}

int rmd_seeds_create(int width, int height, float fx, float fy, float cx, float cy,
                     int patch_side, int device, rmd_seeds_t **out)
{
  RMD_REQUIRE(out, "rmd_seeds_create: out is null");
  *out = NULL;
  RMD_REQUIRE(width > 0 && height > 0, "rmd_seeds_create: bad image size");
  RMD_REQUIRE(patch_side == 5 || patch_side == 7, "rmd_seeds_create: patch_side must be 5 or 7");
  RMD_REQUIRE(width > 2 * patch_side && height > 2 * patch_side,
              "rmd_seeds_create: image smaller than the border ring");
  if(device < 0) RMD_CUDA_TRY(cudaGetDevice(&device));
  DeviceGuard guard(device);
  int major = 0, minor = 0;
  RMD_CUDA_TRY(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device));
  RMD_CUDA_TRY(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device));
  // sm_90a code runs on compute capability 9.0 only (the "a" features do not carry forward)
  if(major != 9 || minor != 0)
    return fail(RMD_ERR_UNSUPPORTED, "rmd_seeds_create: this library is built for sm_90a (H100) only");

  rmd_seeds *s = new(std::nothrow) rmd_seeds();
  if(!s) return fail((int)cudaErrorMemoryAllocation, "rmd_seeds_create: host allocation failed");
  memset(s, 0, sizeof(*s));
  s->device = device;
  s->width = width; s->height = height; s->patch = patch_side;
  s->cam.fx = fx; s->cam.fy = fy; s->cam.cx = cx; s->cam.cy = cy;
  s->one_pix_angle = atan2f(1.0f, 2.0f * fx) * 2.0f;  // pinhole_camera.cuh:55-59
  s->tex_frac_bits = 8;
  s->tune[0] = staged::SPLIT_MAX; s->tune[1] = staged::SPLIT_MIN_ITEMS;
  s->tune[2] = staged::SPLIT_ITEMS_PER_CTA; s->tune[3] = staged::SPARSE_MAX_SEEDS;
  s->tune[4] = staged::HEAVY_MIN_ITEMS; s->tune[5] = staged::SPLIT_AVG_PCT; s->tune[6] = 1;
  s->tune[7] = staged::WARP_TILE_MAX_SEEDS;
  s->tune[10] = staged::WARP_TILE_MAX_CANDS;
  s->tune[11] = 0;
  s->variant = 0;   // staged (the fast path) unless RMD_OPT_KERNEL_VARIANT says otherwise
  s->chain_frames = 1;   // chaining is opt-in (include/rmd_b200.h, RMD_OPT_CHAIN_FRAMES)
  s->seed_mode_pct = 0;   // off by default: measured slower than the tile organisation on the bench workloads (DESIGN.md 4.1c)
  const int rc = seeds_alloc(s);
  if(rc)
  {
    seeds_free(s);
    delete s;
    return rc;
  }
  *out = s;
  return 0;
}

int rmd_seeds_destroy(rmd_seeds_t *s)
{
  if(!s) return 0;
  DeviceGuard guard(s->device);
  seeds_free(s);
  delete s;
  return 0;
}

int rmd_seeds_set_stream(rmd_seeds_t *s, void *cuda_stream)
{
  RMD_REQUIRE(s, "rmd_seeds_set_stream: null handle");
  DeviceGuard guard(s->device);
  RMD_CUDA_TRY(cudaStreamSynchronize(s->stream));
  s->stream = cuda_stream ? (cudaStream_t)cuda_stream : s->own_stream;
  return 0;
}

int rmd_seeds_get_stream(rmd_seeds_t *s, void **cuda_stream)
{
  RMD_REQUIRE(s && cuda_stream, "rmd_seeds_get_stream: null");
  *cuda_stream = (void*)s->stream;
  return 0;
}

int rmd_seeds_set_option(rmd_seeds_t *s, int option, int value)
{
  RMD_REQUIRE(s, "rmd_seeds_set_option: null handle");
  switch(option)
  {
  case RMD_OPT_RECORD_MATCHES: s->record_matches = (value != 0); return 0;
  case RMD_OPT_PINNED_INPUT: s->pinned_input = (value != 0); return 0;
  case RMD_OPT_CHAIN_FRAMES:
    RMD_REQUIRE(value >= 1 && value <= STAGED_BATCH_MAX, "RMD_OPT_CHAIN_FRAMES: 1..8");
    s->chain_frames = value;
    return 0;
  case RMD_OPT_KERNEL_VARIANT:
    RMD_REQUIRE(value == 0 || value == 1, "RMD_OPT_KERNEL_VARIANT: 0 (staged) or 1 (direct)");
    if(value != s->variant)
      leave_seed_mode(s);
    s->variant = value;
    return 0;
  case RMD_OPT_SEED_MODE_PCT:
    RMD_REQUIRE(value >= 0 && value <= 100, "RMD_OPT_SEED_MODE_PCT: 0..100");
    s->seed_mode_pct = value;
    if(value == 0)
      leave_seed_mode(s);
    return 0;
  case RMD_OPT_DEBUG_TIMELINE:
  {
    DeviceGuard guard(s->device);
    if(value && !s->timeline)
    {
      s->timeline_bytes = sizeof(long long) * 16 * (size_t)((s->width + 31) / 32) * (size_t)((s->height + 7) / 8);
      RMD_CUDA_TRY(cudaMalloc(&s->timeline, s->timeline_bytes));
      RMD_CUDA_TRY(cudaMemset(s->timeline, 0, s->timeline_bytes));
    }
    else if(!value && s->timeline)
    {
      RMD_CUDA_TRY(cudaStreamSynchronize(s->stream));
      cudaFree(s->timeline);
      s->timeline = NULL;
    }
    return 0;
  }
  case RMD_OPT_TUNE_SPLIT_MAX: case RMD_OPT_TUNE_SPLIT_MIN_ITEMS: case RMD_OPT_TUNE_SPLIT_ITEMS_PER_CTA:
  case RMD_OPT_TUNE_SPARSE_MAX_SEEDS: case RMD_OPT_TUNE_HEAVY_MIN_ITEMS: case RMD_OPT_TUNE_SPLIT_AVG_PCT: case RMD_OPT_TUNE_PDL:
  case RMD_OPT_TUNE_WARP_TILE_SEEDS: case RMD_OPT_TUNE_GRID_CTAS: case RMD_OPT_TUNE_WARP_TILE_CANDS:
    RMD_REQUIRE(value >= ((option == RMD_OPT_TUNE_SPARSE_MAX_SEEDS || option == RMD_OPT_TUNE_PDL ||
                           option == RMD_OPT_TUNE_WARP_TILE_SEEDS || option == RMD_OPT_TUNE_GRID_CTAS) ? 0 : 1) && value <= 65535, "tuning value out of range");
    // (only these ranges are covered by the bit-equality tests)
    RMD_REQUIRE(option != RMD_OPT_TUNE_WARP_TILE_SEEDS || value <= staged::WARP_TILE_MAX_SEEDS, "RMD_OPT_TUNE_WARP_TILE_SEEDS: 0..8");
    RMD_REQUIRE(option != RMD_OPT_TUNE_WARP_TILE_CANDS || value <= staged::WARP_TILE_MAX_CANDS, "RMD_OPT_TUNE_WARP_TILE_CANDS: 1..64");
    RMD_REQUIRE(option != RMD_OPT_TUNE_SPLIT_MAX || value <= 32, "RMD_OPT_TUNE_SPLIT_MAX: 1..32");
    s->tune[option - RMD_OPT_TUNE_SPLIT_MAX] = value;
    return 0;
  case RMD_OPT_TUNE_CTAS_PER_SM:
    RMD_REQUIRE(value == 0 || value == 2 || value == 3, "RMD_OPT_TUNE_CTAS_PER_SM: 0 (automatic), 2 or 3");
    s->ctas_per_sm = value;
    return 0;
  case RMD_OPT_TUNE_RUN_CHUNKS:
    RMD_REQUIRE(value >= 0 && value <= staged::MAX_CHUNKS, "RMD_OPT_TUNE_RUN_CHUNKS: 0 (automatic)..36");
    s->tune[11] = value;
    return 0;
  case RMD_OPT_TEX_FRAC_BITS:
    RMD_REQUIRE(value >= 0 && value <= 12, "RMD_OPT_TEX_FRAC_BITS: 0..12");
    s->tex_frac_bits = value;
    return 0;
  default: return fail(RMD_ERR_INVALID_ARGUMENT, "rmd_seeds_set_option: unknown option");
  }
}

int rmd_seeds_set_reference(rmd_seeds_t *s, const float *host_img, const float *T_curr_world,
                            float min_depth, float max_depth)
{
  RMD_REQUIRE(s && host_img && T_curr_world, "rmd_seeds_set_reference: null argument");
  DeviceGuard guard(s->device);
  {
    // s->ref may still be read by work another handle enqueued against s (rmd_volume_integrate_seeds)
    const int rc = wait_external(s);
    if(rc) return rc;
  }
  const size_t row = sizeof(float) * (size_t)s->width;
  // pageable source: returns once the data is staged, buffer reusable
  RMD_CUDA_TRY(cudaMemcpy2DAsync(s->ref, s->ref_pitch, host_img, row, row, s->height,
                                 cudaMemcpyHostToDevice, s->stream));
  return finish_set_reference(s, T_curr_world, min_depth, max_depth);
}

int rmd_seeds_set_reference_device(rmd_seeds_t *s, const float *dev_img, size_t pitch_bytes,
                                   const float *T_curr_world, float min_depth, float max_depth)
{
  RMD_REQUIRE(s && dev_img && T_curr_world, "rmd_seeds_set_reference_device: null argument");
  DeviceGuard guard(s->device);
  const size_t row = sizeof(float) * (size_t)s->width;
  RMD_REQUIRE(pitch_bytes >= row, "rmd_seeds_set_reference_device: pitch smaller than a row");
  {
    const int rc = wait_external(s);   // as rmd_seeds_set_reference
    if(rc) return rc;
  }
  RMD_CUDA_TRY(cudaMemcpy2DAsync(s->ref, s->ref_pitch, dev_img, pitch_bytes, row, s->height,
                                 cudaMemcpyDeviceToDevice, s->stream));
  return finish_set_reference(s, T_curr_world, min_depth, max_depth);
}

int rmd_seeds_set_reference_u8(rmd_seeds_t *s, const uint8_t *host_img, const float *T_curr_world,
                               float min_depth, float max_depth)
{
  RMD_REQUIRE(s && host_img && T_curr_world, "rmd_seeds_set_reference_u8: null argument");
  DeviceGuard guard(s->device);
  {
    const int rc = wait_external(s);   // as rmd_seeds_set_reference
    if(rc) return rc;
  }
  // own scratch image: the ring slots belong to frames that may still be in flight
  if(!s->ref_u8)
    RMD_CUDA_TRY(cudaMallocPitch(&s->ref_u8, &s->ref_u8_pitch, (size_t)s->width, s->height));
  RMD_CUDA_TRY(cudaMemcpy2DAsync(s->ref_u8, s->ref_u8_pitch, host_img, (size_t)s->width,
                                 (size_t)s->width, s->height, cudaMemcpyHostToDevice, s->stream));
  RMD_CUDA_TRY(u8_frame_to_float(s, s->ref_u8, s->ref_u8_pitch, s->ref, s->ref_pitch, s->stream));
  s->n_total += 1;
  return finish_set_reference(s, T_curr_world, min_depth, max_depth);
}

int rmd_seeds_set_prior_propagation(rmd_seeds_t *s, float sigma_sq_frac)
{
  RMD_REQUIRE(s, "rmd_seeds_set_prior_propagation: null handle");
  RMD_REQUIRE(sigma_sq_frac >= 0.0f && sigma_sq_frac <= 1.0f,
              "rmd_seeds_set_prior_propagation: sigma_sq_frac must be in [0, 1] (0 = off)");
  s->prior_frac = sigma_sq_frac;
  return 0;
}

int rmd_seeds_propagate_prior(rmd_seeds_t *dst, const rmd_seeds_t *src, float sigma_sq_frac)
{
  RMD_REQUIRE(dst && src, "rmd_seeds_propagate_prior: null handle");
  RMD_REQUIRE(sigma_sq_frac > 0.0f && sigma_sq_frac <= 1.0f, "rmd_seeds_propagate_prior: sigma_sq_frac must be in (0, 1]");
  RMD_REQUIRE(dst != src, "rmd_seeds_propagate_prior: src == dst (use rmd_seeds_set_prior_propagation)");
  RMD_REQUIRE(dst->device == src->device, "rmd_seeds_propagate_prior: handles on different devices");
  if(!dst->has_reference || dst->frame_index != 0)
    return fail(RMD_ERR_NOT_INITIALISED,
                "rmd_seeds_propagate_prior: dst needs a reference frame set since its last update");
  if(!src->has_reference)
    return fail(RMD_ERR_NOT_INITIALISED, "rmd_seeds_propagate_prior: src has no reference frame");
  DeviceGuard guard(dst->device);
  {
    const int rc = wait_external(dst);
    if(rc) return rc;
  }
  // The splat runs on dst's stream after everything that writes src's state: src's own stream, and work
  // another handle enqueued against src's buffers.
  rmd_seeds *s = const_cast<rmd_seeds*>(src);   // only its ordering book-keeping changes
  if(!dst->prior_ev)
    RMD_CUDA_TRY(cudaEventCreateWithFlags(&dst->prior_ev, cudaEventDisableTiming));
  RMD_CUDA_TRY(cudaEventRecord(dst->prior_ev, s->stream));
  RMD_CUDA_TRY(cudaStreamWaitEvent(dst->stream, dst->prior_ev, 0));
  if(s->ext_pending)
    RMD_CUDA_TRY(cudaStreamWaitEvent(dst->stream, s->ext_ev, 0));
  {
    const int rc = prior_splat(dst, s, dst->T_ref_world.m, dst->min_depth, dst->max_depth);
    if(rc) return rc;
  }
  // a later writer of src's seeds (update, set_reference, upload_state) waits for the splat's reads; the wait
  // above already covers any earlier external event, so re-recording ext_ev loses nothing
  RMD_CUDA_TRY(cudaEventRecord(s->ext_ev, dst->stream));
  s->ext_pending = true;
  return prior_apply(dst, sigma_sq_frac);
}

int rmd_seeds_update(rmd_seeds_t *s, const float *host_img, const float *T_curr_world)
{
  RMD_REQUIRE(s && host_img && T_curr_world, "rmd_seeds_update: null argument");
  if(!s->has_reference)
    return fail(RMD_ERR_NOT_INITIALISED, "rmd_seeds_update: set_reference has not been called");
  ProfScope prof(5);
  if(g_prof_on) g_prof[6] += 1.0;
  DeviceGuard guard(s->device);
  int slot = 0;
  const int rc = stage_host_frame(s, host_img, sizeof(float), &slot);
  if(rc) return rc;
  const int rc2 = enqueue_update(s, s->curr[slot], s->curr_pitch, T_curr_world);
  if(rc2) return rc2;
  RMD_CUDA_TRY(cudaEventRecord(s->consumed[slot], s->stream));
  return 0;
}

int rmd_seeds_update_u8(rmd_seeds_t *s, const uint8_t *host_img, const float *T_curr_world)
{
  RMD_REQUIRE(s && host_img && T_curr_world, "rmd_seeds_update_u8: null argument");
  if(!s->has_reference)
    return fail(RMD_ERR_NOT_INITIALISED, "rmd_seeds_update_u8: set_reference has not been called");
  ProfScope prof(5);
  if(g_prof_on) g_prof[6] += 1.0;
  DeviceGuard guard(s->device);
  int slot = 0;
  const int rc = stage_host_frame(s, host_img, sizeof(uint8_t), &slot);
  if(rc) return rc;
  const int rc2 = enqueue_update(s, s->curr[slot], s->curr_pitch, T_curr_world);
  if(rc2) return rc2;
  RMD_CUDA_TRY(cudaEventRecord(s->consumed[slot], s->stream));
  return 0;
}

namespace
{

int update_many(rmd_seeds_t *const *handles, int n, const void *host_img, size_t elem_size, const float *T_curr_world)
{
  RMD_REQUIRE(handles && n >= 1 && host_img && T_curr_world, "rmd_seeds_update_many: null argument");
  rmd_seeds *h0 = handles[0];
  for(int i = 0; i < n; ++i)
  {
    rmd_seeds *h = handles[i];
    RMD_REQUIRE(h, "rmd_seeds_update_many: null handle");
    if(!h->has_reference)
      return fail(RMD_ERR_NOT_INITIALISED, "rmd_seeds_update_many: a handle has no reference frame");
    RMD_REQUIRE(h->width == h0->width && h->height == h0->height && h->device == h0->device,
                "rmd_seeds_update_many: handles differ in image size or device");
    for(int j = 0; j < i; ++j)
      RMD_REQUIRE(handles[j] != h, "rmd_seeds_update_many: the same handle twice");
  }
  ProfScope prof(5);
  if(g_prof_on) g_prof[6] += 1.0;
  DeviceGuard guard(h0->device);
  for(int i = 0; i < n; ++i)
    if(!handles[i]->fan_ev)
      RMD_CUDA_TRY(cudaEventCreateWithFlags(&handles[i]->fan_ev, cudaEventDisableTiming));
  int slot = 0;
  const int rc = stage_host_frame(h0, host_img, elem_size, &slot);   // one pinned copy, one upload (+ ingest kernel)
  if(rc) return rc;
  // ONE launch for all staged keyframes of h0's patch size (groups of STAGED_BATCH_MAX): their work lists
  // are concatenated, so the dependent chains of different keyframes interleave on the GPU from the first
  // cycle.  Keyframes on the direct variant (or of another patch size) are enqueued one by one.  Everything
  // runs on h0's stream, where the frame lives.
  RMD_REQUIRE(n <= 64, "rmd_seeds_update_many: at most 64 keyframes per call");
  int batch_ids[64], single_ids[64], n_batch = 0, n_single = 0;
  for(int i = 0; i < n; ++i)
  {
    const rmd_seeds *h = handles[i];
    rmd_seeds *hm = handles[i];
    if(hm->mode == 1 && !seed_mode_allowed(hm)) leave_seed_mode(hm);
    {
      const int rcm = maybe_enter_seed_mode(hm);
      if(rcm) return rcm;
    }
    if(h0->variant == 0 && h->variant == 0 && h->patch == h0->patch && h->mode == 0 && h0->mode == 0) batch_ids[n_batch++] = i;
    else single_ids[n_single++] = i;
  }
  for(int g = 0; g < n_batch; g += STAGED_BATCH_MAX)
  {
    FilterParams P[STAGED_BATCH_MAX];
    const FilterParams *pp[STAGED_BATCH_MAX];
    const StagedMaps *mm[STAGED_BATCH_MAX];
    const int m = (n_batch - g < STAGED_BATCH_MAX) ? n_batch - g : STAGED_BATCH_MAX;
    for(int k = 0; k < m; ++k)
    {
      rmd_seeds *h = handles[batch_ids[g + k]];
      const int rci = prepare_update(h, h0->curr[slot], h0->curr_pitch, T_curr_world, P[k]);
      if(rci) return rci;
      if(h != h0)
      {
        // whatever is pending on the keyframe's own stream (set_reference, work-list rebuild) comes first
        RMD_CUDA_TRY(cudaEventRecord(h->fan_ev, h->stream));
        RMD_CUDA_TRY(cudaStreamWaitEvent(h0->stream, h->fan_ev, 0));
      }
      pp[k] = &P[k];
      mm[k] = h->maps;
    }
    {
      ProfScope prof_launch(4);
      RMD_CUDA_TRY(launch_depth_filter_staged(pp, mm, m, 0, h0->cursor, h0->patch, h0->stream));
    }
    for(int k = 0; k < m; ++k)
    {
      rmd_seeds *h = handles[batch_ids[g + k]];
      finish_update(h);
      const int rcs = request_stats(h, P[k], h0->stream);    // on the stream the batch ran on
      if(rcs) return rcs;
    }
  }
  for(int j = 0; j < n_single; ++j)
  {
    rmd_seeds *h = handles[single_ids[j]];
    if(h != h0)
    {
      RMD_CUDA_TRY(cudaEventRecord(h->fan_ev, h->stream));
      RMD_CUDA_TRY(cudaStreamWaitEvent(h0->stream, h->fan_ev, 0));
    }
    const cudaStream_t own = h->stream;
    h->stream = h0->stream;
    const int rci = enqueue_update(h, h0->curr[slot], h0->curr_pitch, T_curr_world);
    h->stream = own;
    if(rci) return rci;
  }
  // everything ran on h0's stream: the other keyframes' own streams continue after it
  RMD_CUDA_TRY(cudaEventRecord(h0->fan_ev, h0->stream));
  for(int i = 1; i < n; ++i)
    RMD_CUDA_TRY(cudaStreamWaitEvent(handles[i]->stream, h0->fan_ev, 0));
  RMD_CUDA_TRY(cudaEventRecord(h0->consumed[slot], h0->stream));
  return 0;
}

} // namespace

int rmd_seeds_update_many(rmd_seeds_t *const *handles, int n, const float *host_img, const float *T_curr_world)
{
  return update_many(handles, n, host_img, sizeof(float), T_curr_world);
}

int rmd_seeds_update_many_u8(rmd_seeds_t *const *handles, int n, const uint8_t *host_img, const float *T_curr_world)
{
  return update_many(handles, n, host_img, sizeof(uint8_t), T_curr_world);
}

int rmd_seeds_init_undistortion_map(rmd_seeds_t *s, float k1, float k2, float r1, float r2)
{
  RMD_REQUIRE(s, "rmd_seeds_init_undistortion_map: null handle");
  DeviceGuard guard(s->device);
  const size_t n = (size_t)s->width * s->height;
  if(!s->undist_host_xy)
  {
    s->undist_host_xy = (int16_t*)malloc(n * 2 * sizeof(int16_t));
    s->undist_host_frac = (uint16_t*)malloc(n * sizeof(uint16_t));
    if(!s->undist_host_xy || !s->undist_host_frac)
      return fail((int)cudaErrorMemoryAllocation, "rmd_seeds_init_undistortion_map: host allocation failed");
  }
  compute_undistort_maps(s->width, s->height, s->cam.fx, s->cam.fy, s->cam.cx, s->cam.cy, k1, k2, r1, r2,
                         s->undist_host_xy, s->undist_host_frac);
  short2 *xy = s->undist_xy;
  uint16_t *frac = s->undist_frac;
  if(!xy)
  {
    RMD_CUDA_TRY(cudaMalloc(&xy, n * sizeof(short2)));
    RMD_CUDA_TRY(cudaMalloc(&frac, n * sizeof(uint16_t)));
  }
  RMD_CUDA_TRY(cudaStreamSynchronize(s->copy_stream));   // frames in flight still use the previous maps
  RMD_CUDA_TRY(cudaStreamSynchronize(s->stream));
  RMD_CUDA_TRY(cudaMemcpy(xy, s->undist_host_xy, n * sizeof(short2), cudaMemcpyHostToDevice));
  RMD_CUDA_TRY(cudaMemcpy(frac, s->undist_host_frac, n * sizeof(uint16_t), cudaMemcpyHostToDevice));
  s->undist_xy = xy;
  s->undist_frac = frac;
  return 0;
}

int rmd_seeds_clear_undistortion_map(rmd_seeds_t *s)
{
  RMD_REQUIRE(s, "rmd_seeds_clear_undistortion_map: null handle");
  DeviceGuard guard(s->device);
  RMD_CUDA_TRY(cudaStreamSynchronize(s->copy_stream));   // the ingest kernels run there
  RMD_CUDA_TRY(cudaStreamSynchronize(s->stream));
  cudaFree(s->undist_xy); cudaFree(s->undist_frac);
  s->undist_xy = NULL; s->undist_frac = NULL;
  return 0;
}

int rmd_seeds_get_undistortion_map(rmd_seeds_t *s, int16_t *host_xy, uint16_t *host_frac)
{
  RMD_REQUIRE(s, "rmd_seeds_get_undistortion_map: null handle");
  if(!s->undist_xy)
    return fail(RMD_ERR_NOT_INITIALISED, "rmd_seeds_get_undistortion_map: init_undistortion_map has not been called");
  const size_t n = (size_t)s->width * s->height;
  if(host_xy) memcpy(host_xy, s->undist_host_xy, n * 2 * sizeof(int16_t));
  if(host_frac) memcpy(host_frac, s->undist_host_frac, n * sizeof(uint16_t));
  return 0;
}

int rmd_seeds_undistort_u8(rmd_seeds_t *s, const uint8_t *host_src, uint8_t *host_dst)
{
  RMD_REQUIRE(s && host_src && host_dst, "rmd_seeds_undistort_u8: null argument");
  if(!s->undist_xy)
    return fail(RMD_ERR_NOT_INITIALISED, "rmd_seeds_undistort_u8: init_undistortion_map has not been called");
  DeviceGuard guard(s->device);
  for(int i = 0; i < 2; ++i)
    if(!s->undist_tmp[i])
      RMD_CUDA_TRY(cudaMallocPitch(&s->undist_tmp[i], &s->undist_tmp_pitch, (size_t)s->width, s->height));
  RMD_CUDA_TRY(cudaMemcpy2DAsync(s->undist_tmp[0], s->undist_tmp_pitch, host_src, (size_t)s->width,
                                 (size_t)s->width, s->height, cudaMemcpyHostToDevice, s->stream));
  RMD_CUDA_TRY(launch_undistort_u8(s->undist_tmp[0], (int)s->undist_tmp_pitch, s->undist_xy, s->undist_frac,
                                   NULL, 0, s->undist_tmp[1], (int)s->undist_tmp_pitch, s->width, s->height,
                                   s->stream));
  s->n_total += 1;
  RMD_CUDA_TRY(cudaMemcpy2DAsync(host_dst, (size_t)s->width, s->undist_tmp[1], s->undist_tmp_pitch,
                                 (size_t)s->width, s->height, cudaMemcpyDeviceToHost, s->stream));
  RMD_CUDA_TRY(cudaStreamSynchronize(s->stream));
  return 0;
}

namespace
{

// Runs the two extraction kernels into `out` (device) and returns the number of CONVERGED pixels.
int point_cloud_run(rmd_seeds *s, const float *dev_depth, size_t depth_pitch_bytes, float4 *out, size_t capacity,
                    size_t *count)
{
  if(!s->has_reference)
    return fail(RMD_ERR_NOT_INITIALISED, "rmd_seeds_point_cloud: set_reference has not been called");
  {
    const int rc = wait_external(s);
    if(rc) return rc;
  }
  const int n_pixels = s->width * s->height;
  PointCloudParams P;
  memset(&P, 0, sizeof(P));
  P.n_blocks = (n_pixels + POINT_CLOUD_PIXELS - 1) / POINT_CLOUD_PIXELS;
  if(!s->pc_counts)
  {
    RMD_CUDA_TRY(cudaMalloc(&s->pc_counts, sizeof(unsigned int) * (size_t)P.n_blocks));
    RMD_CUDA_TRY(cudaMalloc(&s->pc_total, 2 * sizeof(unsigned int)));
    RMD_CUDA_TRY(cudaMemsetAsync(s->pc_total, 0, 2 * sizeof(unsigned int), s->stream));
  }
  P.width = s->width; P.height = s->height;
  P.conv = s->conv; P.conv_stride = (int)(s->conv_pitch / sizeof(int));
  if(dev_depth)
  {
    RMD_REQUIRE(depth_pitch_bytes >= sizeof(float) * (size_t)s->width && depth_pitch_bytes % sizeof(float) == 0,
                "rmd_seeds_point_cloud: bad depth pitch");
    P.depth = dev_depth; P.depth_stride = (int)(depth_pitch_bytes / sizeof(float)); P.depth_comps = 1;
  }
  else
  {
    P.depth = reinterpret_cast<const float*>(s->seed); P.depth_stride = s->seed_stride * 4; P.depth_comps = 4;  // mu
  }
  P.ref = s->ref; P.ref_stride = (int)(s->ref_pitch / sizeof(float));
  P.cam = s->cam;
  P.T_world_ref = s->T_world_ref;
  P.out = out;
  P.capacity = (unsigned int)(capacity > (size_t)n_pixels ? (size_t)n_pixels : capacity);
  P.block_counts = s->pc_counts;
  P.total = s->pc_total;
  RMD_CUDA_TRY(launch_point_cloud(P, s->stream));
  s->n_total += 2;
  unsigned int n = 0;
  RMD_CUDA_TRY(cudaMemcpyAsync(&n, s->pc_total, sizeof(n), cudaMemcpyDeviceToHost, s->stream));
  RMD_CUDA_TRY(cudaStreamSynchronize(s->stream));
  *count = n;
  return 0;
}

} // namespace

int rmd_seeds_point_cloud(rmd_seeds_t *s, const float *dev_depth, size_t depth_pitch_bytes,
                          float *host_xyzi, size_t capacity_points, size_t *count)
{
  RMD_REQUIRE(s && count && (host_xyzi || capacity_points == 0), "rmd_seeds_point_cloud: null argument");
  DeviceGuard guard(s->device);
  if(!s->pc_points)
    RMD_CUDA_TRY(cudaMalloc(&s->pc_points, sizeof(float4) * (size_t)s->width * s->height));
  const int rc = point_cloud_run(s, dev_depth, depth_pitch_bytes, s->pc_points, (size_t)s->width * s->height, count);
  if(rc) return rc;
  const size_t n = *count < capacity_points ? *count : capacity_points;
  if(n)
    RMD_CUDA_TRY(cudaMemcpy(host_xyzi, s->pc_points, n * sizeof(float4), cudaMemcpyDeviceToHost));
  return 0;
}

int rmd_seeds_point_cloud_device(rmd_seeds_t *s, const float *dev_depth, size_t depth_pitch_bytes,
                                 float *dev_xyzi, size_t capacity_points, size_t *count)
{
  RMD_REQUIRE(s && count && (dev_xyzi || capacity_points == 0), "rmd_seeds_point_cloud_device: null argument");
  RMD_REQUIRE(((uintptr_t)dev_xyzi % 16) == 0, "rmd_seeds_point_cloud_device: output must be 16-byte aligned");
  DeviceGuard guard(s->device);
  return point_cloud_run(s, dev_depth, depth_pitch_bytes, reinterpret_cast<float4*>(dev_xyzi), capacity_points, count);
}

int rmd_seeds_update_device(rmd_seeds_t *s, const float *dev_img, size_t pitch_bytes,
                            const float *T_curr_world)
{
  RMD_REQUIRE(s && dev_img && T_curr_world, "rmd_seeds_update_device: null argument");
  RMD_REQUIRE(pitch_bytes >= sizeof(float) * (size_t)s->width && pitch_bytes % 16 == 0 &&
              ((uintptr_t)dev_img % 16) == 0,
              "rmd_seeds_update_device: image must be 16-byte aligned with a pitch multiple of 16");
  if(!s->has_reference)
    return fail(RMD_ERR_NOT_INITIALISED, "rmd_seeds_update_device: set_reference has not been called");
  DeviceGuard guard(s->device);
  return enqueue_update(s, dev_img, pitch_bytes, T_curr_world);
}

int rmd_seeds_update_device_batch(rmd_seeds_t *s, const float *dev_frames, size_t frame_stride_bytes,
                                  size_t pitch_bytes, int n_frames, const float *T_curr_world)
{
  RMD_REQUIRE(s && dev_frames && T_curr_world, "rmd_seeds_update_device_batch: null argument");
  RMD_REQUIRE(n_frames >= 0, "rmd_seeds_update_device_batch: negative frame count");
  RMD_REQUIRE(pitch_bytes >= sizeof(float) * (size_t)s->width && pitch_bytes % 16 == 0 &&
              frame_stride_bytes % 16 == 0 && ((uintptr_t)dev_frames % 16) == 0,
              "rmd_seeds_update_device_batch: frames must be 16-byte aligned with pitch/stride multiples of 16");
  if(!s->has_reference)
    return fail(RMD_ERR_NOT_INITIALISED, "rmd_seeds_update_device_batch: set_reference has not been called");
  DeviceGuard guard(s->device);
  const char *base = reinterpret_cast<const char*>(dev_frames);
  for(int i = 0; i < n_frames; i += SEED_FRAMES_MAX)
  {
    const int m = (n_frames - i < SEED_FRAMES_MAX) ? n_frames - i : SEED_FRAMES_MAX;
    const float *frames[SEED_FRAMES_MAX];
    for(int k = 0; k < m; ++k)
      frames[k] = reinterpret_cast<const float*>(base + (size_t)(i + k) * frame_stride_bytes);
    const int rc = enqueue_frames(s, frames, pitch_bytes, T_curr_world + 12 * i, m);
    if(rc) return rc;
  }
  return 0;
}

int rmd_seeds_sync(rmd_seeds_t *s)
{
  RMD_REQUIRE(s, "rmd_seeds_sync: null handle");
  DeviceGuard guard(s->device);
  RMD_CUDA_TRY(cudaStreamSynchronize(s->copy_stream));
  RMD_CUDA_TRY(cudaStreamSynchronize(s->stream));
  unsigned int flag = 0u;
  RMD_CUDA_TRY(cudaMemcpy(&flag, s->cursor + STAGED_BATCH_MAX + 1, sizeof(flag), cudaMemcpyDeviceToHost));
  if(flag)
    return fail(RMD_ERR_DEVICE_WAIT, "rmd_seeds_sync: a bounded wait of a chained launch expired on the device");
  return 0;
}

int rmd_seeds_download(rmd_seeds_t *s, int field, void *host_dst)
{
  RMD_REQUIRE(s && host_dst, "rmd_seeds_download: null argument");
  DeviceGuard guard(s->device);
  const size_t w = s->width, h = s->height;
  if(is_seed_field(field) || is_templ_field(field))
  {
    int rc = ensure_dense_tmp(s);
    if(rc) return rc;
    rc = export_field(s, field, s->dense_tmp, s->width);
    if(rc) return rc;
    RMD_CUDA_TRY(cudaMemcpyAsync(host_dst, s->dense_tmp, sizeof(float) * w * h,
                                 cudaMemcpyDeviceToHost, s->stream));
  }
  else if(field == RMD_FIELD_CONVERGENCE)
  {
    RMD_CUDA_TRY(cudaMemcpy2DAsync(host_dst, sizeof(int) * w, s->conv, s->conv_pitch, sizeof(int) * w,
                                   h, cudaMemcpyDeviceToHost, s->stream));
  }
  else if(field == RMD_FIELD_EPIPOLAR_MATCHES)
  {
    if(!s->matches)
      return fail(RMD_ERR_NOT_INITIALISED,
                  "rmd_seeds_download: matches are only kept with RMD_OPT_RECORD_MATCHES");
    RMD_CUDA_TRY(cudaMemcpy2DAsync(host_dst, sizeof(float2) * w, s->matches, s->matches_pitch,
                                   sizeof(float2) * w, h, cudaMemcpyDeviceToHost, s->stream));
  }
  else if(field == RMD_FIELD_DEBUG_TIMELINE)
  {
    if(!s->timeline)
      return fail(RMD_ERR_NOT_INITIALISED, "rmd_seeds_download: RMD_OPT_DEBUG_TIMELINE is off");
    RMD_CUDA_TRY(cudaMemcpyAsync(host_dst, s->timeline, s->timeline_bytes, cudaMemcpyDeviceToHost, s->stream));
  }
  else if(field == RMD_FIELD_REF_IMG)
  {
    RMD_CUDA_TRY(cudaMemcpy2DAsync(host_dst, sizeof(float) * w, s->ref, s->ref_pitch,
                                   sizeof(float) * w, h, cudaMemcpyDeviceToHost, s->stream));
  }
  else
  {
    return fail(RMD_ERR_INVALID_ARGUMENT, "rmd_seeds_download: unknown field");
  }
  RMD_CUDA_TRY(cudaStreamSynchronize(s->stream));
  return 0;
}

int rmd_seeds_upload_state(rmd_seeds_t *s, int field, const void *host_src)
{
  RMD_REQUIRE(s && host_src, "rmd_seeds_upload_state: null argument");
  DeviceGuard guard(s->device);
  {
    const int rc = wait_external(s);
    if(rc) return rc;
  }
  const size_t w = s->width, h = s->height;
  if(is_seed_field(field))
  {
    const int rc = ensure_dense_tmp(s);
    if(rc) return rc;
    RMD_CUDA_TRY(cudaMemcpyAsync(s->dense_tmp, host_src, sizeof(float) * w * h,
                                 cudaMemcpyHostToDevice, s->stream));
    RMD_CUDA_TRY(launch_import_plane(s->dense_tmp, s->width, reinterpret_cast<float*>(s->seed),
                                     s->seed_stride * 4, 4, field - RMD_FIELD_MU, s->width,
                                     s->height, s->stream));
    s->n_total += 1;
  }
  else if(field == RMD_FIELD_CONVERGENCE)
  {
    RMD_CUDA_TRY(cudaMemcpy2DAsync(s->conv, s->conv_pitch, host_src, sizeof(int) * w, sizeof(int) * w,
                                   h, cudaMemcpyHostToDevice, s->stream));
  }
  else
  {
    return fail(RMD_ERR_INVALID_ARGUMENT, "rmd_seeds_upload_state: field is not writable");
  }
  RMD_CUDA_TRY(cudaStreamSynchronize(s->stream));
  s->trust_conv = false;  // the map may no longer agree with the parameters
  s->worklist_valid = false;
  leave_seed_mode(s);
  return 0;
}

int rmd_seeds_device_ptr(rmd_seeds_t *s, int field, void **dev_ptr, size_t *pitch_bytes)
{
  RMD_REQUIRE(s && dev_ptr && pitch_bytes, "rmd_seeds_device_ptr: null argument");
  DeviceGuard guard(s->device);
  if(field == RMD_FIELD_CONVERGENCE)
  {
    *dev_ptr = s->conv;
    *pitch_bytes = s->conv_pitch;
  }
  else if(field == RMD_FIELD_REF_IMG)
  {
    *dev_ptr = s->ref;
    *pitch_bytes = s->ref_pitch;
  }
  else if(is_seed_field(field) || is_templ_field(field))
  {
    const int slot = is_seed_field(field) ? field - RMD_FIELD_MU : 4 + field - RMD_FIELD_SUM_TEMPL;
    if(!s->planar[slot])
      RMD_CUDA_TRY(cudaMallocPitch(&s->planar[slot], &s->planar_pitch,
                                   sizeof(float) * (size_t)s->width, s->height));
    const int rc = export_field(s, field, s->planar[slot], (int)(s->planar_pitch / sizeof(float)));
    if(rc) return rc;
    *dev_ptr = s->planar[slot];
    *pitch_bytes = s->planar_pitch;
  }
  else if(field == RMD_FIELD_EPIPOLAR_MATCHES)
  {
    if(!s->matches)
      return fail(RMD_ERR_NOT_INITIALISED,
                  "rmd_seeds_device_ptr: matches are only kept with RMD_OPT_RECORD_MATCHES");
    *dev_ptr = s->matches;
    *pitch_bytes = s->matches_pitch;
  }
  else
  {
    return fail(RMD_ERR_INVALID_ARGUMENT, "rmd_seeds_device_ptr: unknown field");
  }
  RMD_CUDA_TRY(cudaStreamSynchronize(s->stream));
  return 0;
}

int rmd_seeds_copy_field_to_device(rmd_seeds_t *s, int field, void *dev_dst, size_t dst_pitch_bytes)
{
  RMD_REQUIRE(s && dev_dst, "rmd_seeds_copy_field_to_device: null argument");
  DeviceGuard guard(s->device);
  const size_t w = s->width, h = s->height;
  if(is_seed_field(field) || is_templ_field(field))
  {
    RMD_REQUIRE(dst_pitch_bytes >= sizeof(float) * w && dst_pitch_bytes % sizeof(float) == 0,
                "rmd_seeds_copy_field_to_device: bad pitch");
    return export_field(s, field, static_cast<float*>(dev_dst), (int)(dst_pitch_bytes / sizeof(float)));
  }
  if(field == RMD_FIELD_CONVERGENCE)
  {
    RMD_REQUIRE(dst_pitch_bytes >= sizeof(int) * w, "rmd_seeds_copy_field_to_device: bad pitch");
    RMD_CUDA_TRY(cudaMemcpy2DAsync(dev_dst, dst_pitch_bytes, s->conv, s->conv_pitch, sizeof(int) * w, h,
                                   cudaMemcpyDeviceToDevice, s->stream));
    return 0;
  }
  return fail(RMD_ERR_INVALID_ARGUMENT, "rmd_seeds_copy_field_to_device: unsupported field");
}

int rmd_seeds_converged_count(rmd_seeds_t *s, size_t *count)
{
  RMD_REQUIRE(s && count, "rmd_seeds_converged_count: null argument");
  DeviceGuard guard(s->device);
  if(s->mode == 1)
  {
    unsigned int total = 0u;
    RMD_CUDA_TRY(cudaMemcpyAsync(&total, s->seed_ctl + 3, sizeof(total), cudaMemcpyDeviceToHost, s->stream));
    RMD_CUDA_TRY(cudaStreamSynchronize(s->stream));
    *count = (size_t)total;
    return 0;
  }
  unsigned int v[4] = {0u, 0u, 0u, 0u};
  if(s->frame_index > 0)
  {
    RMD_CUDA_TRY(cudaMemcpyAsync(v, s->counters, sizeof(v), cudaMemcpyDeviceToHost, s->stream));
    RMD_CUDA_TRY(cudaStreamSynchronize(s->stream));
  }
  // seeds of tiles the staged kernel has retired from its work list are counted in v[3]
  *count = (size_t)v[s->frame_index % 3] + (s->last_staged ? (size_t)v[3] : 0);
  return 0;
}

int rmd_seeds_dist_from_ref(rmd_seeds_t *s, float *dist)
{
  RMD_REQUIRE(s && dist, "rmd_seeds_dist_from_ref: null argument");
  *dist = s->dist_from_ref;
  return 0;
}

int rmd_seeds_size(rmd_seeds_t *s, int *width, int *height, int *patch_side)
{
  RMD_REQUIRE(s, "rmd_seeds_size: null handle");
  if(width) *width = s->width;
  if(height) *height = s->height;
  if(patch_side) *patch_side = s->patch;
  return 0;
}

int rmd_seeds_launch_count(rmd_seeds_t *s, uint64_t *fused, uint64_t *total)
{
  RMD_REQUIRE(s, "rmd_seeds_launch_count: null handle");
  if(fused) *fused = s->n_fused;
  if(total) *total = s->n_total;
  return 0;
}

int rmd_seeds_enable_kernel_timing(rmd_seeds_t *s, int on)
{
  RMD_REQUIRE(s, "rmd_seeds_enable_kernel_timing: null handle");
  s->timing = (on != 0);
  s->t_valid = false;
  return 0;
}

int rmd_seeds_last_kernel_ms(rmd_seeds_t *s, float *ms)
{
  RMD_REQUIRE(s && ms, "rmd_seeds_last_kernel_ms: null argument");
  if(!s->t_valid)
    return fail(RMD_ERR_NOT_INITIALISED, "rmd_seeds_last_kernel_ms: timing not enabled / no kernel yet");
  DeviceGuard guard(s->device);
  RMD_CUDA_TRY(cudaEventSynchronize(s->t1));
  RMD_CUDA_TRY(cudaEventElapsedTime(ms, s->t0, s->t1));
  return 0;
}

} // extern "C"

// ============================================================== denoiser

struct rmd_denoiser
{
  int device;
  int width, height, stride;
  cudaStream_t own_stream, stream;
  // planar solver state (denoiser.cu): one allocation of 10 planes of stride x height floats --
  // (u, u_head, p.x, p.y) twice (ping-pong between launches), then g and the noisy depth
  float *planes;
  float *state[2][4];
  float *g, *noisy;
  CUtensorMap map_state[2][4], map_g, map_noisy;   // TMA descriptors of the planes (fixed for the handle's life)
  float large_sigma_sq;
  uint64_t n_total;
};

namespace
{

int denoiser_iterate(rmd_denoiser *d, float lambda, int iterations, int *final_buf)
{
  DenoiseBlockParams bp;
  memset(&bp, 0, sizeof(bp));
  bp.width = d->width; bp.height = d->height; bp.stride = d->stride;
  bp.g = d->map_g; bp.mu = d->map_noisy;
  const float L = sqrtf(8.0f);          // depthmap_denoiser.cu:130
  bp.tau = 0.02f;                       // :131
  bp.sigma = (1 / (L * L)) / bp.tau;    // :132
  bp.theta = 0.5f;                      // :133
  bp.lambda = lambda;
  int cur = 0;
  // DENOISE_T iterations per launch (temporal blocking); the last launch takes the remainder
  for(int left = iterations; left > 0; left -= DENOISE_T)
  {
    bp.n_it = left < DENOISE_T ? left : DENOISE_T;
    bp.in_u = d->map_state[cur][0]; bp.in_uh = d->map_state[cur][1];
    bp.in_px = d->map_state[cur][2]; bp.in_py = d->map_state[cur][3];
    bp.out_u = d->state[cur ^ 1][0]; bp.out_uh = d->state[cur ^ 1][1];
    bp.out_px = d->state[cur ^ 1][2]; bp.out_py = d->state[cur ^ 1][3];
    RMD_CUDA_TRY(launch_denoise_block(bp, d->stream));
    d->n_total += 1;
    cur ^= 1;
  }
  *final_buf = cur;
  return 0;
}

int denoiser_setup_common(rmd_denoiser *d, DenoiseSetupParams &P)
{
  P.width = d->width; P.height = d->height;
  P.large_sigma_sq = d->large_sigma_sq;
  P.g = d->g; P.noisy = d->noisy;
  P.u = d->state[0][0]; P.u_head = d->state[0][1]; P.p_x = d->state[0][2]; P.p_y = d->state[0][3];
  P.stride = d->stride;
  return 0;
}

int denoiser_emit(rmd_denoiser *d, int buf, float *host_out, float *dev_out, size_t dev_pitch)
{
  const size_t row = sizeof(float) * (size_t)d->width, pitch = sizeof(float) * (size_t)d->stride;
  const float *u = d->state[buf][0];   // the denoised depth is the primal variable itself: no export kernel
  if(dev_out)
  {
    RMD_CUDA_TRY(cudaMemcpy2DAsync(dev_out, dev_pitch, u, pitch, row, d->height, cudaMemcpyDeviceToDevice, d->stream));
    return 0;
  }
  RMD_CUDA_TRY(cudaMemcpy2DAsync(host_out, row, u, pitch, row, d->height, cudaMemcpyDeviceToHost, d->stream));
  RMD_CUDA_TRY(cudaStreamSynchronize(d->stream));  // u_.getDevData is blocking, :223
  return 0;
}

} // namespace

extern "C"
{

int rmd_denoiser_create(int width, int height, int device, rmd_denoiser_t **out)
{
  RMD_REQUIRE(out, "rmd_denoiser_create: out is null");
  *out = NULL;
  RMD_REQUIRE(width > 0 && height > 0, "rmd_denoiser_create: bad image size");
  if(device < 0) RMD_CUDA_TRY(cudaGetDevice(&device));
  DeviceGuard guard(device);
  rmd_denoiser *d = new(std::nothrow) rmd_denoiser();
  if(!d) return fail((int)cudaErrorMemoryAllocation, "rmd_denoiser_create: host allocation failed");
  memset(d, 0, sizeof(*d));
  d->device = device;
  d->width = width; d->height = height;
  d->stride = (int)round_up(width, 32);
  d->large_sigma_sq = -1.0f;  // "not set" (the reference leaves it uninitialised, SURVEY 5)
  cudaError_t err = cudaStreamCreateWithFlags(&d->own_stream, cudaStreamNonBlocking);
  const size_t n = (size_t)d->stride * height;
  if(err == cudaSuccess) err = cudaMalloc(&d->planes, sizeof(float) * n * 10);
  if(err != cudaSuccess)
  {
    rmd_denoiser_destroy(d);
    return fail_cuda(err, "rmd_denoiser_create");
  }
  for(int b = 0; b < 2; ++b)
    for(int k = 0; k < 4; ++k)
      d->state[b][k] = d->planes + n * (size_t)(4 * b + k);
  d->g = d->planes + n * 8;
  d->noisy = d->planes + n * 9;
  int rc = 0;
  for(int b = 0; b < 2 && !rc; ++b)
    for(int k = 0; k < 4 && !rc; ++k)
      rc = encode_tensor_map_2d_f32(&d->map_state[b][k], d->state[b][k], width, height, d->stride,
                                    DENOISE_EXT_W, DENOISE_EXT_H);
  if(!rc) rc = encode_tensor_map_2d_f32(&d->map_g, d->g, width, height, d->stride, DENOISE_EXT_W, DENOISE_EXT_H);
  if(!rc) rc = encode_tensor_map_2d_f32(&d->map_noisy, d->noisy, width, height, d->stride, DENOISE_EXT_W, DENOISE_EXT_H);
  if(rc)
  {
    rmd_denoiser_destroy(d);
    return rc;
  }
  d->stream = d->own_stream;
  *out = d;
  return 0;
}

int rmd_denoiser_destroy(rmd_denoiser_t *d)
{
  if(!d) return 0;
  DeviceGuard guard(d->device);
  cudaDeviceSynchronize();
  if(d->own_stream) cudaStreamDestroy(d->own_stream);
  cudaFree(d->planes);
  cudaGetLastError();
  delete d;
  return 0;
}

int rmd_denoiser_set_stream(rmd_denoiser_t *d, void *cuda_stream)
{
  RMD_REQUIRE(d, "rmd_denoiser_set_stream: null handle");
  DeviceGuard guard(d->device);
  RMD_CUDA_TRY(cudaStreamSynchronize(d->stream));
  d->stream = cuda_stream ? (cudaStream_t)cuda_stream : d->own_stream;
  return 0;
}

int rmd_denoiser_set_large_sigma_sq(rmd_denoiser_t *d, float depth_range)
{
  RMD_REQUIRE(d, "rmd_denoiser_set_large_sigma_sq: null handle");
  d->large_sigma_sq = depth_range * depth_range / 72.0f;  // depthmap_denoiser.cu:228
  return 0;
}

int rmd_denoiser_run(rmd_denoiser_t *d, const float *mu, size_t mu_pitch, const float *sigma_sq,
                     size_t sigma_sq_pitch, const float *a, size_t a_pitch, const float *b,
                     size_t b_pitch, float *host_denoised, float lambda, int iterations)
{
  RMD_REQUIRE(d && mu && sigma_sq && a && b && host_denoised, "rmd_denoiser_run: null argument");
  RMD_REQUIRE(iterations >= 0, "rmd_denoiser_run: negative iteration count");
  if(d->large_sigma_sq < 0.0f)
    return fail(RMD_ERR_NOT_INITIALISED,
                "rmd_denoiser_run: set_large_sigma_sq must be called before this function");
  DeviceGuard guard(d->device);
  // Inputs may have been produced on another stream (the seed matrix' own):
  // the reference runs everything on the legacy default stream, which orders
  // it implicitly; here they must be complete when this is called
  // (rmd_seeds_device_ptr, which hands them out, synchronises that stream).
  DenoiseSetupParams P;
  memset(&P, 0, sizeof(P));
  denoiser_setup_common(d, P);
  P.mu = mu; P.mu_stride = (int)(mu_pitch / sizeof(float));
  P.sigma_sq = sigma_sq; P.sigma_sq_stride = (int)(sigma_sq_pitch / sizeof(float));
  P.a = a; P.a_stride = (int)(a_pitch / sizeof(float));
  P.b = b; P.b_stride = (int)(b_pitch / sizeof(float));
  RMD_CUDA_TRY(launch_denoise_setup(P, false, d->stream));
  d->n_total += 1;
  int buf = 0;
  const int rc = denoiser_iterate(d, lambda, iterations, &buf);
  if(rc) return rc;
  return denoiser_emit(d, buf, host_denoised, NULL, 0);
}

static int run_seeds_common(rmd_denoiser_t *d, rmd_seeds_t *s, float lambda, int iterations, int *buf)
{
  if(d->large_sigma_sq < 0.0f)
    return fail(RMD_ERR_NOT_INITIALISED,
                "rmd_denoiser_run_seeds: set_large_sigma_sq must be called before this function");
  RMD_REQUIRE(s->width == d->width && s->height == d->height && s->device == d->device,
              "rmd_denoiser_run_seeds: seed matrix and denoiser differ in size or device");
  RMD_CUDA_TRY(cudaStreamSynchronize(s->stream));  // the seeds must be final
  DenoiseSetupParams P;
  memset(&P, 0, sizeof(P));
  denoiser_setup_common(d, P);
  P.seed = s->seed; P.seed_stride = s->seed_stride;
  RMD_CUDA_TRY(launch_denoise_setup(P, true, d->stream));
  d->n_total += 1;
  // s->seed has been read once this kernel is done: later writers on s->stream (update,
  // set_reference, upload_state) wait for it
  RMD_CUDA_TRY(cudaEventRecord(s->ext_ev, d->stream));
  s->ext_pending = true;
  return denoiser_iterate(d, lambda, iterations, buf);
}

int rmd_denoiser_run_seeds(rmd_denoiser_t *d, rmd_seeds_t *s, float *host_denoised, float lambda,
                           int iterations)
{
  RMD_REQUIRE(d && s && host_denoised, "rmd_denoiser_run_seeds: null argument");
  RMD_REQUIRE(iterations >= 0, "rmd_denoiser_run_seeds: negative iteration count");
  DeviceGuard guard(d->device);
  int buf = 0;
  const int rc = run_seeds_common(d, s, lambda, iterations, &buf);
  if(rc) return rc;
  return denoiser_emit(d, buf, host_denoised, NULL, 0);
}

int rmd_denoiser_run_seeds_to_device(rmd_denoiser_t *d, rmd_seeds_t *s, float *dev_out,
                                     size_t out_pitch_bytes, float lambda, int iterations)
{
  RMD_REQUIRE(d && s && dev_out, "rmd_denoiser_run_seeds_to_device: null argument");
  RMD_REQUIRE(iterations >= 0, "rmd_denoiser_run_seeds_to_device: negative iteration count");
  RMD_REQUIRE(out_pitch_bytes >= sizeof(float) * (size_t)d->width && out_pitch_bytes % sizeof(float) == 0,
              "rmd_denoiser_run_seeds_to_device: bad pitch");
  DeviceGuard guard(d->device);
  int buf = 0;
  const int rc = run_seeds_common(d, s, lambda, iterations, &buf);
  if(rc) return rc;
  const int rc2 = denoiser_emit(d, buf, NULL, dev_out, out_pitch_bytes);
  if(rc2) return rc2;
  // dev_out is complete when this event fires: rmd_seeds_point_cloud(s, dev_out, ...) and everything
  // else on the seeds' stream waits for it (the two streams are cudaStreamNonBlocking: no implicit order)
  RMD_CUDA_TRY(cudaEventRecord(s->ext_ev, d->stream));
  s->ext_pending = true;
  return 0;
}

int rmd_denoiser_sync(rmd_denoiser_t *d)
{
  RMD_REQUIRE(d, "rmd_denoiser_sync: null handle");
  DeviceGuard guard(d->device);
  RMD_CUDA_TRY(cudaStreamSynchronize(d->stream));
  return 0;
}

int rmd_denoiser_launch_count(rmd_denoiser_t *d, uint64_t *total)
{
  RMD_REQUIRE(d && total, "rmd_denoiser_launch_count: null argument");
  *total = d->n_total;
  return 0;
}

} // extern "C"

// ============================================================ reductions

namespace
{

struct ReduceContext
{
  ReduceScratch scratch;
  bool ready;
};

std::mutex g_reduce_mutex;
ReduceContext g_reduce_ctx[64];

// Scratch of the calling thread's current device (allocated on first use).
int reduce_scratch(ReduceScratch **out)
{
  int device = 0;
  RMD_CUDA_TRY(cudaGetDevice(&device));
  RMD_REQUIRE(device >= 0 && device < 64, "reduce: device index out of range");
  ReduceContext &ctx = g_reduce_ctx[device];
  if(!ctx.ready)
  {
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    ctx.scratch.max_blocks = sms * 4;
    RMD_CUDA_TRY(cudaMalloc(&ctx.scratch.partials, sizeof(double) * 2 * (size_t)ctx.scratch.max_blocks));
    RMD_CUDA_TRY(cudaMalloc(&ctx.scratch.ticket, sizeof(unsigned int)));
    RMD_CUDA_TRY(cudaMemset(ctx.scratch.ticket, 0, sizeof(unsigned int)));
    RMD_CUDA_TRY(cudaMalloc(&ctx.scratch.result, 16));
    ctx.ready = true;
  }
  *out = &ctx.scratch;
  return 0;
}

} // namespace

extern "C"
{

// The reference's reducers run on the legacy default stream and block on a
// 4-byte cudaMemcpy (src/reduction.cu:108,163); same here.  The library's own
// streams are cudaStreamNonBlocking, so the legacy stream does NOT order after
// them: an image produced by a handle must be complete before it is reduced
// (rmd_seeds_device_ptr synchronises; after rmd_seeds_copy_field_to_device call
// rmd_seeds_sync first).
int rmd_reduce_sum_f32(const float *dev_img, size_t stride, size_t width, size_t height, float *out)
{
  RMD_REQUIRE(dev_img && out, "rmd_reduce_sum_f32: null argument");
  std::lock_guard<std::mutex> lock(g_reduce_mutex);
  ReduceScratch *sc = NULL;
  const int rc = reduce_scratch(&sc);
  if(rc) return rc;
  RMD_CUDA_TRY(launch_sum_f32(dev_img, stride, width, height, *sc, 0));
  double r[2];
  RMD_CUDA_TRY(cudaMemcpy(r, sc->result, sizeof(r), cudaMemcpyDeviceToHost));
  *out = (float)r[0];
  return 0;
}

int rmd_reduce_sum_i32(const int32_t *dev_img, size_t stride, size_t width, size_t height,
                       int32_t *out)
{
  RMD_REQUIRE(dev_img && out, "rmd_reduce_sum_i32: null argument");
  std::lock_guard<std::mutex> lock(g_reduce_mutex);
  ReduceScratch *sc = NULL;
  const int rc = reduce_scratch(&sc);
  if(rc) return rc;
  RMD_CUDA_TRY(launch_sum_i32(dev_img, stride, width, height, *sc, 0));
  long long r[2];
  RMD_CUDA_TRY(cudaMemcpy(r, sc->result, sizeof(r), cudaMemcpyDeviceToHost));
  *out = (int32_t)r[0];  // wraps like the reference's int accumulation
  return 0;
}

int rmd_reduce_count_eq_i32(const int32_t *dev_img, size_t stride, size_t width, size_t height,
                            int32_t value, size_t *out)
{
  RMD_REQUIRE(dev_img && out, "rmd_reduce_count_eq_i32: null argument");
  std::lock_guard<std::mutex> lock(g_reduce_mutex);
  ReduceScratch *sc = NULL;
  const int rc = reduce_scratch(&sc);
  if(rc) return rc;
  RMD_CUDA_TRY(launch_count_eq_i32(dev_img, stride, width, height, value, *sc, 0));
  long long r[2];
  RMD_CUDA_TRY(cudaMemcpy(r, sc->result, sizeof(r), cudaMemcpyDeviceToHost));
  *out = (size_t)r[0];
  return 0;
}

int rmd_reduce_min_max_f32(const float *dev_img, size_t stride, size_t width, size_t height,
                           float *out_min, float *out_max)
{
  RMD_REQUIRE(dev_img && out_min && out_max, "rmd_reduce_min_max_f32: null argument");
  std::lock_guard<std::mutex> lock(g_reduce_mutex);
  ReduceScratch *sc = NULL;
  const int rc = reduce_scratch(&sc);
  if(rc) return rc;
  RMD_CUDA_TRY(launch_min_max_f32(dev_img, stride, width, height, *sc, 0));
  double r[2];
  RMD_CUDA_TRY(cudaMemcpy(r, sc->result, sizeof(r), cudaMemcpyDeviceToHost));
  *out_min = (float)r[0];
  *out_max = (float)r[1];
  return 0;
}

// ========================================================== device image

int rmd_image_alloc(size_t width, size_t height, size_t elem_size, void **dev_ptr, size_t *pitch_bytes)
{
  RMD_REQUIRE(dev_ptr && pitch_bytes && width && height && elem_size, "rmd_image_alloc: bad argument");
  RMD_CUDA_TRY(cudaMallocPitch(dev_ptr, pitch_bytes, width * elem_size, height));
  return 0;
}

int rmd_image_free(void *dev_ptr)
{
  RMD_CUDA_TRY(cudaFree(dev_ptr));
  return 0;
}

int rmd_image_upload(void *dev_ptr, size_t pitch_bytes, const void *host_src, size_t width,
                     size_t height, size_t elem_size)
{
  RMD_REQUIRE(dev_ptr && host_src, "rmd_image_upload: null argument");
  RMD_CUDA_TRY(cudaMemcpy2D(dev_ptr, pitch_bytes, host_src, width * elem_size, width * elem_size,
                            height, cudaMemcpyHostToDevice));
  return 0;
}

int rmd_image_download(const void *dev_ptr, size_t pitch_bytes, void *host_dst, size_t width,
                       size_t height, size_t elem_size)
{
  RMD_REQUIRE(dev_ptr && host_dst, "rmd_image_download: null argument");
  RMD_CUDA_TRY(cudaMemcpy2D(host_dst, width * elem_size, dev_ptr, pitch_bytes, width * elem_size,
                            height, cudaMemcpyDeviceToHost));
  return 0;
}

int rmd_image_zero(void *dev_ptr, size_t pitch_bytes, size_t width, size_t height, size_t elem_size)
{
  RMD_REQUIRE(dev_ptr, "rmd_image_zero: null argument");
  RMD_CUDA_TRY(cudaMemset2D(dev_ptr, pitch_bytes, 0, width * elem_size, height));
  return 0;
}

int rmd_image_copy(void *dst, size_t dst_pitch, const void *src, size_t src_pitch, size_t width,
                   size_t height, size_t elem_size)
{
  RMD_REQUIRE(dst && src, "rmd_image_copy: null argument");
  RMD_CUDA_TRY(cudaMemcpy2D(dst, dst_pitch, src, src_pitch, width * elem_size, height,
                            cudaMemcpyDeviceToDevice));
  return 0;
}

} // extern "C"

// ============================================================ TSDF volume
// The volume's entry points are in volume_api.cu; these two read the seeds' internals and order the volume's
// stream against theirs.

extern "C"
{

int rmd_volume_integrate_seeds(rmd_volume_t *v, rmd_seeds_t *s, const float *dev_depth, size_t depth_pitch)
{
  RMD_REQUIRE(v && s, "rmd_volume_integrate_seeds: null handle");
  RMD_REQUIRE(v->device == s->device, "rmd_volume_integrate_seeds: volume and seeds on different devices");
  RMD_REQUIRE(!dev_depth || depth_pitch_ok(depth_pitch, s->width), "rmd_volume_integrate_seeds: bad depth pitch");
  if(!s->has_reference)
    return fail(RMD_ERR_NOT_INITIALISED, "rmd_volume_integrate_seeds: the seeds have no reference frame");
  DeviceGuard guard(v->device);
  // As rmd_seeds_propagate_prior with its source: run after everything that writes the seeds' state (their own
  // stream, and work another handle enqueued against them, e.g. the denoised image) ...
  RMD_CUDA_TRY(cudaEventRecord(v->seeds_ev, s->stream));
  RMD_CUDA_TRY(cudaStreamWaitEvent(v->stream, v->seeds_ev, 0));
  if(s->ext_pending)
    RMD_CUDA_TRY(cudaStreamWaitEvent(v->stream, s->ext_ev, 0));
  VolumeIntegrateParams P;
  memset(&P, 0, sizeof(P));
  P.width = s->width; P.height = s->height;
  P.cam = s->cam;
  P.T_curr_world = s->T_ref_world;
  if(dev_depth)
  {
    P.depth = dev_depth; P.depth_stride = depth_pitch / sizeof(float); P.depth_comps = 1;
  }
  else
  {
    P.depth = reinterpret_cast<const float*>(s->seed); P.depth_stride = (size_t)s->seed_stride * 4; P.depth_comps = 4;
  }
  P.conv = s->conv; P.conv_stride = s->conv_pitch / sizeof(int);
  if(v->col)   // with the intensity channel, the reference image is fused too
  {
    P.intensity = s->ref; P.intensity_stride = s->ref_pitch / sizeof(float);
  }
  const int rc = volume_integrate(v, P);
  if(rc) return rc;
  // ... and a later writer of the seeds (update, set_reference, upload_state) waits for the kernel's reads
  RMD_CUDA_TRY(cudaEventRecord(s->ext_ev, v->stream));
  s->ext_pending = true;
  return 0;
}

} // extern "C"

namespace
{

// rmd_volume_prior_seeds[_box]: box, the box (lo, dims) of the map instead of the window.
int volume_prior_seeds(const char *what, rmd_volume_t *v, rmd_seeds_t *s, float sigma_sq_frac, bool box,
                       const int64_t lo[3], const int dims[3])
{
  const std::string w(what);
  RMD_REQUIRE(v && s, (w + ": null handle").c_str());
  RMD_REQUIRE(v->device == s->device, (w + ": volume and seeds on different devices").c_str());
  RMD_REQUIRE(sigma_sq_frac > 0.0f && sigma_sq_frac <= 1.0f, (w + ": sigma_sq_frac must be in (0, 1]").c_str());
  if(!s->has_reference || s->frame_index != 0)
    return fail(RMD_ERR_NOT_INITIALISED, (w + ": the seeds need a reference frame set since their last update").c_str());
  DeviceGuard guard(s->device);
  VolumeGrid g = v->g;
  if(box)   // the box's records, gathered on the volume's stream: the hand-off below orders the rays after them
  {
    const int rc = volume_box_records(v, lo, dims, g, NULL, what);
    if(rc) return rc;
  }
  {
    const int rc = wait_external(s);
    if(rc) return rc;
  }
  // The rays run on the seeds' stream and read the model as the volume's queued work leaves it (e.g. the
  // integration of the keyframe just left) ...
  RMD_CUDA_TRY(cudaEventRecord(v->seeds_ev, v->stream));
  RMD_CUDA_TRY(cudaStreamWaitEvent(s->stream, v->seeds_ev, 0));
  VolumeRaycastParams P;
  memset(&P, 0, sizeof(P));
  P.g = g;
  P.width = s->width; P.height = s->height;
  P.cam = s->cam;
  P.T_world_curr = s->T_world_ref;   // = pose_inverse(pose_from(T_curr_world)), as rmd_volume_raycast computes it
  VolumePriorSeeds S;
  memset(&S, 0, sizeof(S));
  S.seed = s->seed; S.seed_stride = s->seed_stride;
  S.conv = s->conv; S.conv_stride = (int)(s->conv_pitch / sizeof(int));
  S.min_depth = s->min_depth; S.max_depth = s->max_depth;
  S.sigma_sq = sigma_sq_frac * s->sigma_sq_max;   // as prior_apply
  RMD_CUDA_TRY(launch_volume_prior(P, S, s->stream));
  s->n_total += 1;
  // ... and a later writer of the volume (integrate, reset, upload; for a box also the next gather into the same
  // scratch) waits for the rays' reads.  The wait above has already taken the event's previous record, so recording
  // it again loses nothing.
  RMD_CUDA_TRY(cudaEventRecord(v->seeds_ev, s->stream));
  RMD_CUDA_TRY(cudaStreamWaitEvent(v->stream, v->seeds_ev, 0));
  return 0;
}

} // namespace

extern "C"
{

int rmd_volume_prior_seeds(rmd_volume_t *v, rmd_seeds_t *s, float sigma_sq_frac)
{
  return volume_prior_seeds("rmd_volume_prior_seeds", v, s, sigma_sq_frac, false, NULL, NULL);
}

int rmd_volume_prior_seeds_box(rmd_volume_t *v, rmd_seeds_t *s, float sigma_sq_frac, const int64_t lo[3],
                               const int dims[3])
{
  return volume_prior_seeds("rmd_volume_prior_seeds_box", v, s, sigma_sq_frac, true, lo, dims);
}

} // extern "C"
