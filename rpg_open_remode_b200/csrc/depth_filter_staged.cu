// depth_filter_staged.cu -- fused depth filter, staged variant for sm_90a.
//
// One CTA (8 warps) per listed 32x8 tile of the reference view, one warp per
// pixel row.  Per frame (details and measurements: DESIGN.md section 4.1):
//   W. the CTA looks up its tile in the frame's work list, written by the
//      previous frame's kernel: busy tiles first, tiles that are finished for
//      good not at all, very busy tiles several times (3b);
//   0. classify every seed (convergence check, src/seed_check.cu:29-67);
//      absorbing seeds cost 4 bytes, a tile with nothing to update ends here;
//   1. every active seed projects its depth interval into the current frame
//      (src/epipolar_match.cu:60-75), counts its candidates with the
//      reference's own float accumulation (checkpointing l every 16th), finds
//      the exact contiguous range of candidates inside the image, and the CTA
//      reduces the bounding box and the centroid of all search segments;
//   2. one thread issues TMA loads (cp.async.bulk.tensor.2d -> UTMALDG,
//      mbarrier complete_tx) of the reference tile (+halo) and of the strip of the
//      current frame under that bounding box into shared memory;
//   3. the seeds' candidates are cut into 4-candidate chunks, and a seed's chunks
//      into runs of up to `run` consecutive chunks (chosen per tile); the tile's
//      runs form one run-major work list and all warps take 32-item rounds of it
//      round-robin, so lanes stay busy whatever the mix of search lengths; a
//      candidate's NCC is evaluated by the same code as in the direct variant
//      (depth_filter_math.cuh) on taps from the shared-memory strip (from
//      global memory for the rare block outside it); per-seed arg-max is a
//      shared-memory 64-bit atomicMax on (ncc, -index), which reproduces the
//      reference's "first maximum wins" (epipolar_match.cu:125-129);
//   3b. a tile that was much busier than its share of the previous frame is
//      processed by up to 16 CTAs (listed next to each other), merged through
//      global atomics, the last one to arrive finalising the tile;
//   3c. a tile with at most 16 seeds to update skips staging: one warp per seed,
//      lanes = candidates, warp-shuffle arg-max;
//   4. the owner thread triangulates the best match and updates its seed
//      (src/seed_update.cu:40-121) in registers and writes it back once.
// Results are bit-identical to the direct variant (tests/test_gpu_configs.py).
#include <cudaTypedefs.h>

#include <limits.h>
#include <stdlib.h>

#include <algorithm>
#include <mutex>

#include "depth_filter.cuh"
#include "depth_filter_math.cuh"
#include "depth_filter_seed_steps.cuh"
#include "staged_maps.cuh"
#include "denoiser.cuh"

// 1: the debug timeline also counts the candidates scored from the strip and
// from global memory (slots 8, 9).  Off by default: even predicated off, the
// counters cost the search-heavy frames ~15 %.
#ifndef RMD_DEBUG_COUNTERS
#define RMD_DEBUG_COUNTERS 0
#endif

// Largest patch side whose candidates are scored two at a time (ncc_score_pair, packed_f32x2.cuh);
// tools/build_variant_lib.sh builds the A/B alternatives.
#ifndef RMD_STAGED_PAIR_MAX_PS
#define RMD_STAGED_PAIR_MAX_PS 7
#endif

namespace rmdb
{

using namespace staged;

namespace
{

template<int PS>
struct __align__(128) StagedSmem
{
  float strip[STRIP_FLOATS];
  float ref[REF_BOX_W * ref_box_h(PS)];
  SearchRec rec[NPIX];
  unsigned long long best[NPIX];
  int n_levels;                        // chunks of the tile's longest search
  int dbg[8];                          // debug build (RMD_DEBUG_COUNTERS): see the timeline slots 8.. below
  float l_checkpoint[NPIX][L_CHECKPOINTS];  // l of candidates 0, 16, 32, ... of every seed
  // tile-wide run-major work list: level c = the seeds that have a c-th run of chunks
  unsigned int level_mask[MAX_CHUNKS][TILE_H];              // ... as one ballot per pixel row
  __align__(16) unsigned short level_rowpre[MAX_CHUNKS][TILE_H];  // items of level c in the rows above
  int level_cum[MAX_CHUNKS + 4];                            // items before level c; [n_levels] = all items
  int bbox[4];       // xmin, ymin, xmax, ymax over all segments of the CTA
  int centroid[3];   // sum of x * w, y * w, w over the seeds (w = accepted candidates, x/y = middle of their range)
  int strip_ox, strip_oy, strip_w, strip_rows;
  int is_last;
  unsigned int fetch;                  // index of the work-list entry this CTA processes next (persistent loop)
  unsigned int fetch_heavy, fetch_light, fetch_sparse;  // chain mode: the frame's list sizes, read BEFORE the index was drawn
  int items_acc;                       // work items of the tile (sum of the seeds' chunk counts)
  unsigned int row_active[TILE_H];     // ballot of the seeds to update, per pixel row
  unsigned long long mbar;
};

// ------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ unsigned int smem_addr(const void *p)
{
  return (unsigned int)__cvta_generic_to_shared(p);
}

__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned int count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_addr(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned int bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
               :: "r"(smem_addr(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(unsigned long long *bar, unsigned int parity)
{
  unsigned int ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n" : "=r"(ok) : "r"(smem_addr(bar)), "r"(parity) : "memory");
  return ok != 0u;
}

// Bounded wait: a TMA that never completes (bad descriptor) must fail the
// launch, not hang the GPU.
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned int parity)
{
  for(unsigned int it = 0; !mbar_try_wait(bar, parity); ++it)
    if(it > (1u << 22)) __trap();
}

__device__ __forceinline__ void tma_load_2d(void *smem_dst, const CUtensorMap *map, int c0, int c1,
                                            unsigned long long *bar)
{
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%2, %3}], [%4];"
      :: "r"(smem_addr(smem_dst)), "l"(reinterpret_cast<unsigned long long>(map)), "r"(c0), "r"(c1),
         "r"(smem_addr(bar))
      : "memory");
}

// Texel block of a candidate inside the shared-memory strip.
struct StripTaps
{
  static constexpr bool kEdgeFirst = false;
  const float *origin;
  int stride;
  __device__ __forceinline__ StripTaps(const float *strip, int strip_w, int ox, int oy, const TapFrame &t)
    : origin(strip + (t.j0 - oy) * strip_w + (t.i0 - ox)), stride(strip_w) {}
  __device__ __forceinline__ float at(const int j, const int i) const { return origin[j * stride + i]; }
};

// A lead CTA has appended its tile's entries to the next frame's work list (or retired the tile): when
// every tile listed in THIS frame has done so, the next frame's list is complete.
__device__ __forceinline__ void signal_listed(const FilterParams &P)
{
  __threadfence();            // my entries are written before I count myself ...
  const unsigned int done = atomicAdd(P.counts_next + 5, 1u) + 1u;
  if(done == __ldcg(P.counts_cur + 4))
  {
    __threadfence();          // ... and everybody's (observed through the counter) before the list is published
    atomicMax(P.list_ready, P.frame_no + 1u);
  }
}

// Chunks per work item (run) of a staged tile, phase 3.  Longer runs pay the item's set-up less often, but
// make the warps' last rounds coarser: the run is as long as every warp of each of the tile's zeff CTAs still
// gets RUN_MIN_ROUNDS rounds of it (a function of the tile's chunk count and zeff only, hence the same in all
// CTAs of a split tile).  P.run_chunks > 0 fixes it (RMD_OPT_TUNE_RUN_CHUNKS); results never depend on it.
__device__ __forceinline__ int run_chunks(const FilterParams &P, const int items, const int zeff)
{
  if(P.run_chunks > 0)
    return P.run_chunks;
  return max(1, min(RUN_MAX_CHUNKS, items / (32 * NWARPS * RUN_MIN_ROUNDS * zeff)));
}

} // namespace


// One entry of a keyframe's work list: phases 0-4 for one tile (or one share of a split tile).
// `mbar_phase` is the parity of the CTA's TMA mbarrier, carried from tile to tile.
template<int PS>
__device__ __forceinline__ void process_tile(const FilterParams &P, const StagedTensorMaps &M, StagedSmem<PS> &S,
                                             const unsigned int entry, unsigned int &mbar_phase,
                                             const bool chain, const bool wait_prev, unsigned int *error_flag)
{
  const int lane = threadIdx.x, wid = threadIdx.y;   // warp `wid` owns pixel row `wid` of the tile
  const int tid = wid * TILE_W + lane;
  const int pix = tid;
  // entry = tile | share << 20 | zeff << 26.  A tile that was much busier than the per-slot average of the
  // previous frame is listed zeff times -- its lead CTA and zeff - 1 helpers, each taking every zeff-th round
  // of its work list (once most seeds have converged a frame's duration is bounded below by its busiest
  // tile, up to 9216 items).
  const int tile = (int)(entry & 0xfffffu);
  const int z = (int)((entry >> 20) & 0x3fu);
  const int zeff = (int)(entry >> 26);
  const int x0 = (tile % P.tiles_x) * TILE_W, y0 = (tile / P.tiles_x) * TILE_H;
  const int x = x0 + lane, y = y0 + wid;
  const bool lead = (z == 0);  // the CTA that records what all of them compute identically
  if(wait_prev)
  {
    // chain mode, not the launch's first frame: this tile's seeds are final once the previous frame's
    // finaliser has released them (pixels never interact: frame f of a tile depends on frame f-1 of that tile only)
    if(tid == 0 && !wait_at_least(P.tile_done + tile, P.frame_no - 1u))
      atomicExch(error_flag, 1u);
    __syncthreads();
  }

  // debug timeline (RMD_OPT_DEBUG_TIMELINE), lead CTA only:
  // [0] globaltimer ns at start, [1..4] SM cycles since start after classification /
  // search set-up / TMA arrival / NCC search, [5] globaltimer ns at the end,
  // [6] SM id, [7] work items of the tile, [8] candidates scored from the strip,
  // [9] ... from global memory, [10] bounding box w | h << 16, [11] strip w | rows << 16,
  // [12] seeds to update, [13] zeff | sparse << 8
  long long *const stamps = (P.timeline && lead) ? P.timeline + 16 * (size_t)tile : nullptr;
  const long long stamp_t0 = stamps ? clock64() : 0;
#define RMD_STAMP(i) do { if(stamps && tid == 0) { if((i) == 5) { long long gt_; \
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt_)); stamps[5] = gt_; } \
    else stamps[i] = clock64() - stamp_t0; } } while(0)
  if(stamps && tid == 0)
  {
    unsigned int smid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    stamps[6] = (long long)smid;
    stamps[7] = 0;
    long long gt;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
    stamps[0] = gt;
  }

  // ---- 0. classification
  bool active = false, converged = false;
  int prev = RMD_BORDER, state = RMD_BORDER;
  int *conv_ptr = nullptr;
  float4 *seed_ptr = nullptr;
  float4 seed = make_float4(0.f, 0.f, 0.f, 0.f);
  const bool inside = (x < P.width) && (y < P.height);
  if(inside)
  {
    conv_ptr = P.conv + (size_t)y * P.conv_stride + x;
    seed_ptr = P.seed + (size_t)y * P.seed_stride + x;
    // (L2 loads: in chain mode the previous frame's finaliser may have run on another SM during this launch)
    prev = __ldcg(conv_ptr);
    seed = __ldcg(seed_ptr);   // issued with the state load, not after it: one memory round trip for the tile
    state = classify_pixel<PS>(P, x, y, prev, seed, active);
    converged = (state == RMD_CONVERGED);
    if(lead && !active && state != prev)
      *conv_ptr = state;
  }
  if(tid == 0)
  {
    S.bbox[0] = INT_MAX; S.bbox[1] = INT_MAX; S.bbox[2] = INT_MIN; S.bbox[3] = INT_MIN;
    S.items_acc = 0;
    S.n_levels = 0;
    for(int i = 0; i < 8; ++i) S.dbg[i] = 0;
    S.centroid[0] = 0; S.centroid[1] = 0; S.centroid[2] = 0;
  }
  const unsigned int conv_ballot = __ballot_sync(0xffffffffu, converged);
  const int n_active = __syncthreads_count(active);
  if(n_active == 0)
  {
    // Nothing to search.  If, moreover, every seed is in an absorbing state the
    // tile is finished for good: it leaves the work list and its converged
    // seeds are counted once in the retired total instead of every frame.
    const bool pending = inside && !(state == RMD_BORDER || state == RMD_CONVERGED || state == RMD_DIVERGED);
    const int any_pending = __syncthreads_or(pending);
    if(lead)
    {
      if(lane == 0 && conv_ballot)
        atomicAdd(any_pending ? P.converged_now : P.retired_converged, (unsigned int)__popc(conv_ballot));
      if(tid == 0 && any_pending)
      {
        if(P.warp_tile_max_seeds > 0)
          P.sparse_next[atomicAdd(P.counts_next + 6, 1u)] = (unsigned int)tile;     // nothing to update now: cheapest class
        else
          P.light_next[atomicAdd(P.counts_next + 1, 1u)] = (unsigned int)tile | (1u << 26);
        atomicAdd(P.counts_next + 4, 1u);
      }
      if(chain)
      {
        if(tid == 0)
          signal_listed(P);
        // the state changes written above (conv of newly absorbing seeds) are visible before the tile is
        // released: CTA barrier, then ONE cumulative gpu-scope fence + release by the signalling thread
        __syncthreads();
        if(tid == 0)
        {
          __threadfence();
          st_release(P.tile_done + tile, P.frame_no);
        }
      }
    }
    if(stamps && tid == 0) stamps[1] = -(clock64() - stamp_t0);
    return;
  }
  if(lead && lane == 0 && conv_ballot)
    atomicAdd(P.converged_now, (unsigned int)__popc(conv_ballot));
  RMD_STAMP(1);

  // ---- 1. search segments, candidate counts, bounding box
  EpiSegment seg;
  seg.mean = make_float2(0.f, 0.f); seg.dir = make_float2(0.f, 0.f); seg.half_len = 0.f;
  int n_cand = 0, k_lo = INT_MAX, k_hi = -1;  // candidates, first / last one inside the image
  int bx_lo = INT_MAX, by_lo = INT_MAX, bx_hi = INT_MIN, by_hi = INT_MIN;
  if(active)
  {
    const float2 stats = __ldg(P.templ + (size_t)y * P.templ_stride + x);
    seg = epipolar_segment(P, x, y, seed.x, seed.y);
    n_cand = count_candidates(seg.half_len, S.l_checkpoint[pix]);
    accepted_range<PS>(P, seg, n_cand, S.l_checkpoint[pix], k_lo, k_hi);
    const float ex0 = seg.mean.x - seg.half_len * seg.dir.x, ex1 = seg.mean.x + seg.half_len * seg.dir.x;
    const float ey0 = seg.mean.y - seg.half_len * seg.dir.y, ey1 = seg.mean.y + seg.half_len * seg.dir.y;
    int xl = to_int_clamped(floorf(fminf(ex0, ex1))) - (PS / 2 + 1);
    int xh = to_int_clamped(floorf(fmaxf(ex0, ex1))) + (PS / 2 + 3);
    int yl = to_int_clamped(floorf(fminf(ey0, ey1))) - (PS / 2 + 1);
    int yh = to_int_clamped(floorf(fmaxf(ey0, ey1))) + (PS / 2 + 3);
    // only the part where candidates are accepted matters (epipolar_match.cu:91-97)
    xl = max(xl, PS - PS / 2 - 1); yl = max(yl, PS - PS / 2 - 1);
    xh = min(xh, P.width - 1);     yh = min(yh, P.height - 1);
    if(k_hi >= 0 && xl <= xh && yl <= yh)
    {
      bx_lo = xl; bx_hi = xh; by_lo = yl; by_hi = yh;
    }
    SearchRec r;
    r.mean_x = seg.mean.x; r.mean_y = seg.mean.y; r.dir_x = seg.dir.x; r.dir_y = seg.dir.y;
    r.half_len = seg.half_len; r.sum_templ = stats.x; r.denom = stats.y;
    r.n = (k_hi >= 0) ? (k_lo | (k_hi << 8) | (1 << 16)) : 0;  // accepted candidate range, packed
    S.rec[pix] = r;
  }
  const unsigned long long kNoMatch = K_NO_MATCH;
  S.best[pix] = kNoMatch;
  const int m_chunks = (k_hi >= 0) ? (k_hi / CHUNK - k_lo / CHUNK + 1) : 0;  // chunks with accepted candidates
  {
    const unsigned int act = __ballot_sync(0xffffffffu, active);
    const int m_row = __reduce_add_sync(0xffffffffu, m_chunks);
    const int m_max = __reduce_max_sync(0xffffffffu, m_chunks);
    if(lane == 0)
    {
      S.row_active[wid] = act;
      if(m_row)
      {
        atomicAdd(&S.items_acc, m_row);
        atomicMax(&S.n_levels, m_max);
      }
    }
  }
  bx_lo = __reduce_min_sync(0xffffffffu, bx_lo); by_lo = __reduce_min_sync(0xffffffffu, by_lo);
  bx_hi = __reduce_max_sync(0xffffffffu, bx_hi); by_hi = __reduce_max_sync(0xffffffffu, by_hi);
  if(lane == 0 && bx_lo <= bx_hi)
  {
    atomicMin(&S.bbox[0], bx_lo); atomicMin(&S.bbox[1], by_lo);
    atomicMax(&S.bbox[2], bx_hi); atomicMax(&S.bbox[3], by_hi);
  }
  {
    // where the candidates are, for the strip placement when the box is larger than the strip
    int w = 0, wx = 0, wy = 0;
    if(k_hi >= 0)
    {
      w = k_hi - k_lo + 1;
      const float l_mid = -seg.half_len + RMD_EPIPOLAR_STEP * 0.5f * (float)(k_lo + k_hi);
      wx = w * to_int_clamped(seg.mean.x + l_mid * seg.dir.x);
      wy = w * to_int_clamped(seg.mean.y + l_mid * seg.dir.y);
    }
    w = __reduce_add_sync(0xffffffffu, w);
    wx = __reduce_add_sync(0xffffffffu, wx);
    wy = __reduce_add_sync(0xffffffffu, wy);
    if(lane == 0 && w > 0)
    {
      atomicAdd(&S.centroid[0], wx); atomicAdd(&S.centroid[1], wy); atomicAdd(&S.centroid[2], w);
    }
  }
  __syncthreads();

  RMD_STAMP(2);
  if(lead && tid == 0)
  {
    // this tile's entries in the NEXT frame's work list
    const int items = S.items_acc;
    atomicAdd(P.counts_next + 3, (unsigned int)items);
    atomicAdd(P.counts_next + 7, (unsigned int)n_active);   // seeds updated in this frame (host: when to go seed-major)
    const unsigned int frame_items = __ldcg(P.counts_cur + 3);   // (chain mode: still growing -- a heuristic input only)
    const unsigned int avg_per_slot = frame_items / (unsigned int)P.cta_slots;
    // CTAs in proportion to the tile's share of the frame: about one resident-CTA
    // slot's worth of items each (never fewer than split_items_per_cta, the fixed
    // cost of a CTA must pay off), so the frame's CTAs finish together and the sum
    // of all helpers stays below the number of slots.
    // (no estimate of the frame's total in the first frame of a keyframe: no split)
    int znext = 1;
    if(P.split_max > 1 && items > P.split_min_items && frame_items != 0u)
    {
      const unsigned int target = max((unsigned int)P.split_items_per_cta, avg_per_slot * (unsigned int)P.split_avg_pct / 100u);
      znext = (int)min((unsigned int)P.split_max, ((unsigned int)items + target - 1u) / target);
    }
    if(znext > 1)
    {
      const int reserved = (int)atomicAdd(P.counts_next + 2, (unsigned int)(znext - 1));
      znext = 1 + max(0, min(znext - 1, P.helper_cap - reserved));   // what fits in the list
    }
    if(znext == 1 && n_active <= P.warp_tile_max_seeds && S.centroid[2] <= P.warp_tile_max_cands)
    {
      P.sparse_next[atomicAdd(P.counts_next + 6, 1u)] = (unsigned int)tile;   // a handful of seeds, a few dozen candidates
    }
    else if(znext > 1 || items >= P.heavy_min_items)
    {
      const unsigned int base = atomicAdd(P.counts_next + 0, (unsigned int)znext);
      for(int k = 0; k < znext; ++k)
        P.heavy_next[base + k] = (unsigned int)tile | ((unsigned int)k << 20) | ((unsigned int)znext << 26);
    }
    else
    {
      P.light_next[atomicAdd(P.counts_next + 1, 1u)] = (unsigned int)tile | (1u << 26);
    }
    atomicAdd(P.counts_next + 4, 1u);
    if(chain)
      signal_listed(P);
    if(stamps) { stamps[7] = S.items_acc; stamps[12] = n_active; }
  }

  // ---- sparse tile (the common case once most seeds have converged): a handful
  // of seeds does not pay for a TMA round trip and a CTA-wide work list.  One
  // warp per seed, lanes = candidates, taps straight from global memory (L2),
  // arg-max with warp shuffles on the same (ncc, -index) key.
  const bool sparse = (n_active <= P.sparse_max_seeds) && (zeff == 1);
  if(stamps && tid == 0) stamps[13] = zeff | (sparse ? 256 : 0);
  if(sparse)
  {
    int seen = 0;
    for(int r = 0; r < TILE_H; ++r)
    {
      unsigned int mask = S.row_active[r];
      while(mask)
      {
        const int src = __ffs(mask) - 1;
        mask &= mask - 1;
        if((seen++ % NWARPS) != wid)
          continue;
        const SearchRec R = S.rec[r * TILE_W + src];
        unsigned long long key = kNoMatch;
        if(R.n >> 16)
        {
          const int ka = R.n & 0xff, kb = (R.n >> 8) & 0xff;
          float templ[PS * PS];
#pragma unroll
          for(int j = 0; j < PS; ++j)
#pragma unroll
            for(int i = 0; i < PS; ++i)
              templ[j * PS + i] = __ldg(P.ref + (size_t)(y0 + r - PS / 2 + j) * P.ref_stride + (x0 + src - PS / 2 + i));
          float best_ncc = -1.0f;
          int best_idx = 0;
#pragma unroll 1
          for(int k = ka + lane; k <= kb; k += 32)
          {
            float l = S.l_checkpoint[r * TILE_W + src][k / L_CHECKPOINT_STEP];
            for(int t = 0; t < (k & (L_CHECKPOINT_STEP - 1)); ++t) l += RMD_EPIPOLAR_STEP;
            const float2 px = candidate_px(R.mean_x, R.mean_y, R.dir_x, R.dir_y, l);
            if(candidate_rejected<PS>(px, P.width, P.height))
              continue;
            const TapFrame frame = tap_frame<PS>(px, P.tex_quant);
            const GlobalTaps taps(P.curr, P.curr_stride, frame);
            const float ncc = ncc_score<PS>(taps, frame, templ, R.sum_templ, R.denom);
            if(ncc > best_ncc)
            {
              best_ncc = ncc;
              best_idx = k;
            }
          }
          if(best_ncc > -1.0f)
            key = (((unsigned long long)orderable(best_ncc)) << 32) |
                  (unsigned long long)(0xffffffffu - (unsigned int)best_idx);
        }
#pragma unroll
        for(int off = 16; off > 0; off >>= 1)
        {
          const unsigned long long other = __shfl_xor_sync(0xffffffffu, key, off);
          key = (other > key) ? other : key;
        }
        if(lane == 0)
          S.best[r * TILE_W + src] = key;
      }
    }
    __syncthreads();
    RMD_STAMP(3);
    RMD_STAMP(4);
  }
  else
  {
  // ---- 2. TMA: reference tile and current-image strip -> shared memory
  if(tid == 0)
  {
    const int xmin = S.bbox[0], ymin = S.bbox[1], xmax = S.bbox[2], ymax = S.bbox[3];
    int ox = 0, oy = 0, sw = 0, rows = 0, wi = 0;
    if(xmin <= xmax && ymin <= ymax)
    {
      // A TMA box must start at a 16-byte aligned global address:
      // box origins are multiples of 4 floats.
      const int xmin_a = xmin & ~3;
      const int bw = xmax - xmin_a + 1, bh = ymax - ymin + 1;
      wi = NUM_WIDTHS - 1;
#pragma unroll
      for(int i = NUM_WIDTHS - 1; i >= 0; --i)
        if(strip_width(i) >= bw) wi = i;
      sw = strip_width(wi);
      const int max_rows = (STRIP_FLOATS / sw) / STRIP_BOX_ROWS * STRIP_BOX_ROWS;
      const int want_rows = (bh + STRIP_BOX_ROWS - 1) / STRIP_BOX_ROWS * STRIP_BOX_ROWS;
      rows = min(want_rows, max_rows);
      // a box larger than the strip: centre the strip on the candidates' centroid
      // (a few outliers stretch the box, most candidates cluster), inside the box
      const int cw = max(1, S.centroid[2]);
      const int cx = S.centroid[0] / cw, cy = S.centroid[1] / cw;
      ox = (bw <= sw) ? xmin_a : (min(max(cx - sw / 2, xmin_a), xmax + 1 - sw + 3) & ~3);
      oy = (want_rows <= max_rows) ? ymin : min(max(cy - rows / 2, ymin), ymax + 1 - rows);
    }
    S.strip_ox = ox; S.strip_oy = oy; S.strip_w = sw; S.strip_rows = rows;
    if(stamps)
    {
      stamps[10] = (long long)max(0, xmax - xmin + 1) | ((long long)max(0, ymax - ymin + 1) << 16);
      stamps[11] = (long long)sw | ((long long)rows << 16);
    }
    const unsigned int ref_bytes = REF_BOX_W * ref_box_h(PS) * (unsigned int)sizeof(float);
    mbar_expect_tx(&S.mbar, ref_bytes + (unsigned int)(rows * sw) * (unsigned int)sizeof(float));
    tma_load_2d(S.ref, &M.ref, x0 - REF_ORIGIN_X, y0 - PS / 2, &S.mbar);
    const CUtensorMap *cm = &M.curr[wi];
    for(int r = 0; r < rows; r += STRIP_BOX_ROWS)
      tma_load_2d(S.strip + r * sw, cm, ox, oy + r, &S.mbar);
  }

  // ---- 3. balanced NCC search: one run-major work list for the whole tile
  // A seed's chunks are cut into runs of `run` consecutive chunks (the last one
  // may be shorter); an item is one run, so the item's set-up (list lookup,
  // record, template, restart of l from its checkpoint, arg-max atomic) is paid
  // once per run instead of once per chunk.  Level c of the list = all seeds of
  // the tile that still have a c-th run, in pixel order; item q belongs to
  // level c = max{c : cum[c] <= q}, and is the (q - cum[c])-th such seed.
  // Lanes of a round therefore work on neighbouring pixels' candidates, every
  // round but the last is full, and a round costs about the same whatever the
  // mix of search lengths in the tile.  `run` is the same in every CTA of a
  // split tile (a function of the tile's chunk count and zeff only).
  const int run = run_chunks(P, S.items_acc, zeff);
  const int n_levels = (S.n_levels + run - 1) / run;
  {
    const int m = (m_chunks + run - 1) / run;
    for(int c = 0; c < n_levels; ++c)
    {
      const unsigned int mk = __ballot_sync(0xffffffffu, m > c);
      if(lane == 0)
      {
        S.level_mask[c][wid] = mk;
        S.level_rowpre[c][wid] = (unsigned short)__popc(mk);
      }
    }
  }
  __syncthreads();
  if(wid == 0)
  {
    // row counts -> exclusive row prefixes per level, level totals -> exclusive scan over the levels
    int tot[2];
#pragma unroll
    for(int h = 0; h < 2; ++h)
    {
      const int c = lane + 32 * h;
      int acc = 0;
      if(c < n_levels)
      {
#pragma unroll
        for(int r = 0; r < TILE_H; ++r)
        {
          const int cnt = S.level_rowpre[c][r];
          S.level_rowpre[c][r] = (unsigned short)acc;
          acc += cnt;
        }
      }
      tot[h] = acc;
    }
    int inc0 = tot[0], inc1 = tot[1];
#pragma unroll
    for(int off = 1; off < 32; off <<= 1)
    {
      const int a0 = __shfl_up_sync(0xffffffffu, inc0, off), a1 = __shfl_up_sync(0xffffffffu, inc1, off);
      if(lane >= off) { inc0 += a0; inc1 += a1; }
    }
    const int sum0 = __shfl_sync(0xffffffffu, inc0, 31);
    if(lane <= n_levels) S.level_cum[lane] = inc0 - tot[0];                  // lane == n_levels <= 31: the total
    if(lane + 32 <= n_levels) S.level_cum[lane + 32] = sum0 + inc1 - tot[1];
  }
  __syncthreads();  // publishes the work list and the strip geometry (built while the TMA is in flight)
  const int strip_ox = S.strip_ox, strip_oy = S.strip_oy, strip_w = S.strip_w, strip_rows = S.strip_rows;
  mbar_wait(&S.mbar, mbar_phase);
  mbar_phase ^= 1u;
  RMD_STAMP(3);
  // The warps of the tile's zeff CTAs take 32-item rounds of the list round-robin.
  const int total = S.level_cum[n_levels];
  for(int rho = z * NWARPS + wid; rho * 32 < total; rho += zeff * NWARPS)
  {
    const int q = rho * 32 + lane;
#if RMD_DEBUG_COUNTERS
    const long long dbg_t0 = clock64();
#endif
    if(q < total)
    {
      // largest level c with level_cum[c] <= q (level_cum[n_levels] = total > q)
      int c = 0, hi = n_levels;
#pragma unroll
      for(int step = 0; step < 6; ++step)
      {
        const int mid = (c + hi) >> 1;
        if(S.level_cum[mid] <= q) c = mid; else hi = mid;
      }
      const int rank = q - S.level_cum[c];
      // pixel row: the last one whose prefix does not exceed the rank (prefixes are non-decreasing)
      const uint4 pre = *reinterpret_cast<const uint4*>(&S.level_rowpre[c][0]);
      const int p1 = (int)(pre.x >> 16), p2 = (int)(pre.y & 0xffffu), p3 = (int)(pre.y >> 16);
      const int p4 = (int)(pre.z & 0xffffu), p5 = (int)(pre.z >> 16), p6 = (int)(pre.w & 0xffffu), p7 = (int)(pre.w >> 16);
      const int r = (p1 <= rank) + (p2 <= rank) + (p3 <= rank) + (p4 <= rank) + (p5 <= rank) + (p6 <= rank) + (p7 <= rank);
      const int before = (r == 0) ? 0 : (r == 1) ? p1 : (r == 2) ? p2 : (r == 3) ? p3 : (r == 4) ? p4 : (r == 5) ? p5 : (r == 6) ? p6 : p7;
      const int src = __fns(S.level_mask[c][r], 0, rank - before + 1);  // lane owning the seed

      const SearchRec R = S.rec[r * TILE_W + src];
      float templ[PS * PS];
#pragma unroll
      for(int j = 0; j < PS; ++j)
#pragma unroll
        for(int i = 0; i < PS; ++i)
          templ[j * PS + i] = S.ref[(r + j) * REF_BOX_W + src + i + (REF_ORIGIN_X - PS / 2)];

      // the run's chunks: c * run .. of the seed's (R.n & 0xff) / CHUNK .. (R.n >> 8 & 0xff) / CHUNK
      const int chunk_lo = (R.n & 0xff) / CHUNK, chunk_hi = ((R.n >> 8) & 0xff) / CHUNK;
      const int first = (chunk_lo + c * run) * CHUNK;
      const int n_run = min(run, chunk_hi - chunk_lo + 1 - c * run) * CHUNK;   // candidates of the run
      // l of the run's first candidate: the same float accumulation as the
      // reference's loop (epipolar_match.cu:88), so positions are bit-identical;
      // within the run l keeps accumulating the same way
      float l = S.l_checkpoint[r * TILE_W + src][first / L_CHECKPOINT_STEP];
      for(int k = 0; k < (first & (L_CHECKPOINT_STEP - 1)); ++k) l += RMD_EPIPOLAR_STEP;

      float best_ncc = -1.0f;
      int best_idx = 0;
#if RMD_DEBUG_COUNTERS
      const long long dbg_t1 = clock64();
#endif
      // Two candidates per pass: when both lie in the strip their texel blocks are filtered together with
      // paired operations (ncc_score_pair); otherwise each goes the scalar way (strip or global taps).
      // l advances by the reference's own float accumulation either way.
      static_assert(CHUNK % 2 == 0, "candidates are taken two at a time");
      constexpr bool kPair = (PS <= RMD_STAGED_PAIR_MAX_PS);
#pragma unroll 1
      for(int i = 0; i < n_run; i += 2)
      {
        const float l0 = l;
        l += RMD_EPIPOLAR_STEP;
        const float l1 = l;
        l += RMD_EPIPOLAR_STEP;
        if(!(l0 <= R.half_len)) break;
        const float2 px0 = candidate_px(R.mean_x, R.mean_y, R.dir_x, R.dir_y, l0);
        const float2 px1 = candidate_px(R.mean_x, R.mean_y, R.dir_x, R.dir_y, l1);
        const bool use0 = !candidate_rejected<PS>(px0, P.width, P.height);
        const bool use1 = (l1 <= R.half_len) && !candidate_rejected<PS>(px1, P.width, P.height);
        const TapFrame frame0 = tap_frame<PS>(px0, P.tex_quant);
        const TapFrame frame1 = tap_frame<PS>(px1, P.tex_quant);
        const bool in0 = (frame0.i0 >= strip_ox) && (frame0.i0 + PS < strip_ox + strip_w) &&
                         (frame0.j0 >= strip_oy) && (frame0.j0 + PS < strip_oy + strip_rows);
        const bool in1 = (frame1.i0 >= strip_ox) && (frame1.i0 + PS < strip_ox + strip_w) &&
                         (frame1.j0 >= strip_oy) && (frame1.j0 + PS < strip_oy + strip_rows);
        float ncc0 = -2.0f, ncc1 = -2.0f;     // below every score: a skipped candidate never wins
#if RMD_DEBUG_COUNTERS
        if(P.timeline)
        {
          if(use0) atomicAdd(&S.dbg[in0 ? 0 : 1], 1);              // candidates (lanes)
          if(use1) atomicAdd(&S.dbg[in1 ? 0 : 1], 1);
          const unsigned int am = __activemask();
          if(lane == __ffs(am) - 1) atomicAdd(&S.dbg[(in0 && in1) ? 2 : 3], 1);  // warp-level executions of each path
        }
#endif
        if(!use0 && !use1)
          continue;
        // both usable candidates in the strip (a lone one is paired with itself): packed; otherwise both from global memory
        if(kPair && (in0 || !use0) && (in1 || !use1))
        {
          const TapFrame fa = use0 ? frame0 : frame1, fb = use1 ? frame1 : frame0;
          const StripTaps taps_a(S.strip, strip_w, strip_ox, strip_oy, fa);
          const StripTaps taps_b(S.strip, strip_w, strip_ox, strip_oy, fb);
          const float2 both = ncc_score_pair<PS>(taps_a, fa, taps_b, fb, templ, R.sum_templ, R.denom);
          if(use0) ncc0 = both.x;
          if(use1) ncc1 = both.y;
        }
        else
        {
#pragma unroll 1
          for(int h = 0; h < 2; ++h)
          {
            if(!(h == 0 ? use0 : use1))
              continue;
            const TapFrame frame = (h == 0) ? frame0 : frame1;
            float ncc;
            if(!kPair && (h == 0 ? in0 : in1))
            {
              const StripTaps taps(S.strip, strip_w, strip_ox, strip_oy, frame);
              ncc = ncc_score<PS>(taps, frame, templ, R.sum_templ, R.denom);
            }
            else
            {
              const GlobalTaps taps(P.curr, P.curr_stride, frame);
              ncc = ncc_score<PS>(taps, frame, templ, R.sum_templ, R.denom);
            }
            if(h == 0) ncc0 = ncc; else ncc1 = ncc;
          }
        }
        if(ncc0 > best_ncc)
        {
          best_ncc = ncc0;
          best_idx = first + i;
        }
        if(ncc1 > best_ncc)
        {
          best_ncc = ncc1;
          best_idx = first + i + 1;
        }
      }
      if(best_ncc > -1.0f)
      {
        const unsigned long long key =
            (((unsigned long long)orderable(best_ncc)) << 32) | (unsigned long long)(0xffffffffu - (unsigned int)best_idx);
        atomicMax(&S.best[r * TILE_W + src], key);
      }
#if RMD_DEBUG_COUNTERS
      if(P.timeline && q == rho * 32)
      {
        const long long t2 = clock64();
        atomicAdd(&S.dbg[4], (int)(dbg_t1 - dbg_t0));   // item decode: list lookup, record, template
        atomicAdd(&S.dbg[5], (int)(t2 - dbg_t1));       // the item's candidates (first lane of the round)
        atomicAdd(&S.dbg[6], 1);                        // rounds
      }
#endif
    }
  }
  __syncthreads();
  RMD_STAMP(4);
  // debug build: [8] candidates from the strip, [9] from global memory, [14] decode cycles | rounds << 40,
  // [15] candidate cycles of the rounds' first lanes, [13] also warp-level strip passes << 16 | global passes << 40
  if(stamps && tid == 0)
  {
    stamps[8] = S.dbg[0]; stamps[9] = S.dbg[1];
    stamps[14] = (long long)S.dbg[4] | ((long long)S.dbg[6] << 40);
    stamps[15] = S.dbg[5];
    stamps[13] |= ((long long)S.dbg[2] << 16) | ((long long)S.dbg[3] << 40);
  }
  }  // staged (non-sparse) path

  // ---- 3b. a split tile: merge the partial arg-max of its CTAs in global
  // memory; the last CTA to arrive finalises the tile (and leaves the keys and
  // the arrival counter reset for the next frame).
  unsigned long long key = S.best[pix];
  if(zeff > 1)
  {
    unsigned long long *gkey = P.tile_keys + (size_t)tile * NPIX + pix;
    if(key != kNoMatch)
      atomicMax(gkey, key);
    __threadfence();
    __syncthreads();
    if(tid == 0)
    {
      const unsigned int ticket = atomicAdd(P.tile_arrivals + tile, 1u);
      S.is_last = (ticket == (unsigned int)(zeff - 1)) ? 1 : 0;
      if(S.is_last)
        P.tile_arrivals[tile] = 0u;
    }
    __syncthreads();
    if(!S.is_last)
      return;
    __threadfence();
    key = atomicExch(gkey, kNoMatch);
  }

  // ---- 4. triangulation + Bayesian update by the owner of the seed
  if(active)
    apply_match<PS>(P, x, y, seg, n_cand, key, S.l_checkpoint[pix], seed, seed_ptr, prev, conv_ptr);
  if(chain)
  {
    // seeds and states of this frame are visible before the next frame may read them (barrier, then one
    // cumulative gpu-scope fence + release: a fence per thread would invalidate L1 256 times per tile)
    __syncthreads();
    if(tid == 0)
    {
      __threadfence();
      st_release(P.tile_done + tile, P.frame_no);
    }
  }
  RMD_STAMP(5);
}
#undef RMD_STAMP

// ------------------------------------------------------------------------------------------------ warp tiles
// Late in a keyframe two thirds of the listed tiles have a handful of seeds left to update and a few dozen
// candidates in all.  A 256-thread CTA with 64 KB of shared memory per such tile is mostly idle warps holding a
// resident slot: here ONE WARP does the whole tile (eight tiles per CTA pass), so the slots go to the tiles that
// need them and several keyframes' (or frames') sparse tiles pack eight to a CTA.  Same per-seed steps as the CTA
// path (classify_pixel, epipolar_segment, count_candidates, accepted_range, ncc_score, apply_match), hence the
// same results: lanes = the tile's (seed, candidate) pairs, taps from global memory (L2), per-seed arg-max by
// shared-memory atomicMax on the same (ncc, ~index) key.
struct alignas(16) WarpTileSmem
{
  SearchRec rec[WARP_TILE_MAX_SEEDS];
  unsigned long long best[WARP_TILE_MAX_SEEDS];
  float l_checkpoint[WARP_TILE_MAX_SEEDS][L_CHECKPOINTS];
  int cum[WARP_TILE_MAX_SEEDS];    // candidates of the batch's seeds 0..i (inclusive prefix)
  int pos[WARP_TILE_MAX_SEEDS];    // x | y << 16 of the seed
};
static_assert(sizeof(WarpTileSmem) * NWARPS <= STRIP_FLOATS * sizeof(float), "warp-tile scratch aliases the strip");

template<int PS>
__device__ __forceinline__ void process_warp_tile(const FilterParams &P, StagedSmem<PS> &S, const unsigned int entry,
                                                  const bool chain, const bool wait_prev, unsigned int *error_flag)
{
  const int lane = threadIdx.x, wid = threadIdx.y;
  WarpTileSmem &Wt = reinterpret_cast<WarpTileSmem*>(S.strip)[wid];
  const int tile = (int)(entry & 0xfffffu);
  const int x0 = (tile % P.tiles_x) * TILE_W, y0 = (tile / P.tiles_x) * TILE_H;
  const int x = x0 + lane;
  if(wait_prev)
  {
    if(lane == 0 && !wait_at_least(P.tile_done + tile, P.frame_no - 1u))
      atomicExch(error_flag, 1u);
    __syncwarp();
  }
  // ---- 0. classification of the tile's 8 rows (lane = column)
  unsigned int act[TILE_H];
  int n_conv = 0;
  unsigned int pending_any = 0u;
#pragma unroll
  for(int r = 0; r < TILE_H; ++r)
  {
    const int y = y0 + r;
    const bool inside = (x < P.width) && (y < P.height);
    bool active = false;
    int state = RMD_BORDER;
    if(inside)
    {
      int *conv_ptr = P.conv + (size_t)y * P.conv_stride + x;
      const int prev = __ldcg(conv_ptr);
      const float4 seed = __ldcg(P.seed + (size_t)y * P.seed_stride + x);
      state = classify_pixel<PS>(P, x, y, prev, seed, active);
      if(!active && state != prev)
        *conv_ptr = state;
    }
    act[r] = __ballot_sync(0xffffffffu, active);
    n_conv += __popc(__ballot_sync(0xffffffffu, state == RMD_CONVERGED));
    pending_any |= __ballot_sync(0xffffffffu, inside && !(state == RMD_BORDER || state == RMD_CONVERGED || state == RMD_DIVERGED));
  }
  int n_act = 0;
#pragma unroll
  for(int r = 0; r < TILE_H; ++r) n_act += __popc(act[r]);
  if(n_act == 0)
  {
    if(lane == 0)
    {
      if(n_conv)
        atomicAdd(pending_any ? P.converged_now : P.retired_converged, (unsigned int)n_conv);
      if(pending_any)
      {
        P.sparse_next[atomicAdd(P.counts_next + 6, 1u)] = (unsigned int)tile;
        atomicAdd(P.counts_next + 4, 1u);
      }
      if(chain)
        signal_listed(P);
    }
    if(chain)
    {
      __syncwarp();
      if(lane == 0)
      {
        __threadfence();
        st_release(P.tile_done + tile, P.frame_no);
      }
    }
    return;
  }
  if(lane == 0 && n_conv)
    atomicAdd(P.converged_now, (unsigned int)n_conv);

  // ---- seeds to update, in pixel order, WARP_TILE_MAX_SEEDS at a time (one batch unless the list was stale)
  int items = 0, total_cands = 0;
  for(int base = 0; base < n_act; base += WARP_TILE_MAX_SEEDS)
  {
    const int slot = lane - base;
    const bool mine = (slot >= 0) && (slot < WARP_TILE_MAX_SEEDS) && (lane < n_act);
    // my seed: the lane-th set bit of act[0..7]
    int sx = 0, sy = 0;
    {
      int acc = 0, found = 0;
#pragma unroll
      for(int r = 0; r < TILE_H; ++r)
      {
        const int cnt = __popc(act[r]);
        if(!found && lane < acc + cnt)
        {
          sy = y0 + r;
          sx = x0 + (int)__fns(act[r], 0, lane - acc + 1);
          found = 1;
        }
        acc += cnt;
      }
    }
    // ---- 1. set-up by the seed's lane
    EpiSegment seg;
    seg.mean = make_float2(0.f, 0.f); seg.dir = make_float2(0.f, 0.f); seg.half_len = 0.f;
    float4 seed = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 *seed_ptr = nullptr;
    int *conv_ptr = nullptr;
    int prev = RMD_UPDATE, n_cand = 0, k_lo = INT_MAX, k_hi = -1, cnt = 0;
    if(mine)
    {
      seed_ptr = P.seed + (size_t)sy * P.seed_stride + sx;
      conv_ptr = P.conv + (size_t)sy * P.conv_stride + sx;
      seed = __ldcg(seed_ptr);
      prev = __ldcg(conv_ptr);
      const float2 stats = __ldg(P.templ + (size_t)sy * P.templ_stride + sx);
      seg = epipolar_segment(P, sx, sy, seed.x, seed.y);
      n_cand = count_candidates(seg.half_len, Wt.l_checkpoint[slot]);
      accepted_range<PS>(P, seg, n_cand, Wt.l_checkpoint[slot], k_lo, k_hi);
      cnt = (k_hi >= 0) ? (k_hi - k_lo + 1) : 0;
      SearchRec rec;
      rec.mean_x = seg.mean.x; rec.mean_y = seg.mean.y; rec.dir_x = seg.dir.x; rec.dir_y = seg.dir.y;
      rec.half_len = seg.half_len; rec.sum_templ = stats.x; rec.denom = stats.y;
      rec.n = (k_hi >= 0) ? k_lo : 0;
      Wt.rec[slot] = rec;
      Wt.best[slot] = K_NO_MATCH;
      Wt.pos[slot] = sx | (sy << 16);
      items += (k_hi >= 0) ? (k_hi / CHUNK - k_lo / CHUNK + 1) : 0;
    }
    // inclusive prefix of the batch's candidate counts (lanes base .. base+7)
    {
      int inc = mine ? cnt : 0;
#pragma unroll
      for(int off = 1; off < WARP_TILE_MAX_SEEDS; off <<= 1)
      {
        const int up = __shfl_up_sync(0xffffffffu, inc, off);
        if(slot >= off) inc += up;
      }
      if(slot >= 0 && slot < WARP_TILE_MAX_SEEDS)
        Wt.cum[slot] = inc;     // lanes past n_act carry the running total: cum[] is non-decreasing over all 8 slots
    }
    __syncwarp();
    const int batch_cands = Wt.cum[WARP_TILE_MAX_SEEDS - 1];
    total_cands += batch_cands;
    // ---- 3. NCC search: lane = (seed, candidate) pair of the batch
#pragma unroll 1
    for(int q = lane; q < batch_cands; q += 32)
    {
      int j = 0;
#pragma unroll
      for(int i = 0; i < WARP_TILE_MAX_SEEDS - 1; ++i) j += (Wt.cum[i] <= q) ? 1 : 0;
      const SearchRec R = Wt.rec[j];
      const int k = R.n + q - (j ? Wt.cum[j - 1] : 0);
      const int px0 = Wt.pos[j] & 0xffff, py0 = Wt.pos[j] >> 16;
      const float l = candidate_l(Wt.l_checkpoint[j], k);
      const float2 px = candidate_px(R.mean_x, R.mean_y, R.dir_x, R.dir_y, l);
      if(candidate_rejected<PS>(px, P.width, P.height))
        continue;
      float templ[PS * PS];
#pragma unroll
      for(int jj = 0; jj < PS; ++jj)
#pragma unroll
        for(int ii = 0; ii < PS; ++ii)
          templ[jj * PS + ii] = __ldg(P.ref + (size_t)(py0 - PS / 2 + jj) * P.ref_stride + (px0 - PS / 2 + ii));
      const TapFrame frame = tap_frame<PS>(px, P.tex_quant);
      const GlobalTaps taps(P.curr, P.curr_stride, frame);
      const float ncc = ncc_score<PS>(taps, frame, templ, R.sum_templ, R.denom);
      if(ncc > -1.0f)
        atomicMax(&Wt.best[j], (((unsigned long long)orderable(ncc)) << 32) |
                                   (unsigned long long)(0xffffffffu - (unsigned int)k));
    }
    __syncwarp();
    // ---- 4. update by the seed's lane
    if(mine)
      apply_match<PS>(P, sx, sy, seg, n_cand, Wt.best[slot], Wt.l_checkpoint[slot], seed, seed_ptr, prev, conv_ptr);
    __syncwarp();
  }
  items = __reduce_add_sync(0xffffffffu, items);
  // ---- this tile's entry in the NEXT frame's work list
  if(lane == 0)
  {
    atomicAdd(P.counts_next + 3, (unsigned int)items);
    atomicAdd(P.counts_next + 7, (unsigned int)n_act);
    if(n_act <= P.warp_tile_max_seeds && total_cands <= P.warp_tile_max_cands)
      P.sparse_next[atomicAdd(P.counts_next + 6, 1u)] = (unsigned int)tile;
    else if(items >= P.heavy_min_items)
      P.heavy_next[atomicAdd(P.counts_next + 0, 1u)] = (unsigned int)tile | (1u << 26);
    else
      P.light_next[atomicAdd(P.counts_next + 1, 1u)] = (unsigned int)tile | (1u << 26);
    atomicAdd(P.counts_next + 4, 1u);
    if(chain)
      signal_listed(P);
  }
  if(chain)
  {
    __syncwarp();
    if(lane == 0)
    {
      __threadfence();
      st_release(P.tile_done + tile, P.frame_no);
    }
  }
}

// The launch: a persistent grid (one CTA per resident slot).  Every CTA pulls entries of the frame's work
// list(s) through one cursor until they run out, so a frame costs one wave however many tiles it lists:
// no empty CTAs (the list's capacity is tiles + 1024 entries, of which a steady frame uses a third), no wave
// transition, and the busy tiles -- listed first -- are still started first.  The lead CTAs of the PREVIOUS
// frame wrote this frame's lists: tiles that were busy come first (a frame ends when its slowest CTA does),
// a tile that was much busier than the per-slot average is listed zeff times (3b), light tiles follow; tiles
// with nothing left to update, ever, are not listed.  K > 1: the lists of up to K keyframes (independent
// reference views updated by the same incoming frame) are concatenated -- all heavy lists, then all light
// lists -- so the dependent chains of different keyframes interleave from the first cycle.
// MB = CTAs per SM the register budget is sized for.  The 5x5 kernel exists as 3 x 256 threads x 80 registers
// (24 warps per SM: more issue slots covered when every seed searches its full range) and as 2 x 256 x 128
// (no spills, shorter dependent chains: faster when a frame is the critical path of a few CTAs); the host picks
// per launch (RMD_OPT_TUNE_CTAS_PER_SM, c_api.cu).  The 7x7 kernel needs 128 registers.
template<int PS, int K, int MB>
__global__ void __launch_bounds__(NTHREADS, MB) depth_filter_staged_kernel(
    const __grid_constant__ StagedBatch<K> B)
{
  extern __shared__ unsigned char smem_raw[];
  // 128-byte alignment for the TMA destinations, derived as an offset from
  // smem_raw so that the compiler keeps the shared address space (LDS/STS).
  const unsigned int smem_pad = (128u - (smem_addr(smem_raw) & 127u)) & 127u;
  StagedSmem<PS> &S = *reinterpret_cast<StagedSmem<PS>*>(smem_raw + smem_pad);

  // Launched with programmatic stream serialisation: this grid may be set up
  // while the previous frame's kernel drains; nothing may be read before that
  // kernel has completed and flushed (a no-op for an ordinary launch).
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int n_kf = (K == 1) ? 1 : B.n;
  const int tid = threadIdx.y * TILE_W + threadIdx.x;
  if(blockIdx.x == 0 && tid == 0 && !((K > 1) && (B.chain != 0)))
  {
    for(int k = 0; k < n_kf; ++k)
    {
      const FilterParams &P = B.p[K == 1 ? 0 : k];
      *P.converged_next = 0u;
#pragma unroll
      for(int w = 0; w < 8; ++w) P.counts_zero[w] = 0u;
    }
  }
  if(tid == 0)
    mbar_init(&S.mbar, 1);
  unsigned int mbar_phase = 0u;
  const bool chain = (K > 1) && (B.chain != 0);
  unsigned int *const error_flag = B.cursor + STAGED_BATCH_MAX + 1;
  int g = 0;           // chain mode: frame of the launch this CTA is working on
  for(;;)
  {
    if(tid == 0)
    {
      if(chain)
      {
        const FilterParams &P = B.p[K == 1 ? 0 : g];
        // frame g's work list is written by the lead CTAs of frame g-1, in this launch
        if(g > 0 && !wait_at_least(P.list_ready, P.frame_no))
          atomicExch(error_flag, 1u);
        // The sizes are read BEFORE the index is drawn: the slot is recycled (zeroed) by the first CTA
        // that finds this frame's cursor exhausted, i.e. after every valid index has been drawn.
        S.fetch_heavy = __ldcg(P.counts_cur + 0);
        S.fetch_light = __ldcg(P.counts_cur + 1);
        S.fetch_sparse = __ldcg(P.counts_cur + 6);
        __threadfence();
      }
      S.fetch = atomicAdd(B.cursor + (chain ? g : 0), 1u);
    }
    __syncthreads();   // also: everybody is done with the previous tile's shared memory (and sees the mbarrier)
    const unsigned int i = S.fetch;
    int kf = -1;
    unsigned int entry = 0u;
    int sparse_group = -1;           // >= 0: the index is a group of 8 warp tiles (one per warp) of keyframe / frame kf
    unsigned int n_sparse = 0u;
    if(chain)
    {
      const FilterParams &P = B.p[K == 1 ? 0 : g];
      const unsigned int n_heavy = S.fetch_heavy, n_light = S.fetch_light;
      n_sparse = S.fetch_sparse;
      if(i < n_heavy) { kf = g; entry = __ldcg(P.heavy_cur + i); }
      else if(i - n_heavy < n_light) { kf = g; entry = __ldcg(P.light_cur + (i - n_heavy)); }
      else if(i - n_heavy - n_light < (n_sparse + NWARPS - 1) / NWARPS) { kf = g; sparse_group = (int)(i - n_heavy - n_light); }
      if(i == 0u && tid == 0)
      {
        // whoever starts a frame clears what the NEXT frame will accumulate into (nobody uses those slots
        // any more: their last readers were the lead CTAs of frame g-1, which all finished listing before
        // this frame's list was complete)
        *P.converged_next = 0u;
#pragma unroll
        for(int w = 0; w < 8; ++w) P.counts_zero[w] = 0u;
        if(__ldcg(P.counts_cur + 4) == 0u)
        {
          // nothing listed (every tile has retired): no lead CTA will publish the next frame's (empty) list
          __threadfence();
          atomicMax(P.list_ready, P.frame_no + 1u);
        }
      }
      if(kf < 0)
      {
        g += 1;          // this frame's list is exhausted: on to the next one
        if(g >= n_kf)
          break;
        __syncthreads();   // S.fetch is rewritten next
        continue;
      }
    }
    else
    {
      // entry i of the concatenation: heavy lists of keyframes 0..n-1, then their light lists
      unsigned int base = 0u;
#pragma unroll 1
      for(int k = 0; k < n_kf && kf < 0; ++k)
      {
        const FilterParams &P = B.p[K == 1 ? 0 : k];
        const unsigned int n_heavy = P.counts_cur[0];
        if(i - base < n_heavy) { kf = k; entry = P.heavy_cur[i - base]; }
        base += n_heavy;
      }
#pragma unroll 1
      for(int k = 0; k < n_kf && kf < 0; ++k)
      {
        const FilterParams &P = B.p[K == 1 ? 0 : k];
        const unsigned int n_light = P.counts_cur[1];
        if(i - base < n_light) { kf = k; entry = P.light_cur[i - base]; }
        base += n_light;
      }
#pragma unroll 1
      for(int k = 0; k < n_kf && kf < 0; ++k)
      {
        const FilterParams &P = B.p[K == 1 ? 0 : k];
        const unsigned int ns = P.counts_cur[6], groups = (ns + NWARPS - 1) / NWARPS;
        if(i - base < groups) { kf = k; sparse_group = (int)(i - base); n_sparse = ns; }
        base += groups;
      }
      if(kf < 0)
        break;           // the lists are exhausted (uniform: every thread read the same index)
    }
    if(sparse_group >= 0)
    {
      const FilterParams &P = B.p[K == 1 ? 0 : kf];
      const unsigned int e = (unsigned int)sparse_group * NWARPS + threadIdx.y;
      if(e < n_sparse)
        process_warp_tile<PS>(P, S, __ldcg(P.sparse_cur + e), chain, chain && g > 0, error_flag);
    }
    else
      process_tile<PS>(B.p[K == 1 ? 0 : kf], B.m[K == 1 ? 0 : kf], S, entry, mbar_phase, chain, chain && g > 0, error_flag);
    __syncthreads();   // S.fetch and the tile's shared state are free again
  }
  // the last CTA out rewinds the cursor for the next launch (launches on a stream are ordered)
  if(tid == 0)
  {
    __threadfence();
    const unsigned int done = atomicAdd(B.cursor + STAGED_BATCH_MAX, 1u);
    if(done == gridDim.x - 1u)
    {
#pragma unroll
      for(int w = 0; w <= STAGED_BATCH_MAX; ++w) B.cursor[w] = 0u;
    }
  }
}

// ---------------------------------------------------------------- host side

StagedMaps::StagedMaps()
  : patch(0), ref_ptr(NULL), curr_ptr(NULL), ref_stride(0), curr_stride(0), width(0), height(0)
{
  memset(&maps, 0, sizeof(maps));
}

namespace
{

PFN_cuTensorMapEncodeTiled_v12000 encode_fn()
{
  static PFN_cuTensorMapEncodeTiled_v12000 fn = NULL;
  static bool tried = false;
  if(!tried)
  {
    tried = true;
    void *p = NULL;
    cudaDriverEntryPointQueryResult qres;
    if(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
       qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }
  return fn;
}

int encode_one(CUtensorMap *map, const void *base, int width, int height, int stride_floats,
               int box_w, int box_h)
{
  PFN_cuTensorMapEncodeTiled_v12000 fn = encode_fn();
  if(!fn)
    return fail(RMD_ERR_UNSUPPORTED, "cuTensorMapEncodeTiled is not available in this driver");
  const cuuint64_t dims[2] = {(cuuint64_t)width, (cuuint64_t)height};
  const cuuint64_t strides[1] = {(cuuint64_t)stride_floats * sizeof(float)};
  const cuuint32_t box[2] = {(cuuint32_t)box_w, (cuuint32_t)box_h};
  const cuuint32_t elem_strides[2] = {1, 1};
  const CUresult res = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims, strides,
                          box, elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if(res != CUDA_SUCCESS)
  {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)res));
    return RMD_ERR_INVALID_ARGUMENT;
  }
  return 0;
}

} // namespace

int encode_tensor_map_2d_f32(CUtensorMap *map, const void *base, int width, int height, int stride_floats,
                             int box_w, int box_h)
{
  return encode_one(map, base, width, height, stride_floats, box_w, box_h);
}

int StagedMaps::encode(const FilterParams &P, int patch_side)
{
  if(((uintptr_t)P.ref % 16) != 0 || ((uintptr_t)P.curr % 16) != 0 || (P.ref_stride % 4) != 0 ||
     (P.curr_stride % 4) != 0)
    return fail(RMD_ERR_INVALID_ARGUMENT, "staged kernel: images must be 16-byte aligned with 16-byte pitch");
  const bool geom_same = (width == P.width && height == P.height && patch == patch_side);
  if(!(geom_same && ref_ptr == P.ref && ref_stride == P.ref_stride))
  {
    const int rc = encode_one(&maps.ref, P.ref, P.width, P.height, P.ref_stride, REF_BOX_W,
                              ref_box_h(patch_side));
    if(rc) return rc;
    ref_ptr = P.ref; ref_stride = P.ref_stride;
  }
  if(!(geom_same && curr_ptr == P.curr && curr_stride == P.curr_stride))
  {
    for(int i = 0; i < NUM_WIDTHS; ++i)
    {
      const int rc = encode_one(&maps.curr[i], P.curr, P.width, P.height, P.curr_stride, strip_width(i),
                                STRIP_BOX_ROWS);
      if(rc) return rc;
    }
    curr_ptr = P.curr; curr_stride = P.curr_stride;
  }
  width = P.width; height = P.height; patch = patch_side;
  return 0;
}

namespace
{

template<int PS, int K, int MB>
struct StagedLaunch
{
  static size_t smem_bytes() { return sizeof(StagedSmem<PS>) + 128; }  // slack for the manual 128-byte alignment

  // Resident CTAs on `device` (SMs x occupancy); configures the kernel's shared-memory limit on first use.
  static int slots(int device)
  {
    static std::mutex mutex;
    static int cached[64] = {0};
    std::lock_guard<std::mutex> lock(mutex);
    if(device < 0 || device >= 64)
      return 0;
    if(cached[device] == 0)
    {
      if(cudaFuncSetAttribute(depth_filter_staged_kernel<PS, K, MB>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)smem_bytes()) != cudaSuccess)
        return 0;
      int per_sm = 0, sms = 0;
      if(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, depth_filter_staged_kernel<PS, K, MB>, NTHREADS,
                                                       smem_bytes()) != cudaSuccess ||
         cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess)
        return 0;
      cached[device] = per_sm * sms;
    }
    return cached[device];
  }

  static cudaError_t launch(const FilterParams *const *P, const StagedMaps *const *maps, int n, int chain,
                            unsigned int *cursor, cudaStream_t stream)
  {
    int device = 0;
    cudaError_t err = cudaGetDevice(&device);
    if(err != cudaSuccess) return err;
    const int n_slots = slots(device);
    if(n_slots <= 0)
    {
      err = cudaGetLastError();
      return err != cudaSuccess ? err : cudaErrorInvalidDevice;
    }
    static_assert(sizeof(StagedBatch<K>) <= 32000, "kernel parameter space (32 KB from CUDA 12.1)");
    StagedBatch<K> B;
    memset(&B, 0, sizeof(B));
    int tiles = 0;
    for(int k = 0; k < n; ++k)
    {
      B.p[k] = *P[k];
      B.m[k] = maps[k]->maps;
      tiles += P[k]->n_tiles + P[k]->helper_cap;
    }
    B.cursor = cursor;
    B.n = n;
    B.chain = chain;
    if(chain)
      tiles = P[0]->n_tiles + P[0]->helper_cap;   // the frames of a chain share the CTAs
    const dim3 block(TILE_W, NWARPS);
    int ctas = std::min(n_slots, tiles);         // persistent: never more CTAs than can be resident
    if(P[0]->grid_ctas > 0)
      ctas = std::min(ctas, P[0]->grid_ctas);
    const dim3 grid(ctas);
    cudaLaunchConfig_t cfg = cudaLaunchConfig_t();
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem_bytes(); cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = P[0]->pdl ? 1 : 0;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, depth_filter_staged_kernel<PS, K, MB>, B);
  }
};

} // namespace

cudaError_t launch_depth_filter_staged(const FilterParams *const *P, const StagedMaps *const *maps, int n, int chain,
                                       unsigned int *cursor, int patch_side, cudaStream_t stream)
{
  if(n < 1 || n > STAGED_BATCH_MAX || !P || !maps || !cursor)
    return cudaErrorInvalidValue;
  // RMD_FORCE_BATCH_KERNEL=1 (test hook): single keyframes also go through the batched instantiation
  static const bool force_batch = (getenv("RMD_FORCE_BATCH_KERNEL") != NULL);
  const bool single = (n == 1) && !force_batch && !chain;
  if(patch_side == 5 && P[0]->ctas_per_sm == 2)
    return single ? StagedLaunch<5, 1, 2>::launch(P, maps, n, 0, cursor, stream)
                  : StagedLaunch<5, STAGED_BATCH_MAX, 2>::launch(P, maps, n, chain, cursor, stream);
  if(patch_side == 5)
    return single ? StagedLaunch<5, 1, 3>::launch(P, maps, n, 0, cursor, stream)
                  : StagedLaunch<5, STAGED_BATCH_MAX, 3>::launch(P, maps, n, chain, cursor, stream);
  if(patch_side == 7)
    return single ? StagedLaunch<7, 1, 2>::launch(P, maps, n, 0, cursor, stream)
                  : StagedLaunch<7, STAGED_BATCH_MAX, 2>::launch(P, maps, n, chain, cursor, stream);
  return cudaErrorInvalidValue;
}

int staged_cta_slots(int patch_side, int ctas_per_sm)
{
  int device = 0;
  if(cudaGetDevice(&device) != cudaSuccess)
    return 0;
  if(patch_side == 5) return ctas_per_sm == 2 ? StagedLaunch<5, 1, 2>::slots(device) : StagedLaunch<5, 1, 3>::slots(device);
  if(patch_side == 7) return StagedLaunch<7, 1, 2>::slots(device);
  return 0;
}

} // namespace rmdb
