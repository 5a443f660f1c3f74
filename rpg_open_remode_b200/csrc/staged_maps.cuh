// staged_maps.cuh -- TMA descriptor set of the staged depth filter.
#pragma once

#include <cuda.h>

#include "rmd_common.cuh"

namespace rmdb
{

// Geometry shared by the host encoder and the kernel.
namespace staged
{
constexpr int TILE_W = 32;             // pixels per CTA row (one warp)
constexpr int TILE_H = 8;              // pixel rows per CTA
constexpr int NWARPS = TILE_H;          // one warp per pixel row; all warps share the tile's work list
constexpr int NTHREADS = 32 * NWARPS;
constexpr int NPIX = TILE_W * TILE_H;  // seeds per CTA
constexpr int CHUNK = 4;               // candidates per work item
constexpr int MAX_CHUNKS = 36;         // ceil(143 / CHUNK): 100 px / 0.7 px + 1 = 143 candidates
#ifndef RMD_RUN_MAX_CHUNKS
#define RMD_RUN_MAX_CHUNKS 9
#endif
#ifndef RMD_RUN_MIN_ROUNDS
#define RMD_RUN_MIN_ROUNDS 2
#endif
constexpr int RUN_MAX_CHUNKS = RMD_RUN_MAX_CHUNKS;  // longest run of chunks one work item scores (automatic choice)
constexpr int RUN_MIN_ROUNDS = RMD_RUN_MIN_ROUNDS;  // ... while every warp of the tile still gets this many rounds (2: DESIGN.md 4.1)
#ifndef RMD_STRIP_FLOATS
#define RMD_STRIP_FLOATS 15360
#endif
constexpr int STRIP_FLOATS = RMD_STRIP_FLOATS;    // current-image strip per CTA: 60 KB (40 KB: +1.5 %, 80 KB: -0.4 % but only 18 KB of L1 left; profiles/r02_occupancy_ab.txt)
constexpr int SPLIT_MAX = 16;            // at most this many CTAs share one busy tile
constexpr int HELPER_CAP = 1024;         // most helper CTAs per frame (work list capacity = tiles + this)
constexpr int SPLIT_MIN_ITEMS = 512;     // tiles below this are never split
constexpr int SPLIT_ITEMS_PER_CTA = 384; // a helper CTA must be worth its fixed cost: at least this many items each (tools/tune_probe.py)
constexpr int HEAVY_MIN_ITEMS = 128;     // tiles with at least this many items go to the front of the work list
constexpr int SPLIT_AVG_PCT = 50;        // ... or this percentage of the frame's items per resident-CTA slot, if larger
constexpr int SPARSE_MAX_SEEDS = 16;     // tiles with at most this many seeds to update skip staging
constexpr int WARP_TILE_MAX_SEEDS = 8;   // ... and with at most this many (and WARP_TILE_MAX_CANDS candidates) are done by one warp
constexpr int WARP_TILE_MAX_CANDS = 64;
constexpr int L_CHECKPOINT_STEP = 16;   // l is stored every 16th candidate (power of two)
constexpr int L_CHECKPOINTS = 9;        // ceil(143 / 16)
constexpr int STRIP_BOX_ROWS = 8;      // rows per TMA box of the strip
constexpr int REF_BOX_W = 40;          // covers [x0 - 4, x0 + 36): tile + halo of a 7x7 patch
constexpr int REF_ORIGIN_X = 4;        // the reference box starts at x0 - 4 (16-byte aligned origin)
constexpr int NUM_WIDTHS = 4;
__host__ __device__ constexpr int strip_width(int i)
{
  // multiples of 32 floats, so bank = column mod 32 whatever row a lane is on: the 32 lanes of a round score the
  // candidates of 32 neighbouring pixels, i.e. (nearly) consecutive columns.  Not conflict-free in practice: as soon
  // as the two views differ in scale the 32 blocks span more than 32 columns and two lanes share a bank -- ncu counts
  // 1.9 wavefronts per LDS of the NCC on search-heavy frames (profiles/r02_ncu_staged.md); TMA's swizzle modes
  // only apply to rows of <= 128 bytes, the strip's are 256..640.
  return i == 0 ? 64 : (i == 1 ? 96 : (i == 2 ? 128 : 160));
}
__host__ __device__ constexpr int ref_box_h(int patch) { return TILE_H + patch - 1; }
}

// The descriptors as the kernel receives them (one __grid_constant__ param).
struct alignas(64) StagedTensorMaps
{
  CUtensorMap ref;                         // box REF_BOX_W x ref_box_h(patch)
  CUtensorMap curr[staged::NUM_WIDTHS];    // boxes strip_width(i) x STRIP_BOX_ROWS
};

// Most keyframes one launch can serve (rmd_seeds_update_many: several live reference views against
// one incoming frame, SURVEY.md 8f row 2).
constexpr int STAGED_BATCH_MAX = 8;

// Everything one launch of the staged kernel receives, as ONE __grid_constant__ parameter: the
// descriptors and parameter blocks of 1 (single-keyframe instantiation: all offsets static) or up
// to STAGED_BATCH_MAX keyframes (batched instantiation: indexed by the keyframe an entry belongs
// to), and the launch's work cursor.  8 keyframes = 8 x (640 + sizeof(FilterParams)) bytes: needs
// the 32 KB kernel-parameter space of CUDA >= 12.1.
template<int K>
struct alignas(64) StagedBatch
{
  StagedTensorMaps m[K];
  FilterParams p[K];
  // cursor[g], g < STAGED_BATCH_MAX: next entry of the work list(s) -- batch mode uses cursor[0] over the
  // concatenation (all heavy lists, then all light lists), chain mode one cursor per frame;
  // cursor[STAGED_BATCH_MAX]: CTAs that have run out of work; cursor[STAGED_BATCH_MAX + 1]: error flag
  // (a bounded wait of the chain mode expired).  The last CTA out leaves the cursors and the count at zero.
  unsigned int *cursor;
  int n;                 // keyframes (batch) or consecutive frames (chain) in this launch, 1 <= n <= K
  int chain;             // 0: p[0..n) = n keyframes updated by one frame; 1: p[0..n) = n consecutive frames of one keyframe
};
constexpr int STAGED_CURSOR_WORDS = STAGED_BATCH_MAX + 2;

// Tiled 2-D tensor maps (cuTensorMapEncodeTiled) over the pitched reference
// and current images.  Box shapes are fixed when a map is encoded; the box
// origin is a run-time coordinate of the TMA instruction, so one map per box
// width serves every CTA.  The current image changes address every frame
// (upload ring / caller memory), hence encode() per frame: it is a pure host
// computation of 128-byte descriptors, no driver round trip.
struct StagedMaps
{
  StagedTensorMaps maps;
  int patch;
  const void *ref_ptr, *curr_ptr;
  int ref_stride, curr_stride, width, height;

  StagedMaps();
  // Returns 0 or an error code (and sets the thread's last error string).
  int encode(const FilterParams &P, int patch_side);
};

} // namespace rmdb
