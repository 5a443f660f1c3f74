// volume_store.h -- host side of the TSDF volume's brick store (DESIGN.md 4.8): which 8x8x8 bricks of the unbounded
// grid a shift touches, and the index from brick coordinate to pool slot.  Host-only (no CUDA), so that a CPU test can
// cover it (tests/cpp/volume_store_test.cpp).
//
// Voxel (i, j, k) of the window is voxel u = (i, j, k) + W of the unbounded grid, W the window's total offset; it lies
// in brick floor(u / 8) per axis.  Coordinates are int64 per axis, so there is no packing range.
#pragma once

#include <stddef.h>
#include <stdint.h>

#include <map>
#include <vector>

namespace rmdb
{

constexpr int STORE_BRICK = 8;                                            // voxels per brick edge
constexpr int STORE_BRICK_VOXELS = STORE_BRICK * STORE_BRICK * STORE_BRICK;

struct BrickCoord
{
  int64_t b[3];   // x, y, z
};

// Ascending (z, y, x): the order of candidates, of slot assignment and of rmd_volume_download_store.
struct BrickOrder
{
  bool operator()(const BrickCoord &p, const BrickCoord &q) const
  {
    for(int a = 2; a >= 0; --a)
      if(p.b[a] != q.b[a])
        return p.b[a] < q.b[a];
    return false;
  }
};

inline int64_t brick_floor(int64_t u)
{
  const int64_t q = u / STORE_BRICK;
  return (u % STORE_BRICK < 0) ? q - 1 : q;
}

// Every brick with a voxel in the window [W, W + n) that lies outside the box [W + lo, W + hi) (window indices, per
// axis; an empty box on any axis takes the whole window), in ascending (z, y, x).  The caller guarantees that W + n
// does not overflow.  With the box a shift by d keeps, these are the bricks with a leaving voxel; with the box of
// pre-shift sources after the shift, the bricks with an entering voxel.
inline std::vector<BrickCoord> store_candidates(const int64_t W[3], const int n[3], const int lo[3], const int hi[3])
{
  std::vector<BrickCoord> out;
  int64_t b0[3];
  int s[3], nb[3];
  bool empty_box = false;
  std::vector<char> inside[3];   // per axis and brick: its window voxels all lie in [lo, hi)
  for(int a = 0; a < 3; ++a)
  {
    if(n[a] <= 0)
      return out;
    b0[a] = brick_floor(W[a]);
    s[a] = (int)(b0[a] * STORE_BRICK - W[a]);   // window index of brick b0's first voxel, in [-7, 0]
    nb[a] = (n[a] - 1 - s[a]) / STORE_BRICK + 1;
    empty_box = empty_box || lo[a] >= hi[a];
    inside[a].resize(nb[a]);
    for(int t = 0; t < nb[a]; ++t)
    {
      const int a0 = s[a] + STORE_BRICK * t < 0 ? 0 : s[a] + STORE_BRICK * t;
      const int a1 = s[a] + STORE_BRICK * (t + 1) > n[a] ? n[a] : s[a] + STORE_BRICK * (t + 1);
      inside[a][t] = a0 >= lo[a] && a1 <= hi[a];
    }
  }
  for(int z = 0; z < nb[2]; ++z)
    for(int y = 0; y < nb[1]; ++y)
      for(int x = 0; x < nb[0]; ++x)
        if(empty_box || !(inside[0][x] && inside[1][y] && inside[2][z]))
          out.push_back(BrickCoord{{b0[0] + x, b0[1] + y, b0[2] + z}});
  return out;
}

// The index of the stored bricks: brick coordinate -> pool slot.  Slots are dense, 0 .. size() - 1, in the order the
// bricks were added.
struct BrickIndex
{
  std::map<BrickCoord, int, BrickOrder> slot;

  // The candidates split into those already stored and those not, each in candidate order.
  void split(const std::vector<BrickCoord> &cand, std::vector<BrickCoord> &known, std::vector<BrickCoord> &fresh) const
  {
    for(const BrickCoord &c : cand)
      (slot.count(c) ? known : fresh).push_back(c);
  }

  // Adds the fresh bricks whose flag is set, in their order, each at the next slot; returns them.
  std::vector<BrickCoord> add(const std::vector<BrickCoord> &fresh, const std::vector<int> &flags)
  {
    std::vector<BrickCoord> added;
    for(size_t q = 0; q < fresh.size(); ++q)
      if(flags[q])
      {
        slot.emplace(fresh[q], (int)slot.size());
        added.push_back(fresh[q]);
      }
    return added;
  }
};

// Pool capacity (bricks) for `need` bricks from `cap`: doubled until it fits, at least 64.
inline size_t store_pool_capacity(size_t cap, size_t need)
{
  if(need <= cap)
    return cap;
  size_t c = cap ? cap : 64;
  while(c < need)
    c *= 2;
  return c;
}

} // namespace rmdb
