// The brick store's host side (rpg_open_remode_b200/csrc/volume_store.h): the candidate bricks of a shift against a
// voxel-by-voxel enumeration, and the order in which new bricks get their slots.  Host-only, no GPU.
#include <stdio.h>
#include <stdlib.h>

#include <set>
#include <vector>

#include "../../rpg_open_remode_b200/csrc/volume_store.h"

using namespace rmdb;

static int failures = 0;

#define CHECK(cond, ...)                          \
  do {                                            \
    if(!(cond))                                   \
    {                                             \
      printf("FAIL %s:%d: ", __FILE__, __LINE__); \
      printf(__VA_ARGS__);                        \
      printf("\n");                               \
      ++failures;                                 \
    }                                             \
  } while(0)

// The box a shift by d keeps, in pre-shift window indices (rmd_volume_spill_* / spill_box in volume_api.cu).
static void kept_box(const int n[3], const int d[3], int lo[3], int hi[3])
{
  for(int a = 0; a < 3; ++a)
  {
    const int c = d[a] < -n[a] ? -n[a] : d[a] > n[a] ? n[a] : d[a];
    lo[a] = c > 0 ? c : 0;
    hi[a] = c < 0 ? n[a] + c : n[a];
  }
}

// Every voxel of the window, floor division written out differently: the bricks of the voxels outside the box.
static std::vector<BrickCoord> brute(const int64_t W[3], const int n[3], const int lo[3], const int hi[3])
{
  std::set<BrickCoord, BrickOrder> s;
  for(int k = 0; k < n[2]; ++k)
    for(int j = 0; j < n[1]; ++j)
      for(int i = 0; i < n[0]; ++i)
      {
        const int w[3] = {i, j, k};
        bool inside = true;
        BrickCoord c;
        for(int a = 0; a < 3; ++a)
        {
          inside = inside && w[a] >= lo[a] && w[a] < hi[a];
          const int64_t u = W[a] + w[a];
          c.b[a] = (u - ((u % 8) + 8) % 8) / 8;
        }
        if(!inside)
          s.insert(c);
      }
  return std::vector<BrickCoord>(s.begin(), s.end());
}

static bool same(const std::vector<BrickCoord> &p, const std::vector<BrickCoord> &q)
{
  if(p.size() != q.size())
    return false;
  for(size_t i = 0; i < p.size(); ++i)
    for(int a = 0; a < 3; ++a)
      if(p[i].b[a] != q[i].b[a])
        return false;
  return true;
}

static void check_shift(const int64_t D[3], const int n[3], const int d[3], const char *what)
{
  int lo[3], hi[3], ilo[3], ihi[3];
  kept_box(n, d, lo, hi);
  const std::vector<BrickCoord> leave = store_candidates(D, n, lo, hi);
  CHECK(same(leave, brute(D, n, lo, hi)), "%s: leaving candidates (%zu)", what, leave.size());
  // entering: the box of the post-shift voxels whose source lay in the grid is the kept box of -d
  const int nd[3] = {-d[0], -d[1], -d[2]};
  kept_box(n, nd, ilo, ihi);
  const int64_t Dn[3] = {D[0] + d[0], D[1] + d[1], D[2] + d[2]};
  const std::vector<BrickCoord> enter = store_candidates(Dn, n, ilo, ihi);
  CHECK(same(enter, brute(Dn, n, ilo, ihi)), "%s: entering candidates (%zu)", what, enter.size());
  for(size_t i = 1; i < leave.size(); ++i)
    CHECK(BrickOrder()(leave[i - 1], leave[i]), "%s: not ascending (z, y, x)", what);
  if(!d[0] && !d[1] && !d[2])
    CHECK(leave.empty() && enter.empty(), "%s: d = 0 moves nothing", what);
}

int main()
{
  {
    const int n[3] = {97, 64, 71};
    const int64_t D0[3] = {0, 0, 0}, Dneg[3] = {-13, -64, -1}, Dodd[3] = {5, -3, 1000000000003LL};
    const int ds[][3] = {{0, 0, 0}, {1, 0, 0}, {-3, 5, 0}, {9, -17, 33}, {97, 0, 0}, {0, -64, 0}, {200, -300, 71},
                         {-96, 63, -70}, {8, 8, 8}, {-8, 0, 16}};
    for(const int *d : ds)
    {
      check_shift(D0, n, d, "97x64x71, D = 0");
      check_shift(Dneg, n, d, "97x64x71, negative D");
      check_shift(Dodd, n, d, "97x64x71, D not a multiple of 8");
    }
  }
  {
    const int n[3] = {1, 40, 9};
    const int64_t D[3] = {-7, 3, -9};
    const int ds[][3] = {{1, 0, 0}, {-1, 2, 0}, {0, 0, 9}, {0, -41, 0}, {0, 0, 0}, {3, 5, -2}};
    for(const int *d : ds)
      check_shift(D, n, d, "nx = 1");
  }
  {
    // slot order: fresh bricks with their flag set, in candidate order, after the bricks already stored
    BrickIndex index;
    const std::vector<BrickCoord> a = {{{0, 0, 0}}, {{1, 0, 0}}, {{-1, 1, 0}}, {{0, 0, 1}}};
    const std::vector<BrickCoord> added = index.add(a, std::vector<int>{1, 0, 1, 1});
    CHECK(added.size() == 3 && index.slot.size() == 3, "add: %zu", added.size());
    CHECK(index.slot.at(a[0]) == 0 && index.slot.at(a[2]) == 1 && index.slot.at(a[3]) == 2 && !index.slot.count(a[1]),
          "add: slots");
    std::vector<BrickCoord> known, fresh;
    const std::vector<BrickCoord> cand = {{{1, 0, 0}}, {{0, 0, 1}}, {{5, 5, 5}}, {{0, 0, 0}}};
    index.split(cand, known, fresh);
    CHECK(known.size() == 2 && fresh.size() == 2 && fresh[0].b[0] == 1 && fresh[1].b[0] == 5, "split");
    index.add(fresh, std::vector<int>{0, 1});
    CHECK(index.slot.at(cand[2]) == 3 && index.slot.size() == 4, "add after split");
    // iteration is ascending (z, y, x)
    std::vector<BrickCoord> order;
    for(const auto &e : index.slot)
      order.push_back(e.first);
    for(size_t i = 1; i < order.size(); ++i)
      CHECK(BrickOrder()(order[i - 1], order[i]), "index order");
    CHECK(order[0].b[0] == 0 && order[0].b[1] == 0 && order[0].b[2] == 0 && order[1].b[0] == -1, "index order");
  }
  CHECK(store_pool_capacity(0, 0) == 0 && store_pool_capacity(0, 1) == 64 && store_pool_capacity(64, 65) == 128 &&
        store_pool_capacity(64, 300) == 512 && store_pool_capacity(128, 100) == 128, "pool capacity");
  CHECK(brick_floor(-1) == -1 && brick_floor(-8) == -1 && brick_floor(-9) == -2 && brick_floor(7) == 0 &&
        brick_floor(INT64_MIN) == INT64_MIN / 8, "brick_floor");
  if(failures)
  {
    printf("%d FAILURES\n", failures);
    return 1;
  }
  printf("ALL VOLUME STORE HOST TESTS PASSED\n");
  return 0;
}
