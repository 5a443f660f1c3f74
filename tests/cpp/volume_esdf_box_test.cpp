// The brick table of an ESDF box (rpg_open_remode_b200/csrc/volume_store.h, store_brick_table) against std::map
// lookups: random stored bricks with negative coordinates and coordinates near the int64 limits, random box brick
// ranges that hold some, all or none of them, and a one-brick range.  Host-only, no GPU.
#include <stdint.h>
#include <stdio.h>

#include <random>
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

// Every entry of the table against a lookup of its brick in the index.
static void check_table(const BrickIndex &index, const int64_t b0[3], const int nb[3])
{
  const std::vector<int> table = store_brick_table(index, b0, nb);
  CHECK(table.size() == (size_t)nb[0] * nb[1] * nb[2], "table size %zu", table.size());
  size_t q = 0, found = 0;
  for(int z = 0; z < nb[2]; ++z)
    for(int y = 0; y < nb[1]; ++y)
      for(int x = 0; x < nb[0]; ++x, ++q)
      {
        const BrickCoord c{{b0[0] + x, b0[1] + y, b0[2] + z}};
        const auto it = index.slot.find(c);
        const int want = it == index.slot.end() ? -1 : it->second;
        found += want >= 0;
        if(table[q] != want)
        {
          CHECK(false, "brick (%lld, %lld, %lld): %d, want %d", (long long)c.b[0], (long long)c.b[1],
                (long long)c.b[2], table[q], want);
          return;
        }
      }
  // every stored brick in range is in the table, and nothing else
  size_t in_range = 0;
  for(const auto &e : index.slot)
  {
    bool in = true;
    for(int a = 0; a < 3; ++a)
      in = in && e.first.b[a] >= b0[a] && e.first.b[a] - b0[a] < nb[a];
    in_range += in;
  }
  CHECK(found == in_range, "%zu found, %zu in range", found, in_range);
}

int main()
{
  std::mt19937_64 rng(0xB0C5);
  for(int round = 0; round < 200; ++round)
  {
    BrickIndex index;
    const int64_t centre[3] = {(int64_t)(rng() % 41) - 20, (int64_t)(rng() % 41) - 20, (int64_t)(rng() % 41) - 20};
    const int n = 1 + (int)(rng() % 400);
    for(int q = 0; q < n; ++q)
    {
      BrickCoord c;
      for(int a = 0; a < 3; ++a)
        c.b[a] = centre[a] + (int64_t)(rng() % 25) - 12;
      if(!index.slot.count(c))
        index.slot.emplace(c, (int)index.slot.size());
    }
    int64_t b0[3];
    int nb[3];
    for(int a = 0; a < 3; ++a)
    {
      b0[a] = centre[a] + (int64_t)(rng() % 31) - 15;
      nb[a] = 1 + (int)(rng() % 20);
    }
    check_table(index, b0, nb);
    // a range that holds every brick, one that holds none, one brick
    const int64_t all0[3] = {centre[0] - 12, centre[1] - 12, centre[2] - 12}, none0[3] = {centre[0] + 13, 0, 0};
    const int all_n[3] = {25, 25, 25}, one[3] = {1, 1, 1};
    check_table(index, all0, all_n);
    check_table(index, none0, all_n);
    check_table(index, index.slot.begin()->first.b, one);
  }
  // coordinates near the int64 limits: no overflow in the range test
  BrickIndex edge;
  const int64_t lo = INT64_MIN / STORE_BRICK, hi = INT64_MAX / STORE_BRICK;
  edge.slot.emplace(BrickCoord{{lo, lo, lo}}, 0);
  edge.slot.emplace(BrickCoord{{hi, hi, hi}}, 1);
  edge.slot.emplace(BrickCoord{{lo + 1, hi, 0}}, 2);
  edge.slot.emplace(BrickCoord{{-1, 0, 1}}, 3);
  const int64_t r0[3] = {lo, lo, lo}, r1[3] = {hi - 2, hi - 2, hi - 2}, r2[3] = {lo, hi - 1, -1}, r3[3] = {-3, -2, -1};
  const int three[3] = {3, 3, 3};
  check_table(edge, r0, three);
  check_table(edge, r1, three);
  check_table(edge, r2, three);
  check_table(edge, r3, three);
  const std::vector<int> t3 = store_brick_table(edge, r3, three);
  CHECK(t3[(2 * 3 + 2) * 3 + 2] == 3, "brick (-1, 0, 1) at its entry");
  if(failures)
  {
    printf("%d FAILURES\n", failures);
    return 1;
  }
  printf("ALL VOLUME ESDF BOX HOST TESTS PASSED\n");
  return 0;
}
