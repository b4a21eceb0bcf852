// The parameter-group lookup of the fused optimizer kernels (csrc/cuda/optim_body.cuh: group_seg_find and the per-thread
// cursor group_seg_advance), compiled by g++ and checked against a brute-force map of every shard vector to its row, on
// random sorted segment tables and the grid strides the kernels walk them with.
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>
#include <random>
#include <vector>

#include "cuda/optim_body.cuh"

using bnet::optim::group_seg_advance;
using bnet::optim::group_seg_find;

static int failures = 0;
#define CHECK(cond, ...)                                     \
  do {                                                       \
    if (!(cond)) {                                           \
      if (failures++ < 10) {                                 \
        fprintf(stderr, "FAIL %s:%d: ", __FILE__, __LINE__); \
        fprintf(stderr, __VA_ARGS__);                        \
        fprintf(stderr, "\n");                               \
      }                                                      \
    }                                                        \
  } while (0)

// A random table of `nseg` rows covering `shard` vectors: {vec0, nvec, group, 0}.
static std::vector<int> random_table(std::mt19937& rng, int shard, int nseg, int ngroups) {
  std::vector<int> cuts = {0};
  std::uniform_int_distribution<int> pos(1, shard - 1);
  while ((int)cuts.size() < nseg) {
    const int c = pos(rng);
    bool dup = false;
    for (int x : cuts) dup |= x == c;
    if (!dup) cuts.push_back(c);
  }
  std::sort(cuts.begin(), cuts.end());
  std::vector<int> t;
  std::uniform_int_distribution<int> grp(0, ngroups - 1);
  for (int k = 0; k < nseg; k++) {
    const int end = k + 1 < nseg ? cuts[k + 1] : shard;
    t.insert(t.end(), {cuts[k], end - cuts[k], grp(rng), 0});
  }
  return t;
}

int main() {
  std::mt19937 rng(1234);
  long checks = 0;
  // (shard vectors, rows): one row, rows of one vector, many short rows, a few long ones
  const int shapes[][2] = {{1, 1}, {7, 7}, {8, 3}, {1000, 1}, {1000, 999}, {4096, 161}, {100003, 64}, {1 << 20, 317}};
  // grid strides of 1, 7, 132 and 264 CTAs of 512 threads, and small ones that land on every row
  const int strides[] = {1, 3, 512, 7 * 512, 132 * 512, 264 * 512};
  for (const auto& sh : shapes) {
    const int shard = sh[0], nseg = sh[1];
    for (int rep = 0; rep < 4; rep++) {
      const std::vector<int> t = random_table(rng, shard, nseg, 1 + rep * 20);
      std::vector<int> row_of(shard);
      for (int k = 0; k < nseg; k++)
        for (int v = t[4 * k]; v < t[4 * k] + t[4 * k + 1]; v++) row_of[v] = k;
      for (int v = 0; v < shard; v++) {
        CHECK(group_seg_find(t.data(), nseg, v) == row_of[v], "find: shard %d rows %d vector %d", shard, nseg, v);
        checks++;
      }
      // a cursor per thread, as the kernels keep it: started by the search at the thread's first vector, walked forward
      for (int stride : strides) {
        const int threads = stride < shard ? stride : shard;
        const int step = threads > 4096 ? threads / 4096 : 1;   // (a sample of the threads of the large grids)
        for (int first = 0; first < threads; first += step) {
          int cur = group_seg_find(t.data(), nseg, first);
          for (long v = first; v < shard; v += stride) {
            cur = group_seg_advance(t.data(), nseg, cur, (int)v);
            CHECK(cur == row_of[v], "cursor: shard %d rows %d stride %d vector %ld: row %d, want %d", shard, nseg, stride, v, cur,
                  row_of[v]);
            CHECK(t[4 * cur + 2] == t[4 * row_of[v] + 2], "cursor: wrong group");
            checks++;
          }
        }
      }
    }
  }
  if (failures) {
    fprintf(stderr, "group_lookup_test: %d of %ld checks FAILED\n", failures, checks);
    return 1;
  }
  printf("group_lookup_test: %ld lookups match the brute-force map\n", checks);
  return 0;
}
