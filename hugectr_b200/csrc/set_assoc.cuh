// Warp-cooperative pieces of the set-associative tables (gpu_cache.cu, evict_table.cu): a set is a
// run of `ways` keys (a multiple of 32) probed by one warp with coalesced loads and a ballot, and
// guarded by one lock word.  Only lane 0 takes a lock; a warp holds at most one set lock at a time.
#pragma once
#include <cuda_runtime.h>

#include "ptx.cuh"

namespace hctr {

// slot of `key` inside the set whose keys start at `k`, or -1 (uniform across the warp).  K may be
// volatile-qualified to re-read a set another warp is changing.
template <typename K, typename V>
HCTR_DEVICE int warp_find(K* k, int ways, V key, int lane) {
  for (int w = 0; w < ways; w += 32) {
    const unsigned m = __ballot_sync(0xffffffffu, k[w + lane] == key);
    if (m) return w + __ffs(m) - 1;
  }
  return -1;
}

// lock word `locks[set]` (indexed by lane 0 only)
HCTR_DEVICE void lock_set(int* locks, int set, int lane) {
  if (lane == 0) {
    while (atomicCAS(&locks[set], 0, 1) != 0) {
    }
    __threadfence();
  }
  __syncwarp();
}

HCTR_DEVICE void unlock_set(int* locks, int set, int lane) {
  __syncwarp();
  if (lane == 0) {
    __threadfence();
    atomicExch(&locks[set], 0);
  }
}

}  // namespace hctr
