// S2: gpu_cache -- set-associative LRU hot-row cache in HBM (Query / Replace / Update / Dump).
// Interface and semantics of the reference gpu_cache (gpu_cache/include/nv_gpu_cache.hpp,
// gpu_cache/src/nv_gpu_cache.cu:154-1230, gpu_cache/ReadMe.md): `num_sets` sets x `ways` slots
// (ways is a multiple of 32 so one warp probes a whole set with coalesced key reads + ballot),
// a global 64-bit clock stamps every touch and the LRU victim is the warp-min of the stamps,
// Query returns hit vectors plus a compacted miss list, Replace inserts-or-evicts under a per-set
// lock, Update overwrites hits only, Dump lists the keys of a set range.
#include <cuda_runtime.h>
#include <stdint.h>

#include "embedding.cuh"
#include "set_assoc.cuh"

namespace hctr {

struct CacheView {
  long long* keys;            // [num_sets * ways], -1 = empty
  unsigned long long* stamps; // [num_sets * ways]
  float* vals;                // [num_sets * ways, ev]
  int* locks;                 // [num_sets]
  unsigned long long* clock;  // [1]
  int num_sets, ways, ev;
};

HCTR_DEVICE int set_of(const CacheView& c, long long key) {
  return static_cast<int>(hash64(static_cast<unsigned long long>(key)) % static_cast<unsigned>(c.num_sets));
}

// warp-cooperative find: returns slot index inside the set or -1 (uniform across the warp)
HCTR_DEVICE int warp_find(const CacheView& c, int set, long long key, int lane) {
  return warp_find(c.keys + static_cast<long long>(set) * c.ways, c.ways, key, lane);
}

__global__ void __launch_bounds__(256)
    cache_query_kernel(CacheView c, const long long* __restrict__ keys, long long n,
                       float* __restrict__ out, long long* __restrict__ miss_index,
                       long long* __restrict__ miss_keys, unsigned long long* miss_len) {
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const long long key = keys[w];
  const int set = set_of(c, key);
  const int slot = key < 0 ? -1 : warp_find(c, set, key, lane);
  if (slot >= 0) {
    const long long g = static_cast<long long>(set) * c.ways + slot;
    if (lane == 0) c.stamps[g] = atomicAdd(c.clock, 1ull) + 1ull;
    const float* v = c.vals + g * c.ev;
    for (int e = lane; e < c.ev; e += 32) out[w * c.ev + e] = v[e];
  } else if (lane == 0) {
    const unsigned long long p = atomicAdd(miss_len, 1ull);
    miss_index[p] = w;
    miss_keys[p] = key;
  }
}

HCTR_DEVICE void lock_set(const CacheView& c, int set, int lane) { lock_set(c.locks, set, lane); }
HCTR_DEVICE void unlock_set(const CacheView& c, int set, int lane) { unlock_set(c.locks, set, lane); }

// insert-or-evict (LRU); already-present keys are refreshed with the new value
__global__ void __launch_bounds__(256)
    cache_replace_kernel(CacheView c, const long long* __restrict__ keys,
                         const float* __restrict__ vals, long long n,
                         long long* __restrict__ evicted_keys, float* __restrict__ evicted_vals,
                         unsigned long long* evicted_len) {
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const long long key = keys[w];
  if (key < 0) return;
  const int set = set_of(c, key);
  lock_set(c, set, lane);
  int slot = warp_find(c, set, key, lane);
  long long victim_key = -1;
  if (slot < 0) {
    // empty slot first, else the least recently used
    const long long* k = c.keys + static_cast<long long>(set) * c.ways;
    const unsigned long long* st = c.stamps + static_cast<long long>(set) * c.ways;
    unsigned long long best = ~0ull;
    int best_slot = 0;
    for (int wv = 0; wv < c.ways; wv += 32) {
      unsigned long long s = (k[wv + lane] < 0) ? 0ull : st[wv + lane];
      int sl = wv + lane;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long s2 = __shfl_xor_sync(0xffffffffu, s, o);
        const int sl2 = __shfl_xor_sync(0xffffffffu, sl, o);
        if (s2 < s || (s2 == s && sl2 < sl)) { s = s2; sl = sl2; }
      }
      if (s < best) { best = s; best_slot = sl; }
    }
    slot = best_slot;
    victim_key = k[slot];
  }
  const long long g = static_cast<long long>(set) * c.ways + slot;
  if (victim_key >= 0 && evicted_keys != nullptr) {
    unsigned long long p = 0;
    if (lane == 0) p = atomicAdd(evicted_len, 1ull);
    p = __shfl_sync(0xffffffffu, p, 0);
    if (lane == 0) evicted_keys[p] = victim_key;
    for (int e = lane; e < c.ev; e += 32) evicted_vals[p * c.ev + e] = c.vals[g * c.ev + e];
  }
  for (int e = lane; e < c.ev; e += 32) c.vals[g * c.ev + e] = vals[w * c.ev + e];
  if (lane == 0) {
    c.keys[g] = key;
    c.stamps[g] = atomicAdd(c.clock, 1ull) + 1ull;
  }
  unlock_set(c, set, lane);
}

__global__ void __launch_bounds__(256)
    cache_update_kernel(CacheView c, const long long* __restrict__ keys,
                        const float* __restrict__ vals, long long n) {
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const long long key = keys[w];
  if (key < 0) return;
  const int set = set_of(c, key);
  lock_set(c, set, lane);
  const int slot = warp_find(c, set, key, lane);
  if (slot >= 0) {
    const long long g = static_cast<long long>(set) * c.ways + slot;
    for (int e = lane; e < c.ev; e += 32) c.vals[g * c.ev + e] = vals[w * c.ev + e];
  }
  unlock_set(c, set, lane);
}

__global__ void cache_dump_kernel(CacheView c, int set0, int set1, long long* out_keys,
                                  unsigned long long* out_len) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long n = static_cast<long long>(set1 - set0) * c.ways;
  if (i >= n) return;
  const long long k = c.keys[static_cast<long long>(set0) * c.ways + i];
  if (k >= 0) out_keys[atomicAdd(out_len, 1ull)] = k;
}

}  // namespace hctr

using namespace hctr;

static CacheView mk(void* keys, void* stamps, void* vals, void* locks, void* clock, int num_sets,
                    int ways, int ev) {
  return CacheView{(long long*)keys, (unsigned long long*)stamps, (float*)vals, (int*)locks,
                   (unsigned long long*)clock, num_sets, ways, ev};
}

extern "C" int hctr_cache_query(void* keys_t, void* stamps, void* vals, void* locks, void* clock,
                                int num_sets, int ways, int ev, const long long* keys, long long n,
                                float* out, long long* miss_index, long long* miss_keys,
                                void* miss_len, void* stream) {
  if (n == 0) return 0;
  cache_query_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      mk(keys_t, stamps, vals, locks, clock, num_sets, ways, ev), keys, n, out, miss_index, miss_keys,
      (unsigned long long*)miss_len);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
extern "C" int hctr_cache_replace(void* keys_t, void* stamps, void* vals, void* locks, void* clock,
                                  int num_sets, int ways, int ev, const long long* keys,
                                  const float* v, long long n, long long* ev_keys, float* ev_vals,
                                  void* ev_len, void* stream) {
  if (n == 0) return 0;
  cache_replace_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      mk(keys_t, stamps, vals, locks, clock, num_sets, ways, ev), keys, v, n, ev_keys, ev_vals,
      (unsigned long long*)ev_len);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
extern "C" int hctr_cache_update(void* keys_t, void* stamps, void* vals, void* locks, void* clock,
                                 int num_sets, int ways, int ev, const long long* keys, const float* v,
                                 long long n, void* stream) {
  if (n == 0) return 0;
  cache_update_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      mk(keys_t, stamps, vals, locks, clock, num_sets, ways, ev), keys, v, n);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
extern "C" int hctr_cache_dump(void* keys_t, void* stamps, void* vals, void* locks, void* clock,
                               int num_sets, int ways, int ev, int set0, int set1, long long* out_keys,
                               void* out_len, void* stream) {
  const long long n = static_cast<long long>(set1 - set0) * ways;
  if (n <= 0) return 0;
  cache_dump_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      mk(keys_t, stamps, vals, locks, clock, num_sets, ways, ev), set0, set1, out_keys,
      (unsigned long long*)out_len);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
