// Evicting shards of dynamic embedding-collection tables (EmbeddingTableConfig(evict_strategy="lru" |
// "lfu")): a fixed set-associative key -> row map, S sets of 32 ways, a key lives only in set
// hash64(key) % S and its arena row is row_off + set * 32 + way.  Semantics in docs/embedding.md.
//
// One training lookup of a table is two passes over its key regions, every region of the table through
// the first pass before any region goes through the second:
//   touch   a present key stamps its way with the collection clock and counts the occurrence (an admitting
//           table counts a missing key's occurrence in its admission sketch instead, admit_sketch.cuh);
//   insert  every key gets its row, written in place over the key (the lookup kernels then run as for a
//           static table); a missing key takes, under its set's lock, an empty way or else the unprotected
//           way with the smallest (stamp, key) (LRU) or (count, stamp, key) (LFU).  A way stamped with the
//           current clock is protected, so every key of the running step keeps its row for the whole step.
//           An admitting table first rejects a missing key whose sketch count is below its threshold.
// Then the re-initialisation kernel gives every admitted row fresh weights and optimizer state.
// Evaluation uses the get kernel only.  Everything reads the clock from device memory: no host input,
// so the whole step is captured in one CUDA graph.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "admit_sketch.cuh"
#include "embedding.cuh"
#include "set_assoc.cuh"

namespace hctr {

constexpr int kEvictWays = 32;
constexpr unsigned long long kCountMax = 0xFFFFFFFFull;  // counts compare saturated at this value

struct EvictTableView {
  long long* keys;                  // [capacity] -1 = empty way
  unsigned long long* stamps;       // [capacity] clock of the last touch
  unsigned long long* counts;       // [capacity] touches since admission (read saturated at kCountMax)
  int* locks;                       // [num_sets]
  const unsigned long long* clock;  // [1] the collection's clock
  unsigned long long* stats;        // [3] admitted, evicted, dropped (cumulative)
  int num_sets;
  int lfu;
};

// The keys of one lookup in every source rank's slab: `ranks` blocks of `n` keys, `stride` elements
// apart.  A key is handled iff key >= 0 and key % key_mod == key_rem (the row shard's ownership).
struct KeyRegion {
  void* base;
  long long n;
  long long stride;
  int ranks;
  int key_mod, key_rem;
  int key_bytes;  // 4 or 8
};

template <typename KT>
HCTR_DEVICE KT* key_ptr(const KeyRegion& r, long long i) {
  const long long rk = i / r.n;
  return static_cast<KT*>(r.base) + rk * r.stride + (i - rk * r.n);
}

HCTR_DEVICE bool owned(const KeyRegion& r, long long key) {
  return key >= 0 && (r.key_mod <= 1 ||
                      static_cast<unsigned long long>(key) % static_cast<unsigned long long>(r.key_mod) ==
                          static_cast<unsigned long long>(r.key_rem));
}

HCTR_DEVICE long long evict_set_base(const EvictTableView& t, long long key) {
  const unsigned int set = hash64(static_cast<unsigned long long>(key)) % static_cast<unsigned>(t.num_sets);
  return static_cast<long long>(set) * kEvictWays;
}

// kAdmit (admit_threshold > 1): an occurrence of a missing key is counted in the admission sketch
template <typename KT, bool kAdmit>
__global__ void __launch_bounds__(256) evict_touch_kernel(EvictTableView t, KeyRegion r, AdmitSketch s) {
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= r.n * r.ranks) return;
  const long long key = static_cast<long long>(*key_ptr<KT>(r, w));
  if (!owned(r, key)) return;
  const long long base = evict_set_base(t, key);
  const int slot = warp_find(t.keys + base, kEvictWays, key, lane);
  if constexpr (kAdmit) {
    if (slot < 0 && lane == 0) {
      sketch_count(s, key);
      atomicAdd(&s.stats[0], 1ull);
    }
  }
  if (slot < 0 || lane != 0) return;
  const long long g = base + slot;
  // a hot key is touched by many warps: store the stamp once, count with one atomic each
  const unsigned long long now = *t.clock;
  if (t.stamps[g] != now) t.stamps[g] = now;
  atomicAdd(&t.counts[g], 1ull);
}

// kEvict = false (checkpoint load): only empty ways are taken, a full set drops the key.
// kAdmit: a missing key below the admission threshold is rejected before its set lock (row -1, counted).
// adm (optional): the admitted ways are appended to adm[0 .. *adm_n) for the re-initialisation.
template <typename KT, bool kEvict, bool kAdmit>
__global__ void __launch_bounds__(256) evict_insert_kernel(EvictTableView t, KeyRegion r, long long* __restrict__ adm,
                                                           int* __restrict__ adm_n, AdmitSketch s) {
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= r.n * r.ranks) return;
  KT* kp = key_ptr<KT>(r, w);
  const long long key = static_cast<long long>(*kp);
  __syncwarp();  // every lane read the key before lane 0 overwrites it
  if (!owned(r, key)) {
    if (lane == 0) *kp = static_cast<KT>(-1);
    return;
  }
  const long long base = evict_set_base(t, key);
  // A key of the running step found here stays: it was touched (protected) or inserted this step.
  int slot = warp_find(t.keys + base, kEvictWays, key, lane);
  bool admit = true;
  if constexpr (kAdmit) {
    if (slot < 0 && !sketch_admits(s, key)) {
      admit = false;
      if (lane == 0) atomicAdd(&s.stats[1], 1ull);
    }
  }
  if (slot < 0 && admit) {
    const int set = static_cast<int>(base / kEvictWays);
    lock_set(t.locks, set, lane);
    volatile long long* vk = t.keys + base;
    slot = warp_find(vk, kEvictWays, key, lane);  // a duplicate of the key may have inserted it meanwhile
    if (slot < 0) {
      const unsigned long long now = *t.clock;
      const long long k = vk[lane];
      const unsigned long long st = reinterpret_cast<volatile unsigned long long*>(t.stamps)[base + lane];
      const unsigned long long cnt = reinterpret_cast<volatile unsigned long long*>(t.counts)[base + lane];
      // victim order: (class, count (LFU only), stamp, key); class 0 empty, 1 evictable, 2 protected
      const unsigned long long cls = k < 0 ? 0ull : ((!kEvict || st == now) ? 2ull : 1ull);
      unsigned long long a = (cls << 32) | (k >= 0 && t.lfu ? (cnt < kCountMax ? cnt : kCountMax) : 0ull);
      unsigned long long b = k < 0 ? 0ull : st;
      unsigned long long c = k < 0 ? static_cast<unsigned long long>(lane) : static_cast<unsigned long long>(k);
      int sl = lane;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long a2 = __shfl_xor_sync(0xffffffffu, a, o);
        const unsigned long long b2 = __shfl_xor_sync(0xffffffffu, b, o);
        const unsigned long long c2 = __shfl_xor_sync(0xffffffffu, c, o);
        const int sl2 = __shfl_xor_sync(0xffffffffu, sl, o);
        if (a2 < a || (a2 == a && (b2 < b || (b2 == b && c2 < c)))) {
          a = a2;
          b = b2;
          c = c2;
          sl = sl2;
        }
      }
      const unsigned long long vcls = a >> 32;
      if (vcls == 2) {
        if (lane == 0) atomicAdd(&t.stats[2], 1ull);
      } else {
        slot = sl;
        if (lane == 0) {
          const long long g = base + slot;
          atomicAdd(&t.stats[0], 1ull);
          if (vcls == 1) atomicAdd(&t.stats[1], 1ull);
          t.keys[g] = key;
          t.stamps[g] = now;
          t.counts[g] = 1ull;
          if (adm) adm[atomicAdd(adm_n, 1)] = g;
        }
      }
    }
    unlock_set(t.locks, set, lane);
  }
  if (lane == 0) *kp = static_cast<KT>(slot >= 0 ? base + slot : -1);
}

template <typename KT>
__global__ void __launch_bounds__(256) evict_get_kernel(EvictTableView t, KeyRegion r) {
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= r.n * r.ranks) return;
  KT* kp = key_ptr<KT>(r, w);
  const long long key = static_cast<long long>(*kp);
  __syncwarp();
  int slot = -1;
  long long base = 0;
  if (owned(r, key)) {
    base = evict_set_base(t, key);
    slot = warp_find(t.keys + base, kEvictWays, key, lane);
  }
  if (lane == 0) *kp = static_cast<KT>(slot >= 0 ? base + slot : -1);
}

__global__ void evict_dump_kernel(const long long* __restrict__ keys, long long capacity,
                                  long long* __restrict__ out_keys, long long* __restrict__ out_slots,
                                  unsigned long long* out_n) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= capacity) return;
  const long long k = keys[i];
  if (k >= 0) {
    const unsigned long long p = atomicAdd(out_n, 1ull);
    out_keys[p] = k;
    out_slots[p] = i;
  }
}

// Initial weights of an admitted key: bound * (2u - 1), u = the top 24 bits of a stateless hash of
// (seed, table, key, global column) over 2^24, bf16 arenas rounded to nearest.  A returning key gets
// the same row whatever the sharding plan.  Mirrored bit for bit by embedding/ops.py (evict_init_rows).
HCTR_DEVICE float evict_init_value(unsigned long long init_key, long long key, int col, float bound) {
  const unsigned long long h = fmix64(fmix64(init_key ^ static_cast<unsigned long long>(key)) ^
                                      static_cast<unsigned long long>(col));
  const float u = static_cast<float>(h >> 40) * (1.0f / 16777216.0f);
  return __fmul_rn(bound, __fsub_rn(__fmul_rn(2.0f, u), 1.0f));
}

struct EvictReinit {
  const long long* keys;  // the shard's way keys
  const long long* adm;   // admitted ways
  const int* adm_n;
  void* table;            // arena (fp32 or bf16), row pitch `pitch`
  void* s0;               // optional, pitch s0_pitch (1: row-wise)
  void* s1;               // optional, pitch `pitch` (s1_row: fp32, one value per row)
  long long row_off;      // first arena row of the shard
  unsigned long long init_key;
  float bound, s0_init;
  int pitch, col0, s0_pitch, state_bf16;
  int s1_row;             // 1: s1 is fp32 with one value per row (partial row-wise Adam's second moment)
};

HCTR_DEVICE void store_state(void* p, long long i, float v, int bf16) {
  if (bf16)
    static_cast<__nv_bfloat16*>(p)[i] = __float2bfloat16_rn(v);
  else
    static_cast<float*>(p)[i] = v;
}

// S1_ROW: p.s1_row is set (the other instantiations are those of the optimizers with per-element states)
template <typename WT, bool S1_ROW>
__global__ void __launch_bounds__(256) evict_reinit_kernel(EvictReinit p) {
  const int lane = threadIdx.x & 31;
  const int n = *p.adm_n;
  for (long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; i < n;
       i += (static_cast<long long>(gridDim.x) * blockDim.x) >> 5) {
    const long long g = p.adm[i];
    const long long key = p.keys[g];
    const long long row = p.row_off + g;
    WT* w = static_cast<WT*>(p.table) + row * p.pitch;
    for (int c = lane; c < p.pitch; c += 32) {
      const float v = evict_init_value(p.init_key, key, p.col0 + c, p.bound);
      if constexpr (sizeof(WT) == 2)
        w[c] = __float2bfloat16_rn(v);
      else
        w[c] = v;
      if constexpr (!S1_ROW)
        if (p.s1) store_state(p.s1, row * p.pitch + c, 0.0f, p.state_bf16);
    }
    if (p.s0)
      for (int c = lane; c < p.s0_pitch; c += 32) store_state(p.s0, row * p.s0_pitch + c, p.s0_init, p.state_bf16);
    if constexpr (S1_ROW)
      if (lane == 0) static_cast<float*>(p.s1)[row] = 0.0f;
  }
}

template <template <typename> class K, typename... A>
int launch_by_key(const KeyRegion& r, cudaStream_t st, A... a) {
  const long long n = r.n * r.ranks;
  if (n <= 0) return 0;
  const unsigned grid = static_cast<unsigned>((n * 32 + 255) / 256);
  if (r.key_bytes == 8)
    K<long long>::launch(grid, st, r, a...);
  else if (r.key_bytes == 4)
    K<int>::launch(grid, st, r, a...);
  else
    return -1;
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// s: the shard's admission sketch, or nullptr (no admission: today's instantiations)
template <typename KT>
struct TouchL {
  static void launch(unsigned g, cudaStream_t st, const KeyRegion& r, const EvictTableView& t, const AdmitSketch* s) {
    if (s)
      evict_touch_kernel<KT, true><<<g, 256, 0, st>>>(t, r, *s);
    else
      evict_touch_kernel<KT, false><<<g, 256, 0, st>>>(t, r, AdmitSketch{});
  }
};
template <typename KT>
struct InsertL {
  static void launch(unsigned g, cudaStream_t st, const KeyRegion& r, const EvictTableView& t, long long* adm,
                     int* adm_n, int evict, const AdmitSketch* s) {
    if (s && evict)
      evict_insert_kernel<KT, true, true><<<g, 256, 0, st>>>(t, r, adm, adm_n, *s);
    else if (evict)
      evict_insert_kernel<KT, true, false><<<g, 256, 0, st>>>(t, r, adm, adm_n, AdmitSketch{});
    else
      evict_insert_kernel<KT, false, false><<<g, 256, 0, st>>>(t, r, adm, adm_n, AdmitSketch{});
  }
};
template <typename KT>
struct GetL {
  static void launch(unsigned g, cudaStream_t st, const KeyRegion& r, const EvictTableView& t) {
    evict_get_kernel<KT><<<g, 256, 0, st>>>(t, r);
  }
};

}  // namespace hctr

using namespace hctr;

// s (optional): the admission sketch of an admitting shard; the insert applies it only when evicting
extern "C" int hctr_evict_touch(const EvictTableView* t, const KeyRegion* r, const AdmitSketch* s, void* stream) {
  return launch_by_key<TouchL>(*r, (cudaStream_t)stream, *t, s);
}

extern "C" int hctr_evict_insert(const EvictTableView* t, const KeyRegion* r, long long* adm, int* adm_n,
                                 int evict, const AdmitSketch* s, void* stream) {
  return launch_by_key<InsertL>(*r, (cudaStream_t)stream, *t, adm, adm_n, evict, s);
}

extern "C" int hctr_evict_get(const EvictTableView* t, const KeyRegion* r, void* stream) {
  return launch_by_key<GetL>(*r, (cudaStream_t)stream, *t);
}

extern "C" int hctr_evict_dump(const long long* keys, long long capacity, long long* out_keys, long long* out_slots,
                               void* out_n, void* stream) {
  if (capacity <= 0) return 0;
  evict_dump_kernel<<<(unsigned)((capacity + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      keys, capacity, out_keys, out_slots, (unsigned long long*)out_n);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// max_adm: length of the admitted list (sizes the grid; the kernel reads the count from the device)
extern "C" int hctr_evict_reinit(const EvictReinit* p, long long max_adm, int table_bf16, void* stream) {
  if (max_adm <= 0) return 0;
  const long long warps = max_adm < 8192 ? max_adm : 8192;
  const unsigned grid = static_cast<unsigned>((warps * 32 + 255) / 256);
  auto launch = [&](auto s1_row) {
    if (table_bf16)
      evict_reinit_kernel<__nv_bfloat16, decltype(s1_row)::value><<<grid, 256, 0, (cudaStream_t)stream>>>(*p);
    else
      evict_reinit_kernel<float, decltype(s1_row)::value><<<grid, 256, 0, (cudaStream_t)stream>>>(*p);
  };
  if (p->s1_row && p->s1)
    launch(std::true_type{});
  else
    launch(std::false_type{});
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
