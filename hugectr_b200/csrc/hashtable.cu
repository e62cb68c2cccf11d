// S1: persistent open-addressing hash table (key -> dense row index) for the legacy
// SparseEmbedding path and dynamic tables.  API parity with HashTable<Key,size_t>
// (HugeCTR/src/hashtable/nv_hashtable.cu:36-306): get_insert (new keys receive the next row from an
// atomic counter), get (lookup only; missing -> -1, the reference's "get_mark"), insert/set, dump,
// get_size.  Capacity = max_vocabulary_size / load_factor slots (nv_hashtable.hpp:179).
#include <cuda_runtime.h>
#include <stdint.h>

#include "admit_sketch.cuh"
#include "embedding.cuh"

namespace hctr {

struct HashTableView {
  unsigned long long* keys;   // [capacity] kEmptyKey = empty
  long long* vals;            // [capacity] row index (-1 while being inserted)
  unsigned long long* counter;  // [1] next row index == size
  unsigned long long capacity_mask;
  long long max_rows;         // rows beyond this are an overflow (check_overflow)
};

// Bounded: a full table can neither spin (probe count <= capacity) nor hand out rows past max_rows --
// both cases return -1 and raise the sticky ``overflow`` flag that check_overflow() reads on the host
// outside the step (no per-step host sync; the step stays graph capturable).
__global__ void ht_get_insert_kernel(HashTableView t, const long long* __restrict__ keys,
                                     long long* __restrict__ out, long long n, int insert,
                                     unsigned int* __restrict__ overflow) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long key = keys[i];
  if (key < 0) {
    out[i] = -1;
    return;
  }
  const unsigned long long k = static_cast<unsigned long long>(key);
  unsigned long long h = hash64(k) & t.capacity_mask;
  for (unsigned long long probes = 0; probes <= t.capacity_mask; ++probes) {
    unsigned long long prev = *reinterpret_cast<volatile unsigned long long*>(&t.keys[h]);
    if (prev == kEmptyKey && insert) {
      // rows are exhausted: do not consume another key slot (the table would fill up and probing
      // would never terminate), report the overflow instead
      if (static_cast<long long>(*reinterpret_cast<volatile unsigned long long*>(t.counter)) >= t.max_rows) {
        if (overflow) atomicMax(overflow, 1u);
        out[i] = -1;
        return;
      }
      prev = atomicCAS(&t.keys[h], kEmptyKey, k);
    }
    if (prev == kEmptyKey) {
      if (!insert) {
        out[i] = -1;
        return;
      }
      const unsigned long long row = atomicAdd(t.counter, 1ull);
      atomicExch(reinterpret_cast<unsigned long long*>(&t.vals[h]), row);
      const bool ok = static_cast<long long>(row) < t.max_rows;
      if (!ok && overflow) atomicMax(overflow, 1u);
      out[i] = ok ? static_cast<long long>(row) : -1;
      return;
    }
    if (prev == k) {
      long long v;
      do {
        v = *reinterpret_cast<volatile long long*>(&t.vals[h]);
      } while (v < 0);
      out[i] = v < t.max_rows ? v : -1;
      return;
    }
    h = (h + 1) & t.capacity_mask;
  }
  if (overflow) atomicMax(overflow, 1u);
  out[i] = -1;
}

// Ownership filter + translation in one pass over an inbox of gathered keys [ranks x n_per_rank]
// (legacy embeddings on the fused path): a key is translated iff this rank owns it,
//   Distributed  key % key_mod == key_rem
//   Localized    ((position / slot_div) % slot_num) % key_mod == key_rem     (slot of the key's position)
// everything else becomes -1.  Same bounded insert as ht_get_insert_kernel.
struct OwnFilter {
  long long n_per_rank;
  int key_mod, key_rem;      // key_mod <= 1: no key filter
  int slot_div, slot_num;    // slot_num <= 0: no slot filter
};
__global__ void ht_translate_kernel(HashTableView t, const long long* __restrict__ keys,
                                    long long* __restrict__ out, long long n, int insert,
                                    unsigned int* __restrict__ overflow, OwnFilter f) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long key = keys[i];
  bool own = key >= 0;
  if (own && f.slot_num > 0) {
    const long long pos = i % f.n_per_rank;
    own = (((pos / f.slot_div) % f.slot_num) % f.key_mod) == f.key_rem;
  } else if (own && f.key_mod > 1) {
    own = static_cast<int>(static_cast<unsigned long long>(key) % static_cast<unsigned long long>(f.key_mod)) ==
          f.key_rem;
  }
  if (!own) {
    out[i] = -1;
    return;
  }
  const unsigned long long k = static_cast<unsigned long long>(key);
  unsigned long long h = hash64(k) & t.capacity_mask;
  for (unsigned long long probes = 0; probes <= t.capacity_mask; ++probes) {
    unsigned long long prev = *reinterpret_cast<volatile unsigned long long*>(&t.keys[h]);
    if (prev == kEmptyKey && insert) {
      if (static_cast<long long>(*reinterpret_cast<volatile unsigned long long*>(t.counter)) >= t.max_rows) {
        if (overflow) atomicMax(overflow, 1u);
        out[i] = -1;
        return;
      }
      prev = atomicCAS(&t.keys[h], kEmptyKey, k);
    }
    if (prev == kEmptyKey) {
      if (!insert) {
        out[i] = -1;
        return;
      }
      const unsigned long long row = atomicAdd(t.counter, 1ull);
      atomicExch(reinterpret_cast<unsigned long long*>(&t.vals[h]), row);
      const bool ok = static_cast<long long>(row) < t.max_rows;
      if (!ok && overflow) atomicMax(overflow, 1u);
      out[i] = ok ? static_cast<long long>(row) : -1;
      return;
    }
    if (prev == k) {
      long long v;
      do {
        v = *reinterpret_cast<volatile long long*>(&t.vals[h]);
      } while (v < 0);
      out[i] = v < t.max_rows ? v : -1;
      return;
    }
    h = (h + 1) & t.capacity_mask;
  }
  if (overflow) atomicMax(overflow, 1u);
  out[i] = -1;
}

// ---- admission of a growing dynamic table (admit_threshold > 1, admit_sketch.cuh).  A training lookup runs
// the count kernel over every key region of the table, then the filter kernel and the get-insert per region.

// whether `key` has a slot (read-only probe; no insert of the table runs concurrently)
HCTR_DEVICE bool ht_has(const HashTableView& t, unsigned long long k) {
  unsigned long long h = hash64(k) & t.capacity_mask;
  for (unsigned long long probes = 0; probes <= t.capacity_mask; ++probes) {
    const unsigned long long prev = t.keys[h];
    if (prev == k) return true;
    if (prev == kEmptyKey) return false;
    h = (h + 1) & t.capacity_mask;
  }
  return false;
}

// keys >= 0 (the owned ones) without a slot count one occurrence each
__global__ void __launch_bounds__(256) ht_admit_count_kernel(HashTableView t, const long long* __restrict__ keys,
                                                             long long n, AdmitSketch s) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long key = i < n ? keys[i] : -1;
  const bool miss = key >= 0 && !ht_has(t, static_cast<unsigned long long>(key));
  if (miss) sketch_count(s, key);
  const unsigned m = __ballot_sync(0xffffffffu, miss);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&s.stats[0], static_cast<unsigned long long>(__popc(m)));
}

// keys >= 0 without a slot whose count is below the threshold become -1 (rejected, counted), in place
__global__ void __launch_bounds__(256) ht_admit_filter_kernel(HashTableView t, long long* __restrict__ keys,
                                                              long long n, AdmitSketch s) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long key = i < n ? keys[i] : -1;
  const bool rej = key >= 0 && !ht_has(t, static_cast<unsigned long long>(key)) && !sketch_admits(s, key);
  if (rej) keys[i] = -1;
  const unsigned m = __ballot_sync(0xffffffffu, rej);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&s.stats[1], static_cast<unsigned long long>(__popc(m)));
}

__global__ void ht_set_kernel(HashTableView t, const long long* __restrict__ keys,
                              const long long* __restrict__ vals, long long n) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = static_cast<unsigned long long>(keys[i]);
  unsigned long long h = hash64(k) & t.capacity_mask;
  while (true) {
    const unsigned long long prev = atomicCAS(&t.keys[h], kEmptyKey, k);
    if (prev == kEmptyKey || prev == k) {
      t.vals[h] = vals[i];
      return;
    }
    h = (h + 1) & t.capacity_mask;
  }
}

__global__ void ht_dump_kernel(HashTableView t, long long* __restrict__ out_keys,
                               long long* __restrict__ out_vals, unsigned long long* out_count,
                               unsigned long long capacity) {
  const unsigned long long i = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= capacity) return;
  const unsigned long long k = t.keys[i];
  if (k != kEmptyKey) {
    const unsigned long long pos = atomicAdd(out_count, 1ull);
    out_keys[pos] = static_cast<long long>(k);
    out_vals[pos] = t.vals[i];
  }
}

}  // namespace hctr

using namespace hctr;

extern "C" int hctr_ht_get_insert(void* keys_tab, void* vals_tab, void* counter,
                                  unsigned long long capacity, long long max_rows,
                                  const long long* keys, long long* out, long long n, int insert,
                                  void* stream, void* overflow) {
  if (n == 0) return 0;
  HashTableView t{(unsigned long long*)keys_tab, (long long*)vals_tab, (unsigned long long*)counter,
                  capacity - 1, max_rows};
  ht_get_insert_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      t, keys, out, n, insert, reinterpret_cast<unsigned int*>(overflow));
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int hctr_ht_translate(void* keys_tab, void* vals_tab, void* counter, unsigned long long capacity,
                                 long long max_rows, const long long* keys, long long* out, long long n,
                                 int insert, void* overflow, long long n_per_rank, int key_mod, int key_rem,
                                 int slot_div, int slot_num, void* stream) {
  if (n == 0) return 0;
  HashTableView t{(unsigned long long*)keys_tab, (long long*)vals_tab, (unsigned long long*)counter,
                  capacity - 1, max_rows};
  OwnFilter f{n_per_rank, key_mod, key_rem, slot_div, slot_num};
  ht_translate_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      t, keys, out, n, insert, reinterpret_cast<unsigned int*>(overflow), f);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int hctr_ht_set(void* keys_tab, void* vals_tab, void* counter, unsigned long long capacity,
                           const long long* keys, const long long* vals, long long n, void* stream) {
  if (n == 0) return 0;
  HashTableView t{(unsigned long long*)keys_tab, (long long*)vals_tab, (unsigned long long*)counter,
                  capacity - 1, 0x7fffffffffffffffll};
  ht_set_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(t, keys, vals, n);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int hctr_ht_dump(void* keys_tab, void* vals_tab, unsigned long long capacity,
                            long long* out_keys, long long* out_vals, void* out_count, void* stream) {
  HashTableView t{(unsigned long long*)keys_tab, (long long*)vals_tab, nullptr, capacity - 1, 0};
  ht_dump_kernel<<<(unsigned)((capacity + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      t, out_keys, out_vals, (unsigned long long*)out_count, capacity);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// filter = 0: count the missing keys of `keys`; 1: reject the missing keys below the threshold (in place)
extern "C" int hctr_ht_admit(void* keys_tab, unsigned long long capacity, long long* keys, long long n,
                             const AdmitSketch* sketch, int filter, void* stream) {
  if (n == 0) return 0;
  HashTableView t{(unsigned long long*)keys_tab, nullptr, nullptr, capacity - 1, 0};
  const unsigned grid = (unsigned)((n + 255) / 256);
  if (filter)
    ht_admit_filter_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(t, keys, n, *sketch);
  else
    ht_admit_count_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(t, keys, n, *sketch);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
