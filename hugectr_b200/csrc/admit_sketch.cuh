// Admission sketch of the dynamic embedding-collection tables with admit_threshold > 1: a count-min
// sketch per row shard, 4 rows of `width` saturating uint32 counters (width a power of two).  A training
// lookup counts every owned occurrence of a key that has no row (before any insert of the step), and a
// missing key is offered to the table's insert only when the minimum of its four counters reaches the
// threshold.  Semantics in docs/embedding.md; mirrored bit for bit by embedding/hashtable.py (AdmitSketch).
#pragma once
#include <cuda_runtime.h>

#include "embedding.cuh"

namespace hctr {

constexpr int kSketchRows = 4;
constexpr unsigned int kSketchMax = 0xFFFFFFFFu;
// salt of the sketch hash: its bits are independent of hash64(key), which picks a key's evicting set
// and its growing-table slot
constexpr unsigned long long kSketchSalt = 0x9E3779B97F4A7C15ull;

struct AdmitSketch {
  unsigned int* counters;     // [kSketchRows * width] row-major
  unsigned long long* stats;  // [2] counted occurrences, rejected positions (cumulative)
  unsigned int width_mask;    // width - 1
  unsigned int threshold;
};

// counter of `key` in sketch row `row`: double hashing of h = fmix64(key ^ salt),
// column (lo32(h) + row * (hi32(h) | 1)) mod width
HCTR_DEVICE unsigned int* sketch_counter(const AdmitSketch& s, long long key, int row) {
  const unsigned long long h = fmix64(static_cast<unsigned long long>(key) ^ kSketchSalt);
  const unsigned int col = (static_cast<unsigned int>(h) + static_cast<unsigned int>(row) *
                                                               (static_cast<unsigned int>(h >> 32) | 1u)) &
                           s.width_mask;
  return s.counters + static_cast<long long>(row) * (s.width_mask + 1ull) + col;
}

// one occurrence of a missing key: +1 on its four counters, saturating at kSketchMax (an add that
// wrapped a full counter puts it back; no other add can leave it below the maximum afterwards)
HCTR_DEVICE void sketch_count(const AdmitSketch& s, long long key) {
#pragma unroll
  for (int r = 0; r < kSketchRows; ++r) {
    unsigned int* c = sketch_counter(s, key, r);
    if (atomicAdd(c, 1u) == kSketchMax) atomicExch(c, kSketchMax);
  }
}

// whether a missing key may take a row: min of its counters >= threshold (read after every count of the step)
HCTR_DEVICE bool sketch_admits(const AdmitSketch& s, long long key) {
  unsigned int m = kSketchMax;
#pragma unroll
  for (int r = 0; r < kSketchRows; ++r) m = min(m, *sketch_counter(s, key, r));
  return m >= s.threshold;
}

}  // namespace hctr
