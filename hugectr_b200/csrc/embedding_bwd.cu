// F2: fused embedding backward -- gradient gather ("all-to-all" by peer loads), duplicate-row
// reduction and sparse optimizer in ONE pass over each unique row, with no sort and no float
// atomics on the common path.
//
//   index   (independent of gradients -> overlappable with dense fwd/bwd, like the reference's
//            index calculation on the "dp" stream, model_pipeline.cpp:189-193,303)
//     A  per (bucket,key): uid = hash get_insert(arena row); count[uid]++ ; pair_uid[pair] = uid
//     B  exclusive scan of count -> offsets                      (3 small kernels)
//     C  per pair: bucket_list[offsets[uid] + --count[uid]] = bucket id      (counting sort)
//   reduce+update
//     D1 one warp per unique row: sum the bf16 gradient rows of its buckets (read from the
//        requesters' top-grad tensors: local L2 or peer HBM over NVLink), apply the optimizer,
//        write weight + state, free the hash slot.  Rows with > kHeavy buckets are deferred:
//     D2 heavy rows (power-law heads): kChunk-bucket chunks are reduced by separate blocks,
//        combined with fp32 red.add into a scratch row; the last chunk applies the optimizer.
//
// Replaces the reference chain NetworkBackward -> NCCL all-to-all -> CUB radix/segmented sorts ->
// unique -> multi_to_one_reduce -> update4_kernel
// (HugeCTR/embedding/operators/index_calculation.cu:102-887, multi_to_one_reduce*.cuh,
//  HugeCTR/embedding_storage/ragged_static_embedding.cu:93-345).
#include "embedding.cuh"

namespace hctr {

constexpr int kHeavy = 64;     // buckets per row handled by a single warp
constexpr int kChunk = 512;    // buckets per block for heavy rows

struct BwdIndex {
  unsigned int* count;        // [max_unique] per-uid bucket count (consumed by fill)
  unsigned int* offsets;      // [max_unique + 1]
  unsigned int* block_sums;   // [ceil(max_unique / 1024) + 1]
  int* pair_uid;              // [max_pairs]
  unsigned int* bucket_list;  // [max_pairs] gradient-row locators grouped by uid:
                              //   (src rank << 28) | (element offset of the bucket's grad row >> 2)
  float* bucket_scale;        // [max_pairs] per-entry scale (mean combiner) or null when all sums
  unsigned int* heavy_items;  // [max_heavy_items * 2] (uid, chunk)
  unsigned int* heavy_count;  // [1]
  float* heavy_scratch;       // [max_heavy_rows, ev]
  unsigned int* heavy_ticket; // [max_heavy_rows]
  unsigned int* heavy_slot;   // [1] allocator of scratch rows
  unsigned int max_heavy_rows, max_heavy_items;
  uint2* light_list;          // [max_unique] (uid, offset | (count-1) << 30) of rows with <= 4 entries
  uint2* medium_list;         // [max_unique] (uid, offset) of rows with 5..kHeavy entries
  unsigned int* class_count;  // [2] light / medium list lengths
};

// ---------------------------------------------------------------- scans
HCTR_DEVICE unsigned int warp_inclusive_scan(unsigned int x, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  return x;
}
// Exclusive scan of one value per thread of a 1024-thread block.  w: 32 words of shared memory, free
// again after the caller's next __syncthreads.  Thread 1023's result plus its v is the block's total.
HCTR_DEVICE unsigned int block_exclusive_scan_1024(unsigned int v, unsigned int* w) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned int x = warp_inclusive_scan(v, lane);
  if (lane == 31) w[warp] = x;
  __syncthreads();
  if (warp == 0) w[lane] = warp_inclusive_scan(w[lane], lane);
  __syncthreads();
  return (warp ? w[warp - 1] : 0u) + x - v;
}

// ---------------------------------------------------------------- A: unique ids + counts
// Block-aggregated: a block de-duplicates its kPairsPerBlock (bucket,key) pairs in a shared-memory
// hash first, so a power-law head row costs ONE global CAS + ONE global atomicAdd per block instead
// of one per occurrence (the hottest Criteo-like row appears ~8% of the time).
constexpr int kIdxThreads = 256;
constexpr int kPairsPerThread = 4;
constexpr int kPairsPerBlock = kIdxThreads * kPairsPerThread;
constexpr int kSmemSlots = 2048;  // 2x pairs per block, power of two
constexpr int kMaxSmemLookups = 512;

struct PairInfo {
  int l, src, s, h;
};
HCTR_DEVICE PairInfo decode_pair(const EmbParams& p, const long long* s_pair_off, long long pair) {
  int lo = 0, hi = p.num_lookups - 1;
  while (lo < hi) {  // last lookup with pair_off <= pair
    const int mid = (lo + hi + 1) >> 1;
    if (s_pair_off[mid] <= pair) lo = mid; else hi = mid - 1;
  }
  PairInfo r;
  r.l = lo;
  const unsigned int rem = static_cast<unsigned int>(pair - s_pair_off[lo]);
  const unsigned int H = static_cast<unsigned int>(__ldg(&p.lookups[lo].hotness));
  const unsigned int bucket = rem / H;
  r.h = static_cast<int>(rem - bucket * H);
  r.src = static_cast<int>(bucket / static_cast<unsigned int>(p.batch));
  r.s = static_cast<int>(bucket - static_cast<unsigned int>(r.src) * static_cast<unsigned int>(p.batch));
  return r;
}

template <typename KeyT>
__global__ void __launch_bounds__(kIdxThreads)
    emb_bwd_index_kernel(const EmbParams p, const UniqueTable ut, const BwdIndex ix,
                         const long long total_pairs) {
  __shared__ unsigned long long h_keys[kSmemSlots];
  __shared__ unsigned int h_cnt[kSmemSlots];
  __shared__ long long s_pair_off[kMaxSmemLookups];
  for (int i = threadIdx.x; i < kSmemSlots; i += blockDim.x) {
    h_keys[i] = kEmptyKey;
    h_cnt[i] = 0;
  }
  for (int i = threadIdx.x; i < p.num_lookups; i += blockDim.x) s_pair_off[i] = p.lookups[i].pair_off;
  __syncthreads();
  const long long base = static_cast<long long>(blockIdx.x) * kPairsPerBlock;
  int slot[kPairsPerThread];
#pragma unroll
  for (int q = 0; q < kPairsPerThread; ++q) {
    slot[q] = -1;
    const long long pair = base + q * kIdxThreads + threadIdx.x;
    if (pair >= total_pairs) continue;
    const PairInfo pi = decode_pair(p, s_pair_off, pair);
    const EmbLookup* lk = p.lookups + pi.l;
    if (pi.h >= bucket_nnz(p, __ldg(&lk->hotness), __ldg(&lk->nnz_off), pi.src, pi.s)) continue;
    const KeyT* kp = reinterpret_cast<const KeyT*>(p.keys[pi.src]) + __ldg(&lk->key_off) +
                     static_cast<long long>(pi.s) * __ldg(&lk->key_stride) + pi.h;
    const long long key = static_cast<long long>(*kp);
    const int ns = __ldg(&lk->num_shards);
    if (key < 0) continue;
    long long r = key;
    if (ns > 1) {
      if ((key % ns) != __ldg(&lk->shard_idx)) continue;
      r = key / ns;
    }
    if (r >= __ldg(&lk->rows)) continue;
    const unsigned long long arow = static_cast<unsigned long long>(__ldg(&lk->table_row_off) + r);
    unsigned int hslot = hash64(arow) & (kSmemSlots - 1);
    while (true) {
      const unsigned long long prev = atomicCAS(&h_keys[hslot], kEmptyKey, arow);
      if (prev == kEmptyKey || prev == arow) break;
      hslot = (hslot + 1) & (kSmemSlots - 1);
    }
    atomicAdd(&h_cnt[hslot], 1u);
    slot[q] = static_cast<int>(hslot);
  }
  __syncthreads();
  // One global insert per distinct row of the block.  Unique ids are handed out with ONE atomicAdd
  // on the global counter per block (a per-key atomicAdd on that single address serialises in L2
  // and was the whole kernel's critical path): (1) claim / find the global hash slot of every
  // distinct row without waiting, (2) block-scan the number of newly claimed rows, reserve the id
  // range, publish the ids, (3) only then wait for ids owned by other blocks -- every block
  // publishes before it waits, so the waits cannot form a cycle.
  constexpr int kSlotIters = kSmemSlots / kIdxThreads;
  unsigned int gslot[kSlotIters];
  unsigned int newmask = 0, nnew = 0;
#pragma unroll
  for (int k = 0; k < kSlotIters; ++k) {
    const unsigned long long key = h_keys[threadIdx.x + k * kIdxThreads];
    gslot[k] = kInvalidVal;
    if (key != kEmptyKey) {
      unsigned int h = hash64(key) & ut.mask;
      while (true) {
        const unsigned long long prev = atomicCAS(&ut.keys[h], kEmptyKey, key);
        if (prev == kEmptyKey) {
          newmask |= 1u << k;
          ++nnew;
          break;
        }
        if (prev == key) break;
        h = (h + 1) & ut.mask;
      }
      gslot[k] = h;
    }
  }
  __shared__ unsigned int s_warp_sum[kIdxThreads / 32];
  __shared__ unsigned int s_base;
  const unsigned int incl = warp_inclusive_scan(nnew, threadIdx.x & 31);
  if ((threadIdx.x & 31) == 31) s_warp_sum[threadIdx.x >> 5] = incl;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int tot = 0;
#pragma unroll
    for (int w = 0; w < kIdxThreads / 32; ++w) {
      const unsigned int v = s_warp_sum[w];
      s_warp_sum[w] = tot;
      tot += v;
    }
    s_base = tot ? atomicAdd(ut.counter, tot) : 0u;
  }
  __syncthreads();
  unsigned int next_uid = s_base + s_warp_sum[threadIdx.x >> 5] + incl - nnew;
#pragma unroll
  for (int k = 0; k < kSlotIters; ++k) {
    if (newmask & (1u << k)) {
      const unsigned int uid = next_uid++;
      const unsigned int h = gslot[k];
      if (uid < ut.max_unique) {
        ut.rows[uid] = h_keys[threadIdx.x + k * kIdxThreads];
        ut.slots[uid] = h;
      }
      // rows[]/slots[] are consumed by later kernels only; concurrent blocks need the id alone
      atomicExch(&ut.vals[h], uid);
      gslot[k] = uid | 0x80000000u;  // resolved (ids are < 2^31)
    }
  }
#pragma unroll
  for (int k = 0; k < kSlotIters; ++k) {
    const int i = threadIdx.x + k * kIdxThreads;
    if (h_keys[i] == kEmptyKey) continue;
    unsigned int u;
    if (gslot[k] & 0x80000000u) {
      u = gslot[k] & 0x7FFFFFFFu;
    } else {
      const volatile unsigned int* vp = reinterpret_cast<volatile unsigned int*>(&ut.vals[gslot[k]]);
      do {
        u = *vp;
      } while (u == kInvalidVal);
    }
    if (u < ut.max_unique) {
      atomicAdd(&ix.count[u], h_cnt[i]);
      h_cnt[i] = u;
    } else {
      h_cnt[i] = kInvalidVal;
    }
  }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < kPairsPerThread; ++q) {
    const long long pair = base + q * kIdxThreads + threadIdx.x;
    if (pair >= total_pairs) continue;
    int uid = -1;
    if (slot[q] >= 0) {
      const unsigned int u = h_cnt[slot[q]];
      uid = (u == kInvalidVal) ? -1 : static_cast<int>(u);
    }
    ix.pair_uid[pair] = uid;
  }
}

// ---------------------------------------------------------------- B: exclusive scan (3 phases)
__global__ void __launch_bounds__(1024)
    scan_block_sums_kernel(const unsigned int* __restrict__ in, unsigned int* __restrict__ sums,
                           const unsigned int* n_ptr, unsigned int max_n) {
  const unsigned int n = min(*n_ptr, max_n);
  const unsigned int i = blockIdx.x * 1024 + threadIdx.x;
  if (blockIdx.x * 1024 >= n) return;
  unsigned int v = i < n ? in[i] : 0u;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __shared__ unsigned int w[32];
  if ((threadIdx.x & 31) == 0) w[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    unsigned int x = w[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if (threadIdx.x == 0) sums[blockIdx.x] = x;
  }
}
__global__ void __launch_bounds__(1024)
    scan_sums_kernel(unsigned int* sums, const unsigned int* n_ptr, unsigned int max_n,
                     unsigned int* heavy_count, unsigned int* heavy_slot, unsigned int* class_count) {
  // single block: exclusive scan of the block sums in place
  const unsigned int n = min(*n_ptr, max_n);
  const unsigned int nb = (n + 1023) / 1024;
  __shared__ unsigned int carry_s;
  __shared__ unsigned int w[32];
  if (threadIdx.x == 0) {
    carry_s = 0;
    *heavy_count = 0;
    *heavy_slot = 0;
    class_count[0] = 0;
    class_count[1] = 0;
  }
  __syncthreads();
  for (unsigned int base = 0; base < nb; base += 1024) {
    const unsigned int i = base + threadIdx.x;
    const unsigned int v = i < nb ? sums[i] : 0u;
    const unsigned int scan = block_exclusive_scan_1024(v, w);
    const unsigned int excl = carry_s + scan;
    if (i < nb) sums[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = excl + v;
    __syncthreads();
  }
}
__global__ void __launch_bounds__(1024)
    scan_apply_kernel(const unsigned int* __restrict__ in, const unsigned int* __restrict__ sums,
                      unsigned int* __restrict__ offsets, const unsigned int* n_ptr,
                      unsigned int max_n) {
  const unsigned int n = min(*n_ptr, max_n);
  if (blockIdx.x * 1024 >= n) return;
  const unsigned int i = blockIdx.x * 1024 + threadIdx.x;
  const unsigned int v = i < n ? in[i] : 0u;
  __shared__ unsigned int w[32];
  const unsigned int scan = block_exclusive_scan_1024(v, w);
  const unsigned int excl = sums[blockIdx.x] + scan;
  if (i < n) offsets[i] = excl;
  if (i == n - 1) offsets[n] = excl + v;
}

// ---------------------------------------------------------------- C: fill (counting sort)
// Same block aggregation: positions inside a row's bucket list are reserved once per (block, row).
// An entry's scale is 1/nnz for a mean bag, times the key's weight for a weighted lookup (WGT).
template <bool WGT>
__global__ void __launch_bounds__(kIdxThreads)
    emb_bwd_fill_kernel(const EmbParams p, const BwdIndex ix, const long long total_pairs) {
  __shared__ unsigned int h_uid[kSmemSlots];
  __shared__ unsigned int h_cnt[kSmemSlots];
  __shared__ long long s_pair_off[kMaxSmemLookups];
  for (int i = threadIdx.x; i < kSmemSlots; i += blockDim.x) {
    h_uid[i] = kInvalidVal;
    h_cnt[i] = 0;
  }
  for (int i = threadIdx.x; i < p.num_lookups; i += blockDim.x) s_pair_off[i] = p.lookups[i].pair_off;
  __syncthreads();
  const long long base = static_cast<long long>(blockIdx.x) * kPairsPerBlock;
  int slot[kPairsPerThread];
  unsigned int rank_local[kPairsPerThread];
#pragma unroll
  for (int q = 0; q < kPairsPerThread; ++q) {
    slot[q] = -1;
    const long long pair = base + q * kIdxThreads + threadIdx.x;
    if (pair >= total_pairs) continue;
    const int uid = ix.pair_uid[pair];
    if (uid < 0) continue;
    unsigned int hslot = (static_cast<unsigned int>(uid) * 2654435761u) & (kSmemSlots - 1);
    while (true) {
      const unsigned int prev = atomicCAS(&h_uid[hslot], kInvalidVal, static_cast<unsigned int>(uid));
      if (prev == kInvalidVal || prev == static_cast<unsigned int>(uid)) break;
      hslot = (hslot + 1) & (kSmemSlots - 1);
    }
    rank_local[q] = atomicAdd(&h_cnt[hslot], 1u);
    slot[q] = static_cast<int>(hslot);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kSmemSlots; i += blockDim.x) {
    const unsigned int u = h_uid[i];
    if (u != kInvalidVal) {
      const unsigned int c = h_cnt[i];
      // reserve c consecutive positions at the tail of row u's list (count runs down to zero)
      h_cnt[i] = ix.offsets[u] + atomicSub(&ix.count[u], c) - c;
    }
  }
  __syncthreads();
#pragma unroll
  for (int q = 0; q < kPairsPerThread; ++q) {
    if (slot[q] < 0) continue;
    const long long pair = base + q * kIdxThreads + threadIdx.x;
    const PairInfo pi = decode_pair(p, s_pair_off, pair);
    const EmbLookup* lk = p.lookups + pi.l;
    const long long goff = __ldg(&lk->grad_off) + static_cast<long long>(pi.s) * __ldg(&lk->grad_stride);
    const unsigned int pos = h_cnt[slot[q]] + rank_local[q];
    ix.bucket_list[pos] = (static_cast<unsigned int>(pi.src) << 28) | static_cast<unsigned int>(goff >> 2);
    if (ix.bucket_scale != nullptr) {
      float sc = 1.f;
      if (__ldg(&lk->combiner) == 1) {
        const int nnz = bucket_nnz(p, __ldg(&lk->hotness), __ldg(&lk->nnz_off), pi.src, pi.s);
        sc = 1.f / static_cast<float>(max(nnz, 1));
      }
      if constexpr (WGT) sc *= key_weight(p, *lk, pi.src, pi.s, pi.h);
      ix.bucket_scale[pos] = sc;
    }
  }
}

// ---------------------------------------------------------------- D: reduce + optimizer
template <typename GradT>
HCTR_DEVICE const GradT* locate_grad(const EmbParams& p, unsigned int e) {
  return reinterpret_cast<const GradT*>(p.grad[e >> 28]) + (static_cast<long long>(e & 0x0FFFFFFFu) << 2);
}

// The gather of the update kernels: gather_add issues the gradient loads of N bucket-list entries at one
// column, then adds the scaled rows to acc in index order (kNoEntry: an absent entry, adds zero).  Every
// caller walks a row's entries in list order, which fixes the fp32 sum bit for bit.
constexpr unsigned int kNoEntry = 0xFFFFFFFFu;
template <typename GradT, int N>
HCTR_DEVICE void gather_add(float4& acc, const EmbParams& p, const unsigned int (&ent)[N],
                            const float (&sc)[N], int col) {
  float4 g[N];
#pragma unroll
  for (int u = 0; u < N; ++u)
    g[u] = ent[u] != kNoEntry ? load_vec4<GradT>(locate_grad<GradT>(p, ent[u]) + col)
                              : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int u = 0; u < N; ++u) {
    acc.x += g[u].x * sc[u]; acc.y += g[u].y * sc[u];
    acc.z += g[u].z * sc[u]; acc.w += g[u].w * sc[u];
  }
}
// Sum at one column of the list entries first, first + stride, ... below `end`, N in flight per round
// (the scale of an entry is 1 when the index has none)
template <typename GradT, int N>
HCTR_DEVICE float4 gather_list(const EmbParams& p, const BwdIndex& ix, bool has_scale, unsigned int first,
                               unsigned int stride, unsigned int end, int col) {
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (unsigned int j = first; j < end; j += N * stride) {
    unsigned int ent[N];
    float sc[N];
#pragma unroll
    for (int u = 0; u < N; ++u) {
      ent[u] = kNoEntry;
      sc[u] = 1.f;
      if (u * stride < end - j) {
        ent[u] = ix.bucket_list[j + u * stride];
        if (has_scale) sc[u] = ix.bucket_scale[j + u * stride];
      }
    }
    gather_add<GradT, N>(acc, p, ent, sc, col);
  }
  return acc;
}

// Unique rows are classified by their number of occurrences right after the offsets are known (during
// the index build, off the critical path):
//   light  (<= 4 entries, ~94 % of the rows): compact list of (uid, offset | (count-1) << 30)
//   medium (5..kHeavy):                       compact list of (uid, offset)
//   heavy  (> kHeavy):                        (uid, chunk) work items of the block-per-chunk kernel
// so that the update kernels run UNIFORM work per lane group: with the power-law tail, four rows
// sharing a warp would otherwise wait for the longest of them (2.6x measured slowdown).
// List positions are reserved with one atomicAdd per block and class.
constexpr unsigned int kLightMax = 4;
constexpr unsigned int kMaxHeavyChunks = 4096;   // heavy item = (uid, scratch slot << 12 | chunk)
__global__ void __launch_bounds__(1024)
    emb_bwd_classify_kernel(const UniqueTable ut, const BwdIndex ix) {
  __shared__ unsigned int s_cnt[2][32];
  __shared__ unsigned int s_base[2];
  const unsigned int n = min(*ut.counter, ut.max_unique);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (unsigned int base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
    const unsigned int uid = base + threadIdx.x;
    unsigned int cnt = 0, o0 = 0;
    if (uid < n) {
      o0 = ix.offsets[uid];
      cnt = ix.offsets[uid + 1] - o0;
    }
    const bool is_light = cnt >= 1 && cnt <= kLightMax;
    bool is_medium = cnt > kLightMax && cnt <= kHeavy;
    if (cnt > kHeavy) {
      // a heavy row gets a scratch row and its chunks' work items only if all of them fit (and the
      // chunk index fits its 12 bits); otherwise it falls back to the warp-per-row medium list, which
      // handles any count, so every row is updated exactly once whatever the caps
      const unsigned int nch = (cnt + kChunk - 1) / kChunk;
      bool placed = false;
      if (nch <= kMaxHeavyChunks) {
        const unsigned int slot = atomicAdd(ix.heavy_slot, 1u);
        if (slot < ix.max_heavy_rows) {
          const unsigned int hb = atomicAdd(ix.heavy_count, nch);
          placed = hb + nch <= ix.max_heavy_items;
          // items reserved past the cap by a row that does not fit are marked invalid, so the
          // heavy kernel never picks up a stale item of an earlier step
          for (unsigned int c = 0; c < nch && hb + c < ix.max_heavy_items; ++c) {
            ix.heavy_items[2 * (hb + c)] = placed ? uid : kInvalidVal;
            ix.heavy_items[2 * (hb + c) + 1] = (slot << 12) | c;
          }
        }
      }
      is_medium = !placed;
    }
    const unsigned int bl = __ballot_sync(0xffffffffu, is_light);
    const unsigned int bm = __ballot_sync(0xffffffffu, is_medium);
    if (lane == 0) {
      s_cnt[0][warp] = __popc(bl);
      s_cnt[1][warp] = __popc(bm);
    }
    __syncthreads();
    if (warp < 2) {   // warp 0 scans the light counts, warp 1 the medium counts
      const unsigned int v = s_cnt[warp][lane], x = warp_inclusive_scan(v, lane);
      s_cnt[warp][lane] = x - v;
      if (lane == 31) s_base[warp] = x ? atomicAdd(&ix.class_count[warp], x) : 0u;
    }
    __syncthreads();
    const unsigned int below = (1u << lane) - 1u;
    if (is_light) {
      const unsigned int pos = s_base[0] + s_cnt[0][warp] + __popc(bl & below);
      ix.light_list[pos] = make_uint2(uid, o0 | ((cnt - 1u) << 30));
    } else if (is_medium) {
      const unsigned int pos = s_base[1] + s_cnt[1][warp] + __popc(bm & below);
      ix.medium_list[pos] = make_uint2(uid, o0);
    }
    __syncthreads();
  }
}

// Light + medium rows: fused gradient reduction and optimizer step.
// Light part: G lanes per row (G = 8: four rows per warp, every lane owns 4 float4 chunks of the
// row), exactly one gather round per row.  The chain  record -> (arena row, bucket entries) ->
// (weight, state, gradient rows)  is software-pipelined over the rows a lane group visits: record i+2
// and the row id / entries of i+1 are in flight while row i is reduced, and the weight / state
// vectors are requested together with the gradients, so ONE DRAM latency is exposed per row.
// Medium part: one warp per row, 8 gradient rows in flight per round.
// WT: weight type of the arena (fp32, or bf16 moved 8 bytes per 4 columns and stored with stochastic
// rounding); the reduction and the optimizer run in fp32 either way.
template <int OPT, typename StateT, typename GradT, int G, typename WT>
__global__ void __launch_bounds__(256, (G == 8) ? 3 : 2)
    emb_bwd_reduce_update_kernel(const EmbParams p, const UniqueTable ut, const BwdIndex ix,
                                 StateT* __restrict__ s0, StateT* __restrict__ s1, const OptHyper hp,
                                 const float grad_scale) {
  constexpr bool kHasS0 = (OPT != OPT_SGD);
  const OptStep step = opt_step<OPT>(hp);
  const float inv_scaler = grad_scale / hp.scaler;
  const unsigned long long srk = sr_key<WT>(hp.sr_seed, hp.step_ptr);
  const int lane = threadIdx.x & 31;
  const int ev = p.ev_size;
  const bool has_scale = ix.bucket_scale != nullptr;
  const unsigned int n_light = min(ix.class_count[0], ut.max_unique);
  const unsigned int n_medium = min(ix.class_count[1], ut.max_unique);
  const unsigned int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned int num_warps = (gridDim.x * blockDim.x) >> 5;

  // ------------------------------------------------------------------ light rows
  {
    const int gl = lane % G, gi = lane / G;
    constexpr int GPW = 32 / G;
    constexpr int NC = (G == 8) ? 4 : 8;             // chunks per lane
    const unsigned int groups = num_warps * GPW;
    const unsigned int first = warp_global * GPW + gi;
    uint2 rec[3];                 // stage R: list records of rows i, i+1, i+2
    unsigned long long row[2];    // stage A: arena row of rows i, i+1
    unsigned int ent[2][4];       //          and their bucket entries / scales
    float esc[2][4];
    auto load_r = [&](unsigned int i, int k) {
      rec[k] = make_uint2(0u, 0u);
      if (i < n_light) rec[k] = ix.light_list[i];
    };
    auto load_a = [&](unsigned int i, int kr, int ka) {
      row[ka] = 0ull;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        ent[ka][u] = kNoEntry;
        esc[ka][u] = 1.f;
      }
      if (i < n_light) {
        const unsigned int o0 = rec[kr].y & 0x3FFFFFFFu, cnt = (rec[kr].y >> 30) + 1u;
        row[ka] = ut.rows[rec[kr].x];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (u < cnt) {
            ent[ka][u] = ix.bucket_list[o0 + u];
            if (has_scale) esc[ka][u] = ix.bucket_scale[o0 + u];
          }
        }
      }
    };
    load_r(first, 0);
    load_r(first + groups, 1);
    load_a(first, 0, 0);
    for (unsigned int i = first; i < n_light; i += groups) {
      load_r(i + 2 * groups, 2);
      load_a(i + groups, 1, 1);
      const unsigned int uid = rec[0].x;
      const long long base = static_cast<long long>(row[0]) * ev;
      if constexpr (kRowRule<OPT>) {
        // The row-reduced rules (row-wise AdaGrad, partial row-wise Adam) need the whole row's sum of
        // g^2 before any of its weights is stored.  The gradient sums of all NC chunks stay in
        // registers (they take the place of the per-element state vectors of the other optimizers),
        // so a row is gathered exactly once even when it spans two passes (G == 32, ev > 512).  The
        // weights of the first four chunks and the row's state (one 4-byte load by the group's first
        // lane) are requested with the gradients; a second pass loads its weights, and partial
        // row-wise Adam its first moments, once the factor is known.
        const unsigned int gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (gi * G));
        float* const rs = row_state<OPT>(s0, s1);
        typename Row4<WT>::type wv[4];
        float4 acc[NC];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int col = (c * G + gl) * 4;
          wv[c] = {};
          if (col < ev) wv[c] = load_row4<WT>(static_cast<const WT*>(p.table) + base + col);
        }
        const float s_old = gl == 0 ? rs[row[0]] : 0.f;
        float sq = 0.f;
#pragma unroll
        for (int c = 0; c < NC; ++c) {
          const int col = (c * G + gl) * 4;
          acc[c] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (col < ev) {
            gather_add<GradT, 4>(acc[c], p, ent[0], esc[0], col);
            acc[c] = scale4(acc[c], inv_scaler);
            sq += sumsq4(acc[c]);
          }
        }
        const float f = row_reduce_step<OPT, G>(gmask, gi * G, lane, sq, s_old, rs + row[0], ev, hp, step);
#pragma unroll
        for (int c = 0; c < NC; ++c) {
          const int col = (c * G + gl) * 4;
          if (col < ev) {
            float4 w;
            if (c < 4) w = widen4(wv[c & 3]);
            else w = load_vec4<WT>(static_cast<const WT*>(p.table) + base + col);
            row_apply4<OPT, StateT>(w, acc[c], f, s0, base + col, hp);
            store_w4<WT>(static_cast<WT*>(p.table) + base + col, w, srk, base + col);
          }
        }
      } else {
        // the row in passes of at most 4 chunks: weights, state and sums of one pass stay within the
        // 128 registers of two resident blocks per SM for G == 32 (8 chunks per lane)
#pragma unroll
        for (int c0 = 0; c0 < NC; c0 += 4) {
          typename Row4<WT>::type wv[4];
          float4 sv[4], acc[4];
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int col = ((c0 + c) * G + gl) * 4;
            wv[c] = {};
            sv[c] = acc[c] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (col < ev) {
              wv[c] = load_row4<WT>(static_cast<const WT*>(p.table) + base + col);
              if constexpr (kHasS0) sv[c] = load_vec4<StateT>(s0 + base + col);
            }
          }
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int col = ((c0 + c) * G + gl) * 4;
            if (col < ev) gather_add<GradT, 4>(acc[c], p, ent[0], esc[0], col);
          }
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int col = ((c0 + c) * G + gl) * 4;
            if (col < ev) {
              float4 w = widen4(wv[c]);
              apply_opt4_pre<OPT, StateT>(w, scale4(acc[c], inv_scaler), sv[c], s0, s1, base + col, hp, step);
              store_w4<WT>(static_cast<WT*>(p.table) + base + col, w, srk, base + col);
            }
          }
        }
      }
      if (gl == 0) unique_release(ut, uid);
      rec[0] = rec[1];
      rec[1] = rec[2];
      row[0] = row[1];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        ent[0][u] = ent[1][u];
        esc[0][u] = esc[1][u];
      }
    }
  }

  // ------------------------------------------------------------------ medium rows: warp per row
  for (unsigned int i = warp_global; i < n_medium; i += num_warps) {
    const uint2 r = ix.medium_list[i];
    const unsigned int uid = r.x, o0 = r.y;
    const unsigned int o1 = ix.offsets[uid + 1];
    const long long base = static_cast<long long>(ut.rows[uid]) * ev;
    if constexpr (kRowRule<OPT>) {
      // as the light rows: the sums of all (up to 8) column iterations stay in registers until the
      // row's sum of g^2 is known, then every column takes the row's factor
      const unsigned long long arow = ut.rows[uid];
      float* const rs = row_state<OPT>(s0, s1);
      const float s_old = lane == 0 ? rs[arow] : 0.f;
      constexpr int kIters = (G == 8) ? 1 : kMaxEmbWidth / 128;   // G == 8 launches have ev <= 128
      float4 acc[kIters];
      float sq = 0.f;
#pragma unroll
      for (int c = 0; c < kIters; ++c) {
        const int col = lane * 4 + c * 128;
        acc[c] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (col < ev) {
          acc[c] = scale4(gather_list<GradT, 8>(p, ix, has_scale, o0, 1u, o1, col), inv_scaler);
          sq += sumsq4(acc[c]);
        }
      }
      const float f = row_reduce_step<OPT, 32>(0xffffffffu, 0, lane, sq, s_old, rs + arow, ev, hp, step);
#pragma unroll
      for (int c = 0; c < kIters; ++c) {
        const int col = lane * 4 + c * 128;
        if (col < ev) {
          float4 w = load_vec4<WT>(static_cast<const WT*>(p.table) + base + col);
          row_apply4<OPT, StateT>(w, acc[c], f, s0, base + col, hp);
          store_w4<WT>(static_cast<WT*>(p.table) + base + col, w, srk, base + col);
        }
      }
    } else
    for (int col = lane * 4; col < ev; col += 128) {
      float4 w = load_vec4<WT>(static_cast<const WT*>(p.table) + base + col);
      float4 sv = make_float4(0.f, 0.f, 0.f, 0.f);
      if constexpr (kHasS0) sv = load_vec4<StateT>(s0 + base + col);
      const float4 acc = gather_list<GradT, 8>(p, ix, has_scale, o0, 1u, o1, col);
      apply_opt4_pre<OPT, StateT>(w, scale4(acc, inv_scaler), sv, s0, s1, base + col, hp, step);
      store_w4<WT>(static_cast<WT*>(p.table) + base + col, w, srk, base + col);
    }
    if (lane == 0) unique_release(ut, uid);
  }
}

// heavy rows: one block per (uid, chunk)
template <int OPT, typename StateT, typename GradT, typename WT>
__global__ void __launch_bounds__(256)
    emb_bwd_heavy_kernel(const EmbParams p, const UniqueTable ut, const BwdIndex ix,
                         StateT* __restrict__ s0, StateT* __restrict__ s1, const OptHyper hp,
                         const float grad_scale) {
  const unsigned int nitems = min(*ix.heavy_count, ix.max_heavy_items);
  const int ev = p.ev_size;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  extern __shared__ float sm[];  // [8 warps][ev]
  __shared__ unsigned int last_s;
  const OptStep step = opt_step<OPT>(hp);
  const float inv_scaler = grad_scale / hp.scaler;
  const bool has_scale = ix.bucket_scale != nullptr;
  for (unsigned int it = blockIdx.x; it < nitems; it += gridDim.x) {
    const unsigned int uid = ix.heavy_items[2 * it];
    if (uid == kInvalidVal) continue;   // reserved by a row that fell back to the medium list
    const unsigned int sc_ = ix.heavy_items[2 * it + 1];
    const unsigned int slot = sc_ >> 12, chunk = sc_ & 0xFFFu;
    const unsigned int o0 = ix.offsets[uid] + chunk * kChunk;
    const unsigned int o1 = min(ix.offsets[uid + 1], o0 + kChunk);
    const unsigned int nch = (ix.offsets[uid + 1] - ix.offsets[uid] + kChunk - 1) / kChunk;
    float* scratch = ix.heavy_scratch + static_cast<long long>(slot) * ev;
    for (int col0 = 0; col0 < ev; col0 += 128) {
      const int col = col0 + lane * 4;
      // warp w sums the chunk's entries w, w + 8, ..., four in flight per round
      if (col < ev)
        *reinterpret_cast<float4*>(sm + warp * ev + col) =
            gather_list<GradT, 4>(p, ix, has_scale, o0 + warp, 8u, o1, col);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < ev; c += blockDim.x) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < 8; ++w) v += sm[w * ev + c];
      atomicAdd(scratch + c, v);
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last_s = (atomicAdd(&ix.heavy_ticket[slot], 1u) == nch - 1) ? 1u : 0u;
    __syncthreads();
    if (last_s) {
      __threadfence();
      const unsigned long long row = ut.rows[uid];
      const long long base = static_cast<long long>(row) * ev;
      const unsigned long long srk = sr_key<WT>(hp.sr_seed, hp.step_ptr);
      if constexpr (kRowRule<OPT>) {
        // the block reduces the row's sum of g^2 over the scratch row, thread 0 updates the row
        // state once, then every column is applied; scratch is zeroed only by this second read
        __shared__ float sq_s[8];
        __shared__ float f_s;
        float sq = 0.f;
        for (int c = threadIdx.x; c < ev; c += blockDim.x) {
          const float g = __ldcg(scratch + c) * inv_scaler;
          sq += g * g;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
        if (lane == 0) sq_s[warp] = sq;
        __syncthreads();
        if (threadIdx.x == 0) {
          float t = 0.f;
#pragma unroll
          for (int w = 0; w < 8; ++w) t += sq_s[w];
          float* const rs = row_state<OPT>(s0, s1);
          f_s = row_state_step<OPT>(rs[row], t, rs + row, ev, hp, step);
        }
        __syncthreads();
        const float f = f_s;
        for (int c = threadIdx.x; c < ev; c += blockDim.x) {
          const float g = __ldcg(scratch + c) * inv_scaler;
          scratch[c] = 0.f;
          float w = to_f<WT>(static_cast<const WT*>(p.table)[base + c]);
          row_apply1<OPT, StateT>(w, g, f, s0, base + c, hp);
          store_w<WT>(static_cast<WT*>(p.table) + base + c, w, srk, base + c);
        }
      } else
      for (int c = threadIdx.x; c < ev; c += blockDim.x) {
        const float g = __ldcg(scratch + c);
        scratch[c] = 0.f;
        float w = to_f<WT>(static_cast<const WT*>(p.table)[base + c]);
        apply_opt<OPT, StateT>(w, g * inv_scaler, s0, s1, base + c, hp, step);
        store_w<WT>(static_cast<WT*>(p.table) + base + c, w, srk, base + c);
      }
      if (threadIdx.x == 0) {
        ix.heavy_ticket[slot] = 0;
        unique_release(ut, uid);
      }
    }
    __syncthreads();
  }
}

}  // namespace hctr

using namespace hctr;

// ABI self-check: the Python side mirrors these structs with ctypes (embedding/ops.py) and compares
// the sizes at load time, so a layout drift fails loudly instead of corrupting kernel arguments.
extern "C" int hctr_abi_sizes_emb(int* out) {
  out[0] = static_cast<int>(sizeof(EmbLookup));
  out[1] = static_cast<int>(sizeof(EmbParams));
  out[2] = static_cast<int>(sizeof(UniqueTable));
  out[3] = static_cast<int>(sizeof(BwdIndex));
  out[4] = static_cast<int>(sizeof(OptHyper));
  return 5;
}

extern "C" int hctr_emb_bwd_index(const EmbParams* p, const UniqueTable* ut, const BwdIndex* ix,
                                  long long total_pairs, int key_bytes, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (total_pairs == 0) return 0;
  if (p->num_lookups > kMaxSmemLookups) return -5;
  if (ix->max_heavy_rows > (1u << 20)) return -6;   // 20-bit scratch slot field of a heavy item
  const unsigned int blocks = static_cast<unsigned int>((total_pairs + kPairsPerBlock - 1) / kPairsPerBlock);
  with_key(key_bytes, [&](auto k) {
    emb_bwd_index_kernel<type_of<decltype(k)>><<<blocks, kIdxThreads, 0, st>>>(*p, *ut, *ix, total_pairs);
  });
  const unsigned int nb = (ut->max_unique + 1023) / 1024;
  scan_block_sums_kernel<<<nb, 1024, 0, st>>>(ix->count, ix->block_sums, ut->counter, ut->max_unique);
  scan_sums_kernel<<<1, 1024, 0, st>>>(ix->block_sums, ut->counter, ut->max_unique, ix->heavy_count,
                                       ix->heavy_slot, ix->class_count);
  scan_apply_kernel<<<nb, 1024, 0, st>>>(ix->count, ix->block_sums, ix->offsets, ut->counter,
                                         ut->max_unique);
  emb_bwd_classify_kernel<<<num_sms(), 1024, 0, st>>>(*ut, *ix);
  with_weighted(*p, [&](auto wgt) {
    emb_bwd_fill_kernel<decltype(wgt)::value><<<blocks, kIdxThreads, 0, st>>>(*p, *ix, total_pairs);
  });
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// fork/join helper: the heavy-row kernel runs on an internal side stream next to the light-row
// kernel (event dependencies are captured into CUDA graphs like any other cross-stream edge)
struct SideStream {
  cudaStream_t s = nullptr;
  cudaEvent_t fork = nullptr, join = nullptr;
  bool ok() {
    if (s) return true;
    // highest priority: the (small) heavy-row blocks must become resident before the light-row
    // kernel occupies every SM, whatever order the graph scheduler releases the two nodes in
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    if (cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, hi) != cudaSuccess) return false;
    cudaEventCreateWithFlags(&fork, cudaEventDisableTiming);
    cudaEventCreateWithFlags(&join, cudaEventDisableTiming);
    return true;
  }
};
static SideStream g_heavy_side;

template <int OPT, typename StateT, typename WT>
static void launch_reduce(const EmbParams* p, const UniqueTable* ut, const BwdIndex* ix, void* s0,
                         void* s1, const OptHyper* hp, float grad_scale, int grad_bf16, int num_sms,
                         cudaStream_t st) {
  const size_t smem = 8 * static_cast<size_t>(p->ev_size) * sizeof(float);
  const bool g8 = p->ev_size <= 128;
  const int blocks = num_sms * (g8 ? 3 : 2);   // one resident wave of grid-stride blocks
  // heavy rows first, on the side stream: its (small, latency-bound) blocks become resident before
  // the bandwidth-bound light-row kernel fills the rest of every SM
  const bool fork = g_heavy_side.ok();
  cudaStream_t hs = fork ? g_heavy_side.s : st;
  if (fork) {
    cudaEventRecord(g_heavy_side.fork, st);
    cudaStreamWaitEvent(hs, g_heavy_side.fork, 0);
  }
  with_elem(grad_bf16, [&](auto g) {
    using GradT = type_of<decltype(g)>;
    emb_bwd_heavy_kernel<OPT, StateT, GradT, WT><<<num_sms * 4, 256, smem, hs>>>(
        *p, *ut, *ix, (StateT*)s0, (StateT*)s1, *hp, grad_scale);
    if (fork) cudaEventRecord(g_heavy_side.join, hs);
    auto light = [&](auto lanes) {
      emb_bwd_reduce_update_kernel<OPT, StateT, GradT, decltype(lanes)::value, WT><<<blocks, 256, 0, st>>>(
          *p, *ut, *ix, (StateT*)s0, (StateT*)s1, *hp, grad_scale);
    };
    if (g8) light(Int<8>{});
    else light(Int<32>{});
  });
  if (fork) cudaStreamWaitEvent(st, g_heavy_side.join, 0);
}

extern "C" int hctr_emb_bwd_reduce_update(const EmbParams* p, const UniqueTable* ut,
                                          const BwdIndex* ix, void* s0, void* s1, int opt,
                                          int state_bf16, const OptHyper* hp, float grad_scale,
                                          int grad_bf16, unsigned int* overflow_flag, int num_sms,
                                          int table_bf16, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (p->ev_size % 4) return -3;
  if (p->ev_size > kMaxEmbWidth) return -4;
  const int rc = dispatch_opt(opt, state_bf16, table_bf16, [&](auto o, auto s, auto w) {
    launch_reduce<decltype(o)::value, type_of<decltype(s)>, type_of<decltype(w)>>(
        p, ut, ix, s0, s1, hp, grad_scale, grad_bf16, num_sms, st);
  });
  if (rc) return rc;
  // heavy rows past the caps take the medium path (emb_bwd_classify_kernel): only the unique-row
  // capacity can overflow
  emb_finish_kernel<<<1, 1, 0, st>>>(ut->counter, overflow_flag, ut->max_unique);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
