// Shared declarations of the embedding kernels (see embedding.cu / embedding_bwd.cu).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "optim.cuh"
#include "ptx.cuh"

namespace hctr {

constexpr int kMaxRanks = 16;
constexpr unsigned long long kEmptyKey = 0xFFFFFFFFFFFFFFFFull;
constexpr unsigned int kInvalidVal = 0xFFFFFFFFu;
// widest row the lookup / accumulate / fused-update kernels cover (32 lanes x 32 columns per lane);
// the entry points reject wider tables instead of truncating them
constexpr int kMaxEmbWidth = 1024;

struct EmbLookup {
  long long table_row_off;  // first row of this table shard inside the local arena
  long long key_off;        // element offset of the lookup's keys in a rank's feature-major buffer
  long long nnz_off;        // element offset of per-bucket nnz (variable hotness) or -1
  long long out_off;        // element offset of the lookup's output block inside the output slab
  long long grad_off;       // element offset of the lookup's top-grad block inside the grad slab
  int hotness;              // fixed / max hotness (keys read per bucket)
  int key_stride;           // keys per sample in the key block (>= hotness; concat combiner: H)
  int num_shards;           // row sharding: owned iff key % num_shards == shard_idx
  int shard_idx;
  int out_stride;           // elements per sample row of the output block
  int grad_stride;          // elements per sample row of the grad block
  int combiner;             // 0 = sum, 1 = mean
  int ev_size;
  int rows;                 // rows of the local shard (bounds guard)
  int weighted;             // 1: every key carries an fp32 weight at its element offset in weights[src]
  long long pair_off;       // first (bucket,key) pair index of this lookup (backward index)
};

struct EmbParams {
  int num_ranks, my_rank, batch, num_lookups;
  const void* keys[kMaxRanks];   // per source rank: feature-major keys
  const int* nnz[kMaxRanks];     // per source rank: per-bucket nnz (optional)
  void* out[kMaxRanks];          // per source rank: output activation base
  const void* grad[kMaxRanks];   // per source rank: top-grad base
  const EmbLookup* lookups;      // device array [num_lookups]
  void* table;                   // [rows, ev] arena of fp32, bf16 or e4m3 weights (the launcher's table_type)
  int ev_size;                   // row pitch of the arena (all tables of a group share it)
  // per source rank: fp32 per-key weights in the layout of keys (same element offsets); all null
  // when no lookup of the launch is weighted, which selects the unweighted kernels
  const float* weights[kMaxRanks];
  // e4m3 arena: one byte e + 127 per arena row, the row dequantizes to q * 2^e; null for fp32 and bf16
  const uint8_t* row_exp;
};

// Weight of key h of bucket (src, s) of a lookup: 1 unless the lookup is weighted
HCTR_DEVICE float key_weight(const EmbParams& p, const EmbLookup& lk, int src, int s, int h) {
  return lk.weighted ? p.weights[src][lk.key_off + static_cast<long long>(s) * lk.key_stride + h] : 1.f;
}

struct PeerStage {
  void* dst[kMaxRanks];
};

struct UniqueTable {
  unsigned long long* keys;  // [capacity] hash keys (arena row index)
  unsigned int* vals;        // [capacity] compact unique id
  unsigned int* counter;     // [1] number of unique rows
  unsigned long long* rows;  // [max_unique] uid -> arena row
  unsigned int* slots;       // [max_unique] uid -> hash slot (for O(n) clearing)
  unsigned int mask;         // capacity - 1
  unsigned int max_unique;
};

// MurmurHash3 64-bit finaliser (a bijection of 64-bit words)
HCTR_DEVICE unsigned long long fmix64(unsigned long long k) {
  k ^= k >> 33;
  k *= 0xff51afd7ed558ccdull;
  k ^= k >> 33;
  k *= 0xc4ceb9fe1a85ec53ull;
  k ^= k >> 33;
  return k;
}

HCTR_DEVICE unsigned int hash64(unsigned long long k) { return static_cast<unsigned int>(fmix64(k)); }

// ------------------------------------------------------------------ bf16 weights: stochastic rounding
// Every optimizer store of a bf16 weight rounds stochastically: the stored value is the upper 16 bits
// of (fp32 bits + r), r = 16 pseudo-random bits, so it rounds away from zero with probability equal to
// the dropped fraction of an ulp and the expected stored value is the fp32 result (updates far below
// one bf16 ulp still move the weights on average).  Inf / NaN are stored as round-to-nearest does.
// r is a stateless hash of (seed, device step counter, arena index i = row * pitch + col): no host
// input, capturable in a CUDA graph, independent across steps and kernels, and reproduced by a resumed
// run.  One 64-bit hash serves four consecutive elements: r(i) = 16-bit lane i % 4 of
// fmix64(step key ^ i / 4), so a 4-wide store hashes once.
// Mirrored bit for bit by embedding/ops.py (sr_step_key, sr_bits, sr_round_bf16).
HCTR_DEVICE unsigned long long sr_step_key(unsigned int seed, unsigned int step) {
  return fmix64((static_cast<unsigned long long>(seed) << 32) | step);
}
HCTR_DEVICE unsigned long long sr_hash4(unsigned long long key, long long idx) {
  return fmix64(key ^ (static_cast<unsigned long long>(idx) >> 2));
}
HCTR_DEVICE unsigned short sr_round(float v, unsigned int r) {
  const unsigned int b = __float_as_uint(v);
  if ((b & 0x7f800000u) == 0x7f800000u) return __bfloat16_as_ushort(__float2bfloat16_rn(v));
  return static_cast<unsigned short>((b + r) >> 16);
}

// Weight rows of the arena: WT = float or __nv_bfloat16.  Loads widen to fp32 (load_vec4 / to_f);
// the optimizer stores go through store_w / store_w4 with the launch's key (sr_key), which the fp32
// instantiations never compute.
template <typename WT>
HCTR_DEVICE unsigned long long sr_key(unsigned int seed, const unsigned int* step_ptr) {
  if constexpr (sizeof(WT) == 2) return sr_step_key(seed, step_ptr ? *step_ptr : 1u);
  return 0ull;
}
template <typename WT>
HCTR_DEVICE void store_w(WT* p, float w, unsigned long long key, long long idx);
template <>
HCTR_DEVICE void store_w<float>(float* p, float w, unsigned long long, long long) { *p = w; }
template <>
HCTR_DEVICE void store_w<__nv_bfloat16>(__nv_bfloat16* p, float w, unsigned long long key, long long idx) {
  const unsigned int r = static_cast<unsigned int>(sr_hash4(key, idx) >> (16 * (idx & 3))) & 0xFFFFu;
  *reinterpret_cast<unsigned short*>(p) = sr_round(w, r);
}
template <typename WT>
HCTR_DEVICE void store_w4(WT* p, float4 w, unsigned long long key, long long idx);
template <>
HCTR_DEVICE void store_w4<float>(float* p, float4 w, unsigned long long, long long) {
  *reinterpret_cast<float4*>(p) = w;
}
template <>
HCTR_DEVICE void store_w4<__nv_bfloat16>(__nv_bfloat16* p, float4 w, unsigned long long key, long long idx) {
  // idx % 4 == 0 (4-aligned rows and columns): the four lanes of one hash
  const unsigned long long h = sr_hash4(key, idx);
  const unsigned int lo = static_cast<unsigned int>(h), hi = static_cast<unsigned int>(h >> 32);
  const unsigned int a = sr_round(w.x, lo & 0xFFFFu), b = sr_round(w.y, lo >> 16);
  const unsigned int c = sr_round(w.z, hi & 0xFFFFu), d = sr_round(w.w, hi >> 16);
  *reinterpret_cast<uint2*>(p) = make_uint2(a | (b << 16), c | (d << 16));
}
// A 4-column slice of a weight row as loaded: float4 (fp32) or the packed bf16 pairs (uint2), widened
// to fp32 where the optimizer needs it, so a bf16 row held across the gradient gather takes half the
// registers.
template <typename WT>
struct Row4 {
  using type = float4;
};
template <>
struct Row4<__nv_bfloat16> {
  using type = uint2;
};
template <typename WT>
HCTR_DEVICE typename Row4<WT>::type load_row4(const WT* p) {
  return *reinterpret_cast<const typename Row4<WT>::type*>(p);
}
HCTR_DEVICE float4 widen4(float4 v) { return v; }
HCTR_DEVICE float4 widen4(uint2 v) { return make_float4(bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y)); }
// read-only (non-coherent cache) row loads of the lookup
HCTR_DEVICE float4 ldg_row4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
HCTR_DEVICE float4 ldg_row4(const __nv_bfloat16* p) {
  const uint2 v = __ldg(reinterpret_cast<const uint2*>(p));
  return make_float4(bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y));
}
HCTR_DEVICE float ldg_row1(const float* p) { return __ldg(p); }
HCTR_DEVICE float ldg_row1(const __nv_bfloat16* p) { return __bfloat162float(__ldg(p)); }
// e4m3 rows (serving arenas): 4 bytes per 4 columns, unpacked by the hardware conversion; the row's
// power-of-two scale is applied by the caller (row_scale)
HCTR_DEVICE float4 e4m3x4_to_float4(unsigned int v) {
  const float2 lo = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2(
      static_cast<__nv_fp8x2_storage_t>(v & 0xFFFFu), __NV_E4M3)));
  const float2 hi = __half22float2(__half2(__nv_cvt_fp8x2_to_halfraw2(
      static_cast<__nv_fp8x2_storage_t>(v >> 16), __NV_E4M3)));
  return make_float4(lo.x, lo.y, hi.x, hi.y);
}
HCTR_DEVICE float4 ldg_row4(const __nv_fp8_e4m3* p) {
  return e4m3x4_to_float4(__ldg(reinterpret_cast<const unsigned int*>(p)));
}
// 4-byte word k of a 16-byte load (k known at compile time)
HCTR_DEVICE unsigned int word_of(const uint4& v, int k) {
  return k == 0 ? v.x : (k == 1 ? v.y : (k == 2 ? v.z : v.w));
}
HCTR_DEVICE float ldg_row1(const __nv_fp8_e4m3* p) {
  const unsigned char b = __ldg(reinterpret_cast<const unsigned char*>(p));
  return __half2float(__half(__nv_cvt_fp8_to_halfraw(static_cast<__nv_fp8_storage_t>(b), __NV_E4M3)));
}
// 2^e of arena row `row` of an e4m3 arena (exps[row] = e + 127), exact for bytes 1..254.  Byte 0 gives 0 instead
// of the subnormal 2^-127, which the fast-math (flush-to-zero) weight multiply would flush anyway: a row with
// e = -127 -- all-zero, or amax at most 448 * 2^-127 (about 2^-118.2) with nonzero codes -- pools to zero in the
// fp8 lookup (docs/embedding.md, fp8 serving tables: exactness).
HCTR_DEVICE float row_scale(const uint8_t* exps, long long row) {
  return __uint_as_float(static_cast<unsigned int>(__ldg(exps + row)) << 23);
}

// ------------------------------------------------------------------ unique (transient hash)
HCTR_DEVICE unsigned int unique_get_insert(const UniqueTable& t, unsigned long long row) {
  unsigned int h = hash64(row) & t.mask;
  while (true) {
    const unsigned long long prev = atomicCAS(&t.keys[h], kEmptyKey, row);
    if (prev == kEmptyKey) {
      const unsigned int uid = atomicAdd(t.counter, 1u);
      if (uid < t.max_unique) {
        t.rows[uid] = row;
        t.slots[uid] = h;
      }
      // rows[]/slots[] are only consumed by later kernels (kernel boundary orders them); concurrent
      // threads of this kernel need the uid alone, so no membar is required before publishing it
      atomicExch(&t.vals[h], uid);
      return uid;
    }
    if (prev == row) {
      unsigned int v;
      do {
        v = *reinterpret_cast<volatile unsigned int*>(&t.vals[h]);
      } while (v == kInvalidVal);
      return v;
    }
    h = (h + 1) & t.mask;
  }
}

// An update kernel is done with unique row uid: empties its hash slot for the next step
HCTR_DEVICE void unique_release(const UniqueTable& t, unsigned int uid) {
  const unsigned int slot = t.slots[uid];
  t.keys[slot] = kEmptyKey;
  t.vals[slot] = kInvalidVal;
}

// Keys of bucket (src rank, sample s) of a lookup with the given hotness and nnz_off: the hotness, or
// the bucket's own count below it for a variable-hotness lookup
HCTR_DEVICE int bucket_nnz(const EmbParams& p, int hotness, long long nnz_off, int src, int s) {
  int nnz = hotness;
  if (nnz_off >= 0) nnz = min(hotness, p.nnz[src][nnz_off + s]);
  return nnz;
}

// Clears the counter of unique rows after an update and records an overflow of it (the update kernels
// release their rows' hash slots, so the table is empty again)
__global__ void emb_finish_kernel(unsigned int* counter, unsigned int* overflow_flag, unsigned int max_unique);

// Host dispatch of the kernels' template arguments: each helper calls a generic lambda with a tag
// (type_of<decltype(tag)> is the type, decltype(tag)::value the integer).
template <typename T>
struct Tag {
  using type = T;
};
template <typename TagT>
using type_of = typename TagT::type;
template <int V>
using Int = std::integral_constant<int, V>;
// element type of activations, gradients, state or weights
template <typename Fn>
inline void with_elem(int is_bf16, Fn&& fn) {
  if (is_bf16) fn(Tag<__nv_bfloat16>{});
  else fn(Tag<float>{});
}
// weight type of an arena: 0 fp32, 1 bf16, 2 e4m3 (serving arenas, lookup only)
template <typename Fn>
inline void with_table(int table_type, Fn&& fn) {
  if (table_type == 2) fn(Tag<__nv_fp8_e4m3>{});
  else with_elem(table_type, fn);
}
// key type: 8-byte or 4-byte integers
template <typename Fn>
inline void with_key(int key_bytes, Fn&& fn) {
  if (key_bytes == 8) fn(Tag<long long>{});
  else fn(Tag<int>{});
}
// weighted lookups in the launch (p.weights set): the instantiations that read per-key weights
template <typename Fn>
inline void with_weighted(const EmbParams& p, Fn&& fn) {
  if (p.weights[0] != nullptr) fn(std::true_type{});
  else fn(std::false_type{});
}
// The sparse optimizers: calls fn(Int<OPT>, Tag<StateT>, Tag<WT>) for optimizer `opt`, state type (bf16
// when state_bf16) and weight type (bf16 when table_bf16).  SGD (no state) and row-wise AdaGrad (a
// [rows] fp32 accumulator, never bf16: a value that only grows would drop small increments) run with the
// fp32 state type.  Partial row-wise Adam's StateT is the type of its first moment s0; its second moment
// s1 is one fp32 value per row whatever StateT is (the kernels read it through row_state).  Returns 0, -2
// for an unknown optimizer, or -7 for row-wise AdaGrad with bf16 state.
template <typename Fn>
inline int dispatch_opt(int opt, int state_bf16, int table_bf16, Fn&& fn) {
  auto run = [&](auto o) {
    constexpr int O = decltype(o)::value;
    auto with_w = [&](auto s) { with_elem(table_bf16, [&](auto w) { fn(o, s, w); }); };
    if constexpr (O != OPT_SGD && O != OPT_ROWWISE_ADAGRAD) {
      if (state_bf16) return with_w(Tag<__nv_bfloat16>{});
    }
    with_w(Tag<float>{});
  };
  if (opt == OPT_ROWWISE_ADAGRAD && state_bf16) return -7;
  switch (opt) {
    case OPT_SGD: run(Int<OPT_SGD>{}); break;
    case OPT_ADAGRAD: run(Int<OPT_ADAGRAD>{}); break;
    case OPT_ADAM: run(Int<OPT_ADAM>{}); break;
    case OPT_FTRL: run(Int<OPT_FTRL>{}); break;
    case OPT_MOMENTUM: run(Int<OPT_MOMENTUM>{}); break;
    case OPT_NESTEROV: run(Int<OPT_NESTEROV>{}); break;
    case OPT_RMSPROP: run(Int<OPT_RMSPROP>{}); break;
    case OPT_ROWWISE_ADAGRAD: run(Int<OPT_ROWWISE_ADAGRAD>{}); break;
    case OPT_PARTIAL_ROWWISE_ADAM: run(Int<OPT_PARTIAL_ROWWISE_ADAM>{}); break;
    default: return -2;
  }
  return 0;
}

}  // namespace hctr
