// Position-weighted inputs (DataReaderSparseParam(..., position_weighted=True), docs/embedding.md): key h of every
// bag of such an input weighs P[f, h], a dense fp32 parameter of the network.
//   fill   : before the key exchange, P[f, h] is written into the weight slab at every key position of the input
//            (0 at padding keys), with a 0 / 1 mask of the valid positions; from there on the weighted lookup,
//            exchange and update kernels run unchanged.
//   dot    : after the gradient push and before the sparse update overwrites the rows, one warp per owned bag
//            computes <T[row_h], g> (times 1/nnz for mean) for every owned key and adds it at the key's position
//            of an fp32 buffer laid out like the key slab, one slot per source rank.
//   reduce : the column sums of that buffer, in a fixed order, are added into P's gradient (one launch, a block per
//            element of P).
// No float atomics anywhere: a position is owned by exactly one row shard, so the ranks' partial gradients add up
// to the full gradient in the dense all-reduce, and a replay from the same state gives the same bits.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "embedding.cuh"

namespace hctr {

struct PwFillRegion {
  const float* p;      // P[f, 0..hotness) of the lookup's input
  long long key_off;   // first key of the lookup's block in the key slab
  long long n;         // keys of the block (batch * hotness)
  int hotness;
  int pad_;
};

// grid.y = region
template <typename KeyT>
__global__ void __launch_bounds__(256)
    emb_pw_fill_kernel(const KeyT* __restrict__ keys, float* __restrict__ weights, float* __restrict__ valid,
                       const PwFillRegion* __restrict__ regions) {
  const PwFillRegion rg = regions[blockIdx.y];
  const long long step = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < rg.n; i += step) {
    const long long o = rg.key_off + i;
    const bool ok = keys[o] >= 0;
    weights[o] = ok ? __ldg(rg.p + static_cast<int>(i % rg.hotness)) : 0.f;
    valid[o] = ok ? 1.f : 0.f;
  }
}

HCTR_DEVICE float4 ld_f4(const float* p) { return *reinterpret_cast<const float4*>(p); }
HCTR_DEVICE float4 ld_f4(const __nv_bfloat16* p) { return widen4(*reinterpret_cast<const uint2*>(p)); }
HCTR_DEVICE float ld_f1(const float* p) { return *p; }
HCTR_DEVICE float ld_f1(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// One warp per (source rank, selected lookup, sample) bag; lane j covers columns j*VEC + 32*VEC*i.  The lane sums
// and the xor butterfly run in a fixed order, and only lane 0 writes, to a position no other warp owns.
template <typename KeyT, typename GT, typename WT, int VEC>
__global__ void __launch_bounds__(256)
    emb_pw_dot_kernel(const EmbParams p, const int* __restrict__ sel, const int nsel, float* __restrict__ dots,
                      const long long dot_stride) {
  const int lane = threadIdx.x & 31;
  const unsigned int warps = blockDim.x >> 5;
  const unsigned int batch = static_cast<unsigned int>(p.batch), ns = static_cast<unsigned int>(nsel);
  const unsigned int bags = static_cast<unsigned int>(p.num_ranks) * ns * batch;
  for (unsigned int item = blockIdx.x * warps + (threadIdx.x >> 5); item < bags; item += gridDim.x * warps) {
    const unsigned int rl = item / batch;
    const int s = static_cast<int>(item - rl * batch);
    const int src = static_cast<int>(rl / ns);
    const EmbLookup& lk = p.lookups[sel[rl - static_cast<unsigned int>(src) * ns]];
    const long long kpos = lk.key_off + static_cast<long long>(s) * lk.key_stride;
    const KeyT* kb = static_cast<const KeyT*>(p.keys[src]) + kpos;
    const GT* g = static_cast<const GT*>(p.grad[src]) + lk.grad_off + static_cast<long long>(s) * lk.grad_stride;
    float* d = dots + static_cast<long long>(src) * dot_stride + kpos;
    const int nnz = bucket_nnz(p, lk.hotness, lk.nnz_off, src, s);
    const float scale = (lk.combiner == 1 && nnz > 0) ? 1.f / static_cast<float>(nnz) : 1.f;
    const int ev = lk.ev_size;
    const unsigned int shards = static_cast<unsigned int>(lk.num_shards);
    for (int h = 0; h < nnz; ++h) {
      const long long key = static_cast<long long>(kb[h]);
      if (key < 0) continue;
      const unsigned long long uk = static_cast<unsigned long long>(key);
      unsigned long long r = uk;
      if (shards > 1) {
        unsigned int rem;
        if (uk <= 0xFFFFFFFFull) {   // 32-bit fast path (no 64-bit division)
          const unsigned int k32 = static_cast<unsigned int>(uk);
          r = k32 / shards;
          rem = k32 - static_cast<unsigned int>(r) * shards;
        } else {
          r = uk / shards;
          rem = static_cast<unsigned int>(uk - r * shards);
        }
        if (rem != static_cast<unsigned int>(lk.shard_idx)) continue;
      }
      if (r >= static_cast<unsigned long long>(lk.rows)) continue;
      const WT* row = static_cast<const WT*>(p.table) + (lk.table_row_off + static_cast<long long>(r)) * p.ev_size;
      float acc = 0.f;
      for (int c = lane * VEC; c < ev; c += 32 * VEC) {
        if constexpr (VEC == 4) {
          const float4 w = ld_f4(row + c), gv = ld_f4(g + c);
          acc = fmaf(w.x, gv.x, acc);
          acc = fmaf(w.y, gv.y, acc);
          acc = fmaf(w.z, gv.z, acc);
          acc = fmaf(w.w, gv.w, acc);
        } else {
          acc = fmaf(ld_f1(row + c), ld_f1(g + c), acc);
        }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) d[h] += acc * scale;
    }
  }
}

// A column of the dot products: position h of a lookup whose buffer region starts at element off (row r of source
// rank r's slot, sample s at off + s * hotness)
struct PwReduceCol {
  long long off;
  int hotness;
  int h;
};
// One element of P's gradient and the columns that add into it (the lookups of its input), in order
struct PwReduceTarget {
  float* dst;
  int col_begin;
  int ncols;
};

// One block per element of P's gradient: each of its columns is summed over the ranks * batch rows -- thread t takes
// rows t, t + 256, ... in order, then a fixed shared-memory tree -- and the column sums are added in order.
__global__ void __launch_bounds__(256)
    emb_pw_reduce_kernel(const float* __restrict__ dots, const long long row_stride, const int batch, const int ranks,
                         const PwReduceCol* __restrict__ cols, const PwReduceTarget* __restrict__ targets) {
  __shared__ float part[256];
  const PwReduceTarget t = targets[blockIdx.x];
  const int rows = ranks * batch;
  float total = 0.f;
  for (int c = 0; c < t.ncols; ++c) {
    const PwReduceCol col = cols[t.col_begin + c];
    const float* base = dots + col.off + col.h;
    float acc = 0.f;
    for (int i = threadIdx.x; i < rows; i += blockDim.x) {
      const int r = i / batch;
      acc += base[r * row_stride + static_cast<long long>(i - r * batch) * col.hotness];
    }
    part[threadIdx.x] = acc;
    __syncthreads();
    for (int w = 128; w > 0; w >>= 1) {
      if (threadIdx.x < w) part[threadIdx.x] += part[threadIdx.x + w];
      __syncthreads();
    }
    if (threadIdx.x == 0) total += part[0];
    __syncthreads();
  }
  if (threadIdx.x == 0) *t.dst += total;
}

}  // namespace hctr

using namespace hctr;

// ABI self-check of the descriptors' ctypes mirrors (embedding/ops.py)
extern "C" void hctr_abi_sizes_pw(int* sz) {
  sz[0] = static_cast<int>(sizeof(PwFillRegion));
  sz[1] = static_cast<int>(sizeof(PwReduceCol));
  sz[2] = static_cast<int>(sizeof(PwReduceTarget));
}

extern "C" int hctr_emb_pw_fill(const void* keys, int key_bytes, float* weights, float* valid,
                                const PwFillRegion* regions, int num_regions, long long max_n, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (num_regions <= 0 || max_n <= 0) return 0;
  long long bx = (max_n + 255) / 256;
  if (bx > 4 * num_sms()) bx = 4 * num_sms();
  const dim3 grid(static_cast<unsigned>(bx), num_regions);
  with_key(key_bytes, [&](auto k) {
    emb_pw_fill_kernel<type_of<decltype(k)>><<<grid, 256, 0, st>>>(
        static_cast<const type_of<decltype(k)>*>(keys), weights, valid, regions);
  });
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// table_bf16: the arena's weight type (fp32 or bf16; serving arenas take no gradient); vec4: every selected
// lookup's width, gradient offset and stride, the pitch and the table and gradient pointers are 4-element aligned
extern "C" int hctr_emb_pw_dot(const EmbParams* p, const int* sel, int nsel, float* dots, long long dot_stride,
                               int key_bytes, int grad_bf16, int table_bf16, int vec4, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  const long long bags = static_cast<long long>(p->num_ranks) * nsel * p->batch;
  if (bags == 0) return 0;
  if (bags >= (1ll << 31)) return -4;
  long long blocks = (bags + 7) / 8;
  if (blocks > 16 * num_sms()) blocks = 16 * num_sms();
  with_key(key_bytes, [&](auto k) { with_elem(grad_bf16, [&](auto g) { with_elem(table_bf16, [&](auto w) {
    using K = type_of<decltype(k)>;
    using G = type_of<decltype(g)>;
    using W = type_of<decltype(w)>;
    if (vec4) emb_pw_dot_kernel<K, G, W, 4><<<static_cast<unsigned>(blocks), 256, 0, st>>>(*p, sel, nsel, dots, dot_stride);
    else emb_pw_dot_kernel<K, G, W, 1><<<static_cast<unsigned>(blocks), 256, 0, st>>>(*p, sel, nsel, dots, dot_stride);
  }); }); });
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int hctr_emb_pw_reduce(const float* dots, long long row_stride, int batch, int ranks,
                                  const PwReduceCol* cols, const PwReduceTarget* targets, int num_targets,
                                  void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (num_targets <= 0 || batch <= 0 || ranks <= 0) return 0;
  if (static_cast<long long>(ranks) * batch >= (1ll << 31)) return -4;
  emb_pw_reduce_kernel<<<num_targets, 256, 0, st>>>(dots, row_stride, batch, ranks, cols, targets);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
