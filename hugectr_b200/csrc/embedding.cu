// Sparse hot path: model-parallel embedding lookup / pooling and fused backward + optimizer.
//
// Owner-side design (one process per GPU, tables sharded table-wise and/or row-wise):
//   forward  : ONE kernel on the owner pulls the requesters' keys straight out of their (peer
//              mapped) key buffers, gathers + pools the rows from local HBM and stores the pooled
//              vectors straight into the requester's activation tensor over NVLink.  This replaces
//              the reference chain  key all-to-all (X11/X12, with a host sync)  ->  lookup  ->
//              ModelForward -> NCCL all-to-all (X14) -> NetworkForward
//              (HugeCTR/embedding/model_parallel_embedding.cpp:213-231,
//               HugeCTR/embedding/operators/generic_lookup.cuh:319-716).
//   backward : gradient rows are read from the requesters' (peer) top-grad tensors, de-duplicated
//              with a transient open-addressing hash (no sort, no host sync) and accumulated in
//              fp32; a fused per-unique-row optimizer kernel then updates weights + state.
//              Replaces NetworkBackward + all-to-all + index calculation (CUB sorts) + LocalReduce
//              + update (HugeCTR/embedding/operators/index_calculation.cu:102-887,
//              HugeCTR/embedding_storage/ragged_static_embedding.cu:93-345).
// With num_ranks == 1 all "peer" pointers are local and the same kernels serve a single GPU.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "embedding.cuh"

namespace hctr {

// ------------------------------------------------------------------ forward
// One group of G lanes per (src rank, lookup, sample) bucket; each lane owns VEC consecutive
// floats per 32*VEC-wide column chunk.  G*VEC >= ev for ev <= 128 (VEC=4), wider rows loop over
// up to MAXC chunks per lane: one launch covers columns [col_base, col_base + MAXC * G * VEC).
// WT: weight type of the arena (fp32, bf16 loaded 8 bytes per 4 columns, or e4m3: VEC = 16 columns in one
// 16-byte load per lane when the rows are whole 16-byte units, else 4 or 1 columns); pooling is in fp32.
// WGT: weighted lookups may be present; a row enters as fma(w, row, acc) (w = 1 for unweighted
// lookups and 0 for skipped keys: fma(1, v, acc) == acc + v, so all-ones weights pool bit for bit as
// the unweighted kernel does).
// e4m3 arenas (FP8) always take the fma path: the lane that resolves a key also reads its row's
// exponent byte and folds 2^e into the key's weight, which travels with the row as the weights do.
// w * 2^e and q * 2^e are exact, so fma(w * 2^e, q, acc) == fma(w, q * 2^e, acc): the lookup pools bit
// for bit as the fp32 kernel over the dequantized rows.
template <typename KeyT, typename OutT, int VEC, int U, typename WT, bool WGT>
__global__ void __launch_bounds__(256, 3)
    emb_fwd_kernel(const EmbParams p, const int G, const int col_base) {
  // grid.y = (src rank, lookup): uniform per block, no per-thread integer division
  const int lane = threadIdx.x & 31;
  const int groups_per_warp = 32 / G;
  const int gl = lane % G;  // lane inside group
  const int gi = lane / G;  // group inside warp
  const int l = blockIdx.y % p.num_lookups;
  const int src = blockIdx.y / p.num_lookups;
  const int s = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * groups_per_warp + gi;
  const bool active = s < p.batch;
  const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (gi * G));
  const EmbLookup lk = p.lookups[l];
  const int ev = lk.ev_size;
  int nnz = lk.hotness;
  const KeyT* kbase = reinterpret_cast<const KeyT*>(p.keys[src]) + lk.key_off +
                      static_cast<long long>(s) * lk.key_stride;
  if (active && lk.nnz_off >= 0) nnz = min(lk.hotness, p.nnz[src][lk.nnz_off + s]);
  if (!active) nnz = 0;
  const WT* table = static_cast<const WT*>(p.table);
  constexpr bool FP8 = std::is_same<WT, __nv_fp8_e4m3>::value;
  constexpr bool SCALED = WGT || FP8;   // rows enter as fma(factor, row, acc)
  const bool lw = WGT && lk.weighted;
  const float* wbase = WGT ? p.weights[src] + lk.key_off + static_cast<long long>(s) * lk.key_stride : nullptr;

  // chunks per lane.  Weighted vector rows keep 8 chunks at 4 rows in flight: the U weights beside 8 rows' loads
  // and the accumulators exceed the 80 registers of __launch_bounds__(256, 3) and spill
  // (e4m3 rows: exactly the chunks kMaxEmbWidth needs at 32 lanes, so that no chunk's accumulators are held in vain)
  constexpr int MAXC = (FP8 && VEC >= 4) ? kMaxEmbWidth / (32 * VEC) : ((U >= 8 || (WGT && VEC == 4)) ? 8 : 4);
  float acc[MAXC][VEC];
#pragma unroll
  for (int c = 0; c < MAXC; ++c)
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[c][v] = 0.f;
  const int nchunk = (ev - col_base + G * VEC - 1) / (G * VEC);

  // gathers U rows (rp[u] == nullptr: skip) with factors wv (SCALED only) into the accumulators
  auto gather = [&](const WT* const (&rp)[U], const float (&wv)[U]) {
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      if (c < nchunk) {
        const int col = col_base + (c * G + gl) * VEC;
        if (col < ev) {
          if constexpr (VEC == 4) {
            float4 v[U];
#pragma unroll
            for (int u = 0; u < U; ++u)
              v[u] = rp[u] ? ldg_row4(rp[u] + col) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int u = 0; u < U; ++u) {
              if constexpr (SCALED) {
                acc[c][0] = fmaf(wv[u], v[u].x, acc[c][0]); acc[c][1] = fmaf(wv[u], v[u].y, acc[c][1]);
                acc[c][2] = fmaf(wv[u], v[u].z, acc[c][2]); acc[c][3] = fmaf(wv[u], v[u].w, acc[c][3]);
              } else {
                acc[c][0] += v[u].x; acc[c][1] += v[u].y; acc[c][2] += v[u].z; acc[c][3] += v[u].w;
              }
            }
          } else if constexpr (VEC == 16) {
            // e4m3 rows only: 16 bytes per lane and chunk in one load per row (docs/performance.md: faster than
            // 4 or 8 bytes per lane at ev 128 and 256)
            uint4 v[U];
#pragma unroll
            for (int u = 0; u < U; ++u)
              v[u] = rp[u] ? __ldg(reinterpret_cast<const uint4*>(rp[u] + col)) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
            for (int u = 0; u < U; ++u) {
#pragma unroll
              for (int k = 0; k < VEC / 4; ++k) {
                const float4 f = e4m3x4_to_float4(word_of(v[u], k));
                acc[c][4 * k] = fmaf(wv[u], f.x, acc[c][4 * k]);
                acc[c][4 * k + 1] = fmaf(wv[u], f.y, acc[c][4 * k + 1]);
                acc[c][4 * k + 2] = fmaf(wv[u], f.z, acc[c][4 * k + 2]);
                acc[c][4 * k + 3] = fmaf(wv[u], f.w, acc[c][4 * k + 3]);
              }
            }
          } else {
            float v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) v[u] = rp[u] ? ldg_row1(rp[u] + col) : 0.f;
#pragma unroll
            for (int u = 0; u < U; ++u) {
              if constexpr (SCALED) acc[c][0] = fmaf(wv[u], v[u], acc[c][0]);
              else acc[c][0] += v[u];
            }
          }
        }
      }
    }
  };

  if (lk.num_shards > 1) {
    // Row-sharded table (block-uniform branch): this shard owns ~1/num_shards of the bag, so the
    // owned keys are compacted first -- every lane fetches up to 4 keys, a group ballot marks the
    // owned ones, and rows are gathered U at a time from the compacted set.  (Gathering in key order
    // would issue one row per round for an 8-way shard: a chain of dependent DRAM latencies.)
    const int KPL = (G >= 32) ? 1 : ((G >= 16) ? 2 : 4);   // keys per lane and round; KPL * G <= 32
    const unsigned int ns = static_cast<unsigned int>(lk.num_shards);
    for (int h0 = 0; h0 < nnz; h0 += KPL * G) {
      unsigned int rowv[4] = {0u, 0u, 0u, 0u};
      float wtv[4] = {1.f, 1.f, 1.f, 1.f};   // SCALED: the weights (times 2^e) travel with rowv
      unsigned int m = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (i < KPL) {
          const int h = h0 + i * G + gl;
          bool ok = false;
          if (h < nnz) {
            const long long key = static_cast<long long>(kbase[h]);
            if (key >= 0) {
              const unsigned long long uk = static_cast<unsigned long long>(key);
              unsigned long long q;
              unsigned int rem;
              if (uk <= 0xFFFFFFFFull) {        // 32-bit fast path (no 64-bit division)
                const unsigned int k32 = static_cast<unsigned int>(uk);
                q = k32 / ns;
                rem = k32 - static_cast<unsigned int>(q) * ns;
              } else {
                q = uk / ns;
                rem = static_cast<unsigned int>(uk - q * ns);
              }
              ok = rem == static_cast<unsigned int>(lk.shard_idx) && q < static_cast<unsigned long long>(lk.rows);
              rowv[i] = static_cast<unsigned int>(q);
              if (lw && ok) wtv[i] = wbase[h];
              if constexpr (FP8) {
                if (ok) wtv[i] *= row_scale(p.row_exp, lk.table_row_off + static_cast<long long>(q));
              }
            }
          }
          const unsigned int bal = (__ballot_sync(gmask, ok) >> (gi * G)) & ((G == 32) ? 0xffffffffu : ((1u << G) - 1u));
          m |= bal << (i * G);
        }
      }
      while (m) {               // group-uniform
        const WT* rp[U];
        float wv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          rp[u] = nullptr;
          const bool take = m != 0u;
          const int b = take ? (__ffs(m) - 1) : 0;
          if (take) m &= m - 1u;
          const int i = b / G, sl = b - i * G;
          const unsigned int cand = i == 0 ? rowv[0] : (i == 1 ? rowv[1] : (i == 2 ? rowv[2] : rowv[3]));
          const unsigned int r = __shfl_sync(gmask, cand, gi * G + sl);
          if (take) rp[u] = table + (lk.table_row_off + r) * static_cast<long long>(p.ev_size);
          if constexpr (SCALED) {
            const float cw = i == 0 ? wtv[0] : (i == 1 ? wtv[1] : (i == 2 ? wtv[2] : wtv[3]));
            const float w = __shfl_sync(gmask, cw, gi * G + sl);
            wv[u] = take ? w : 0.f;
          }
        }
        gather(rp, wv);
      }
    }
  } else {
    for (int h0 = 0; h0 < nnz; h0 += G) {
      // lanes of the group fetch up to G keys at once (coalesced peer/local read)
      long long mykey = -1;
      if (h0 + gl < nnz) mykey = static_cast<long long>(kbase[h0 + gl]);
      float myw = 1.f;
      if (lw && h0 + gl < nnz) myw = wbase[h0 + gl];
      if constexpr (FP8) {
        if (mykey >= 0 && mykey < lk.rows) myw *= row_scale(p.row_exp, lk.table_row_off + mykey);
      }
      const int cnt = min(G, nnz - h0);
      for (int j0 = 0; j0 < cnt; j0 += U) {
        const WT* rp[U];
        float wv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int j = j0 + u;
          const long long key = __shfl_sync(gmask, mykey, gi * G + (j < cnt ? j : 0));
          const bool ok = (j < cnt) && key >= 0 && key < lk.rows;
          rp[u] = ok ? table + (lk.table_row_off + key) * static_cast<long long>(p.ev_size) : nullptr;
          if constexpr (SCALED) {
            const float w = __shfl_sync(gmask, myw, gi * G + (j < cnt ? j : 0));
            wv[u] = ok ? w : 0.f;
          }
        }
        gather(rp, wv);
      }
    }
  }
  if (!active) return;
  float scale = 1.f;
  if (lk.combiner == 1 && nnz > 0) scale = 1.f / static_cast<float>(nnz);
  OutT* o = reinterpret_cast<OutT*>(p.out[src]) + lk.out_off +
            static_cast<long long>(s) * lk.out_stride;
#pragma unroll
  for (int c = 0; c < MAXC; ++c) {
    if (c < nchunk) {
      const int col = col_base + (c * G + gl) * VEC;
      if (col < ev) {
        if constexpr (VEC >= 4) {
#pragma unroll
          for (int k = 0; k < VEC / 4; ++k)
            store_vec4<OutT>(o + col + 4 * k, acc[c][4 * k] * scale, acc[c][4 * k + 1] * scale,
                             acc[c][4 * k + 2] * scale, acc[c][4 * k + 3] * scale);
        } else {
          o[col] = from_f<OutT>(acc[c][0] * scale);
        }
      }
    }
  }
}

// ------------------------------------------------------------------ backward accumulate
// Same bucket decomposition as forward.  Each group loads its bucket's gradient row once and
// red.adds it (fp32) into wgrad_unique[uid] for every owned key of the bucket; WGT: times the key's
// weight (weighted lookups).
template <typename KeyT, typename GradT, int VEC, bool WGT>
__global__ void __launch_bounds__(256)
    emb_bwd_accum_kernel(const EmbParams p, const UniqueTable ut, float* __restrict__ wgrad_unique,
                         const float grad_scale, const int G, const long long total_items) {
  const int lane = threadIdx.x & 31;
  const int groups_per_warp = 32 / G;
  const int gl = lane % G;
  const int gi = lane / G;
  const long long warp_global = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const long long item = warp_global * groups_per_warp + gi;
  const bool active = item < total_items;
  const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (gi * G));
  int s = 0, l = 0, src = 0;
  if (active) {
    s = static_cast<int>(item % p.batch);
    const long long t = item / p.batch;
    l = static_cast<int>(t % p.num_lookups);
    src = static_cast<int>(t / p.num_lookups);
  }
  const EmbLookup lk = p.lookups[l];
  const int ev = lk.ev_size;
  int nnz = lk.hotness;
  const KeyT* kbase = reinterpret_cast<const KeyT*>(p.keys[src]) + lk.key_off +
                      static_cast<long long>(s) * lk.key_stride;
  if (active && lk.nnz_off >= 0) nnz = min(lk.hotness, p.nnz[src][lk.nnz_off + s]);
  if (!active) nnz = 0;

  constexpr int MAXC = 32 / VEC;   // ev <= MAXC * G * VEC = kMaxEmbWidth at G = 32
  float g[MAXC][VEC];
  const int nchunk = (ev + G * VEC - 1) / (G * VEC);
  float scale = grad_scale;
  if (lk.combiner == 1 && nnz > 0) scale /= static_cast<float>(nnz);
  if (active) {
    const GradT* gp = reinterpret_cast<const GradT*>(p.grad[src]) + lk.grad_off +
                      static_cast<long long>(s) * lk.grad_stride;
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      if (c < nchunk) {
        const int col = (c * G + gl) * VEC;
        if (col < ev) {
          if constexpr (VEC == 4) {
            const float4 v = load_vec4<GradT>(gp + col);
            g[c][0] = v.x * scale; g[c][1] = v.y * scale; g[c][2] = v.z * scale; g[c][3] = v.w * scale;
          } else {
            g[c][0] = to_f<GradT>(gp[col]) * scale;
          }
        }
      }
    }
  }
  for (int h0 = 0; h0 < nnz; h0 += G) {
    long long mykey = -1;
    if (h0 + gl < nnz) mykey = static_cast<long long>(kbase[h0 + gl]);
    float myw = 1.f;
    if (WGT && h0 + gl < nnz) myw = key_weight(p, lk, src, s, h0 + gl);
    // every lane resolves the unique id of ITS key (parallel hash probes), then broadcast
    unsigned int myuid = kInvalidVal;
    if (mykey >= 0 && (lk.num_shards == 1 || (mykey % lk.num_shards) == lk.shard_idx)) {
      const long long r = mykey / lk.num_shards;
      if (r < lk.rows) {
        const unsigned long long arow = static_cast<unsigned long long>(lk.table_row_off + r);
        // ut.keys == nullptr : dense wgrad [rows, ev] (data-parallel tables), uid == arena row
        myuid = ut.keys ? unique_get_insert(ut, arow) : static_cast<unsigned int>(arow);
      }
    }
    const int cnt = min(G, nnz - h0);
    for (int j = 0; j < cnt; ++j) {
      const unsigned int uid = __shfl_sync(gmask, myuid, gi * G + j);
      float w = 1.f;
      if constexpr (WGT) w = __shfl_sync(gmask, myw, gi * G + j);
      if (uid == kInvalidVal || uid >= ut.max_unique) continue;
      float* dst = wgrad_unique + static_cast<long long>(uid) * p.ev_size;
#pragma unroll
      for (int c = 0; c < MAXC; ++c) {
        if (c < nchunk) {
          const int col = (c * G + gl) * VEC;
          if (col < ev) {
            if constexpr (VEC == 4) {
              if constexpr (WGT) {
                asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + col),
                             "f"(g[c][0] * w), "f"(g[c][1] * w), "f"(g[c][2] * w), "f"(g[c][3] * w)
                             : "memory");
              } else {
                asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + col),
                             "f"(g[c][0]), "f"(g[c][1]), "f"(g[c][2]), "f"(g[c][3])
                             : "memory");
              }
            } else {
              atomicAdd(dst + col, WGT ? g[c][0] * w : g[c][0]);
            }
          }
        }
      }
    }
  }
}

// Data-parallel tables (small, replicated): dense wgrad [rows, pitch] += scattered bag gradients of
// the LOCAL batch.  Hot rows of tiny tables would serialise global reductions on a handful of L2
// lines, so a block (one lookup x one chunk of samples) first accumulates into a shared-memory copy
// of the table when it fits and flushes it with one vector reduction per non-zero 16-byte group.
// WGT: every key's share is scaled by its weight (weighted lookups).
template <typename KeyT, typename GradT, bool WGT>
__global__ void __launch_bounds__(256)
    emb_dp_wgrad_kernel(const EmbParams p, float* __restrict__ wgrad, const float grad_scale,
                        const int smem_floats) {
  extern __shared__ float dp_acc[];
  const EmbLookup lk = p.lookups[blockIdx.y];
  const int ev = lk.ev_size, pitch = p.ev_size;
  const long long tbl_floats = static_cast<long long>(lk.rows) * ev;
  const bool priv = tbl_floats <= smem_floats;
  const int per = (p.batch + gridDim.x - 1) / gridDim.x;
  const int s0 = blockIdx.x * per, s1 = min(p.batch, s0 + per);
  if (priv) {
    for (int i = threadIdx.x; i < tbl_floats; i += blockDim.x) dp_acc[i] = 0.f;
    __syncthreads();
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const KeyT* keys = reinterpret_cast<const KeyT*>(p.keys[0]) + lk.key_off;
  const GradT* grads = reinterpret_cast<const GradT*>(p.grad[0]) + lk.grad_off;
  for (int s = s0 + warp; s < s1; s += 8) {
    const int nnz = bucket_nnz(p, lk.hotness, lk.nnz_off, 0, s);
    if (nnz <= 0) continue;
    float scale = grad_scale;
    if (lk.combiner == 1) scale /= static_cast<float>(nnz);
    const KeyT* kb = keys + static_cast<long long>(s) * lk.key_stride;
    const GradT* gp = grads + static_cast<long long>(s) * lk.grad_stride;
    for (int col = lane * 4; col < ev; col += 128) {
      float4 v = load_vec4<GradT>(gp + col);
      v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
      for (int h = 0; h < nnz; ++h) {
        const long long key = static_cast<long long>(kb[h]);
        if (key < 0 || key >= lk.rows) continue;
        float4 u = v;
        if constexpr (WGT) u = scale4(v, key_weight(p, lk, 0, s, h));
        if (priv) {
          float* d = dp_acc + key * ev + col;
          atomicAdd(d, u.x); atomicAdd(d + 1, u.y); atomicAdd(d + 2, u.z); atomicAdd(d + 3, u.w);
        } else {
          float* d = wgrad + (lk.table_row_off + key) * pitch + col;
          asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d), "f"(u.x), "f"(u.y),
                       "f"(u.z), "f"(u.w) : "memory");
        }
      }
    }
  }
  if (priv) {
    __syncthreads();
    for (long long i = threadIdx.x * 4ll; i < tbl_floats; i += blockDim.x * 4ll) {
      const float4 v = *reinterpret_cast<const float4*>(dp_acc + i);
      if (v.x == 0.f && v.y == 0.f && v.z == 0.f && v.w == 0.f) continue;
      const long long r = i / ev;
      const int c = static_cast<int>(i - r * ev);
      float* d = wgrad + (lk.table_row_off + r) * pitch + c;
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d), "f"(v.x), "f"(v.y),
                   "f"(v.z), "f"(v.w) : "memory");
    }
  }
}

// A row-reduced rule (row-wise AdaGrad, partial row-wise Adam) on one row by one warp (accumulate path
// and data-parallel tables): a warp-reduced pass over the row's fp32 gradient gives sum g^2,
// row_reduce_step updates the row's state *s, then the update pass applies the factor to every column
// (partial row-wise Adam: through the first moments m0 of the arena's element indices) and zeroes the
// gradient.
template <int OPT, typename StateT, typename WT>
HCTR_DEVICE void rowwise_update_warp(WT* table, float* s, StateT* m0, float* gsrc, long long base, int ev,
                                      float inv_scaler, const OptHyper& hp, const OptStep& st,
                                      unsigned long long srk, int lane) {
  const bool v4 = (ev & 3) == 0;
  float sq = 0.f;
  if (v4) {
    for (int col = lane * 4; col < ev; col += 128) {
      const float4 g = *reinterpret_cast<const float4*>(gsrc + col);
      sq += sumsq4(scale4(g, inv_scaler));
    }
  } else {
    for (int col = lane; col < ev; col += 32) {
      const float g = gsrc[col] * inv_scaler;
      sq += g * g;
    }
  }
  const float s_old = lane == 0 ? *s : 0.f;
  const float f = row_reduce_step<OPT, 32>(0xffffffffu, 0, lane, sq, s_old, s, ev, hp, st);
  if (v4) {
    for (int col = lane * 4; col < ev; col += 128) {
      const float4 g = *reinterpret_cast<float4*>(gsrc + col);
      *reinterpret_cast<float4*>(gsrc + col) = make_float4(0.f, 0.f, 0.f, 0.f);
      float4 w = load_vec4<WT>(table + base + col);
      row_apply4<OPT, StateT>(w, scale4(g, inv_scaler), f, m0, base + col, hp);
      store_w4<WT>(table + base + col, w, srk, base + col);
    }
  } else {
    for (int col = lane; col < ev; col += 32) {
      const float g = gsrc[col] * inv_scaler;
      gsrc[col] = 0.f;
      float w = to_f<WT>(table[base + col]);
      row_apply1<OPT, StateT>(w, g, f, m0, base + col, hp);
      store_w<WT>(table + base + col, w, srk, base + col);
    }
  }
}

// One warp per unique row: reads the accumulated fp32 gradient (and zeroes it for the next step),
// updates weight + optimizer state in place and releases the row's hash slot.
template <int OPT, typename StateT, typename WT>
__global__ void __launch_bounds__(256)
    emb_update_kernel(WT* __restrict__ table, StateT* __restrict__ s0, StateT* __restrict__ s1,
                      float* __restrict__ wgrad_unique, const UniqueTable ut, const int ev,
                      const OptHyper hp) {
  const unsigned int n = min(*ut.counter, ut.max_unique);
  const OptStep step = opt_step<OPT>(hp);
  const float inv_scaler = 1.f / hp.scaler;
  const unsigned long long srk = sr_key<WT>(hp.sr_seed, hp.step_ptr);
  const int lane = threadIdx.x & 31;
  const unsigned int warps = (gridDim.x * blockDim.x) >> 5;
  for (unsigned int uid = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; uid < n; uid += warps) {
    const unsigned long long row = ut.rows[uid];
    float* gsrc = wgrad_unique + static_cast<long long>(uid) * ev;
    const long long base = static_cast<long long>(row) * ev;
    if constexpr (kRowRule<OPT>) {
      rowwise_update_warp<OPT, StateT, WT>(table, row_state<OPT>(s0, s1) + row, s0, gsrc, base, ev, inv_scaler,
                                           hp, step, srk, lane);
    } else if ((ev & 3) == 0) {
      for (int col = lane * 4; col < ev; col += 128) {
        float4 g = *reinterpret_cast<float4*>(gsrc + col);
        *reinterpret_cast<float4*>(gsrc + col) = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 w = load_vec4<WT>(table + base + col);
        apply_opt4<OPT, StateT>(w, scale4(g, inv_scaler), s0, s1, base + col, hp, step);
        store_w4<WT>(table + base + col, w, srk, base + col);
      }
    } else {
      for (int col = lane; col < ev; col += 32) {
        const float g = gsrc[col];
        gsrc[col] = 0.f;
        float w = to_f<WT>(table[base + col]);
        apply_opt<OPT, StateT>(w, g * inv_scaler, s0, s1, base + col, hp, step);
        store_w<WT>(table + base + col, w, srk, base + col);
      }
    }
    if (lane == 0) unique_release(ut, uid);
  }
}

// Data-parallel tables with row-wise AdaGrad: every row of the all-reduced dense wgrad [rows, pitch]
// takes the row rule (one warp per row) and is zeroed.  An all-zero row leaves s and w as they are,
// as the element-wise AdaGrad of the dense optimizer does.
__global__ void __launch_bounds__(256)
    emb_dp_rowwise_update_kernel(float* __restrict__ table, float* __restrict__ s,
                                 float* __restrict__ wgrad, const long long rows, const int pitch,
                                 const OptHyper hp) {
  const OptStep step = opt_step<OPT_ROWWISE_ADAGRAD>(hp);
  const float inv_scaler = 1.f / hp.scaler;
  const int lane = threadIdx.x & 31;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  for (long long r = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; r < rows;
       r += warps)
    rowwise_update_warp<OPT_ROWWISE_ADAGRAD, float, float>(table, s + r, nullptr, wgrad + r * pitch, r * pitch,
                                                          pitch, inv_scaler, hp, step, 0ull, lane);
}

// Data-parallel tables with partial row-wise Adam: table and first moments m [rows, pitch] fp32, second
// moments v [rows] fp32.  A row whose all-reduced gradient is all zero is skipped: its weights and both
// moments stay as they are, as an all-zero row leaves them under row-wise AdaGrad (a model-parallel row that
// was looked up takes the step with g = 0 instead, and its moments decay).
__global__ void __launch_bounds__(256)
    emb_dp_prow_adam_update_kernel(float* __restrict__ table, float* __restrict__ m, float* __restrict__ v,
                                   float* __restrict__ wgrad, const long long rows, const int pitch,
                                   const OptHyper hp) {
  const OptStep step = opt_step<OPT_PARTIAL_ROWWISE_ADAM>(hp);
  const float inv_scaler = 1.f / hp.scaler;
  const int lane = threadIdx.x & 31;
  const long long warps = (static_cast<long long>(gridDim.x) * blockDim.x) >> 5;
  for (long long r = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; r < rows;
       r += warps) {
    const float* g = wgrad + r * pitch;
    bool any = false;
    for (int c = lane; c < pitch; c += 32) any |= g[c] != 0.f;
    if (!__any_sync(0xffffffffu, any)) continue;
    rowwise_update_warp<OPT_PARTIAL_ROWWISE_ADAM, float, float>(table, v + r, m, wgrad + r * pitch, r * pitch,
                                                               pitch, inv_scaler, hp, step, 0ull, lane);
  }
}

__global__ void emb_finish_kernel(unsigned int* counter, unsigned int* overflow_flag,
                                  unsigned int max_unique) {
  if (*counter > max_unique) atomicMax(overflow_flag, *counter);
  *counter = 0;
}

// plain gather (no pooling): out[i] = table[rows[i]]  (concat combiner / dense lookups / SOK)
template <typename OutT, typename WT>
__global__ void emb_gather_rows_kernel(const WT* __restrict__ table, const long long* rows,
                                       OutT* out, long long n, int ev) {
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const long long r = rows[w];
  for (int c = lane; c < ev; c += 32)
    out[w * ev + c] = from_f<OutT>(r < 0 ? 0.f : to_f<WT>(table[r * ev + c]));
}

// Serving arenas: quantizes fp32 rows src [n, pitch] into arena rows rows[i] of the e4m3 arena q
// [*, pitch], one warp per row: exps[row] = e + 127 with e = e4m3_scale_exp(amax of the row) and
// q = e4m3_satfinite_rn(x * 2^-e) (mirrored by embedding/ops.py::fp8_rows_quantize).  A non-finite
// value sets *bad; the caller reads the flag once per load and rejects the load.
__global__ void __launch_bounds__(256)
    emb_quantize_rows_kernel(const float* __restrict__ src, const long long* __restrict__ rows, long long n,
                             int pitch, uint8_t* __restrict__ q, uint8_t* __restrict__ exps, int* bad) {
  const long long w = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n) return;
  const float* x = src + w * pitch;
  float amax = 0.f;
  bool finite = true;
  for (int c = lane; c < pitch; c += 32) {
    const float v = x[c];
    finite &= isfinite(v);
    amax = fmaxf(amax, fabsf(v));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  if (!__all_sync(0xffffffffu, finite) && lane == 0) *bad = 1;
  const int e = e4m3_scale_exp(amax);
  const long long r = rows[w];
  uint8_t* d = q + r * pitch;
  for (int c = lane; c < pitch; c += 32)
    d[c] = static_cast<uint8_t>(__nv_cvt_float_to_fp8(e4m3_scale_down(x[c], e), __NV_SATFINITE, __NV_E4M3));
  if (lane == 0) exps[r] = static_cast<uint8_t>(e + 127);
}

// Update tracking (embedding/collection.py, track_updates): stamp[rows[i]] = *clock for the first
// min(*counter, max_unique) entries of a step's unique-row list.  The count and the clock are read on the
// device, so a replayed graph stamps with the clock of its own step.  The rows of a list are distinct: plain
// stores.  Rows at or beyond row_bound are skipped.  Every thread loads kStampIlp list entries before it stores
// any, so that each thread keeps that many independent loads in flight.
constexpr int kStampIlp = 4;
__global__ void __launch_bounds__(256)
    emb_stamp_rows_kernel(int* __restrict__ stamp, const unsigned long long* __restrict__ rows,
                          const unsigned int* __restrict__ counter, unsigned int max_unique,
                          long long row_bound, const long long* __restrict__ clock) {
  const unsigned int n = min(*counter, max_unique);
  const int c = static_cast<int>(*clock);
  const unsigned int stride = gridDim.x * blockDim.x;
  for (unsigned int i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < n; i0 += kStampIlp * stride) {
    unsigned long long r[kStampIlp];
#pragma unroll
    for (int k = 0; k < kStampIlp; ++k) {
      const unsigned long long i = i0 + static_cast<unsigned long long>(k) * stride;
      r[k] = i < n ? __ldg(rows + i) : ~0ull;
    }
#pragma unroll
    for (int k = 0; k < kStampIlp; ++k)
      if (r[k] < static_cast<unsigned long long>(row_bound)) stamp[r[k]] = c;
  }
}

}  // namespace hctr

using namespace hctr;

static inline int pick_group(int ev, int vec) {
  int g = (ev + vec - 1) / vec;
  int p = 1;
  while (p < g && p < 32) p <<= 1;
  return p;
}

// key_bytes: 4 or 8 ; out_bf16 / grad_bf16 : element type of activations ; table_bf16 : of the arena
// (hctr_emb_forward's table_type: 0 fp32, 1 bf16, 2 e4m3 with p->row_exp)
// aligned4 (4, or 16 for an e4m3 arena whose lookup widths and pitch are multiples of 16): every lookup's
// ev_size, out_off and out_stride, the table pitch and the base pointers are
// multiples of 4 elements (whole-vector table rows and output stores); 0 selects scalar accesses
extern "C" int hctr_emb_forward(const EmbParams* p, int max_ev, int key_bytes, int out_bf16,
                                int aligned4, int table_type, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (max_ev > kMaxEmbWidth) return -4;
  int vec = (aligned4 && max_ev % 4 == 0) ? 4 : 1;
  // e4m3 arenas whose rows are whole 16-byte units (aligned4 == 16): one 16-byte load per lane and row
  if (table_type == 2 && aligned4 == 16 && max_ev % 16 == 0) vec = 16;
  int G = pick_group(max_ev, vec);
  // wide rows: 8 lanes per bucket, every lane owns up to 4 float4 chunks of the row -> 4 buckets
  // per warp and 16 independent 16-byte loads in flight per lane (latency-bound -> bandwidth-bound)
  const bool narrow = (vec == 4 && max_ev >= 64 && max_ev <= 128);
  if (narrow) G = 8;
  const long long items = static_cast<long long>(p->num_ranks) * p->num_lookups * p->batch;
  if (items == 0) return 0;
  const int threads = 256;
  const int buckets_per_block = (threads / 32) * (32 / G);
  const dim3 blocks((p->batch + buckets_per_block - 1) / buckets_per_block,
                    p->num_ranks * p->num_lookups);
  // one pass covers every column, except scalar rows wider than 8 chunks x 32 lanes: those take
  // passes of 256 columns (keeps the accumulators of the scalar kernel in registers)
  const int pass = (vec >= 4) ? max_ev : 8 * G;
  for (int c0 = 0; c0 < max_ev; c0 += pass) {
    with_key(key_bytes, [&](auto k) { with_elem(out_bf16, [&](auto o) { with_table(table_type, [&](auto w) {
      with_weighted(*p, [&](auto wgt) {
        auto launch = [&](auto v, auto u) {   // vector width, rows in flight per gather round
          emb_fwd_kernel<type_of<decltype(k)>, type_of<decltype(o)>, decltype(v)::value, decltype(u)::value,
                         type_of<decltype(w)>, decltype(wgt)::value><<<blocks, threads, 0, st>>>(*p, G, c0);
        };
        if constexpr (std::is_same<type_of<decltype(w)>, __nv_fp8_e4m3>::value) {
          if (vec == 16) launch(Int<16>{}, Int<4>{});
          else if (vec == 4) launch(Int<4>{}, Int<2>{});
          else launch(Int<1>{}, Int<8>{});
        } else {
          if (vec == 1) launch(Int<1>{}, Int<8>{});
          else if (narrow) launch(Int<4>{}, Int<4>{});
          else launch(Int<4>{}, Int<decltype(wgt)::value ? 4 : 8>{});
        }
      });
    }); }); });
  }
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int hctr_emb_backward_accum(const EmbParams* p, const UniqueTable* ut,
                                       float* wgrad_unique, float grad_scale, int max_ev,
                                       int key_bytes, int grad_bf16, int dp_ev4, void* stream_) {
  // dp_ev4: every lookup's ev_size, grad_off and grad_stride, the pitch and the base pointers are
  // multiples of 4 elements (whole-vector gradient loads); 0 selects scalar accesses
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  const int vec = (dp_ev4 && max_ev % 4 == 0) ? 4 : 1;
  const int G = pick_group(max_ev, vec);
  const long long items = static_cast<long long>(p->num_ranks) * p->num_lookups * p->batch;
  if (items == 0) return 0;
  if (ut->keys == nullptr && p->num_ranks == 1 && dp_ev4 && p->ev_size % 4 == 0) {
    // dense wgrad of replicated tables: privatised block-level accumulation
    constexpr int kSmem = 96 * 1024;
    int chunks = (2 * num_sms() + p->num_lookups - 1) / p->num_lookups;
    if (chunks > 64) chunks = 64;
    if (chunks * 8 > p->batch) chunks = (p->batch + 7) / 8;
    if (chunks < 1) chunks = 1;
    const dim3 grid(chunks, p->num_lookups);
    with_key(key_bytes, [&](auto k) { with_elem(grad_bf16, [&](auto g) { with_weighted(*p, [&](auto wgt) {
      const auto kernel = emb_dp_wgrad_kernel<type_of<decltype(k)>, type_of<decltype(g)>, decltype(wgt)::value>;
      // once per instantiation: this static belongs to the (k, g, wgt) instance of the lambda
      static const cudaError_t attr =
          cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
      (void)attr;
      kernel<<<grid, 256, kSmem, st>>>(*p, wgrad_unique, grad_scale, kSmem / 4);
    }); }); });
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
  }
  if (max_ev > kMaxEmbWidth) return -4;
  const long long warps = (items + (32 / G) - 1) / (32 / G);
  const int threads = 256;
  const long long blocks = (warps * 32 + threads - 1) / threads;
  with_key(key_bytes, [&](auto k) { with_elem(grad_bf16, [&](auto g) { with_weighted(*p, [&](auto wgt) {
    auto launch = [&](auto v) {
      emb_bwd_accum_kernel<type_of<decltype(k)>, type_of<decltype(g)>, decltype(v)::value, decltype(wgt)::value>
          <<<(unsigned)blocks, threads, 0, st>>>(*p, *ut, wgrad_unique, grad_scale, G, items);
    };
    if (vec == 4) launch(Int<4>{});
    else launch(Int<1>{});
  }); }); });
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int hctr_emb_update(void* table, void* s0, void* s1, float* wgrad_unique,
                               const UniqueTable* ut, int ev, int opt, int state_bf16,
                               const OptHyper* hp, unsigned int* overflow_flag, int num_sms,
                               int table_bf16, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  const int threads = 256;
  const int blocks = num_sms * 8;
  const int rc = dispatch_opt(opt, state_bf16, table_bf16, [&](auto o, auto s, auto w) {
    using StateT = type_of<decltype(s)>;
    using WT = type_of<decltype(w)>;
    emb_update_kernel<decltype(o)::value, StateT, WT><<<blocks, threads, 0, st>>>(
        (WT*)table, (StateT*)s0, (StateT*)s1, wgrad_unique, *ut, ev, *hp);
  });
  if (rc) return rc;
  emb_finish_kernel<<<1, 1, 0, st>>>(ut->counter, overflow_flag, ut->max_unique);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// Row-wise AdaGrad of a data-parallel table: table [rows, pitch] fp32, s [rows] fp32, wgrad the
// all-reduced dense gradient [rows, pitch] (zeroed on return)
extern "C" int hctr_emb_dp_rowwise_update(float* table, float* s, float* wgrad, long long rows,
                                          int pitch, const OptHyper* hp, int num_sms, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (rows <= 0) return 0;
  long long blocks = (rows * 32 + 255) / 256;
  if (blocks > num_sms * 8ll) blocks = num_sms * 8ll;
  emb_dp_rowwise_update_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(table, s, wgrad, rows,
                                                                              pitch, *hp);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// Partial row-wise Adam of a data-parallel table: table and m [rows, pitch] fp32, v [rows] fp32, wgrad the
// all-reduced dense gradient [rows, pitch] (zeroed on return; all-zero rows are skipped)
extern "C" int hctr_emb_dp_prow_adam_update(float* table, float* m, float* v, float* wgrad, long long rows,
                                            int pitch, const OptHyper* hp, int num_sms, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (rows <= 0) return 0;
  long long blocks = (rows * 32 + 255) / 256;
  if (blocks > num_sms * 8ll) blocks = num_sms * 8ll;
  emb_dp_prow_adam_update_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(table, m, v, wgrad, rows,
                                                                                pitch, *hp);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int hctr_emb_gather_rows(const void* table, const long long* rows, void* out,
                                    long long n, int ev, int out_bf16, int table_bf16, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (n == 0) return 0;
  const unsigned blocks = static_cast<unsigned>((n * 32 + 255) / 256);
  with_elem(out_bf16, [&](auto o) { with_elem(table_bf16, [&](auto w) {
    using OutT = type_of<decltype(o)>;
    using WT = type_of<decltype(w)>;
    emb_gather_rows_kernel<OutT, WT><<<blocks, 256, 0, st>>>((const WT*)table, rows, (OutT*)out, n, ev);
  }); });
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// rows: int64 [n] arena rows (distinct), src: fp32 [n, pitch] contiguous, q / exps: the e4m3 arena and
// its exponent bytes, bad: int32 flag set on a non-finite value
extern "C" int hctr_emb_quantize_rows(const float* src, const long long* rows, long long n, int pitch, void* q,
                                      unsigned char* exps, int* bad, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (n == 0) return 0;
  const unsigned blocks = static_cast<unsigned>((n * 32 + 255) / 256);
  emb_quantize_rows_kernel<<<blocks, 256, 0, st>>>(src, rows, n, pitch, static_cast<uint8_t*>(q), exps, bad);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// stamp: int32 [row_bound] per-row step stamps; rows / counter / max_unique: a unique-row list (UniqueTable's
// rows and counter); clock: int64 device clock.  The grid covers max_unique and exits at the device count.
extern "C" int hctr_emb_stamp_rows(int* stamp, const unsigned long long* rows, const unsigned int* counter,
                                   unsigned int max_unique, long long row_bound, const long long* clock,
                                   int num_sms, void* stream_) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream_);
  if (max_unique == 0) return 0;
  // one entry per thread up to 16 blocks per SM; longer lists take kStampIlp entries per thread and pass
  long long blocks = (static_cast<long long>(max_unique) + 255) / 256;
  if (blocks > num_sms * 16ll) blocks = num_sms * 16ll;
  emb_stamp_rows_kernel<<<static_cast<unsigned>(blocks), 256, 0, st>>>(stamp, rows, counter, max_unique,
                                                                       row_bound, clock);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
