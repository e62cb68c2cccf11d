// D1 / D3: persistent warp-specialised bf16 GEMM on Hopper tensor cores (wgmma.mma_async, register
// accumulators, TMA operand staging, mbarrier pipelines) with fused epilogues:
//   bias + ReLU            (MLP fprop;       replaces cuBLASLt RELU_AUX_BIAS epilogue,
//                           reference HugeCTR/src/layers/functors/fused_gemm_functors.cu:21-289)
//   dReLU mask multiply    (MLP dgrad;       reference DRELU_BGRAD epilogue)
//   fp32 (atomic) accum    (MLP/Cross wgrad; reference beta=1 wgrad, fused_fc_layer_functors.cu:161)
//   x0 * (acc + b) + xl    (DCNv2 cross;     reference HugeCTR/src/layers/multi_cross_layer.cu:625-672)
// Operands may be K-major or MN-major, so fprop (X*W, W=[in,out]), dgrad (dY*W^T) and wgrad
// (X^T*dY) all run from the same row-major tensors without any transposed copies.
//
// CTA = three warpgroups: warpgroup 0 is the TMA producer, warpgroups 1 and 2 each own 64 rows of the
// 128 x BN tile (one m64nBNk16 wgmma per 16-wide K step) and run the epilogue of their rows.
//
// Two epilogues, chosen on the host per call:
//  * TMA epilogue (TMA_EPI; bf16 outputs whose epilogue tensors TMA can address).  Warp 1 of the producer
//    warpgroup TMA-loads the x0 / xl / mask boxes of each 64-column group into a per-warpgroup ring while the
//    tile's main loop runs.  The consumers combine them with the accumulators in place, at the wgmma fragment
//    positions, and one thread TMA-stores the bf16 box (and aux) asynchronously; the slot is handed back to the
//    producer once the store has read it, which for a tile's last group happens in the next tile's main loop.
//  * Slab epilogue (fp32 / atomic outputs, tensors TMA cannot address): the accumulators leave the registers
//    through a per-warpgroup [64 x 64] fp32 staging slab, so the fused epilogue works on one row x 32 columns per
//    thread with vectorised global accesses.
#include <cstdio>
#include <cstring>

#include "gemm_epilogue.cuh"

namespace hctr {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 B = one SWIZZLE_128B row
constexpr int WG_K = 16;
constexpr int kNumThreads = 384;
constexpr int kSmemLimit = 232448;  // 227 KB opt-in shared memory per block on sm_90

// TMA epilogue ring: kEpiBoxes [64 rows x 64 columns] bf16 boxes (SWIZZLE_128B) per consumer warpgroup.  A
// 64-column group takes one box per tensor it reads (epi_in_boxes, at least one for the output), so the ring has
// 4 slots for EPI_ADD / EPI_MASK / output-only flag sets and 2 for EPI_CROSS.
constexpr int kEpiBoxBytes = 64 * 64 * 2;
constexpr int kEpiBoxes = 4;

// boxes of x0 / xl / mask (in that order within a slot) the TMA epilogue loads per 64-column group
__host__ __device__ inline int epi_in_boxes(int flags) {
  return ((flags & EPI_CROSS) ? 2 : (flags & EPI_ADD) ? 1 : 0) + ((flags & EPI_MASK) ? 1 : 0);
}

// Operand stages that fit beside the epilogue staging (slab / TMA ring): BN = 64: 7 / 6, BN = 128: 5 / 5,
// BN = 256: 3 / 3.
template <int BN, bool TMA_EPI>
struct SmemLayout {
  static constexpr int kABytes = BLOCK_M * BLOCK_K * 2;
  static constexpr int kBBytes = BN * BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kEpiBytes = TMA_EPI ? 2 * kEpiBoxes * kEpiBoxBytes : 2 * kEpiSlabBytes;
  static constexpr int kBarBytes = 1024;
  static constexpr int kFit = (kSmemLimit - kEpiBytes - kBarBytes - 1024) / kStageBytes;
  static constexpr int kStages = kFit < 8 ? kFit : 8;
  static constexpr int kTotal = kStages * kStageBytes + kEpiBytes + kBarBytes + 1024;  // +1024 align slack
  static_assert(kStages == (BN == 64 ? (TMA_EPI ? 6 : 7) : BN == 128 ? 5 : 3), "stage count per BN changed");
  static_assert((kStageBytes % 1024) == 0, "the TMA ring needs 1024-byte aligned boxes");
};

// TMA epilogue of one warpgroup's m64 x BN accumulator tile (rows m_base.., columns n_base..).  `ring` holds the
// warpgroup's kEpiBoxes boxes; `pos` walks it in step with the producer (full / empty barriers, used only when the
// flags read tensors), and `pending` is the slot whose TMA store has not been confirmed to have read it.  Every
// element goes through the same fp32 expressions, in the same order, as epilogue_chunk.
template <int BN>
HCTR_DEVICE void epilogue_tile_tma(const GemmParams& p, const int flags, const float (&acc)[BN / 2],
                                   uint8_t* ring, uint64_t* full, uint64_t* empty, const CUtensorMap* tm_out,
                                   const CUtensorMap* tm_aux, const int m_base, const int n_base, const int wg,
                                   RingPos& pos, int& pending) {
  const int n_in = epi_in_boxes(flags);
  const int nbox = n_in > 0 ? n_in : 1;
  const int slots = kEpiBoxes / nbox;
  const int xl_box = (flags & EPI_CROSS) ? 1 : 0;
  const int mask_box = n_in - 1;
  const bool aux = (flags & EPI_CROSS) && p.aux != nullptr;
  const bool leader = (threadIdx.x & 127) == 0;
  const int lane = threadIdx.x & 31;
  const int r0 = ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2);
  // SWIZZLE_128B: the 16-byte chunk j of box row r sits at chunk j ^ (r % 8); r % 8 == lane / 4 for both rows
  const uint32_t lane_off = static_cast<uint32_t>(r0 * 128 + (lane & 3) * 4);
  const int sw = lane >> 2;
#pragma unroll
  for (int g = 0; g < BN / 64; ++g) {
    const int n0 = n_base + g * 64;
    if (n0 >= p.N) break;
    uint8_t* box = ring + pos.slot * nbox * kEpiBoxBytes;
    float2 bv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + 8 * j + 2 * (lane & 3);
      bv[j] = make_float2(0.f, 0.f);
      if (p.bias != nullptr) {
        if (n + 1 < p.N) bv[j] = __ldg(reinterpret_cast<const float2*>(p.bias + n));
        else if (n < p.N) bv[j].x = __ldg(p.bias + n);
      }
    }
    if (n_in > 0) mbar_wait(&full[pos.slot], pos.phase);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t off = lane_off + h * (8 * 128) + ((j ^ sw) << 4);
        const float* a2 = acc + (8 * g + j) * 4 + 2 * h;
        float v0 = a2[0] * p.alpha, v1 = a2[1] * p.alpha;
        if (p.bias != nullptr) {
          v0 += bv[j].x;
          v1 += bv[j].y;
        }
        if (flags & EPI_CROSS) {
          const uint32_t xa = *reinterpret_cast<const uint32_t*>(box + off);
          const uint32_t xb = *reinterpret_cast<const uint32_t*>(box + kEpiBoxBytes + off);
          if (aux) *reinterpret_cast<uint32_t*>(box + kEpiBoxBytes + off) = pack_bf16x2(v0, v1);
          v0 = bf16_lo(xa) * v0 + bf16_lo(xb);
          v1 = bf16_hi(xa) * v1 + bf16_hi(xb);
        }
        if (flags & EPI_ADD) {
          const uint32_t xb = *reinterpret_cast<const uint32_t*>(box + xl_box * kEpiBoxBytes + off);
          v0 += bf16_lo(xb);
          v1 += bf16_hi(xb);
        }
        if (flags & EPI_MASK) {
          const uint32_t mk = *reinterpret_cast<const uint32_t*>(box + mask_box * kEpiBoxBytes + off);
          if (!(bf16_lo(mk) > 0.f)) v0 = 0.f;
          if (!(bf16_hi(mk) > 0.f)) v1 = 0.f;
        }
        if (flags & EPI_RELU) {
          v0 = fmaxf(v0, 0.f);
          v1 = fmaxf(v1, 0.f);
        }
        if (flags & EPI_SIGMOID) {
          v0 = 1.f / (1.f + __expf(-v0));
          v1 = 1.f / (1.f + __expf(-v1));
        }
        *reinterpret_cast<uint32_t*>(box + off) = pack_bf16x2(v0, v1);
      }
    }
    fence_proxy_async();  // the box writes above become visible to the TMA store
    if (leader) {
      // every earlier store has read its box: the slot of the previous group goes back to the producer, and
      // (output-only flag sets) the next group may write into its slot once past the barrier below
      bulk_wait_read<0>();
      if (pending >= 0 && n_in > 0) mbar_arrive(&empty[pending]);
    }
    named_bar_sync(1 + wg, 128);
    if (leader) {
      tma_store_2d(tm_out, box, n0, m_base);
      if (aux) tma_store_2d(tm_aux, box + kEpiBoxBytes, n0, m_base);
      bulk_commit();
    }
    pending = pos.slot;
    pos.advance(slots);
  }
}

template <int BN, int TA, int TB>
HCTR_DEVICE void wgmma_tile(float (&acc)[BN / 2], uint64_t a, uint64_t b, uint32_t accumulate) {
  if constexpr (BN == 64) wgmma_bf16_n64<TA, TB>(acc, a, b, accumulate);
  else if constexpr (BN == 128) wgmma_bf16_n128<TA, TB>(acc, a, b, accumulate);
  else wgmma_bf16_n256<TA, TB>(acc, a, b, accumulate);
}

// Work item t of the persistent walk is (m-group of MC tiles, n tile, k split), n fastest; the CTAs of a cluster take
// the MC consecutive m tiles of one item.  Both producers and the consumers walk the items through this one mapping:
// if they disagreed, they would wait on each other's barrier phases forever.
struct TileWork {
  int m_blk, n_blk, kb0, kb1;  // k blocks [kb0, kb1)
};
template <int MC>
HCTR_DEVICE TileWork tile_work(const GemmParams& p, const int t, const int m_groups, const int cta_rank) {
  const int split = t / (p.n_tiles * m_groups);
  const int kb0 = split * p.kb_per_split;
  return {((t / p.n_tiles) % m_groups) * MC + cta_rank, t % p.n_tiles, kb0, min(p.k_blocks, kb0 + p.kb_per_split)};
}

// hands an operand stage back to the producer of every CTA of the cluster (each of them multicast into it)
template <int MC>
HCTR_DEVICE void release_stage(uint64_t* empty) {
  if constexpr (MC == 1) mbar_arrive(empty);
  else
    for (int r = 0; r < MC; ++r) mbar_arrive_cluster(empty, r);
}

// MC == 2: thread-block cluster of two CTAs stacked along M that share the B tile -- each CTA loads
// half of it and TMA-multicasts it into both shared memories (halves the L2->SM operand traffic of B).
// TMA_EPI: bf16 output through the TMA epilogue; tmOut / tmAux / tmX0 / tmXl / tmMask are the [64 x 64] box maps of
// the tensors the flags use (the others are not read).
template <int BN, bool A_MN, bool B_MN, int MC, bool TMA_EPI>
__global__ void __launch_bounds__(kNumThreads, 1)
    gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const __grid_constant__ CUtensorMap tmOut, const __grid_constant__ CUtensorMap tmAux,
                   const __grid_constant__ CUtensorMap tmX0, const __grid_constant__ CUtensorMap tmXl,
                   const __grid_constant__ CUtensorMap tmMask, const GemmParams p) {
  using L = SmemLayout<BN, TMA_EPI>;
  constexpr int kStages = L::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * L::kABytes;
  uint8_t* epi = smem + kStages * L::kStageBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * L::kStageBytes + L::kEpiBytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + kStages;
  // TMA epilogue ring barriers, kEpiBoxes per consumer warpgroup (one per slot at most)
  uint64_t* epi_full = bars + 2 * kStages;
  uint64_t* epi_empty = epi_full + 2 * kEpiBoxes;

  const int wg = threadIdx.x >> 7;
  const int warp_idx = threadIdx.x >> 5;
  const int m_groups = (p.m_tiles + MC - 1) / MC;
  const int total_tiles = m_groups * p.n_tiles * p.splits;
  const int cta_rank = (MC > 1) ? static_cast<int>(cluster_ctarank()) : 0;
  const int cluster_id = (MC > 1) ? (blockIdx.x / MC) : blockIdx.x;
  const int num_clusters = (MC > 1) ? (gridDim.x / MC) : gridDim.x;

  if (warp_idx == 0 && elect_one()) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (TMA_EPI) tma_prefetch_desc(&tmOut);
  }
  if (warp_idx == 1 && elect_one()) {
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8 * MC);  // every consumer warp of every CTA of the cluster
    }
    if constexpr (TMA_EPI) {
      for (int i = 0; i < 2 * kEpiBoxes; ++i) {
        mbar_init(&epi_full[i], 1);
        mbar_init(&epi_empty[i], 1);  // the store-issuing thread of the warpgroup
      }
    }
    fence_barrier_init();
  }
  __syncthreads();
  if constexpr (MC > 1) cluster_sync_all();  // peers' barriers are initialised before any remote arrive

  if (wg == 0) {
    // ===================== TMA producer =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp_idx == 0 && elect_one()) {
      RingPos s;
      for (int t = cluster_id; t < total_tiles; t += num_clusters) {
        const TileWork w = tile_work<MC>(p, t, m_groups, cta_rank);
        const int m0 = w.m_blk * BLOCK_M, n0 = w.n_blk * BN;
        for (int kb = w.kb0; kb < w.kb1; ++kb) {
          mbar_wait(&empty_bar[s.slot], s.phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[s.slot], L::kStageBytes);
          uint8_t* sa = smem_a + s.slot * L::kABytes;
          uint8_t* sb = smem_b + s.slot * L::kBBytes;
          const int k0 = kb * BLOCK_K;
          if constexpr (A_MN) {
#pragma unroll
            for (int c = 0; c < BLOCK_M / 64; ++c)
              tma_load_2d(sa + c * (BLOCK_K * 128), &tmA, &full_bar[s.slot], m0 + c * 64, k0);
          } else {
            tma_load_2d(sa, &tmA, &full_bar[s.slot], k0, m0);
          }
          if constexpr (MC == 1) {
            if constexpr (B_MN) {
#pragma unroll
              for (int c = 0; c < BN / 64; ++c)
                tma_load_2d(sb + c * (BLOCK_K * 128), &tmB, &full_bar[s.slot], n0 + c * 64, k0);
            } else {
              tma_load_2d(sb, &tmB, &full_bar[s.slot], k0, n0);
            }
          } else {
            // this CTA fetches its 1/MC share of the B tile and multicasts it to the whole cluster
            constexpr uint16_t kMask = (1u << MC) - 1;
            if constexpr (B_MN) {
              constexpr int kChunks = BN / 64 / MC;
              if constexpr (kChunks > 0) {
#pragma unroll
                for (int c = 0; c < kChunks; ++c) {
                  const int cc = cta_rank * kChunks + c;
                  tma_load_2d_mc(sb + cc * (BLOCK_K * 128), &tmB, &full_bar[s.slot], n0 + cc * 64, k0, kMask);
                }
              } else if (cta_rank == 0) {  // BN == 64: one chunk, fetched by the first CTA
                tma_load_2d_mc(sb, &tmB, &full_bar[s.slot], n0, k0, kMask);
              }
            } else {
              constexpr int kRowsPer = BN / MC;
              tma_load_2d_mc(sb + cta_rank * (kRowsPer * 128), &tmB, &full_bar[s.slot], k0,
                             n0 + cta_rank * kRowsPer, kMask);
            }
          }
          s.advance(kStages);
        }
      }
    } else if (TMA_EPI && warp_idx == 1 && epi_in_boxes(p.flags) > 0 && elect_one()) {
      // epilogue operands: the x0 / xl / mask boxes of every 64-column group of this CTA's rows, in the order
      // the consumers walk them; skipped where the group or the warpgroup's rows lie wholly outside the output
      const int flags = p.flags;
      const int n_in = epi_in_boxes(flags);
      const int slots = kEpiBoxes / n_in;
      if (flags & EPI_CROSS) tma_prefetch_desc(&tmX0);
      if (flags & (EPI_CROSS | EPI_ADD)) tma_prefetch_desc(&tmXl);
      if (flags & EPI_MASK) tma_prefetch_desc(&tmMask);
      RingPos pos[2];  // one ring per consumer warpgroup
      for (int t = cluster_id; t < total_tiles; t += num_clusters) {
        const TileWork w = tile_work<MC>(p, t, m_groups, cta_rank);
        for (int g = 0; g < BN / 64; ++g) {
          const int n0 = w.n_blk * BN + g * 64;
          if (n0 >= p.N) break;
#pragma unroll
          for (int cw = 0; cw < 2; ++cw) {
            const int m0 = w.m_blk * BLOCK_M + cw * 64;
            if (m0 >= p.M) continue;
            const int s = cw * kEpiBoxes + pos[cw].slot;
            mbar_wait(&epi_empty[s], pos[cw].phase ^ 1);
            mbar_arrive_expect_tx(&epi_full[s], n_in * kEpiBoxBytes);
            uint8_t* box = epi + (cw * kEpiBoxes + pos[cw].slot * n_in) * kEpiBoxBytes;
            if (flags & EPI_CROSS) {
              tma_load_2d(box, &tmX0, &epi_full[s], n0, m0);
              tma_load_2d(box + kEpiBoxBytes, &tmXl, &epi_full[s], n0, m0);
            } else if (flags & EPI_ADD) {
              tma_load_2d(box, &tmXl, &epi_full[s], n0, m0);
            }
            if (flags & EPI_MASK) tma_load_2d(box + (n_in - 1) * kEpiBoxBytes, &tmMask, &epi_full[s], n0, m0);
            pos[cw].advance(slots);
          }
        }
      }
    }
  } else {
    // ===================== wgmma consumers + epilogue (64 rows each) =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = wg - 1;                       // 0 / 1: rows [64 cw, 64 cw + 64) of the tile
    const int lane = threadIdx.x & 31;
    uint32_t* slab = reinterpret_cast<uint32_t*>(epi + cw * kEpiSlabBytes);
    uint8_t* ring = epi + cw * kEpiBoxes * kEpiBoxBytes;
    const int flags = p.flags;
    RingPos s, epi_pos;
    int epi_pending = -1;
    float acc[BN / 2];
    for (int t = cluster_id; t < total_tiles; t += num_clusters) {
      const TileWork w = tile_work<MC>(p, t, m_groups, cta_rank);
      int prev = -1;
      for (int kb = w.kb0; kb < w.kb1; ++kb) {
        mbar_wait(&full_bar[s.slot], s.phase);
        const uint32_t a_addr = smem_u32(smem_a + s.slot * L::kABytes) + cw * (64 * 128);
        const uint32_t b_addr = smem_u32(smem_b + s.slot * L::kBBytes);
        // K-major SW128 : 8-row atoms of 1024 B ; MN-major SW128: 64-wide chunks BLOCK_K*128 B
        // apart (LBO), 8-k-row groups 1024 B apart (SBO)
        const uint64_t a_desc = A_MN ? make_smem_desc_sw128(a_addr, BLOCK_K * 128, 1024)
                                     : make_smem_desc_sw128(a_addr, 16, 1024);
        const uint64_t b_desc = B_MN ? make_smem_desc_sw128(b_addr, BLOCK_K * 128, 1024)
                                     : make_smem_desc_sw128(b_addr, 16, 1024);
        constexpr uint32_t a_step = A_MN ? (WG_K * 128) >> 4 : (WG_K * 2) >> 4;
        constexpr uint32_t b_step = B_MN ? (WG_K * 128) >> 4 : (WG_K * 2) >> 4;
        wgmma_fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WG_K; ++k)
          wgmma_tile<BN, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, a_desc + static_cast<uint64_t>(k * a_step),
                                                      b_desc + static_cast<uint64_t>(k * b_step),
                                                      (kb > w.kb0 || k > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_fence_regs(acc);
        if (TMA_EPI && epi_pending >= 0) {
          // the previous tile's last TMA store, deferred to here so that it overlaps this tile's first wgmma
          if ((threadIdx.x & 127) == 0) {
            bulk_wait_read<0>();
            if (epi_in_boxes(flags) > 0) mbar_arrive(&epi_empty[cw * kEpiBoxes + epi_pending]);
          }
          epi_pending = -1;
        }
        if (prev >= 0) {
          wgmma_wait<1>();  // the previous k block's wgmma has finished reading its slot
          if (lane == 0) release_stage<MC>(&empty_bar[prev]);
        }
        prev = s.slot;
        s.advance(kStages);
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev >= 0 && lane == 0) release_stage<MC>(&empty_bar[prev]);
      const int m_base = w.m_blk * BLOCK_M + cw * 64;
      if constexpr (TMA_EPI) {
        if (m_base < p.M)
          epilogue_tile_tma<BN>(p, flags, acc, ring, epi_full + cw * kEpiBoxes, epi_empty + cw * kEpiBoxes,
                                &tmOut, &tmAux, m_base, w.n_blk * BN, cw, epi_pos, epi_pending);
      } else {
        epilogue_tile_wg<BN>(p, flags, acc, slab, m_base, w.n_blk * BN, cw);
      }
    }
    if (TMA_EPI && (threadIdx.x & 127) == 0) bulk_wait<0>();  // the stores are complete before the CTA exits
  }

  __syncthreads();
  if constexpr (MC > 1) cluster_sync_all();  // no CTA may exit while a peer can still multicast into it
}

// ------------------------------------------------------------------ host side
// 2-D bf16 row-major tensor [outer, inner] with leading dimension ld (elements)
static int make_tmap_bf16(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer,
                          uint64_t ld, uint32_t box_inner, uint32_t box_outer) {
  PFN_encodeTiled enc = get_encode();
  if (enc == nullptr) return -1;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -2;
}

// [64 x 64] boxes of the TMA epilogue's bf16 tensors; only the maps the flags use are encoded
struct EpiMaps {
  CUtensorMap out, aux, x0, xl, mask;
};

// one launcher per (BN, MC, TMA_EPI) over the four operand layouts (A_MN, B_MN)
template <int BN, int MC, bool TMA_EPI>
static int launch(const int a_mn, const int b_mn, const CUtensorMap& ta, const CUtensorMap& tb, const EpiMaps& em,
                  const GemmParams& p, cudaStream_t stream) {
  using L = SmemLayout<BN, TMA_EPI>;
  decltype(&gemm_tc_kernel<BN, false, false, MC, TMA_EPI>) const kernels[4] = {
      gemm_tc_kernel<BN, false, false, MC, TMA_EPI>, gemm_tc_kernel<BN, false, true, MC, TMA_EPI>,
      gemm_tc_kernel<BN, true, false, MC, TMA_EPI>, gemm_tc_kernel<BN, true, true, MC, TMA_EPI>};
  const int layout = 2 * (a_mn != 0) + (b_mn != 0);
  static bool attr_set[4] = {};
  auto kern = kernels[layout];
  if (!attr_set[layout]) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kTotal) !=
        cudaSuccess)
      return -3;
    attr_set[layout] = true;
  }
  const int m_groups = (p.m_tiles + MC - 1) / MC;
  const int total = m_groups * p.n_tiles * p.splits;       // cluster work items
  int clusters = num_sms() / MC;
  if (total < clusters) clusters = total;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(clusters * MC);
  cfg.blockDim = dim3(kNumThreads);
  cfg.dynamicSmemBytes = L::kTotal;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = MC;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (cudaLaunchKernelEx(&cfg, kern, ta, tb, em.out, em.aux, em.x0, em.xl, em.mask, p) != cudaSuccess)
    return -4;
  return cudaGetLastError() == cudaSuccess ? 0 : -4;
}

template <bool TMA_EPI>
static int dispatch(int BN, int mc, int a_mn, int b_mn, const CUtensorMap& ta, const CUtensorMap& tb,
                    const EpiMaps& em, const GemmParams& p, cudaStream_t stream) {
  if (mc == 2) {
    if (BN == 256) return launch<256, 2, TMA_EPI>(a_mn, b_mn, ta, tb, em, p, stream);
    if (BN == 64) return launch<64, 2, TMA_EPI>(a_mn, b_mn, ta, tb, em, p, stream);
    return launch<128, 2, TMA_EPI>(a_mn, b_mn, ta, tb, em, p, stream);
  }
  if (BN == 256) return launch<256, 1, TMA_EPI>(a_mn, b_mn, ta, tb, em, p, stream);
  if (BN == 64) return launch<64, 1, TMA_EPI>(a_mn, b_mn, ta, tb, em, p, stream);
  return launch<128, 1, TMA_EPI>(a_mn, b_mn, ta, tb, em, p, stream);
}

// The TMA epilogue takes bf16 outputs whose slot holds at most two boxes, and whose epilogue tensors TMA can address
// (16-byte bases and pitches) and bias, if any, is 8-byte aligned (float2 loads); it encodes their maps into em.
// Everything else runs the slab epilogue.
static bool tma_epilogue_maps(EpiMaps* em, int M, int N, int flags, const void* out, long long ldo, const void* aux,
                              long long ldaux, const void* x0, const void* xl, long long ldx, const void* mask,
                              long long ldmask, const float* bias) {
  if ((flags & (EPI_OUT_F32 | EPI_ATOMIC)) || epi_in_boxes(flags) > 2) return false;
  if (bias != nullptr && reinterpret_cast<uintptr_t>(bias) % 8) return false;
  auto map = [&](CUtensorMap* m, const void* ptr, long long ld) {
    return ptr != nullptr && reinterpret_cast<uintptr_t>(ptr) % 16 == 0 && ld >= N &&
           make_tmap_bf16(m, ptr, N, M, ld, 64, 64) == 0;
  };
  memset(em, 0, sizeof(*em));
  if (!map(&em->out, out, ldo)) return false;
  if ((flags & EPI_CROSS) && aux != nullptr && !map(&em->aux, aux, ldaux)) return false;
  if ((flags & EPI_CROSS) && !map(&em->x0, x0, ldx)) return false;
  if ((flags & (EPI_CROSS | EPI_ADD)) && !map(&em->xl, xl, ldx)) return false;
  if ((flags & EPI_MASK) && !map(&em->mask, mask, ldmask)) return false;
  return true;
}

}  // namespace hctr

using namespace hctr;

// A: a_mn ? [K, M] row-major (lda) : [M, K] row-major (lda)
// B: b_mn ? [K, N] row-major (ldb) : [N, K] row-major (ldb)
// out: [M, N] row-major (ldo) bf16 (default) or fp32 (EPI_OUT_F32 | EPI_ATOMIC)
// block_n: BN in {64, 128, 256} (one CTA per tile) or 1000 + BN (2-CTA cluster sharing the B tile); other codes
// >= 1000 are rejected (rc -11)
extern "C" int hctr_gemm_bf16(const void* A, const void* B, void* out, int M, int N, int K,
                              long long lda, long long ldb, long long ldo, int a_mn, int b_mn,
                              const float* bias, const void* mask, long long ldmask,
                              const void* x0, const void* xl, long long ldx, void* aux,
                              long long ldaux, float alpha, int flags, int splits, int block_n,
                              void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if (block_n >= 2000) return -11;
  const int mc = (block_n >= 1000) ? 2 : 1;
  block_n %= 1000;
  const int BN = (block_n == 256 || block_n == 64) ? block_n : 128;
  GemmParams p;
  p.M = M; p.N = N; p.K = K;
  p.m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
  p.n_tiles = (N + BN - 1) / BN;
  p.k_blocks = (K + BLOCK_K - 1) / BLOCK_K;
  if (splits < 1) splits = 1;
  if (splits > p.k_blocks) splits = p.k_blocks;
  p.kb_per_split = (p.k_blocks + splits - 1) / splits;
  p.splits = (p.k_blocks + p.kb_per_split - 1) / p.kb_per_split;
  if (p.splits > 1 && !(flags & EPI_ATOMIC)) return -10;
  p.out = out; p.ldo = ldo; p.aux = aux; p.ldaux = ldaux; p.bias = bias;
  p.mask = reinterpret_cast<const __nv_bfloat16*>(mask); p.ldmask = ldmask;
  p.x0 = reinterpret_cast<const __nv_bfloat16*>(x0);
  p.xl = reinterpret_cast<const __nv_bfloat16*>(xl); p.ldx = ldx;
  p.alpha = alpha; p.flags = flags;

  CUtensorMap ta, tb;
  int rc;
  if (a_mn) rc = make_tmap_bf16(&ta, A, M, K, lda, 64, BLOCK_K);
  else      rc = make_tmap_bf16(&ta, A, K, M, lda, BLOCK_K, BLOCK_M);
  if (rc) return rc;
  if (b_mn) rc = make_tmap_bf16(&tb, B, N, K, ldb, 64, BLOCK_K);
  else      rc = make_tmap_bf16(&tb, B, K, N, ldb, BLOCK_K, BN / mc);
  if (rc) return rc - 10;

  EpiMaps em;
  if (tma_epilogue_maps(&em, M, N, flags, out, ldo, aux, ldaux, x0, xl, ldx, mask, ldmask, bias))
    return dispatch<true>(BN, mc, a_mn, b_mn, ta, tb, em, p, stream);
  return dispatch<false>(BN, mc, a_mn, b_mn, ta, tb, em, p, stream);
}
