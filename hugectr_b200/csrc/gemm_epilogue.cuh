// Shared declarations, the tensor-map encoder, the pipeline-ring position and the fused epilogue of the wgmma GEMM
// kernels (gemm_tc.cu, gemm_mxfp8.cu).
#pragma once
#include "ptx.cuh"

namespace hctr {

enum EpiFlags : int {
  EPI_RELU = 1,
  EPI_OUT_F32 = 2,
  EPI_ATOMIC = 4,   // fp32 red.add into out (split-K / beta=1)
  EPI_CROSS = 16,   // out = x0 * (acc + bias) + xl ; aux (optional) = acc + bias
  EPI_MASK = 32,    // out = acc * (mask > 0)
  EPI_SIGMOID = 64, // out = sigmoid(acc + bias)
  EPI_ADD = 128,    // out = acc + xl (bf16)   (residual / gradient accumulation)
};

struct GemmParams {
  int M, N, K;
  int m_tiles, n_tiles, splits, kb_per_split, k_blocks;
  void* out;
  long long ldo;
  void* aux;
  long long ldaux;
  const float* bias;
  const __nv_bfloat16* mask;
  long long ldmask;
  const __nv_bfloat16* x0;
  const __nv_bfloat16* xl;
  long long ldx;
  float alpha;
  int flags;
  // Unused.  Keeps the struct at its earlier size: without these 16 bytes nvcc 12.9 duplicates the TMA epilogue
  // loop of gemm_tc_kernel, and its bf16-output GEMMs ran 10-17% slower on an H100 80GB HBM3 (700 W).
  long long reserved[2];
};

// cuTensorMapEncodeTiled, looked up once through the runtime's driver entry point (nullptr if the driver lacks it)
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) !=
            cudaSuccess ||
        ptr == nullptr)
      return nullptr;
    fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  }
  return fn;
}

// The dynamic shared-memory base rounded up to 1024 bytes (SWIZZLE_128B tiles).  It is an offset from `smem_raw`
// rather than an integer cast, so that the compiler keeps every derived pointer in the shared window and addresses
// it with 32-bit LDS / STS instead of 64-bit generic loads and stores.
HCTR_DEVICE uint8_t* smem_align1024(uint8_t* smem_raw) {
  return smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
}

// Position in a ring of mbarrier-guarded slots: the slot, and the parity of the current pass over the ring.
struct RingPos {
  int slot = 0;
  uint32_t phase = 0;
  HCTR_DEVICE void advance(const int slots) {
    if (++slot == slots) {
      slot = 0;
      phase ^= 1;
    }
  }
};


// One thread owns row `m`, columns [n0, n0+32) of the tile: r[] are the fp32 accumulators (bit patterns)
// read back from the kernel's staging slab.
HCTR_DEVICE void epilogue_chunk(const GemmParams& p, const int flags, const int m, const bool row_ok,
                                const int n0, const uint32_t (&r)[32]) {
        if (n0 >= p.N) return;  // warp-uniform
  const int nvalid = min(32, p.N - n0);
  float v[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(r[j]) * p.alpha;
  if (p.bias != nullptr) {
    if (nvalid == 32) {
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + n0 + j));
        v[j] += b.x; v[j + 1] += b.y; v[j + 2] += b.z; v[j + 3] += b.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j < nvalid) v[j] += __ldg(p.bias + n0 + j);
    }
  }
  if (!row_ok) return;
  if (flags & EPI_CROSS) {
    // aux = acc + bias ; out = x0 * aux + xl
    const __nv_bfloat16* px0 = p.x0 + static_cast<long long>(m) * p.ldx + n0;
    const __nv_bfloat16* pxl = p.xl + static_cast<long long>(m) * p.ldx + n0;
    if (p.aux != nullptr && nvalid == 32) {
      uint4* pa = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.aux) +
                                           static_cast<long long>(m) * p.ldaux + n0);
#pragma unroll
      for (int j = 0; j < 4; ++j)
        pa[j] = make_uint4(pack_bf16x2(v[8 * j], v[8 * j + 1]),
                           pack_bf16x2(v[8 * j + 2], v[8 * j + 3]),
                           pack_bf16x2(v[8 * j + 4], v[8 * j + 5]),
                           pack_bf16x2(v[8 * j + 6], v[8 * j + 7]));
    } else if (p.aux != nullptr) {
      __nv_bfloat16* pa = reinterpret_cast<__nv_bfloat16*>(p.aux) +
                          static_cast<long long>(m) * p.ldaux + n0;
      _Pragma("unroll") for (int j = 0; j < 32; ++j) if (j < nvalid) pa[j] = __float2bfloat16(v[j]);
    }
    if (nvalid == 32) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(px0) + j);
        const uint4 b = __ldg(reinterpret_cast<const uint4*>(pxl) + j);
        const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
        const uint32_t bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          v[8 * j + 2 * q] = bf16_lo(aw[q]) * v[8 * j + 2 * q] + bf16_lo(bw[q]);
          v[8 * j + 2 * q + 1] = bf16_hi(aw[q]) * v[8 * j + 2 * q + 1] + bf16_hi(bw[q]);
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j < nvalid) v[j] = __bfloat162float(px0[j]) * v[j] + __bfloat162float(pxl[j]);
    }
  }
  if (flags & EPI_ADD) {
    const __nv_bfloat16* pxl = p.xl + static_cast<long long>(m) * p.ldx + n0;
    if (nvalid == 32) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint4 b = __ldg(reinterpret_cast<const uint4*>(pxl) + j);
        const uint32_t bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          v[8 * j + 2 * q] += bf16_lo(bw[q]);
          v[8 * j + 2 * q + 1] += bf16_hi(bw[q]);
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j < nvalid) v[j] += __bfloat162float(pxl[j]);
    }
  }
  if (flags & EPI_MASK) {
    const __nv_bfloat16* pm = p.mask + static_cast<long long>(m) * p.ldmask + n0;
    if (nvalid == 32) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(pm) + j);
        const uint32_t aw[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          if (!(bf16_lo(aw[q]) > 0.f)) v[8 * j + 2 * q] = 0.f;
          if (!(bf16_hi(aw[q]) > 0.f)) v[8 * j + 2 * q + 1] = 0.f;
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j)
        if (j < nvalid && !(__bfloat162float(pm[j]) > 0.f)) v[j] = 0.f;
    }
  }
  if (flags & EPI_RELU) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
  }
  if (flags & EPI_SIGMOID) {
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = 1.f / (1.f + __expf(-v[j]));
  }
  if (flags & (EPI_OUT_F32 | EPI_ATOMIC)) {
    float* po = reinterpret_cast<float*>(p.out) + static_cast<long long>(m) * p.ldo + n0;
    if (flags & EPI_ATOMIC) {
      if (nvalid == 32) {
#pragma unroll
        for (int j = 0; j < 32; j += 4)
          asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(po + j),
                       "f"(v[j]), "f"(v[j + 1]), "f"(v[j + 2]), "f"(v[j + 3])
                       : "memory");
      } else {
        _Pragma("unroll") for (int j = 0; j < 32; ++j) if (j < nvalid) atomicAdd(po + j, v[j]);
      }
    } else if (nvalid == 32) {
#pragma unroll
      for (int j = 0; j < 32; j += 4)
        *reinterpret_cast<float4*>(po + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
    } else {
      _Pragma("unroll") for (int j = 0; j < 32; ++j) if (j < nvalid) po[j] = v[j];
    }
  } else {
    __nv_bfloat16* po =
        reinterpret_cast<__nv_bfloat16*>(p.out) + static_cast<long long>(m) * p.ldo + n0;
    if (nvalid == 32) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        reinterpret_cast<uint4*>(po)[j] =
            make_uint4(pack_bf16x2(v[8 * j], v[8 * j + 1]),
                       pack_bf16x2(v[8 * j + 2], v[8 * j + 3]),
                       pack_bf16x2(v[8 * j + 4], v[8 * j + 5]),
                       pack_bf16x2(v[8 * j + 6], v[8 * j + 7]));
    } else {
      _Pragma("unroll") for (int j = 0; j < 32; ++j) if (j < nvalid) po[j] = __float2bfloat16(v[j]);
    }
  }
}


// ---------------------------------------------------------------------------------------------
// Epilogue of one warpgroup's m64 x BN wgmma accumulator tile (layout in wgmma.cuh): 64-column groups go
// through a [64 x kStagePitch] fp32 staging slab in shared memory so that every thread then owns one row
// x 32 consecutive columns for epilogue_chunk.  `slab` is private to the warpgroup (named barrier 1 + wg).
constexpr int kStagePitch = 64 + 4;  // fp32 words per staged row (+4: conflict-free 16-byte reads)
constexpr int kEpiSlabBytes = 64 * kStagePitch * 4;

HCTR_DEVICE void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

template <int BN>
HCTR_DEVICE void epilogue_tile_wg(const GemmParams& p, const int flags, const float (&acc)[BN / 2], uint32_t* slab,
                                  const int m_base, const int n_base, const int wg) {
  const int w4 = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int erow = (w4 & 1) * 32 + lane;
  const int m = m_base + erow;
  const bool row_ok = m < p.M;
  const int r0 = w4 * 16 + (lane >> 2);
  const int c = w4 >> 1;
#pragma unroll
  for (int g = 0; g < BN / 64; ++g) {
    named_bar_sync(1 + wg, 128);  // the slab's previous readers are done
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = 8 * j + 2 * (lane & 3);
      const float* a4 = acc + (8 * g + j) * 4;
      *reinterpret_cast<uint2*>(slab + r0 * kStagePitch + col) =
          make_uint2(__float_as_uint(a4[0]), __float_as_uint(a4[1]));
      *reinterpret_cast<uint2*>(slab + (r0 + 8) * kStagePitch + col) =
          make_uint2(__float_as_uint(a4[2]), __float_as_uint(a4[3]));
    }
    named_bar_sync(1 + wg, 128);
    uint32_t r[32];
    const uint4* src = reinterpret_cast<const uint4*>(slab + erow * kStagePitch + c * 32);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const uint4 v = src[q];
      r[4 * q] = v.x; r[4 * q + 1] = v.y; r[4 * q + 2] = v.z; r[4 * q + 3] = v.w;
    }
    epilogue_chunk(p, flags, m, row_ok, n_base + g * 64 + c * 32, r);
  }
}

}  // namespace hctr
