// D1-fp8: block-scaled (MX) fp8 GEMM on Hopper tensor cores.
//   out[M, N] (bf16 / fp32) = epilogue( sum_k  (A_q[m, k] * 2^(SFA[m, k/32] - 127)) * (B_q[n, k] * 2^(SFB[n, k/32] - 127)) )
// A_q [M, K], B_q [N, K]: e4m3, K-major.  SFA / SFB: one UE8M0 scale per 32 consecutive K elements (OCP MX
// format).  Hopper's fp8 wgmma has no block scaling, and one m64n128k32 wgmma covers exactly one 32-wide scale
// slice, so every slice is accumulated into a temporary register tile and promoted into the fp32 accumulator
// with the product of its row and column scales (powers of two: the promotion is exact up to fp32 rounding).
// Scale range: the product s0 * sc = 2^(ea + eb - 254) of scale bytes ea, eb is a fast-math (flush-to-zero) fp32
// multiply, so a slice is promoted exactly only while ea + eb - 254 lies in [-126, 127] and neither byte is 0.  A
// slice with ea + eb < 128, or a scale byte of 0 (read as zero, not 2^-127), adds nothing, even where its products
// times the scales would be normal fp32 numbers; above the range the scale product is +inf (and a zero partial sum
// times it NaN).  Quantised activations and weights of a trained model sit far inside the range
// (tests/test_mxfp8_fp64_gpu.py pins its ends).
// CTA (one 128 x 128 output tile) = three warpgroups:
//   warpgroup 0   TMA producer: A / B tiles (128 rows x 128 bytes, SWIZZLE_128B) + the 512-byte scale blocks of
//                 the k-block (1-D bulk copies) into a ring of stages, completion on the stage's mbarrier
//   warpgroups 1-2  64 rows each: 4 slices per k-block (wgmma -> wait -> scaled promotion), then the fused
//                 epilogue (bias / ReLU / ...) through the shared staging slab
// Scale layout in global memory: a k-block's scales are ONE contiguous 512-byte block per 128 rows:
//   block (row / 128, k / 128), byte offset (row % 32) * 16 + ((row % 128) / 32) * 4 + (k % 128) / 32
// The quantiser (mx_quantize_kernel) writes exactly this; it is the reference's cublasLt path replaced
// (HugeCTR/src/layers/functors/fused_gemm_functors.cu:21-289 has no fp8 at all).
#include <cuda_fp8.h>

#include "gemm_epilogue.cuh"

namespace hctr {

constexpr int MX_BM = 128, MX_BN = 128, MX_BK = 128, MX_STAGES = 4, MX_THREADS = 384;
constexpr int MX_TILE_BYTES = MX_BM * MX_BK;          // 16 KB (fp8)
constexpr int MX_SF_BYTES = 512;
constexpr int MX_SMEM = MX_STAGES * (2 * MX_TILE_BYTES + 2 * MX_SF_BYTES) + 2 * kEpiSlabBytes + 1024 + 1024;

HCTR_DEVICE void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// UE8M0 byte -> 2^(e - 127) (e = 0, i.e. 2^-127, flushes to zero)
HCTR_DEVICE float ue8m0_to_float(uint32_t e) { return __uint_as_float(e << 23); }

__global__ void __launch_bounds__(MX_THREADS, 1)
    gemm_mxfp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      const uint8_t* __restrict__ sfa, const uint8_t* __restrict__ sfb, const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align1024(smem_raw);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + MX_STAGES * MX_TILE_BYTES;
  uint8_t* smem_sfa = smem + 2 * MX_STAGES * MX_TILE_BYTES;
  uint8_t* smem_sfb = smem_sfa + MX_STAGES * MX_SF_BYTES;
  uint32_t* epi = reinterpret_cast<uint32_t*>(smem_sfb + MX_STAGES * MX_SF_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(epi) + 2 * kEpiSlabBytes);
  uint64_t* empty_bar = full_bar + MX_STAGES;

  const int wg = threadIdx.x >> 7, warp_idx = threadIdx.x >> 5;
  const int n_blk = blockIdx.x, m_blk = blockIdx.y;
  const int k_blocks = p.k_blocks;

  if (warp_idx == 0 && elect_one()) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  if (warp_idx == 1 && elect_one()) {
    for (int i = 0; i < MX_STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);   // every consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp_idx == 0 && elect_one()) {
      RingPos s;
      for (int kb = 0; kb < k_blocks; ++kb) {
        mbar_wait(&empty_bar[s.slot], s.phase ^ 1);
        mbar_arrive_expect_tx(&full_bar[s.slot], 2 * MX_TILE_BYTES + 2 * MX_SF_BYTES);
        tma_load_2d(smem_a + s.slot * MX_TILE_BYTES, &tmA, &full_bar[s.slot], kb * MX_BK, m_blk * MX_BM);
        tma_load_2d(smem_b + s.slot * MX_TILE_BYTES, &tmB, &full_bar[s.slot], kb * MX_BK, n_blk * MX_BN);
        bulk_load_1d(smem_sfa + s.slot * MX_SF_BYTES,
                     sfa + (static_cast<long long>(m_blk) * k_blocks + kb) * MX_SF_BYTES, MX_SF_BYTES, &full_bar[s.slot]);
        bulk_load_1d(smem_sfb + s.slot * MX_SF_BYTES,
                     sfb + (static_cast<long long>(n_blk) * k_blocks + kb) * MX_SF_BYTES, MX_SF_BYTES, &full_bar[s.slot]);
        s.advance(MX_STAGES);
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = wg - 1;
    const int w4 = warp_idx & 3, lane = threadIdx.x & 31;
    const int row0 = cw * 64 + w4 * 16 + (lane >> 2);   // tile rows row0 and row0 + 8
    float acc[64], part[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    RingPos s;
    for (int kb = 0; kb < k_blocks; ++kb) {
      mbar_wait(&full_bar[s.slot], s.phase);
      const uint64_t a_desc = make_smem_desc_sw128(smem_u32(smem_a + s.slot * MX_TILE_BYTES) + cw * (64 * 128), 16, 1024);
      const uint64_t b_desc = make_smem_desc_sw128(smem_u32(smem_b + s.slot * MX_TILE_BYTES), 16, 1024);
      const uint8_t* sa = smem_sfa + s.slot * MX_SF_BYTES;
      const uint8_t* sb = smem_sfb + s.slot * MX_SF_BYTES;
#pragma unroll
      for (int k = 0; k < MX_BK / 32; ++k) {
        wgmma_fence_regs(part);
        wgmma_fence();
        wgmma_e4m3_n128(part, a_desc + static_cast<uint64_t>(k * 2), b_desc + static_cast<uint64_t>(k * 2), 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(part);
        const float s0 = ue8m0_to_float(sa[(row0 & 31) * 16 + (row0 >> 5) * 4 + k]);
        const float s1 = ue8m0_to_float(sa[((row0 + 8) & 31) * 16 + ((row0 + 8) >> 5) * 4 + k]);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * j + 2 * (lane & 3) + e;
            const float sc = ue8m0_to_float(sb[(col & 31) * 16 + (col >> 5) * 4 + k]);
            acc[4 * j + e] = fmaf(part[4 * j + e], s0 * sc, acc[4 * j + e]);
            acc[4 * j + 2 + e] = fmaf(part[4 * j + 2 + e], s1 * sc, acc[4 * j + 2 + e]);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[s.slot]);
      s.advance(MX_STAGES);
    }
    epilogue_tile_wg<MX_BN>(p, p.flags, acc, epi + cw * (kEpiSlabBytes / 4), m_blk * MX_BM + cw * 64,
                            n_blk * MX_BN, cw);
  }
}

// ------------------------------------------------------------------ MX quantiser
// x [rows, cols] (bf16 / fp32, row-major, cols % 128 == 0) -> q [rows_pad, cols] e4m3 + scales in the block layout
// above (rows_pad = rows rounded up to 128; padding rows are zero with scale 2^-127).  One thread per 32-wide block.
template <typename T>
__global__ void __launch_bounds__(256)
    mx_quantize_kernel(const T* __restrict__ x, long long ldx, uint8_t* __restrict__ q, uint8_t* __restrict__ sf,
                       int rows, int rows_pad, int cols, int transposed) {
  const int blocks_per_row = cols / 32;
  const long long total = static_cast<long long>(rows_pad) * blocks_per_row;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / blocks_per_row);
    const int cb = static_cast<int>(i - static_cast<long long>(r) * blocks_per_row);
    float v[32];
    float amax = 0.f;
    if (r < rows) {
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        v[j] = static_cast<float>(transposed ? x[static_cast<long long>(cb * 32 + j) * ldx + r]
                                             : x[static_cast<long long>(r) * ldx + cb * 32 + j]);
        amax = fmaxf(amax, fabsf(v[j]));
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = 0.f;
    }
    const int e = e4m3_scale_exp(amax);
    uint32_t w[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const __nv_fp8x2_storage_t lo = __nv_cvt_float2_to_fp8x2(
          make_float2(e4m3_scale_down(v[4 * j], e), e4m3_scale_down(v[4 * j + 1], e)), __NV_SATFINITE, __NV_E4M3);
      const __nv_fp8x2_storage_t hi = __nv_cvt_float2_to_fp8x2(
          make_float2(e4m3_scale_down(v[4 * j + 2], e), e4m3_scale_down(v[4 * j + 3], e)), __NV_SATFINITE, __NV_E4M3);
      w[j] = static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
    }
    uint4* dst = reinterpret_cast<uint4*>(q + static_cast<long long>(r) * cols + cb * 32);
    dst[0] = make_uint4(w[0], w[1], w[2], w[3]);
    dst[1] = make_uint4(w[4], w[5], w[6], w[7]);
    const int kb = cb >> 2, k = cb & 3;
    const long long blk = static_cast<long long>(r >> 7) * (cols / 128) + kb;
    sf[blk * 512 + (r & 31) * 16 + ((r & 127) >> 5) * 4 + k] = static_cast<uint8_t>(e + 127);
  }
}

static int make_tmap_u8(CUtensorMap* m, const void* ptr, uint64_t inner, uint64_t outer, uint64_t ld_bytes) {
  PFN_encodeTiled enc = get_encode();
  if (enc == nullptr) return -1;
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {ld_bytes};
  cuuint32_t box[2] = {128, 128};
  cuuint32_t estr[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS ? 0 : -2;
}

}  // namespace hctr

using namespace hctr;

// x: bf16 (is_bf16) or fp32 [rows, cols], row pitch ldx elements (transposed: stored [cols, rows], pitch ldx);
// q: [rows_pad, cols] bytes; sf: (rows_pad/128)*(cols/128)*512 bytes
extern "C" int hctr_mx_quantize(const void* x, long long ldx, void* q, void* sf, int rows, int cols, int is_bf16,
                                int transposed, void* stream) {
  if (cols % 128) return -2;
  const int rows_pad = (rows + 127) / 128 * 128;
  const long long total = static_cast<long long>(rows_pad) * (cols / 32);
  long long blocks = (total + 255) / 256;
  if (blocks > num_sms() * 16) blocks = num_sms() * 16;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (is_bf16)
    mx_quantize_kernel<__nv_bfloat16><<<static_cast<unsigned>(blocks), 256, 0, st>>>(
        reinterpret_cast<const __nv_bfloat16*>(x), ldx, reinterpret_cast<uint8_t*>(q), reinterpret_cast<uint8_t*>(sf),
        rows, rows_pad, cols, transposed);
  else
    mx_quantize_kernel<float><<<static_cast<unsigned>(blocks), 256, 0, st>>>(
        reinterpret_cast<const float*>(x), ldx, reinterpret_cast<uint8_t*>(q), reinterpret_cast<uint8_t*>(sf), rows,
        rows_pad, cols, transposed);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// A_q [M_pad, K], B_q [N_pad, K] e4m3 (row pitch K bytes), scales in block layout; out [M, N] bf16 (or fp32 with
// EPI_OUT_F32), bias fp32 [N] optional, flags: EPI_RELU / EPI_SIGMOID / EPI_OUT_F32
extern "C" int hctr_gemm_mxfp8(const void* Aq, const void* sfa, const void* Bq, const void* sfb, void* out, int M,
                               int N, int K, long long ldo, const float* bias, float alpha, int flags,
                               void* stream_) {
  if (M <= 0 || N <= 0 || K <= 0) return 0;
  if (K % 128) return -2;
  const int m_pad = (M + 127) / 128 * 128, n_pad = (N + 127) / 128 * 128;
  CUtensorMap ta, tb;
  if (make_tmap_u8(&ta, Aq, K, m_pad, K)) return -3;
  if (make_tmap_u8(&tb, Bq, K, n_pad, K)) return -4;
  GemmParams p{};
  p.M = M; p.N = N; p.K = K;
  p.m_tiles = m_pad / 128; p.n_tiles = n_pad / 128; p.k_blocks = K / 128; p.splits = 1; p.kb_per_split = p.k_blocks;
  p.out = out; p.ldo = ldo; p.bias = bias; p.alpha = alpha; p.flags = flags;
  static bool attr = false;
  if (!attr) {
    if (cudaFuncSetAttribute(gemm_mxfp8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MX_SMEM) != cudaSuccess)
      return -5;
    attr = true;
  }
  gemm_mxfp8_kernel<<<dim3(p.n_tiles, p.m_tiles), MX_THREADS, MX_SMEM, reinterpret_cast<cudaStream_t>(stream_)>>>(
      ta, tb, reinterpret_cast<const uint8_t*>(sfa), reinterpret_cast<const uint8_t*>(sfb), p);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
