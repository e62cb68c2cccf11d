// D2: DLRM dot-product interaction on Hopper wgmma (fwd + bwd), bf16, n <= 32 rows, D <= 128, D % 16 == 0.
//   fwd : out[s] = [ mlp[s] | strict lower triangle of X X^T (row-major) | 0 ],  X = [mlp[s]; emb[s]]
//   bwd : dX = (G + G^T) X  with G the lower-triangular gradient matrix;  dmlp = dX[0] + dout[:, :D],
//         demb = dX[1:] (both overwritten)
// Reference: HugeCTR/src/layers/interaction_layer.cu:47-596 (Volta wmma 16x16x16, one warp per
// sample).  Here FOUR samples share one tile: their (zero padded) 32-row blocks are stacked into a
// 128-row operand that sits in shared memory in the canonical SWIZZLE_128B layout.  Each of the two
// warpgroups owns two samples (64 rows): one m64n64 wgmma chain with A = B = its 64 rows produces both
// 32x32 Gram blocks on the diagonal, and the triangle is stored straight from the accumulator
// fragments.  The backward builds a block-diagonal (G+G^T) operand and multiplies it with the same X
// tile used as an MN-major B (m64n128 per warpgroup).
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ptx.cuh"

namespace hctr {

using bf16 = __nv_bfloat16;
constexpr int kSPT = 4;          // samples per tile
[[maybe_unused]] constexpr int kRows = 32;  // padded rows per sample (layout constant, documents kSPT * kRows == 128)
constexpr int kHalfBytes = 128 * 128;  // one 64-column half of a 128-row tile

// byte offset of 16-byte chunk `c` (0..15 over D=128) of tile row `row` in the SW128 layout
HCTR_DEVICE uint32_t tile_off(int row, int c) {
  return static_cast<uint32_t>((c >> 3) * kHalfBytes + row * 128 + (((c & 7) ^ (row & 7)) << 4));
}

// cooperative fill of the stacked X tile for samples [s0, s0+4)
HCTR_DEVICE void fill_x_tile(uint8_t* smem_x, const bf16* __restrict__ mlp,
                             const bf16* __restrict__ emb, int s0, int B, int n, int D) {
  const int chunks = D >> 3;  // 16-byte chunks per row
  for (int t = threadIdx.x; t < 128 * 16; t += blockDim.x) {
    const int row = t >> 4, c = t & 15;
    const int i = row >> 5, j = row & 31;
    const int s = s0 + i;
    int4 v = make_int4(0, 0, 0, 0);
    if (c < chunks && s < B && j < n) {
      const bf16* src = (j == 0) ? mlp + static_cast<long long>(s) * D
                                 : emb + (static_cast<long long>(s) * (n - 1) + (j - 1)) * D;
      v = ld_nc_v4(reinterpret_cast<const int4*>(src) + c);
    }
    *reinterpret_cast<int4*>(smem_x + tile_off(row, c)) = v;
  }
}

__global__ void __launch_bounds__(256, 2)
    interaction_fwd_kernel(const bf16* __restrict__ mlp, const bf16* __restrict__ emb,
                           bf16* __restrict__ out, int B, int n, int D, int out_w) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem_x = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                               ~static_cast<uintptr_t>(1023));
  const int wg = threadIdx.x >> 7, w4 = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int ntiles = (B + kSPT - 1) / kSPT;
  const int ntri = n * (n - 1) / 2;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int s0 = tile * kSPT;
    fill_x_tile(smem_x, mlp, emb, s0, B, n, D);
    fence_proxy_async();   // generic-proxy smem writes -> visible to the tensor-core (async) proxy
    __syncthreads();
    // passthrough of the bottom-MLP output + zero pad column
    for (int t = threadIdx.x; t < kSPT * D; t += blockDim.x) {
      const int i = t / D, c = t - i * D, s = s0 + i;
      if (s >= B) continue;
      bf16* o = out + static_cast<long long>(s) * out_w;
      if ((out_w & 7) == 0) {
        if ((c & 7) == 0)
          reinterpret_cast<int4*>(o)[c >> 3] =
              ld_nc_v4(reinterpret_cast<const int4*>(mlp + static_cast<long long>(s) * D) + (c >> 3));
      } else {
        o[c] = mlp[static_cast<long long>(s) * D + c];
      }
      if (c == 0) o[D + ntri] = __float2bfloat16(0.f);
    }
    float acc[32];
    {
      const uint32_t base = smem_u32(smem_x) + wg * (64 * 128);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k) {              // D <= 128: at most 8 steps of 16
        if (k >= (D >> 4)) break;
        const uint64_t d = make_smem_desc_sw128(base + (k >> 2) * kHalfBytes + (k & 3) * 32, 16, 1024);
        wgmma_bf16_n64<0, 0>(acc, d, d, k > 0 ? 1u : 0u);   // Z = X X^T : A and B are the same rows
      }
      wgmma_commit();
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);
    // rows 16 w4 + lane / 4 (+ 8) of this warpgroup's 64; the sample's Gram block is n8 blocks [4 h, 4 h + 4)
    const int h = w4 >> 1, s = s0 + 2 * wg + h;
    if (s < B) {
      bf16* o = out + static_cast<long long>(s) * out_w + D;
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int i = (16 * w4 + (lane >> 2) + 8 * half) & 31;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int c = 8 * jj + 2 * (lane & 3) + e;
            const float v = h ? acc[16 + 4 * jj + 2 * half + e] : acc[4 * jj + 2 * half + e];
            if (i < n && c < i) o[i * (i - 1) / 2 + c] = __float2bfloat16(v);
          }
        }
      }
    }
    __syncthreads();   // smem tile consumed before the next tile overwrites it
  }
}

__global__ void __launch_bounds__(256, 2)
    interaction_bwd_kernel(const bf16* __restrict__ mlp, const bf16* __restrict__ emb,
                           const bf16* __restrict__ dout, bf16* __restrict__ dmlp,
                           bf16* __restrict__ demb, int B, int n, int D, int out_w) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem_x = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                               ~static_cast<uintptr_t>(1023));
  uint8_t* smem_g = smem_x + 2 * kHalfBytes;   // block-diagonal (G + G^T), K-major, 2 halves
  const int wg = threadIdx.x >> 7, w4 = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int ntiles = (B + kSPT - 1) / kSPT;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int s0 = tile * kSPT;
    fill_x_tile(smem_x, mlp, emb, s0, B, n, D);
    // zero the G tile, then write the four 32x32 diagonal blocks
    for (int t = threadIdx.x; t < 2 * kHalfBytes / 16; t += blockDim.x)
      reinterpret_cast<int4*>(smem_g)[t] = make_int4(0, 0, 0, 0);
    __syncthreads();
    for (int t = threadIdx.x; t < 128 * 4; t += blockDim.x) {
      const int row = t >> 2, cc = t & 3;       // cc: 8-column chunk inside the sample's block
      const int i = row >> 5, r = row & 31, s = s0 + i;
      if (s >= B || r >= n) continue;
      const bf16* g = dout + static_cast<long long>(s) * out_w + D;
      uint32_t w[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        float v[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = cc * 8 + q * 2 + e;
          float x = 0.f;
          if (c < n && c != r) {
            const int hi = max(r, c), lo = min(r, c);
            x = __bfloat162float(g[hi * (hi - 1) / 2 + lo]);
          }
          v[e] = x;
        }
        w[q] = pack_bf16x2(v[0], v[1]);
      }
      const int col_chunk = i * 4 + cc;          // 16-byte chunk index along K (0..15)
      *reinterpret_cast<int4*>(smem_g + tile_off(row, col_chunk)) =
          make_int4(static_cast<int>(w[0]), static_cast<int>(w[1]), static_cast<int>(w[2]),
                    static_cast<int>(w[3]));
    }
    fence_proxy_async();
    __syncthreads();
    // D[64 rows of this warpgroup, N = 128] = A[64, K = 128] (K-major) * B (MN-major: rows = K, 64-wide N chunks)
    float acc[64];
    {
      const uint32_t ga = smem_u32(smem_g) + wg * (64 * 128), xb = smem_u32(smem_x);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 8; ++k) {            // K = 128 stacked rows
        const uint64_t a = make_smem_desc_sw128(ga + (k >> 2) * kHalfBytes + (k & 3) * 32, 16, 1024);
        const uint64_t b = make_smem_desc_sw128(xb + k * 2048, kHalfBytes, 1024);
        wgmma_bf16_n128<0, 1>(acc, a, b, k > 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
    }
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int row = 64 * wg + 16 * w4 + (lane >> 2) + 8 * half;
      const int s = s0 + (row >> 5), j = row & 31;
      if (s >= B || j >= n) continue;
      bf16* dst = j == 0 ? dmlp + static_cast<long long>(s) * D
                         : demb + (static_cast<long long>(s) * (n - 1) + (j - 1)) * D;
      const bf16* pass = j == 0 ? dout + static_cast<long long>(s) * out_w : nullptr;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        const int c = 8 * jj + 2 * (lane & 3);
        if (c >= D) continue;
        float v0 = acc[4 * jj + 2 * half], v1 = acc[4 * jj + 2 * half + 1];
        if (pass) {
          v0 += __bfloat162float(pass[c]);
          v1 += __bfloat162float(pass[c + 1]);
        }
        *reinterpret_cast<uint32_t*>(dst + c) = pack_bf16x2(v0, v1);
      }
    }
    __syncthreads();
  }
}

}  // namespace hctr

using namespace hctr;

extern "C" int hctr_interaction_fwd(const void* mlp, const void* emb, void* out, int B, int n, int D,
                                    void* stream) {
  if (n > 32 || D > 128 || (D & 15)) return -2;
  static bool attr = false;
  const int smem = 2 * kHalfBytes + 1024;
  if (!attr) {
    cudaFuncSetAttribute(interaction_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr = true;
  }
  const int out_w = D + n * (n - 1) / 2 + 1;
  const int tiles = (B + kSPT - 1) / kSPT;
  const int grid = tiles < 2 * num_sms() ? tiles : 2 * num_sms();
  interaction_fwd_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(
      (const bf16*)mlp, (const bf16*)emb, (bf16*)out, B, n, D, out_w);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int hctr_interaction_bwd(const void* mlp, const void* emb, const void* dout, void* dmlp,
                                    void* demb, int B, int n, int D, void* stream) {
  if (n > 32 || D > 128 || (D & 15)) return -2;
  static bool attr = false;
  const int smem = 4 * kHalfBytes + 1024;
  if (!attr) {
    cudaFuncSetAttribute(interaction_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    attr = true;
  }
  const int out_w = D + n * (n - 1) / 2 + 1;
  const int tiles = (B + kSPT - 1) / kSPT;
  const int grid = tiles < 2 * num_sms() ? tiles : 2 * num_sms();
  interaction_bwd_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(
      (const bf16*)mlp, (const bf16*)emb, (const bf16*)dout, (bf16*)dmlp, (bf16*)demb, B, n, D, out_w);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
