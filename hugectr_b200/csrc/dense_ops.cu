// D4 elementwise / reduction family + fused dense optimizers + loss kernels (sm_90a).
//   fused optimizers over the flat parameter arena  (reference HugeCTR/src/optimizers/*.cu)
//   BinaryCrossEntropy fwd+bwd in one pass           (reference HugeCTR/src/loss.cu:231-264)
//   bias-grad column reduction, skinny (N==1) FC fwd/bwd, DCNv2 backward elementwise fusion
//   (reference HugeCTR/src/layers/multi_cross_layer.cu:60-222), strided 2-D copies for
//   concat/slice, fp32->bf16 cast with K padding, ReLU/Sigmoid fwd/bwd.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "optim.cuh"
#include "ptx.cuh"

namespace hctr {

using bf16 = __nv_bfloat16;

// ------------------------------------------------------------------ dense optimizers
struct DenseOptArgs {
  float* w;            // fp32 master weights (flat)
  float* g;            // fp32 wgrad (flat) ; zeroed after use when zero_grad
  bf16* w16;           // optional bf16 copy (flat, same indexing) or null
  float* s0;
  float* s1;
  long long n;
  OptHyper hp;         // the rule's hyper-parameters, device learning rate and step counter
  int zero_grad;
};

template <int OPT>
__global__ void __launch_bounds__(256) dense_opt_kernel(const DenseOptArgs a) {
  constexpr bool kHasS0 = OPT != OPT_SGD;
  constexpr bool kHasS1 = OPT == OPT_ADAM || OPT == OPT_FTRL;
  const OptHyper& hp = a.hp;
  const OptStep step = opt_step<OPT>(hp);
  const float inv_scaler = 1.f / hp.scaler;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x * 4;
  for (long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4; i < a.n;
       i += stride) {
    float w[4], g[4], s0[4], s1[4];
    const int cnt = static_cast<int>(min(4ll, a.n - i));
    if (cnt == 4) {
      const float4 wv = *reinterpret_cast<const float4*>(a.w + i);
      const float4 gv = *reinterpret_cast<const float4*>(a.g + i);
      w[0] = wv.x; w[1] = wv.y; w[2] = wv.z; w[3] = wv.w;
      g[0] = gv.x; g[1] = gv.y; g[2] = gv.z; g[3] = gv.w;
      if constexpr (kHasS0) {
        const float4 sv = *reinterpret_cast<const float4*>(a.s0 + i);
        s0[0] = sv.x; s0[1] = sv.y; s0[2] = sv.z; s0[3] = sv.w;
      }
      if constexpr (kHasS1) {
        const float4 sv = *reinterpret_cast<const float4*>(a.s1 + i);
        s1[0] = sv.x; s1[1] = sv.y; s1[2] = sv.z; s1[3] = sv.w;
      }
    } else {
      for (int j = 0; j < 4; ++j) {
        const bool ok = j < cnt;
        w[j] = ok ? a.w[i + j] : 0.f;
        g[j] = ok ? a.g[i + j] : 0.f;
        s0[j] = (ok && kHasS0) ? a.s0[i + j] : 0.f;
        s1[j] = (ok && kHasS1) ? a.s1[i + j] : 0.f;
      }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
      apply_opt<OPT, float>(w[j], g[j] * inv_scaler, s0 + j, s1 + j, 0, hp, step);
    if (cnt == 4) {
      *reinterpret_cast<float4*>(a.w + i) = make_float4(w[0], w[1], w[2], w[3]);
      if (a.zero_grad) *reinterpret_cast<float4*>(a.g + i) = make_float4(0.f, 0.f, 0.f, 0.f);
      if constexpr (kHasS0)
        *reinterpret_cast<float4*>(a.s0 + i) = make_float4(s0[0], s0[1], s0[2], s0[3]);
      if constexpr (kHasS1)
        *reinterpret_cast<float4*>(a.s1 + i) = make_float4(s1[0], s1[1], s1[2], s1[3]);
      if (a.w16)
        *reinterpret_cast<uint2*>(a.w16 + i) =
            make_uint2(pack_bf16x2(w[0], w[1]), pack_bf16x2(w[2], w[3]));
    } else {
      for (int j = 0; j < cnt; ++j) {
        a.w[i + j] = w[j];
        if (a.zero_grad) a.g[i + j] = 0.f;
        if (kHasS0) a.s0[i + j] = s0[j];
        if (kHasS1) a.s1[i + j] = s1[j];
        if (a.w16) a.w16[i + j] = __float2bfloat16(w[j]);
      }
    }
  }
}

// learning-rate schedule on device (reference gpu_learning_rate_scheduler.cu:26)
struct LrSched {
  float base_lr, end_lr, decay_power;
  unsigned int warmup, decay_start, decay_steps;
};
__global__ void lr_step_kernel(unsigned int* step, float* lr, const LrSched s) {
  const unsigned int t = *step + 1;
  *step = t;
  float v;
  if (t <= s.warmup) v = s.base_lr * static_cast<float>(t) / static_cast<float>(s.warmup);
  else if (s.decay_start == 0 || t <= s.decay_start) v = s.base_lr;
  else if (t <= s.decay_start + s.decay_steps) {
    const float f = static_cast<float>(s.decay_start + s.decay_steps - t) / static_cast<float>(s.decay_steps);
    v = fmaxf(s.base_lr * powf(f, s.decay_power), s.end_lr);
  } else v = s.end_lr;
  *lr = v;
}

// ------------------------------------------------------------------ BCE loss (fwd + in-place bwd)
// logits [n] (T), labels [n] fp32.  train: grad[i] = (sigmoid(x)-y) * grad_scale written to `dx`
// (may alias logits); eval: dx[i] = sigmoid(x).  loss_out += mean loss * loss_weight (atomic).
template <typename T>
__global__ void __launch_bounds__(256)
    bce_loss_kernel(const T* __restrict__ x, const float* __restrict__ y, T* dx, float* loss_out,
                    int n, float grad_scale, float loss_scale, int is_train, int want_loss) {
  float local = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float v = static_cast<float>(x[i]);
    const float t = y[i];
    const float ex = __expf(-fabsf(v));
    // stable: max(x,0) - x*y + log(1+exp(-|x|))
    local += fmaxf(v, 0.f) - v * t + log1pf(ex);
    const float sig = v >= 0.f ? 1.f / (1.f + ex) : ex / (1.f + ex);
    dx[i] = static_cast<T>(is_train ? (sig - t) * grad_scale : sig);
  }
  if (!want_loss) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  __shared__ float red[8];
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) red[w] = local;
  __syncthreads();
  if (w == 0) {
    float v = l < (blockDim.x >> 5) ? red[l] : 0.f;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (l == 0) atomicAdd(loss_out, v * loss_scale);
  }
}

// ------------------------------------------------------------------ column sum (bias grad)
// out[n] += sum_m x[m, n]   (x bf16/fp32 row-major, ld).  Block = 32 column-groups (8 columns each,
// one 16-byte load per row) x 8 row lanes; grid (ceil(N/256), row splits); fp32 atomics at the end.
template <typename T>
__global__ void __launch_bounds__(256)
    colsum_kernel(const T* __restrict__ x, float* __restrict__ out, int M, int N, long long ld) {
  constexpr int VEC = 16 / sizeof(T);  // 8 bf16 or 4 fp32
  __shared__ float sm[8][32 * VEC];
  const int cg = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int col = (blockIdx.x * 32 + cg) * VEC;
  const int rows_per = (M + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * rows_per, r1 = min(M, r0 + rows_per);
  float acc[VEC];
#pragma unroll
  for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
  const bool vec_ok = (col + VEC <= N) && ((ld * sizeof(T)) % 16 == 0) &&
                      (reinterpret_cast<uintptr_t>(x) % 16 == 0);
  if (col < N) {
    if (vec_ok) {
      for (int r = r0 + rl; r < r1; r += 8) {
        const uint4 v = *reinterpret_cast<const uint4*>(x + r * ld + col);
        if constexpr (sizeof(T) == 2) {
          const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            acc[2 * q] += bf16_lo(w[q]);
            acc[2 * q + 1] += bf16_hi(w[q]);
          }
        } else {
          acc[0] += __uint_as_float(v.x); acc[1] += __uint_as_float(v.y);
          acc[2] += __uint_as_float(v.z); acc[3] += __uint_as_float(v.w);
        }
      }
    } else {
      for (int r = r0 + rl; r < r1; r += 8)
#pragma unroll
        for (int j = 0; j < VEC; ++j)
          if (col + j < N) acc[j] += static_cast<float>(x[r * ld + col + j]);
    }
  }
#pragma unroll
  for (int j = 0; j < VEC; ++j) sm[rl][cg * VEC + j] = acc[j];
  __syncthreads();
  for (int c = threadIdx.x; c < 32 * VEC; c += 256) {
    const int gc = blockIdx.x * 32 * VEC + c;
    if (gc < N) {
      float v = 0.f;
#pragma unroll
      for (int r = 0; r < 8; ++r) v += sm[r][c];
      atomicAdd(out + gc, v);
    }
  }
}

// ------------------------------------------------------------------ skinny FC (num_output == 1)
// y[m] = act(dot(x[m,:], w) + b) ; one warp per row
template <typename T>
__global__ void __launch_bounds__(256)
    fc1_fwd_kernel(const T* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                   T* __restrict__ y, int M, int K, long long ldx, int relu) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  float acc = 0.f;
  for (int k = lane; k < K; k += 32) acc += static_cast<float>(x[row * ldx + k]) * __ldg(w + k);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) {
    acc += b ? b[0] : 0.f;
    if (relu) acc = fmaxf(acc, 0.f);
    y[row] = static_cast<T>(acc);
  }
}
// dx[m,k] = dy[m] * w[k] * (mask[m,k] > 0 if mask) ; dw[k] += sum_m x[m,k]*dy[m] ; db += sum dy
template <typename T>
__global__ void __launch_bounds__(256)
    fc1_bwd_kernel(const T* __restrict__ x, const float* __restrict__ w, const T* __restrict__ dy,
                   T* __restrict__ dx, float* __restrict__ dw, float* __restrict__ db, int M, int K,
                   long long ldx, long long lddx, int mask_relu, int rows_per_block) {
  // block handles rows_per_block rows; thread k-strided; accumulates dw in registers
  const int r0 = blockIdx.x * rows_per_block, r1 = min(M, r0 + rows_per_block);
  float dbl = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float wk = w[k];
    float acc = 0.f;
    for (int r = r0; r < r1; ++r) {
      const float g = static_cast<float>(dy[r]);
      const float xv = static_cast<float>(x[r * ldx + k]);
      acc += xv * g;
      if (dx) {
        float d = g * wk;
        if (mask_relu && !(xv > 0.f)) d = 0.f;
        dx[r * lddx + k] = static_cast<T>(d);
      }
    }
    atomicAdd(dw + k, acc);
  }
  if (db && threadIdx.x == 0) {
    for (int r = r0; r < r1; ++r) dbl += static_cast<float>(dy[r]);
    atomicAdd(db, dbl);
  }
}

// ------------------------------------------------------------------ elementwise helpers
// generic strided 2-D copy (concat / slice): dst[r, c] = src[r, c], 16-byte vectorised when possible
template <typename T>
__global__ void copy2d_kernel(const T* __restrict__ src, T* __restrict__ dst, long long rows,
                              int cols, long long lds, long long ldd, int accumulate) {
  const long long total = rows * cols;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / cols;
    const int c = static_cast<int>(i - r * cols);
    if (accumulate)
      dst[r * ldd + c] = static_cast<T>(static_cast<float>(dst[r * ldd + c]) +
                                        static_cast<float>(src[r * lds + c]));
    else
      dst[r * ldd + c] = src[r * lds + c];
  }
}
__global__ void copy2d_vec_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst,
                                  long long rows, int cols16, long long lds16, long long ldd16) {
  const long long total = rows * cols16;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / cols16;
    const int c = static_cast<int>(i - r * cols16);
    dst[r * ldd16 + c] = src[r * lds16 + c];
  }
}

// fp32 [M, K] -> bf16 [M, Kp] with zero padding of columns K..Kp
__global__ void cast_pad_kernel(const float* __restrict__ src, bf16* __restrict__ dst, long long M,
                                int K, int Kp, long long lds) {
  const long long total = M * Kp;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / Kp;
    const int c = static_cast<int>(i - r * Kp);
    dst[i] = __float2bfloat16(c < K ? src[r * lds + c] : 0.f);
  }
}

// op codes for the unary / binary elementwise kernels
enum EwOp : int { EW_RELU = 0, EW_RELU_BWD, EW_SIGMOID, EW_SIGMOID_BWD, EW_ADD, EW_SUB, EW_MUL,
                  EW_SCALE, EW_ELU, EW_ELU_BWD, EW_COPY, EW_ADD_INPLACE };

template <typename T>
__global__ void ew_kernel(const T* __restrict__ a, const T* __restrict__ b, T* __restrict__ o,
                          long long n, int op, float alpha) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float x = static_cast<float>(a[i]);
    const float y = b ? static_cast<float>(b[i]) : 0.f;
    float r;
    switch (op) {
      case EW_RELU: r = fmaxf(x, 0.f); break;
      case EW_RELU_BWD: r = y > 0.f ? x : 0.f; break;          // a = dy, b = fwd output
      case EW_SIGMOID: r = 1.f / (1.f + __expf(-x)); break;
      case EW_SIGMOID_BWD: r = x * y * (1.f - y); break;       // a = dy, b = fwd output
      case EW_ADD: r = x + y; break;
      case EW_SUB: r = x - y; break;
      case EW_MUL: r = x * y; break;
      case EW_SCALE: r = x * alpha; break;
      case EW_ELU: r = x > 0.f ? x : alpha * (__expf(x) - 1.f); break;
      case EW_ELU_BWD: r = y > 0.f ? x : x * (y + alpha); break;  // b = fwd output
      case EW_ADD_INPLACE: r = static_cast<float>(o[i]) + x; break;
      default: r = x; break;
    }
    o[i] = static_cast<T>(r);
  }
}

// DCNv2 backward elementwise fusion for one cross layer (bf16, vectorised x8):
//   dt  = dy * x0                                   (input of the V^T dgrad GEMM)
//   dx0 = (first ? 0 : dx0) + dy * t (+ dy if last) (accumulated over layers; on the last layer the
//         residual dy is folded in so the final dgrad GEMM epilogue adds ONE bf16 tensor)
//   db += column sums of dt                         (bias gradient, fused: no separate reduction)
// block = 16 column groups (128 columns) x 16 row lanes; a thread owns 8 fixed columns and walks
// rows ry, ry+16, ... of its row split with 4 rows of 16-byte loads in flight; bias partials stay in
// registers, are combined through shared memory and leave as one atomicAdd per column per block.
template <typename AccT>
__global__ void __launch_bounds__(256)
    cross_bwd_ew_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x0,
                        const bf16* __restrict__ t, bf16* __restrict__ dt, AccT* __restrict__ dx0,
                        float* __restrict__ db, int rows, int cols, int mode) {
  constexpr bool kAccBf16 = sizeof(AccT) == 2;
  __shared__ float red[16][16][9];
  const int cx = threadIdx.x & 15, ry = threadIdx.x >> 4;
  const int ngroups = cols >> 3;
  const int c8 = blockIdx.x * 16 + cx;
  const bool col_ok = c8 < ngroups;
  const int rows_per = (rows + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * rows_per, r1 = min(rows, r0 + rows_per);
  const bool first = mode & 1, last = mode & 2;
  float bsum[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) bsum[j] = 0.f;
  constexpr int NR = 4;
  if (col_ok) {
    for (int rb = r0 + ry; rb < r1; rb += 16 * NR) {
      uint4 a[NR], b[NR], c[NR], pb[NR];
      float4 p0[NR], p1[NR];
#pragma unroll
      for (int u = 0; u < NR; ++u) {
        const int r = rb + 16 * u;
        if (r < r1) {
          const long long i = static_cast<long long>(r) * ngroups + c8;
          a[u] = reinterpret_cast<const uint4*>(dy)[i];
          b[u] = reinterpret_cast<const uint4*>(x0)[i];
          c[u] = reinterpret_cast<const uint4*>(t)[i];
          if (!first) {
            if constexpr (kAccBf16) {
              pb[u] = reinterpret_cast<const uint4*>(dx0)[i];
            } else {
              p0[u] = reinterpret_cast<const float4*>(dx0)[2 * i];
              p1[u] = reinterpret_cast<const float4*>(dx0)[2 * i + 1];
            }
          }
        }
      }
#pragma unroll
      for (int u = 0; u < NR; ++u) {
        const int r = rb + 16 * u;
        if (r >= r1) continue;
        const long long i = static_cast<long long>(r) * ngroups + c8;
        const uint32_t aw[4] = {a[u].x, a[u].y, a[u].z, a[u].w}, bw[4] = {b[u].x, b[u].y, b[u].z, b[u].w},
                       cw[4] = {c[u].x, c[u].y, c[u].z, c[u].w};
        uint32_t ow[4];
        float acc[8];
        if (!first) {
          if constexpr (kAccBf16) {
            const uint32_t pw[4] = {pb[u].x, pb[u].y, pb[u].z, pb[u].w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              acc[2 * q] = bf16_lo(pw[q]);
              acc[2 * q + 1] = bf16_hi(pw[q]);
            }
          } else {
            acc[0] = p0[u].x; acc[1] = p0[u].y; acc[2] = p0[u].z; acc[3] = p0[u].w;
            acc[4] = p1[u].x; acc[5] = p1[u].y; acc[6] = p1[u].z; acc[7] = p1[u].w;
          }
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[j] = 0.f;
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float d0 = bf16_lo(aw[q]), d1 = bf16_hi(aw[q]);
          const float e0 = d0 * bf16_lo(bw[q]), e1 = d1 * bf16_hi(bw[q]);
          ow[q] = pack_bf16x2(e0, e1);
          bsum[2 * q] += bf16_lo(ow[q]);       // bias grad sums the bf16-rounded dt (what the GEMMs consume)
          bsum[2 * q + 1] += bf16_hi(ow[q]);
          acc[2 * q] += d0 * bf16_lo(cw[q]) + (last ? d0 : 0.f);
          acc[2 * q + 1] += d1 * bf16_hi(cw[q]) + (last ? d1 : 0.f);
        }
        reinterpret_cast<uint4*>(dt)[i] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
        if constexpr (kAccBf16) {
          reinterpret_cast<uint4*>(dx0)[i] =
              make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]),
                         pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
        } else {
          reinterpret_cast<float4*>(dx0)[2 * i] = make_float4(acc[0], acc[1], acc[2], acc[3]);
          reinterpret_cast<float4*>(dx0)[2 * i + 1] = make_float4(acc[4], acc[5], acc[6], acc[7]);
        }
      }
    }
  }
  if (db != nullptr) {
#pragma unroll
    for (int j = 0; j < 8; ++j) red[ry][cx][j] = bsum[j];
    __syncthreads();
    if (threadIdx.x < 128) {
      const int gx_ = threadIdx.x >> 3, j = threadIdx.x & 7;
      const int col = (blockIdx.x * 16 + gx_) * 8 + j;
      if (col < cols) {
        float sacc = 0.f;
#pragma unroll
        for (int y = 0; y < 16; ++y) sacc += red[y][gx_][j];
        atomicAdd(db + col, sacc);
      }
    }
  }
}
// out(bf16) = a(bf16) + b(bf16) [+ c(fp32)]   (vectorised x8) : dxl = dy + dxl_gemm (+ dx0 on last)
__global__ void __launch_bounds__(256)
    add3_kernel(const bf16* __restrict__ a, const bf16* __restrict__ b, const float* __restrict__ c,
                bf16* __restrict__ o, long long n8) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const uint4 av = reinterpret_cast<const uint4*>(a)[i];
    const uint4 bv = reinterpret_cast<const uint4*>(b)[i];
    const uint32_t aw[4] = {av.x, av.y, av.z, av.w}, bw[4] = {bv.x, bv.y, bv.z, bv.w};
    float r[8];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      r[2 * q] = bf16_lo(aw[q]) + bf16_lo(bw[q]);
      r[2 * q + 1] = bf16_hi(aw[q]) + bf16_hi(bw[q]);
    }
    if (c) {
      const float4 p0 = reinterpret_cast<const float4*>(c)[2 * i];
      const float4 p1 = reinterpret_cast<const float4*>(c)[2 * i + 1];
      r[0] += p0.x; r[1] += p0.y; r[2] += p0.z; r[3] += p0.w;
      r[4] += p1.x; r[5] += p1.y; r[6] += p1.z; r[7] += p1.w;
    }
    reinterpret_cast<uint4*>(o)[i] = make_uint4(pack_bf16x2(r[0], r[1]), pack_bf16x2(r[2], r[3]),
                                               pack_bf16x2(r[4], r[5]), pack_bf16x2(r[6], r[7]));
  }
}

static inline int grid_for(long long n, int threads, int max_blocks = num_sms() * 16) {
  long long b = (n + threads - 1) / threads;
  if (b > max_blocks) b = max_blocks;
  if (b < 1) b = 1;
  return static_cast<int>(b);
}

}  // namespace hctr

using namespace hctr;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define OK() (cudaGetLastError() == cudaSuccess ? 0 : -1)

extern "C" int hctr_abi_size_dense_opt() { return static_cast<int>(sizeof(DenseOptArgs)); }

extern "C" int hctr_dense_opt(const DenseOptArgs* a, int opt, void* stream) {
  if (a->n == 0) return 0;
  const int threads = 256;
  const int blocks = grid_for((a->n + 3) / 4, threads, num_sms() * 8);
  switch (opt) {
    case OPT_SGD: dense_opt_kernel<OPT_SGD><<<blocks, threads, 0, ST(stream)>>>(*a); break;
    case OPT_ADAGRAD: dense_opt_kernel<OPT_ADAGRAD><<<blocks, threads, 0, ST(stream)>>>(*a); break;
    case OPT_ADAM: dense_opt_kernel<OPT_ADAM><<<blocks, threads, 0, ST(stream)>>>(*a); break;
    case OPT_FTRL: dense_opt_kernel<OPT_FTRL><<<blocks, threads, 0, ST(stream)>>>(*a); break;
    case OPT_MOMENTUM: dense_opt_kernel<OPT_MOMENTUM><<<blocks, threads, 0, ST(stream)>>>(*a); break;
    case OPT_NESTEROV: dense_opt_kernel<OPT_NESTEROV><<<blocks, threads, 0, ST(stream)>>>(*a); break;
    case OPT_RMSPROP: dense_opt_kernel<OPT_RMSPROP><<<blocks, threads, 0, ST(stream)>>>(*a); break;
    default: return -2;
  }
  return OK();
}

extern "C" int hctr_lr_step(unsigned int* step, float* lr, float base_lr, float end_lr,
                            float decay_power, unsigned int warmup, unsigned int decay_start,
                            unsigned int decay_steps, void* stream) {
  LrSched s{base_lr, end_lr, decay_power, warmup, decay_start, decay_steps};
  lr_step_kernel<<<1, 1, 0, ST(stream)>>>(step, lr, s);
  return OK();
}

extern "C" int hctr_bce_loss(const void* x, const float* y, void* dx, float* loss_out, int n,
                             float grad_scale, float loss_scale, int is_train, int want_loss,
                             int is_bf16, void* stream) {
  const int blocks = grid_for(n, 256, num_sms() * 4);
  if (is_bf16)
    bce_loss_kernel<bf16><<<blocks, 256, 0, ST(stream)>>>((const bf16*)x, y, (bf16*)dx, loss_out, n,
                                                          grad_scale, loss_scale, is_train, want_loss);
  else
    bce_loss_kernel<float><<<blocks, 256, 0, ST(stream)>>>((const float*)x, y, (float*)dx, loss_out,
                                                           n, grad_scale, loss_scale, is_train, want_loss);
  return OK();
}

extern "C" int hctr_colsum(const void* x, float* out, int M, int N, long long ld, int is_bf16,
                           void* stream) {
  const int cols_per_block = is_bf16 ? 256 : 128;
  const int gx = (N + cols_per_block - 1) / cols_per_block;
  int gy = 1;
  while (gx * gy < 2 * num_sms() && M / (gy * 2) >= 64) gy *= 2;   // ~2 waves of blocks
  dim3 grid(gx, gy);
  if (is_bf16) colsum_kernel<bf16><<<grid, 256, 0, ST(stream)>>>((const bf16*)x, out, M, N, ld);
  else colsum_kernel<float><<<grid, 256, 0, ST(stream)>>>((const float*)x, out, M, N, ld);
  return OK();
}

extern "C" int hctr_fc1_fwd(const void* x, const float* w, const float* b, void* y, int M, int K,
                            long long ldx, int relu, int is_bf16, void* stream) {
  const int blocks = (M * 32 + 255) / 256;
  if (is_bf16) fc1_fwd_kernel<bf16><<<blocks, 256, 0, ST(stream)>>>((const bf16*)x, w, b, (bf16*)y, M, K, ldx, relu);
  else fc1_fwd_kernel<float><<<blocks, 256, 0, ST(stream)>>>((const float*)x, w, b, (float*)y, M, K, ldx, relu);
  return OK();
}

extern "C" int hctr_fc1_bwd(const void* x, const float* w, const void* dy, void* dx, float* dw,
                            float* db, int M, int K, long long ldx, long long lddx, int mask_relu,
                            int is_bf16, void* stream) {
  const int rows_per_block = 32;
  const int blocks = (M + rows_per_block - 1) / rows_per_block;
  if (is_bf16)
    fc1_bwd_kernel<bf16><<<blocks, 256, 0, ST(stream)>>>((const bf16*)x, w, (const bf16*)dy, (bf16*)dx, dw, db, M, K, ldx, lddx, mask_relu, rows_per_block);
  else
    fc1_bwd_kernel<float><<<blocks, 256, 0, ST(stream)>>>((const float*)x, w, (const float*)dy, (float*)dx, dw, db, M, K, ldx, lddx, mask_relu, rows_per_block);
  return OK();
}

extern "C" int hctr_copy2d(const void* src, void* dst, long long rows, int cols, long long lds,
                           long long ldd, int elem_bytes, int accumulate, void* stream) {
  if (rows == 0 || cols == 0) return 0;
  const long long row_bytes = static_cast<long long>(cols) * elem_bytes;
  if (!accumulate && row_bytes % 16 == 0 && (lds * elem_bytes) % 16 == 0 &&
      (ldd * elem_bytes) % 16 == 0 && reinterpret_cast<uintptr_t>(src) % 16 == 0 &&
      reinterpret_cast<uintptr_t>(dst) % 16 == 0) {
    const int c16 = static_cast<int>(row_bytes / 16);
    copy2d_vec_kernel<<<grid_for(rows * c16, 256), 256, 0, ST(stream)>>>(
        (const uint4*)src, (uint4*)dst, rows, c16, lds * elem_bytes / 16, ldd * elem_bytes / 16);
    return OK();
  }
  const int blocks = grid_for(rows * cols, 256);
  if (elem_bytes == 2) copy2d_kernel<bf16><<<blocks, 256, 0, ST(stream)>>>((const bf16*)src, (bf16*)dst, rows, cols, lds, ldd, accumulate);
  else if (elem_bytes == 4) copy2d_kernel<float><<<blocks, 256, 0, ST(stream)>>>((const float*)src, (float*)dst, rows, cols, lds, ldd, accumulate);
  else return -2;
  return OK();
}

extern "C" int hctr_cast_pad(const float* src, void* dst, long long M, int K, int Kp,
                             long long lds, void* stream) {
  cast_pad_kernel<<<grid_for(M * Kp, 256), 256, 0, ST(stream)>>>(src, (bf16*)dst, M, K, Kp, lds);
  return OK();
}

extern "C" int hctr_elementwise(const void* a, const void* b, void* o, long long n, int op,
                                float alpha, int is_bf16, void* stream) {
  if (n == 0) return 0;
  const int blocks = grid_for(n, 256);
  if (is_bf16) ew_kernel<bf16><<<blocks, 256, 0, ST(stream)>>>((const bf16*)a, (const bf16*)b, (bf16*)o, n, op, alpha);
  else ew_kernel<float><<<blocks, 256, 0, ST(stream)>>>((const float*)a, (const float*)b, (float*)o, n, op, alpha);
  return OK();
}

extern "C" int hctr_cross_bwd_ew(const void* dy, const void* x0, const void* t, void* dt,
                                 void* dx0, float* db, int rows, int cols, int mode,
                                 int dx0_bf16, int row_splits, void* stream) {
  if (cols % 8) return -2;
  const int gx = (cols / 8 + 15) / 16;
  int gy = row_splits > 0 ? row_splits : (num_sms() * 4 + gx - 1) / gx;
  if (gy * 16 > rows) gy = (rows + 15) / 16;
  if (gy < 1) gy = 1;
  if (dx0_bf16)
    cross_bwd_ew_kernel<bf16><<<dim3(gx, gy), 256, 0, ST(stream)>>>(
        (const bf16*)dy, (const bf16*)x0, (const bf16*)t, (bf16*)dt, (bf16*)dx0, db, rows, cols, mode);
  else
    cross_bwd_ew_kernel<float><<<dim3(gx, gy), 256, 0, ST(stream)>>>(
        (const bf16*)dy, (const bf16*)x0, (const bf16*)t, (bf16*)dt, (float*)dx0, db, rows, cols, mode);
  return OK();
}

// out[s, col0 + j] = sum_i part[s, i, j]   (partial pooled vectors of a row-sharded table, k shards)
template <typename T>
__global__ void __launch_bounds__(256)
    partial_sum_kernel(const T* __restrict__ part, T* __restrict__ out, int rows, int k, int w,
                       long long out_stride, int col0) {
  const long long total = static_cast<long long>(rows) * w;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long s = i / w;
    const int j = static_cast<int>(i - s * w);
    const T* p = part + s * k * w + j;
    float acc = 0.f;
    for (int q = 0; q < k; ++q) acc += static_cast<float>(p[static_cast<long long>(q) * w]);
    out[s * out_stride + col0 + j] = static_cast<T>(acc);
  }
}

extern "C" int hctr_partial_sum(const void* part, void* out, int rows, int k, int w,
                                long long out_stride, int col0, int is_bf16, void* stream) {
  const long long total = static_cast<long long>(rows) * w;
  if (total == 0) return 0;
  const int blocks = grid_for(total, 256);
  if (is_bf16)
    partial_sum_kernel<bf16><<<blocks, 256, 0, ST(stream)>>>((const bf16*)part, (bf16*)out, rows, k, w,
                                                             out_stride, col0);
  else
    partial_sum_kernel<float><<<blocks, 256, 0, ST(stream)>>>((const float*)part, (float*)out, rows, k,
                                                              w, out_stride, col0);
  return OK();
}

extern "C" int hctr_add3(const void* a, const void* b, const float* c, void* o, long long n,
                         void* stream) {
  if (n % 8) return -2;
  add3_kernel<<<grid_for(n / 8, 256), 256, 0, ST(stream)>>>((const bf16*)a, (const bf16*)b, c,
                                                             (bf16*)o, n / 8);
  return OK();
}
