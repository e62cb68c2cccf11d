// Native forward / backward kernels of the long-tail dense layers (SURVEY 2.2): normalisation (LayerNorm,
// BatchNorm, PReLU_Dice), Softmax / MaskedSoftmax, FmOrder2, WeightMultiply, ReduceSum / ReduceMean, generic
// strided copies (Scale, Select, Gather, FusedReshapeConcat), strided batched matmul (MatrixMultiply,
// MultiHeadAttention) and the GRU gate math.  Reference files: HugeCTR/src/layers/{layer_norm_layer.cu:43-239,
// batch_norm_layer.cu:155-185 (cuDNN there), prelu_dice_layer.cu:45-86, softmax_layer.cu:53-173,
// masked_softmax_layer.cu:33-140, fm_order2_layer.cu:24-91, weight_multiply_layer.cu:32-82, reduce_sum_layer.cu,
// reduce_mean_layer.cu, scale_layer.cu:32-78, multi_head_attention_layer.cu:324-481, gru_layer.cu:265 (cuDNN)}.
// All math in fp32; T = float or bf16 storage.  With these the zoo models (DIN, BST, DeepFM, W&D, MMoE, NCF)
// run without a single at:: kernel in the step and are CUDA-graph capturable.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ptx.cuh"

namespace hctr {

using bf16 = __nv_bfloat16;
template <typename T> __device__ __forceinline__ float ldf(const T* p, long long i) { return static_cast<float>(p[i]); }
template <typename T> __device__ __forceinline__ void stf(T* p, long long i, float v) { p[i] = static_cast<T>(v); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------ row-wise: softmax, layer norm
// one warp per row of length n
template <typename T>
__global__ void __launch_bounds__(256)
    softmax_fwd_kernel(const T* __restrict__ x, const T* __restrict__ mask, T* __restrict__ y, long long rows,
                       int n) {
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const T* xr = x + row * n;
  const T* mr = mask ? mask + row * n : nullptr;
  float mx = -3.0e38f;
  for (int i = lane; i < n; i += 32) {
    float v = ldf(xr, i);
    if (mr && !(ldf(mr, i) > 0.f)) v = -10000.f;
    mx = fmaxf(mx, v);
  }
  mx = warp_max(mx);
  float s = 0.f;
  for (int i = lane; i < n; i += 32) {
    float v = ldf(xr, i);
    if (mr && !(ldf(mr, i) > 0.f)) v = -10000.f;
    s += __expf(v - mx);
  }
  s = warp_sum(s);
  const float inv = 1.f / s;
  for (int i = lane; i < n; i += 32) {
    float v = ldf(xr, i);
    if (mr && !(ldf(mr, i) > 0.f)) v = -10000.f;
    stf(y + row * n, i, __expf(v - mx) * inv);
  }
}

// dx = y * (dy - sum(dy * y)); masked positions get the gradient of the constant (0)
template <typename T>
__global__ void __launch_bounds__(256)
    softmax_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ y, const T* __restrict__ mask,
                       T* __restrict__ dx, long long rows, int n) {
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float dot = 0.f;
  for (int i = lane; i < n; i += 32) dot += ldf(dy, row * n + i) * ldf(y, row * n + i);
  dot = warp_sum(dot);
  for (int i = lane; i < n; i += 32) {
    float g = ldf(y, row * n + i) * (ldf(dy, row * n + i) - dot);
    if (mask && !(ldf(mask, row * n + i) > 0.f)) g = 0.f;
    stf(dx, row * n + i, g);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
    layernorm_fwd_kernel(const T* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                         T* __restrict__ y, float* __restrict__ mean, float* __restrict__ rstd, long long rows,
                         int n, float eps) {
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float s = 0.f;
  for (int i = lane; i < n; i += 32) s += ldf(x, row * n + i);
  const float mu = warp_sum(s) / n;
  float v = 0.f;
  for (int i = lane; i < n; i += 32) {
    const float d = ldf(x, row * n + i) - mu;
    v += d * d;
  }
  const float rs = rsqrtf(warp_sum(v) / n + eps);
  if (lane == 0) {
    mean[row] = mu;
    rstd[row] = rs;
  }
  for (int i = lane; i < n; i += 32)
    stf(y, row * n + i, (ldf(x, row * n + i) - mu) * rs * gamma[i] + beta[i]);
}

// dx = rstd * (g - mean(g) - xhat * mean(g * xhat)),  g = dy * gamma
template <typename T>
__global__ void __launch_bounds__(256)
    layernorm_bwd_dx_kernel(const T* __restrict__ dy, const T* __restrict__ x, const float* __restrict__ gamma,
                            const float* __restrict__ mean, const float* __restrict__ rstd, T* __restrict__ dx,
                            long long rows, int n) {
  const long long row = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float mu = mean[row], rs = rstd[row];
  float a = 0.f, b = 0.f;
  for (int i = lane; i < n; i += 32) {
    const float g = ldf(dy, row * n + i) * gamma[i];
    const float xh = (ldf(x, row * n + i) - mu) * rs;
    a += g;
    b += g * xh;
  }
  a = warp_sum(a) / n;
  b = warp_sum(b) / n;
  for (int i = lane; i < n; i += 32) {
    const float g = ldf(dy, row * n + i) * gamma[i];
    const float xh = (ldf(x, row * n + i) - mu) * rs;
    stf(dx, row * n + i, rs * (g - a - xh * b));
  }
}

// ------------------------------------------------------------------ column reductions (two sums per column)
// out0[c] += sum_r u(r, c), out1[c] += sum_r v(r, c);  block = 32 columns x 8 row lanes, grid.y splits rows
//   MODE 0  u = x           v = x * x                      (batch statistics)
//   MODE 1  u = dy          v = dy * (x - m[c]) * s[c]     (BatchNorm dbeta / dgamma; m, s per column)
//   MODE 2  u = dy          v = dy * (x - m[r]) * s[r]     (LayerNorm dbeta / dgamma; m, s per row)
//   MODE 3  u = a           v = a * (x - m[c]),  a = dy * (1 - alpha) * x * p * (1 - p), p = sigmoid((x - m[c]) * s[c])
template <typename T, int MODE>
__global__ void __launch_bounds__(256)
    colreduce2_kernel(const T* __restrict__ x, const T* __restrict__ dy, const float* __restrict__ m,
                      const float* __restrict__ s, float* __restrict__ out0, float* __restrict__ out1,
                      long long rows, int cols, float alpha) {
  __shared__ float r0[8][33], r1[8][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx;
  const long long per = (rows + gridDim.y - 1) / gridDim.y;
  const long long lo = blockIdx.y * per, hi = min(rows, lo + per);
  float a0 = 0.f, a1 = 0.f;
  if (c < cols) {
    for (long long r = lo + ry; r < hi; r += 8) {
      const float xv = ldf(x, r * cols + c);
      if constexpr (MODE == 0) {
        a0 += xv;
        a1 += xv * xv;
      } else if constexpr (MODE == 1) {
        const float g = ldf(dy, r * cols + c);
        a0 += g;
        a1 += g * (xv - m[c]) * s[c];
      } else if constexpr (MODE == 2) {
        const float g = ldf(dy, r * cols + c);
        a0 += g;
        a1 += g * (xv - m[r]) * s[r];
      } else {
        const float p = 1.f / (1.f + __expf(-(xv - m[c]) * s[c]));
        const float a = ldf(dy, r * cols + c) * (1.f - alpha) * xv * p * (1.f - p);
        a0 += a;
        a1 += a * (xv - m[c]);
      }
    }
  }
  r0[ry][cx] = a0;
  r1[ry][cx] = a1;
  __syncthreads();
  if (ry == 0 && c < cols) {
#pragma unroll
    for (int j = 1; j < 8; ++j) {
      a0 += r0[j][cx];
      a1 += r1[j][cx];
    }
    atomicAdd(out0 + c, a0);
    atomicAdd(out1 + c, a1);
  }
}

// stats[0..cols) = sum x, stats[cols..2cols) = sum x^2  ->  mean, rstd (biased variance); optional running
// statistics update  run = momentum * run + (1 - momentum) * batch
__global__ void bn_finalize_kernel(const float* __restrict__ sum, const float* __restrict__ sumsq,
                                   float* __restrict__ mean, float* __restrict__ rstd, float* __restrict__ var_out,
                                   float* __restrict__ run_mean, float* __restrict__ run_var, int cols, float inv_n,
                                   float eps, float momentum) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  const float mu = sum[c] * inv_n;
  const float var = fmaxf(sumsq[c] * inv_n - mu * mu, 0.f);
  mean[c] = mu;
  rstd[c] = rsqrtf(var + eps);
  if (var_out) var_out[c] = var;
  if (run_mean) {
    run_mean[c] = momentum * run_mean[c] + (1.f - momentum) * mu;
    run_var[c] = momentum * run_var[c] + (1.f - momentum) * var;
  }
}

// elementwise with per-column parameters
//   OP 0  BatchNorm fwd   y = (x - m) * s * gamma + beta
//   (BatchNorm backward: bn_bwd_dx_kernel below)
//   OP 2  Dice fwd        y = x * (alpha + (1 - alpha) * p),  p = sigmoid((x - m) * s)
//   OP 3  Dice bwd        dx = dy * (alpha + (1 - alpha) * (p + x p (1 - p) s)) - s / N * A - (x - m) s^3 / N * B
template <typename T, int OP>
__global__ void __launch_bounds__(256)
    colwise_kernel(const T* __restrict__ x, const T* __restrict__ dy, const float* __restrict__ m,
                   const float* __restrict__ s, const float* __restrict__ p0, const float* __restrict__ p1,
                   T* __restrict__ out, long long total, int cols, float alpha, float inv_n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % cols);
    const float xv = ldf(x, i);
    float r;
    if constexpr (OP == 0) {
      r = (xv - m[c]) * s[c] * p0[c] + p1[c];
    } else if constexpr (OP == 2) {
      const float p = 1.f / (1.f + __expf(-(xv - m[c]) * s[c]));
      r = xv * (alpha + (1.f - alpha) * p);
    } else {
      const float sc = s[c];
      const float p = 1.f / (1.f + __expf(-(xv - m[c]) * sc));
      r = ldf(dy, i) * (alpha + (1.f - alpha) * (p + xv * p * (1.f - p) * sc)) - sc * inv_n * p0[c] -
          (xv - m[c]) * sc * sc * sc * inv_n * p1[c];
    }
    stf(out, i, r);
  }
}

// ------------------------------------------------------------------ FmOrder2 / WeightMultiply / reductions
// x [b, S, D] -> y [b, D] = 0.5 * ((sum_s x)^2 - sum_s x^2)
template <typename T>
__global__ void fm_order2_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, long long b, int S, int D) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= b * D) return;
  const long long r = i / D;
  const int d = static_cast<int>(i - r * D);
  float s = 0.f, q = 0.f;
  for (int k = 0; k < S; ++k) {
    const float v = ldf(x, (r * S + k) * D + d);
    s += v;
    q += v * v;
  }
  stf(y, i, 0.5f * (s * s - q));
}
// dx[b, s, d] = dy[b, d] * (sum_s' x[b, s', d] - x[b, s, d])
template <typename T>
__global__ void fm_order2_bwd_kernel(const T* __restrict__ x, const T* __restrict__ dy, T* __restrict__ dx,
                                     long long b, int S, int D) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= b * D) return;
  const long long r = i / D;
  const int d = static_cast<int>(i - r * D);
  float s = 0.f;
  for (int k = 0; k < S; ++k) s += ldf(x, (r * S + k) * D + d);
  const float g = ldf(dy, i);
  for (int k = 0; k < S; ++k) {
    const long long j = (r * S + k) * D + d;
    stf(dx, j, g * (s - ldf(x, j)));
  }
}

// y[b, s * V + j] = x[b, s] * W[s, j]
template <typename T>
__global__ void weight_mul_fwd_kernel(const T* __restrict__ x, const float* __restrict__ w, T* __restrict__ y,
                                      long long total, int S, int V) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long bs = i / V;
    const int j = static_cast<int>(i - bs * V);
    const int s = static_cast<int>(bs % S);
    stf(y, i, ldf(x, bs) * w[s * V + j]);
  }
}
// dx[b, s] = sum_j dy[b, s, j] * W[s, j]
template <typename T>
__global__ void weight_mul_bwd_dx_kernel(const T* __restrict__ dy, const float* __restrict__ w,
                                         T* __restrict__ dx, long long bs_total, int S, int V) {
  const long long bs = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (bs >= bs_total) return;
  const int s = static_cast<int>(bs % S);
  float a = 0.f;
  for (int j = 0; j < V; ++j) a += ldf(dy, bs * V + j) * w[s * V + j];
  stf(dx, bs, a);
}
// dW[s, j] += sum_b dy[b, s, j] * x[b, s] : grid (ceil(S*V / 256), row splits)
template <typename T>
__global__ void __launch_bounds__(256)
    weight_mul_bwd_dw_kernel(const T* __restrict__ dy, const T* __restrict__ x, float* __restrict__ dw, long long b,
                             int S, int V) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= S * V) return;
  const int s = c / V;
  const long long per = (b + gridDim.y - 1) / gridDim.y;
  const long long lo = blockIdx.y * per, hi = min(b, lo + per);
  float a = 0.f;
  for (long long r = lo; r < hi; ++r) a += ldf(dy, r * S * V + c) * ldf(x, r * S + s);
  atomicAdd(dw + c, a);
}

// x [outer, R, inner] -> y [outer, inner] = scale * sum_r ; backward broadcasts
template <typename T>
__global__ void reduce_mid_fwd_kernel(const T* __restrict__ x, T* __restrict__ y, long long outer, int R,
                                      long long inner, float scale) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= outer * inner) return;
  const long long o = i / inner, k = i - o * inner;
  float a = 0.f;
  for (int r = 0; r < R; ++r) a += ldf(x, (o * R + r) * inner + k);
  stf(y, i, a * scale);
}
template <typename T>
__global__ void reduce_mid_bwd_kernel(const T* __restrict__ dy, T* __restrict__ dx, long long outer, int R,
                                      long long inner, float scale) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= outer * R * inner) return;
  const long long o = i / (R * inner), k = i % inner;
  stf(dx, i, ldf(dy, o * inner + k) * scale);
}

// ------------------------------------------------------------------ generic 4-D strided copy / accumulate
struct Copy4D {
  long long d[4];     // extents (outermost first)
  long long ss[4];    // source element strides (0 = broadcast)
  long long ds[4];    // destination element strides
};
template <typename T>
__global__ void copy4d_kernel(const T* __restrict__ src, T* __restrict__ dst, Copy4D c, int accumulate) {
  const long long total = c.d[0] * c.d[1] * c.d[2] * c.d[3];
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    long long t = i;
    const long long i3 = t % c.d[3]; t /= c.d[3];
    const long long i2 = t % c.d[2]; t /= c.d[2];
    const long long i1 = t % c.d[1]; t /= c.d[1];
    const long long so = t * c.ss[0] + i1 * c.ss[1] + i2 * c.ss[2] + i3 * c.ss[3];
    const long long dofs = t * c.ds[0] + i1 * c.ds[1] + i2 * c.ds[2] + i3 * c.ds[3];
    if (accumulate) stf(dst, dofs, ldf(dst, dofs) + ldf(src, so));
    else dst[dofs] = src[so];
  }
}

// ------------------------------------------------------------------ strided batched matmul (CUDA cores)
// C[z](m, n) = alpha * sum_k A[z](m, k) * B[z](k, n) (+ C if accumulate); z = (z0, z1) two-level batch;
// every operand is addressed by element strides, so transposes and head splits need no copies.
struct BmmDesc {
  int M, N, K, Z1;                 // batch = Z0 * Z1 (grid.z = Z0 * Z1)
  long long a_z0, a_z1, a_m, a_k;
  long long b_z0, b_z1, b_k, b_n;
  long long c_z0, c_z1, c_m, c_n;
  float alpha;
  int accumulate;
};
template <typename TA, typename TB, typename TC>
__global__ void __launch_bounds__(256)
    bmm_kernel(const TA* __restrict__ A, const TB* __restrict__ B, TC* __restrict__ C, BmmDesc d) {
  __shared__ float sa[16][17], sb[16][17];
  const int z = blockIdx.z, z0 = z / d.Z1, z1 = z - z0 * d.Z1;
  const TA* a = A + z0 * d.a_z0 + z1 * d.a_z1;
  const TB* b = B + z0 * d.b_z0 + z1 * d.b_z1;
  TC* c = C + z0 * d.c_z0 + z1 * d.c_z1;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m = blockIdx.y * 16 + ty, n = blockIdx.x * 16 + tx;
  float acc = 0.f;
  for (int k0 = 0; k0 < d.K; k0 += 16) {
    const int ka = k0 + tx, kb = k0 + ty;
    sa[ty][tx] = (m < d.M && ka < d.K) ? static_cast<float>(a[m * d.a_m + ka * d.a_k]) : 0.f;
    sb[ty][tx] = (kb < d.K && n < d.N) ? static_cast<float>(b[kb * d.b_k + n * d.b_n]) : 0.f;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) acc += sa[ty][k] * sb[k][tx];
    __syncthreads();
  }
  if (m < d.M && n < d.N) {
    const long long o = m * d.c_m + n * d.c_n;
    float r = acc * d.alpha;
    if (d.accumulate) r += static_cast<float>(c[o]);
    c[o] = static_cast<TC>(r);
  }
}

// ------------------------------------------------------------------ GRU gates (PyTorch / cuDNN gate order r, z, n)
// gi, gh: [b, 3h] pre-activations (bias included); h' = (1 - z) * n + z * h
__global__ void gru_gate_fwd_kernel(const float* __restrict__ gi, const float* __restrict__ gh,
                                    const float* __restrict__ hprev, float* __restrict__ hnew,
                                    float* __restrict__ save, long long b, int H) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= b * H) return;
  const long long r_ = i / H;
  const int j = static_cast<int>(i - r_ * H);
  const long long o = r_ * 3 * H;
  const float r = 1.f / (1.f + __expf(-(gi[o + j] + gh[o + j])));
  const float z = 1.f / (1.f + __expf(-(gi[o + H + j] + gh[o + H + j])));
  const float hn = gh[o + 2 * H + j];
  const float n = tanhf(gi[o + 2 * H + j] + r * hn);
  hnew[i] = (1.f - z) * n + z * hprev[i];
  save[o + j] = r;
  save[o + H + j] = z;
  save[o + 2 * H + j] = n;
}
// dh' -> dgi, dgh (pre-activation grads), dhprev (direct path); hn = gh_n is re-read
__global__ void gru_gate_bwd_kernel(const float* __restrict__ dh, const float* __restrict__ save,
                                    const float* __restrict__ gh, const float* __restrict__ hprev,
                                    float* __restrict__ dgi, float* __restrict__ dgh, float* __restrict__ dhprev,
                                    long long b, int H) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= b * H) return;
  const long long r_ = i / H;
  const int j = static_cast<int>(i - r_ * H);
  const long long o = r_ * 3 * H;
  const float r = save[o + j], z = save[o + H + j], n = save[o + 2 * H + j];
  const float g = dh[i];
  const float dn = g * (1.f - z) * (1.f - n * n);
  const float dz = g * (hprev[i] - n) * z * (1.f - z);
  const float hn = gh[o + 2 * H + j];
  const float dr = dn * hn * r * (1.f - r);
  dgi[o + j] = dr;
  dgi[o + H + j] = dz;
  dgi[o + 2 * H + j] = dn;
  dgh[o + j] = dr;
  dgh[o + H + j] = dz;
  dgh[o + 2 * H + j] = dn * r;
  dhprev[i] = g * z;
}

}  // namespace hctr

using namespace hctr;
#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define OK() (cudaGetLastError() == cudaSuccess ? 0 : -1)
static inline unsigned grid1(long long n, int threads = 256, long long cap = hctr::num_sms() * 32LL) {
  long long b = (n + threads - 1) / threads;
  if (b > cap) b = cap;
  return static_cast<unsigned>(b < 1 ? 1 : b);
}
static inline unsigned gridx(long long n, int threads = 256) { return static_cast<unsigned>((n + threads - 1) / threads); }
#define DISPATCH_T(bf, CALL_F, CALL_B) do { if (bf) { CALL_B; } else { CALL_F; } } while (0)

extern "C" int hctr_softmax_fwd(const void* x, const void* mask, void* y, long long rows, int n, int bf, void* s) {
  if (rows == 0) return 0;
  const unsigned g = gridx(rows * 32);
  DISPATCH_T(bf, (softmax_fwd_kernel<float><<<g, 256, 0, ST(s)>>>((const float*)x, (const float*)mask, (float*)y, rows, n)),
             (softmax_fwd_kernel<bf16><<<g, 256, 0, ST(s)>>>((const bf16*)x, (const bf16*)mask, (bf16*)y, rows, n)));
  return OK();
}
extern "C" int hctr_softmax_bwd(const void* dy, const void* y, const void* mask, void* dx, long long rows, int n,
                                int bf, void* s) {
  if (rows == 0) return 0;
  const unsigned g = gridx(rows * 32);
  DISPATCH_T(bf, (softmax_bwd_kernel<float><<<g, 256, 0, ST(s)>>>((const float*)dy, (const float*)y, (const float*)mask, (float*)dx, rows, n)),
             (softmax_bwd_kernel<bf16><<<g, 256, 0, ST(s)>>>((const bf16*)dy, (const bf16*)y, (const bf16*)mask, (bf16*)dx, rows, n)));
  return OK();
}
extern "C" int hctr_layernorm_fwd(const void* x, const float* gamma, const float* beta, void* y, float* mean,
                                  float* rstd, long long rows, int n, float eps, int bf, void* s) {
  if (rows == 0) return 0;
  const unsigned g = gridx(rows * 32);
  DISPATCH_T(bf, (layernorm_fwd_kernel<float><<<g, 256, 0, ST(s)>>>((const float*)x, gamma, beta, (float*)y, mean, rstd, rows, n, eps)),
             (layernorm_fwd_kernel<bf16><<<g, 256, 0, ST(s)>>>((const bf16*)x, gamma, beta, (bf16*)y, mean, rstd, rows, n, eps)));
  return OK();
}
extern "C" int hctr_layernorm_bwd(const void* dy, const void* x, const float* gamma, const float* mean,
                                  const float* rstd, void* dx, float* dgamma, float* dbeta, long long rows, int n,
                                  int bf, void* s) {
  if (rows == 0) return 0;
  const unsigned g = gridx(rows * 32);
  if (dx) {
    DISPATCH_T(bf, (layernorm_bwd_dx_kernel<float><<<g, 256, 0, ST(s)>>>((const float*)dy, (const float*)x, gamma, mean, rstd, (float*)dx, rows, n)),
               (layernorm_bwd_dx_kernel<bf16><<<g, 256, 0, ST(s)>>>((const bf16*)dy, (const bf16*)x, gamma, mean, rstd, (bf16*)dx, rows, n)));
  }
  long long gy = (rows + 255) / 256;
  if (gy > 64) gy = 64;
  const dim3 gr((n + 31) / 32, static_cast<unsigned>(gy));
  DISPATCH_T(bf, (colreduce2_kernel<float, 2><<<gr, 256, 0, ST(s)>>>((const float*)x, (const float*)dy, mean, rstd, dbeta, dgamma, rows, n, 0.f)),
             (colreduce2_kernel<bf16, 2><<<gr, 256, 0, ST(s)>>>((const bf16*)x, (const bf16*)dy, mean, rstd, dbeta, dgamma, rows, n, 0.f)));
  return OK();
}

// mode: 0 stats (out0 = sum x, out1 = sum x^2), 1 BatchNorm grads, 3 Dice sums
extern "C" int hctr_colreduce2(const void* x, const void* dy, const float* m, const float* sc, float* out0,
                               float* out1, long long rows, int cols, float alpha, int mode, int bf, void* s) {
  if (rows == 0) return 0;
  long long gy = (rows + 255) / 256;
  if (gy > 64) gy = 64;
  const dim3 gr((cols + 31) / 32, static_cast<unsigned>(gy));
#define CR(T, M) colreduce2_kernel<T, M><<<gr, 256, 0, ST(s)>>>((const T*)x, (const T*)dy, m, sc, out0, out1, rows, cols, alpha)
  if (mode == 0) DISPATCH_T(bf, (CR(float, 0)), (CR(bf16, 0)));
  else if (mode == 1) DISPATCH_T(bf, (CR(float, 1)), (CR(bf16, 1)));
  else if (mode == 3) DISPATCH_T(bf, (CR(float, 3)), (CR(bf16, 3)));
  else return -2;
#undef CR
  return OK();
}
extern "C" int hctr_bn_finalize(const float* sum, const float* sumsq, float* mean, float* rstd, float* var_out,
                                float* run_mean, float* run_var, int cols, long long n, float eps, float momentum,
                                void* s) {
  bn_finalize_kernel<<<(cols + 255) / 256, 256, 0, ST(s)>>>(sum, sumsq, mean, rstd, var_out, run_mean, run_var, cols,
                                                             1.f / static_cast<float>(n), eps, momentum);
  return OK();
}
// op: 0 bn fwd (p0 = gamma, p1 = beta), 2 dice fwd, 3 dice bwd (p0 = A, p1 = B)
extern "C" int hctr_colwise(const void* x, const void* dy, const float* m, const float* sc, const float* p0,
                            const float* p1, void* out, long long rows, int cols, float alpha, int op, int bf,
                            void* s) {
  const long long total = rows * cols;
  if (total == 0) return 0;
  const unsigned g = grid1(total);
  const float inv_n = 1.f / static_cast<float>(rows);
#define CW(T, O) colwise_kernel<T, O><<<g, 256, 0, ST(s)>>>((const T*)x, (const T*)dy, m, sc, p0, p1, (T*)out, total, cols, alpha, inv_n)
  if (op == 0) DISPATCH_T(bf, (CW(float, 0)), (CW(bf16, 0)));
  else if (op == 2) DISPATCH_T(bf, (CW(float, 2)), (CW(bf16, 2)));
  else if (op == 3) DISPATCH_T(bf, (CW(float, 3)), (CW(bf16, 3)));
  else return -2;
#undef CW
  return OK();
}

namespace hctr {
// BatchNorm dx needs gamma AND rstd: dx = gamma * rstd * (dy - dbeta / N - xhat * dgamma / N)
template <typename T>
__global__ void __launch_bounds__(256)
    bn_bwd_dx_kernel(const T* __restrict__ x, const T* __restrict__ dy, const float* __restrict__ mean,
                     const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ dbeta,
                     const float* __restrict__ dgamma, T* __restrict__ dx, long long total, int cols, float inv_n) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % cols);
    const float xh = (ldf(x, i) - mean[c]) * rstd[c];
    stf(dx, i, gamma[c] * rstd[c] * (ldf(dy, i) - dbeta[c] * inv_n - xh * dgamma[c] * inv_n));
  }
}
}  // namespace hctr
extern "C" int hctr_bn_bwd_dx(const void* x, const void* dy, const float* mean, const float* rstd,
                              const float* gamma, const float* dbeta, const float* dgamma, void* dx, long long rows,
                              int cols, int bf, void* s) {
  const long long total = rows * cols;
  if (total == 0) return 0;
  const unsigned g = grid1(total);
  const float inv_n = 1.f / static_cast<float>(rows);
  DISPATCH_T(bf, (bn_bwd_dx_kernel<float><<<g, 256, 0, ST(s)>>>((const float*)x, (const float*)dy, mean, rstd, gamma, dbeta, dgamma, (float*)dx, total, cols, inv_n)),
             (bn_bwd_dx_kernel<bf16><<<g, 256, 0, ST(s)>>>((const bf16*)x, (const bf16*)dy, mean, rstd, gamma, dbeta, dgamma, (bf16*)dx, total, cols, inv_n)));
  return OK();
}

extern "C" int hctr_fm_order2(const void* x, const void* dy, void* out, long long b, int S, int D, int backward,
                              int bf, void* s) {
  if (b * D == 0) return 0;
  const unsigned g = gridx(b * D);
  if (!backward)
    DISPATCH_T(bf, (fm_order2_fwd_kernel<float><<<g, 256, 0, ST(s)>>>((const float*)x, (float*)out, b, S, D)),
               (fm_order2_fwd_kernel<bf16><<<g, 256, 0, ST(s)>>>((const bf16*)x, (bf16*)out, b, S, D)));
  else
    DISPATCH_T(bf, (fm_order2_bwd_kernel<float><<<g, 256, 0, ST(s)>>>((const float*)x, (const float*)dy, (float*)out, b, S, D)),
               (fm_order2_bwd_kernel<bf16><<<g, 256, 0, ST(s)>>>((const bf16*)x, (const bf16*)dy, (bf16*)out, b, S, D)));
  return OK();
}
extern "C" int hctr_weight_mul_fwd(const void* x, const float* w, void* y, long long b, int S, int V, int bf, void* s) {
  const long long total = b * S * V;
  if (total == 0) return 0;
  DISPATCH_T(bf, (weight_mul_fwd_kernel<float><<<grid1(total), 256, 0, ST(s)>>>((const float*)x, w, (float*)y, total, S, V)),
             (weight_mul_fwd_kernel<bf16><<<grid1(total), 256, 0, ST(s)>>>((const bf16*)x, w, (bf16*)y, total, S, V)));
  return OK();
}
extern "C" int hctr_weight_mul_bwd(const void* dy, const void* x, const float* w, void* dx, float* dw, long long b,
                                   int S, int V, int bf, void* s) {
  if (b == 0) return 0;
  if (dx) {
    DISPATCH_T(bf, (weight_mul_bwd_dx_kernel<float><<<gridx(b * S), 256, 0, ST(s)>>>((const float*)dy, w, (float*)dx, b * S, S, V)),
               (weight_mul_bwd_dx_kernel<bf16><<<gridx(b * S), 256, 0, ST(s)>>>((const bf16*)dy, w, (bf16*)dx, b * S, S, V)));
  }
  long long gy = (b + 127) / 128;
  if (gy > 128) gy = 128;
  const dim3 gr((S * V + 255) / 256, static_cast<unsigned>(gy));
  DISPATCH_T(bf, (weight_mul_bwd_dw_kernel<float><<<gr, 256, 0, ST(s)>>>((const float*)dy, (const float*)x, dw, b, S, V)),
             (weight_mul_bwd_dw_kernel<bf16><<<gr, 256, 0, ST(s)>>>((const bf16*)dy, (const bf16*)x, dw, b, S, V)));
  return OK();
}
extern "C" int hctr_reduce_mid(const void* in, void* out, long long outer, int R, long long inner, float scale,
                               int backward, int bf, void* s) {
  if (outer * inner == 0) return 0;
  if (!backward)
    DISPATCH_T(bf, (reduce_mid_fwd_kernel<float><<<gridx(outer * inner), 256, 0, ST(s)>>>((const float*)in, (float*)out, outer, R, inner, scale)),
               (reduce_mid_fwd_kernel<bf16><<<gridx(outer * inner), 256, 0, ST(s)>>>((const bf16*)in, (bf16*)out, outer, R, inner, scale)));
  else
    DISPATCH_T(bf, (reduce_mid_bwd_kernel<float><<<gridx(outer * R * inner), 256, 0, ST(s)>>>((const float*)in, (float*)out, outer, R, inner, scale)),
               (reduce_mid_bwd_kernel<bf16><<<gridx(outer * R * inner), 256, 0, ST(s)>>>((const bf16*)in, (bf16*)out, outer, R, inner, scale)));
  return OK();
}
extern "C" int hctr_copy4d(const void* src, void* dst, const long long* dims, const long long* sstr,
                           const long long* dstr, int accumulate, int elem_bytes, void* s) {
  Copy4D c;
  long long total = 1;
  for (int i = 0; i < 4; ++i) {
    c.d[i] = dims[i];
    c.ss[i] = sstr[i];
    c.ds[i] = dstr[i];
    total *= dims[i];
  }
  if (total == 0) return 0;
  if (elem_bytes == 2) copy4d_kernel<bf16><<<grid1(total), 256, 0, ST(s)>>>((const bf16*)src, (bf16*)dst, c, accumulate);
  else if (elem_bytes == 4) copy4d_kernel<float><<<grid1(total), 256, 0, ST(s)>>>((const float*)src, (float*)dst, c, accumulate);
  else return -2;
  return OK();
}
extern "C" int hctr_abi_size_bmm() { return static_cast<int>(sizeof(BmmDesc)); }
// dtype codes: 0 = fp32, 1 = bf16 for a / b / c
extern "C" int hctr_bmm(const void* A, const void* B, void* C, const BmmDesc* d, int Z0, int ta, int tb, int tc,
                        void* s) {
  if (d->M == 0 || d->N == 0 || Z0 * d->Z1 == 0) return 0;
  const dim3 g((d->N + 15) / 16, (d->M + 15) / 16, Z0 * d->Z1);
#define BM(TA, TB, TC) bmm_kernel<TA, TB, TC><<<g, 256, 0, ST(s)>>>((const TA*)A, (const TB*)B, (TC*)C, *d)
  const int code = ta * 4 + tb * 2 + tc;
  switch (code) {
    case 0: BM(float, float, float); break;
    case 1: BM(float, float, bf16); break;
    case 2: BM(float, bf16, float); break;
    case 3: BM(float, bf16, bf16); break;
    case 4: BM(bf16, float, float); break;
    case 5: BM(bf16, float, bf16); break;
    case 6: BM(bf16, bf16, float); break;
    default: BM(bf16, bf16, bf16); break;
  }
#undef BM
  return OK();
}
extern "C" int hctr_gru_gate(const float* a0, const float* a1, const float* a2, const float* a3, float* o0, float* o1,
                             float* o2, long long b, int H, int backward, void* s) {
  if (b * H == 0) return 0;
  if (!backward) gru_gate_fwd_kernel<<<gridx(b * H), 256, 0, ST(s)>>>(a0, a1, a2, o0, o1, b, H);
  else gru_gate_bwd_kernel<<<gridx(b * H), 256, 0, ST(s)>>>(a0, a1, a2, a3, o0, o1, o2, b, H);
  return OK();
}
