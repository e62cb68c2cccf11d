// Element-wise optimizer rules shared by the dense optimizer (dense_ops.cu) and the fused sparse-update
// kernels (embedding.cu / embedding_bwd.cu): one definition of each rule and of its hyper-parameters.
// Mirrored on the host by ops/optim.py (OPT_CODE, COptHyper, opt_reference).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "ptx.cuh"

namespace hctr {

template <typename T>
HCTR_DEVICE void store_vec4(T* p, float a, float b, float c, float d);
template <>
HCTR_DEVICE void store_vec4<float>(float* p, float a, float b, float c, float d) {
  *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d);
}
template <>
HCTR_DEVICE void store_vec4<__nv_bfloat16>(__nv_bfloat16* p, float a, float b, float c, float d) {
  *reinterpret_cast<uint2*>(p) = make_uint2(pack_bf16x2(a, b), pack_bf16x2(c, d));
}
template <typename T>
HCTR_DEVICE float4 load_vec4(const T* p);
template <>
HCTR_DEVICE float4 load_vec4<float>(const float* p) {
  return *reinterpret_cast<const float4*>(p);
}
template <>
HCTR_DEVICE float4 load_vec4<__nv_bfloat16>(const __nv_bfloat16* p) {
  const uint2 v = *reinterpret_cast<const uint2*>(p);
  return make_float4(bf16_lo(v.x), bf16_hi(v.x), bf16_lo(v.y), bf16_hi(v.y));
}
template <typename T>
HCTR_DEVICE float to_f(T v);
template <>
HCTR_DEVICE float to_f<float>(float v) { return v; }
template <>
HCTR_DEVICE float to_f<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T>
HCTR_DEVICE T from_f(float v);
template <>
HCTR_DEVICE float from_f<float>(float v) { return v; }
template <>
HCTR_DEVICE __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16(v); }

// ------------------------------------------------------------------ optimizer rules
enum SparseOpt : int { OPT_SGD = 0, OPT_ADAGRAD, OPT_ADAM, OPT_FTRL, OPT_MOMENTUM, OPT_NESTEROV,
                       OPT_RMSPROP, OPT_ROWWISE_ADAGRAD, OPT_PARTIAL_ROWWISE_ADAM };

struct OptHyper {
  const float* lr_ptr;    // device learning rate (graph friendly)
  float lr_scale;         // extra multiplier (1)
  float scaler;           // loss scaler: g /= scaler
  float beta1, beta2, epsilon;
  float lambda1, lambda2, ftrl_beta;
  float momentum;
  float initial_accu;
  const unsigned int* step_ptr;  // device step counter (Adam bias correction), 1-based
  unsigned int sr_seed;          // seed of the stochastic rounding of bf16 weights (sr_step_key)
  unsigned int pad_;
};

// Scalars every element of one optimizer step shares: the learning rate and Adam's bias corrections
// (1 elsewhere).  A null lr_ptr / step_ptr reads as learning rate 1 / step 1.
struct OptStep {
  float lr, bc1, bc2;
};
template <int OPT>
HCTR_DEVICE OptStep opt_step(const OptHyper& hp) {
  OptStep st = {(hp.lr_ptr ? *hp.lr_ptr : 1.f) * hp.lr_scale, 1.f, 1.f};
  if constexpr (OPT == OPT_ADAM || OPT == OPT_PARTIAL_ROWWISE_ADAM) {
    const float t = static_cast<float>(hp.step_ptr ? *hp.step_ptr : 1u);
    st.bc1 = 1.f - powf(hp.beta1, t);
    st.bc2 = 1.f - powf(hp.beta2, t);
  }
  return st;
}

template <int OPT, typename StateT>
HCTR_DEVICE void apply_opt(float& w, float g, StateT* s0, StateT* s1, long long idx,
                           const OptHyper& hp, const OptStep& st) {
  const float lr = st.lr;
  if constexpr (OPT == OPT_SGD) {
    w -= lr * g;
  } else if constexpr (OPT == OPT_ADAGRAD) {
    float a = to_f<StateT>(s0[idx]) + g * g;
    s0[idx] = from_f<StateT>(a);
    w -= lr * g / (sqrtf(a) + hp.epsilon);
  } else if constexpr (OPT == OPT_ADAM) {
    float m = hp.beta1 * to_f<StateT>(s0[idx]) + (1.f - hp.beta1) * g;
    float v = hp.beta2 * to_f<StateT>(s1[idx]) + (1.f - hp.beta2) * g * g;
    s0[idx] = from_f<StateT>(m);
    s1[idx] = from_f<StateT>(v);
    const float alpha = lr * sqrtf(st.bc2) / st.bc1;
    w -= alpha * m / (sqrtf(v) + hp.epsilon);
  } else if constexpr (OPT == OPT_FTRL) {
    // state0 = z, state1 = n (reference ftrl_optimizer.cu:28-42)
    const float n = to_f<StateT>(s1[idx]);
    const float n_new = n + g * g;
    const float ef = hp.ftrl_beta;
    float z = to_f<StateT>(s0[idx]) + g + (sqrtf(n + ef) - sqrtf(n_new + ef)) * w / lr;
    s0[idx] = from_f<StateT>(z);
    s1[idx] = from_f<StateT>(n_new);
    const float p = (z > 0.f ? 1.f : -1.f) * hp.lambda1 - z;
    const float q = sqrtf(n_new + ef) / lr + hp.lambda2;
    w = (fabsf(z) > hp.lambda1) ? p / q : 0.f;
  } else if constexpr (OPT == OPT_MOMENTUM) {
    float m = hp.momentum * to_f<StateT>(s0[idx]) - lr * g;
    s0[idx] = from_f<StateT>(m);
    w += m;
  } else if constexpr (OPT == OPT_NESTEROV) {
    const float a = to_f<StateT>(s0[idx]);
    const float a_new = hp.momentum * a - lr * g;
    s0[idx] = from_f<StateT>(a_new);
    w += -hp.momentum * a + (1.f + hp.momentum) * a_new;
  } else if constexpr (OPT == OPT_RMSPROP) {
    float v = hp.beta2 * to_f<StateT>(s0[idx]) + (1.f - hp.beta2) * g * g;
    s0[idx] = from_f<StateT>(v);
    w -= lr * g / (sqrtf(v) + hp.epsilon);
  }
}

// 4-wide variant: optimizer state is loaded / stored as one vector (16 B fp32, 8 B bf16) instead of
// four scalar accesses per lane.
template <int OPT, typename StateT>
HCTR_DEVICE void apply_opt4(float4& w, const float4 g, StateT* s0, StateT* s1, long long idx,
                            const OptHyper& hp, const OptStep& st) {
  constexpr bool kHasS0 = (OPT != OPT_SGD);
  constexpr bool kHasS1 = (OPT == OPT_ADAM || OPT == OPT_FTRL);
  float a[4] = {0.f, 0.f, 0.f, 0.f}, b[4] = {0.f, 0.f, 0.f, 0.f};
  if constexpr (kHasS0) {
    const float4 v = load_vec4<StateT>(s0 + idx);
    a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w;
  }
  if constexpr (kHasS1) {
    const float4 v = load_vec4<StateT>(s1 + idx);
    b[0] = v.x; b[1] = v.y; b[2] = v.z; b[3] = v.w;
  }
  float ww[4] = {w.x, w.y, w.z, w.w};
  const float gg[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    // run the scalar rule on local copies of the state
    float sa = a[j], sb = b[j];
    apply_opt<OPT, float>(ww[j], gg[j], &sa, &sb, 0, hp, st);
    a[j] = sa; b[j] = sb;
  }
  w = make_float4(ww[0], ww[1], ww[2], ww[3]);
  if constexpr (kHasS0) store_vec4<StateT>(s0 + idx, a[0], a[1], a[2], a[3]);
  if constexpr (kHasS1) store_vec4<StateT>(s1 + idx, b[0], b[1], b[2], b[3]);
}

// variant with the weight / first state vector already in registers (loaded early by the caller so
// their latency overlaps the gradient gather); the caller stores w, this stores the states.
template <int OPT, typename StateT>
HCTR_DEVICE void apply_opt4_pre(float4& w, const float4 g, const float4 s0v, StateT* s0, StateT* s1,
                                long long idx, const OptHyper& hp, const OptStep& st) {
  constexpr bool kHasS0 = (OPT != OPT_SGD);
  constexpr bool kHasS1 = (OPT == OPT_ADAM || OPT == OPT_FTRL);
  float a[4] = {s0v.x, s0v.y, s0v.z, s0v.w}, b[4] = {0.f, 0.f, 0.f, 0.f};
  if constexpr (kHasS1) {
    const float4 v = load_vec4<StateT>(s1 + idx);
    b[0] = v.x; b[1] = v.y; b[2] = v.z; b[3] = v.w;
  }
  float ww[4] = {w.x, w.y, w.z, w.w};
  const float gg[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float sa = a[j], sb = b[j];
    apply_opt<OPT, float>(ww[j], gg[j], &sa, &sb, 0, hp, st);
    a[j] = sa; b[j] = sb;
  }
  w = make_float4(ww[0], ww[1], ww[2], ww[3]);
  if constexpr (kHasS0) store_vec4<StateT>(s0 + idx, a[0], a[1], a[2], a[3]);
  if constexpr (kHasS1) store_vec4<StateT>(s1 + idx, b[0], b[1], b[2], b[3]);
}

// Row-wise AdaGrad (OPT_ROWWISE_ADAGRAD): ONE fp32 accumulator per row, s[row] (never bf16).
//   s += (1/ev) * sum_c g[c]^2 ;  w[c] -= lr * g[c] / (sqrt(s) + eps)  for every column of the row
// The caller reduces sum_c g[c]^2 over the whole row first (row_reduce_step over the row's lanes, or
// its own block reduction followed by rowwise_state_step), and applies the returned factor
// f = lr / (sqrt(s) + eps) to every column.  Square root and divisions round to nearest even whatever the fast-math flags, so a row
// whose update is exact in fp32 is reproduced bit for bit by the CPU path (ops/optim.py).
HCTR_DEVICE float rowwise_accumulate(float s, float sumsq, int ev) {
  return s + __fdiv_rn(sumsq, static_cast<float>(ev));
}
HCTR_DEVICE float rowwise_factor(float s_new, const OptHyper& hp, float lr) {
  return __fdiv_rn(lr, __fsqrt_rn(s_new) + hp.epsilon);
}
// one thread per row: *s = s_old + sumsq / ev, returns the row's factor
HCTR_DEVICE float rowwise_state_step(float s_old, float sumsq, float* s, int ev, const OptHyper& hp, float lr) {
  const float s_new = rowwise_accumulate(s_old, sumsq, ev);
  *s = s_new;
  return rowwise_factor(s_new, hp, lr);
}
HCTR_DEVICE void apply_rowwise4(float4& w, const float4 g, float f) {
  w.x -= f * g.x; w.y -= f * g.y; w.z -= f * g.z; w.w -= f * g.w;
}
HCTR_DEVICE float sumsq4(const float4 g) { return g.x * g.x + g.y * g.y + g.z * g.z + g.w * g.w; }
HCTR_DEVICE float4 scale4(const float4 g, float a) { return make_float4(g.x * a, g.y * a, g.z * a, g.w * a); }

// Partial row-wise Adam (OPT_PARTIAL_ROWWISE_ADAM): the first moment m per element (state 0, StateT) and
// the second moment ONE fp32 value per row, v[row] (state 1, never bf16: an EMA of a small quantity would
// lose its increments).  For a row that receives gradients, t = the device step counter:
//   m[c] = b1 m[c] + (1 - b1) g[c] ;  v = b2 v + (1 - b2) (1/ev) sum_c g[c]^2
//   w[c] -= alpha m[c] / (sqrt(v) + eps),  alpha = lr sqrt(1 - b2^t) / (1 - b1^t)
// with Adam's bias correction and epsilon placement (apply_opt<OPT_ADAM>).  As for row-wise AdaGrad the
// caller reduces sum_c g[c]^2 over the whole row before it stores any weight or m of the row; the row step
// updates v once and returns the row's factor f = alpha / (sqrt(v) + eps), and the element step updates m
// and applies w -= f m.
HCTR_DEVICE float prow_adam_state_step(float v_old, float sumsq, float* v, int ev, const OptHyper& hp,
                                       const OptStep& st) {
  const float v_new = hp.beta2 * v_old + (1.f - hp.beta2) * __fdiv_rn(sumsq, static_cast<float>(ev));
  *v = v_new;
  const float alpha = st.lr * sqrtf(st.bc2) / st.bc1;   // as apply_opt<OPT_ADAM>
  return __fdiv_rn(alpha, __fsqrt_rn(v_new) + hp.epsilon);
}
template <typename StateT>
HCTR_DEVICE void prow_adam_step4(float4& w, const float4 g, StateT* m, const OptHyper& hp, float f) {
  float4 a = load_vec4<StateT>(m);
  const float c = 1.f - hp.beta1;
  a.x = hp.beta1 * a.x + c * g.x; a.y = hp.beta1 * a.y + c * g.y;
  a.z = hp.beta1 * a.z + c * g.z; a.w = hp.beta1 * a.w + c * g.w;
  store_vec4<StateT>(m, a.x, a.y, a.z, a.w);
  w.x -= f * a.x; w.y -= f * a.y; w.z -= f * a.z; w.w -= f * a.w;
}
template <typename StateT>
HCTR_DEVICE void prow_adam_step1(float& w, float g, StateT* m, const OptHyper& hp, float f) {
  const float a = hp.beta1 * to_f<StateT>(*m) + (1.f - hp.beta1) * g;
  *m = from_f<StateT>(a);
  w -= f * a;
}

// The two row-reduced rules behind one interface, for the kernels that hold a whole row's sum of g^2
// before they store any of it: the fp32 row state (row-wise AdaGrad: s0 [rows]; partial row-wise Adam:
// s1 [rows], whatever StateT is), the row step of one thread (row_state_step) or of the lanes that own
// the row (row_reduce_step), and the element steps (row_apply4 / row_apply1) on the gradient g of arena
// element idx with the row's factor f.
template <int OPT>
constexpr bool kRowRule = (OPT == OPT_ROWWISE_ADAGRAD || OPT == OPT_PARTIAL_ROWWISE_ADAM);
template <int OPT, typename StateT>
HCTR_DEVICE float* row_state(StateT* s0, StateT* s1) {
  if constexpr (OPT == OPT_ROWWISE_ADAGRAD) return reinterpret_cast<float*>(s0);
  else return reinterpret_cast<float*>(s1);
}
template <int OPT>
HCTR_DEVICE float row_state_step(float s_old, float sumsq, float* s, int ev, const OptHyper& hp, const OptStep& st) {
  if constexpr (OPT == OPT_ROWWISE_ADAGRAD) return rowwise_state_step(s_old, sumsq, s, ev, hp, st.lr);
  else return prow_adam_state_step(s_old, sumsq, s, ev, hp, st);
}
// The WIDTH lanes of `mask` (a power of two, aligned) own one row and hold partial sums of g^2 in sq;
// lane `leader`, the first of them, has s_old = *s (loaded early by the caller) and updates *s.  Every
// lane returns the row's factor.
template <int OPT, int WIDTH>
HCTR_DEVICE float row_reduce_step(unsigned int mask, int leader, int lane, float sq, float s_old, float* s,
                                  int ev, const OptHyper& hp, const OptStep& st) {
#pragma unroll
  for (int o = WIDTH / 2; o > 0; o >>= 1) sq += __shfl_xor_sync(mask, sq, o);
  float f = 0.f;
  if (lane == leader) f = row_state_step<OPT>(s_old, sq, s, ev, hp, st);
  return __shfl_sync(mask, f, leader);
}
template <int OPT, typename StateT>
HCTR_DEVICE void row_apply4(float4& w, const float4 g, float f, StateT* s0, long long idx, const OptHyper& hp) {
  if constexpr (OPT == OPT_ROWWISE_ADAGRAD) apply_rowwise4(w, g, f);
  else prow_adam_step4<StateT>(w, g, s0 + idx, hp, f);
}
template <int OPT, typename StateT>
HCTR_DEVICE void row_apply1(float& w, float g, float f, StateT* s0, long long idx, const OptHyper& hp) {
  if constexpr (OPT == OPT_ROWWISE_ADAGRAD) w -= f * g;
  else prow_adam_step1<StateT>(w, g, s0 + idx, hp, f);
}

}  // namespace hctr
