// Hopper (sm_90a) PTX wrappers: mbarrier, TMA, clusters, wgmma (wgmma.cuh), peer-memory ld/st.
// Hand-written inline PTX; no CUTLASS dependency.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace hctr {

#define HCTR_DEVICE __device__ __forceinline__

HCTR_DEVICE uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// Exponent e of the power-of-two scale of a block (or row) of e4m3 values whose largest magnitude is amax >= 0:
// the smallest 2^e with amax / 2^e <= 448 (e4m3 max), clamped to [-127, 127]; -127 when amax == 0.
// Integer arithmetic on the bits of amax = m * 2^ex (m in [0.5, 1)): 448 = 0.875 * 2^9, so e = ex - 9 + (m > 0.875).
// A float multiply (amax * (1 / 448)) flushes to zero under --use_fast_math for amax below 448 * 2^-126; amax below
// 2^-126 gives e < -127 anyway.  Mirrored by ops/mxfp8.py::e4m3_scale_exponent.
HCTR_DEVICE int e4m3_scale_exp(float amax) {
  const uint32_t b = __float_as_uint(amax);
  if (b < 0x00800000u) return -127;                               // zero or subnormal
  const int e = static_cast<int>(b >> 23) - 126 - 9 + ((b & 0x7fffffu) > 0x600000u);
  return min(127, max(-127, e));
}

// x * 2^-e for an e4m3_scale_exp exponent e, rounded once as IEEE fp32 (subnormal operands and results kept):
// fast math turns every fp32 multiply, __fmul_rn included, into mul.ftz, which would zero x below 2^-126.
HCTR_DEVICE float e4m3_scale_down(float x, int e) {
  float r;
  asm("mul.rn.f32 %0, %1, %2;" : "=f"(r) : "f"(x), "f"(__uint_as_float(static_cast<uint32_t>(127 - e) << 23)));
  return r;
}

HCTR_DEVICE uint32_t lane_id() {
  uint32_t l;
  asm volatile("mov.u32 %0, %%laneid;" : "=r"(l));
  return l;
}

HCTR_DEVICE bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// streaming multiprocessors of the current device: grid size of persistent / grid-stride kernels
inline int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
  }
  return n;
}

// ---------------------------------------------------------------- mbarrier
HCTR_DEVICE void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
HCTR_DEVICE void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
HCTR_DEVICE void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

HCTR_DEVICE void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
HCTR_DEVICE void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
HCTR_DEVICE bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
HCTR_DEVICE void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ---------------------------------------------------------------- TMA
HCTR_DEVICE void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2D tile load global -> shared, completion on mbarrier (complete_tx::bytes)
HCTR_DEVICE void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, "
      "{%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// multicast variant: the tile lands at the same CTA-relative smem offset of every CTA in cta_mask and
// performs complete_tx on the mbarrier at the same offset in each of them
HCTR_DEVICE void tma_load_2d_mc(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster "
      "[%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}
// 2D tile store shared -> global, tracked by this thread's bulk async-groups (out-of-bounds parts are not written)
HCTR_DEVICE void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
HCTR_DEVICE void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's bulk groups still read their shared-memory source
template <int N>
HCTR_DEVICE void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// at most N of this thread's bulk groups are still in flight (writes included)
template <int N>
HCTR_DEVICE void bulk_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
HCTR_DEVICE uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
HCTR_DEVICE void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `cta` of the cluster.  Release at CTA scope (the
// default): the arrival only reports that this thread's reads of a stage are done, which is ordered before the
// peer's next TMA write into it by the barrier itself.  A .release.cluster arrive compiles to a GPU-wide memory
// barrier (MEMBAR.ALL.GPU) ahead of every arrival, i.e. once per consumer warp and k block of the GEMM main loop.
HCTR_DEVICE void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t"
      ".reg .b32 remote;\n\t"
      "mapa.shared::cluster.u32 remote, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [remote];\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(cta)
      : "memory");
}

// ------------------------------------------------------- misc
HCTR_DEVICE uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
HCTR_DEVICE float bf16_lo(uint32_t v) { return __uint_as_float(v << 16); }
HCTR_DEVICE float bf16_hi(uint32_t v) { return __uint_as_float(v & 0xFFFF0000u); }

// system-scope release/acquire for cross-GPU flags in peer-mapped memory
HCTR_DEVICE void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
HCTR_DEVICE uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
HCTR_DEVICE uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
HCTR_DEVICE void red_add_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
HCTR_DEVICE int4 ld_nc_v4(const void* p) {
  int4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
HCTR_DEVICE void st_na_v4(void* p, const int4& v) {
  asm volatile("st.global.L1::no_allocate.v4.s32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

}  // namespace hctr

#include "wgmma.cuh"
