// Decay of the admission sketches (admit_sketch.cuh): with admit_decay_steps = P > 0, every counter is
// halved (rounding down) at the start of each training step whose clock is a multiple of P.  One launch
// per sketch per training step; it reads the clock from device memory, so the step graph replays it.
#include <cuda_runtime.h>
#include <stdint.h>

#include "admit_sketch.cuh"

namespace hctr {

__global__ void __launch_bounds__(256) admit_decay_kernel(uint4* __restrict__ c, long long n4,
                                                          const unsigned long long* clock,
                                                          unsigned long long period) {
  if (*clock % period != 0) return;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    uint4 v = c[i];
    v.x >>= 1;
    v.y >>= 1;
    v.z >>= 1;
    v.w >>= 1;
    c[i] = v;
  }
}

}  // namespace hctr

using namespace hctr;

// n: counters of the sketch (a multiple of 4, 16-byte aligned)
extern "C" int hctr_admit_decay(void* counters, long long n, const void* clock, unsigned long long period,
                                void* stream) {
  if (n <= 0 || period == 0 || (n & 3)) return n & 3 ? -1 : 0;
  const long long n4 = n / 4;
  const long long blocks = (n4 + 255) / 256;
  admit_decay_kernel<<<(unsigned)(blocks < 1056 ? blocks : 1056), 256, 0, (cudaStream_t)stream>>>(
      static_cast<uint4*>(counters), n4, static_cast<const unsigned long long*>(clock), period);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
