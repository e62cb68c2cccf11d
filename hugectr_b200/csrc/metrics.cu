// Device side of the distributed exact AUC (hugectr_b200/metrics.py).  Pipeline per evaluation round, the
// GPU reading of the reference's histogram -> pivots -> all-to-all -> local sort -> halo pipeline
// (HugeCTR/src/metrics.cu:1017-1240):
//   1. auc_hist_kernel       every rank bins its (prediction, label) pairs by an order-preserving 20-bit key
//                            of the fp32 prediction into positive / negative histograms (2 x 4 MB)
//   2. all-reduce of the histograms; a prefix sum assigns contiguous bin ranges to ranks so that every rank
//      receives ~N/W pairs (ties share a bin, hence a rank: no halo exchange is needed afterwards)
//   3. auc_partition_kernel  counting-sort scatter of the local pairs into per-destination segments of the
//                            send buffer (warp-aggregated cursors), then one variable-size all-to-all
//   4. local sort + tie-aware rank statistic on N/W elements per rank, scalar all-reduce of the partial areas.
// Memory per rank is O(N / W) + the histograms, never the whole evaluation set.
#include <cuda_runtime.h>
#include <stdint.h>

#include "ptx.cuh"

namespace hctr {

__device__ __forceinline__ unsigned int ordered_key(float f) {
  const unsigned int u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);     // monotone: a < b  <=>  key(a) < key(b)
}

__global__ void __launch_bounds__(256)
    auc_hist_kernel(const float* __restrict__ pred, const float* __restrict__ label, long long n,
                    unsigned int* __restrict__ hist_pos, unsigned int* __restrict__ hist_neg, int shift) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const unsigned int b = ordered_key(pred[i]) >> shift;
    atomicAdd((label[i] > 0.5f ? hist_pos : hist_neg) + b, 1u);
  }
}

// cursors[d] starts at the first slot of destination d's segment in the send buffer
__global__ void __launch_bounds__(256)
    auc_partition_kernel(const float* __restrict__ pred, const float* __restrict__ label, long long n,
                         const unsigned char* __restrict__ bin2dst, unsigned int* __restrict__ cursors,
                         float* __restrict__ send_pred, float* __restrict__ send_label, int shift) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long n_round = (n + 31) / 32 * 32;
  const unsigned int lane = threadIdx.x & 31u;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_round; i += stride) {
    const bool act = i < n;
    float p = 0.f, y = 0.f;
    unsigned int d = 0xFFu;
    if (act) {
      p = pred[i];
      y = label[i];
      d = bin2dst[ordered_key(p) >> shift];
    }
    // warp-aggregated reservation: one atomic per distinct destination in the warp
    const unsigned int peers = __match_any_sync(0xffffffffu, d);
    const unsigned int leader = __ffs(peers) - 1;
    unsigned int base = 0;
    if (act && lane == leader) base = atomicAdd(cursors + d, static_cast<unsigned int>(__popc(peers)));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (act) {
      const unsigned int pos = base + __popc(peers & ((1u << lane) - 1u));
      send_pred[pos] = p;
      send_label[pos] = y;
    }
  }
}

}  // namespace hctr

using namespace hctr;

extern "C" int hctr_auc_hist(const float* pred, const float* label, long long n, void* hist_pos,
                             void* hist_neg, int bits, void* stream) {
  if (n <= 0) return 0;
  long long blocks = (n + 255) / 256;
  if (blocks > hctr::num_sms() * 16) blocks = hctr::num_sms() * 16;
  auc_hist_kernel<<<static_cast<unsigned>(blocks), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      pred, label, n, reinterpret_cast<unsigned int*>(hist_pos), reinterpret_cast<unsigned int*>(hist_neg),
      32 - bits);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

extern "C" int hctr_auc_partition(const float* pred, const float* label, long long n, const void* bin2dst,
                                  void* cursors, float* send_pred, float* send_label, int bits,
                                  void* stream) {
  if (n <= 0) return 0;
  long long blocks = (n + 255) / 256;
  if (blocks > hctr::num_sms() * 16) blocks = hctr::num_sms() * 16;
  auc_partition_kernel<<<static_cast<unsigned>(blocks), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      pred, label, n, reinterpret_cast<const unsigned char*>(bin2dst), reinterpret_cast<unsigned int*>(cursors),
      send_pred, send_label, 32 - bits);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
