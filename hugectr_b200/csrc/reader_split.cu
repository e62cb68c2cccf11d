// Device side of the RawAsync reader (C13): one kernel splits a batch of raw fixed-size records that was copied to
// the device as ONE contiguous block into the model's input tensors
//   record = [label_dim x 4 B][dense_dim x 4 B][sum(hotness) x key bytes]
//   label [b, L] fp32 (int32 -> float; stored floats when flag bit 1 is set), dense [b, D] fp32 (log(x + 1) of
//   integer features; the stored floats when flag bit 0 is set), keys FEATURE-major: feature f at keys[key_off[f] + s * hot[f] + h]
// Reference: HugeCTR/src/data_readers/multi_hot/split_batch.cu:43-88 (one thread per record column, per-column
// bucket tables); here the column -> (feature, position) tables sit in shared memory and the keys land directly in
// the embedding collection's key slab (no per-feature tensors, no second copy).
#include <cuda_runtime.h>
#include <stdint.h>

#include "ptx.cuh"

namespace hctr {

struct SplitDesc {
  const uint8_t* raw;      // [b, rec_bytes] (device), starts at the first record
  float* label;
  float* dense;
  void* keys;
  const int* col_feat;     // [sparse cols] feature of the column
  const int* col_pos;      // [sparse cols] position inside the feature's bag
  const long long* key_off;  // [features] element offset of the feature's block in `keys`
  const int* hot;          // [features]
  int batch, valid, label_dim, dense_dim, sparse_cols, rec_bytes;
  int key_bytes_in, key_bytes_out, dense_is_float;
};

__global__ void __launch_bounds__(256) raw_split_kernel(const SplitDesc d) {
  extern __shared__ int sh[];
  int* s_feat = sh;
  int* s_pos = sh + d.sparse_cols;
  for (int i = threadIdx.x; i < d.sparse_cols; i += blockDim.x) {
    s_feat[i] = d.col_feat[i];
    s_pos[i] = d.col_pos[i];
  }
  __syncthreads();
  const int cols = d.label_dim + d.dense_dim + d.sparse_cols;
  const long long total = static_cast<long long>(d.batch) * cols;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int s = static_cast<int>(i / cols);
    const int c = static_cast<int>(i - static_cast<long long>(s) * cols);
    const bool ok = s < d.valid;                    // incomplete last batch: padding rows
    const uint8_t* rec = d.raw + static_cast<long long>(ok ? s : 0) * d.rec_bytes;
    if (c < d.label_dim) {
      float v = 0.f;
      if (ok) {
        const uint32_t w = *reinterpret_cast<const uint32_t*>(rec + 4 * c);
        v = (d.dense_is_float & 2) ? __uint_as_float(w) : static_cast<float>(static_cast<int>(w));
      }
      d.label[static_cast<long long>(s) * d.label_dim + c] = v;
    } else if (c < d.label_dim + d.dense_dim) {
      float v = 0.f;
      if (ok) {
        const uint32_t w = *reinterpret_cast<const uint32_t*>(rec + 4 * c);
        v = (d.dense_is_float & 1) ? __uint_as_float(w) : logf(static_cast<float>(w) + 1.f);
      }
      d.dense[static_cast<long long>(s) * d.dense_dim + (c - d.label_dim)] = v;
    } else {
      const int sc = c - d.label_dim - d.dense_dim;
      const int f = s_feat[sc];
      long long k = -1;
      if (ok) {
        const uint8_t* kp = rec + 4 * (d.label_dim + d.dense_dim) + static_cast<long long>(sc) * d.key_bytes_in;
        k = d.key_bytes_in == 4 ? static_cast<long long>(*reinterpret_cast<const uint32_t*>(kp))
                                : *reinterpret_cast<const long long*>(kp);
      }
      const long long o = d.key_off[f] + static_cast<long long>(s) * d.hot[f] + s_pos[sc];
      if (d.key_bytes_out == 4) reinterpret_cast<int*>(d.keys)[o] = static_cast<int>(k);
      else reinterpret_cast<long long*>(d.keys)[o] = k;
    }
  }
}

}  // namespace hctr

extern "C" int hctr_raw_split(const void* raw, void* label, void* dense, void* keys, const int* col_feat,
                              const int* col_pos, const long long* key_off, const int* hot, int batch, int valid,
                              int label_dim, int dense_dim, int sparse_cols, int rec_bytes, int key_bytes_in,
                              int key_bytes_out, int dense_is_float, void* stream) {
  if (batch <= 0) return 0;
  hctr::SplitDesc d{reinterpret_cast<const uint8_t*>(raw), reinterpret_cast<float*>(label),
                    reinterpret_cast<float*>(dense), keys, col_feat, col_pos, key_off, hot, batch, valid, label_dim,
                    dense_dim, sparse_cols, rec_bytes, key_bytes_in, key_bytes_out, dense_is_float};
  const long long total = static_cast<long long>(batch) * (label_dim + dense_dim + sparse_cols);
  long long blocks = (total + 255) / 256;
  if (blocks > hctr::num_sms() * 8) blocks = hctr::num_sms() * 8;
  hctr::raw_split_kernel<<<static_cast<unsigned>(blocks), 256, 2 * sparse_cols * sizeof(int),
                           reinterpret_cast<cudaStream_t>(stream)>>>(d);
  return cudaGetLastError() == cudaSuccess ? 0 : -1;
}
