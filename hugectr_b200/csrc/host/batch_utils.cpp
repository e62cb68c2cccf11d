// Host-side batch assembly helpers shared by the file readers.
// hctr_csr_to_padded: one multi-hot (list) column of a row group slice, given as CSR offsets + values,
// scattered into the [b, S, H] key block of a batch (row stride S*H, -1 padding already in place) with
// bags truncated to H and the per-sample counts written to the [S, b] nnz block -- the CPU counterpart
// of the reference's dense/sparse column conversion kernels
// (HugeCTR/src/data_readers/parquet_data_converter.cu) done before the H2D copy, so the device
// receives the final layout.
#include <stdint.h>

// T = long long (keys, + add) or float (the per-key weights of a weighted input, add unused)
template <typename T>
static void csr_to_padded(const void* offs, int off_bytes, const T* vals, int n, int H, T add, T* out,
                          long long row_stride, int32_t* nnz) {
#pragma omp parallel for schedule(static) if (n > 2048)
  for (int i = 0; i < n; ++i) {
    long long lo, hi;
    if (off_bytes == 4) {
      lo = static_cast<const int32_t*>(offs)[i];
      hi = static_cast<const int32_t*>(offs)[i + 1];
    } else {
      lo = static_cast<const int64_t*>(offs)[i];
      hi = static_cast<const int64_t*>(offs)[i + 1];
    }
    long long c = hi - lo;
    if (c > H) c = H;
    if (c < 0) c = 0;
    T* o = out + static_cast<long long>(i) * row_stride;
    for (long long h = 0; h < c; ++h) o[h] = vals[lo + h] + add;
    if (nnz) nnz[i] = static_cast<int32_t>(c);
  }
}

extern "C" void hctr_csr_to_padded(const void* offs, int off_bytes, const long long* vals, int n, int H,
                                   long long add, long long* out, long long row_stride, int32_t* nnz) {
  csr_to_padded<long long>(offs, off_bytes, vals, n, H, add, out, row_stride, nnz);
}

// hctr_csr_to_padded_f32: the weight column of a weighted multi-hot slot into the [b, S, H] fp32 weight block, in
// the positions hctr_csr_to_padded gives the keys (0 padding already in place)
extern "C" void hctr_csr_to_padded_f32(const void* offs, int off_bytes, const float* vals, int n, int H, float* out,
                                       long long row_stride) {
  csr_to_padded<float>(offs, off_bytes, vals, n, H, 0.f, out, row_stride, nullptr);
}

// hctr_onehot_block: S one-hot (scalar) columns of a row-group slice -> the [b, S] key block of a batch in
// the model's key dtype, per-slot offset added, rows >= nloc padded with -1, and the [S, b] bag-length block.
// One call per block instead of S strided numpy stores under the GIL.
extern "C" void hctr_onehot_block(const long long* const* cols, const long long* add, int S, long long lo,
                                  long long nloc, long long b, void* keys_out, int key_bytes, int32_t* nnz) {
#pragma omp parallel for schedule(static) if (b > 2048)
  for (long long i = 0; i < b; ++i) {
    if (key_bytes == 8) {
      long long* o = static_cast<long long*>(keys_out) + i * S;
      for (int s = 0; s < S; ++s) o[s] = i < nloc ? cols[s][lo + i] + (add ? add[s] : 0) : -1;
    } else {
      int32_t* o = static_cast<int32_t*>(keys_out) + i * S;
      for (int s = 0; s < S; ++s)
        o[s] = i < nloc ? static_cast<int32_t>(cols[s][lo + i] + (add ? add[s] : 0)) : -1;
    }
  }
  for (int s = 0; s < S; ++s) {
    int32_t* z = nnz + static_cast<long long>(s) * b;
    for (long long i = 0; i < b; ++i) z[i] = i < nloc ? 1 : 0;
  }
}

// hctr_rows_f32: dst[b, w] = src[lo:lo+nloc, w] (float32), zero rows behind nloc
extern "C" void hctr_rows_f32(const float* src, long long lo, long long nloc, long long b, int w, float* dst) {
  for (long long i = 0; i < b * w; ++i) dst[i] = i < nloc * w ? src[lo * w + i] : 0.f;
}
