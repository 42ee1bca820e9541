// session.cu — K10: the session operators ListSlice and DifferenceLag, on sm_90a.
//
// Replaces, per partition:
//   ListSlice      reference nvtabular/ops/list_slice.py:78-144 (row[start:end], padded with
//                  pad_value up to max_elements) and its GPU kernels _calculate_row_sizes /
//                  _slice_rows (list_slice.py:180-228).  The unpadded copy is nvtb_gb_list_rows
//                  (groupby.cu) over the bounds written here.
//   DifferenceLag  reference nvtabular/ops/difference_lag.py:65-80:
//                    mask = (df[partition_cols] == df[partition_cols].shift(shift)).all(axis=1)
//                    out  = ((df[col] - df[col].shift(shift)) * mask).astype(float32)
//                  as one pass over the partition columns (a same-key bitmask) and one pass over up
//                  to 16 value columns.
// Every kernel is one streaming pass in which a lane owns 8 consecutive rows or output elements,
// i.e. one byte of every bitmask it writes: no atomics, and the outputs are bit-identical from run
// to run.  Row indices are int64 throughout.
#include "common.cuh"

namespace nvtb {
namespace {

constexpr int kSessThreads = 256;
constexpr int kMaxLagKeys = 8;
constexpr int kMaxLagCols = 16;

struct LagKeys {
  const void* data[kMaxLagKeys];
  const uint8_t* valid[kMaxLagKeys];
  int32_t dtype[kMaxLagKeys];
  int32_t n;
};

struct LagCols {
  const void* src[kMaxLagCols];
  const uint8_t* src_valid[kMaxLagCols];
  float* out[kMaxLagCols];
  uint8_t* out_valid[kMaxLagCols];
  int32_t dtype[kMaxLagCols];
  int32_t ncols;
};

// ---------------------------------------------------------------------------------------
// ListSlice
// ---------------------------------------------------------------------------------------
// Python's row[start:end] on a row of `len` elements: [s, e) with 0 <= s <= e <= len.  A negative
// index counts from the row end (start + len cannot overflow: start < 0 <= len).
__device__ __forceinline__ void slice_range(int64_t len, int64_t start, int64_t end, int64_t& s, int64_t& e) {
  s = start < 0 ? start + len : start;
  e = end < 0 ? end + len : end;
  s = s < 0 ? 0 : (s > len ? len : s);
  e = e < 0 ? 0 : (e > len ? len : e);
  if (e < s) e = s;
}

__global__ void __launch_bounds__(kSessThreads)
list_slice_bounds_kernel(const int64_t* __restrict__ off, int64_t n, int64_t start, int64_t end,
                         int64_t* __restrict__ lo, int64_t* __restrict__ hi) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t a = __ldg(off + i);
    int64_t s, e;
    slice_range(__ldg(off + i + 1) - a, start, end, s, e);
    lo[i] = a + s;
    hi[i] = a + e;
  }
}

// Dense output: row r is out[r * L, (r + 1) * L).  A lane owns output elements [p0, p0 + 8): the
// row of p0 is one division, the rest follow by stepping through the row.  Elements past the
// slice are `pad` and valid; copied elements carry the leaf validity.
template <typename T>
__global__ void __launch_bounds__(kSessThreads)
list_slice_pad_kernel(const T* __restrict__ src, const uint8_t* __restrict__ src_valid, const int64_t* __restrict__ off,
                      int64_t n, int64_t start, int64_t end, int64_t L, T pad, T* __restrict__ out,
                      uint8_t* __restrict__ out_valid, int64_t* __restrict__ off_out) {
  const int64_t total = n * L;
  const int64_t nchunks = (total + 7) / 8;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += stride) {
    const int64_t p0 = c * 8;
    int64_t row = p0 / L;
    int64_t k = p0 - row * L;
    int64_t base, cnt;
    {
      const int64_t a = __ldg(off + row);
      int64_t s, e;
      slice_range(__ldg(off + row + 1) - a, start, end, s, e);
      base = a + s;
      cnt = e - s;
    }
    T v[8];
    unsigned vb = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t p = p0 + j;
      v[j] = pad;
      if (p < total) {
        if (k < cnt) {
          v[j] = src[base + k];
          if (valid1(src_valid, base + k)) vb |= 1u << j;
        } else {
          vb |= 1u << j;
        }
        if (++k == L && p + 1 < total) {
          k = 0;
          ++row;
          const int64_t a = __ldg(off + row);
          int64_t s, e;
          slice_range(__ldg(off + row + 1) - a, start, end, s, e);
          base = a + s;
          cnt = e - s;
        }
      }
    }
    if (p0 + 8 <= total) {
      st_rows8<T>(out + p0, v);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) if (p0 + j < total) out[p0 + j] = v[j];
    }
    if (out_valid != nullptr) out_valid[p0 >> 3] = (uint8_t)vb;
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= n; i += stride) off_out[i] = i * L;
}

// ---------------------------------------------------------------------------------------
// DifferenceLag
// ---------------------------------------------------------------------------------------
// clears bit k of m where key[i0 + k] != key[i0 + k - shift] (IEEE ==: -0.0 == +0.0, NaN never)
template <typename T>
__device__ __forceinline__ unsigned keep_equal8(const void* d, int64_t i0, int64_t shift, unsigned m) {
  const T* __restrict__ x = static_cast<const T*>(d);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if ((m >> k) & 1u) {
      const int64_t i = i0 + k;
      if (!(__ldg(x + i) == __ldg(x + i - shift))) m &= ~(1u << k);
    }
  }
  return m;
}

// same[i / 8] bit i % 8: 0 <= i - shift < n and every key is valid and equal at i and i - shift
__global__ void __launch_bounds__(kSessThreads)
lag_same_key_kernel(LagKeys keys, int64_t n, int64_t shift, uint8_t* __restrict__ same) {
  const int64_t nchunks = (n + 7) / 8;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i0 = c * 8;
    unsigned m = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int64_t i = i0 + k, j = i - shift;
      if (i < n && j >= 0 && j < n) m |= 1u << k;
    }
    for (int q = 0; q < keys.n && m != 0; ++q) {
      const uint8_t* v = keys.valid[q];
      if (v != nullptr) {
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if (((m >> k) & 1u) && !(valid1(v, i0 + k) && valid1(v, i0 + k - shift))) m &= ~(1u << k);
      }
      switch (keys.dtype[q]) {
        case NVTB_I32: m = keep_equal8<int32_t>(keys.data[q], i0, shift, m); break;
        case NVTB_F32: m = keep_equal8<float>(keys.data[q], i0, shift, m); break;
        case NVTB_F64: m = keep_equal8<double>(keys.data[q], i0, shift, m); break;
        case NVTB_U8: m = keep_equal8<uint8_t>(keys.data[q], i0, shift, m); break;
        default: m = keep_equal8<int64_t>(keys.data[q], i0, shift, m); break;
      }
    }
    same[c] = (uint8_t)m;
  }
}

// x[i] - x[i - shift] as float32: integers subtract in int64 (wrapping) and round once; float32
// subtracts in float32; float64 subtracts in float64 and rounds once
template <typename T>
__device__ __forceinline__ float lag_diff(T a, T b) {
  if constexpr (std::is_same<T, float>::value) {
    return a - b;
  } else if constexpr (std::is_same<T, double>::value) {
    return (float)(a - b);
  } else {
    return (float)(int64_t)((uint64_t)(int64_t)a - (uint64_t)(int64_t)b);
  }
}

template <typename T>
__device__ __forceinline__ void lag8(const LagCols& c, int q, int64_t i0, int64_t n, int64_t shift, unsigned m) {
  const T* __restrict__ x = static_cast<const T*>(c.src[q]);
  const uint8_t* __restrict__ xv = c.src_valid[q];
  float o[8];
  unsigned vb = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    o[k] = 0.0f;
    const int64_t i = i0 + k;
    if (((m >> k) & 1u) && valid1(xv, i) && valid1(xv, i - shift)) {
      o[k] = lag_diff<T>(__ldg(x + i), __ldg(x + i - shift));
      vb |= 1u << k;
    }
  }
  float* out = c.out[q];
  if (i0 + 8 <= n) {
    st_rows8<float>(out + i0, o);
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) if (i0 + k < n) out[i0 + k] = o[k];
  }
  c.out_valid[q][i0 >> 3] = (uint8_t)vb;
}

__global__ void __launch_bounds__(kSessThreads)
difference_lag_kernel(LagCols c, int64_t n, int64_t shift, const uint8_t* __restrict__ same) {
  const int64_t nchunks = (n + 7) / 8;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < nchunks; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i0 = g * 8;
    const unsigned m = __ldg(same + g);
    for (int q = 0; q < c.ncols; ++q) {
      switch (c.dtype[q]) {
        case NVTB_I32: lag8<int32_t>(c, q, i0, n, shift, m); break;
        case NVTB_I64: lag8<int64_t>(c, q, i0, n, shift, m); break;
        case NVTB_F32: lag8<float>(c, q, i0, n, shift, m); break;
        case NVTB_F64: lag8<double>(c, q, i0, n, shift, m); break;
        default: lag8<uint8_t>(c, q, i0, n, shift, m); break;
      }
    }
  }
}

// |shift| >= n leaves no row inside the partition: clamping keeps i - shift from overflowing
inline int64_t clamp_shift(int64_t shift, int64_t n) {
  return shift > n ? n : (shift < -n ? -n : shift);
}

}  // namespace
}  // namespace nvtb

using namespace nvtb;

extern "C" {

int nvtb_list_slice_bounds(const int64_t* offsets, int64_t n, int64_t start, int64_t end, int64_t* lo_out,
                           int64_t* hi_out, void* stream) {
  NVTB_REQUIRE(n >= 0, "n < 0");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(offsets && lo_out && hi_out, "NULL offsets / outputs");
  list_slice_bounds_kernel<<<plain_grid(n), kSessThreads, 0, (cudaStream_t)stream>>>(offsets, n, start, end, lo_out,
                                                                                    hi_out);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

int nvtb_list_slice_pad(const nvtb_col_t* leaves, const int64_t* offsets, int64_t n, int64_t start, int64_t end,
                        int64_t L, uint64_t pad_bits, void* out, uint8_t* out_valid, int64_t* off_out, void* stream) {
  NVTB_REQUIRE(leaves != nullptr && n >= 0 && L >= 1 && off_out != nullptr, "bad arguments");
  NVTB_REQUIRE(n <= INT64_MAX / L, "n * L overflows int64");
  const int sz = (int)dtype_size(leaves->dtype);
  NVTB_REQUIRE(sz == 1 || sz == 4 || sz == 8, "unsupported leaf dtype");
  NVTB_REQUIRE(offsets != nullptr, "NULL offsets");
  NVTB_REQUIRE(n == 0 || out != nullptr, "NULL out");
  NVTB_REQUIRE(sz == 1 ? (reinterpret_cast<uintptr_t>(out) & 7u) == 0 : is_aligned32(out),
               "out must be 32-byte aligned (1-byte leaves: 8-byte)");
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = plain_grid((n * L + 7) / 8 > n + 1 ? (n * L + 7) / 8 : n + 1);
  switch (sz) {
#define NVTB_PAD_LAUNCH(T)                                                                                  \
  {                                                                                                         \
    T pad;                                                                                                  \
    memcpy(&pad, &pad_bits, sizeof(T));                                                                     \
    list_slice_pad_kernel<T><<<grid, kSessThreads, 0, st>>>((const T*)leaves->data, leaves->validity, offsets, \
                                                            n, start, end, L, pad, (T*)out, out_valid, off_out); \
  }
    case 1: NVTB_PAD_LAUNCH(uint8_t) break;
    case 4: NVTB_PAD_LAUNCH(uint32_t) break;
    default: NVTB_PAD_LAUNCH(uint64_t) break;
#undef NVTB_PAD_LAUNCH
  }
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

int nvtb_lag_same_key(const nvtb_col_t* keys, int n_keys, int64_t n, int64_t shift, uint8_t* same_out, void* stream) {
  NVTB_REQUIRE(keys != nullptr && n >= 0, "bad arguments");
  NVTB_REQUIRE(n_keys >= 1 && n_keys <= kMaxLagKeys, "n_keys must be in [1, 8]");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(same_out != nullptr, "NULL same_out");
  LagKeys k;
  memset(&k, 0, sizeof(k));
  k.n = n_keys;
  for (int q = 0; q < n_keys; ++q) {
    NVTB_REQUIRE(dtype_size(keys[q].dtype) != 0, "unsupported key dtype");
    NVTB_REQUIRE(keys[q].data != nullptr, "NULL key data");
    k.data[q] = keys[q].data;
    k.valid[q] = keys[q].validity;
    k.dtype[q] = keys[q].dtype;
  }
  lag_same_key_kernel<<<plain_grid((n + 7) / 8), kSessThreads, 0, (cudaStream_t)stream>>>(k, n, clamp_shift(shift, n),
                                                                                         same_out);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

int nvtb_difference_lag(const nvtb_col_t* cols, int ncols, int64_t n, int64_t shift, const uint8_t* same,
                        float* const* outs, uint8_t* const* out_valids, void* stream) {
  NVTB_REQUIRE(cols != nullptr && outs != nullptr && out_valids != nullptr && n >= 0, "bad arguments");
  NVTB_REQUIRE(ncols >= 1 && ncols <= kMaxLagCols, "ncols must be in [1, 16]");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(same != nullptr, "NULL same-key bitmask");
  LagCols c;
  memset(&c, 0, sizeof(c));
  c.ncols = ncols;
  for (int q = 0; q < ncols; ++q) {
    const int dt = cols[q].dtype;
    NVTB_REQUIRE(dt == NVTB_I32 || dt == NVTB_I64 || dt == NVTB_F32 || dt == NVTB_F64 || dt == NVTB_U8,
                 "unsupported value dtype");
    NVTB_REQUIRE(cols[q].data != nullptr && outs[q] != nullptr && out_valids[q] != nullptr, "NULL column / output");
    NVTB_REQUIRE(is_aligned32(outs[q]), "outputs must be 32-byte aligned");
    c.src[q] = cols[q].data;
    c.src_valid[q] = cols[q].validity;
    c.out[q] = outs[q];
    c.out_valid[q] = out_valids[q];
    c.dtype[q] = dt;
  }
  difference_lag_kernel<<<plain_grid((n + 7) / 8), kSessThreads, 0, (cudaStream_t)stream>>>(c, n, clamp_shift(shift, n),
                                                                                           same);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

}  // extern "C"
