// scan_kernels.cu — the streaming (HBM-bound) kernels of libnvtb200:
//   K1  fused FillMissing + moments/min/max reduction   (Normalize.fit)
//   K2  fused FillMissing + Normalize / NormalizeMinMax (transform)
//       standalone FillMissing (+ `_filled` indicator)
//   K6  HashBucket (pandas-compatible value hash % num_buckets)
//       key images of columns: raw value hashes, two int32 keys packed into one int64
//
// Reference behaviour restated (not ported — the reference calls cuDF/pandas):
//   nvtabular/ops/moments.py:64-116, nvtabular/ops/normalize.py:71-90,150-161,
//   nvtabular/ops/fill.py:49-57, nvtabular/ops/hash_bucket.py:86-100.
//
// Every kernel is a single coalesced pass: 256-bit loads/stores (common.cuh),
// all columns of a call in ONE launch (blockIdx.y = column), grid.x sized as a
// multiple of the SM count.  Algorithmic bytes per row and column:
//   K1: sizeof(T) + 1/8 read;            K2: sizeof(T) + 1/8 read, sizeof(Out) write
//   K6: sizeof(T) + 1/8 read, 4 write.
#include <cstdarg>
#include <limits>

#include <cstdlib>

#include "common.cuh"

namespace nvtb {

// --------------------------------------------------------------------------
// error state + device info (shared by all translation units)
// --------------------------------------------------------------------------
static thread_local char g_err[512] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int sm_count() {
  ensure_pool_configured();
  static thread_local int cached_dev = -1;
  static thread_local int cached = 132;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev != cached_dev) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) ==
            cudaSuccess && v > 0)
      cached = v;
    cached_dev = dev;
  }
  return cached;
}

void ensure_pool_configured() {
  static thread_local int done_dev = -1;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev == done_dev) return;
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
    unsigned long long keep = ~0ull;   // never trim: the engine re-uses these buffers every batch
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
  // NVTB_L2_FETCH=32|64|128: L2 fetch granularity hint.  The lookups of the large vocabularies are
  // one random 32-byte sector per row; when the L2 fetches more than that sector per miss, the rest
  // of the fetch is unused, so a smaller granularity leaves more DRAM bandwidth to useful sectors.
  if (const char* e = getenv("NVTB_L2_FETCH")) {
    const size_t g = (size_t)atoll(e);
    if (g == 32 || g == 64 || g == 128) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, g);
  }
  done_dev = dev;
}

constexpr int kMaxCols = 32;  // columns per launch (kernel-parameter budget)

struct ColBatch {
  const void* data[kMaxCols];
  const uint8_t* mask[kMaxCols];
  void* out[kMaxCols];
  uint8_t* filled[kMaxCols];
  double fill[kMaxCols];   // NaN = no fill
  double p0[kMaxCols];     // mean | min
  double p1[kMaxCols];     // std  | max
  int32_t dtype[kMaxCols];
};

__device__ __forceinline__ bool has_fill(double f) { return f == f; }

// --------------------------------------------------------------------------
// K1: moments.  partials layout: [col][block][5]
// --------------------------------------------------------------------------
struct Moments {
  double cnt, sum, sumsq, mn, mx;
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_down_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_down_sync(0xffffffffu, v, o));
  return v;
}

template <typename T>
__device__ __forceinline__ void moments_column(const T* __restrict__ data,
                                               const uint8_t* __restrict__ mask,
                                               int64_t n, double fill,
                                               double* __restrict__ partial) {
  const bool filling = has_fill(fill);
  const T fill_t = filling ? (T)fill : (T)0;
  // integer sums are exact in int64 (pandas: int column .sum() is int64, then
  // .astype(float64), moments.py:72); squares are accumulated in fp64
  // (moments.py:73 casts to float64 before pow(2)).
  using SumT = typename std::conditional<std::is_integral<T>::value, int64_t,
                                         double>::type;
  SumT sum = 0;
  double sumsq = 0.0;
  int64_t cnt = 0;
  double mn = INFINITY, mx = -INFINITY;
  const bool aligned = is_aligned32(data);
  for_each_row<T>(data, mask, n, aligned,
                  [&](int64_t, T x, bool valid) {
                    bool isnull = !valid;
                    if constexpr (std::is_floating_point<T>::value)
                      isnull = isnull || (x != x);  // NaN == null (pandas)
                    if (isnull) {
                      if (!filling) return;
                      x = fill_t;
                    }
                    const double xd = (double)x;
                    cnt += 1;
                    sum += (SumT)x;
                    sumsq = fma(xd, xd, sumsq);
                    mn = fmin(mn, xd);
                    mx = fmax(mx, xd);
                  });
  __shared__ double s[5][kThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double c = warp_sum((double)cnt);
  double su = warp_sum((double)sum);
  double sq = warp_sum(sumsq);
  double a = warp_min(mn);
  double b = warp_max(mx);
  if (lane == 0) {
    s[0][warp] = c; s[1][warp] = su; s[2][warp] = sq; s[3][warp] = a; s[4][warp] = b;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double r0 = 0, r1 = 0, r2 = 0, r3 = INFINITY, r4 = -INFINITY;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
      r0 += s[0][w]; r1 += s[1][w]; r2 += s[2][w];
      r3 = fmin(r3, s[3][w]); r4 = fmax(r4, s[4][w]);
    }
    partial[0] = r0; partial[1] = r1; partial[2] = r2; partial[3] = r3; partial[4] = r4;
  }
}

__global__ void __launch_bounds__(kThreads)
moments_kernel(ColBatch cb, int64_t n, double* __restrict__ partials) {
  const int c = blockIdx.y;
  double* partial = partials + ((int64_t)c * gridDim.x + blockIdx.x) * 5;
  switch (cb.dtype[c]) {
    case NVTB_I32: moments_column<int32_t>((const int32_t*)cb.data[c], cb.mask[c], n, cb.fill[c], partial); break;
    case NVTB_I64: moments_column<int64_t>((const int64_t*)cb.data[c], cb.mask[c], n, cb.fill[c], partial); break;
    case NVTB_F32: moments_column<float>((const float*)cb.data[c], cb.mask[c], n, cb.fill[c], partial); break;
    default:       moments_column<double>((const double*)cb.data[c], cb.mask[c], n, cb.fill[c], partial); break;
  }
}

// ordered (deterministic) reduction of the per-block partials into acc
__global__ void moments_reduce_kernel(const double* __restrict__ partials,
                                      int nblocks, double* __restrict__ acc) {
  const int c = blockIdx.x;
  const double* p = partials + (int64_t)c * nblocks * 5;
  double r0 = 0, r1 = 0, r2 = 0, r3 = INFINITY, r4 = -INFINITY;
  for (int b = threadIdx.x; b < nblocks; b += 32) {
    r0 += p[b * 5 + 0]; r1 += p[b * 5 + 1]; r2 += p[b * 5 + 2];
    r3 = fmin(r3, p[b * 5 + 3]); r4 = fmax(r4, p[b * 5 + 4]);
  }
  r0 = warp_sum(r0); r1 = warp_sum(r1); r2 = warp_sum(r2);
  r3 = warp_min(r3); r4 = warp_max(r4);
  if (threadIdx.x == 0) {
    double* a = acc + c * 5;
    a[0] += r0; a[1] += r1; a[2] += r2;
    a[3] = fmin(a[3], r3); a[4] = fmax(a[4], r4);
  }
}

__global__ void moments_init_kernel(double* acc, int ncols) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < ncols) {
    acc[c * 5 + 0] = 0; acc[c * 5 + 1] = 0; acc[c * 5 + 2] = 0;
    acc[c * 5 + 3] = INFINITY; acc[c * 5 + 4] = -INFINITY;
  }
}

// --------------------------------------------------------------------------
// K2: transforms
// --------------------------------------------------------------------------
enum { OP_FILL = 0, OP_NORMALIZE = 1, OP_MINMAX = 2, OP_CLIP = 3, OP_CLIPLOG = 4 };

template <typename T, typename OutT, int OP>
__device__ __forceinline__ void transform_column(const ColBatch& cb, int c,
                                                 int64_t n) {
  const T* data = (const T*)cb.data[c];
  const uint8_t* mask = cb.mask[c];
  OutT* out = (OutT*)cb.out[c];
  const double fill = cb.fill[c];
  const bool filling = has_fill(fill);
  const T fill_t = filling ? (T)fill : (T)0;
  const bool aligned = is_aligned32(data) && is_aligned32(out);
  // numpy semantics (normalize.py:80-85): a float32 column minus a python
  // float stays float32, every other dtype is promoted to float64.
  using CT = typename std::conditional<std::is_same<T, float>::value, float,
                                       double>::type;
  const CT p0 = (CT)cb.p0[c];
  const CT p1 = (CT)cb.p1[c];
  const OutT out_null = std::is_floating_point<OutT>::value
                            ? (OutT)NAN : (OutT)0;
  if constexpr (OP == OP_FILL) {
    uint8_t* filled = cb.filled[c];
    map_rows<T, OutT>(data, mask, out, n, aligned,
                      [&](int64_t, T x, bool valid) -> OutT {
                        bool isnull = !valid;
                        if constexpr (std::is_floating_point<T>::value)
                          isnull = isnull || (x != x);
                        return (OutT)(isnull ? fill_t : x);
                      });
    if (filled != nullptr) {
      const bool al2 = is_aligned32(data) &&
                       ((reinterpret_cast<uintptr_t>(filled) & 7u) == 0);
      map_rows<T, uint8_t>(data, mask, filled, n, al2,
                           [&](int64_t, T x, bool valid) -> uint8_t {
                             bool isnull = !valid;
                             if constexpr (std::is_floating_point<T>::value)
                               isnull = isnull || (x != x);
                             return isnull ? 1 : 0;
                           });
    }
  } else if constexpr (OP == OP_NORMALIZE) {
    const bool divide = p1 > (CT)0;  // std > 0 (false for NaN std too)
    map_rows<T, OutT>(data, mask, out, n, aligned,
                      [&](int64_t, T x, bool valid) -> OutT {
                        bool isnull = !valid;
                        if constexpr (std::is_floating_point<T>::value)
                          isnull = isnull || (x != x);
                        if (isnull) {
                          if (!filling) return out_null;
                          x = fill_t;
                        }
                        CT r = (CT)x - p0;
                        if (divide) r = r / p1;
                        return (OutT)r;
                      });
  } else if constexpr (OP == OP_CLIP || OP == OP_CLIPLOG) {
    // Clip (reference nvtabular/ops/clip.py:46-53): values below p0 become p0, above p1 become
    // p1 (NaN bound = none; nulls stay nulls unless an upstream FillMissing is fused in), then
    // for OP_CLIPLOG LogOp (ops/logop.py:47-56): log(x.astype(out dtype) + 1) in that dtype —
    // evaluated in fp64 and rounded once, i.e. the correctly rounded value
    const double lo = cb.p0[c], hi = cb.p1[c];
    const bool has_lo = lo == lo, has_hi = hi == hi;
    const T lo_t = has_lo ? (T)lo : (T)0, hi_t = has_hi ? (T)hi : (T)0;
    map_rows<T, OutT>(data, mask, out, n, aligned,
                      [&](int64_t, T x, bool valid) -> OutT {
                        bool isnull = !valid;
                        if constexpr (std::is_floating_point<T>::value)
                          isnull = isnull || (x != x);
                        if (isnull) {
                          if (!filling) return out_null;
                          x = fill_t;
                        }
                        if (has_lo && x < lo_t) x = lo_t;
                        if (has_hi && x > hi_t) x = hi_t;
                        if constexpr (OP == OP_CLIPLOG) {
                          const OutT xo = (OutT)x + (OutT)1;
                          return (OutT)log((double)xo);
                        } else {
                          return (OutT)x;
                        }
                      });
  } else {  // OP_MINMAX: p0 = min, p1 = max
    const CT dif = p1 - p0;
    map_rows<T, OutT>(data, mask, out, n, aligned,
                      [&](int64_t, T x, bool valid) -> OutT {
                        bool isnull = !valid;
                        if constexpr (std::is_floating_point<T>::value)
                          isnull = isnull || (x != x);
                        if (isnull) {
                          if (!filling) return out_null;
                          x = fill_t;
                        }
                        CT r;
                        if (dif > (CT)0) r = ((CT)x - p0) / dif;
                        else r = (CT)x / ((CT)2 * (CT)x);  // normalize.py:158-159
                        return (OutT)r;
                      });
  }
}

template <int OP, typename OutT>
__global__ void __launch_bounds__(kThreads)
transform_kernel(ColBatch cb, int64_t n) {
  const int c = blockIdx.y;
  switch (cb.dtype[c]) {
    case NVTB_I32: transform_column<int32_t, OutT, OP>(cb, c, n); break;
    case NVTB_I64: transform_column<int64_t, OutT, OP>(cb, c, n); break;
    case NVTB_F32: transform_column<float, OutT, OP>(cb, c, n); break;
    default:       transform_column<double, OutT, OP>(cb, c, n); break;
  }
}

// FillMissing keeps the dtype, so OutT == T per column
__global__ void __launch_bounds__(kThreads)
fill_kernel(ColBatch cb, int64_t n) {
  const int c = blockIdx.y;
  switch (cb.dtype[c]) {
    case NVTB_I32: transform_column<int32_t, int32_t, OP_FILL>(cb, c, n); break;
    case NVTB_I64: transform_column<int64_t, int64_t, OP_FILL>(cb, c, n); break;
    case NVTB_F32: transform_column<float, float, OP_FILL>(cb, c, n); break;
    default:       transform_column<double, double, OP_FILL>(cb, c, n); break;
  }
}

// Clip keeps the dtype, so OutT == T per column (nulls of an unfilled integer column come out
// as 0 under an unchanged validity mask)
__global__ void __launch_bounds__(kThreads)
clip_kernel(ColBatch cb, int64_t n) {
  const int c = blockIdx.y;
  switch (cb.dtype[c]) {
    case NVTB_I32: transform_column<int32_t, int32_t, OP_CLIP>(cb, c, n); break;
    case NVTB_I64: transform_column<int64_t, int64_t, OP_CLIP>(cb, c, n); break;
    case NVTB_F32: transform_column<float, float, OP_CLIP>(cb, c, n); break;
    default:       transform_column<double, double, OP_CLIP>(cb, c, n); break;
  }
}

// --------------------------------------------------------------------------
// K6: hash bucket.  Up to 4 columns are XOR-combined (combo / HashedCross).
// --------------------------------------------------------------------------
constexpr int kMaxHashCols = 8;
struct HashCols {
  const void* data[kMaxHashCols];
  const uint8_t* mask[kMaxHashCols];
  int32_t dtype[kMaxHashCols];
  int32_t ncols;
};

__device__ __forceinline__ uint64_t hash_one(const HashCols& hc, int c,
                                             int64_t i) {
  uint64_t bits;
  if (!valid1(hc.mask[c], i)) {
    bits = kNaNBits;
  } else {
    switch (hc.dtype[c]) {
      case NVTB_I32: bits = value_bits<int32_t>(((const int32_t*)hc.data[c])[i]); break;
      case NVTB_I64: bits = value_bits<int64_t>(((const int64_t*)hc.data[c])[i]); break;
      case NVTB_F32: bits = value_bits<float>(((const float*)hc.data[c])[i]); break;
      case NVTB_F64: bits = value_bits<double>(((const double*)hc.data[c])[i]); break;
      case NVTB_H64: return (uint64_t)((const int64_t*)hc.data[c])[i];  // already a hash
      default:       bits = value_bits<uint8_t>(((const uint8_t*)hc.data[c])[i]); break;
    }
  }
  return pandas_mix64(bits);
}

// h % d without the ~100-instruction software 64-bit division: with M = floor(2^64 / d) (host),
// q = mulhi(h, M) is the true quotient or one below it, so r = h - q d lies in [0, 2d): one
// conditional subtraction makes it exact for every d >= 2 (d == 1: M does not fit, result 0).
__device__ __forceinline__ uint64_t fast_mod_u64(uint64_t h, uint64_t d, uint64_t M) {
  if (d == 1) return 0;
  const uint64_t r = h - __umul64hi(h, M) * d;
  return r >= d ? r - d : r;
}
static uint64_t fast_mod_magic(uint64_t d) {
  return d > 1 ? (uint64_t)((((unsigned __int128)1) << 64) / d) : 0;
}

// single-column fast path: tiled 256-bit loads
template <typename T, typename OutT>
__device__ __forceinline__ void hash_bucket_column(const T* __restrict__ data,
                                                   const uint8_t* __restrict__ mask,
                                                   OutT* __restrict__ out,
                                                   int64_t n, uint64_t nb, uint64_t nb_magic,
                                                   int64_t add) {
  const bool aligned = is_aligned32(data) && is_aligned32(out);
  map_rows<T, OutT>(data, mask, out, n, aligned,
                    [&](int64_t, T x, bool valid) -> OutT {
                      const uint64_t bits = valid ? value_bits<T>(x) : kNaNBits;
                      return (OutT)((int64_t)fast_mod_u64(pandas_mix64(bits), nb, nb_magic) + add);
                    });
}

template <typename OutT>
__global__ void __launch_bounds__(kThreads)
hash_bucket1_kernel(const void* data, const uint8_t* mask, int dtype, OutT* out,
                    int64_t n, uint64_t nb, uint64_t nb_magic, int64_t add) {
  switch (dtype) {
    case NVTB_I32: hash_bucket_column<int32_t, OutT>((const int32_t*)data, mask, out, n, nb, nb_magic, add); break;
    case NVTB_I64: hash_bucket_column<int64_t, OutT>((const int64_t*)data, mask, out, n, nb, nb_magic, add); break;
    case NVTB_F32: hash_bucket_column<float, OutT>((const float*)data, mask, out, n, nb, nb_magic, add); break;
    default:       hash_bucket_column<double, OutT>((const double*)data, mask, out, n, nb, nb_magic, add); break;
  }
}

template <typename OutT>
__global__ void __launch_bounds__(kThreads)
hash_bucketN_kernel(HashCols hc, OutT* __restrict__ out, int64_t n, uint64_t nb, uint64_t nb_magic,
                    int64_t add) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    uint64_t h = 0;
    for (int c = 0; c < hc.ncols; ++c) h ^= hash_one(hc, c, i);
    out[i] = (OutT)((int64_t)fast_mod_u64(h, nb, nb_magic) + add);
  }
}

__global__ void __launch_bounds__(kThreads)
hash_values_kernel(HashCols hc, uint64_t* __restrict__ out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    out[i] = hash_one(hc, 0, i);
}

// two int32 key columns -> one order-preserving int64 key (multi-column keys of the group-by)
__global__ void __launch_bounds__(kThreads)
pack_keys2_kernel(const int32_t* __restrict__ a, const uint8_t* __restrict__ ma,
                  const int32_t* __restrict__ b, const uint8_t* __restrict__ mb,
                  int64_t n, int64_t* __restrict__ out, uint8_t* __restrict__ vout) {
  // one thread per 8 rows so each thread owns one validity byte
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t n8 = (n + 7) / 8;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n8; g += stride) {
    unsigned vb = 0;
    for (int k = 0; k < 8; ++k) {
      const int64_t i = g * 8 + k;
      if (i >= n) break;
      const bool va = valid1(ma, i), vb_ = valid1(mb, i);
      const int32_t x = va ? a[i] : INT32_MIN;
      const int32_t y = vb_ ? b[i] : INT32_MIN;
      out[i] = (int64_t)(((uint64_t)(uint32_t)x << 32) |
                         (uint64_t)((uint32_t)y ^ 0x80000000u));
      if (va || vb_) vb |= 1u << k;
    }
    if (vout) vout[g] = (uint8_t)vb;
  }
}

static int check_cols(const nvtb_col_t* cols, int ncols, int64_t n) {
  NVTB_REQUIRE(ncols >= 0, "ncols < 0");
  NVTB_REQUIRE(n >= 0, "n < 0");
  NVTB_REQUIRE(ncols == 0 || cols != nullptr, "cols is NULL");
  for (int c = 0; c < ncols; ++c) {
    NVTB_REQUIRE(cols[c].dtype >= NVTB_I32 && cols[c].dtype <= NVTB_F64,
                 "column dtype must be int32/int64/float32/float64");
    NVTB_REQUIRE(n == 0 || cols[c].data != nullptr, "column data is NULL");
  }
  return NVTB_OK;
}

}  // namespace nvtb

using namespace nvtb;

extern "C" {

int nvtb_version(void) { return 1000 * 0 + 1; }

const char* nvtb_last_error(void) { return g_err; }

int nvtb_device_sm_count(int* out_host) {
  NVTB_REQUIRE(out_host != nullptr, "out is NULL");
  int dev = 0, v = 0;
  NVTB_CUDA_OK(cudaGetDevice(&dev));
  NVTB_CUDA_OK(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev));
  *out_host = v;
  return NVTB_OK;
}

int nvtb_moments_init(double* acc, int ncols, void* stream) {
  NVTB_REQUIRE(acc != nullptr && ncols > 0, "acc NULL or ncols <= 0");
  moments_init_kernel<<<(ncols + 127) / 128, 128, 0, (cudaStream_t)stream>>>(acc, ncols);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

int nvtb_moments_accumulate(const nvtb_col_t* cols, int ncols, int64_t n,
                            const double* fill_vals, double* acc, void* stream) {
  int rc = check_cols(cols, ncols, n);
  if (rc) return rc;
  NVTB_REQUIRE(acc != nullptr, "acc is NULL");
  if (n == 0 || ncols == 0) return NVTB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = scan_grid(n, 4);
  for (int c0 = 0; c0 < ncols; c0 += kMaxCols) {
    const int nc = (ncols - c0 < kMaxCols) ? ncols - c0 : kMaxCols;
    ColBatch cb;
    memset(&cb, 0, sizeof(cb));
    for (int c = 0; c < nc; ++c) {
      cb.data[c] = cols[c0 + c].data;
      cb.mask[c] = cols[c0 + c].validity;
      cb.dtype[c] = cols[c0 + c].dtype;
      cb.fill[c] = fill_vals ? fill_vals[c0 + c] : NAN;
    }
    double* partials = nullptr;
    NVTB_CUDA_OK(cudaMallocAsync(&partials, sizeof(double) * 5 * grid * nc, st));
    moments_kernel<<<dim3(grid, nc), kThreads, 0, st>>>(cb, n, partials);
    NVTB_LAUNCH_OK();
    moments_reduce_kernel<<<nc, 32, 0, st>>>(partials, grid, acc + (int64_t)c0 * 5);
    NVTB_LAUNCH_OK();
    NVTB_CUDA_OK(cudaFreeAsync(partials, st));
  }
  return NVTB_OK;
}

int nvtb_moments_finalize(const double* acc, int ncols, double* out) {
  NVTB_REQUIRE(acc != nullptr && out != nullptr && ncols >= 0, "NULL argument");
  for (int c = 0; c < ncols; ++c) {
    const double n = acc[c * 5 + 0], x = acc[c * 5 + 1], x2 = acc[c * 5 + 2];
    // moments.py:98-107: var = x2 - x**2/n; div = n-1 clamped to >= 1;
    // NaN where n-1 == 0
    double var = x2 - x * x / n;
    double div = n - 1.0;
    if (div < 1.0) div = 1.0;
    var /= div;
    if (n - 1.0 == 0.0) var = NAN;
    out[c * 3 + 0] = x / n;
    out[c * 3 + 1] = var;
    out[c * 3 + 2] = sqrt(var);
  }
  return NVTB_OK;
}

static int launch_transform(int op, const nvtb_col_t* cols, int ncols, int64_t n,
                            const double* fill_vals, const double* p0,
                            const double* p1, void* const* out,
                            uint8_t* const* filled, int out_dtype, void* stream) {
  int rc = check_cols(cols, ncols, n);
  if (rc) return rc;
  NVTB_REQUIRE(out != nullptr || ncols == 0, "out is NULL");
  if (op != OP_FILL && op != OP_CLIP)
    NVTB_REQUIRE(out_dtype == NVTB_F32 || out_dtype == NVTB_F64,
                 "out_dtype must be float32 or float64");
  if (n == 0 || ncols == 0) return NVTB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = scan_grid(n, 8);
  for (int c0 = 0; c0 < ncols; c0 += kMaxCols) {
    const int nc = (ncols - c0 < kMaxCols) ? ncols - c0 : kMaxCols;
    ColBatch cb;
    memset(&cb, 0, sizeof(cb));
    for (int c = 0; c < nc; ++c) {
      cb.data[c] = cols[c0 + c].data;
      cb.mask[c] = cols[c0 + c].validity;
      cb.dtype[c] = cols[c0 + c].dtype;
      cb.fill[c] = fill_vals ? fill_vals[c0 + c] : NAN;
      const double none = (op == OP_CLIP || op == OP_CLIPLOG) ? NAN : 0.0;
      cb.p0[c] = p0 ? p0[c0 + c] : none;
      cb.p1[c] = p1 ? p1[c0 + c] : none;
      NVTB_REQUIRE(out[c0 + c] != nullptr, "out column is NULL");
      cb.out[c] = out[c0 + c];
      cb.filled[c] = filled ? filled[c0 + c] : nullptr;
    }
    dim3 g(grid, nc);
    if (op == OP_FILL) {
      fill_kernel<<<g, kThreads, 0, st>>>(cb, n);
    } else if (op == OP_CLIP) {
      clip_kernel<<<g, kThreads, 0, st>>>(cb, n);
    } else if (op == OP_CLIPLOG) {
      if (out_dtype == NVTB_F64) transform_kernel<OP_CLIPLOG, double><<<g, kThreads, 0, st>>>(cb, n);
      else                        transform_kernel<OP_CLIPLOG, float><<<g, kThreads, 0, st>>>(cb, n);
    } else if (op == OP_NORMALIZE) {
      if (out_dtype == NVTB_F64) transform_kernel<OP_NORMALIZE, double><<<g, kThreads, 0, st>>>(cb, n);
      else                        transform_kernel<OP_NORMALIZE, float><<<g, kThreads, 0, st>>>(cb, n);
    } else {
      if (out_dtype == NVTB_F64) transform_kernel<OP_MINMAX, double><<<g, kThreads, 0, st>>>(cb, n);
      else                        transform_kernel<OP_MINMAX, float><<<g, kThreads, 0, st>>>(cb, n);
    }
    NVTB_LAUNCH_OK();
  }
  return NVTB_OK;
}

int nvtb_fill_apply(const nvtb_col_t* cols, int ncols, int64_t n,
                    const double* fill_vals, void* const* out,
                    uint8_t* const* filled_out, void* stream) {
  NVTB_REQUIRE(fill_vals != nullptr || ncols == 0, "fill_vals is NULL");
  return launch_transform(OP_FILL, cols, ncols, n, fill_vals, nullptr, nullptr,
                          out, filled_out, 0, stream);
}

int nvtb_normalize_apply(const nvtb_col_t* cols, int ncols, int64_t n,
                         const double* fill_vals, const double* means,
                         const double* stds, void* const* out, int out_dtype,
                         void* stream) {
  NVTB_REQUIRE((means && stds) || ncols == 0, "means/stds NULL");
  return launch_transform(OP_NORMALIZE, cols, ncols, n, fill_vals, means, stds,
                          out, nullptr, out_dtype, stream);
}

int nvtb_minmax_apply(const nvtb_col_t* cols, int ncols, int64_t n,
                      const double* fill_vals, const double* mins,
                      const double* maxs, void* const* out, int out_dtype,
                      void* stream) {
  NVTB_REQUIRE((mins && maxs) || ncols == 0, "mins/maxs NULL");
  return launch_transform(OP_MINMAX, cols, ncols, n, fill_vals, mins, maxs, out,
                          nullptr, out_dtype, stream);
}

int nvtb_cliplog_apply(const nvtb_col_t* cols, int ncols, int64_t n,
                       const double* fill_vals, const double* min_vals,
                       const double* max_vals, int take_log, void* const* out,
                       int out_dtype, void* stream) {
  return launch_transform(take_log ? OP_CLIPLOG : OP_CLIP, cols, ncols, n, fill_vals, min_vals, max_vals,
                          out, nullptr, out_dtype, stream);
}

int nvtb_hash_bucket_apply(const nvtb_col_t* cols, int ncols, int64_t n,
                           uint64_t num_buckets, int64_t add, void* out,
                           int out_dtype, void* stream) {
  NVTB_REQUIRE(ncols >= 1 && ncols <= kMaxHashCols, "ncols must be in [1, 8]");
  NVTB_REQUIRE(num_buckets >= 1, "num_buckets must be >= 1");
  NVTB_REQUIRE(out_dtype == NVTB_I32 || out_dtype == NVTB_I64,
               "out_dtype must be int32 or int64");
  NVTB_REQUIRE(n >= 0 && cols != nullptr, "bad n/cols");
  for (int c = 0; c < ncols; ++c)
    NVTB_REQUIRE(cols[c].dtype >= NVTB_I32 && cols[c].dtype <= NVTB_H64 &&
                     (n == 0 || cols[c].data),
                 "bad hash column");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(out != nullptr, "out is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = scan_grid(n, 8);
  const uint64_t magic = fast_mod_magic(num_buckets);
  if (ncols == 1 && cols[0].dtype <= NVTB_F64) {
    if (out_dtype == NVTB_I32)
      hash_bucket1_kernel<int32_t><<<grid, kThreads, 0, st>>>(
          cols[0].data, cols[0].validity, cols[0].dtype, (int32_t*)out, n, num_buckets, magic, add);
    else
      hash_bucket1_kernel<int64_t><<<grid, kThreads, 0, st>>>(
          cols[0].data, cols[0].validity, cols[0].dtype, (int64_t*)out, n, num_buckets, magic, add);
  } else {
    HashCols hc;
    memset(&hc, 0, sizeof(hc));
    hc.ncols = ncols;
    for (int c = 0; c < ncols; ++c) {
      hc.data[c] = cols[c].data; hc.mask[c] = cols[c].validity; hc.dtype[c] = cols[c].dtype;
    }
    if (out_dtype == NVTB_I32)
      hash_bucketN_kernel<int32_t><<<grid, kThreads, 0, st>>>(hc, (int32_t*)out, n, num_buckets, magic, add);
    else
      hash_bucketN_kernel<int64_t><<<grid, kThreads, 0, st>>>(hc, (int64_t*)out, n, num_buckets, magic, add);
  }
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

int nvtb_hash_values(const nvtb_col_t* col, int64_t n, uint64_t* out, void* stream) {
  NVTB_REQUIRE(col != nullptr && n >= 0, "bad col/n");
  NVTB_REQUIRE(col->dtype >= NVTB_I32 && col->dtype <= NVTB_H64, "bad dtype");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(col->data && out, "NULL data/out");
  HashCols hc;
  memset(&hc, 0, sizeof(hc));
  hc.ncols = 1; hc.data[0] = col->data; hc.mask[0] = col->validity; hc.dtype[0] = col->dtype;
  hash_values_kernel<<<scan_grid(n, 8), kThreads, 0, (cudaStream_t)stream>>>(hc, out, n);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

int nvtb_pack_keys2(const nvtb_col_t* a, const nvtb_col_t* b, int64_t n,
                    int64_t* keys_out, uint8_t* validity_out, void* stream) {
  NVTB_REQUIRE(a && b && n >= 0, "NULL column or n < 0");
  NVTB_REQUIRE(a->dtype == NVTB_I32 && b->dtype == NVTB_I32, "pack_keys2 needs int32 columns");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(a->data && b->data && keys_out, "NULL data");
  pack_keys2_kernel<<<plain_grid((n + 7) / 8), kThreads, 0, (cudaStream_t)stream>>>(
      (const int32_t*)a->data, a->validity, (const int32_t*)b->data, b->validity, n, keys_out, validity_out);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

}  // extern "C"
