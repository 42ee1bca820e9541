// filter.cu — K11: the row-selection operators Filter and Dropna, on sm_90a.
//
// Replaces, per partition:
//   Filter  reference nvtabular/ops/filter.py:51-62: f(df) returns a bool Series (a comparison of
//           a column with a scalar or another column, isnull / notnull, & | ^ ~ of those) and the
//           frame is indexed by it, pandas boolean indexing, then reset_index(drop=True).
//   Dropna  reference nvtabular/ops/dropna.py:33-37: df.dropna(subset=<selected columns>).
// Predicates are row masks in the validity layout (LSB-first, one bit per row, padded to 32 bytes
// like pack_validity, bits at positions >= n zero).  A mask is counted per tile of 2048 rows, the
// tile counts are scanned by the multi-CTA scan of scan.cuh, and the kept row ids are written in
// ascending order.  The compaction itself is the external-table join's gather (nvtb_join_gather)
// and the sub-list copy (nvtb_gb_list_rows) at those row ids.
// Every mask kernel is one streaming pass in which a lane owns 8 consecutive rows, i.e. one mask
// byte: no atomics, and the outputs are bit-identical from run to run.  Row indices are int64.
#include "common.cuh"
#include "scan.cuh"

namespace nvtb {
namespace {

constexpr int kFiltThreads = 256;
constexpr int kMaxNotnullCols = 16;
constexpr int kMaskTile = kScanTile;   // rows per tile of the count / select passes (256 mask bytes)

struct NotnullCols {
  const void* data[kMaxNotnullCols];
  const uint8_t* valid[kMaxNotnullCols];
  int32_t dtype[kMaxNotnullCols];
  uint32_t vec;                         // bit q: column q may use 128-bit loads
  int32_t n;
};

inline int filt_grid(int64_t items) {
  int64_t g = (items + kFiltThreads - 1) / kFiltThreads;
  const int64_t cap = (int64_t)sm_count() * 8;
  if (g > cap) g = cap;
  return (int)(g < 1 ? 1 : g);
}

// bytes of an n-row mask: ceil(n / 8) rounded up to whole 32-byte blocks (pack_validity's padding)
__host__ __device__ __forceinline__ int64_t mask_bytes(int64_t n) {
  return ((n + 7) / 8 + 31) / 32 * 32;
}

// the bits of mask byte c that are rows below n
__device__ __forceinline__ unsigned tail8(int64_t c, int64_t n) {
  const int64_t left = n - c * 8;
  return left >= 8 ? 0xFFu : ((1u << left) - 1u);
}

// can rows [8c, 8c + 8) of this column be moved as one vector?
inline bool vec_ok(const void* p, int dtype) {
  return dtype_size(dtype) == 1 ? (reinterpret_cast<uintptr_t>(p) & 7u) == 0 : is_aligned32(p);
}

// rows [i0, i0 + 8) of a column (0 past n); `vec`: 32-byte aligned (1-byte columns: 8-byte)
template <typename T>
__device__ __forceinline__ void load8(const void* p, int64_t i0, int64_t n, bool vec, T (&v)[8]) {
  const T* __restrict__ x = static_cast<const T*>(p);
  if (vec && i0 + 8 <= n) {
    if constexpr (sizeof(T) == 1) {
      const uint2 w = __ldg(reinterpret_cast<const uint2*>(x + i0));
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = (T)(((k < 4 ? w.x : w.y) >> (8 * (k & 3))) & 0xFFu);
    } else {
      ld_rows8<T>(x + i0, v);
    }
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = i0 + k < n ? x[i0 + k] : (T)0;
  }
}

template <typename T, typename C>
__device__ __forceinline__ void load8_cvt(const void* p, int64_t i0, int64_t n, bool vec, C (&c)[8]) {
  T v[8];
  load8<T>(p, i0, n, vec, v);
#pragma unroll
  for (int k = 0; k < 8; ++k) c[k] = (C)v[k];
}

// rows [i0, i0 + 8) of a column of any engine dtype, converted to the comparison type C
template <typename C>
__device__ __forceinline__ void load8_as(const void* p, int dt, int64_t i0, int64_t n, bool vec, C (&c)[8]) {
  switch (dt) {
    case NVTB_I32: load8_cvt<int32_t, C>(p, i0, n, vec, c); break;
    case NVTB_I64: load8_cvt<int64_t, C>(p, i0, n, vec, c); break;
    case NVTB_F32: load8_cvt<float, C>(p, i0, n, vec, c); break;
    case NVTB_F64: load8_cvt<double, C>(p, i0, n, vec, c); break;
    default: load8_cvt<uint8_t, C>(p, i0, n, vec, c); break;
  }
}

// bit k = x[k] op y[k] (IEEE: a NaN operand is false for every op but NE)
template <typename C>
__device__ __forceinline__ unsigned cmp8(int op, const C (&x)[8], const C (&y)[8]) {
  unsigned m = 0;
  switch (op) {
    case NVTB_CMP_EQ:
#pragma unroll
      for (int k = 0; k < 8; ++k) m |= (unsigned)(x[k] == y[k]) << k;
      break;
    case NVTB_CMP_NE:
#pragma unroll
      for (int k = 0; k < 8; ++k) m |= (unsigned)(x[k] != y[k]) << k;
      break;
    case NVTB_CMP_LT:
#pragma unroll
      for (int k = 0; k < 8; ++k) m |= (unsigned)(x[k] < y[k]) << k;
      break;
    case NVTB_CMP_LE:
#pragma unroll
      for (int k = 0; k < 8; ++k) m |= (unsigned)(x[k] <= y[k]) << k;
      break;
    case NVTB_CMP_GT:
#pragma unroll
      for (int k = 0; k < 8; ++k) m |= (unsigned)(x[k] > y[k]) << k;
      break;
    default:
#pragma unroll
      for (int k = 0; k < 8; ++k) m |= (unsigned)(x[k] >= y[k]) << k;
      break;
  }
  return m;
}

// out byte c: rows [8c, 8c + 8) of a op (b or the scalar s), in type C.  A null operand gives true
// for NE and false otherwise.  Bytes from ceil(n / 8) to the padded end are written as 0.
template <typename C>
__global__ void __launch_bounds__(kFiltThreads)
mask_compare_kernel(nvtb_col_t a, bool avec, nvtb_col_t b, bool bvec, C s, int op, int64_t n,
                    uint8_t* __restrict__ out) {
  const int64_t nchunks = (n + 7) / 8;
  const int64_t nbytes = mask_bytes(n);
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nbytes; c += (int64_t)gridDim.x * blockDim.x) {
    if (c >= nchunks) {
      out[c] = 0;
      continue;
    }
    const int64_t i0 = c * 8;
    C x[8], y[8];
    load8_as<C>(a.data, a.dtype, i0, n, avec, x);
    unsigned valid = valid8(a.validity, i0);
    if (b.data != nullptr) {
      load8_as<C>(b.data, b.dtype, i0, n, bvec, y);
      valid &= valid8(b.validity, i0);
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) y[k] = s;
    }
    unsigned m = cmp8<C>(op, x, y);
    m = op == NVTB_CMP_NE ? (m | ~valid) : (m & valid);
    out[c] = (uint8_t)(m & tail8(c, n));
  }
}

template <typename T>
__device__ __forceinline__ unsigned not_nan8(const void* p, int64_t i0, int64_t n, bool vec) {
  T v[8];
  load8<T>(p, i0, n, vec, v);
  unsigned m = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) m |= (unsigned)(v[k] == v[k]) << k;
  return m;
}

// out byte c: the rows of [8c, 8c + 8) at which every column is valid and, if it is a float, not NaN
__global__ void __launch_bounds__(kFiltThreads)
mask_notnull_kernel(NotnullCols cols, int64_t n, uint8_t* __restrict__ out) {
  const int64_t nchunks = (n + 7) / 8;
  const int64_t nbytes = mask_bytes(n);
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nbytes; c += (int64_t)gridDim.x * blockDim.x) {
    if (c >= nchunks) {
      out[c] = 0;
      continue;
    }
    const int64_t i0 = c * 8;
    unsigned m = tail8(c, n);
    for (int q = 0; q < cols.n && m != 0; ++q) {
      m &= valid8(cols.valid[q], i0);
      const bool vec = (cols.vec >> q) & 1u;
      if (cols.dtype[q] == NVTB_F32) m &= not_nan8<float>(cols.data[q], i0, n, vec);
      else if (cols.dtype[q] == NVTB_F64) m &= not_nan8<double>(cols.data[q], i0, n, vec);
    }
    out[c] = (uint8_t)m;
  }
}

__device__ __forceinline__ uint32_t logic32(int op, uint32_t x, uint32_t y) {
  switch (op) {
    case NVTB_MASK_AND: return x & y;
    case NVTB_MASK_OR: return x | y;
    case NVTB_MASK_XOR: return x ^ y;
    default: return ~x;
  }
}

// 16 mask bytes per lane (one 128-bit access); bits at rows >= n are cleared
__global__ void __launch_bounds__(kFiltThreads)
mask_logic_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, int64_t n, int op,
                  uint4* __restrict__ out) {
  const int64_t nwords = mask_bytes(n) / 16;
  for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += (int64_t)gridDim.x * blockDim.x) {
    const uint4 x = __ldg(a + w);
    const uint4 y = b != nullptr ? __ldg(b + w) : make_uint4(0, 0, 0, 0);
    uint32_t r[4] = {logic32(op, x.x, y.x), logic32(op, x.y, y.y), logic32(op, x.z, y.z), logic32(op, x.w, y.w)};
    const int64_t r0 = w * 128;            // first row of this word
    if (r0 + 128 > n) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int64_t left = n - (r0 + 32 * j);
        r[j] &= left >= 32 ? 0xFFFFFFFFu : (left <= 0 ? 0u : ((1u << left) - 1u));
      }
    }
    out[w] = make_uint4(r[0], r[1], r[2], r[3]);
  }
}

// tile_count[t] = the set bits of rows [t * 2048, (t + 1) * 2048) below n: one warp per tile, 8
// mask bytes per lane
__global__ void __launch_bounds__(kFiltThreads)
mask_tile_count_kernel(const uint8_t* __restrict__ mask, int64_t n, int64_t ntiles, int64_t* __restrict__ tile_count) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x / 32);
  for (int64_t t = (int64_t)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); t < ntiles; t += warps) {
    const int64_t r0 = t * kMaskTile + (int64_t)lane * 64;
    unsigned cnt = 0;
    if (r0 < n) {
      const uint2 w = __ldg(reinterpret_cast<const uint2*>(mask + (r0 >> 3)));
      uint64_t bits = ((uint64_t)w.y << 32) | w.x;
      if (r0 + 64 > n) bits &= (1ull << (n - r0)) - 1ull;
      cnt = (unsigned)__popcll(bits);
    }
    cnt = __reduce_add_sync(0xFFFFFFFFu, cnt);
    if (lane == 0) tile_count[t] = (int64_t)cnt;
  }
}

// one CTA per tile, one mask byte per lane: the lane's output position is the tile base plus a
// block exclusive scan of the bytes' popcounts
__global__ void __launch_bounds__(kScanTileThreads)
mask_select_kernel(const uint8_t* __restrict__ mask, int64_t n, const int64_t* __restrict__ tile_off,
                   int64_t* __restrict__ rows_out) {
  __shared__ long long ws[kScanTileThreads / 32 + 1];
  const int64_t i0 = (int64_t)blockIdx.x * kMaskTile + (int64_t)threadIdx.x * 8;
  unsigned m = 0;
  if (i0 < n) m = __ldg(mask + (i0 >> 3)) & tail8(i0 >> 3, n);
  long long tot;
  long long pos = __ldg(tile_off + blockIdx.x) + block_excl_scan_i64<kScanTileThreads>(__popc(m), ws, &tot);
  while (m != 0) {
    rows_out[pos++] = i0 + (__ffs(m) - 1);
    m &= m - 1;
  }
}

template <typename C>
int launch_compare(const nvtb_col_t* a, const nvtb_col_t* b, C s, int op, int64_t n, uint8_t* out, cudaStream_t st) {
  nvtb_col_t none;
  memset(&none, 0, sizeof(none));
  const nvtb_col_t bb = b != nullptr ? *b : none;
  mask_compare_kernel<C><<<filt_grid(mask_bytes(n)), kFiltThreads, 0, st>>>(
      *a, vec_ok(a->data, a->dtype), bb, b != nullptr && vec_ok(b->data, b->dtype), s, op, n, out);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

inline bool is_fixed(int dt) {
  return dt == NVTB_I32 || dt == NVTB_I64 || dt == NVTB_F32 || dt == NVTB_F64 || dt == NVTB_U8;
}

}  // namespace
}  // namespace nvtb

using namespace nvtb;

extern "C" {

int nvtb_mask_compare(const nvtb_col_t* a, const nvtb_col_t* b, int op, int cmp_type, uint64_t scalar_bits,
                      int64_t n, uint8_t* mask_out, void* stream) {
  NVTB_REQUIRE(a != nullptr && n >= 0, "bad arguments");
  NVTB_REQUIRE(op >= NVTB_CMP_EQ && op <= NVTB_CMP_GE, "unknown comparison");
  NVTB_REQUIRE(cmp_type == NVTB_I64 || cmp_type == NVTB_F32 || cmp_type == NVTB_F64, "cmp_type must be I64, F32 or F64");
  NVTB_REQUIRE(is_fixed(a->dtype) && (b == nullptr || is_fixed(b->dtype)), "unsupported operand dtype");
  const auto is_float = [](int dt) { return dt == NVTB_F32 || dt == NVTB_F64; };
  NVTB_REQUIRE(cmp_type != NVTB_I64 || (!is_float(a->dtype) && (b == nullptr || !is_float(b->dtype))),
               "a float operand cannot be compared as int64");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(a->data != nullptr && (b == nullptr || b->data != nullptr) && mask_out != nullptr, "NULL operand / mask");
  cudaStream_t st = (cudaStream_t)stream;
  switch (cmp_type) {
    case NVTB_I64: return launch_compare<int64_t>(a, b, (int64_t)scalar_bits, op, n, mask_out, st);
    case NVTB_F32: {
      float s;
      const uint32_t lo = (uint32_t)scalar_bits;
      memcpy(&s, &lo, sizeof(s));
      return launch_compare<float>(a, b, s, op, n, mask_out, st);
    }
    default: {
      double s;
      memcpy(&s, &scalar_bits, sizeof(s));
      return launch_compare<double>(a, b, s, op, n, mask_out, st);
    }
  }
}

int nvtb_mask_notnull(const nvtb_col_t* cols, int ncols, int64_t n, uint8_t* mask_out, void* stream) {
  NVTB_REQUIRE(cols != nullptr && n >= 0, "bad arguments");
  NVTB_REQUIRE(ncols >= 1 && ncols <= kMaxNotnullCols, "ncols must be in [1, 16]");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(mask_out != nullptr, "NULL mask");
  NotnullCols c;
  memset(&c, 0, sizeof(c));
  c.n = ncols;
  for (int q = 0; q < ncols; ++q) {
    NVTB_REQUIRE(is_fixed(cols[q].dtype), "unsupported column dtype");
    NVTB_REQUIRE(cols[q].data != nullptr, "NULL column data");
    c.data[q] = cols[q].data;
    c.valid[q] = cols[q].validity;
    c.dtype[q] = cols[q].dtype;
    if (vec_ok(cols[q].data, cols[q].dtype)) c.vec |= 1u << q;
  }
  mask_notnull_kernel<<<filt_grid(mask_bytes(n)), kFiltThreads, 0, (cudaStream_t)stream>>>(c, n, mask_out);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

int nvtb_mask_logic(const uint8_t* a, const uint8_t* b, int64_t n, int op, uint8_t* out, void* stream) {
  NVTB_REQUIRE(n >= 0, "n < 0");
  NVTB_REQUIRE(op >= NVTB_MASK_AND && op <= NVTB_MASK_NOT, "unknown mask operation");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(a != nullptr && out != nullptr && (op == NVTB_MASK_NOT || b != nullptr), "NULL mask");
  const auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
  NVTB_REQUIRE(al16(a) && al16(out) && (b == nullptr || al16(b)), "masks must be 16-byte aligned");
  mask_logic_kernel<<<filt_grid(mask_bytes(n) / 16), kFiltThreads, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const uint4*>(a), op == NVTB_MASK_NOT ? nullptr : reinterpret_cast<const uint4*>(b), n, op,
      reinterpret_cast<uint4*>(out));
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

int nvtb_mask_count(const uint8_t* mask, int64_t n, int64_t* tile_off, int64_t* n_kept_host, void* stream) {
  NVTB_REQUIRE(n >= 0 && n_kept_host != nullptr, "bad arguments");
  *n_kept_host = 0;
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(mask != nullptr && (reinterpret_cast<uintptr_t>(mask) & 7u) == 0, "mask must be 8-byte aligned");
  NVTB_REQUIRE(tile_off != nullptr && is_aligned32(tile_off), "tile_off must be non-NULL and 32-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t ntiles = (n + kMaskTile - 1) / kMaskTile;
  mask_tile_count_kernel<<<filt_grid(ntiles * 32), kFiltThreads, 0, st>>>(mask, n, ntiles, tile_off);
  NVTB_LAUNCH_OK();
  return excl_scan_i64(tile_off, ntiles, n_kept_host, st);
}

int nvtb_mask_select(const uint8_t* mask, int64_t n, const int64_t* tile_off, int64_t* rows_out, void* stream) {
  NVTB_REQUIRE(n >= 0, "n < 0");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(mask != nullptr && tile_off != nullptr && rows_out != nullptr, "NULL argument");
  const int64_t ntiles = (n + kMaskTile - 1) / kMaskTile;
  mask_select_kernel<<<(unsigned)ntiles, kScanTileThreads, 0, (cudaStream_t)stream>>>(mask, n, tile_off, rows_out);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

}  // extern "C"
