// groupby.cu — K8: the session group-by (Groupby operator) and the row routing of
// Dataset.shuffle_by_keys, on sm_90a.
//
// Replaces, per partition, the cuDF / pandas calls of reference nvtabular/ops/groupby.py:
//   df.sort_values(sort_cols, ascending=...)                              groupby.py:118-120
//   df.groupby(groupby_cols).agg({col: [count, sum, ..., list]})          groupby.py:222-227
//   _first_or_last: x.list.get(0) / x.list.get(-1)                        groupby.py:290-313
// and, for shuffle_by_keys, merlin.io.Dataset.shuffle_by_keys's hash partition + concat.
//
// Stages (nvtabular_b200/ops/groupby.py drives them):
//   1. order codes   one streaming pass per key / sort column: a uint64 code per row whose
//                    unsigned order is the column's order, a validity bitmask (null or NaN =
//                    invalid), and {min, max, n_valid} of the valid codes
//   2. order rows    LSD rounds of the radix primitive (radix.cuh, rx_sort_bits) over elements
//                    (packed fields << r) | row; every round rewrites the high bits in place
//   3. segments      boundary flags of the sorted rows + a tile scan -> int64 group offsets
//   4. gather        the value columns into group order (the `list` leaves; gather.cu)
//   5. reduce        count / sum / mean / var / std / min / max per segment in fp64, in a
//                    fixed order (warp per segment; long segments one CTA each)
//   6. rank stats    median / nunique over rows ordered by (group, value) with stage 2
// No floating-point atomics anywhere: outputs are bit-identical from run to run.
#include "common.cuh"
#include "radix.cuh"
#include "scan.cuh"

namespace nvtb {
namespace {

constexpr int kGbThreads = 256;
constexpr int kGbTileRows = kGbThreads * kRows;        // 2048 positions per tile: one flag byte per lane
constexpr int64_t kLongSegment = 1 << 14;              // segments above this are reduced by a whole CTA
constexpr int kLongThreads = 256;
constexpr int kMaxChunks = 16;
constexpr int kMaxKeys = 16;

struct Chunk {
  const uint64_t* codes;
  const uint8_t* valid;
  uint64_t min;
  uint64_t span;   // max - min of the valid codes
  int32_t mode;    // 0 key value, 1 ascending (null slot last), 2 descending (null slot last), 3 null flag
  int32_t lo;      // lowest bit of the field value this chunk takes
  int32_t nbits;
  int32_t _pad;
};
struct RoundDesc {
  Chunk c[kMaxChunks];
  int n;
};
struct KeyCodes {
  const uint64_t* codes[kMaxKeys];
  int n;
};

// ---------------------------------------------------------------------------------------
// 1. order codes
// ---------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ uint64_t order_code(T x, bool& ok) {
  if constexpr (std::is_same<T, int32_t>::value) {
    return (uint64_t)((uint32_t)x ^ 0x80000000u);
  } else if constexpr (std::is_same<T, int64_t>::value) {
    return (uint64_t)x ^ 0x8000000000000000ull;
  } else if constexpr (std::is_same<T, float>::value) {
    if (isnan(x)) { ok = false; return 0; }
    const uint32_t u = __float_as_uint(x + 0.0f);                 // -0.0 -> +0.0
    return (uint64_t)((u & 0x80000000u) ? ~u : (u | 0x80000000u));
  } else if constexpr (std::is_same<T, double>::value) {
    if (isnan(x)) { ok = false; return 0; }
    const uint64_t u = (uint64_t)__double_as_longlong(x + 0.0);
    return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
  } else {
    return (uint64_t)x;                                            // uint8 / bool
  }
}

// every lane owns 8 consecutive rows (one validity byte); the vector path loads them with the
// two-128-bit-access layout of common.cuh.  stats: {min, max, n_valid} of the valid codes.
template <typename T>
__global__ void __launch_bounds__(kGbThreads)
codes_kernel(const T* __restrict__ data, const uint8_t* __restrict__ mask, int64_t n, bool aligned,
             uint64_t* __restrict__ codes, uint8_t* __restrict__ valid_out, uint8_t* __restrict__ key_valid,
             int and_key_valid, unsigned long long* __restrict__ stats) {
  uint64_t mn = ~0ull, mx = 0ull, cnt = 0;
  const int64_t ngroups = (n + 7) / 8;
  for (int64_t gi = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; gi < ngroups; gi += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = gi * 8;
    T v[8];
    unsigned m;
    if (aligned && i + 8 <= n) {
      if constexpr (sizeof(T) == 1) {
        const uint2 q = __ldg(reinterpret_cast<const uint2*>(data + i));
#pragma unroll
        for (int k = 0; k < 4; ++k) { v[k] = (T)(q.x >> (8 * k)); v[4 + k] = (T)(q.y >> (8 * k)); }
      } else {
        ld_rows8<T>(data + i, v);
      }
      m = valid8(mask, i);
    } else {
      m = 0;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const bool in = i + k < n;
        v[k] = in ? data[i + k] : (T)0;
        if (in && valid1(mask, i + k)) m |= 1u << k;
      }
    }
    uint64_t c[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      bool ok = (m >> k) & 1u;
      c[k] = order_code<T>(v[k], ok);
      if (!ok) { m &= ~(1u << k); c[k] = 0; }
      if ((m >> k) & 1u) { mn = c[k] < mn ? c[k] : mn; mx = c[k] > mx ? c[k] : mx; ++cnt; }
    }
    if (i + 8 <= n) {
      st_rows8<uint64_t>(codes + i, c);
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) if (i + k < n) codes[i + k] = c[k];
    }
    valid_out[gi] = (uint8_t)m;
    if (key_valid != nullptr) key_valid[gi] = and_key_valid ? (uint8_t)(key_valid[gi] & m) : (uint8_t)m;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const uint64_t a = __shfl_xor_sync(0xFFFFFFFFu, mn, o);
    const uint64_t b = __shfl_xor_sync(0xFFFFFFFFu, mx, o);
    mn = a < mn ? a : mn;
    mx = b > mx ? b : mx;
    cnt += __shfl_xor_sync(0xFFFFFFFFu, cnt, o);
  }
  if ((threadIdx.x & 31) == 0 && cnt) {
    atomicMin(stats + 0, (unsigned long long)mn);
    atomicMax(stats + 1, (unsigned long long)mx);
    atomicAdd(stats + 2, (unsigned long long)cnt);
  }
}

// ---------------------------------------------------------------------------------------
// 2. one LSD round: rewrite the high bits of every element from its row's codes
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t field_value(const Chunk& c, uint64_t row) {
  const bool ok = valid1(c.valid, (int64_t)row);
  switch (c.mode) {
    case 0: return c.codes[row] - c.min;
    case 1: return ok ? c.codes[row] - c.min : c.span + 1;
    case 2: return ok ? c.span - (c.codes[row] - c.min) : c.span + 1;
    default: return ok ? 0ull : 1ull;
  }
}

__global__ void __launch_bounds__(kGbThreads)
round_pack_kernel(uint64_t* __restrict__ elems, int64_t n, int row_bits, int first, RoundDesc rd) {
  const uint64_t row_mask = row_bits >= 64 ? ~0ull : ((1ull << row_bits) - 1ull);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint64_t row = first ? (uint64_t)i : (elems[i] & row_mask);
    uint64_t packed = 0;
    int pos = 0;
    for (int j = 0; j < rd.n; ++j) {
      const Chunk& c = rd.c[j];
      const uint64_t v = field_value(c, row) >> c.lo;
      const uint64_t m = c.nbits >= 64 ? ~0ull : ((1ull << c.nbits) - 1ull);
      packed |= (v & m) << pos;
      pos += c.nbits;
    }
    elems[i] = (row_bits >= 64 ? 0ull : (packed << row_bits)) | row;
  }
}

// ---------------------------------------------------------------------------------------
// 3. segments
// ---------------------------------------------------------------------------------------
template <int T>
__device__ __forceinline__ uint32_t block_excl_scan_u32(uint32_t v, uint32_t* ws /*[T/32 + 1]*/, uint32_t* total) {
  uint32_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if ((threadIdx.x & 31) >= o) incl += y;
  }
  if ((threadIdx.x & 31) == 31) ws[threadIdx.x >> 5] = incl;
  __syncthreads();
  if (threadIdx.x < 32) {
    const uint32_t w = threadIdx.x < T / 32 ? ws[threadIdx.x] : 0u;
    uint32_t wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, wi, o);
      if (threadIdx.x >= o) wi += y;
    }
    if (threadIdx.x < T / 32) ws[threadIdx.x] = wi - w;
    if (threadIdx.x == T / 32 - 1) ws[T / 32] = wi;
  }
  __syncthreads();
  const uint32_t out = ws[threadIdx.x >> 5] + incl - v;
  *total = ws[T / 32];
  __syncthreads();
  return out;
}

// a position starts a group when its row has valid keys and its key codes differ from the
// previous position's (null-key rows are sorted behind every valid one, so they form a suffix)
__global__ void __launch_bounds__(kGbThreads)
seg_flags_kernel(const uint64_t* __restrict__ order, int64_t n, int row_bits, KeyCodes keys,
                 const uint8_t* __restrict__ key_valid, uint8_t* __restrict__ flags,
                 uint32_t* __restrict__ tile_cnt, uint32_t* __restrict__ tile_kv) {
  __shared__ uint32_t ws[kGbThreads / 32 + 1];
  const uint64_t row_mask = (1ull << row_bits) - 1ull;
  const int64_t p0 = (int64_t)blockIdx.x * kGbTileRows + (int64_t)threadIdx.x * 8;
  unsigned f = 0, kv = 0;
  if (p0 < n) {
    uint64_t prev = p0 > 0 ? (order[p0 - 1] & row_mask) : 0;
    for (int k = 0; k < 8 && p0 + k < n; ++k) {
      const int64_t p = p0 + k;
      const uint64_t row = order[p] & row_mask;
      if (valid1(key_valid, (int64_t)row)) {
        kv |= 1u << k;
        bool differs = p == 0;
        for (int j = 0; j < keys.n && !differs; ++j) differs = keys.codes[j][row] != keys.codes[j][prev];
        if (differs) f |= 1u << k;
      }
      prev = row;
    }
    flags[p0 >> 3] = (uint8_t)f;
  }
  uint32_t tot_f, tot_kv;
  block_excl_scan_u32<kGbThreads>((uint32_t)__popc(f), ws, &tot_f);
  block_excl_scan_u32<kGbThreads>((uint32_t)__popc(kv), ws, &tot_kv);
  if (threadIdx.x == 0) { tile_cnt[blockIdx.x] = tot_f; tile_kv[blockIdx.x] = tot_kv; }
}

// one CTA: exclusive scan of the tile flag counts; totals[0] = groups, totals[1] = rows kept
__global__ void __launch_bounds__(1024)
tile_scan_kernel(const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ kv, int64_t ntiles,
                 uint32_t* __restrict__ scan, unsigned long long* __restrict__ totals) {
  __shared__ uint32_t ws[1024 / 32 + 1];
  uint64_t carry = 0, kept = 0;
  for (int64_t c0 = 0; c0 < ntiles; c0 += 1024) {
    const int64_t i = c0 + threadIdx.x;
    const uint32_t v = i < ntiles ? cnt[i] : 0u;
    uint32_t tot;
    const uint32_t ex = block_excl_scan_u32<1024>(v, ws, &tot);
    if (i < ntiles) scan[i] = (uint32_t)(carry + ex);
    carry += tot;
    const uint32_t k = i < ntiles ? kv[i] : 0u;
    uint32_t ktot;
    block_excl_scan_u32<1024>(k, ws, &ktot);
    kept += ktot;
  }
  if (threadIdx.x == 0) { totals[0] = carry; totals[1] = kept; }
}

__global__ void __launch_bounds__(kGbThreads)
seg_offsets_kernel(const uint8_t* __restrict__ flags, const uint32_t* __restrict__ scan, int64_t n,
                   int64_t n_groups, int64_t n_kept, int64_t* __restrict__ off) {
  __shared__ uint32_t ws[kGbThreads / 32 + 1];
  const int64_t p0 = (int64_t)blockIdx.x * kGbTileRows + (int64_t)threadIdx.x * 8;
  const unsigned f = p0 < n ? flags[p0 >> 3] : 0u;
  uint32_t tot;
  uint32_t g = scan[blockIdx.x] + block_excl_scan_u32<kGbThreads>((uint32_t)__popc(f), ws, &tot);
  for (int k = 0; k < 8; ++k)
    if ((f >> k) & 1u) off[g++] = p0 + k;
  if (blockIdx.x == 0 && threadIdx.x == 0) off[n_groups] = n_kept;
}

// gid[p] = g for off[g] <= p < off[g + 1] (binary search: balanced whatever the lengths)
__global__ void __launch_bounds__(kGbThreads)
segment_ids_kernel(const int64_t* __restrict__ off, int64_t n_groups, int64_t n, uint64_t* __restrict__ gid) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = n_groups;             // last g with off[g] <= p
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) >> 1;
      if (__ldg(off + mid) <= p) lo = mid; else hi = mid;
    }
    gid[p] = (uint64_t)lo;
  }
}

// ---------------------------------------------------------------------------------------
// 5. segmented reductions
// ---------------------------------------------------------------------------------------
struct ReduceOut {
  int32_t* count;
  float* sum;
  float* mean;
  float* var;
  float* stdev;
  void* min;
  void* max;
  uint32_t* min_valid;   // int min / max: bit g clear when the group has no value
  uint32_t* max_valid;
};

struct Acc {
  double cnt, sum, mn, mx;   // mn / mx of the value as double (float columns)
  int64_t imn, imx;          // exact min / max of integer columns
};

template <typename T>
__device__ __forceinline__ bool load_value(const T* __restrict__ d, const uint8_t* __restrict__ v, int64_t p, T& x) {
  if (!valid1(v, p)) return false;
  x = d[p];
  if constexpr (std::is_floating_point<T>::value) return !isnan(x);
  return true;
}

__device__ __forceinline__ void acc_merge(Acc& a, const Acc& b) {
  a.cnt += b.cnt;
  a.sum += b.sum;
  a.mn = fmin(a.mn, b.mn);
  a.mx = fmax(a.mx, b.mx);
  a.imn = b.imn < a.imn ? b.imn : a.imn;
  a.imx = b.imx > a.imx ? b.imx : a.imx;
}

__device__ __forceinline__ Acc acc_shfl(const Acc& a, int o) {
  Acc b;
  b.cnt = __shfl_xor_sync(0xFFFFFFFFu, a.cnt, o);
  b.sum = __shfl_xor_sync(0xFFFFFFFFu, a.sum, o);
  b.mn = __shfl_xor_sync(0xFFFFFFFFu, a.mn, o);
  b.mx = __shfl_xor_sync(0xFFFFFFFFu, a.mx, o);
  b.imn = __shfl_xor_sync(0xFFFFFFFFu, a.imn, o);
  b.imx = __shfl_xor_sync(0xFFFFFFFFu, a.imx, o);
  return b;
}

template <typename T>
__device__ __forceinline__ void write_result(const ReduceOut& o, int64_t g, const Acc& a, double m2) {
  const int64_t n = (int64_t)a.cnt;
  const double nan = __longlong_as_double(0x7FF8000000000000ll);
  if (o.count) o.count[g] = (int32_t)n;
  if (o.sum) o.sum[g] = (float)a.sum;
  if (o.mean) o.mean[g] = n ? (float)(a.sum / a.cnt) : (float)nan;
  const double var = n >= 2 ? m2 / (a.cnt - 1.0) : nan;
  if (o.var) o.var[g] = (float)var;
  if (o.stdev) o.stdev[g] = (float)sqrt(var);
  if constexpr (std::is_floating_point<T>::value) {
    if (o.min) static_cast<T*>(o.min)[g] = n ? (T)a.mn : (T)nan;
    if (o.max) static_cast<T*>(o.max)[g] = n ? (T)a.mx : (T)nan;
  } else {
    if (o.min) static_cast<T*>(o.min)[g] = n ? (T)a.imn : (T)0;
    if (o.max) static_cast<T*>(o.max)[g] = n ? (T)a.imx : (T)0;
    if (n && o.min_valid) atomicOr(o.min_valid + (g >> 5), 1u << (g & 31));
    if (n && o.max_valid) atomicOr(o.max_valid + (g >> 5), 1u << (g & 31));
  }
}

template <typename T>
__device__ __forceinline__ void acc_add(Acc& a, T x) {
  a.cnt += 1.0;
  a.sum += (double)x;
  if constexpr (std::is_floating_point<T>::value) {
    a.mn = fmin(a.mn, (double)x);
    a.mx = fmax(a.mx, (double)x);
  } else {
    a.imn = (int64_t)x < a.imn ? (int64_t)x : a.imn;
    a.imx = (int64_t)x > a.imx ? (int64_t)x : a.imx;
  }
}

__device__ __forceinline__ Acc acc_empty() {
  const double nan = __longlong_as_double(0x7FF8000000000000ll);
  return Acc{0.0, 0.0, nan, nan, INT64_MAX, INT64_MIN};
}

// warp per segment: lane l takes rows s + l, s + l + 32, ... (a fixed assignment), the
// butterfly combine is symmetric, so the result never depends on timing.  var is a second pass
// around the mean (sum of squares minus square of sums loses every digit on timestamps).
template <typename T>
__global__ void __launch_bounds__(kGbThreads)
reduce_warp_kernel(const T* __restrict__ d, const uint8_t* __restrict__ v, const int64_t* __restrict__ off,
                   int64_t n_groups, ReduceOut o, bool need_m2, uint32_t* __restrict__ long_list,
                   unsigned int* __restrict__ n_long) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x / 32);
  for (int64_t g = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; g < n_groups; g += warps) {
    const int64_t s = off[g], e = off[g + 1];
    if (e - s > kLongSegment) {
      if (lane == 0) long_list[atomicAdd(n_long, 1u)] = (uint32_t)g;
      continue;
    }
    Acc a = acc_empty();
    for (int64_t p = s + lane; p < e; p += 32) {
      T x;
      if (load_value(d, v, p, x)) acc_add(a, x);
    }
#pragma unroll
    for (int o2 = 16; o2 > 0; o2 >>= 1) acc_merge(a, acc_shfl(a, o2));
    double m2 = 0.0;
    if (need_m2 && a.cnt >= 2.0) {
      const double mean = a.sum / a.cnt;
      for (int64_t p = s + lane; p < e; p += 32) {
        T x;
        if (load_value(d, v, p, x)) { const double dx = (double)x - mean; m2 += dx * dx; }
      }
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) m2 += __shfl_xor_sync(0xFFFFFFFFu, m2, o2);
    }
    if (lane == 0) write_result<T>(o, g, a, m2);
  }
}

// one CTA per long segment; thread t takes rows s + t, s + t + kLongThreads, ..., and the
// partials combine in a fixed tree
template <typename T>
__global__ void __launch_bounds__(kLongThreads)
reduce_long_kernel(const T* __restrict__ d, const uint8_t* __restrict__ v, const int64_t* __restrict__ off,
                   ReduceOut o, bool need_m2, const uint32_t* __restrict__ long_list,
                   const unsigned int* __restrict__ n_long) {
  __shared__ Acc sa[kLongThreads / 32];
  __shared__ double sm[kLongThreads / 32];
  __shared__ double s_mean;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned nl = *n_long;
  for (unsigned li = blockIdx.x; li < nl; li += gridDim.x) {
    const int64_t g = long_list[li];
    const int64_t s = off[g], e = off[g + 1];
    Acc a = acc_empty();
    for (int64_t p = s + threadIdx.x; p < e; p += kLongThreads) {
      T x;
      if (load_value(d, v, p, x)) acc_add(a, x);
    }
#pragma unroll
    for (int o2 = 16; o2 > 0; o2 >>= 1) acc_merge(a, acc_shfl(a, o2));
    if (lane == 0) sa[warp] = a;
    __syncthreads();
    if (warp == 0) {
      Acc w = lane < kLongThreads / 32 ? sa[lane] : acc_empty();
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) acc_merge(w, acc_shfl(w, o2));
      if (lane == 0) { sa[0] = w; s_mean = w.cnt > 0 ? w.sum / w.cnt : 0.0; }
    }
    __syncthreads();
    const Acc tot = sa[0];
    double m2 = 0.0;
    if (need_m2 && tot.cnt >= 2.0) {
      const double mean = s_mean;
      for (int64_t p = s + threadIdx.x; p < e; p += kLongThreads) {
        T x;
        if (load_value(d, v, p, x)) { const double dx = (double)x - mean; m2 += dx * dx; }
      }
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) m2 += __shfl_xor_sync(0xFFFFFFFFu, m2, o2);
      if (lane == 0) sm[warp] = m2;
      __syncthreads();
      if (warp == 0) {
        m2 = lane < kLongThreads / 32 ? sm[lane] : 0.0;
#pragma unroll
        for (int o2 = 16; o2 > 0; o2 >>= 1) m2 += __shfl_xor_sync(0xFFFFFFFFu, m2, o2);
      }
    }
    if (threadIdx.x == 0) write_result<T>(o, g, tot, m2);
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------
// 6. median / nunique over positions ordered by (group, value code), nulls last in a group
// ---------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kGbThreads)
rank_stats_kernel(const T* __restrict__ d, const uint64_t* __restrict__ codes, const uint8_t* __restrict__ cvalid,
                  const uint64_t* __restrict__ order, uint64_t row_mask, const int64_t* __restrict__ off,
                  int64_t n_groups, float* __restrict__ median, int32_t* __restrict__ nunique) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x / 32);
  for (int64_t g = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; g < n_groups; g += warps) {
    const int64_t s = off[g], e = off[g + 1];
    // the valid values are a prefix of the segment: find its end
    int64_t lo = s, hi = e;                   // first invalid position in [s, e]
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (valid1(cvalid, (int64_t)(order[mid] & row_mask))) lo = mid + 1; else hi = mid;
    }
    const int64_t cnt = lo - s;
    if (nunique != nullptr) {
      int32_t c = 0;
      for (int64_t p = s + lane; p < s + cnt; p += 32)
        c += (p == s || codes[order[p] & row_mask] != codes[order[p - 1] & row_mask]) ? 1 : 0;
#pragma unroll
      for (int o2 = 16; o2 > 0; o2 >>= 1) c += __shfl_xor_sync(0xFFFFFFFFu, c, o2);
      if (lane == 0) nunique[g] = c;
    }
    if (median != nullptr && lane == 0) {
      if (cnt == 0) {
        median[g] = __int_as_float(0x7FC00000);
      } else {
        const double a = (double)d[order[s + (cnt - 1) / 2] & row_mask];
        const double b = (double)d[order[s + cnt / 2] & row_mask];
        median[g] = (float)((cnt & 1) ? a : (a + b) / 2.0);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------
// sub-lists of a list column (first / last of a list input, ListSlice): output row g holds
// leaves[lo[g], hi[g]).  Its offsets are the exclusive scan (scan.cuh) of the lengths.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kGbThreads)
list_lengths_kernel(const int64_t* __restrict__ lo, const int64_t* __restrict__ hi, int64_t m,
                    int64_t* __restrict__ len) {
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < m; g += (int64_t)gridDim.x * blockDim.x)
    len[g] = __ldg(hi + g) - __ldg(lo + g);
}

// last g in [a, b) with off[g] <= p (off[a] <= p is given)
__device__ __forceinline__ int64_t last_at_or_below(const int64_t* __restrict__ off, int64_t a, int64_t b, int64_t p) {
  while (b - a > 1) {
    const int64_t mid = (a + b) >> 1;
    if (__ldg(off + mid) <= p) a = mid; else b = mid;
  }
  return a;
}

// Balanced over OUTPUT positions: every lane owns 8 consecutive ones (one validity byte, so no
// atomics) and finds the sub-list of each by binary search over off, inside the bracket of its
// first and last position's sub-lists.  A table of 10^7 short lists keeps every lane busy.
template <typename T>
__global__ void __launch_bounds__(kGbThreads)
list_copy_kernel(const T* __restrict__ src, const uint8_t* __restrict__ src_valid, const int64_t* __restrict__ lo,
                 const int64_t* __restrict__ off, int64_t m, int64_t total, bool aligned, T* __restrict__ out,
                 uint8_t* __restrict__ out_valid) {
  const int64_t nchunks = (total + 7) / 8;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p0 = c * 8;
    const int64_t pe = p0 + 7 < total ? p0 + 7 : total - 1;
    const int64_t g0 = last_at_or_below(off, 0, m, p0);
    const int64_t g1 = last_at_or_below(off, g0, m, pe);
    T v[8];
    unsigned vb = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int64_t p = p0 + k <= pe ? p0 + k : pe;
      const int64_t g = last_at_or_below(off, g0, g1 + 1, p);
      const int64_t s = __ldg(lo + g) + (p - __ldg(off + g));
      v[k] = src[s];
      if (p0 + k <= pe && valid1(src_valid, s)) vb |= 1u << k;
    }
    if (aligned && p0 + 8 <= total) {
      st_rows8<T>(out + p0, v);
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) if (p0 + k < total) out[p0 + k] = v[k];
    }
    if (out_valid != nullptr) out_valid[p0 >> 3] = (uint8_t)vb;
  }
}

}  // namespace
}  // namespace nvtb

using namespace nvtb;

extern "C" {

int nvtb_gb_order_codes(const nvtb_col_t* col, int64_t n, uint64_t* codes_out, uint8_t* valid_out,
                        uint8_t* key_valid, int and_key_valid, uint64_t* stats_dev, void* stream) {
  NVTB_REQUIRE(col != nullptr && n >= 0 && stats_dev != nullptr, "NULL column / stats or n < 0");
  cudaStream_t st = (cudaStream_t)stream;
  NVTB_CUDA_OK(cudaMemsetAsync(stats_dev, 0xFF, sizeof(uint64_t), st));
  NVTB_CUDA_OK(cudaMemsetAsync(stats_dev + 1, 0, 2 * sizeof(uint64_t), st));
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(col->data && codes_out && valid_out, "NULL data / codes / validity");
  NVTB_REQUIRE(is_aligned32(codes_out), "codes_out must be 32-byte aligned");
  const bool aligned = is_aligned32(col->data);
  const int grid = grid_for((n + 7) / 8, kGbThreads);
  unsigned long long* s = reinterpret_cast<unsigned long long*>(stats_dev);
  switch (col->dtype) {
    case NVTB_I32: codes_kernel<int32_t><<<grid, kGbThreads, 0, st>>>((const int32_t*)col->data, col->validity, n, aligned, codes_out, valid_out, key_valid, and_key_valid, s); break;
    case NVTB_I64: codes_kernel<int64_t><<<grid, kGbThreads, 0, st>>>((const int64_t*)col->data, col->validity, n, aligned, codes_out, valid_out, key_valid, and_key_valid, s); break;
    case NVTB_F32: codes_kernel<float><<<grid, kGbThreads, 0, st>>>((const float*)col->data, col->validity, n, aligned, codes_out, valid_out, key_valid, and_key_valid, s); break;
    case NVTB_F64: codes_kernel<double><<<grid, kGbThreads, 0, st>>>((const double*)col->data, col->validity, n, aligned, codes_out, valid_out, key_valid, and_key_valid, s); break;
    case NVTB_U8: codes_kernel<uint8_t><<<grid, kGbThreads, 0, st>>>((const uint8_t*)col->data, col->validity, n, aligned && ((reinterpret_cast<uintptr_t>(col->data) & 7u) == 0), codes_out, valid_out, key_valid, and_key_valid, s); break;
    default: set_error("nvtb_gb_order_codes: unsupported dtype %d", (int)col->dtype); return NVTB_EINVAL;
  }
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

int nvtb_gb_order_rows(const nvtb_gb_chunk_t* chunks_host, const int* round_sizes_host, int n_rounds, int64_t n,
                       int row_bits, uint64_t* elems, uint64_t* tmp, int* result_in_tmp_host, void* stream) {
  static_assert(sizeof(nvtb_gb_chunk_t) == sizeof(Chunk), "chunk layout");
  NVTB_REQUIRE(result_in_tmp_host != nullptr && n >= 0 && n_rounds >= 0, "bad arguments");
  NVTB_REQUIRE(n < ((int64_t)1 << 32), "a partition holds at most 2^32 - 1 rows");
  NVTB_REQUIRE(row_bits >= 0 && row_bits <= 32 && (n <= 1 || ((n - 1) >> row_bits) == 0), "row_bits too small for n");
  *result_in_tmp_host = 0;
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(elems != nullptr && tmp != nullptr, "NULL element buffers");
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = grid_for(n, kGbThreads);
  if (n_rounds == 0) {
    RoundDesc rd{};
    rd.n = 0;
    round_pack_kernel<<<grid, kGbThreads, 0, st>>>(elems, n, row_bits, 1, rd);
    NVTB_LAUNCH_OK();
    return NVTB_OK;
  }
  const size_t sbytes = rx_scratch_bytes<uint64_t>(n);
  void* scratch = nullptr;
  NVTB_CUDA_OK(cudaMallocAsync(&scratch, sbytes, st));
  NVTB_CUDA_OK(cudaMemsetAsync(scratch, 0, 256, st));
  uint64_t* a = elems;
  uint64_t* b = tmp;
  int ci = 0, rc = NVTB_OK;
  for (int r = 0; r < n_rounds && rc == NVTB_OK; ++r) {
    const int k = round_sizes_host[r];
    RoundDesc rd{};
    int width = 0;
    if (k < 1 || k > kMaxChunks) { set_error("a round packs 1..%d chunks", kMaxChunks); rc = NVTB_EINVAL; break; }
    for (int j = 0; j < k; ++j) {
      memcpy(&rd.c[j], &chunks_host[ci + j], sizeof(Chunk));
      width += rd.c[j].nbits;
    }
    ci += k;
    rd.n = k;
    if (width < 1 || width > 64 - row_bits) { set_error("round width %d does not fit beside %d row bits", width, row_bits); rc = NVTB_EINVAL; break; }
    round_pack_kernel<<<grid, kGbThreads, 0, st>>>(a, n, row_bits, r == 0, rd);
    if (cudaGetLastError() != cudaSuccess) { set_error("round_pack_kernel launch failed"); rc = NVTB_ECUDA; break; }
    int in_b = 0;
    rc = rx_sort_bits<uint64_t>(nullptr, a, b, nullptr, n, row_bits, row_bits + width, false, scratch, sbytes, st, &in_b);
    if (in_b) { uint64_t* t = a; a = b; b = t; }
  }
  NVTB_CUDA_OK(cudaFreeAsync(scratch, st));
  *result_in_tmp_host = a == tmp ? 1 : 0;
  return rc;
}

int nvtb_gb_segments_count(const uint64_t* order, int64_t n, int row_bits, const uint64_t* const* key_codes_host,
                           int n_keys, const uint8_t* key_valid, uint8_t* flags, uint32_t* tile_scan,
                           int64_t* counts_host, void* stream) {
  NVTB_REQUIRE(n >= 0 && n_keys >= 0 && n_keys <= kMaxKeys && counts_host != nullptr, "bad arguments");
  counts_host[0] = counts_host[1] = 0;
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(order && flags && tile_scan, "NULL buffers");
  cudaStream_t st = (cudaStream_t)stream;
  KeyCodes kc{};
  kc.n = n_keys;
  for (int j = 0; j < n_keys; ++j) kc.codes[j] = key_codes_host[j];
  const int64_t ntiles = (n + kGbTileRows - 1) / kGbTileRows;
  uint32_t* tmp = nullptr;
  NVTB_CUDA_OK(cudaMallocAsync(&tmp, sizeof(uint32_t) * 2 * ntiles + 64, st));
  unsigned long long* totals = reinterpret_cast<unsigned long long*>(tmp + 2 * ntiles);
  seg_flags_kernel<<<(unsigned)ntiles, kGbThreads, 0, st>>>(order, n, row_bits, kc, key_valid, flags, tmp, tmp + ntiles);
  NVTB_LAUNCH_OK();
  tile_scan_kernel<<<1, 1024, 0, st>>>(tmp, tmp + ntiles, ntiles, tile_scan, totals);
  NVTB_LAUNCH_OK();
  unsigned long long h[2] = {0, 0};
  NVTB_CUDA_OK(cudaMemcpyAsync(h, totals, sizeof(h), cudaMemcpyDeviceToHost, st));
  NVTB_CUDA_OK(cudaFreeAsync(tmp, st));
  NVTB_CUDA_OK(cudaStreamSynchronize(st));
  counts_host[0] = (int64_t)h[0];
  counts_host[1] = (int64_t)h[1];
  return NVTB_OK;
}

int nvtb_gb_segments_write(const uint8_t* flags, const uint32_t* tile_scan, int64_t n, int64_t n_groups,
                           int64_t n_kept, int64_t* off_out, void* stream) {
  NVTB_REQUIRE(n >= 0 && n_groups >= 0 && off_out != nullptr, "bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0 || n_groups == 0) {
    const int64_t z = n_kept;
    NVTB_CUDA_OK(cudaMemcpyAsync(off_out + n_groups, &z, sizeof(z), cudaMemcpyHostToDevice, st));
    return cudaStreamSynchronize(st) == cudaSuccess ? NVTB_OK : NVTB_ECUDA;
  }
  const int64_t ntiles = (n + kGbTileRows - 1) / kGbTileRows;
  seg_offsets_kernel<<<(unsigned)ntiles, kGbThreads, 0, st>>>(flags, tile_scan, n, n_groups, n_kept, off_out);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

int nvtb_gb_segment_ids(const int64_t* off, int64_t n_groups, int64_t n, uint64_t* gid_out, void* stream) {
  NVTB_REQUIRE(n >= 0 && n_groups >= 0, "bad sizes");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(off && gid_out && n_groups > 0, "NULL buffers");
  segment_ids_kernel<<<grid_for(n, kGbThreads), kGbThreads, 0, (cudaStream_t)stream>>>(off, n_groups, n, gid_out);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

int nvtb_gb_reduce(const nvtb_col_t* col, const int64_t* off, int64_t n_groups, void* const* outs_host,
                   uint8_t* const* valid_host, void* stream) {
  NVTB_REQUIRE(col != nullptr && n_groups >= 0 && outs_host != nullptr, "bad arguments");
  NVTB_REQUIRE(n_groups < ((int64_t)1 << 32), "too many groups");
  if (n_groups == 0) return NVTB_OK;
  NVTB_REQUIRE(off != nullptr, "NULL offsets");
  cudaStream_t st = (cudaStream_t)stream;
  ReduceOut o;
  o.count = (int32_t*)outs_host[0];
  o.sum = (float*)outs_host[1];
  o.mean = (float*)outs_host[2];
  o.var = (float*)outs_host[3];
  o.stdev = (float*)outs_host[4];
  o.min = outs_host[5];
  o.max = outs_host[6];
  o.min_valid = valid_host ? reinterpret_cast<uint32_t*>(valid_host[0]) : nullptr;
  o.max_valid = valid_host ? reinterpret_cast<uint32_t*>(valid_host[1]) : nullptr;
  const bool need_m2 = o.var != nullptr || o.stdev != nullptr;
  unsigned int* n_long = nullptr;
  NVTB_CUDA_OK(cudaMallocAsync(&n_long, 256 + sizeof(uint32_t) * (size_t)n_groups, st));
  NVTB_CUDA_OK(cudaMemsetAsync(n_long, 0, sizeof(unsigned int), st));
  uint32_t* long_list = reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(n_long) + 256);
  const int gw = grid_for(n_groups, kGbThreads / 32);
  const int gl = sm_count() * 2;
  const void* d = col->data;
  const uint8_t* v = col->validity;
  switch (col->dtype) {
#define NVTB_GB_REDUCE(T)                                                                                   \
  reduce_warp_kernel<T><<<gw, kGbThreads, 0, st>>>((const T*)d, v, off, n_groups, o, need_m2, long_list, n_long); \
  reduce_long_kernel<T><<<gl, kLongThreads, 0, st>>>((const T*)d, v, off, o, need_m2, long_list, n_long);
    case NVTB_I32: NVTB_GB_REDUCE(int32_t) break;
    case NVTB_I64: NVTB_GB_REDUCE(int64_t) break;
    case NVTB_F32: NVTB_GB_REDUCE(float) break;
    case NVTB_F64: NVTB_GB_REDUCE(double) break;
    case NVTB_U8: NVTB_GB_REDUCE(uint8_t) break;
#undef NVTB_GB_REDUCE
    default: set_error("nvtb_gb_reduce: unsupported dtype %d", (int)col->dtype); return NVTB_EINVAL;
  }
  NVTB_LAUNCH_OK();
  NVTB_CUDA_OK(cudaFreeAsync(n_long, st));
  return NVTB_OK;
}

int nvtb_gb_rank_stats(const nvtb_col_t* col, const uint64_t* codes, const uint8_t* codes_valid, const uint64_t* order,
                       uint64_t row_mask, const int64_t* off, int64_t n_groups, float* median_out,
                       int32_t* nunique_out, void* stream) {
  NVTB_REQUIRE(col != nullptr && n_groups >= 0, "bad arguments");
  if (n_groups == 0) return NVTB_OK;
  NVTB_REQUIRE(codes && codes_valid && order && off, "NULL buffers");
  cudaStream_t st = (cudaStream_t)stream;
  const int g = grid_for(n_groups, kGbThreads / 32);
  switch (col->dtype) {
    case NVTB_I32: rank_stats_kernel<int32_t><<<g, kGbThreads, 0, st>>>((const int32_t*)col->data, codes, codes_valid, order, row_mask, off, n_groups, median_out, nunique_out); break;
    case NVTB_I64: rank_stats_kernel<int64_t><<<g, kGbThreads, 0, st>>>((const int64_t*)col->data, codes, codes_valid, order, row_mask, off, n_groups, median_out, nunique_out); break;
    case NVTB_F32: rank_stats_kernel<float><<<g, kGbThreads, 0, st>>>((const float*)col->data, codes, codes_valid, order, row_mask, off, n_groups, median_out, nunique_out); break;
    case NVTB_F64: rank_stats_kernel<double><<<g, kGbThreads, 0, st>>>((const double*)col->data, codes, codes_valid, order, row_mask, off, n_groups, median_out, nunique_out); break;
    case NVTB_U8: rank_stats_kernel<uint8_t><<<g, kGbThreads, 0, st>>>((const uint8_t*)col->data, codes, codes_valid, order, row_mask, off, n_groups, median_out, nunique_out); break;
    default: set_error("nvtb_gb_rank_stats: unsupported dtype %d", (int)col->dtype); return NVTB_EINVAL;
  }
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

int nvtb_gb_list_rows(const nvtb_col_t* leaves, const int64_t* lo, const int64_t* hi, int64_t m, int64_t* off_out,
                      void* out, uint8_t* out_valid, int64_t* total_host, void* stream) {
  NVTB_REQUIRE(leaves != nullptr && m >= 0 && off_out != nullptr && total_host != nullptr, "bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (out == nullptr) {
    *total_host = 0;
    NVTB_REQUIRE(m == 0 || (lo && hi), "NULL bounds");
    // the scan needs 32-byte aligned offsets: scan in a scratch copy when off_out is not
    const bool aligned = is_aligned32(off_out);
    int64_t* buf = off_out;
    if (!aligned) NVTB_CUDA_OK(cudaMallocAsync(&buf, sizeof(int64_t) * (m + 1), st));
    if (m > 0) {
      list_lengths_kernel<<<grid_for(m, kGbThreads), kGbThreads, 0, st>>>(lo, hi, m, buf);
      NVTB_LAUNCH_OK();
    }
    const int rc = excl_scan_i64(buf, m, total_host, st);
    if (!aligned) {
      NVTB_CUDA_OK(cudaMemcpyAsync(off_out, buf, sizeof(int64_t) * (m + 1), cudaMemcpyDeviceToDevice, st));
      NVTB_CUDA_OK(cudaFreeAsync(buf, st));
      NVTB_CUDA_OK(cudaStreamSynchronize(st));
    }
    return rc;
  }
  const int64_t total = *total_host;
  if (m == 0 || total == 0) return NVTB_OK;
  NVTB_REQUIRE(leaves->data && lo, "NULL leaves / bounds");
  const int grid = grid_for((total + 7) / 8, kGbThreads);
  const uintptr_t a = reinterpret_cast<uintptr_t>(out);
  switch (dtype_size(leaves->dtype)) {
    case 1: list_copy_kernel<uint8_t><<<grid, kGbThreads, 0, st>>>((const uint8_t*)leaves->data, leaves->validity, lo, off_out, m, total, (a & 7u) == 0, (uint8_t*)out, out_valid); break;
    case 4: list_copy_kernel<uint32_t><<<grid, kGbThreads, 0, st>>>((const uint32_t*)leaves->data, leaves->validity, lo, off_out, m, total, (a & 31u) == 0, (uint32_t*)out, out_valid); break;
    case 8: list_copy_kernel<uint64_t><<<grid, kGbThreads, 0, st>>>((const uint64_t*)leaves->data, leaves->validity, lo, off_out, m, total, (a & 31u) == 0, (uint64_t*)out, out_valid); break;
    default: set_error("nvtb_gb_list_rows: unsupported dtype %d", (int)leaves->dtype); return NVTB_EINVAL;
  }
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

}  // extern "C"
