// common.cuh — shared device helpers for libnvtb200 (sm_90a).
//
// Nothing here is a port: the reference (NVTabular) has no CUDA sources on this
// path; it calls cuDF/pandas through merlin.core.dispatch.  These helpers give
// the kernels a common column model (typed data + Arrow validity bitmask),
// 128-bit coalesced tile loads, and the two hash functions of the engine.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <type_traits>

#include "../../include/nvtb200.h"

namespace nvtb {

// ---------------------------------------------------------------------------
// error plumbing (thread-local message, status codes; no exceptions escape)
// ---------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int sm_count();
// keep stream-ordered frees cached in the device's default memory pool instead of
// returning them to the OS at every synchronisation (the CUDA default)
void ensure_pool_configured();

#define NVTB_CUDA_OK(expr)                                                    \
  do {                                                                        \
    cudaError_t _e = (expr);                                                  \
    if (_e != cudaSuccess) {                                                  \
      ::nvtb::set_error("%s failed: %s (%s:%d)", #expr,                       \
                        cudaGetErrorString(_e), __FILE__, __LINE__);          \
      return _e == cudaErrorMemoryAllocation ? NVTB_ENOMEM : NVTB_ECUDA;      \
    }                                                                         \
  } while (0)

#define NVTB_REQUIRE(cond, msg)                                               \
  do {                                                                        \
    if (!(cond)) {                                                            \
      ::nvtb::set_error("invalid argument: %s (%s:%d)", msg, __FILE__,        \
                        __LINE__);                                            \
      return NVTB_EINVAL;                                                     \
    }                                                                         \
  } while (0)

#define NVTB_LAUNCH_OK()                                                      \
  do {                                                                        \
    cudaError_t _e = cudaGetLastError();                                      \
    if (_e != cudaSuccess) {                                                  \
      ::nvtb::set_error("kernel launch failed: %s (%s:%d)",                   \
                        cudaGetErrorString(_e), __FILE__, __LINE__);          \
      return NVTB_ECUDA;                                                      \
    }                                                                         \
  } while (0)

inline size_t dtype_size(int dt) {
  switch (dt) {
    case NVTB_I32: return 4;
    case NVTB_I64: return 8;
    case NVTB_F32: return 4;
    case NVTB_F64: return 8;
    case NVTB_U8: return 1;
    case NVTB_H64: return 8;
    default: return 0;
  }
}

// ---------------------------------------------------------------------------
// tile geometry.  Every lane owns kRows = 8 CONSECUTIVE rows per group, i.e.
// one 32-byte sector for 4-byte types and two for 8-byte types.  sm_90 has no
// 256-bit global access, so a sector is moved as two back-to-back 128-bit
// accesses (LDG.E.128 / STG.E.128) from the same thread; both halves fall in
// the same sector, so DRAM traffic is one sector per 8 rows either way.
// A warp therefore touches 1 KB (or 2 KB) of contiguous memory per group, and
// because 8 rows == one validity byte, the Arrow bitmask costs one byte load
// per lane and never straddles lanes or tiles.
// ---------------------------------------------------------------------------
constexpr int kThreads = 256;
constexpr int kRows = 8;                            // rows per lane per group
constexpr int kGroups = 2;                          // groups per thread per tile
constexpr int kTile = kThreads * kRows * kGroups;   // 4096 rows

// L2 eviction policies.  Column data is streamed once: mark it evict-first so that
// hundreds of MB of input/output do not wash the (much smaller) hash / lookup tables
// out of the 50 MB L2; table sectors are marked evict-last.  (Non-volatile asm: the
// compiler hoists the createpolicy out of the tile loops.)
__device__ __forceinline__ uint64_t l2_evict_first() {
  uint64_t p;
  asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_evict_last() {
  uint64_t p;
  asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}

// streaming loads: read-only path, no L1 allocation, L2 evict-first (each byte is used once).
// One 32-byte sector (p 32-byte aligned) as two 128-bit accesses issued back to back.
__device__ __forceinline__ void ld256(const void* __restrict__ p,
                                      uint32_t (&w)[8]) {
  const uint64_t pol = l2_evict_first();
  const char* q = static_cast<const char*>(p);
  asm volatile(
      "ld.global.nc.L1::no_allocate.L2::cache_hint.v4.b32 {%0,%1,%2,%3}, [%4], %5;"
      : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3])
      : "l"(q), "l"(pol));
  asm volatile(
      "ld.global.nc.L1::no_allocate.L2::cache_hint.v4.b32 {%0,%1,%2,%3}, [%4], %5;"
      : "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7])
      : "l"(q + 16), "l"(pol));
}
__device__ __forceinline__ void st256(void* p, const uint32_t (&w)[8]) {
  const uint64_t pol = l2_evict_first();
  char* q = static_cast<char*>(p);
  asm volatile(
      "st.global.L1::no_allocate.L2::cache_hint.v4.b32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(q),
      "r"(w[0]), "r"(w[1]), "r"(w[2]), "r"(w[3]), "l"(pol)
      : "memory");
  asm volatile(
      "st.global.L1::no_allocate.L2::cache_hint.v4.b32 [%0], {%1,%2,%3,%4}, %5;" ::"l"(q + 16),
      "r"(w[4]), "r"(w[5]), "r"(w[6]), "r"(w[7]), "l"(pol)
      : "memory");
}

template <typename T>
__device__ __forceinline__ T from_words(uint32_t lo, uint32_t hi);
template <>
__device__ __forceinline__ int64_t from_words<int64_t>(uint32_t lo,
                                                       uint32_t hi) {
  return (int64_t)(((uint64_t)hi << 32) | lo);
}
template <>
__device__ __forceinline__ double from_words<double>(uint32_t lo, uint32_t hi) {
  return __hiloint2double((int)hi, (int)lo);
}

// load rows [p, p+8) of T (p 32-byte aligned)
template <typename T>
__device__ __forceinline__ void ld_rows8(const T* __restrict__ p, T (&v)[8]) {
  if constexpr (sizeof(T) == 4) {
    uint32_t w[8];
    ld256(p, w);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if constexpr (std::is_same<T, float>::value) v[k] = __uint_as_float(w[k]);
      else v[k] = (T)w[k];
    }
  } else {
    uint32_t a[8], b[8];
    ld256(p, a);
    ld256(p + 4, b);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      v[k] = from_words<T>(a[2 * k], a[2 * k + 1]);
      v[4 + k] = from_words<T>(b[2 * k], b[2 * k + 1]);
    }
  }
}

// store rows [p, p+8) of T.  4/8-byte types need 32-byte alignment, uint8 8.
template <typename T>
__device__ __forceinline__ void st_rows8(T* p, const T (&v)[8]) {
  if constexpr (sizeof(T) == 1) {
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      lo |= (uint32_t)(uint8_t)v[k] << (8 * k);
      hi |= (uint32_t)(uint8_t)v[4 + k] << (8 * k);
    }
    asm volatile("st.global.L1::no_allocate.v2.b32 [%0], {%1,%2};" ::"l"(p),
                 "r"(lo), "r"(hi)
                 : "memory");
  } else if constexpr (sizeof(T) == 4) {
    uint32_t w[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if constexpr (std::is_same<T, float>::value) w[k] = __float_as_uint(v[k]);
      else w[k] = (uint32_t)v[k];
    }
    st256(p, w);
  } else {
    uint32_t a[8], b[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      uint64_t x, y;
      if constexpr (std::is_same<T, double>::value) {
        x = (uint64_t)__double_as_longlong(v[k]);
        y = (uint64_t)__double_as_longlong(v[4 + k]);
      } else {
        x = (uint64_t)v[k];
        y = (uint64_t)v[4 + k];
      }
      a[2 * k] = (uint32_t)x; a[2 * k + 1] = (uint32_t)(x >> 32);
      b[2 * k] = (uint32_t)y; b[2 * k + 1] = (uint32_t)(y >> 32);
    }
    st256(p, a);
    st256(p + 4, b);
  }
}

// validity byte for rows [i, i+8), i % 8 == 0.  NULL mask = all valid.
__device__ __forceinline__ unsigned valid8(const uint8_t* __restrict__ mask,
                                           int64_t i) {
  if (mask == nullptr) return 0xFFu;
  return (unsigned)__ldg(mask + (i >> 3));
}
__device__ __forceinline__ bool valid1(const uint8_t* __restrict__ mask,
                                       int64_t i) {
  if (mask == nullptr) return true;
  return (__ldg(mask + (i >> 3)) >> (i & 7)) & 1u;
}

// Visit every row of [0, n) assigned to this block (grid-stride over tiles of
// kTile rows).  f(row_index, value, is_valid) is called once per row.  The
// vector path needs 32-byte aligned data; otherwise a scalar path is taken.
// All loads of a tile are issued before any row is consumed (MLP = kGroups
// x 32 B x 256 threads = 16 KB in flight per CTA for 4-byte types).
template <typename T, typename F>
__device__ __forceinline__ void for_each_row(const T* __restrict__ data,
                                             const uint8_t* __restrict__ mask,
                                             int64_t n, bool aligned, F&& f) {
  const int64_t n_tiles = (n + kTile - 1) / kTile;
  for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const int64_t base = t * kTile;
    if (aligned && base + kTile <= n) {
      T v[kGroups][kRows];
      unsigned m[kGroups];
#pragma unroll
      for (int g = 0; g < kGroups; ++g) {
        const int64_t i = base + (int64_t)g * (kThreads * kRows) +
                          (int64_t)threadIdx.x * kRows;
        ld_rows8<T>(data + i, v[g]);
        m[g] = valid8(mask, i);
      }
#pragma unroll
      for (int g = 0; g < kGroups; ++g) {
        const int64_t i = base + (int64_t)g * (kThreads * kRows) +
                          (int64_t)threadIdx.x * kRows;
#pragma unroll
        for (int k = 0; k < kRows; ++k) f(i + k, v[g][k], (m[g] >> k) & 1u);
      }
    } else {
      const int64_t end = (base + kTile < n) ? base + kTile : n;
      for (int64_t i = base + threadIdx.x; i < end; i += kThreads)
        f(i, data[i], valid1(mask, i));
    }
  }
}

// Map every row through f(value, is_valid) -> OutT and store it.  Same tiling
// as for_each_row; the vector path needs 32-byte aligned in AND out.
template <typename T, typename OutT, typename F>
__device__ __forceinline__ void map_rows(const T* __restrict__ data,
                                         const uint8_t* __restrict__ mask,
                                         OutT* __restrict__ out, int64_t n,
                                         bool aligned, F&& f) {
  const int64_t n_tiles = (n + kTile - 1) / kTile;
  for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const int64_t base = t * kTile;
    if (aligned && base + kTile <= n) {
      T v[kGroups][kRows];
      unsigned m[kGroups];
#pragma unroll
      for (int g = 0; g < kGroups; ++g) {
        const int64_t i = base + (int64_t)g * (kThreads * kRows) +
                          (int64_t)threadIdx.x * kRows;
        ld_rows8<T>(data + i, v[g]);
        m[g] = valid8(mask, i);
      }
#pragma unroll
      for (int g = 0; g < kGroups; ++g) {
        const int64_t i = base + (int64_t)g * (kThreads * kRows) +
                          (int64_t)threadIdx.x * kRows;
        OutT o[kRows];
#pragma unroll
        for (int k = 0; k < kRows; ++k) o[k] = f(i + k, v[g][k], (m[g] >> k) & 1u);
        st_rows8<OutT>(out + i, o);
      }
    } else {
      const int64_t end = (base + kTile < n) ? base + kTile : n;
      for (int64_t i = base + threadIdx.x; i < end; i += kThreads)
        out[i] = f(i, data[i], valid1(mask, i));
    }
  }
}

__host__ __device__ __forceinline__ bool is_aligned32(const void* p) {
  return (reinterpret_cast<uintptr_t>(p) & 31u) == 0;
}


// grid for a streaming kernel over n rows: enough CTAs to fill every SM a
// few times over, never more than there are tiles.
inline int scan_grid(int64_t n, int ctas_per_sm) {
  int64_t tiles = (n + kTile - 1) / kTile;
  int64_t g = (int64_t)sm_count() * ctas_per_sm;
  if (g > tiles) g = tiles;
  if (g < 1) g = 1;
  return (int)g;
}

// grid for a grid-stride loop of one item per thread (per_block items per CTA): at most 8 CTAs
// per SM
inline int grid_for(int64_t items, int per_block) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((items + per_block - 1) / per_block, (int64_t)sm_count() * 8));
}
inline int plain_grid(int64_t n) { return grid_for(n, kThreads); }

// ---------------------------------------------------------------------------
// shared-memory table hash (fold_i32.cuh, the shared-memory encode in vocab.cu): a
// BIJECTION of the 32-bit key, so a shared table can store h instead of the key
// ---------------------------------------------------------------------------
constexpr uint32_t kFoldC1 = 0x9E3779B1u;
constexpr uint32_t kFoldC2 = 0x85EBCA6Bu;
constexpr uint32_t kFoldC1Inv = 0x0E8B2F51u;
constexpr uint32_t kFoldC2Inv = 0xA5CB9243u;
static_assert((uint32_t)(kFoldC1 * kFoldC1Inv) == 1u, "kFoldC1Inv");
static_assert((uint32_t)(kFoldC2 * kFoldC2Inv) == 1u, "kFoldC2Inv");
constexpr uint32_t kFoldEmpty = 0xFFFFFFFFu;   // the one h that is never stored in shared memory

__host__ __device__ __forceinline__ uint32_t fold_hash(uint32_t k) {
  uint32_t h = k * kFoldC1;
  h ^= h >> 15;
  return h * kFoldC2;
}
__host__ __device__ __forceinline__ uint32_t fold_unhash(uint32_t h) {
  h *= kFoldC2Inv;
  h ^= h >> 15;
  h ^= h >> 30;
  return h * kFoldC1Inv;
}


// ---------------------------------------------------------------------------
// hashes
// ---------------------------------------------------------------------------
// (1) the reference-visible hash: pandas.util.hash_array on numeric data
//     (pandas/core/util/hashing.py::_hash_ndarray — splitmix64 finaliser over
//     the value's bits zero-extended to 64).  Used by HashBucket and the
//     Categorify OOV buckets; bit-exact with the CPU reference path.
__host__ __device__ __forceinline__ uint64_t pandas_mix64(uint64_t v) {
  v ^= v >> 30;
  v *= 0xBF58476D1CE4E5B9ull;
  v ^= v >> 27;
  v *= 0x94D049BB133111EBull;
  v ^= v >> 31;
  return v;
}
template <typename T>
__host__ __device__ __forceinline__ uint64_t value_bits(T x);
template <>
__host__ __device__ __forceinline__ uint64_t value_bits<int32_t>(int32_t x) {
  return (uint64_t)(uint32_t)x;
}
template <>
__host__ __device__ __forceinline__ uint64_t value_bits<int64_t>(int64_t x) {
  return (uint64_t)x;
}
template <>
__host__ __device__ __forceinline__ uint64_t value_bits<float>(float x) {
#ifdef __CUDA_ARCH__
  return (uint64_t)__float_as_uint(x);
#else
  uint32_t u; memcpy(&u, &x, 4); return u;
#endif
}
template <>
__host__ __device__ __forceinline__ uint64_t value_bits<double>(double x) {
#ifdef __CUDA_ARCH__
  return (uint64_t)__double_as_longlong(x);
#else
  uint64_t u; memcpy(&u, &x, 8); return u;
#endif
}
template <>
__host__ __device__ __forceinline__ uint64_t value_bits<uint8_t>(uint8_t x) {
  return (uint64_t)x;
}
constexpr uint64_t kNaNBits = 0x7FF8000000000000ull;  // what pandas sees for a null

// (2) the internal table hash (never visible in results): murmur3 fmix64.
__host__ __device__ __forceinline__ uint64_t table_mix64(uint64_t k) {
  k ^= k >> 33;
  k *= 0xFF51AFD7ED558CCDull;
  k ^= k >> 33;
  k *= 0xC4CEB9FE1A85EC53ull;
  k ^= k >> 33;
  return k;
}

// 32-bit variant (murmur3 fmix32) for the narrow (int32-key) tables: a third of the
// instructions of the 64-bit mixer, which matters in the per-row paths.
__host__ __device__ __forceinline__ uint32_t table_mix32(uint32_t h) {
  h ^= h >> 16;
  h *= 0x85EBCA6Bu;
  h ^= h >> 13;
  h *= 0xC2B2AE35u;
  h ^= h >> 16;
  return h;
}

constexpr int64_t kEmptyKey = INT64_MIN;  // table sentinel (see hashagg.cu)

// dtype dispatch for column-typed kernels
#define NVTB_DISPATCH_NUMERIC(dt, T, ...)                                     \
  switch (dt) {                                                               \
    case NVTB_I32: { using T = int32_t; __VA_ARGS__; } break;                 \
    case NVTB_I64: { using T = int64_t; __VA_ARGS__; } break;                 \
    case NVTB_F32: { using T = float; __VA_ARGS__; } break;                   \
    case NVTB_F64: { using T = double; __VA_ARGS__; } break;                  \
    default:                                                                  \
      ::nvtb::set_error("unsupported dtype %d", (int)(dt));                   \
      return NVTB_EINVAL;                                                     \
  }

#define NVTB_DISPATCH_KEY(dt, T, ...)                                         \
  switch (dt) {                                                               \
    case NVTB_I32: { using T = int32_t; __VA_ARGS__; } break;                 \
    case NVTB_I64: { using T = int64_t; __VA_ARGS__; } break;                 \
    default:                                                                  \
      ::nvtb::set_error("key dtype must be int32 or int64, got %d",           \
                        (int)(dt));                                           \
      return NVTB_EINVAL;                                                     \
  }

}  // namespace nvtb
