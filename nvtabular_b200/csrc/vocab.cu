// vocab.cu — K4 vocabulary ordering/cut, K5 lookup build + encode, and the
// group-statistics gather used by JoinGroupby / TargetEncoding.
//
// Reference behaviour restated (the reference does this with cuDF sort_values,
// merge and a second sort back to row order):
//   _write_uniques / _save_encodings  nvtabular/ops/categorify.py:1149-1337, 719-822
//   _encode                           nvtabular/ops/categorify.py:1558-1807
//   JoinGroupby.transform             nvtabular/ops/join_groupby.py:175-217
//
// Ordering rule: (size desc, key asc) — the stable form of the reference's
// sort_values(key) followed by sort_values(size, ascending=False)
// (categorify.py:1300,1316; SURVEY.md §0.5).  Implemented as two stable LSD
// radix sorts (hand-written passes of radix.cuh for int32 keys; cub::DeviceRadixSort - library code - only for 64-bit keys; on U distinct keys, not on
// the N-row stream).  The encode is a single in-order probe pass: no join, no
// sort back to row order.
#include <algorithm>
#include <cstddef>
#include <cub/cub.cuh>
#include <mutex>
#include <new>
#include <vector>

#include "common.cuh"
#include "hashagg.cuh"
#include "radix.cuh"
#include "lookup.cuh"

namespace nvtb {

// ---------------------------------------------------------------------------
// encode
// ---------------------------------------------------------------------------
constexpr int kMaxHashCols = 8;
struct HashCols {
  const void* data[kMaxHashCols];
  const uint8_t* mask[kMaxHashCols];
  int32_t dtype[kMaxHashCols];
  int32_t ncols;
};

__device__ __forceinline__ uint64_t hash_cols_at(const HashCols& hc, int64_t i) {
  uint64_t h = 0;
  for (int c = 0; c < hc.ncols; ++c) {
    uint64_t bits;
    if (!valid1(hc.mask[c], i)) {
      bits = kNaNBits;
    } else {
      switch (hc.dtype[c]) {
        case NVTB_I32: bits = value_bits<int32_t>(((const int32_t*)hc.data[c])[i]); break;
        case NVTB_I64: bits = value_bits<int64_t>(((const int64_t*)hc.data[c])[i]); break;
        case NVTB_F32: bits = value_bits<float>(((const float*)hc.data[c])[i]); break;
        case NVTB_F64: bits = value_bits<double>(((const double*)hc.data[c])[i]); break;
        case NVTB_H64: h ^= (uint64_t)((const int64_t*)hc.data[c])[i]; continue;  // already a hash
        default:       bits = value_bits<uint8_t>(((const uint8_t*)hc.data[c])[i]); break;
      }
    }
    h ^= pandas_mix64(bits);
  }
  return h;
}

struct EncodeParams {
  int64_t null_label, oov_label, first_label;
  uint64_t num_buckets;  // <= 1: single OOV index
};

// label of one row from scratch: full lookup + OOV hashing.  Out of line on purpose: the
// 16-row-unrolled fast paths below only FLAG the rows that need it (continued probing, OOV
// hash buckets), which keeps them ~3x smaller (the fully inlined version spent a quarter
// of its issue slots waiting for instructions).
template <typename KeyT>
static __device__ __noinline__ long long encode_slow(const Lookup& t, const EncodeParams& p,
                                                     const HashCols& hc, int64_t i, KeyT x) {
  const int64_t pos = lookup_find(t, (int64_t)x);
  if (pos >= 0) return (long long)(p.first_label + pos);
  int64_t lab = p.oov_label;
  if (p.num_buckets > 1) {
    const uint64_t h = hc.ncols > 0 ? hash_cols_at(hc, i) : pandas_mix64(value_bits<KeyT>(x));
    lab += (int64_t)(h % p.num_buckets);
  }
  return (long long)lab;
}

template <typename KeyT, typename OutT, bool NARROW>
__global__ void __launch_bounds__(kThreads, 4)
encode_kernel(const KeyT* __restrict__ keys, const uint8_t* __restrict__ mask,
              int64_t n, Lookup t, EncodeParams p, HashCols hc,
              OutT* __restrict__ out) {
  const bool aligned = is_aligned32(keys) && is_aligned32(out);
  auto in_range = [](long long k) -> bool {
    return !NARROW || (k >= (long long)INT32_MIN && k <= (long long)INT32_MAX);
  };
  const long long fl1 = (long long)p.first_label - 1;     // label = fl1 + (pos + 1)
  const bool hash_oov = p.num_buckets > 1;
  const int64_t n_tiles = (n + kTile - 1) / kTile;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t base = tile * kTile;
    if (aligned && base + kTile <= n) {
      KeyT v[kGroups][kRows];
      unsigned m[kGroups];
#pragma unroll
      for (int g = 0; g < kGroups; ++g) {
        const int64_t i = base + (int64_t)g * (kThreads * kRows) + (int64_t)threadIdx.x * kRows;
        ld_rows8<KeyT>(keys + i, v[g]);
        m[g] = valid8(mask, i);
      }
#pragma unroll
      for (int g = 0; g < kGroups; ++g) {
        const int64_t i = base + (int64_t)g * (kThreads * kRows) + (int64_t)threadIdx.x * kRows;
        // per half of 4 rows: (1) first-probe sector loads back to back, (2) resolve what the
        // first bucket decides, flag the rest; then one 256-bit store (two for 8-byte labels)
        OutT o[kRows];
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          unsigned pend = 0;
          LProbe<NARROW> pr[4];
#pragma unroll
          for (int k = 0; k < 4; ++k)
            lookup_load<NARROW>(t, lookup_home<NARROW>(t, (long long)v[g][4 * half + k]), pr[k]);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int r = 4 * half + k;
            const bool valid = (m[g] >> r) & 1u;
            const long long key = (long long)v[g][r];
            long long lab = (long long)p.oov_label;
            bool decided;
            if constexpr (NARROW) {
              // slot = ((pos + 1) << 32) | key; a free slot has pos + 1 == 0, so "low word
              // equals the key" needs no separate emptiness test
              unsigned pos1 = 0, hi_and = 0xFFFFFFFFu;
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const unsigned lo = (unsigned)pr[k].w[j], hi = (unsigned)(pr[k].w[j] >> 32);
                pos1 |= (lo == (unsigned)key) ? hi : 0u;
                hi_and = (hi == 0u) ? 0u : hi_and;
              }
              if (sizeof(KeyT) == 8 && !in_range(key)) pos1 = 0u;    // cannot be in a narrow table
              if (pos1) lab = fl1 + (long long)pos1;
              // not found: final only if the bucket has a free slot (else the probe goes on)
              decided = pos1 != 0u || ((hi_and == 0u || (sizeof(KeyT) == 8 && !in_range(key))) && !hash_oov);
            } else {
              decided = false;
              if (key != kEmptyKey && pr[k].k == key) { lab = fl1 + 1 + (long long)pr[k].v; decided = true; }
              else if (key != kEmptyKey && pr[k].k == kEmptyKey && !hash_oov) decided = true;
            }
            if (!valid) { lab = (long long)p.null_label; decided = true; }
            if (!decided) pend |= 1u << r;
            o[r] = (OutT)lab;
          }
          if (pend) {
#pragma unroll
            for (int k = 0; k < 4; ++k)
              if ((pend >> (4 * half + k)) & 1u)
                o[4 * half + k] = (OutT)encode_slow<KeyT>(t, p, hc, i + 4 * half + k, v[g][4 * half + k]);
          }
          if constexpr (sizeof(OutT) == 8) {      // 4 labels = one 32-byte sector; frees their registers
            uint32_t w[8];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              w[2 * k] = (uint32_t)(uint64_t)o[4 * half + k];
              w[2 * k + 1] = (uint32_t)((uint64_t)o[4 * half + k] >> 32);
            }
            st256(out + i + 4 * half, w);
          }
        }
        if constexpr (sizeof(OutT) != 8)
          st_rows8<OutT>(out + i, o);
      }
    } else {
      const int64_t end = (base + kTile < n) ? base + kTile : n;
      for (int64_t i = base + threadIdx.x; i < end; i += kThreads) {
        const KeyT x = keys[i];
        out[i] = valid1(mask, i) ? (OutT)encode_slow<KeyT>(t, p, hc, i, x) : (OutT)p.null_label;
      }
    }
  }
}

// ---------------------------------------------------------------------------
// encode with the vocabulary in SHARED memory (int32 keys, vocabularies of <= 14 336 keys:
// 16 of the 26 Criteo columns).  A row of the global-lookup kernel above costs one random
// 32-byte L2 sector (and every CTA hammers the same few sectors when the vocabulary is
// tiny); here every CTA first builds
// its own copy of the vocabulary as a 4-way-bucket table of h = fold_hash(key) (+ position)
// in 224 KB of shared memory, and a row costs one LDS.128 + one LDS.32.  A key that found
// its bucket full at build time is simply not in the shared copy: a row that meets a FULL
// bucket without a match falls back to the global lookup, so the result never depends on
// the build order.
// ---------------------------------------------------------------------------
constexpr int kEncSmemThreads = 1024;
constexpr unsigned kEncSmemBuckets = 7168;                       // x 4 slots x 8 B = 224 KB
constexpr int64_t kEncSmemMaxKeys = (int64_t)kEncSmemBuckets * 2;  // load <= 0.5

template <typename OutT>
__global__ void __launch_bounds__(kEncSmemThreads, 1)
encode_smem_kernel(const int32_t* __restrict__ keys, const uint8_t* __restrict__ mask, int64_t n,
                   const int64_t* __restrict__ vkeys, int n_keep, Lookup t, EncodeParams p,
                   HashCols hc, OutT* __restrict__ out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t* hk = reinterpret_cast<uint32_t*>(smem_raw);
  uint32_t* ps = hk + 4 * kEncSmemBuckets;
  constexpr unsigned nb = kEncSmemBuckets;
  for (unsigned s = threadIdx.x; s < 4 * nb; s += kEncSmemThreads) hk[s] = kFoldEmpty;
  __syncthreads();
  for (int i = threadIdx.x; i < n_keep; i += kEncSmemThreads) {
    const uint32_t h = fold_hash((uint32_t)(int32_t)vkeys[i]);
    if (h == kFoldEmpty) continue;                 // reserved value: served by the fallback
    const unsigned b = __umulhi(h, nb);
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (atomicCAS(hk + 4 * b + j, kFoldEmpty, h) == kFoldEmpty) { ps[4 * b + j] = (uint32_t)i; break; }
  }
  __syncthreads();

  const long long fl = (long long)p.first_label;
  const bool hash_oov = p.num_buckets > 1;

  constexpr int64_t step = (int64_t)kEncSmemThreads * 8;
  for (int64_t base = (int64_t)blockIdx.x * step; base < n; base += (int64_t)gridDim.x * step) {
    const int64_t i = base + (int64_t)threadIdx.x * 8;
    if (i + 8 <= n) {
      int32_t v[8];
      ld_rows8<int32_t>(keys + i, v);
      const unsigned m = valid8(mask, i);
      OutT o[8];
      unsigned pend = 0;
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        uint4 c[4];
        uint32_t h[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          h[k] = fold_hash((uint32_t)v[4 * half + k]);
          const unsigned addr = (unsigned)__cvta_generic_to_shared(hk + 4 * __umulhi(h[k], nb));
          asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                       : "=r"(c[k].x), "=r"(c[k].y), "=r"(c[k].z), "=r"(c[k].w) : "r"(addr));
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int r = 4 * half + k;
          const bool valid = (m >> r) & 1u;
          const int j = (c[k].x == h[k]) ? 0 : (c[k].y == h[k]) ? 1 : (c[k].z == h[k]) ? 2 : (c[k].w == h[k]) ? 3 : -1;
          long long lab = (long long)p.oov_label;
          bool decided = !hash_oov;              // a miss in a non-full bucket is OOV
          if (j >= 0 && h[k] != kFoldEmpty) {
            lab = fl + (long long)ps[4 * __umulhi(h[k], nb) + j];
            decided = true;
          } else if (c[k].w != kFoldEmpty || h[k] == kFoldEmpty) {
            decided = false;                     // full bucket (slots fill in order) or reserved h
          }
          if (!valid) { lab = (long long)p.null_label; decided = true; }
          if (!decided) pend |= 1u << r;
          o[r] = (OutT)lab;
        }
      }
      if (pend) {
#pragma unroll
        for (int r = 0; r < 8; ++r)
          if ((pend >> r) & 1u) o[r] = (OutT)encode_slow<int32_t>(t, p, hc, i + r, v[r]);
      }
      st_rows8<OutT>(out + i, o);
    } else {
      for (int64_t q = i; q < n; ++q)
        out[q] = valid1(mask, q) ? (OutT)encode_slow<int32_t>(t, p, hc, q, keys[q]) : (OutT)p.null_label;
    }
  }
}

// ---------------------------------------------------------------------------
// group-statistics gather
// ---------------------------------------------------------------------------
constexpr int kMaxGatherCols = 16;
struct GatherOut {
  void* out[kMaxGatherCols];
  uint32_t* valid[kMaxGatherCols];   // optional validity bitmask of out[j], or nullptr
  double miss[kMaxGatherCols];
  int32_t col[kMaxGatherCols];
  int32_t dtype[kMaxGatherCols];
  int32_t ncols;
};

// A row of out[j] is valid when its key has a row in the matrix and that value is not NaN.  An
// integer output holds 0 where it is not valid, so the bitmask is what tells a missing statistic
// from a real 0.  A warp covers 32 consecutive rows (blockDim and the grid stride are multiples
// of 32), so one ballot gives one 32-bit word of the LSB-first bitmask.
template <typename KeyT>
__global__ void __launch_bounds__(kThreads)
gather_stats_kernel(const KeyT* __restrict__ keys, const uint8_t* __restrict__ mask,
                    int64_t n, Lookup t, int64_t null_row,
                    const double* __restrict__ stats, int width, GatherOut go) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int lane = threadIdx.x & 31;
  // whole warps iterate together (the ballot below needs every lane)
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i - lane < n; i += stride) {
    const bool in = i < n;
    const int64_t row = !in ? -1 : valid1(mask, i) ? lookup_find(t, (int64_t)keys[i]) : null_row;
    for (int j = 0; j < go.ncols; ++j) {
      const double v = row >= 0 ? __ldg(stats + row * width + go.col[j]) : go.miss[j];
      const bool ok = row >= 0 && v == v;
      if (in) {
        switch (go.dtype[j]) {
          case NVTB_I32: ((int32_t*)go.out[j])[i] = v == v ? (int32_t)v : 0; break;
          case NVTB_I64: ((int64_t*)go.out[j])[i] = v == v ? (int64_t)v : 0; break;
          case NVTB_F32: ((float*)go.out[j])[i] = (float)v; break;
          default:       ((double*)go.out[j])[i] = v; break;
        }
      }
      if (go.valid[j] != nullptr) {
        const unsigned bits = __ballot_sync(0xFFFFFFFFu, in && ok);
        if (lane == 0) go.valid[j][i >> 5] = bits;
      }
    }
  }
}

// ---- vocabularies from packed, key-ordered pairs (sorted accumulator of hashagg.cu) ------
__device__ __forceinline__ long long packed_key(uint64_t w) { return (long long)(int32_t)((uint32_t)(w >> 32) ^ 0x80000000u); }

__global__ void __launch_bounds__(kThreads)
packed_unpack_kernel(const uint64_t* __restrict__ p, int64_t n, int64_t* __restrict__ keys, int64_t* __restrict__ sizes) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint64_t w = p[i];
    if (keys) keys[i] = packed_key(w);
    if (sizes) sizes[i] = (int64_t)(uint32_t)w;
  }
}

// narrow lookup (4-way sector buckets of ((pos + 1) << 32) | key) from the kept pairs; keys are distinct
__global__ void __launch_bounds__(kThreads)
lookup_build_packed_kernel(const uint64_t* __restrict__ p, int64_t n, unsigned long long* __restrict__ slots,
                           int64_t capacity) {
  const int64_t bmask = (capacity >> 2) - 1;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t key = (uint32_t)(p[i] >> 32) ^ 0x80000000u;
    narrow_claim(slots, (int64_t)((uint64_t)table_mix32(key) & (uint64_t)bmask), bmask + 1,
                 ((unsigned long long)(unsigned)(i + 1) << 32) | key);
  }
}

// ---------------------------------------------------------------------------------------
// slice-wise build of a large narrow lookup.  One random insert per key into a multi-GB table is
// one DRAM-resident atomic per key (every warp waiting on its CAS, far from the DRAM peak).  Instead the (position, key) items are partitioned by the table slice
// their home bucket lies in (order-free: shared-memory counts, one reservation per tile and
// slice), and one CTA then builds ITS slice: in shared memory when the slice is 8192 buckets
// (slice_build_smem_kernel), else in place in the L2 (slice_build_kernel).  Every table line
// reaches HBM once.
// ---------------------------------------------------------------------------------------
constexpr int kSlThreads = 512;
// items per tile of the scatter (128 KB staged, one CTA per SM): with up to 8192 slices a tile
// puts several items into each slice's run, so a run grows by whole sectors more often and there
// are fewer cursor reservations per item
constexpr int kSlTile = 16384;

__device__ __forceinline__ uint32_t slice_of(uint32_t key, uint32_t bmask, int lg_slice) {
  return (table_mix32(key) & bmask) >> lg_slice;
}

static __global__ void __launch_bounds__(kSlThreads)
slice_hist_kernel(const uint64_t* __restrict__ p, int64_t n, uint32_t bmask, int lg_slice, int P,
                  uint32_t* __restrict__ total) {
  extern __shared__ __align__(16) uint32_t sl_smem[];
  uint32_t* cnt = sl_smem;
  for (int d = threadIdx.x; d < P; d += kSlThreads) cnt[d] = 0u;
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * kSlThreads;
  for (int64_t i = (int64_t)blockIdx.x * kSlThreads + threadIdx.x; i < n; i += stride)
    atomicAdd(&cnt[slice_of((uint32_t)(p[i] >> 32) ^ 0x80000000u, bmask, lg_slice)], 1u);
  __syncthreads();
  for (int d = threadIdx.x; d < P; d += kSlThreads)
    if (cnt[d]) atomicAdd(&total[d], cnt[d]);
}

// total[P] -> starts[P + 1] (exclusive) and cursor[P]
static __global__ void __launch_bounds__(kSlThreads)
slice_scan_kernel(const uint32_t* __restrict__ total, int P, uint32_t* __restrict__ starts, uint32_t* __restrict__ cursor) {
  extern __shared__ __align__(16) uint32_t sl_smem[];
  __shared__ uint32_t ws[kSlThreads / 32 + 1];
  uint32_t* v = sl_smem;
  uint32_t* o = sl_smem + P;
  for (int d = threadIdx.x; d < P; d += kSlThreads) v[d] = total[d];
  __syncthreads();
  const uint32_t tot = rx_block_excl_scan<kSlThreads>(v, o, P, ws);
  for (int d = threadIdx.x; d < P; d += kSlThreads) { starts[d] = o[d]; cursor[d] = o[d]; }
  if (threadIdx.x == 0) starts[P] = tot;
}

// items[...] = ((pos + 1) << 32) | key, grouped by slice
static __global__ void __launch_bounds__(kSlThreads, 1)
slice_scatter_kernel(const uint64_t* __restrict__ p, int64_t n, uint32_t bmask, int lg_slice, int P,
                     uint32_t* __restrict__ cursor, uint64_t* __restrict__ items) {
  extern __shared__ __align__(16) unsigned char sl_raw[];
  uint64_t* stage = reinterpret_cast<uint64_t*>(sl_raw);                        // [kSlTile]
  uint32_t* cnt = reinterpret_cast<uint32_t*>(stage + kSlTile);                 // [P]
  uint32_t* delta = cnt + P;                                                    // [P]
  __shared__ uint32_t ws[kSlThreads / 32 + 1];
  constexpr int kPer = kSlTile / kSlThreads;                                    // 32 items per thread
  const int64_t n_tiles = (n + kSlTile - 1) / kSlTile;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    for (int d = threadIdx.x; d < P; d += kSlThreads) cnt[d] = 0u;
    __syncthreads();
    uint32_t key[kPer];
    uint16_t bin[kPer];
    const int64_t base = tile * kSlTile;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int64_t i = base + (int64_t)j * kSlThreads + threadIdx.x;
      key[j] = i < n ? ((uint32_t)(p[i] >> 32) ^ 0x80000000u) : 0u;
      bin[j] = (uint16_t)slice_of(key[j], bmask, lg_slice);
      if (i < n) atomicAdd(&cnt[bin[j]], 1u);
    }
    __syncthreads();
    const uint32_t total = rx_block_excl_scan<kSlThreads>(cnt, delta, P, ws);   // staged offsets
    for (int d = threadIdx.x; d < P; d += kSlThreads) {
      const uint32_t c = cnt[d], off = delta[d];
      uint32_t g0 = 0;
      if (c) g0 = atomicAdd(&cursor[d], c);
      delta[d] = g0 - off;            // global index = delta + staged index (mod 2^32)
      cnt[d] = off;                   // running staged cursor
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int64_t i = base + (int64_t)j * kSlThreads + threadIdx.x;
      if (i < n) {
        const uint32_t q = atomicAdd(&cnt[bin[j]], 1u);
        stage[q] = ((uint64_t)(uint32_t)(i + 1) << 32) | key[j];
      }
    }
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < total; j += kSlThreads) {
      const uint64_t it = stage[j];
      items[delta[slice_of((uint32_t)it, bmask, lg_slice)] + j] = it;
    }
    __syncthreads();
  }
}

// one CTA per slice: zero-fill, then claim the first free slot of the home bucket (or of the
// following buckets of the SAME slice)
static __global__ void __launch_bounds__(1024)
slice_build_kernel(const uint64_t* __restrict__ items, const uint32_t* __restrict__ starts,
                   unsigned long long* __restrict__ slots, uint32_t bmask, int lg_slice) {
  const int sl = blockIdx.x;
  const int64_t slice_buckets = (int64_t)1 << lg_slice;
  unsigned long long* base = slots + (int64_t)sl * slice_buckets * 4;
  ulonglong2* z = reinterpret_cast<ulonglong2*>(base);
  for (int64_t i = threadIdx.x; i < slice_buckets * 2; i += blockDim.x) z[i] = make_ulonglong2(0ull, 0ull);
  __syncthreads();
  const uint32_t s = starts[sl], e = starts[sl + 1];
  for (uint32_t i = s + threadIdx.x; i < e; i += blockDim.x) {
    const unsigned long long want = items[i];
    narrow_claim(slots, (int64_t)(table_mix32((uint32_t)want) & bmask), (int64_t)bmask + 1, want);
  }
}

// One CTA per slice of kSliceBuckets buckets, built in shared memory: a claim counter per bucket
// (32 KB) and, per slot, the index (+ 1) of the item that claimed it within the slice's run (16
// bits: a slice holds at most 4 * kSliceBuckets items; 64 KB).  An item takes the next slot of its
// home bucket, or of the first bucket after it in the slice that is not yet full — the placement
// narrow_claim makes in the table.  Then each table slot is written once, in order: the item it
// holds (re-read from the run, which this CTA has just read) or 0.  The inserts are shared-memory
// atomicAdds, and the table is written without a zero-fill pass or a read-modify-write of its lines.
constexpr int kSlBuildThreads = 1024;
constexpr int kSlBuildSlots = 4 * (int)kSliceBuckets;
constexpr int kSlBuildSmem = (int)kSliceBuckets * 4 + kSlBuildSlots * 2;    // 96 KB: 2 CTAs per SM

static __global__ void __launch_bounds__(kSlBuildThreads, 2)
slice_build_smem_kernel(const uint64_t* __restrict__ items, const uint32_t* __restrict__ starts,
                        unsigned long long* __restrict__ slots, uint32_t bmask) {
  extern __shared__ __align__(16) uint32_t sb_fill[];                         // [kSliceBuckets]
  unsigned short* sb_item = reinterpret_cast<unsigned short*>(sb_fill + kSliceBuckets);   // [kSlBuildSlots]
  constexpr uint32_t kBm = (uint32_t)kSliceBuckets - 1;
  constexpr int kUnroll = 4;
  const int sl = blockIdx.x;
  for (int i = threadIdx.x; i < (int)kSliceBuckets / 4; i += kSlBuildThreads)
    reinterpret_cast<uint4*>(sb_fill)[i] = make_uint4(0u, 0u, 0u, 0u);
  __syncthreads();
  const uint32_t s = starts[sl], e = starts[sl + 1];
  for (uint32_t i0 = s + threadIdx.x; i0 < e; i0 += kUnroll * kSlBuildThreads) {
    uint32_t key[kUnroll];
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) {
      const uint32_t i = i0 + k * kSlBuildThreads;
      key[k] = i < e ? (uint32_t)items[i] : 0u;
    }
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) {
      const uint32_t i = i0 + k * kSlBuildThreads;
      if (i >= e) continue;
      uint32_t b = (table_mix32(key[k]) & bmask) & kBm;
      uint32_t j;
      while ((j = atomicAdd(sb_fill + b, 1u)) >= 4u) b = (b + 1) & kBm;
      sb_item[4 * b + j] = (unsigned short)(i - s + 1);
    }
  }
  __syncthreads();
  unsigned long long* base = slots + (int64_t)sl * kSlBuildSlots;
  for (int q0 = threadIdx.x; q0 < kSlBuildSlots; q0 += kUnroll * kSlBuildThreads) {
    uint32_t r[kUnroll];
    unsigned long long w[kUnroll];
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) {
      const int q = q0 + k * kSlBuildThreads;
      r[k] = (uint32_t)(q & 3) < sb_fill[q >> 2] ? (uint32_t)sb_item[q] : 0u;
    }
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) w[k] = r[k] ? items[s + r[k] - 1] : 0ull;
#pragma unroll
    for (int k = 0; k < kUnroll; ++k) base[q0 + k * kSlBuildThreads] = w[k];
  }
}

static int64_t pow2_at_least(int64_t v) {
  int64_t p = 16;
  while (p < v) p <<= 1;
  return p;
}

struct VocabScalars {
  long long n_keep;
  long long sum_kept;
  long long sum_all;
  int fit_i32;             // 1 while every kept key fits int32
  long long min_key_pos;   // position of the INT64_MIN key, or -1
};

__global__ void __launch_bounds__(kThreads)
xor_copy_kernel(const int64_t* src, int64_t* dst, int64_t n, long long mask) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = src[i] ^ mask;
}

// The two row layouts of an ordered vocabulary: int64 key and size arrays, or packed pairs
// ((key ^ 2^31) << 32) | size.
struct ArrayRows {
  const int64_t* __restrict__ keys;
  const int64_t* __restrict__ sizes;
  __device__ __forceinline__ long long key(int64_t i) const { return keys[i]; }
  __device__ __forceinline__ long long size(int64_t i) const { return sizes[i]; }
};
struct PackedRows {
  const uint64_t* __restrict__ p;
  __device__ __forceinline__ long long key(int64_t i) const { return packed_key(p[i]); }
  __device__ __forceinline__ long long size(int64_t i) const { return (long long)(uint32_t)p[i]; }
};

// number of leading rows with size >= threshold in size-descending rows
template <typename Rows>
__global__ void __launch_bounds__(kThreads)
cut_kernel(Rows r, int64_t n, int64_t threshold, long long* out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (r.size(i) >= threshold && (i == n - 1 || r.size(i + 1) < threshold)) *out = i + 1;
  }
}

// sums of the kept / all sizes, and "do the kept keys fit int32?"
template <typename Rows>
__global__ void __launch_bounds__(kThreads)
sums_kernel(Rows r, int64_t n, int64_t n_keep, VocabScalars* sc) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  long long kept = 0, all = 0;
  bool bad = false;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const long long sz = r.size(i);
    all += sz;
    if (i < n_keep) {
      kept += sz;
      const long long k = r.key(i);
      bad = bad || (k < (long long)INT32_MIN) || (k > (long long)INT32_MAX);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    kept += __shfl_down_sync(0xffffffffu, kept, o);
    all += __shfl_down_sync(0xffffffffu, all, o);
  }
  if ((threadIdx.x & 31) == 0) {
    if (kept) atomicAdd(reinterpret_cast<unsigned long long*>(&sc->sum_kept), (unsigned long long)kept);
    if (all) atomicAdd(reinterpret_cast<unsigned long long*>(&sc->sum_all), (unsigned long long)all);
  }
  if (bad) sc->fit_i32 = 0;
}

// build either layout; which one is decided by a DEVICE flag so no host sync is needed
__global__ void __launch_bounds__(kThreads)
lookup_build_any_kernel(const int64_t* __restrict__ keys, int64_t n, int64_t* slots,
                        int64_t capacity, const int* fit_i32, long long* min_key_pos) {
  const bool narrow = (fit_i32 != nullptr) && (*fit_i32 != 0);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const long long k = keys[i];
    if (narrow) {             // keys are distinct here: they come out of a group-by
      const int64_t nbuckets = capacity >> 2;
      narrow_claim(reinterpret_cast<unsigned long long*>(slots),
                   (int64_t)((uint64_t)table_mix32((uint32_t)(int32_t)k) & (uint64_t)(nbuckets - 1)), nbuckets,
                   ((unsigned long long)(unsigned)(i + 1) << 32) | (unsigned)(int)k);
    } else if (k == kEmptyKey) {
      // a repeated key keeps its smallest position, like wide_claim: min of the positions as
      // unsigned, over the -1 (all ones) the slot starts at
      atomicMin(reinterpret_cast<unsigned long long*>(min_key_pos), (unsigned long long)i);
    } else {
      wide_claim(slots, capacity, k, (long long)i);
    }
  }
}

__global__ void lookup_init_any_kernel(int64_t* slots, int64_t capacity, const int* fit_i32) {
  const bool narrow = (fit_i32 != nullptr) && (*fit_i32 != 0);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < capacity; s += stride) {
    if (narrow) {
      slots[s] = 0;                 // narrow table uses the first `capacity` words only
    } else {
      slots[2 * s] = kEmptyKey;
      slots[2 * s + 1] = INT64_MAX;
    }
  }
}

// ---------------------------------------------------------------------------
// small vocabularies (n <= 8192): ONE single-CTA kernel does everything —
// bitonic sort in shared memory on (size desc, key asc), freq_threshold /
// max_size cut, meta sums, int32 check, and the lookup-table build.  Most
// Criteo columns are this small; the general path (two sorts and a dozen
// tiny launches) is launch-latency bound for them.
// ---------------------------------------------------------------------------
constexpr int kSmallVocabMax = 8192;
constexpr int kSmallThreads = 1024;

__device__ __forceinline__ bool vocab_before(long long sa, long long ka, long long sb, long long kb) {
  return (sa > sb) || (sa == sb && ka < kb);
}

__global__ void __launch_bounds__(kSmallThreads)
small_vocab_kernel(const int64_t* __restrict__ keys_in, const int64_t* __restrict__ sizes_in,
                   int n, int n2, long long freq_threshold, long long max_keep,
                   int64_t* __restrict__ keys_out, int64_t* __restrict__ sizes_out,
                   int64_t* slots, long long capacity, VocabScalars* sc) {
  extern __shared__ __align__(16) unsigned char small_raw[];
  long long* k = reinterpret_cast<long long*>(small_raw);
  long long* s = k + n2;
  __shared__ long long red[3][kSmallThreads / 32];
  __shared__ int s_keep, s_bad;
  const int tid = threadIdx.x;
  for (int i = tid; i < n2; i += kSmallThreads) {
    k[i] = i < n ? (long long)keys_in[i] : (long long)INT64_MAX;
    s[i] = i < n ? (long long)sizes_in[i] : -1ll;           // padding sorts last
  }
  if (tid == 0) { s_keep = 0; s_bad = 0; }
  __syncthreads();
  for (int size = 2; size <= n2; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = tid; i < (n2 >> 1); i += kSmallThreads) {
        const int pos = 2 * i - (i & (stride - 1));
        const int par = pos + stride;
        const bool up = ((pos & size) == 0);
        const long long sa = s[pos], ka = k[pos], sb = s[par], kb = k[par];
        if (vocab_before(sb, kb, sa, ka) == up) { s[pos] = sb; k[pos] = kb; s[par] = sa; k[par] = ka; }
      }
      __syncthreads();
    }
  }
  // cut
  int n_keep = n;
  if (freq_threshold > 0) {
    int c = 0;
    for (int i = tid; i < n; i += kSmallThreads) c += (s[i] >= freq_threshold) ? 1 : 0;
    if (c) atomicAdd(&s_keep, c);
    __syncthreads();
    n_keep = s_keep;
  } else if (max_keep >= 0) {
    n_keep = (int)(max_keep < (long long)n ? max_keep : (long long)n);
  }
  // sums + int32 check
  long long kept = 0, all = 0;
  bool bad = false;
  for (int i = tid; i < n; i += kSmallThreads) {
    all += s[i];
    if (i < n_keep) {
      kept += s[i];
      bad = bad || (k[i] < (long long)INT32_MIN) || (k[i] > (long long)INT32_MAX);
    }
    keys_out[i] = k[i];
    sizes_out[i] = s[i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    kept += __shfl_down_sync(0xffffffffu, kept, o);
    all += __shfl_down_sync(0xffffffffu, all, o);
  }
  if ((tid & 31) == 0) { red[0][tid >> 5] = kept; red[1][tid >> 5] = all; }
  if (bad) s_bad = 1;
  __syncthreads();
  const bool narrow = (s_bad == 0);
  // lookup table: init, then build from the first n_keep sorted keys
  for (long long i = tid; i < capacity; i += kSmallThreads) {
    if (narrow) slots[i] = 0;
    else { slots[2 * i] = kEmptyKey; slots[2 * i + 1] = INT64_MAX; }
  }
  __syncthreads();
  for (int i = tid; i < n_keep; i += kSmallThreads) {
    const long long key = k[i];
    if (narrow) {                                         // keys are distinct
      const long long nbuckets = capacity >> 2;
      narrow_claim(reinterpret_cast<unsigned long long*>(slots),
                   (long long)((uint64_t)table_mix32((uint32_t)(int32_t)key) & (uint64_t)(nbuckets - 1)), nbuckets,
                   ((unsigned long long)(unsigned)(i + 1) << 32) | (unsigned)(int)key);
    } else if (key == kEmptyKey) {
      atomicMin(reinterpret_cast<unsigned long long*>(&sc->min_key_pos), (unsigned long long)i);   // as lookup_build_any_kernel
    } else {
      wide_claim(slots, capacity, key, i);
    }
  }
  if (tid == 0) {
    long long a = 0, b = 0;
    for (int w = 0; w < kSmallThreads / 32; ++w) { a += red[0][w]; b += red[1][w]; }
    sc->n_keep = n_keep;
    sc->sum_kept = a;
    sc->sum_all = b;
    sc->fit_i32 = narrow ? 1 : 0;
  }
}

// Allocates for the wide layout.  With `sc` (device) the layout is selected at kernel run time by
// sc->fit_i32 and the position of the INT64_MIN key goes to sc->min_key_pos; without it the table
// is wide and that position goes to *d_min_key_pos.  The CALLER sets t->narrow / t->min_key_pos
// after its sync.
static int lookup_create(Lookup* t, const int64_t* keys, int64_t n, VocabScalars* sc, long long* d_min_key_pos,
                         cudaStream_t st) {
  t->capacity = pow2_at_least(2 * n);
  t->min_key_pos = -1;
  t->slots = nullptr;
  t->narrow = 0;
  NVTB_CUDA_OK(cudaMallocAsync(&t->slots, sizeof(int64_t) * 2 * t->capacity, st));
  const int* fit_i32 = sc ? &sc->fit_i32 : nullptr;
  const int g0 = (int)std::min<int64_t>((t->capacity + kThreads - 1) / kThreads, (int64_t)sm_count() * 8);
  lookup_init_any_kernel<<<g0, kThreads, 0, st>>>(t->slots, t->capacity, fit_i32);
  NVTB_LAUNCH_OK();
  if (n > 0) {
    lookup_build_any_kernel<<<plain_grid(n), kThreads, 0, st>>>(keys, n, t->slots, t->capacity, fit_i32,
                                                               sc ? &sc->min_key_pos : d_min_key_pos);
    NVTB_LAUNCH_OK();
  }
  return NVTB_OK;
}

// wide-only variant with its own sync (user vocabs, group-stats tables)
static int lookup_create_wide(Lookup* t, const int64_t* keys, int64_t n, cudaStream_t st) {
  long long* d_min = nullptr;
  NVTB_CUDA_OK(cudaMallocAsync(&d_min, sizeof(long long), st));
  NVTB_CUDA_OK(cudaMemsetAsync(d_min, 0xFF, sizeof(long long), st));  // -1
  int rc = lookup_create(t, keys, n, nullptr, d_min, st);
  if (rc) return rc;
  long long h_min = -1;
  NVTB_CUDA_OK(cudaMemcpyAsync(&h_min, d_min, sizeof(long long), cudaMemcpyDeviceToHost, st));
  NVTB_CUDA_OK(cudaStreamSynchronize(st));
  NVTB_CUDA_OK(cudaFreeAsync(d_min, st));
  t->min_key_pos = h_min;
  return NVTB_OK;
}

}  // namespace nvtb

struct nvtb_vocab {
  nvtb::Lookup t;
  int64_t* keys;   // device [n_kept], label order
  int64_t* sizes;  // device [n_kept] or nullptr
  // vocabularies built from a sorted accumulator keep the ordered PACKED pairs
  // ((key ^ 2^31) << 32 | size) instead of two int64 arrays; keys[] is then only
  // materialised for the shared-memory encode (<= kEncSmemMaxKeys keys)
  uint64_t* packed;
  nvtb_vocab_info_t info;
  // nvtb_vocab_build enqueues everything and returns; the scalars it needs on the host
  // (n_kept, meta sums, table layout) arrive in a pinned mailbox and are read by the first
  // call that needs them (finalize) — so the 26 vocabularies of a Criteo fit are built
  // back to back without a host round trip in between.
  nvtb::VocabScalars* d_sc;
  nvtb::VocabScalars* h_sc;   // slot in the pinned pool
  cudaEvent_t ev;
  bool pending;
};

struct nvtb_groupstats {
  nvtb::Lookup t;
  double* stats;  // device [n_groups * width]
  int64_t n_groups;
  int width;
  int64_t null_row;
};

namespace nvtb {

// tiny pinned slab for the per-vocabulary mailboxes (cudaMallocHost per handle is slow)
static std::mutex g_pin_mu;
static VocabScalars* g_pin_slab = nullptr;
static std::vector<int> g_pin_free;
constexpr int kPinSlots = 8192;

static VocabScalars* pin_acquire() {
  std::lock_guard<std::mutex> lk(g_pin_mu);
  if (g_pin_slab == nullptr) {
    if (cudaMallocHost(&g_pin_slab, sizeof(VocabScalars) * kPinSlots) != cudaSuccess) return nullptr;
    for (int i = kPinSlots - 1; i >= 0; --i) g_pin_free.push_back(i);
  }
  if (g_pin_free.empty()) return nullptr;
  const int i = g_pin_free.back();
  g_pin_free.pop_back();
  return g_pin_slab + i;
}
static void pin_release(VocabScalars* p) {
  if (p == nullptr) return;
  std::lock_guard<std::mutex> lk(g_pin_mu);
  g_pin_free.push_back((int)(p - g_pin_slab));
}

// serialised: the artefact writer threads (artifacts.cu) and the thread running transform may
// both ask for the scalars of the same vocabulary first
static std::mutex g_fin_mu;

// the scalars of a finished build -> the handle's host-side fields
static void vocab_apply(nvtb_vocab* v, const VocabScalars& h) {
  v->info.n_kept = h.n_keep;
  v->info.unique_size = h.sum_kept;
  v->info.oov_size = h.sum_all - h.sum_kept;
  v->t.narrow = h.fit_i32 ? 1 : 0;   // exactly what the device-side init/build kernels used
  v->t.min_key_pos = h.min_key_pos;
}

static int vocab_finalize(nvtb_vocab* v) {
  cudaEvent_t ev = nullptr;
  {
    std::lock_guard<std::mutex> lk(g_fin_mu);
    if (!v->pending) return NVTB_OK;
    ev = v->ev;
  }
  // wait without the lock: a writer thread waiting for a large build must not hold up the
  // finalize of a vocabulary that is already built (the event lives as long as the handle)
  NVTB_CUDA_OK(cudaEventSynchronize(ev));
  std::lock_guard<std::mutex> lk(g_fin_mu);
  if (!v->pending) return NVTB_OK;
  vocab_apply(v, *v->h_sc);
  v->pending = false;
  if (v->d_sc) { cudaFreeAsync(v->d_sc, 0); v->d_sc = nullptr; }
  pin_release(v->h_sc);
  v->h_sc = nullptr;
  return NVTB_OK;
}

// the event that completes v's enqueued build (its kept rows are final once it has fired), or
// nullptr when the build was finished on the host or the handle was made by from_arrays
cudaEvent_t vocab_build_event(const nvtb_vocab* v) { return v->ev; }

// enqueue the readback of the device scalars; falls back to a blocking read when the
// pinned pool is exhausted
static int vocab_post(nvtb_vocab* v, cudaStream_t st) {
  v->h_sc = pin_acquire();
  if (v->h_sc != nullptr && cudaEventCreateWithFlags(&v->ev, cudaEventDisableTiming) == cudaSuccess) {
    NVTB_CUDA_OK(cudaMemcpyAsync(v->h_sc, v->d_sc, sizeof(VocabScalars), cudaMemcpyDeviceToHost, st));
    NVTB_CUDA_OK(cudaEventRecord(v->ev, st));
    v->pending = true;
    return NVTB_OK;
  }
  pin_release(v->h_sc);
  v->h_sc = nullptr;
  v->ev = nullptr;
  VocabScalars h;
  NVTB_CUDA_OK(cudaMemcpyAsync(&h, v->d_sc, sizeof(h), cudaMemcpyDeviceToHost, st));
  NVTB_CUDA_OK(cudaStreamSynchronize(st));
  vocab_apply(v, h);
  cudaFreeAsync(v->d_sc, st);
  v->d_sc = nullptr;
  return NVTB_OK;
}

// (key, size) rows -> packed pairs (key ^ 2^31) << 32 | size (int32-valued keys, sizes < 2^32)
__global__ void __launch_bounds__(kThreads)
pack_pairs_kernel(const int64_t* __restrict__ keys, const int64_t* __restrict__ sizes, int64_t n,
                  uint64_t* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    out[i] = ((uint64_t)((uint32_t)(int32_t)keys[i] ^ 0x80000000u) << 32) | (uint64_t)(uint32_t)sizes[i];
}

// the cut of a build (categorify.py:766-785): at most one of the two is active
struct VocabCut {
  int64_t freq_threshold;   // > 0: keep the rows with size >= freq_threshold
  int64_t max_keep;         // >= 0: keep at most this many rows (max_size - num_buckets - 2)
};

// Argument checks shared by the builds (categorify.py:1206-1211), then a new handle for n rows.
static int vocab_new(nvtb_vocab** v, VocabCut* cut, int64_t n, int64_t null_size, int64_t freq_threshold,
                     int64_t max_size, int64_t num_buckets) {
  NVTB_REQUIRE(!(freq_threshold > 0 && max_size > 0), "cannot use freq_threshold together with max_size");
  const int64_t oov_count = num_buckets > 0 ? num_buckets : 1;
  NVTB_REQUIRE(!(max_size > 0 && max_size < oov_count + 2),
               "`max_size` can never be less than the maximum of `num_buckets + 2` and `3`");
  ensure_pool_configured();
  *cut = VocabCut{freq_threshold, max_size > 0 ? max_size - (oov_count + 2) : -1};
  *v = new (std::nothrow) nvtb_vocab();
  NVTB_REQUIRE(*v != nullptr, "host allocation failed");
  (*v)->info.n_total = n;
  (*v)->info.null_size = null_size;
  return NVTB_OK;
}

// hands out a built vocabulary, or destroys it when the build failed
static int vocab_out(nvtb_vocab_t** out, nvtb_vocab* v, int rc) {
  if (rc) {
    nvtb_vocab_destroy(v);
    return rc;
  }
  *out = v;
  return NVTB_OK;
}

// Cut and meta sums of n ordered rows, on the device into v->d_sc; the host waits only when a
// freq_threshold makes the kept count data-dependent.
template <typename Rows>
static int vocab_cut(nvtb_vocab* v, Rows r, int64_t n, const VocabCut& cut, cudaStream_t st, int64_t* n_keep) {
  *n_keep = cut.freq_threshold > 0 ? 0 : (cut.max_keep >= 0 ? std::min(n, cut.max_keep) : n);
  NVTB_CUDA_OK(cudaMallocAsync(&v->d_sc, sizeof(VocabScalars), st));
  // fit_i32 starts at 1 only if positions fit the 31-bit field of the narrow layout
  const VocabScalars init = {*n_keep, 0, 0, (n < (int64_t)0x7FFFFFF0) ? 1 : 0, -1};
  NVTB_CUDA_OK(cudaMemcpyAsync(v->d_sc, &init, sizeof(init), cudaMemcpyHostToDevice, st));
  const int g = plain_grid(n);
  if (cut.freq_threshold > 0) {
    cut_kernel<Rows><<<g, kThreads, 0, st>>>(r, n, cut.freq_threshold, &v->d_sc->n_keep);
    NVTB_LAUNCH_OK();
    long long h = 0;
    NVTB_CUDA_OK(cudaMemcpyAsync(&h, &v->d_sc->n_keep, sizeof(h), cudaMemcpyDeviceToHost, st));
    NVTB_CUDA_OK(cudaStreamSynchronize(st));
    *n_keep = h;
  }
  sums_kernel<Rows><<<g, kThreads, 0, st>>>(r, n, *n_keep, v->d_sc);
  NVTB_LAUNCH_OK();
  v->info.n_kept = *n_keep;
  return NVTB_OK;
}

// Tail shared by the packed-pair builds: `sorted` (owned by v from here on) holds n pairs
// (key ^ 2^31) << 32 | count in (count desc, key asc) order.  Cut, meta sums and a narrow
// lookup of the kept keys, all read from the pairs.
static int finish_packed_vocab(nvtb_vocab* v, uint64_t* sorted, int64_t n, const VocabCut& cut, cudaStream_t st) {
  v->packed = sorted;
  int64_t n_keep = 0;
  int rc = vocab_cut(v, PackedRows{sorted}, n, cut, st, &n_keep);
  if (rc) return rc;
  // Load 0.31 .. 0.625 of the 4-way buckets (a power of two at least 1.6 n): these are the
  // vocabularies of 1e7 .. 3e8 keys, where a table twice the size costs 4 GB more HBM and memset /
  // build traffic per column, while a present key still resolves in its first bucket more than 9
  // times out of 10
  v->t.capacity = pow2_at_least(std::max<int64_t>(n_keep + n_keep * 3 / 5, 64));
  v->t.min_key_pos = -1;
  v->t.narrow = 1;
  NVTB_CUDA_OK(cudaMallocAsync(&v->t.slots, sizeof(int64_t) * v->t.capacity, st));
  const int64_t nbuckets = v->t.capacity >> 2;
  const int64_t slice_buckets = narrow_slice_buckets(nbuckets);
  const int64_t n_slices = nbuckets / slice_buckets;
  const bool sliced = n_keep >= ((int64_t)1 << 20) && n_slices >= kSlThreads && n_keep < (int64_t)0xFFFFFFF0ll;
  if (!sliced) NVTB_CUDA_OK(cudaMemsetAsync(v->t.slots, 0, sizeof(int64_t) * v->t.capacity, st));
  if (n_keep > 0) {
    const int g1 = plain_grid(n_keep);
    if (sliced) {
      static bool sl_attrs = false;
      const bool smem_build = slice_buckets == kSliceBuckets;
      const int P = (int)n_slices;                                   // a power of two <= 8192
      int lg_slice = 0;
      while (((int64_t)1 << lg_slice) < slice_buckets) ++lg_slice;
      const int scatter_smem = kSlTile * 8 + 2 * 4 * kSliceParts;
      if (!sl_attrs) {
        NVTB_CUDA_OK(cudaFuncSetAttribute(slice_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * 4 * kSliceParts));
        NVTB_CUDA_OK(cudaFuncSetAttribute(slice_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, scatter_smem));
        NVTB_CUDA_OK(cudaFuncSetAttribute(slice_build_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSlBuildSmem));
        sl_attrs = true;
      }
      uint32_t* meta = nullptr;                                      // total[P] | starts[P + 1] | cursor[P]
      uint64_t* items = nullptr;
      NVTB_CUDA_OK(cudaMallocAsync(&meta, sizeof(uint32_t) * (3 * (size_t)P + 8), st));
      NVTB_CUDA_OK(cudaMallocAsync(&items, sizeof(uint64_t) * (size_t)n_keep, st));
      NVTB_CUDA_OK(cudaMemsetAsync(meta, 0, sizeof(uint32_t) * P, st));
      const uint32_t bmask = (uint32_t)(nbuckets - 1);
      const int sms = sm_count();
      slice_hist_kernel<<<4 * sms, kSlThreads, 4 * P, st>>>(sorted, n_keep, bmask, lg_slice, P, meta);
      NVTB_LAUNCH_OK();
      slice_scan_kernel<<<1, kSlThreads, 2 * 4 * P, st>>>(meta, P, meta + P, meta + 2 * P + 1);
      NVTB_LAUNCH_OK();
      const int64_t tiles = (n_keep + kSlTile - 1) / kSlTile;
      slice_scatter_kernel<<<(int)std::min<int64_t>(tiles, sms), kSlThreads, kSlTile * 8 + 2 * 4 * P, st>>>(
          sorted, n_keep, bmask, lg_slice, P, meta + 2 * P + 1, items);
      NVTB_LAUNCH_OK();
      if (smem_build)
        slice_build_smem_kernel<<<P, kSlBuildThreads, kSlBuildSmem, st>>>(items, meta + P,
                                                                          reinterpret_cast<unsigned long long*>(v->t.slots), bmask);
      else
        slice_build_kernel<<<P, 1024, 0, st>>>(items, meta + P, reinterpret_cast<unsigned long long*>(v->t.slots), bmask, lg_slice);
      NVTB_LAUNCH_OK();
      NVTB_CUDA_OK(cudaFreeAsync(items, st));
      NVTB_CUDA_OK(cudaFreeAsync(meta, st));
    } else {
      lookup_build_packed_kernel<<<g1, kThreads, 0, st>>>(sorted, n_keep, reinterpret_cast<unsigned long long*>(v->t.slots),
                                                          v->t.capacity);
      NVTB_LAUNCH_OK();
    }
    if (n_keep <= kEncSmemMaxKeys) {        // the shared-memory encode reads int64 keys
      NVTB_CUDA_OK(cudaMallocAsync(&v->keys, sizeof(int64_t) * n_keep, st));
      packed_unpack_kernel<<<g1, kThreads, 0, st>>>(sorted, n_keep, v->keys, nullptr);
      NVTB_LAUNCH_OK();
    }
  }
  return vocab_post(v, st);
}

// Rows of (key, size) in any order, n of them.
static int vocab_from_rows(nvtb_vocab* v, const int64_t* keys, const int64_t* sizes, int64_t n, const VocabCut& cut,
                           int key_bits, int64_t size_bound, cudaStream_t st) {
  if (n == 0) {                          // a wide table with nothing in it
    int rc = lookup_create(&v->t, nullptr, 0, nullptr, nullptr, st);
    if (rc) return rc;
    NVTB_CUDA_OK(cudaStreamSynchronize(st));
    return NVTB_OK;
  }
  if (n <= kSmallVocabMax) {
    int n2 = 2;
    while (n2 < n) n2 <<= 1;
    NVTB_CUDA_OK(cudaMallocAsync(&v->keys, sizeof(int64_t) * n, st));
    NVTB_CUDA_OK(cudaMallocAsync(&v->sizes, sizeof(int64_t) * n, st));
    NVTB_CUDA_OK(cudaMallocAsync(&v->d_sc, sizeof(VocabScalars), st));
    const VocabScalars init = {n, 0, 0, 1, -1};
    NVTB_CUDA_OK(cudaMemcpyAsync(v->d_sc, &init, sizeof(init), cudaMemcpyHostToDevice, st));
    v->t.capacity = pow2_at_least(2 * n);
    v->t.min_key_pos = -1;
    v->t.narrow = 0;
    NVTB_CUDA_OK(cudaMallocAsync(&v->t.slots, sizeof(int64_t) * 2 * v->t.capacity, st));
    const int smem = n2 * 16;
    NVTB_CUDA_OK(cudaFuncSetAttribute(small_vocab_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmallVocabMax * 16));
    small_vocab_kernel<<<1, kSmallThreads, smem, st>>>(keys, sizes, (int)n, n2, (long long)cut.freq_threshold,
                                                        (long long)cut.max_keep, v->keys, v->sizes, v->t.slots,
                                                        (long long)v->t.capacity, v->d_sc);
    NVTB_LAUNCH_OK();
    return vocab_post(v, st);
  }
  // (1) key asc, (2) stable size desc  =>  (size desc, key asc).  Radix passes are the cost
  // here: sort only the bits that can differ.  Keys known to be int32 values (sign-extended)
  // are biased by 2^31 (flip bit 31) so that their low 32 bits order them; sizes are bounded
  // by the number of rows seen.
  const bool key32 = (key_bits > 0 && key_bits <= 32);
  int size_bits = 64;
  if (size_bound > 0) {
    size_bits = 1;
    while (size_bits < 63 && ((int64_t)1 << size_bits) <= size_bound) ++size_bits;
  }
  const int g_x = plain_grid(n);
  if (key32 && size_bound > 0 && size_bound < ((int64_t)1 << 32) && n < (int64_t)0x7FFFFFF0) {
    // int32 keys, counts below 2^32 (every Categorify column of the Criteo workload): the rows
    // become packed pairs (key ^ 2^31) << 32 | size and the order (size desc, key asc) is two runs
    // of the hand-written stable radix passes (radix.cuh) over the bits that can differ — key
    // bits ascending, then size bits descending — followed by the same tail as the sorted
    // accumulators (cut, meta sums, narrow lookup).  No library sort on this path.
    uint64_t *p0 = nullptr, *p1 = nullptr;
    void* scratch = nullptr;
    const size_t sbytes = rx_scratch_bytes<uint64_t>(n);
    NVTB_CUDA_OK(cudaMallocAsync(&p0, sizeof(uint64_t) * n, st));
    NVTB_CUDA_OK(cudaMallocAsync(&p1, sizeof(uint64_t) * n, st));
    NVTB_CUDA_OK(cudaMallocAsync(&scratch, sbytes, st));
    NVTB_CUDA_OK(cudaMemsetAsync(scratch, 0, 256, st));
    pack_pairs_kernel<<<g_x, kThreads, 0, st>>>(keys, sizes, n, p0);
    NVTB_LAUNCH_OK();
    int in_b = 0;
    int rc = rx_sort_bits<uint64_t>(nullptr, p0, p1, nullptr, n, 32, 64, false, scratch, sbytes, st, &in_b);
    if (rc) return rc;
    uint64_t* cur = in_b ? p1 : p0;
    uint64_t* oth = in_b ? p0 : p1;
    int in_o = 0;
    rc = rx_sort_bits<uint64_t>(nullptr, cur, oth, nullptr, n, 0, std::min(size_bits, 32), true, scratch, sbytes, st,
                                &in_o);
    if (rc) return rc;
    NVTB_CUDA_OK(cudaFreeAsync(in_o ? cur : oth, st));
    NVTB_CUDA_OK(cudaFreeAsync(scratch, st));
    return finish_packed_vocab(v, in_o ? oth : cur, n, cut, st);
  }
  // any other keys or sizes: cub::DeviceRadixSort (library code), the only sort for 64-bit
  // keys.  The sorted arrays ARE the vocabulary (first n_keep rows); no second copy.
  int64_t *k1 = nullptr, *s1 = nullptr;
  NVTB_CUDA_OK(cudaMallocAsync(&k1, sizeof(int64_t) * n, st));
  NVTB_CUDA_OK(cudaMallocAsync(&s1, sizeof(int64_t) * n, st));
  NVTB_CUDA_OK(cudaMallocAsync(&v->keys, sizeof(int64_t) * n, st));
  NVTB_CUDA_OK(cudaMallocAsync(&v->sizes, sizeof(int64_t) * n, st));
  int64_t* k2 = v->keys;
  int64_t* s2 = v->sizes;
  const int64_t* sort_in = keys;
  if (key32) {
    xor_copy_kernel<<<g_x, kThreads, 0, st>>>(keys, k2, n, 0x80000000ll);   // k2 is free until the 2nd sort
    NVTB_LAUNCH_OK();
    sort_in = k2;
  }
  const int kb = key32 ? 32 : 64;
  size_t tmp_a = 0, tmp_b = 0;
  NVTB_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_a, sort_in, k1, sizes, s1, n, 0, kb, st));
  NVTB_CUDA_OK(cub::DeviceRadixSort::SortPairsDescending(nullptr, tmp_b, s1, s2, k1, k2, n, 0, size_bits, st));
  size_t tmp_bytes = std::max(tmp_a, tmp_b);
  void* tmp = nullptr;
  NVTB_CUDA_OK(cudaMallocAsync(&tmp, tmp_bytes ? tmp_bytes : 1, st));
  NVTB_CUDA_OK(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, sort_in, k1, sizes, s1, n, 0, kb, st));
  if (key32) {
    xor_copy_kernel<<<g_x, kThreads, 0, st>>>(k1, k1, n, 0x80000000ll);     // undo the bias
    NVTB_LAUNCH_OK();
  }
  NVTB_CUDA_OK(cub::DeviceRadixSort::SortPairsDescending(tmp, tmp_bytes, s1, s2, k1, k2, n, 0, size_bits, st));
  NVTB_CUDA_OK(cudaFreeAsync(k1, st));
  NVTB_CUDA_OK(cudaFreeAsync(s1, st));
  NVTB_CUDA_OK(cudaFreeAsync(tmp, st));
  int64_t n_keep = 0;
  int rc = vocab_cut(v, ArrayRows{k2, s2}, n, cut, st, &n_keep);
  if (rc) return rc;
  rc = lookup_create(&v->t, k2, n_keep, v->d_sc, nullptr, st);
  if (rc) return rc;
  return vocab_post(v, st);
}

// Pairs of a sorted accumulator, already in key order: (size desc, key asc) is ONE stable radix
// sort on the size bits in use (max size from the handle's counters: 8-10 bits = one pass for the
// high-cardinality columns this path exists for), none when every size is 1.  The first pass
// reads the accumulator, which stays as it is.
static int vocab_from_key_order(nvtb_vocab* v, const uint64_t* pairs, int64_t n, uint64_t max_count,
                                const VocabCut& cut, cudaStream_t st) {
  int bits = 0;
  while (bits < 32 && (max_count >> bits) != 0) ++bits;
  if (bits <= 1) bits = 0;
  uint64_t *p0 = nullptr, *p1 = nullptr;
  void* scratch = nullptr;
  const size_t sbytes = bits ? rx_scratch_bytes<uint64_t>(n) : 0;
  NVTB_CUDA_OK(cudaMallocAsync(&p0, sizeof(uint64_t) * n, st));
  if (sbytes) {
    NVTB_CUDA_OK(cudaMallocAsync(&scratch, sbytes, st));
    NVTB_CUDA_OK(cudaMemsetAsync(scratch, 0, 256, st));
  }
  if (rx_plan(bits).passes > 1) NVTB_CUDA_OK(cudaMallocAsync(&p1, sizeof(uint64_t) * n, st));
  int in_b = 0;
  int rc = rx_sort_bits<uint64_t>(pairs, p0, p1, nullptr, n, 0, bits, true, scratch, sbytes, st, &in_b);
  if (rc) return rc;
  if (scratch) NVTB_CUDA_OK(cudaFreeAsync(scratch, st));
  if (p1) NVTB_CUDA_OK(cudaFreeAsync(in_b ? p0 : p1, st));
  return finish_packed_vocab(v, in_b ? p1 : p0, n, cut, st);
}

}  // namespace nvtb

using namespace nvtb;

extern "C" {

int nvtb_vocab_build(nvtb_vocab_t** out, const int64_t* keys, const int64_t* sizes,
                     int64_t n, int64_t null_size, int64_t freq_threshold,
                     int64_t max_size, int64_t num_buckets, int key_bits,
                     int64_t size_bound, void* stream) {
  NVTB_REQUIRE(out != nullptr && n >= 0, "out NULL or n < 0");
  NVTB_REQUIRE(n == 0 || (keys && sizes), "NULL keys/sizes");
  nvtb_vocab* v = nullptr;
  VocabCut cut;
  int rc = vocab_new(&v, &cut, n, null_size, freq_threshold, max_size, num_buckets);
  if (rc) return rc;
  return vocab_out(out, v, vocab_from_rows(v, keys, sizes, n, cut, key_bits, size_bound, (cudaStream_t)stream));
}

// Vocabulary straight from a group-by handle (single GPU: no int64 export round trip).  A
// sorted accumulator's pairs are ordered in place of the handle (vocab_from_key_order); a hash
// table is exported into temporaries and handed to nvtb_vocab_build.
int nvtb_vocab_build_from_hashagg(nvtb_vocab_t** out, nvtb_hashagg_t* h, int64_t freq_threshold,
                                  int64_t max_size, int64_t num_buckets, int key_bits,
                                  int64_t size_bound, void* stream) {
  NVTB_REQUIRE(out != nullptr && h != nullptr, "NULL argument");
  cudaStream_t st = (cudaStream_t)stream;
  const uint64_t* pairs = nullptr;
  int64_t n = 0, null_size = 0;
  uint64_t maxc = 0;
  int is_i32 = 0;
  int rc = hashagg_sorted_view(h, &pairs, &n, &null_size, &maxc, &is_i32, st);
  if (rc) return rc;
  if (pairs == nullptr || n == 0 || n >= (int64_t)0x7FFFFFF0) {
    int64_t *k = nullptr, *s = nullptr;
    if (n > 0) {
      NVTB_CUDA_OK(cudaMallocAsync(&k, sizeof(int64_t) * n, st));
      NVTB_CUDA_OK(cudaMallocAsync(&s, sizeof(int64_t) * n, st));
      rc = nvtb_hashagg_export(h, k, s, nullptr, nullptr, stream);
      if (rc) return rc;
    }
    rc = nvtb_vocab_build(out, k, s, n, null_size, freq_threshold, max_size, num_buckets,
                          (key_bits > 0 || is_i32) ? 32 : 0, size_bound, stream);
    if (k) cudaFreeAsync(k, st);
    if (s) cudaFreeAsync(s, st);
    return rc;
  }
  nvtb_vocab* v = nullptr;
  VocabCut cut;
  rc = vocab_new(&v, &cut, n, null_size, freq_threshold, max_size, num_buckets);
  if (rc) return rc;
  return vocab_out(out, v, vocab_from_key_order(v, pairs, n, maxc, cut, st));
}

// Vocabulary from packed pairs that are ALREADY in (count desc, key asc) order — the cross-GPU
// merge (nvtabular_b200/dist.py) assembles that order from the owners' shards.  The array is
// copied; cut, meta sums and the lookup table are the single-GPU code.
int nvtb_vocab_build_from_pairs(nvtb_vocab_t** out, const uint64_t* ordered_pairs, int64_t n, int64_t null_size,
                                int64_t freq_threshold, int64_t max_size, int64_t num_buckets, void* stream) {
  NVTB_REQUIRE(out != nullptr && n >= 0 && n < (int64_t)0x7FFFFFF0, "NULL out or n out of range");
  NVTB_REQUIRE(n == 0 || ordered_pairs != nullptr, "NULL pairs");
  nvtb_vocab* v = nullptr;
  VocabCut cut;
  int rc = vocab_new(&v, &cut, n, null_size, freq_threshold, max_size, num_buckets);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rc = [&]() -> int {
    uint64_t* p0 = nullptr;
    NVTB_CUDA_OK(cudaMallocAsync(&p0, sizeof(uint64_t) * (n > 0 ? n : 1), st));
    v->packed = p0;
    if (n > 0) NVTB_CUDA_OK(cudaMemcpyAsync(p0, ordered_pairs, sizeof(uint64_t) * n, cudaMemcpyDeviceToDevice, st));
    return finish_packed_vocab(v, p0, n, cut, st);
  }();
  return vocab_out(out, v, rc);
}

int nvtb_vocab_from_arrays(nvtb_vocab_t** out, const int64_t* keys, const int64_t* sizes,
                           int64_t n, void* stream) {
  NVTB_REQUIRE(out != nullptr && n >= 0, "out NULL or n < 0");
  NVTB_REQUIRE(n == 0 || keys, "NULL keys");
  cudaStream_t st = (cudaStream_t)stream;
  nvtb_vocab* v = new (std::nothrow) nvtb_vocab();
  NVTB_REQUIRE(v != nullptr, "host allocation failed");
  memset(v, 0, sizeof(*v));
  v->info.n_kept = n;
  v->info.n_total = n;
  if (n > 0) {
    NVTB_CUDA_OK(cudaMallocAsync(&v->keys, sizeof(int64_t) * n, st));
    NVTB_CUDA_OK(cudaMemcpyAsync(v->keys, keys, sizeof(int64_t) * n, cudaMemcpyDeviceToDevice, st));
    if (sizes) {
      NVTB_CUDA_OK(cudaMallocAsync(&v->sizes, sizeof(int64_t) * n, st));
      NVTB_CUDA_OK(cudaMemcpyAsync(v->sizes, sizes, sizeof(int64_t) * n, cudaMemcpyDeviceToDevice, st));
    }
  }
  int rc = lookup_create_wide(&v->t, v->keys, n, st);
  if (rc) { nvtb_vocab_destroy(v); return rc; }
  *out = v;
  return NVTB_OK;
}

int nvtb_vocab_destroy(nvtb_vocab_t* v) {
  if (v == nullptr) return NVTB_OK;
  vocab_finalize(v);
  if (v->ev) cudaEventDestroy(v->ev);
  // stream-ordered frees on the legacy default stream: ordered after every kernel
  // that may still probe the table, without a device-wide host sync
  if (v->t.slots) cudaFreeAsync(v->t.slots, 0);
  if (v->keys) cudaFreeAsync(v->keys, 0);
  if (v->sizes) cudaFreeAsync(v->sizes, 0);
  if (v->packed) cudaFreeAsync(v->packed, 0);
  if (v->d_sc) cudaFreeAsync(v->d_sc, 0);      // a build that failed before its readback
  delete v;
  return NVTB_OK;
}

int nvtb_vocab_info(const nvtb_vocab_t* v, nvtb_vocab_info_t* info) {
  NVTB_REQUIRE(v != nullptr && info != nullptr, "NULL argument");
  { int frc = vocab_finalize(const_cast<nvtb_vocab_t*>(v)); if (frc) return frc; }
  *info = v->info;
  return NVTB_OK;
}

int nvtb_vocab_export(const nvtb_vocab_t* v, int64_t* keys_out, int64_t* sizes_out, void* stream) {
  NVTB_REQUIRE(v != nullptr, "NULL vocab");
  { int frc = vocab_finalize(const_cast<nvtb_vocab_t*>(v)); if (frc) return frc; }
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n = v->info.n_kept;
  if (n == 0) return NVTB_OK;
  if (v->packed != nullptr) {
    packed_unpack_kernel<<<plain_grid(n), kThreads, 0, st>>>(v->packed, n, keys_out, sizes_out);
    NVTB_LAUNCH_OK();
    return NVTB_OK;
  }
  if (keys_out)
    NVTB_CUDA_OK(cudaMemcpyAsync(keys_out, v->keys, sizeof(int64_t) * n, cudaMemcpyDeviceToDevice, st));
  if (sizes_out) {
    NVTB_REQUIRE(v->sizes != nullptr, "vocab has no sizes");
    NVTB_CUDA_OK(cudaMemcpyAsync(sizes_out, v->sizes, sizeof(int64_t) * n, cudaMemcpyDeviceToDevice, st));
  }
  return NVTB_OK;
}

int nvtb_encode_apply(const nvtb_vocab_t* v, const nvtb_col_t* key, int64_t n,
                      int64_t null_label, int64_t oov_label, int64_t first_label,
                      uint64_t num_buckets, const nvtb_col_t* hash_cols, int n_hash_cols,
                      void* out, int out_dtype, void* stream) {
  NVTB_REQUIRE(v != nullptr && key != nullptr && n >= 0, "NULL argument or n < 0");
  { int frc = vocab_finalize(const_cast<nvtb_vocab_t*>(v)); if (frc) return frc; }
  NVTB_REQUIRE(key->dtype == NVTB_I32 || key->dtype == NVTB_I64, "key dtype must be int32 or int64");
  NVTB_REQUIRE(out_dtype == NVTB_I32 || out_dtype == NVTB_I64, "out_dtype must be int32 or int64");
  NVTB_REQUIRE(n_hash_cols >= 0 && n_hash_cols <= kMaxHashCols, "n_hash_cols must be in [0, 8]");
  NVTB_REQUIRE(n_hash_cols == 0 || hash_cols != nullptr, "hash_cols is NULL");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(key->data && out, "NULL data/out");
  HashCols hc;
  memset(&hc, 0, sizeof(hc));
  hc.ncols = n_hash_cols;
  for (int c = 0; c < n_hash_cols; ++c) {
    NVTB_REQUIRE(hash_cols[c].data != nullptr && hash_cols[c].dtype >= NVTB_I32 && hash_cols[c].dtype <= NVTB_H64,
                 "bad hash column");
    hc.data[c] = hash_cols[c].data; hc.mask[c] = hash_cols[c].validity; hc.dtype[c] = hash_cols[c].dtype;
  }
  EncodeParams p{null_label, oov_label, first_label, num_buckets};
  cudaStream_t st = (cudaStream_t)stream;
  if (key->dtype == NVTB_I32 && v->t.narrow && v->info.n_kept > 0 && v->info.n_kept <= kEncSmemMaxKeys &&
      n >= ((int64_t)1 << 18) && is_aligned32(key->data) && is_aligned32(out)) {
    constexpr int kSmem = (int)(kEncSmemBuckets * 4 * 8);
    constexpr int64_t kStep = (int64_t)kEncSmemThreads * 8;
    const int g = (int)std::min<int64_t>(sm_count(), (n + kStep - 1) / kStep);
    if (out_dtype == NVTB_I64) {
      NVTB_CUDA_OK(cudaFuncSetAttribute(encode_smem_kernel<int64_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
      encode_smem_kernel<int64_t><<<g, kEncSmemThreads, kSmem, st>>>(
          (const int32_t*)key->data, key->validity, n, v->keys, (int)v->info.n_kept, v->t, p, hc, (int64_t*)out);
    } else {
      NVTB_CUDA_OK(cudaFuncSetAttribute(encode_smem_kernel<int32_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
      encode_smem_kernel<int32_t><<<g, kEncSmemThreads, kSmem, st>>>(
          (const int32_t*)key->data, key->validity, n, v->keys, (int)v->info.n_kept, v->t, p, hc, (int32_t*)out);
    }
    NVTB_LAUNCH_OK();
    return NVTB_OK;
  }
  const int grid = scan_grid(n, 8);
#define NVTB_ENCODE(KT, OT)                                                                        \
  do {                                                                                             \
    if (v->t.narrow)                                                                               \
      encode_kernel<KT, OT, true><<<grid, kThreads, 0, st>>>((const KT*)key->data, key->validity, n, v->t, p, hc, (OT*)out); \
    else                                                                                           \
      encode_kernel<KT, OT, false><<<grid, kThreads, 0, st>>>((const KT*)key->data, key->validity, n, v->t, p, hc, (OT*)out); \
  } while (0)
  if (key->dtype == NVTB_I32) {
    if (out_dtype == NVTB_I64) NVTB_ENCODE(int32_t, int64_t); else NVTB_ENCODE(int32_t, int32_t);
  } else {
    if (out_dtype == NVTB_I64) NVTB_ENCODE(int64_t, int64_t); else NVTB_ENCODE(int64_t, int32_t);
  }
#undef NVTB_ENCODE
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

int nvtb_groupstats_create(nvtb_groupstats_t** out, const int64_t* keys, int64_t n_groups,
                           const double* stats, int width, int64_t null_row, void* stream) {
  NVTB_REQUIRE(out != nullptr && n_groups >= 0 && width >= 1, "bad arguments");
  NVTB_REQUIRE(n_groups == 0 || (keys && stats), "NULL keys/stats");
  NVTB_REQUIRE(null_row >= -1, "null_row must be >= -1");
  cudaStream_t st = (cudaStream_t)stream;
  nvtb_groupstats* g = new (std::nothrow) nvtb_groupstats();
  NVTB_REQUIRE(g != nullptr, "host allocation failed");
  memset(g, 0, sizeof(*g));
  g->n_groups = n_groups; g->width = width; g->null_row = null_row;
  // the stats matrix may have more rows than keys (the null group's row)
  const int64_t n_rows = std::max<int64_t>(n_groups, null_row + 1);
  if (n_rows > 0) {
    NVTB_CUDA_OK(cudaMallocAsync(&g->stats, sizeof(double) * n_rows * width, st));
    NVTB_CUDA_OK(cudaMemcpyAsync(g->stats, stats, sizeof(double) * n_rows * width, cudaMemcpyDeviceToDevice, st));
  }
  int rc = lookup_create_wide(&g->t, keys, n_groups, st);
  if (rc) { nvtb_groupstats_destroy(g); return rc; }
  *out = g;
  return NVTB_OK;
}

int nvtb_groupstats_destroy(nvtb_groupstats_t* g) {
  if (g == nullptr) return NVTB_OK;
  if (g->t.slots) cudaFreeAsync(g->t.slots, 0);
  if (g->stats) cudaFreeAsync(g->stats, 0);
  delete g;
  return NVTB_OK;
}

int nvtb_groupstats_gather(const nvtb_groupstats_t* g, const nvtb_col_t* key, int64_t n,
                           const int* cols, int ncols_out, const double* miss_vals,
                           void* const* out, const int* out_dtypes, uint8_t* const* valid_out,
                           void* stream) {
  NVTB_REQUIRE(g != nullptr && key != nullptr && n >= 0, "NULL argument or n < 0");
  NVTB_REQUIRE(key->dtype == NVTB_I32 || key->dtype == NVTB_I64, "key dtype must be int32 or int64");
  NVTB_REQUIRE(ncols_out >= 1 && ncols_out <= kMaxGatherCols, "ncols_out must be in [1, 16]");
  NVTB_REQUIRE(cols && miss_vals && out && out_dtypes, "NULL argument");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(key->data != nullptr, "key data is NULL");
  GatherOut go;
  memset(&go, 0, sizeof(go));
  go.ncols = ncols_out;
  for (int j = 0; j < ncols_out; ++j) {
    NVTB_REQUIRE(cols[j] >= 0 && cols[j] < g->width, "stats column out of range");
    NVTB_REQUIRE(out[j] != nullptr, "out column is NULL");
    NVTB_REQUIRE(out_dtypes[j] >= NVTB_I32 && out_dtypes[j] <= NVTB_F64, "bad out dtype");
    go.out[j] = out[j]; go.miss[j] = miss_vals[j]; go.col[j] = cols[j]; go.dtype[j] = out_dtypes[j];
    go.valid[j] = valid_out != nullptr ? reinterpret_cast<uint32_t*>(valid_out[j]) : nullptr;
    NVTB_REQUIRE((reinterpret_cast<uintptr_t>(go.valid[j]) & 3u) == 0, "validity output must be 4-byte aligned");
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = (int)std::min<int64_t>((n + kThreads - 1) / kThreads, (int64_t)sm_count() * 8);
  if (key->dtype == NVTB_I32)
    gather_stats_kernel<int32_t><<<grid, kThreads, 0, st>>>((const int32_t*)key->data, key->validity, n, g->t, g->null_row, g->stats, g->width, go);
  else
    gather_stats_kernel<int64_t><<<grid, kThreads, 0, st>>>((const int64_t*)key->data, key->validity, n, g->t, g->null_row, g->stats, g->width, go);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

}  // extern "C"
