// sortagg.cuh — K3 for HIGH-CARDINALITY int32 key columns: a sort-based group-by.
// Included by sortacc.cu after partition.cuh (its kernels with PartKeyLow are the first,
// order-free radix pass).
//
// Why: once the resident hash table of a column no longer fits the 50 MB L2 (Criteo's
// C20/C1/C22/C10: 1.3e8-2.9e8 distinct keys, tables of 2-4 GB), every row of a batch costs a
// random DRAM sector + atomic in the table instead of an L2 hit, and the vocabulary build then has to radix-sort all U (key, size) pairs twice.  The
// reference meets the same wall with a per-partition cuDF groupby and a tree of
// concat+groupby over host memory (nvtabular/ops/categorify.py:955-1137).
//
// Here the accumulator of such a column is a SORTED array of packed pairs
//     word = (uint32)(key ^ 2^31) << 32 | (uint32)count        (unsigned order == key order)
// and a batch is folded in with streaming passes only:
//     1. LSD radix sort of the batch's valid keys: low 12 bits with the order-free partition
//        kernels of partition.cuh (shared-memory atomics, nulls dropped and counted on the way),
//        bits 12-21 and 22-31 with the stable passes of radix.cuh
//     2. run-length encode the sorted keys -> (key, first index) per distinct key
//     3. merge the batch's distinct keys with the accumulator, adding counts (merge-path
//        tiles of 4096 elements, cross-ranked by binary search in shared memory)
// No table sizing, no cardinality estimate, no overflow arena; the result is key-ordered, so
// the vocabulary build only needs a stable sort on the COUNT (one 8-10 bit pass for these
// columns) and the cross-GPU exchange can split by key range.
#pragma once

#include "radix.cuh"

namespace nvtb {

constexpr int kRunThreads = 512;
constexpr int kRleTile = 8192;           // keys per CTA in the run-length kernels
constexpr int kRleItems = kRleTile / kRunThreads;
constexpr int kMergeTile = 4096;         // merged elements per CTA
constexpr int kSortLowBits = 12;         // first (order-free) pass

__device__ __forceinline__ uint32_t pk_hi(uint64_t w) { return (uint32_t)(w >> 32); }
__device__ __forceinline__ uint32_t pk_lo(uint64_t w) { return (uint32_t)w; }
__host__ __device__ __forceinline__ int32_t ukey_to_key(uint32_t u) { return (int32_t)(u ^ 0x80000000u); }

// block-wide sum of a small per-thread value (kRunThreads threads)
__device__ __forceinline__ uint32_t run_block_sum(uint32_t v, uint32_t* ws /*[kRunThreads/32]*/) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, o);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t t = 0;
  if (threadIdx.x < 32) {
    t = threadIdx.x < kRunThreads / 32 ? ws[threadIdx.x] : 0u;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xFFFFFFFFu, t, o);
    if (threadIdx.x == 0) ws[0] = t;
  }
  __syncthreads();
  t = ws[0];
  __syncthreads();
  return t;
}

// block-wide exclusive scan of one value per thread; returns the exclusive prefix, *total
// receives the block total
__device__ __forceinline__ uint32_t run_block_excl(uint32_t v, uint32_t* ws /*[kRunThreads/32 + 1]*/, uint32_t* total) {
  uint32_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if ((threadIdx.x & 31) >= o) incl += y;
  }
  if ((threadIdx.x & 31) == 31) ws[threadIdx.x >> 5] = incl;
  __syncthreads();
  if (threadIdx.x < 32) {
    uint32_t w = threadIdx.x < kRunThreads / 32 ? ws[threadIdx.x] : 0u;
    uint32_t wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, wi, o);
      if (threadIdx.x >= o) wi += y;
    }
    if (threadIdx.x < kRunThreads / 32) ws[threadIdx.x] = wi - w;
    if (threadIdx.x == kRunThreads / 32 - 1) ws[kRunThreads / 32] = wi;
  }
  __syncthreads();
  const uint32_t ex = ws[threadIdx.x >> 5] + incl - v;
  *total = ws[kRunThreads / 32];
  __syncthreads();
  return ex;
}

// exclusive scan of vals[0..T) in place (ONE CTA); the total goes to total32 / total64
// (either may be NULL)
static __global__ void __launch_bounds__(kRunThreads)
scan_tiles_kernel(uint32_t* __restrict__ vals, int T, uint32_t* total32, unsigned long long* total64) {
  __shared__ uint32_t ws[kRunThreads / 32 + 1];
  constexpr int kPer = 8;
  uint32_t carry = 0;
  for (int c0 = 0; c0 < T; c0 += kRunThreads * kPer) {
    uint32_t v[kPer], local = 0;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int i = c0 + threadIdx.x * kPer + j;
      v[j] = i < T ? vals[i] : 0u;
      local += v[j];
    }
    uint32_t tot;
    uint32_t run = carry + run_block_excl(local, ws, &tot);
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int i = c0 + threadIdx.x * kPer + j;
      if (i < T) vals[i] = run;
      run += v[j];
    }
    carry += tot;
  }
  if (threadIdx.x == 0) {
    if (total32) *total32 = carry;
    if (total64) *total64 = (unsigned long long)carry;
  }
}

// ---------------------------------------------------------------------------------------
// run-length encoding of the sorted keys
// ---------------------------------------------------------------------------------------
// kRleItems consecutive keys of one thread (128-bit loads; `keys` is 16-byte aligned and
// `base` a multiple of kRleItems)
__device__ __forceinline__ void rle_load(const uint32_t* __restrict__ keys, int64_t base, int64_t n,
                                         uint32_t (&k)[kRleItems]) {
#pragma unroll
  for (int q = 0; q < kRleItems / 4; ++q) {
    const int64_t i = base + 4 * q;
    if (i + 4 <= n) {
      const uint4 v = *reinterpret_cast<const uint4*>(keys + i);
      k[4 * q] = v.x; k[4 * q + 1] = v.y; k[4 * q + 2] = v.z; k[4 * q + 3] = v.w;
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) k[4 * q + e] = (i + e < n) ? keys[i + e] : 0u;
    }
  }
}

// number of run heads per tile (a head: first key, or a key different from its predecessor)
static __global__ void __launch_bounds__(kRunThreads)
rle_count_kernel(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ n_ptr, int64_t n_max,
                 uint32_t* __restrict__ tile_heads) {
  __shared__ uint32_t ws[kRunThreads / 32];
  const int64_t n = rx_count(n_ptr, n_max);
  const int64_t base = (int64_t)blockIdx.x * kRleTile + (int64_t)threadIdx.x * kRleItems;
  uint32_t heads = 0;
  if (base < n) {
    uint32_t k[kRleItems];
    rle_load(keys, base, n, k);
    uint32_t prev = base > 0 ? keys[base - 1] : 0u;
    bool first = (base == 0);
#pragma unroll
    for (int j = 0; j < kRleItems; ++j) {
      if (base + j < n) {
        heads += (first || k[j] != prev) ? 1u : 0u;
        prev = k[j];
        first = false;
      }
    }
  }
  const uint32_t tot = run_block_sum(heads, ws);
  if (threadIdx.x == 0) tile_heads[blockIdx.x] = tot;
}

// out[tile_off + r] = key << 32 | index of the run's first element; out[U] = sentinel whose
// low word is n (so that count of run r = lo(out[r + 1]) - lo(out[r]))
static __global__ void __launch_bounds__(kRunThreads)
rle_write_kernel(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ n_ptr, int64_t n_max,
                 const uint32_t* __restrict__ tile_off, const uint32_t* __restrict__ n_unique,
                 uint64_t* __restrict__ out) {
  __shared__ uint32_t ws[kRunThreads / 32 + 1];
  const int64_t n = rx_count(n_ptr, n_max);
  if (blockIdx.x == 0 && threadIdx.x == 0) out[*n_unique] = (0xFFFFFFFFull << 32) | (uint64_t)(uint32_t)n;
  const int64_t base = (int64_t)blockIdx.x * kRleTile + (int64_t)threadIdx.x * kRleItems;
  uint32_t k[kRleItems];
  uint32_t flags = 0;
  if (base < n) {
    rle_load(keys, base, n, k);
    uint32_t prev = base > 0 ? keys[base - 1] : 0u;
    bool first = (base == 0);
#pragma unroll
    for (int j = 0; j < kRleItems; ++j) {
      if (base + j < n) {
        if (first || k[j] != prev) flags |= 1u << j;
        prev = k[j];
        first = false;
      }
    }
  }
  uint32_t tot;
  uint32_t r = tile_off[blockIdx.x] + run_block_excl(__popc(flags), ws, &tot);
#pragma unroll
  for (int j = 0; j < kRleItems; ++j)
    if ((flags >> j) & 1u) out[r++] = ((uint64_t)k[j] << 32) | (uint64_t)(uint32_t)(base + j);
}

// ---------------------------------------------------------------------------------------
// merge (A: accumulator pairs, sorted unique; B: run heads of the batch, sorted unique)
// ---------------------------------------------------------------------------------------
// merge-path split of every tile boundary: splits[t] = (a, b) with a + b = t * kMergeTile
// (A first on ties), then b is advanced by one when the boundary would separate a key of A
// from the same key in B, so that a key never straddles two tiles.
static __global__ void __launch_bounds__(256)
merge_split_kernel(const uint64_t* __restrict__ A, uint32_t ua, const uint64_t* __restrict__ B,
                   const uint32_t* __restrict__ ub_ptr, int MT, uint2* __restrict__ splits) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > MT) return;
  const uint32_t ub = *ub_ptr;
  const uint64_t total = (uint64_t)ua + ub;
  uint64_t diag = (uint64_t)t * kMergeTile;
  if (diag > total) diag = total;
  uint32_t lo = diag > ub ? (uint32_t)(diag - ub) : 0u;
  uint32_t hi = diag < ua ? (uint32_t)diag : ua;
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;              // a = mid, b = diag - mid  (b >= 1 here)
    const uint32_t ka = pk_hi(A[mid]);
    const uint32_t kb = pk_hi(B[diag - mid - 1]);
    if (ka <= kb) lo = mid + 1; else hi = mid;
  }
  uint32_t a = lo, b = (uint32_t)(diag - lo);
  if (a > 0 && b < ub && pk_hi(A[a - 1]) == pk_hi(B[b])) b += 1;
  splits[t] = make_uint2(a, b);
}

__device__ __forceinline__ uint32_t lower_bound_u32(const uint32_t* s, uint32_t n, uint32_t key) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (s[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// outputs of tile t = la + lb - (keys present in both parts)
static __global__ void __launch_bounds__(kRunThreads)
merge_count_kernel(const uint64_t* __restrict__ A, const uint64_t* __restrict__ B,
                   const uint2* __restrict__ splits, uint32_t* __restrict__ tile_out) {
  __shared__ uint32_t sA[kMergeTile + 2];
  __shared__ uint32_t ws[kRunThreads / 32];
  const uint2 s0 = splits[blockIdx.x], s1 = splits[blockIdx.x + 1];
  const uint32_t la = s1.x - s0.x, lb = s1.y - s0.y;
  for (uint32_t i = threadIdx.x; i < la; i += kRunThreads) sA[i] = pk_hi(A[s0.x + i]);
  __syncthreads();
  uint32_t dups = 0;
  for (uint32_t j = threadIdx.x; j < lb; j += kRunThreads) {
    const uint32_t kb = pk_hi(B[s0.y + j]);
    const uint32_t p = lower_bound_u32(sA, la, kb);
    dups += (p < la && sA[p] == kb) ? 1u : 0u;
  }
  const uint32_t tot = run_block_sum(dups, ws);
  if (threadIdx.x == 0) tile_out[blockIdx.x] = la + lb - tot;
}

struct MergeSmem {
  uint64_t a[kMergeTile + 2];        // A part (packed pairs)
  uint32_t bk[kMergeTile + 2];       // B part keys
  uint32_t bc[kMergeTile + 2];       // B part counts
  uint16_t lba[kMergeTile + 2];      // lower bound of every B key in the A part
  uint16_t dx[kMergeTile + 2];       // exclusive prefix of "B key also in A"
};

// B_PACKED = false: B holds run heads (key << 32 | first index, sentinel at B[ub]) of a sorted
// batch; true: B holds packed pairs (key << 32 | count) like A (cross-GPU shard merges)
template <bool B_PACKED>
static __global__ void __launch_bounds__(kRunThreads)
merge_write_kernel(const uint64_t* __restrict__ A, const uint64_t* __restrict__ B,
                   const uint2* __restrict__ splits, const uint32_t* __restrict__ tile_off,
                   uint64_t* __restrict__ out, unsigned long long* max_count) {
  extern __shared__ __align__(16) unsigned char run_smem[];
  MergeSmem& sm = *reinterpret_cast<MergeSmem*>(run_smem);
  __shared__ uint32_t ws[kRunThreads / 32 + 1];
  const uint2 s0 = splits[blockIdx.x], s1 = splits[blockIdx.x + 1];
  const uint32_t la = s1.x - s0.x, lb = s1.y - s0.y;
  if (la + lb == 0) return;
  for (uint32_t i = threadIdx.x; i < la; i += kRunThreads) sm.a[i] = A[s0.x + i];
  for (uint32_t j = threadIdx.x; j < lb; j += kRunThreads) {
    const uint64_t w = B[s0.y + j];
    sm.bk[j] = pk_hi(w);
    if (B_PACKED) sm.bc[j] = pk_lo(w);
    else sm.bc[j] = pk_lo(B[s0.y + j + 1]) - pk_lo(w);           // B[ub] is the sentinel
  }
  __syncthreads();
  // B -> A: lower bounds and duplicate flags; blocked so that the prefix is in index order
  constexpr int kPer = (kMergeTile + 2 + kRunThreads - 1) / kRunThreads;
  uint32_t dflags = 0;
#pragma unroll
  for (int q = 0; q < kPer; ++q) {
    const uint32_t j = threadIdx.x * kPer + q;
    if (j < lb) {
      const uint32_t kb = sm.bk[j];
      uint32_t lo = 0, hi = la;
      while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (pk_hi(sm.a[mid]) < kb) lo = mid + 1; else hi = mid; }
      sm.lba[j] = (uint16_t)lo;
      if (lo < la && pk_hi(sm.a[lo]) == kb) dflags |= 1u << q;
    }
  }
  uint32_t tot;
  uint32_t run = run_block_excl(__popc(dflags), ws, &tot);
#pragma unroll
  for (int q = 0; q < kPer; ++q) {
    const uint32_t j = threadIdx.x * kPer + q;
    if (j <= lb) sm.dx[j] = (uint16_t)run;
    run += (dflags >> q) & 1u;
  }
  __syncthreads();
  const uint64_t off = tile_off[blockIdx.x];
  uint32_t mx = 0;
  // B elements that are new keys
#pragma unroll
  for (int q = 0; q < kPer; ++q) {
    const uint32_t j = threadIdx.x * kPer + q;
    if (j < lb && !((dflags >> q) & 1u)) {
      const uint32_t c = sm.bc[j];
      out[off + sm.lba[j] + (j - sm.dx[j])] = ((uint64_t)sm.bk[j] << 32) | c;
      mx = c > mx ? c : mx;
    }
  }
  // A elements (+ the count of the same key in B)
  for (uint32_t i = threadIdx.x; i < la; i += kRunThreads) {
    const uint64_t w = sm.a[i];
    const uint32_t ka = pk_hi(w);
    const uint32_t p = lower_bound_u32(sm.bk, lb, ka);
    uint32_t c = pk_lo(w);
    if (p < lb && sm.bk[p] == ka) c += sm.bc[p];
    out[off + i + (p - sm.dx[p])] = ((uint64_t)ka << 32) | c;
    mx = c > mx ? c : mx;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const uint32_t y = __shfl_down_sync(0xFFFFFFFFu, mx, o); mx = y > mx ? y : mx; }
  if ((threadIdx.x & 31) == 0 && mx) atomicMax(max_count, (unsigned long long)mx);
}

// accumulator -> int64 key / size arrays (nvtb_hashagg_export of a sorted handle; key order)
static __global__ void __launch_bounds__(kThreads)
runs_unpack_kernel(const uint64_t* __restrict__ acc, int64_t n, int64_t* __restrict__ keys,
                   int64_t* __restrict__ sizes) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint64_t w = acc[i];
    keys[i] = (int64_t)ukey_to_key(pk_hi(w));
    if (sizes) sizes[i] = (int64_t)pk_lo(w);
  }
}

// lower bound of every unsigned key bound[j] in the key-sorted packed pairs: out[j] = number of
// pairs whose key is < bound[j] (one thread per bound)
static __global__ void pairs_lower_bound_kernel(const uint64_t* __restrict__ pairs, int64_t n,
                                                const uint32_t* __restrict__ bound, int m,
                                                long long* __restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= m) return;
  const uint32_t b = bound[j];
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (pk_hi(pairs[mid]) < b) lo = mid + 1; else hi = mid;
  }
  out[j] = (long long)lo;
}

// dst[seg_dst[s] + (i - seg_src[s])] = src[i] for i in [seg_src[s], seg_src[s + 1]): copies
// nseg contiguous segments (seg_src ascending, seg_src[nseg] = n) to their destinations.  Used
// to interleave the owners' count-ordered shards into the global (count desc, key asc) order:
// a segment = the pairs of one count value on one owner.  4 elements per thread; the segment
// of the first is found by binary search, the others usually share it.
static __global__ void __launch_bounds__(kThreads)
segment_copy_kernel(const uint64_t* __restrict__ src, uint64_t* __restrict__ dst,
                    const long long* __restrict__ seg_src, const long long* __restrict__ seg_dst,
                    int nseg, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x * 4;
  for (int64_t i0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; i0 < n; i0 += stride) {
    int lo = 0, hi = nseg;                       // last s with seg_src[s] <= i0
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (seg_src[mid] <= i0) lo = mid; else hi = mid;
    }
    int s = lo;
    long long s_end = seg_src[s + 1], d0 = seg_dst[s], shift = d0 - seg_src[s];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int64_t i = i0 + e;
      if (i >= n) break;
      while (i >= s_end) { ++s; s_end = seg_src[s + 1]; d0 = seg_dst[s]; shift = d0 - seg_src[s]; }
      if (d0 >= 0) dst[i + shift] = src[i];          // seg_dst < 0: padding, skipped
    }
  }
}

}  // namespace nvtb
