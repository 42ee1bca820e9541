// lookup.cuh — the read-only key -> position table shared by the vocabulary encode and
// group-statistics gather (vocab.cu, K5 / K7) and the external-table join probe (join.cu, K9).
#pragma once
#include "common.cuh"

namespace nvtb {

// read-only lookup table: slot = {key, position}; immutable after build so the
// probes go through the read-only (L1-cacheable) path.
// Two slot layouts, like the aggregation table:
//   wide   (16 B) {int64 key, int64 position}; empty key = INT64_MIN
//   narrow ( 8 B) ((uint32)(position + 1) << 32) | (uint32)key; empty = 0.  Used when
//                 every key fits int32 and n < 2^31: half the footprint, so more of
//                 the table stays in L1/L2, and one 8-byte load per probe.
// Narrow (int32-key) tables probe WITHIN a slice of the table: bucket b is followed by the next
// bucket of the same slice, wrapping at the slice end.  A slice is 8192 buckets (256 KB) — more
// when the table has more than 8192 slices — so that one CTA can build a whole slice while it
// stays in the L2 (slice_build_kernel), and no probe sequence ever leaves the CTA's slice.
constexpr int64_t kSliceBuckets = 8192;
constexpr int kSliceParts = 8192;                 // at most this many slices
__host__ __device__ __forceinline__ int64_t narrow_slice_buckets(int64_t nbuckets) {
  int64_t s = nbuckets / kSliceParts;
  if (s < kSliceBuckets) s = kSliceBuckets;
  return s < nbuckets ? s : nbuckets;             // powers of two throughout
}
__host__ __device__ __forceinline__ int64_t narrow_next(int64_t b, int64_t nbuckets) {
  const int64_t sm = narrow_slice_buckets(nbuckets) - 1;
  return (b & ~sm) | ((b + 1) & sm);
}

struct Lookup {
  int64_t* slots;     // wide: [2*capacity]; narrow: [capacity]
  int64_t capacity;   // power of two, >= 2 * n
  int64_t min_key_pos;  // position of key INT64_MIN (the EMPTY sentinel) or -1
  int narrow;
};

// Inserts of one key into either layout.
// narrow: keys are distinct.  Claim the first free slot of bucket b (the key's home), else of
//         the buckets after it in the same slice (narrow_next); word = ((pos + 1) << 32) | key.
__device__ __forceinline__ void narrow_claim(unsigned long long* slots, int64_t b, int64_t nbuckets,
                                             unsigned long long word) {
  for (;; b = narrow_next(b, nbuckets))
    for (int j = 0; j < 4; ++j)
      if (atomicCAS(slots + 4 * b + j, 0ull, word) == 0ull) return;
}

// wide: linear probing from the key's home; a repeated key (user vocab) keeps its smallest
// position (slots start at {kEmptyKey, INT64_MAX}).  kEmptyKey itself cannot be stored: the
// caller records its position in Lookup::min_key_pos.
__device__ __forceinline__ void wide_claim(int64_t* slots, int64_t capacity, long long key, long long pos) {
  const int64_t mask = capacity - 1;
  for (int64_t slot = (int64_t)(table_mix64((uint64_t)key) & (uint64_t)mask);; slot = (slot + 1) & mask) {
    const long long prev = (long long)atomicCAS(reinterpret_cast<unsigned long long*>(slots + 2 * slot),
                                                (unsigned long long)kEmptyKey, (unsigned long long)key);
    if (prev == kEmptyKey || prev == key) {
      atomicMin(reinterpret_cast<long long*>(slots + 2 * slot + 1), pos);
      return;
    }
  }
}

// A probe = the table words fetched for one key.
//   narrow: one 32-byte sector = a 4-way bucket of packed (position+1, key) words,
//           fetched with two 128-bit read-only loads of the same sector (L1-cacheable: the
//           table is immutable).
//   wide:   one {key, position} slot (128-bit load), linear probing.
template <bool NARROW> struct LProbe;
template <> struct LProbe<true>  { int64_t b; unsigned long long w[4]; };
template <> struct LProbe<false> { int64_t b; long long k, v; };

template <bool NARROW>
__device__ __forceinline__ void lookup_load(const Lookup& t, int64_t b, LProbe<NARROW>& p) {
  p.b = b;
  if constexpr (NARROW) {
    const unsigned long long* a = reinterpret_cast<const unsigned long long*>(t.slots) + 4 * b;
    const uint64_t pol = l2_evict_last();
    asm volatile("ld.global.nc.L2::cache_hint.v2.u64 {%0,%1}, [%2], %3;"
                 : "=l"(p.w[0]), "=l"(p.w[1]) : "l"(a), "l"(pol));
    asm volatile("ld.global.nc.L2::cache_hint.v2.u64 {%0,%1}, [%2], %3;"
                 : "=l"(p.w[2]), "=l"(p.w[3]) : "l"(a + 2), "l"(pol));
  } else {
    const longlong2 kv = __ldg(reinterpret_cast<const longlong2*>(t.slots + 2 * b));
    p.k = kv.x; p.v = kv.y;
  }
}

template <bool NARROW>
__device__ __forceinline__ int64_t lookup_home(const Lookup& t, int64_t key) {
  if constexpr (NARROW)
    return (int64_t)((uint64_t)table_mix32((uint32_t)(int32_t)key) & (uint64_t)((t.capacity >> 2) - 1));
  return (int64_t)(table_mix64((uint64_t)key) & (uint64_t)(t.capacity - 1));
}

// position of `key` or -1, starting from a prefetched first probe.  Single exit: the
// lanes of a warp iterate together; with 4-way buckets almost every key resolves in
// the first iteration.
template <bool NARROW>
__device__ __forceinline__ int64_t lookup_resolve(const Lookup& t, int64_t key, LProbe<NARROW> p) {
  if (!NARROW && key == kEmptyKey) return t.min_key_pos;
  const int64_t mask = NARROW ? (t.capacity >> 2) - 1 : t.capacity - 1;
  int64_t pos = -1;
  bool done = false;
#pragma unroll 1
  while (!done) {
    if constexpr (NARROW) {
      bool has_empty = false;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const unsigned long long w = p.w[j];
        has_empty = has_empty || (w == 0ull);
        if (w != 0ull && (unsigned)w == (unsigned)key) pos = (int64_t)(w >> 32) - 1;
      }
      done = (pos >= 0) || has_empty;       // a bucket with a free slot ends the probe sequence
    } else {
      if (p.k == key) { pos = p.v; done = true; }
      else if (p.k == kEmptyKey) done = true;
    }
    if (!done) lookup_load<NARROW>(t, NARROW ? narrow_next(p.b, mask + 1) : ((p.b + 1) & mask), p);
  }
  return pos;
}

__device__ __forceinline__ int64_t lookup_find(const Lookup& t, int64_t key) {
  if (t.narrow) {
    if (key < (int64_t)INT32_MIN || key > (int64_t)INT32_MAX) return -1;
    LProbe<true> p;
    lookup_load<true>(t, lookup_home<true>(t, key), p);
    return lookup_resolve<true>(t, key, p);
  }
  LProbe<false> p;
  lookup_load<false>(t, lookup_home<false>(t, key), p);
  return lookup_resolve<false>(t, key, p);
}

}  // namespace nvtb
