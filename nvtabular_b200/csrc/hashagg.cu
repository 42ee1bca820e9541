// hashagg.cu — K3: device hash aggregation  groupby(key, dropna=False).agg(...)
//
// The group-by handle's hash table: its layouts, inserts, merges of pre-aggregated rows, the
// overflow arena and settle, export, and the hand-off of high-cardinality int32 columns to
// the sorted accumulator (sortacc.cu).
//
// Replaces the reference's per-partition cuDF groupby + concat/groupby tree
// (nvtabular/ops/categorify.py:955-1137, graph built at :1344-1540) with ONE
// resident open-addressing table per column group that every batch is folded
// into.  Design (GPU-first, not a translation of cuDF's groupby, which sizes a
// fresh 2N-slot table per partition):
//
//   * two slot layouts (see `struct Table`): wide {int64 key, int64 size} (+ optional
//     per-slot payload {sum, sumsq, min, max} per cont column) and narrow 8-byte packed
//     slots in 4-way sector buckets for int32 keys without payload.
//   * int32 keys without payload (every Categorify column of the Criteo workload) take
//     the path of fold_i32.cuh: rows are absorbed in SHARED memory (find-or-claim tables
//     of 110-224 KB per CTA), after a one-pass hash partition of the column when the
//     expected number of distinct keys exceeds what one table holds; the global table
//     only sees one (key, count) pair per distinct key per CTA / partition.
//   * other keys: ONE launch per (column, batch); insert_keys_kernel streams the key
//     column with 256-bit loads and first folds rows into a per-CTA shared-memory table
//     (64 KB) - a CTA whose first tile shows < 25 % reuse bypasses it; insert_agg_kernel
//     (payload) updates the global table row by row.
//   * the table is sized from a CARDINALITY ESTIMATE (exact distinct count of
//     the first 2^20 rows, inverted through U = K(1 - exp(-s/K)), or the
//     caller's hint), not from the worst case.  Correctness never depends on
//     the estimate: a probe gives up after 128 buckets and the refused
//     (key, count) pair goes to an overflow ARENA sized for the launch.  The
//     next call on the handle ("settle") reads the counters back, grows the
//     table if the arena is non-empty and merges the arena into it.
//   * the null key (dropna=False) and the one key equal to the EMPTY sentinel
//     (INT64_MIN) live in two "special" groups outside the table.
//
// Throughput bound: the shared-memory pipe and L2 atomics / random 32-B sector traffic,
// not the HBM stream; see DESIGN.md "K3 design and its real roofline".
#include <algorithm>
#include <mutex>
#include <new>

#include "hashagg.cuh"

namespace nvtb {

constexpr int kSmemProbes = 4;
constexpr int kMaxProbes = 128;    // global probe limit before a pair is refused
constexpr int64_t kSampleRows = (int64_t)1 << 20;
constexpr int64_t kMinCapacity = 1 << 16;
constexpr int kInsertCtasPerSm = 3;

// min/max are kept as order-preserving int64 images of the double so that the
// native 64-bit atomicMin/atomicMax can be used.
__host__ __device__ __forceinline__ int64_t enc_ordered(double x) {
#ifdef __CUDA_ARCH__
  int64_t b = __double_as_longlong(x);
#else
  int64_t b; memcpy(&b, &x, 8);
#endif
  return b >= 0 ? b : (b ^ 0x7FFFFFFFFFFFFFFFll);
}
__host__ __device__ __forceinline__ double dec_ordered(int64_t e) {
  int64_t b = e >= 0 ? e : (e ^ 0x7FFFFFFFFFFFFFFFll);
#ifdef __CUDA_ARCH__
  return __longlong_as_double(b);
#else
  double x; memcpy(&x, &b, 8); return x;
#endif
}
// INT64_MAX / INT64_MIN decode to NaN: "no value seen" == pandas NaN min/max.
constexpr int64_t kMinInit = INT64_MAX;
constexpr int64_t kMaxInit = INT64_MIN;

// Two slot layouts:
//   wide   (16 B)  {int64 key, int64 size}; empty key = INT64_MIN
//   narrow ( 8 B)  (uint32 size << 32) | uint32 key; empty = 0 (a live slot has
//                  size >= 1).  Used for int32 keys without payload while the
//                  handle has seen < 2^32 rows: half the footprint (tables of a
//                  few million keys stay L2-resident), a new key costs ONE
//                  64-bit CAS that also deposits the count, a known key one
//                  32-bit RED.
struct Table {
  int64_t* slots;   // wide: [2*capacity]; narrow: [capacity] packed words
  double* vals;     // [capacity * 4 * n_agg] or nullptr (wide only)
  int64_t capacity; // power of two
  int n_agg;
  int narrow;
};

struct Arena {
  int64_t* keys;
  int64_t* sizes;
  double* vals;      // [cap * 4 * n_agg] or nullptr
  int64_t cap;
  int slot;          // index in the shared arena pool, -1 = private allocation
};

}  // namespace nvtb

struct nvtb_hashagg {
  nvtb::Table t;
  nvtb::Counters* ctr;       // device
  double* special_vals;      // device [2][4*n_agg]
  nvtb::Counters* mailbox;   // pinned host
  cudaEvent_t ev;
  bool pending;              // a launch whose counters have not been read back
  nvtb::Arena arena;         // arena of the pending launch
  cudaStream_t pending_stream;
  int64_t u_known;           // distinct keys at the last settle
  int64_t rows_total;        // rows folded in so far
  double k_est;              // cardinality estimate (0 = none yet)
  double predicted;          // distinct keys expected after the batch being prepared
  int64_t hint;
  int n_agg;
  bool mailbox_valid;        // mailbox == device counters (no launch / host edit since the readback)
  nvtb::SortedAcc* acc;      // set once the handle has become a sorted accumulator (sortacc.cu); t is then unused
};

namespace nvtb {

__device__ __forceinline__ void vals_combine(double* __restrict__ dst,
                                             double sum, double sumsq,
                                             double mn, double mx) {
  atomicAdd(dst + 0, sum);
  atomicAdd(dst + 1, sumsq);
  if (mn == mn) atomicMin(reinterpret_cast<long long*>(dst + 2), (long long)enc_ordered(mn));
  if (mx == mx) atomicMax(reinterpret_cast<long long*>(dst + 3), (long long)enc_ordered(mx));
}

// append one refused pair (rare path: a plain atomic, safe under any divergence)
__device__ __forceinline__ int64_t arena_claim(Counters* ctr) {
  return (int64_t)atomicAdd(&ctr->ovf_count, 1ull);
}

// A probe = the table words fetched for one key.
//   narrow: one 32-byte SECTOR = a 4-way bucket of packed slots, fetched with two
//           back-to-back 128-bit loads of that sector.  A key displaced by collisions is
//           still found on the inlined fast path unless its bucket holds > 4 keys; with one slot per
//           probe ~load% of ALL rows took the divergent out-of-line path.
//   wide:   one 16-byte slot (key word only), linear probing.
template <bool NARROW> struct Probe;
template <> struct Probe<true>  { int64_t b; unsigned long long w[4]; };
template <> struct Probe<false> { int64_t b; unsigned long long w[1]; };

template <bool NARROW>
__device__ __forceinline__ void probe_load(const Table& t, int64_t b, Probe<NARROW>& p) {
  p.b = b;
  if constexpr (NARROW) {
    const unsigned long long* a = reinterpret_cast<const unsigned long long*>(t.slots) + 4 * b;
    const uint64_t pol = l2_evict_last();
    asm volatile("ld.global.cg.L2::cache_hint.v2.u64 {%0,%1}, [%2], %3;"
                 : "=l"(p.w[0]), "=l"(p.w[1]) : "l"(a), "l"(pol));
    asm volatile("ld.global.cg.L2::cache_hint.v2.u64 {%0,%1}, [%2], %3;"
                 : "=l"(p.w[2]), "=l"(p.w[3]) : "l"(a + 2), "l"(pol));
  } else {
    p.w[0] = __ldcg(reinterpret_cast<const unsigned long long*>(t.slots) + 2 * b);
  }
}

template <bool NARROW>
__device__ __forceinline__ int64_t probe_home(const Table& t, int64_t key) {
  if constexpr (NARROW)   // int32 keys: 32-bit mixer, low bits pick the bucket
    return (int64_t)((uint64_t)table_mix32((uint32_t)(int32_t)key) & (uint64_t)((t.capacity >> 2) - 1));
  return (int64_t)(table_mix64((uint64_t)key) & (uint64_t)(t.capacity - 1));
}

template <bool NARROW>
__device__ __forceinline__ void probe_first(const Table& t, int64_t key, Probe<NARROW>& p) {
  probe_load<NARROW>(t, probe_home<NARROW>(t, key), p);
}

// Everything that is not "the key sits in the prefetched bucket": claim an empty slot
// (64-bit CAS; on the narrow layout the CAS also deposits the count), walk to the next
// bucket, give up after kMaxProbes buckets (-> -1, the pair is refused).  ONE out-of-line
// copy keeps the 16-row-unrolled kernel small enough for the instruction cache.
// There is no load-factor guard: a table that is too small simply fills up, probes start
// failing, refused pairs go to the arena and settle() regrows the table.
template <bool NARROW>
__device__ __noinline__ int64_t upsert_slow(const Table& t, int64_t key, int64_t add,
                                            Probe<NARROW> p, unsigned& n_new) {
  unsigned long long* base = reinterpret_cast<unsigned long long*>(t.slots);
  const int64_t mask = NARROW ? (t.capacity >> 2) - 1 : t.capacity - 1;
  int64_t result = -1;
  bool done = false;
#pragma unroll 1
  for (int probe = 0; probe < kMaxProbes && !done; ++probe) {
    if constexpr (NARROW) {
      const unsigned long long want =
          ((unsigned long long)(unsigned)add << 32) | (unsigned long long)(unsigned)key;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (!done) {
          unsigned long long cur = p.w[j];
          if (cur == 0ull) {
            cur = atomicCAS(base + 4 * p.b + j, 0ull, want);
            if (cur == 0ull) { ++n_new; result = 4 * p.b + j; done = true; }   // count deposited
          }
          if (!done && (unsigned)cur == (unsigned)key) {        // cur != 0 here
            atomicAdd(reinterpret_cast<unsigned*>(base + 4 * p.b + j) + 1, (unsigned)add);
            result = 4 * p.b + j; done = true;
          }
        }
      }
    } else {
      bool match = ((long long)p.w[0] == key);
      if ((long long)p.w[0] == kEmptyKey) {
        const unsigned long long prev = atomicCAS(base + 2 * p.b, (unsigned long long)kEmptyKey,
                                                  (unsigned long long)key);
        if ((long long)prev == kEmptyKey) { ++n_new; match = true; }
        else match = ((long long)prev == key);
      }
      if (match) {
        atomicAdd(base + 2 * p.b + 1, (unsigned long long)add);
        result = p.b; done = true;
      }
    }
    if (!done) probe_load<NARROW>(t, (p.b + 1) & mask, p);
  }
  return result;
}

// Fold (key, add) into the table starting from a PREFETCHED first probe: callers issue
// the first-probe loads of several keys back to back and only then resolve them, so a
// thread keeps several table sectors in flight.  Returns the slot, or -1 (refused).
template <bool NARROW>
__device__ __forceinline__ int64_t upsert_add(const Table& t, int64_t key, int64_t add,
                                              const Probe<NARROW>& p, unsigned& n_new) {
  unsigned long long* base = reinterpret_cast<unsigned long long*>(t.slots);
  if constexpr (NARROW) {
    int hit = -1;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (p.w[j] != 0ull && (unsigned)p.w[j] == (unsigned)key) hit = j;
    if (hit >= 0) {
      atomicAdd(reinterpret_cast<unsigned*>(base + 4 * p.b + hit) + 1, (unsigned)add);
      return 4 * p.b + hit;
    }
  } else {
    if ((long long)p.w[0] == key) {
      atomicAdd(base + 2 * p.b + 1, (unsigned long long)add);
      return p.b;
    }
  }
  return upsert_slow<NARROW>(t, key, add, p, n_new);
}

// one-key convenience form (cold paths: merge, scalar tails)
template <bool NARROW>
__device__ __forceinline__ int64_t upsert_one(const Table& t, int64_t key, int64_t add, unsigned& n_new) {
  Probe<NARROW> p;
  probe_first<NARROW>(t, key, p);
  return upsert_add<NARROW>(t, key, add, p, n_new);
}

template <bool NARROW>
__device__ __forceinline__ void upsert_or_spill(const Table& t, const Arena& a, Counters* ctr,
                                                int64_t key, int64_t add, const Probe<NARROW>& p,
                                                unsigned& n_new) {
  if (upsert_add<NARROW>(t, key, add, p, n_new) < 0) {
    const int64_t o = arena_claim(ctr);
    if (o < a.cap) { a.keys[o] = key; a.sizes[o] = add; }
  }
}

__global__ void table_init_kernel(Table t) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
       s < t.capacity; s += stride) {
    if (t.narrow) { t.slots[s] = 0; continue; }
    t.slots[2 * s] = kEmptyKey;
    t.slots[2 * s + 1] = 0;
    for (int j = 0; j < t.n_agg; ++j) {
      double* v = t.vals + (s * t.n_agg + j) * 4;
      v[0] = 0.0; v[1] = 0.0;
      reinterpret_cast<int64_t*>(v)[2] = kMinInit;
      reinterpret_cast<int64_t*>(v)[3] = kMaxInit;
    }
  }
}

__global__ void arm_launch_kernel(Counters* ctr) {
  ctr->ovf_count = 0ull;
}

__global__ void special_init_kernel(Counters* ctr, double* special_vals, int n_agg) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    ctr->n_unique = 0; ctr->size[0] = 0; ctr->size[1] = 0; ctr->ovf_count = 0; ctr->max_count = 0;
    for (int g = 0; g < 2; ++g)
      for (int j = 0; j < n_agg; ++j) {
        double* v = special_vals + (g * n_agg + j) * 4;
        v[0] = 0.0; v[1] = 0.0;
        reinterpret_cast<int64_t*>(v)[2] = kMinInit;
        reinterpret_cast<int64_t*>(v)[3] = kMaxInit;
      }
  }
}

}  // namespace nvtb
#include "partition.cuh"
#include "fold_i32.cuh"
namespace nvtb {

// ---------------------------------------------------------------------------
// insert, keys only (Categorify)
// ---------------------------------------------------------------------------
// Per-CTA shared-memory pre-aggregation table.
//   int32 keys: 8192 packed slots (count << 32 | key; 0 = empty), 64 KB
//   int64 keys: 4096 slots of {int64 key, uint32 count}, 48 KB
template <typename KeyT> struct SmemAgg;

template <> struct SmemAgg<int32_t> {
  // 4096 two-way buckets: one 128-bit shared load fetches both candidate slots of a key,
  // so a key displaced by a collision is still found on the inlined fast path (with
  // one-slot-per-probe linear probing ~load% of ALL rows took the divergent slow path).
  static constexpr int kBuckets = 4096;
  static constexpr int kSlots = 2 * kBuckets;
  static constexpr int kBytes = kSlots * 8;
  unsigned long long* w;
  __device__ __forceinline__ explicit SmemAgg(unsigned char* raw) : w(reinterpret_cast<unsigned long long*>(raw)) {}
  __device__ __forceinline__ void clear() {
    for (int s = threadIdx.x; s < kSlots; s += kThreads) w[s] = 0ull;
  }
  // claim one of the two slots of bucket b for `key` (or find it there); false = bucket full
  static __device__ __noinline__ bool fold_slow(unsigned long long* w, unsigned key, unsigned b) {
    bool done = false;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      if (!done) {
        unsigned long long* p = w + 2 * b + j;
        unsigned long long cur = *reinterpret_cast<volatile unsigned long long*>(p);
        if (cur == 0ull) {
          cur = atomicCAS(p, 0ull, (1ull << 32) | (unsigned long long)key);
          if (cur == 0ull) done = true;                          // claimed with count 1
        }
        if (!done && cur != 0ull && (unsigned)cur == key) {
          atomicAdd(reinterpret_cast<unsigned*>(p) + 1, 1u);
          done = true;
        }
      }
    }
    return done;
  }
  // fold one key; true = absorbed.  `hits` counts keys that were already present.
  __device__ __forceinline__ bool fold(long long k, unsigned& hits) {
    const unsigned key = (unsigned)(int)k;
    const unsigned b = (table_mix32(key) >> 20) & (kBuckets - 1);   // top bits; the global bucket uses the low bits
    unsigned long long x, y;
    const unsigned addr = (unsigned)__cvta_generic_to_shared(w + 2 * b);
    asm volatile("ld.volatile.shared.v2.u64 {%0, %1}, [%2];" : "=l"(x), "=l"(y) : "r"(addr));
    const bool mx = (x != 0ull) && ((unsigned)x == key);
    const bool my = (y != 0ull) && ((unsigned)y == key);
    if (mx || my) {
      atomicAdd(reinterpret_cast<unsigned*>(w + 2 * b + (mx ? 0 : 1)) + 1, 1u);
      hits++;
      return true;
    }
    return fold_slow(w, key, b);
  }
  __device__ __forceinline__ bool get(int s, long long* key, unsigned* cnt) const {
    const unsigned long long cur = w[s];
    *key = (long long)(int)(unsigned)cur;
    *cnt = (unsigned)(cur >> 32);
    return cur != 0ull;
  }
};

template <> struct SmemAgg<int64_t> {
  static constexpr int kSlots = 4096;
  static constexpr int kBytes = kSlots * 12;
  long long* keys;
  unsigned* cnt;
  __device__ __forceinline__ explicit SmemAgg(unsigned char* raw)
      : keys(reinterpret_cast<long long*>(raw)), cnt(reinterpret_cast<unsigned*>(raw + sizeof(long long) * kSlots)) {}
  __device__ __forceinline__ void clear() {
    for (int s = threadIdx.x; s < kSlots; s += kThreads) { keys[s] = kEmptyKey; cnt[s] = 0u; }
  }
  static __device__ __noinline__ bool fold_slow(long long* keys, unsigned* cnt, long long k, unsigned s) {
    bool done = false;
#pragma unroll 1
    for (int p = 0; p < kSmemProbes && !done; ++p) {
      long long cur = *reinterpret_cast<volatile long long*>(&keys[s]);
      if (cur == kEmptyKey)
        cur = (long long)atomicCAS(reinterpret_cast<unsigned long long*>(&keys[s]),
                                   (unsigned long long)kEmptyKey, (unsigned long long)k);
      if (cur == kEmptyKey || cur == k) {
        atomicAdd(&cnt[s], 1u);
        done = true;
      }
      s = (s + 1) & (kSlots - 1);
    }
    return done;
  }
  __device__ __forceinline__ bool fold(long long k, unsigned& hits) {
    const unsigned s = (unsigned)(table_mix64((uint64_t)k) >> 40) & (kSlots - 1);
    if (*reinterpret_cast<volatile long long*>(&keys[s]) == k) {
      atomicAdd(&cnt[s], 1u);
      hits++;
      return true;
    }
    return fold_slow(keys, cnt, k, s);
  }
  __device__ __forceinline__ bool get(int s, long long* key, unsigned* c) const {
    *key = keys[s];
    *c = cnt[s];
    return keys[s] != kEmptyKey;
  }
};

template <typename KeyT, bool NARROW>
__global__ void __launch_bounds__(kThreads, 3)
insert_keys_kernel(const KeyT* __restrict__ keys,
                   const uint8_t* __restrict__ mask, int64_t n, Table t,
                   Counters* ctr, Arena arena) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SmemAgg<KeyT> sm(smem_raw);
  __shared__ unsigned long long s_null, s_min;
  __shared__ unsigned int s_hits, s_rows, s_new;
  __shared__ int s_bypass;
  sm.clear();
  if (threadIdx.x == 0) { s_null = 0ull; s_min = 0ull; s_hits = 0u; s_rows = 0u; s_new = 0u; s_bypass = 0; }
  __syncthreads();

  unsigned int n_null = 0, n_min = 0, n_new = 0;
  bool bypass = false;
  const bool aligned = is_aligned32(keys);

  // 8 rows of one lane: (1) shared-memory fold, (2) first-probe loads of every key
  // that still has to reach the global table, issued back to back, (3) resolve
  auto fold8 = [&](const KeyT (&v)[kRows], unsigned m, unsigned& hits, unsigned& rows) {
    unsigned pend = 0;
#pragma unroll
    for (int k = 0; k < kRows; ++k) {
      const bool valid = (m >> k) & 1u;
      const long long key = (long long)v[k];
      const bool is_min = valid && sizeof(KeyT) == 8 && key == kEmptyKey;
      n_null += valid ? 0u : 1u;
      n_min += is_min ? 1u : 0u;
      if (valid && !is_min) {
        rows++;
        if (bypass || !sm.fold(key, hits)) pend |= 1u << k;
      }
    }
    // global phase in two halves of 4 keys: 4 sector loads in flight per thread
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const unsigned hp = (pend >> (4 * half)) & 0xFu;
      if (hp != 0) {
        Probe<NARROW> pr[4];
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if ((hp >> k) & 1u) probe_first<NARROW>(t, (long long)v[4 * half + k], pr[k]);
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if ((hp >> k) & 1u)
            upsert_or_spill<NARROW>(t, arena, ctr, (long long)v[4 * half + k], 1, pr[k], n_new);
      }
    }
  };

  const int64_t n_tiles = (n + kTile - 1) / kTile;
  bool first = true;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t base = tile * kTile;
    unsigned hits = 0, rows = 0;
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
      for (int g = 0; g < kGroups; ++g) fold8(v[g], m[g], hits, rows);
    } else {
      const int64_t end = (base + kTile < n) ? base + kTile : n;
      for (int64_t i = base + threadIdx.x; i < end; i += kThreads) {
        if (!valid1(mask, i)) { n_null++; continue; }
        const long long key = (long long)keys[i];
        if (sizeof(KeyT) == 8 && key == kEmptyKey) { n_min++; continue; }
        rows++;
        if (!bypass && sm.fold(key, hits)) continue;
        Probe<NARROW> pr;
        probe_first<NARROW>(t, key, pr);
        upsert_or_spill<NARROW>(t, arena, ctr, key, 1, pr, n_new);
      }
    }
    if (first) {
      // after its first tile the CTA decides whether shared-memory folding pays:
      // < 25 % of the rows met an already-present key  =>  go straight to global
      first = false;
      if (hits) atomicAdd(&s_hits, hits);
      if (rows) atomicAdd(&s_rows, rows);
      __syncthreads();
      if (threadIdx.x == 0) s_bypass = (s_hits * 4u < s_rows) ? 1 : 0;
      __syncthreads();
      bypass = (s_bypass != 0);
    }
  }

  if (n_null) atomicAdd(&s_null, (unsigned long long)n_null);
  if (n_min) atomicAdd(&s_min, (unsigned long long)n_min);
  __syncthreads();
  // flush the CTA-local aggregates: one global update per distinct key per CTA
  for (int s0 = 0; s0 < SmemAgg<KeyT>::kSlots; s0 += kThreads * 4) {
    long long k[4];
    unsigned c[4];
    bool live[4];
    Probe<NARROW> pr[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      live[j] = sm.get(s0 + j * kThreads + threadIdx.x, &k[j], &c[j]);
      if (live[j]) probe_first<NARROW>(t, k[j], pr[j]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (live[j]) upsert_or_spill<NARROW>(t, arena, ctr, k[j], (int64_t)c[j], pr[j], n_new);
  }
  if (n_new) atomicAdd(&s_new, n_new);
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_null) atomicAdd(&ctr->size[0], s_null);
    if (s_min) atomicAdd(&ctr->size[1], s_min);
    if (s_new) atomicAdd(&ctr->n_unique, (unsigned long long)s_new);
  }
}

// ---------------------------------------------------------------------------
// insert with continuous payload (JoinGroupby / TargetEncoding)
// ---------------------------------------------------------------------------
constexpr int kMaxAgg = 8;
struct AggCols {
  const void* data[kMaxAgg];
  const uint8_t* mask[kMaxAgg];
  int32_t dtype[kMaxAgg];
};

__device__ __forceinline__ bool load_agg(const AggCols& a, int j, int64_t i,
                                         double* out) {
  if (!valid1(a.mask[j], i)) return false;
  double v;
  switch (a.dtype[j]) {
    case NVTB_I32: v = (double)((const int32_t*)a.data[j])[i]; break;
    case NVTB_I64: v = (double)((const int64_t*)a.data[j])[i]; break;
    case NVTB_F32: v = (double)((const float*)a.data[j])[i]; break;
    case NVTB_U8:  v = (double)((const uint8_t*)a.data[j])[i]; break;
    default:       v = ((const double*)a.data[j])[i]; break;
  }
  if (v != v) return false;  // NaN == null
  *out = v;
  return true;
}

template <typename KeyT>
__global__ void __launch_bounds__(kThreads)
insert_agg_kernel(const KeyT* __restrict__ keys,
                  const uint8_t* __restrict__ mask, AggCols agg, int64_t n,
                  Table t, Counters* ctr, double* special_vals, Arena arena) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned n_new = 0;
  const double nan = __longlong_as_double(0x7FF8000000000000ll);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += stride) {
    const bool valid = valid1(mask, i);
    const long long k = valid ? (long long)keys[i] : 0;
    double* vdst = nullptr;
    if (!valid) {
      atomicAdd(&ctr->size[0], 1ull);
      vdst = special_vals;
    } else if (sizeof(KeyT) == 8 && k == kEmptyKey) {
      atomicAdd(&ctr->size[1], 1ull);
      vdst = special_vals + (int64_t)t.n_agg * 4;
    } else {
      const int64_t slot = upsert_one<false>(t, k, 1, n_new);
      if (slot >= 0) {
        vdst = t.vals + slot * t.n_agg * 4;
      } else {
        const int64_t o = arena_claim(ctr);
        if (o < arena.cap) {
          arena.keys[o] = k;
          arena.sizes[o] = 1;
          for (int j = 0; j < t.n_agg; ++j) {
            double v;
            double* w = arena.vals + (o * t.n_agg + j) * 4;
            if (load_agg(agg, j, i, &v)) { w[0] = v; w[1] = v * v; w[2] = v; w[3] = v; }
            else { w[0] = 0.0; w[1] = 0.0; w[2] = nan; w[3] = nan; }
          }
        }
        continue;
      }
    }
    for (int j = 0; j < t.n_agg; ++j) {
      double v;
      if (load_agg(agg, j, i, &v)) vals_combine(vdst + j * 4, v, v * v, v, v);
    }
  }
  if (n_new) atomicAdd(&ctr->n_unique, (unsigned long long)n_new);
}

// merge pre-aggregated rows (other GPUs' partials, or a drained arena)
template <bool NARROW>
__global__ void __launch_bounds__(kThreads)
merge_kernel(const int64_t* __restrict__ keys, const int64_t* __restrict__ sizes,
             const double* __restrict__ vals, int64_t n, Table t, Counters* ctr,
             double* special_vals, Arena arena) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned n_new = 0;
  // four rows per thread per step: their first probes are issued back to back
  for (int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < n; i0 += 4 * stride) {
    long long k[4];
    bool live[4];
    Probe<NARROW> pr[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t i = i0 + j * stride;
      live[j] = i < n;
      k[j] = live[j] ? keys[i] : 0;
      if (live[j] && (NARROW || k[j] != kEmptyKey)) probe_first<NARROW>(t, k[j], pr[j]);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (!live[j]) continue;
      const int64_t i = i0 + j * stride;
      double* vdst;
      if (!NARROW && k[j] == kEmptyKey) {
        atomicAdd(&ctr->size[1], (unsigned long long)sizes[i]);
        vdst = special_vals + (int64_t)t.n_agg * 4;
      } else {
        const int64_t slot = upsert_add<NARROW>(t, k[j], sizes[i], pr[j], n_new);
        if (slot < 0) {
          const int64_t o = arena_claim(ctr);
          if (o < arena.cap) {
            arena.keys[o] = k[j];
            arena.sizes[o] = sizes[i];
            if (vals != nullptr)
              for (int q = 0; q < t.n_agg * 4; ++q)
                arena.vals[o * t.n_agg * 4 + q] = vals[i * t.n_agg * 4 + q];
          }
          continue;
        }
        vdst = NARROW ? nullptr : t.vals + slot * t.n_agg * 4;
      }
      if (vals != nullptr && vdst != nullptr)
        for (int q = 0; q < t.n_agg; ++q) {
          const double* v = vals + (i * t.n_agg + q) * 4;
          vals_combine(vdst + q * 4, v[0], v[1], v[2], v[3]);
        }
    }
  }
  if (n_new) atomicAdd(&ctr->n_unique, (unsigned long long)n_new);
}

// rehash an old table into a new one (larger, and/or narrow -> wide).  Keys are
// distinct: plain stores after the claim; n_unique is unchanged.  The new table is
// at most half full, so the probe loop terminates.
__global__ void __launch_bounds__(kThreads)
rehash_kernel(Table old_t, Table new_t) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t mask = new_t.capacity - 1;
  unsigned long long* nb = reinterpret_cast<unsigned long long*>(new_t.slots);
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
       s < old_t.capacity; s += stride) {
    long long k, sz;
    if (old_t.narrow) {
      const unsigned long long w = (unsigned long long)old_t.slots[s];
      if (w == 0ull) continue;
      k = (long long)(int)(unsigned)w;
      sz = (long long)(w >> 32);
    } else {
      k = old_t.slots[2 * s];
      if (k == kEmptyKey) continue;
      sz = old_t.slots[2 * s + 1];
    }
    int64_t slot = (int64_t)(table_mix64((uint64_t)k) & (uint64_t)mask);
    if (new_t.narrow) {
      const unsigned long long want = ((unsigned long long)sz << 32) | (unsigned long long)(unsigned)k;
      const int64_t bmask = (new_t.capacity >> 2) - 1;
      int64_t b = (int64_t)((uint64_t)table_mix32((uint32_t)(int32_t)k) & (uint64_t)bmask);
      bool placed = false;
      while (!placed) {
        for (int j = 0; j < 4 && !placed; ++j)
          placed = (atomicCAS(nb + 4 * b + j, 0ull, want) == 0ull);
        b = (b + 1) & bmask;
      }
    } else {
      while ((long long)atomicCAS(nb + 2 * slot, (unsigned long long)kEmptyKey, (unsigned long long)k) != kEmptyKey)
        slot = (slot + 1) & mask;
      new_t.slots[2 * slot + 1] = sz;
      if (!old_t.narrow)
        for (int j = 0; j < old_t.n_agg * 4; ++j)
          new_t.vals[slot * old_t.n_agg * 4 + j] = old_t.vals[s * old_t.n_agg * 4 + j];
    }
  }
}

constexpr int kExportPerThread = 4;

// A CTA compacts 1024 slots at a time and reserves its output range with ONE atomic: a
// per-warp atomicAdd on the single cursor (500 k same-address atomics for a 16 M-slot table)
// serialised at ~1 ns each and cost ~20x the time the scan itself needs.  `mine` = the lane's
// live slots; returns the lane's first output index.  The caller syncs before reusing
// s_warp / s_base.
__device__ __forceinline__ int64_t reserve_range(unsigned mine, unsigned* s_warp, unsigned long long* s_base,
                                                 unsigned long long* cursor) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned tot = 0;
    for (int w = 0; w < kThreads / 32; ++w) { const unsigned x = s_warp[w]; s_warp[w] = tot; tot += x; }
    *s_base = tot ? atomicAdd(cursor, (unsigned long long)tot) : 0ull;
  }
  __syncthreads();
  return (int64_t)*s_base + s_warp[warp] + (incl - mine);
}

// payload {sum, sumsq, min, max} of one group as stored (min / max order-encoded) -> doubles
__device__ __forceinline__ void decode_payload(const double* v, double* w) {
  w[0] = v[0]; w[1] = v[1];
  w[2] = dec_ordered(reinterpret_cast<const int64_t*>(v)[2]);
  w[3] = dec_ordered(reinterpret_cast<const int64_t*>(v)[3]);
}

// compaction: table -> dense (unordered) arrays
__global__ void __launch_bounds__(kThreads)
export_kernel(Table t, int64_t* __restrict__ keys_out,
              int64_t* __restrict__ sizes_out, double* __restrict__ vals_out,
              unsigned long long* cursor) {
  __shared__ unsigned s_warp[kThreads / 32];
  __shared__ unsigned long long s_base;
  constexpr int64_t kChunk = (int64_t)kThreads * kExportPerThread;
  // capacity is a power of two >= 65536: every chunk is full
  for (int64_t c0 = (int64_t)blockIdx.x * kChunk; c0 < t.capacity; c0 += (int64_t)gridDim.x * kChunk) {
    long long k[kExportPerThread], sz[kExportPerThread];
    unsigned live = 0;
#pragma unroll
    for (int j = 0; j < kExportPerThread; ++j) {
      const int64_t s = c0 + (int64_t)j * kThreads + threadIdx.x;
      sz[j] = 0;
      if (t.narrow) {
        const unsigned long long w = (unsigned long long)t.slots[s];
        if (w != 0ull) live |= 1u << j;
        k[j] = (long long)(int)(unsigned)w;
        sz[j] = (long long)(w >> 32);
      } else {
        k[j] = t.slots[2 * s];
        if (k[j] != kEmptyKey) { live |= 1u << j; sz[j] = t.slots[2 * s + 1]; }
      }
    }
    int64_t o = reserve_range(__popc(live), s_warp, &s_base, cursor);
#pragma unroll
    for (int j = 0; j < kExportPerThread; ++j) {
      if (!((live >> j) & 1u)) continue;
      keys_out[o] = k[j];
      if (sizes_out) sizes_out[o] = sz[j];
      if (vals_out) {
        const int64_t s = c0 + (int64_t)j * kThreads + threadIdx.x;
        for (int q = 0; q < t.n_agg; ++q)
          decode_payload(t.vals + (s * t.n_agg + q) * 4, vals_out + (o * t.n_agg + q) * 4);
      }
      ++o;
    }
    __syncthreads();     // s_warp / s_base are reused by the next chunk
  }
}

// narrow hash table -> packed pairs (unordered)
static __global__ void __launch_bounds__(kThreads)
table_to_pairs_kernel(Table t, uint64_t* __restrict__ out, unsigned long long* cursor,
                      unsigned long long* max_count) {
  __shared__ unsigned s_warp[kThreads / 32];
  __shared__ unsigned long long s_base;
  const int lane = threadIdx.x & 31;
  constexpr int64_t kChunk = (int64_t)kThreads * kExportPerThread;
  uint32_t mx = 0;
  for (int64_t c0 = (int64_t)blockIdx.x * kChunk; c0 < t.capacity; c0 += (int64_t)gridDim.x * kChunk) {
    unsigned long long w[kExportPerThread];
    unsigned live = 0;
#pragma unroll
    for (int j = 0; j < kExportPerThread; ++j) {
      w[j] = (unsigned long long)t.slots[c0 + (int64_t)j * kThreads + threadIdx.x];
      if (w[j] != 0ull) live |= 1u << j;
    }
    int64_t o = reserve_range(__popc(live), s_warp, &s_base, cursor);
#pragma unroll
    for (int j = 0; j < kExportPerThread; ++j) {
      if (!((live >> j) & 1u)) continue;
      const uint32_t key = (uint32_t)w[j], cnt = (uint32_t)(w[j] >> 32);
      out[o++] = ((uint64_t)(key ^ 0x80000000u) << 32) | cnt;
      mx = cnt > mx ? cnt : mx;
    }
    __syncthreads();
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { const uint32_t y = __shfl_down_sync(0xFFFFFFFFu, mx, o); mx = y > mx ? y : mx; }
  if (lane == 0 && mx) atomicMax(max_count, (unsigned long long)mx);
}

__global__ void decode_special_kernel(const double* special_vals, int n_agg,
                                      double* out) {
  const int i = threadIdx.x;
  if (i < 2 * n_agg) decode_payload(special_vals + i * 4, out + i * 4);
}

// ---------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------
static int table_alloc(Table* t, int64_t capacity, int n_agg, bool narrow, cudaStream_t st) {
  t->capacity = capacity;
  t->n_agg = n_agg;
  t->narrow = narrow ? 1 : 0;
  t->slots = nullptr;
  t->vals = nullptr;
  NVTB_CUDA_OK(cudaMallocAsync(&t->slots, sizeof(int64_t) * (narrow ? 1 : 2) * capacity, st));
  if (n_agg > 0)
    NVTB_CUDA_OK(cudaMallocAsync(&t->vals, sizeof(double) * 4 * n_agg * capacity, st));
  table_init_kernel<<<plain_grid(capacity), kThreads, 0, st>>>(*t);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

static int table_free(Table* t, cudaStream_t st) {
  if (t->slots) NVTB_CUDA_OK(cudaFreeAsync(t->slots, st));
  if (t->vals) NVTB_CUDA_OK(cudaFreeAsync(t->vals, st));
  t->slots = nullptr; t->vals = nullptr;
  return NVTB_OK;
}

static int64_t next_pow2(int64_t v) {
  int64_t p = kMinCapacity;
  while (p < v) p <<= 1;
  return p;
}

static int settle(nvtb_hashagg* h);

static int arena_alloc(Arena* a, int64_t cap, int n_agg, cudaStream_t st) {
  a->cap = cap; a->keys = nullptr; a->sizes = nullptr; a->vals = nullptr; a->slot = -1;
  if (cap <= 0) return NVTB_OK;
  NVTB_CUDA_OK(cudaMallocAsync(&a->keys, sizeof(int64_t) * cap, st));
  NVTB_CUDA_OK(cudaMallocAsync(&a->sizes, sizeof(int64_t) * cap, st));
  if (n_agg > 0) NVTB_CUDA_OK(cudaMallocAsync(&a->vals, sizeof(double) * 4 * n_agg * cap, st));
  return NVTB_OK;
}

// The arena of a launch must be able to hold one pair per input row, but is
// almost never touched.  Two pooled arenas (double buffering) serve every
// handle: acquiring a slot that still belongs to an unsettled launch settles
// that launch first, so at most two arenas exist however many columns are fitted.
struct ArenaSlot {
  int64_t* keys; int64_t* sizes; double* vals;
  int64_t cap_alloc; int64_t vals_alloc;
  nvtb_hashagg* owner;
  uint64_t stamp;
};
static ArenaSlot g_slots[2] = {};
static uint64_t g_stamp = 0;
static std::recursive_mutex g_arena_mu;

static int arena_acquire(nvtb_hashagg* h, Arena* out, int64_t cap, int n_agg) {
  std::lock_guard<std::recursive_mutex> lk(g_arena_mu);
  int pick = -1;
  for (int i = 0; i < 2; ++i)
    if (g_slots[i].owner == nullptr) { pick = i; break; }
  if (pick < 0) {
    pick = g_slots[0].stamp < g_slots[1].stamp ? 0 : 1;
    int rc = settle(g_slots[pick].owner);   // releases the slot
    if (rc) return rc;
  }
  ArenaSlot& sl = g_slots[pick];
  const int64_t need_vals = cap * 4 * n_agg;
  if (sl.cap_alloc < cap) {
    NVTB_CUDA_OK(cudaDeviceSynchronize());
    if (sl.keys) cudaFree(sl.keys);
    if (sl.sizes) cudaFree(sl.sizes);
    sl.keys = nullptr; sl.sizes = nullptr; sl.cap_alloc = 0;
    NVTB_CUDA_OK(cudaMalloc(&sl.keys, sizeof(int64_t) * cap));
    NVTB_CUDA_OK(cudaMalloc(&sl.sizes, sizeof(int64_t) * cap));
    sl.cap_alloc = cap;
  }
  if (sl.vals_alloc < need_vals) {
    NVTB_CUDA_OK(cudaDeviceSynchronize());
    if (sl.vals) cudaFree(sl.vals);
    sl.vals = nullptr; sl.vals_alloc = 0;
    NVTB_CUDA_OK(cudaMalloc(&sl.vals, sizeof(double) * need_vals));
    sl.vals_alloc = need_vals;
  }
  sl.owner = h;
  sl.stamp = ++g_stamp;
  out->keys = sl.keys; out->sizes = sl.sizes; out->vals = n_agg > 0 ? sl.vals : nullptr;
  out->cap = cap; out->slot = pick;
  return NVTB_OK;
}

static int arena_free(Arena* a, cudaStream_t st) {
  if (a->slot >= 0) {
    std::lock_guard<std::recursive_mutex> lk(g_arena_mu);
    g_slots[a->slot].owner = nullptr;
  } else {
    if (a->keys) NVTB_CUDA_OK(cudaFreeAsync(a->keys, st));
    if (a->sizes) NVTB_CUDA_OK(cudaFreeAsync(a->sizes, st));
    if (a->vals) NVTB_CUDA_OK(cudaFreeAsync(a->vals, st));
  }
  a->keys = nullptr; a->sizes = nullptr; a->vals = nullptr; a->cap = 0; a->slot = -1;
  return NVTB_OK;
}

// distinct keys expected among `rows` uniform draws from K values
static double expected_unique(double K, double rows) {
  if (K <= 0) return 0;
  return K * -std::expm1(-rows / K);
}

// invert U = K (1 - exp(-s/K)) for K (bisection); U >= 0.98 s  =>  "all distinct"
static double estimate_cardinality(double U, double s) {
  if (U <= 0) return 1.0;
  if (U >= 0.98 * s) return 1e18;
  double lo = U, hi = 1e18;
  for (int it = 0; it < 200; ++it) {
    const double mid = std::sqrt(lo * hi);
    if (expected_unique(mid, s) < U) lo = mid; else hi = mid;
    if (hi / lo < 1.0 + 1e-9) break;
  }
  return lo;
}

// move to a table of `new_cap` slots and/or the other layout (narrow -> wide only)
static int grow_to(nvtb_hashagg* h, int64_t new_cap, cudaStream_t st, bool force_wide = false) {
  const bool narrow = h->t.narrow && !force_wide;
  new_cap = std::max(new_cap, h->t.capacity);
  if (new_cap == h->t.capacity && narrow == (bool)h->t.narrow) return NVTB_OK;
  Table nt;
  int rc = table_alloc(&nt, new_cap, h->n_agg, narrow, st);
  if (rc) return rc;
  if (h->u_known > 0 || h->rows_total > 0) {
    rehash_kernel<<<plain_grid(h->t.capacity), kThreads, 0, st>>>(h->t, nt);
    NVTB_LAUNCH_OK();
  }
  rc = table_free(&h->t, st);
  if (rc) return rc;
  h->t = nt;
  return NVTB_OK;
}

static int launch_merge(nvtb_hashagg* h, const int64_t* keys, const int64_t* sizes,
                        const double* vals, int64_t n, const Arena& arena, cudaStream_t st) {
  const int grid = plain_grid(n);
  arm_launch_kernel<<<1, 1, 0, st>>>(h->ctr);
  NVTB_LAUNCH_OK();
  if (h->t.narrow)
    merge_kernel<true><<<grid, kThreads, 0, st>>>(keys, sizes, vals, n, h->t, h->ctr, h->special_vals, arena);
  else
    merge_kernel<false><<<grid, kThreads, 0, st>>>(keys, sizes, vals, n, h->t, h->ctr, h->special_vals, arena);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

// wait for the pending launch, read its counters, and fold a non-empty arena
// back in after growing the table.  Leaves no pending state.
static int settle(nvtb_hashagg* h) {
  if (h == nullptr) return NVTB_OK;
  while (h->pending) {
    cudaStream_t st = h->pending_stream;
    NVTB_CUDA_OK(cudaEventSynchronize(h->ev));
    h->pending = false;
    h->mailbox_valid = true;
    const Counters c = *h->mailbox;
    h->u_known = (int64_t)c.n_unique;
    const int64_t ovf = (int64_t)std::min<unsigned long long>(c.ovf_count, (unsigned long long)h->arena.cap);
    Arena old = h->arena;
    h->arena = Arena{nullptr, nullptr, nullptr, 0, -1};
    if (ovf > 0) {
      // every refused pair may be a new key: size for all of them at load <= 0.25
      int rc = grow_to(h, next_pow2(4 * (h->u_known + ovf)), st);
      if (rc) return rc;
      // a pair that is still refused (128
      // probes) lands in a fresh private arena and is settled by the loop
      rc = arena_alloc(&h->arena, ovf, h->n_agg, st);
      if (rc) return rc;
      rc = launch_merge(h, old.keys, old.sizes, old.vals, ovf, h->arena, st);
      if (rc) return rc;
      NVTB_CUDA_OK(cudaMemcpyAsync(h->mailbox, h->ctr, sizeof(Counters), cudaMemcpyDeviceToHost, st));
      NVTB_CUDA_OK(cudaEventRecord(h->ev, st));
      h->pending = true;
      h->pending_stream = st;
    }
    int rc = arena_free(&old, st);
    if (rc) return rc;
  }
  if (h->rows_total > 0) {
    // draws = VALID rows: the null rows of the sample are not draws from the key distribution.
    // (Counting them made a column with 8 % nulls look 8 % "duplicated": a high-cardinality
    // column was estimated far below its key count, its first batch filled the table and took
    // the 128-bucket probe path.)
    int64_t draws = h->rows_total;
    if (h->mailbox_valid) draws -= (int64_t)h->mailbox->size[0];
    h->k_est = estimate_cardinality((double)std::max<int64_t>(h->u_known, 1), (double)std::max<int64_t>(draws, 1));
  }
  return NVTB_OK;
}

// after a launch: async readback of the counters
static int post(nvtb_hashagg* h, cudaStream_t st) {
  NVTB_CUDA_OK(cudaMemcpyAsync(h->mailbox, h->ctr, sizeof(Counters), cudaMemcpyDeviceToHost, st));
  NVTB_CUDA_OK(cudaEventRecord(h->ev, st));
  h->pending = true;
  h->mailbox_valid = false;
  h->pending_stream = st;
  return NVTB_OK;
}

// distinct keys expected in the table after `rows` more rows (-> h->predicted)
static void predict(nvtb_hashagg* h, int64_t rows) {
  double predicted;
  if (h->hint > 0) {
    predicted = (double)std::max<int64_t>(h->hint, h->u_known);
  } else if (h->k_est > 0) {
    predicted = expected_unique(h->k_est, (double)(h->rows_total + rows));
    predicted = std::max(predicted, (double)h->u_known);
  } else {
    predicted = (double)h->u_known + (double)rows;   // no information: worst case
  }
  predicted = std::min(predicted, (double)h->u_known + (double)rows);
  h->predicted = predicted;
}

// size the table for `rows` more rows: load <= 0.5 for the ESTIMATED distinct count
static int prepare(nvtb_hashagg* h, int64_t rows, cudaStream_t st) {
  predict(h, rows);
  const int64_t want = next_pow2((int64_t)(2.5 * h->predicted) + 1);
  return grow_to(h, want, st);
}

int SharedScratch::acquire(size_t need, size_t alloc, cudaStream_t st, void** out, bool* grown) {
  std::lock_guard<std::mutex> lk(mu);
  *grown = false;
  if (bytes < need) {
    NVTB_CUDA_OK(cudaDeviceSynchronize());
    if (ptr) cudaFree(ptr);
    ptr = nullptr; bytes = 0;
    NVTB_CUDA_OK(cudaMalloc(&ptr, alloc));
    bytes = alloc;
    used = false;               // the device is idle: no earlier use to wait for
    *grown = true;
  }
  if (ev == nullptr) NVTB_CUDA_OK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  if (used && last != st) NVTB_CUDA_OK(cudaStreamWaitEvent(st, ev, 0));
  *out = ptr;
  return NVTB_OK;
}

int SharedScratch::release(cudaStream_t st) {
  std::lock_guard<std::mutex> lk(mu);
  NVTB_CUDA_OK(cudaEventRecord(ev, st));
  used = true;
  last = st;
  return NVTB_OK;
}

// partition buffer of the PARTS mode
static SharedScratch g_part;

// int32 keys, narrow table, no payload: shared-memory fold, hash-partitioned first when the
// expected number of distinct keys exceeds what one SM's shared memory holds (fold_i32.cuh)
static int launch_fold_i32(nvtb_hashagg* h, const int32_t* kp, const uint8_t* mp, int64_t m,
                           cudaStream_t st) {
  static bool attrs = false;
  constexpr int kDirectSmem = (int)(kFoldBucketsDirect * kFoldWays * kFoldSlotBytes);
  constexpr int kPartsSmem = (int)(kFoldBucketsParts * kFoldWays * kFoldSlotBytes);
  constexpr int kScatterSmemMax = kPartTile * 4 + 2 * 4 * kMaxParts;
  if (!attrs) {
    NVTB_CUDA_OK(cudaFuncSetAttribute(fold_i32_kernel<kFoldThreadsDirect, 1, false>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, kDirectSmem));
    NVTB_CUDA_OK(cudaFuncSetAttribute(fold_i32_kernel<kFoldThreadsParts, 2, true>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, kPartsSmem));
    NVTB_CUDA_OK(cudaFuncSetAttribute(part_scatter_kernel<PartHashTop>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, kScatterSmemMax));
    attrs = true;
  }
  const int sms = sm_count();
  const bool aligned = is_aligned32(kp);
  // distinct keys this batch is expected to show (the table may already hold some of them)
  const double fresh = std::min(h->predicted, (double)m);
  const bool parts = aligned && m >= ((int64_t)1 << 18) && m < (int64_t)0xFFFF0000ll &&
                     fresh > kFoldMaxLoad * (double)(kFoldWays * kFoldBucketsDirect);
  if (!parts) {
    constexpr int64_t kStep = (int64_t)kFoldThreadsDirect * 8;
    int64_t units = std::min<int64_t>(sms, (m + kStep - 1) / kStep);
    int64_t chunk = ((m + units - 1) / units + kStep - 1) / kStep * kStep;
    units = (m + chunk - 1) / chunk;
    fold_i32_kernel<kFoldThreadsDirect, 1, false><<<(int)units, kFoldThreadsDirect, kDirectSmem, st>>>(
        kp, mp, m, nullptr, nullptr, (int)units, chunk, 0, kFoldBucketsDirect, aligned ? 1 : 0,
        h->t, h->ctr, h->arena);
    NVTB_LAUNCH_OK();
    return NVTB_OK;
  }
  int lg = 9;
  while ((1 << lg) < kMinParts) ++lg;
  while ((1 << lg) < kMaxParts &&
         fresh / (double)(1 << lg) > kFoldMaxLoad * (double)(kFoldWays * kFoldBucketsParts)) ++lg;
  const int P = 1 << lg;
  const size_t need = sizeof(uint32_t) * 3 * kMaxParts + sizeof(int32_t) * (size_t)(m + 8 * (int64_t)kMaxParts);
  void* part = nullptr;
  bool grown = false;
  int rc = g_part.acquire(need, need, st, &part, &grown);
  if (rc) return rc;
  uint32_t* meta = reinterpret_cast<uint32_t*>(part);      // total[P] | starts[P] | cursor[P]
  int32_t* buf = reinterpret_cast<int32_t*>(meta + 3 * kMaxParts);
  NVTB_CUDA_OK(cudaMemsetAsync(meta, 0, sizeof(uint32_t) * P, st));
  const int64_t tiles = (m + kPartTile - 1) / kPartTile;
  part_hist_kernel<PartHashTop><<<(int)std::min<int64_t>(tiles, 3 * sms), kPartThreads, 4 * P, st>>>(
      kp, mp, m, PartHashTop{lg}, meta, h->ctr, 1);
  NVTB_LAUNCH_OK();
  part_scan_kernel<<<1, kPartThreads, 0, st>>>(meta, lg, meta + P, meta + 2 * P, 8u, nullptr);
  NVTB_LAUNCH_OK();
  part_scatter_kernel<PartHashTop><<<(int)std::min<int64_t>(tiles, 2 * sms), kPartThreads, kPartTile * 4 + 2 * 4 * P, st>>>(
      kp, mp, m, PartHashTop{lg}, meta + 2 * P, buf, 1);
  NVTB_LAUNCH_OK();
  fold_i32_kernel<kFoldThreadsParts, 2, true><<<std::min(P, 2 * sms), kFoldThreadsParts, kPartsSmem, st>>>(
      buf, nullptr, m + 8 * (int64_t)P, meta + P, meta + 2 * P, P, 0, lg, kFoldBucketsParts, 1,
      h->t, h->ctr, h->arena);
  NVTB_LAUNCH_OK();
  return g_part.release(st);
}


// ---------------------------------------------------------------------------------------
// sorted accumulator (sortacc.cu)
// ---------------------------------------------------------------------------------------
// expected distinct keys above which an int32 column leaves the hash table for the sorted
// accumulator: the table (2.5 slots x 8 B per key) then no longer stays in H100's 50 MB L2
static int64_t runs_min_keys() {
  const char* e = getenv("NVTB_RUNS_MIN_KEYS");      // read every time: tests flip it
  int64_t v = e ? atoll(e) : ((int64_t)3 << 20);
  return v < 1 ? 1 : v;
}

// hash table -> sorted accumulator (the handle must be settled and its table narrow): the
// u_known (key, count) pairs are exported into the accumulator, which sorts them by key
static int table_to_runs(nvtb_hashagg* h, cudaStream_t st) {
  const int64_t nu = h->u_known;
  uint64_t* pairs = nullptr;
  int rc = sortacc_create(&h->acc, nu, st, &pairs);
  if (rc) return rc;
  if (nu > 0) {
    unsigned long long* cursor = nullptr;
    NVTB_CUDA_OK(cudaMallocAsync(&cursor, sizeof(unsigned long long), st));
    NVTB_CUDA_OK(cudaMemsetAsync(cursor, 0, sizeof(unsigned long long), st));
    table_to_pairs_kernel<<<plain_grid(h->t.capacity / kExportPerThread), kThreads, 0, st>>>(
        h->t, pairs, cursor, &h->ctr->max_count);
    NVTB_LAUNCH_OK();
    NVTB_CUDA_OK(cudaFreeAsync(cursor, st));
    rc = sortacc_sort_pairs(h->acc, nu, st);
    if (rc) return rc;
  }
  // the table itself is no longer used: keep a minimal one so that the handle stays uniform
  rc = table_free(&h->t, st);
  if (rc) return rc;
  return table_alloc(&h->t, kMinCapacity, 0, true, st);
}

// group + merge the batches a sorted accumulator has staged (leaves a pending launch)
static int acc_flush(nvtb_hashagg* h, cudaStream_t st) {
  if (h->acc == nullptr || sortacc_staged_rows(h->acc) == 0) return NVTB_OK;
  int rc = settle(h);
  if (rc) return rc;
  rc = sortacc_flush(h->acc, h->u_known, h->ctr, st);
  if (rc) return rc;
  return post(h, st);
}

template <typename KeyT>
static int launch_insert(nvtb_hashagg* h, const KeyT* kp, const uint8_t* mp, const AggCols& ac,
                         int64_t m, cudaStream_t st) {
  int rc = arena_acquire(h, &h->arena, m, h->n_agg);
  if (rc) return rc;
  arm_launch_kernel<<<1, 1, 0, st>>>(h->ctr);
  NVTB_LAUNCH_OK();
  if (h->n_agg == 0 && sizeof(KeyT) == 4 && h->t.narrow) {
    rc = launch_fold_i32(h, reinterpret_cast<const int32_t*>(kp), mp, m, st);
    if (rc) return rc;
  } else if (h->n_agg == 0) {
    const int grid = scan_grid(m, kInsertCtasPerSm);
    constexpr int kSmemBytes = SmemAgg<KeyT>::kBytes;
    if (h->t.narrow) {
      NVTB_CUDA_OK(cudaFuncSetAttribute(insert_keys_kernel<KeyT, true>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
      insert_keys_kernel<KeyT, true><<<grid, kThreads, kSmemBytes, st>>>(kp, mp, m, h->t, h->ctr, h->arena);
    } else {
      NVTB_CUDA_OK(cudaFuncSetAttribute(insert_keys_kernel<KeyT, false>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
      insert_keys_kernel<KeyT, false><<<grid, kThreads, kSmemBytes, st>>>(kp, mp, m, h->t, h->ctr, h->arena);
    }
  } else {
    const int grid = plain_grid(m);
    insert_agg_kernel<KeyT><<<grid, kThreads, 0, st>>>(kp, mp, ac, m, h->t, h->ctr,
                                                       h->special_vals, h->arena);
  }
  NVTB_LAUNCH_OK();
  h->rows_total += m;
  return post(h, st);
}

int hashagg_sorted_view(nvtb_hashagg* h, const uint64_t** pairs, int64_t* n_unique, int64_t* null_size,
                        uint64_t* max_count, int* is_i32_table, cudaStream_t st) {
  int64_t nu = 0, ns = 0;
  int rc = nvtb_hashagg_size(h, &nu, &ns, (void*)st);
  if (rc) return rc;
  *n_unique = nu;
  *null_size = ns;
  *max_count = (uint64_t)h->mailbox->max_count;
  *pairs = h->acc ? sortacc_pairs(h->acc) : nullptr;
  *is_i32_table = (!h->acc && h->t.narrow) ? 1 : 0;
  return NVTB_OK;
}

}  // namespace nvtb

using namespace nvtb;

extern "C" {

int nvtb_hashagg_create(nvtb_hashagg_t** out, int n_agg, int64_t capacity_hint) {
  NVTB_REQUIRE(out != nullptr, "out is NULL");
  ensure_pool_configured();
  NVTB_REQUIRE(n_agg >= 0 && n_agg <= kMaxAgg, "n_agg must be in [0, 8]");
  nvtb_hashagg* h = new (std::nothrow) nvtb_hashagg();
  NVTB_REQUIRE(h != nullptr, "host allocation failed");
  memset(h, 0, sizeof(*h));
  h->n_agg = n_agg;
  h->hint = capacity_hint > 0 ? capacity_hint : 0;
  cudaStream_t st = 0;
  int rc = table_alloc(&h->t, next_pow2(std::max<int64_t>((int64_t)(2.5 * capacity_hint), kMinCapacity)), n_agg, false, st);
  if (rc) { delete h; return rc; }
  NVTB_CUDA_OK(cudaMalloc(&h->ctr, sizeof(Counters)));
  NVTB_CUDA_OK(cudaMalloc(&h->special_vals, sizeof(double) * 8 * (n_agg > 0 ? n_agg : 1)));
  special_init_kernel<<<1, 32, 0, st>>>(h->ctr, h->special_vals, n_agg);
  NVTB_LAUNCH_OK();
  NVTB_CUDA_OK(cudaMallocHost(&h->mailbox, sizeof(Counters)));
  NVTB_CUDA_OK(cudaEventCreateWithFlags(&h->ev, cudaEventDisableTiming));
  NVTB_CUDA_OK(cudaStreamSynchronize(st));
  *out = h;
  return NVTB_OK;
}

int nvtb_hashagg_reset(nvtb_hashagg_t* h, void* stream) {
  NVTB_REQUIRE(h != nullptr, "NULL handle");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = settle(h);
  if (rc) return rc;
  // the table keeps its capacity (and the estimate its value): a second fit over
  // similar data needs no growth and no sampling pass
  h->hint = std::max<int64_t>(h->hint, h->u_known);
  if (h->acc == nullptr) {      // a sorted accumulator is emptied by zeroing its counters below
    table_init_kernel<<<plain_grid(h->t.capacity), kThreads, 0, st>>>(h->t);
    NVTB_LAUNCH_OK();
  }
  special_init_kernel<<<1, 32, 0, st>>>(h->ctr, h->special_vals, h->n_agg);
  NVTB_LAUNCH_OK();
  if (h->acc) sortacc_reset(h->acc, h->rows_total);
  h->u_known = 0;
  h->rows_total = 0;
  h->mailbox_valid = false;
  return NVTB_OK;
}

int nvtb_hashagg_destroy(nvtb_hashagg_t* h) {
  if (h == nullptr) return NVTB_OK;
  settle(h);              // hands a pooled arena back
  cudaDeviceSynchronize();
  if (h->t.slots) cudaFree(h->t.slots);
  if (h->t.vals) cudaFree(h->t.vals);
  if (h->ctr) cudaFree(h->ctr);
  if (h->special_vals) cudaFree(h->special_vals);
  if (h->mailbox) cudaFreeHost(h->mailbox);
  if (h->ev) cudaEventDestroy(h->ev);
  if (h->acc) sortacc_destroy(h->acc);
  delete h;
  return NVTB_OK;
}

int nvtb_hashagg_insert(nvtb_hashagg_t* h, const nvtb_col_t* key,
                        const nvtb_col_t* agg_cols, int64_t n, void* stream) {
  NVTB_REQUIRE(h != nullptr && key != nullptr, "NULL handle/key");
  NVTB_REQUIRE(n >= 0, "n < 0");
  NVTB_REQUIRE(key->dtype == NVTB_I32 || key->dtype == NVTB_I64,
               "key dtype must be int32 or int64");
  NVTB_REQUIRE(h->n_agg == 0 || agg_cols != nullptr, "agg_cols is NULL");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(key->data != nullptr, "key data is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  AggCols ac;
  memset(&ac, 0, sizeof(ac));
  for (int j = 0; j < h->n_agg; ++j) {
    NVTB_REQUIRE(agg_cols[j].data != nullptr, "agg column data is NULL");
    NVTB_REQUIRE(agg_cols[j].dtype >= NVTB_I32 && agg_cols[j].dtype <= NVTB_U8, "bad agg dtype");
    ac.data[j] = agg_cols[j].data; ac.mask[j] = agg_cols[j].validity; ac.dtype[j] = agg_cols[j].dtype;
  }
  const size_t ksz = dtype_size(key->dtype);
  {
    int rc = settle(h);
    if (rc) return rc;
    const bool can_narrow = h->n_agg == 0 && key->dtype == NVTB_I32 &&
                            h->rows_total + n < (int64_t)0xFFFFFFF0ll;
    if (h->acc) {
      // sorted accumulator: nothing to switch
    } else if (h->rows_total == 0 && h->u_known == 0 && can_narrow && !h->t.narrow) {
      // empty table: switch to the 8-byte layout in place
      const int64_t cap = h->t.capacity;
      rc = table_free(&h->t, st);
      if (rc) return rc;
      rc = table_alloc(&h->t, cap, 0, true, st);
      if (rc) return rc;
    } else if (h->t.narrow && !can_narrow) {
      rc = grow_to(h, h->t.capacity, st, /*force_wide=*/true);   // int64 keys or >= 2^32 rows
      if (rc) return rc;
    }
  }
  // batches: [sample of 2^20 rows when nothing is known about the cardinality] + the rest
  int64_t off = 0;
  while (off < n) {
    int rc = settle(h);
    if (rc) return rc;
    int64_t m = n - off;
    const bool blind = (h->acc == nullptr && h->hint == 0 && h->k_est == 0);
    if (blind && m > 4 * kSampleRows) m = kSampleRows;
    const void* kp = (const char*)key->data + off * ksz;
    const uint8_t* mp = key->validity ? key->validity + (off >> 3) : nullptr;  // off % 8 == 0
    if (h->acc == nullptr) {
      // a column whose table would leave the L2 moves to the sorted accumulator (sortacc.cu)
      predict(h, m);
      const bool eligible = h->n_agg == 0 && key->dtype == NVTB_I32 && h->t.narrow &&
                            h->rows_total + n < (int64_t)0xFFFFFFF0ll && m < (int64_t)0xFFFF0000ll;
      if (eligible && h->predicted > (double)runs_min_keys()) {
        rc = table_to_runs(h, st);
        if (rc) return rc;
      }
    }
    if (h->acc) {
      NVTB_REQUIRE(h->n_agg == 0 && key->dtype == NVTB_I32, "a sorted accumulator takes int32 keys without payload");
      NVTB_REQUIRE(h->rows_total + m < (int64_t)0xFFFFFFF0ll, "more than 2^32 rows in one int32 accumulator");
      const int64_t mm = m < (int64_t)0xFFFF0000ll ? m : (int64_t)0x80000000ll;
      const bool stage = sortacc_stages(h->acc, mm);
      if (!stage || sortacc_stage_full(h->acc, mm)) {
        rc = acc_flush(h, st);
        if (rc) return rc;
      }
      if (stage) {                        // copy now, sort later together with the other batches of this fit
        rc = sortacc_stage(h->acc, (const int32_t*)kp, mp, mm, h->rows_total, st);
        if (rc) return rc;
      } else {                            // ragged tail waiting, or a batch larger than the stage
        rc = settle(h);
        if (rc) return rc;
        rc = sortacc_insert(h->acc, (const int32_t*)kp, mp, mm, h->u_known, h->ctr, st);
        if (rc) return rc;
        rc = post(h, st);
        if (rc) return rc;
      }
      h->rows_total += mm;
      off += mm;
      continue;
    }
    rc = prepare(h, m, st);
    if (rc) return rc;
    AggCols a2 = ac;
    for (int j = 0; j < h->n_agg; ++j) {
      a2.data[j] = (const char*)ac.data[j] + off * dtype_size(ac.dtype[j]);
      a2.mask[j] = ac.mask[j] ? ac.mask[j] + (off >> 3) : nullptr;
    }
    if (key->dtype == NVTB_I32) rc = launch_insert<int32_t>(h, (const int32_t*)kp, mp, a2, m, st);
    else                        rc = launch_insert<int64_t>(h, (const int64_t*)kp, mp, a2, m, st);
    if (rc) return rc;
    off += m;
  }
  return NVTB_OK;
}

int nvtb_hashagg_merge(nvtb_hashagg_t* h, const int64_t* keys,
                       const int64_t* sizes, const double* vals, int64_t n,
                       void* stream) {
  NVTB_REQUIRE(h != nullptr && n >= 0, "NULL handle or n < 0");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(keys != nullptr && sizes != nullptr, "NULL keys/sizes");
  NVTB_REQUIRE(h->n_agg == 0 || vals != nullptr, "vals is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = settle(h);
  if (rc) return rc;
  if (h->acc) {
    set_error("nvtb_hashagg_merge: the handle holds a sorted accumulator (raw int32 rows only)");
    return NVTB_ESTATE;
  }
  // pre-aggregated rows: distinct keys within the batch => every row may be new; sizes are
  // arbitrary int64 => wide layout
  rc = grow_to(h, next_pow2((int64_t)(2.5 * (double)(h->u_known + n)) + 1), st, /*force_wide=*/true);
  if (rc) return rc;
  rc = arena_acquire(h, &h->arena, n, h->n_agg);
  if (rc) return rc;
  rc = launch_merge(h, keys, sizes, vals, n, h->arena, st);
  if (rc) return rc;
  h->rows_total += n;
  return post(h, st);
}

int nvtb_hashagg_add_null_group(nvtb_hashagg_t* h, int64_t size, const double* vals_host) {
  NVTB_REQUIRE(h != nullptr && size >= 0, "NULL handle or size < 0");
  // tiny, synchronous: used once per rank in the cross-GPU merge
  int rc = settle(h);
  if (rc) return rc;
  Counters s;
  NVTB_CUDA_OK(cudaDeviceSynchronize());
  NVTB_CUDA_OK(cudaMemcpy(&s, h->ctr, sizeof(s), cudaMemcpyDeviceToHost));
  s.size[0] += (unsigned long long)size;
  NVTB_CUDA_OK(cudaMemcpy(h->ctr, &s, sizeof(s), cudaMemcpyHostToDevice));
  h->mailbox_valid = false;
  if (h->n_agg > 0 && vals_host != nullptr) {
    double cur[4 * kMaxAgg];
    NVTB_CUDA_OK(cudaMemcpy(cur, h->special_vals, sizeof(double) * 4 * h->n_agg, cudaMemcpyDeviceToHost));
    for (int j = 0; j < h->n_agg; ++j) {
      cur[j * 4 + 0] += vals_host[j * 4 + 0];
      cur[j * 4 + 1] += vals_host[j * 4 + 1];
      int64_t mn, mx;
      memcpy(&mn, &cur[j * 4 + 2], 8);
      memcpy(&mx, &cur[j * 4 + 3], 8);
      const double a = vals_host[j * 4 + 2], b = vals_host[j * 4 + 3];
      if (a == a) mn = std::min<int64_t>(mn, enc_ordered(a));
      if (b == b) mx = std::max<int64_t>(mx, enc_ordered(b));
      memcpy(&cur[j * 4 + 2], &mn, 8);
      memcpy(&cur[j * 4 + 3], &mx, 8);
    }
    NVTB_CUDA_OK(cudaMemcpy(h->special_vals, cur, sizeof(double) * 4 * h->n_agg, cudaMemcpyHostToDevice));
  }
  return NVTB_OK;
}

int nvtb_hashagg_size(nvtb_hashagg_t* h, int64_t* n_unique, int64_t* null_size, void* stream) {
  NVTB_REQUIRE(h != nullptr, "NULL handle");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = settle(h);
  if (rc) return rc;
  if (h->acc && sortacc_staged_rows(h->acc) > 0) {   // batches still waiting: group them in now
    rc = acc_flush(h, st);
    if (rc) return rc;
    rc = settle(h);
    if (rc) return rc;
  }
  if (!h->mailbox_valid) {   // e.g. right after create/reset/add_null_group: read the counters
    NVTB_CUDA_OK(cudaMemcpyAsync(h->mailbox, h->ctr, sizeof(Counters), cudaMemcpyDeviceToHost, st));
    NVTB_CUDA_OK(cudaStreamSynchronize(st));
    h->mailbox_valid = true;
  }
  const Counters s = *h->mailbox;
  h->u_known = (int64_t)s.n_unique;
  if (n_unique) *n_unique = (int64_t)s.n_unique + (s.size[1] ? 1 : 0);
  if (null_size) *null_size = (int64_t)s.size[0];
  return NVTB_OK;
}

int nvtb_hashagg_export(nvtb_hashagg_t* h, int64_t* keys_out, int64_t* sizes_out,
                        double* vals_out, double* null_vals_host, void* stream) {
  NVTB_REQUIRE(h != nullptr, "NULL handle");
  cudaStream_t st = (cudaStream_t)stream;
  int64_t nu = 0, ns = 0;
  int rc = nvtb_hashagg_size(h, &nu, &ns, stream);
  if (rc) return rc;
  const Counters s = *h->mailbox;
  double dec[8 * kMaxAgg];
  if (h->n_agg > 0) {
    double* d_dec = nullptr;
    NVTB_CUDA_OK(cudaMallocAsync(&d_dec, sizeof(double) * 8 * h->n_agg, st));
    decode_special_kernel<<<1, 64, 0, st>>>(h->special_vals, h->n_agg, d_dec);
    NVTB_LAUNCH_OK();
    NVTB_CUDA_OK(cudaMemcpyAsync(dec, d_dec, sizeof(double) * 8 * h->n_agg, cudaMemcpyDeviceToHost, st));
    NVTB_CUDA_OK(cudaFreeAsync(d_dec, st));
    NVTB_CUDA_OK(cudaStreamSynchronize(st));
    if (null_vals_host) memcpy(null_vals_host, dec, sizeof(double) * 4 * h->n_agg);
  }
  if (nu == 0) return NVTB_OK;
  NVTB_REQUIRE(keys_out != nullptr, "keys_out is NULL");
  NVTB_REQUIRE(h->n_agg == 0 || vals_out != nullptr, "vals_out is NULL");
  if (h->acc) return sortacc_unpack(h->acc, nu, keys_out, sizes_out, st);   // the rows come out in key order
  unsigned long long* cursor = nullptr;
  NVTB_CUDA_OK(cudaMallocAsync(&cursor, sizeof(unsigned long long), st));
  NVTB_CUDA_OK(cudaMemsetAsync(cursor, 0, sizeof(unsigned long long), st));
  export_kernel<<<plain_grid(h->t.capacity / kExportPerThread), kThreads, 0, st>>>(h->t, keys_out, sizes_out, vals_out, cursor);
  NVTB_LAUNCH_OK();
  NVTB_CUDA_OK(cudaFreeAsync(cursor, st));
  if (s.size[1]) {  // the INT64_MIN key lives outside the table: append it last
    const int64_t o = (int64_t)s.n_unique;
    const int64_t k = kEmptyKey, sz = (int64_t)s.size[1];
    NVTB_CUDA_OK(cudaMemcpyAsync(keys_out + o, &k, 8, cudaMemcpyHostToDevice, st));
    if (sizes_out) NVTB_CUDA_OK(cudaMemcpyAsync(sizes_out + o, &sz, 8, cudaMemcpyHostToDevice, st));
    if (vals_out && h->n_agg > 0)
      NVTB_CUDA_OK(cudaMemcpyAsync(vals_out + o * h->n_agg * 4, dec + 4 * h->n_agg,
                                   sizeof(double) * 4 * h->n_agg, cudaMemcpyHostToDevice, st));
    NVTB_CUDA_OK(cudaStreamSynchronize(st));  // host temporaries above
  }
  return NVTB_OK;
}

// ---------------------------------------------------------------------------------------
// sorted accumulators in the cross-GPU vocabulary merge (nvtabular_b200/dist.py)
// ---------------------------------------------------------------------------------------
// Turn an int32 key-count handle into a sorted accumulator (no-op when it already is one), so
// that every rank of a fit holds the same representation of a high-cardinality column.
int nvtb_hashagg_to_sorted(nvtb_hashagg_t* h, void* stream) {
  NVTB_REQUIRE(h != nullptr, "NULL handle");
  cudaStream_t st = (cudaStream_t)stream;
  int rc = settle(h);
  if (rc) return rc;
  if (h->acc) return NVTB_OK;
  int64_t nu = 0, ns = 0;
  rc = nvtb_hashagg_size(h, &nu, &ns, stream);
  if (rc) return rc;
  if (h->n_agg != 0 || (h->u_known > 0 && !h->t.narrow) || h->mailbox->size[1] != 0 ||
      h->rows_total >= (int64_t)0xFFFFFFF0ll) {
    set_error("nvtb_hashagg_to_sorted: only int32 key-count tables below 2^32 rows can become sorted accumulators");
    return NVTB_ESTATE;
  }
  return table_to_runs(h, st);
}

// packed pairs (key ^ 2^31) << 32 | count of a sorted accumulator, in key order.  out == NULL:
// only *n_host is set.
int nvtb_hashagg_export_packed(nvtb_hashagg_t* h, uint64_t* out, int64_t* n_host, void* stream) {
  NVTB_REQUIRE(h != nullptr && n_host != nullptr, "NULL argument");
  cudaStream_t st = (cudaStream_t)stream;
  int64_t nu = 0, ns = 0;
  int rc = nvtb_hashagg_size(h, &nu, &ns, stream);
  if (rc) return rc;
  if (h->acc == nullptr) {
    set_error("nvtb_hashagg_export_packed: the handle is not a sorted accumulator");
    return NVTB_ESTATE;
  }
  *n_host = h->u_known;
  if (out != nullptr && h->u_known > 0)
    NVTB_CUDA_OK(cudaMemcpyAsync(out, sortacc_pairs(h->acc), sizeof(uint64_t) * (size_t)h->u_known,
                                 cudaMemcpyDeviceToDevice, st));
  return NVTB_OK;
}

// Sort / run-length encode / merge the batches a sorted accumulator has staged (no-op for a hash
// table or when nothing is waiting).  Reads of the handle do this implicitly; a caller that
// wants the cost attributed to the group-by (bench.py) calls it at the end of the last batch.
int nvtb_hashagg_flush(nvtb_hashagg_t* h, void* stream) {
  NVTB_REQUIRE(h != nullptr, "NULL handle");
  return acc_flush(h, (cudaStream_t)stream);
}

int nvtb_hashagg_mode(nvtb_hashagg_t* h, int* mode_host) {
  NVTB_REQUIRE(h != nullptr && mode_host != nullptr, "NULL argument");
  *mode_host = h->acc != nullptr ? 1 : 0;
  return NVTB_OK;
}

}  // extern "C"
