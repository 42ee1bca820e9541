// fold_i32.cuh — K3 fast path for int32 keys without payload (every Categorify column of
// the Criteo workload).  Included by hashagg.cu after the global-table primitives and
// partition.cuh (the PARTS mode's hash partition).
//
// Why it looks like this (tools/microbench_atomics.cu compares the primitives): a count
// absorbed by a shared-memory RED costs little more than streaming the key, while one that
// reaches the global table costs a global RED (L2-resident) or a sector probe plus a RED,
// and a DRAM round trip once the table leaves L2 — roughly an order of magnitude more.
// The reference's answer to the same problem is a per-partition cuDF groupby followed by
// a concat+groupby tree (nvtabular/ops/categorify.py:955-1137); here:
//
//   DIRECT mode  (expected distinct keys <= what one SM's shared memory holds):
//     fold_i32_kernel streams the column once; every CTA owns a find-or-claim table in
//     shared memory (4-way buckets, 28 672 slots = 224 KB, filled to <= 20 %) and flushes one
//     (key, count) pair per distinct key into the resident global table at the end.
//   PARTS mode  (more distinct keys): one 512..4096-way hash partition of the keys
//     (partition.cuh with PartHashTop: part_hist_kernel -> part_scan_kernel ->
//     part_scatter_kernel), then the SAME fold kernel
//     runs once per partition: a partition holds ~U/P distinct keys, which fit.
//   Either way a key that finds its shared bucket full goes straight to the global
//   table (and from there, if the table is too small, to the overflow arena): the
//   cardinality estimate only ever costs time, never correctness.
//
// The shared table stores h = fold_hash(key), a BIJECTION of the 32-bit key, instead of
// the key: the top lg(P) bits of h are the partition, the following bits pick the bucket,
// and the flush recovers the key with fold_unhash().
#pragma once

namespace nvtb {

// fold_hash / fold_unhash / kFoldEmpty: common.cuh

constexpr int kFoldThreadsDirect = 1024;   // 1 CTA / SM, 224 KB table
constexpr int kFoldThreadsParts = 512;     // 2 CTAs / SM, 110 KB tables
constexpr int kFoldWays = 4;                       // slots per bucket = one 128-bit shared load
constexpr int kFoldSlotBytes = 10;                 // hash + count + one entry of the live list
constexpr unsigned kFoldBucketsDirect = 5728;      // x 4 slots x 10 B = 224 KB
constexpr unsigned kFoldBucketsParts = 2816;       // 110 KB
// 4-way buckets without displacement overflow for ~0.2 % of the keys at load 0.2 and ~2 % at
// load 0.4; an overflowing key costs every one of its rows the divergent slow path
constexpr double kFoldMaxLoad = 0.2;
constexpr int kMinParts = 512;

// ---------------------------------------------------------------------------------------
// shared-memory find-or-claim table
// ---------------------------------------------------------------------------------------
struct FoldTable {
  uint32_t* hk;    // [4 * nb] hashes, bucket b = hk[4b .. 4b+3]; kFoldEmpty = free
  uint32_t* cnt;   // [4 * nb]
  uint16_t* live;  // [4 * nb] slots claimed since the last flush, in claim order
  unsigned* n_live;
  unsigned nb;
  int lg;          // partition bits already consumed at the top of h

  __device__ __forceinline__ unsigned bucket(uint32_t h) const { return __umulhi(h << lg, nb); }

  template <int T> __device__ __forceinline__ void clear() {
    for (unsigned s = threadIdx.x; s < kFoldWays * nb; s += T) { hk[s] = kFoldEmpty; cnt[s] = 0u; }
  }

  // claim a slot of bucket b for h (or find it there after losing a race); false = full.
  // A fresh claim is appended to the live list: flush and re-clear then touch only the
  // slots in use (a partition of a high-cardinality column fills ~15 % of its table, and a
  // flush that walks every slot serialises ~14 dependent DRAM round trips per thread).
  static __device__ __forceinline__ bool claim(uint32_t* hk, uint32_t* cnt, uint16_t* live,
                                               unsigned* n_live, uint32_t h, unsigned b) {
    bool done = false;
#pragma unroll
    for (int j = 0; j < kFoldWays; ++j) {
      if (!done) {
        const unsigned s = kFoldWays * b + j;
        uint32_t cur = *reinterpret_cast<volatile uint32_t*>(hk + s);
        if (cur == kFoldEmpty) {
          cur = atomicCAS(hk + s, kFoldEmpty, h);
          if (cur == kFoldEmpty) live[atomicAdd(n_live, 1u)] = (uint16_t)s;
        }
        if (cur == kFoldEmpty || cur == h) {
          atomicAdd(cnt + s, 1u);
          done = true;
        }
      }
    }
    return done;
  }

  // candidates of h's bucket (issued early, resolved later: several LDS in flight per lane)
  __device__ __forceinline__ uint4 peek(uint32_t h) const {
    uint4 c;
    const unsigned addr = (unsigned)__cvta_generic_to_shared(hk + kFoldWays * bucket(h));
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(c.x), "=r"(c.y), "=r"(c.z), "=r"(c.w) : "r"(addr));
    return c;
  }
  // fast path only: true = h sat in its bucket and was counted
  __device__ __forceinline__ bool hit(uint32_t h, uint4 c) {
    if (h == kFoldEmpty) return false;            // would "match" a free slot
    const int j = (c.x == h) ? 0 : (c.y == h) ? 1 : (c.z == h) ? 2 : (c.w == h) ? 3 : -1;
    if (j < 0) return false;
    atomicAdd(cnt + kFoldWays * bucket(h) + j, 1u);
    return true;
  }
};

// Everything that is not "h already sits in its shared bucket": claim a shared slot, or -
// bucket full, or h is the one reserved value - update the global table directly.  ONE
// out-of-line copy, called from a cold block after the fast loop, so that the values the
// fast loop keeps in registers are not saved and restored around a call per row.
// Returns the number of keys it added to the GLOBAL table (0 or 1).
static __device__ __noinline__ unsigned fold_slow(const FoldTable& ft, uint32_t h, const Table& t,
                                                  const Arena& arena, Counters* ctr) {
  if (h != kFoldEmpty && FoldTable::claim(ft.hk, ft.cnt, ft.live, ft.n_live, h, ft.bucket(h))) return 0u;
  unsigned n_new = 0;
  const long long key = (long long)(int32_t)fold_unhash(h);
  Probe<true> pr;
  probe_first<true>(t, key, pr);
  upsert_or_spill<true>(t, arena, ctr, key, 1, pr, n_new);
  return n_new;
}

// One work unit = a contiguous row range folded into a freshly cleared shared table and
// flushed.  DIRECT: unit u = rows [u*chunk, (u+1)*chunk) of the column (with its validity
// mask).  PARTS: unit p = partition p = rows [starts[p], ends[p]) of the partition buffer.
template <int T, int MINB, bool PREHASHED>
__global__ void __launch_bounds__(T, MINB)
fold_i32_kernel(const int32_t* __restrict__ keys, const uint8_t* __restrict__ mask, int64_t n,
                const uint32_t* __restrict__ starts, const uint32_t* __restrict__ ends,
                int n_units, int64_t chunk, int lg, unsigned nb, int aligned,
                Table t, Counters* ctr, Arena arena) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FoldTable ft;
  ft.hk = reinterpret_cast<uint32_t*>(smem_raw);
  ft.cnt = ft.hk + kFoldWays * nb;
  ft.live = reinterpret_cast<uint16_t*>(ft.cnt + kFoldWays * nb);
  ft.nb = nb;
  ft.lg = lg;
  __shared__ unsigned int s_null, s_new, s_live;
  ft.n_live = &s_live;
  if (threadIdx.x == 0) { s_null = 0u; s_new = 0u; s_live = 0u; }
  unsigned n_null = 0, n_new = 0;
  ft.clear<T>();      // once: a flush hands the table back empty

  // 8 rows of one lane.  The hash replaces the key in registers (fold_unhash recovers it
  // where needed); bucket candidates are fetched four rows at a time; rows that are not
  // plain hits are only FLAGGED in the fast loop and resolved afterwards.
  auto fold8 = [&](Rows8& r) {
    n_null += __popc(r.lv & ~r.m);
    unsigned pend = 0;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      uint4 c[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (!PREHASHED) r.v[4 * half + k] = (int32_t)fold_hash((uint32_t)r.v[4 * half + k]);
        c[k] = ft.peek((uint32_t)r.v[4 * half + k]);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (((r.m >> (4 * half + k)) & 1u) && !ft.hit((uint32_t)r.v[4 * half + k], c[k]))
          pend |= 1u << (4 * half + k);
    }
    if (pend) {
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if ((pend >> k) & 1u)
          n_new += fold_slow(ft, (uint32_t)r.v[k], t, arena, ctr);
    }
  };

  for (int unit = blockIdx.x; unit < n_units; unit += gridDim.x) {
    int64_t r0, r1;
    if (starts != nullptr) { r0 = (int64_t)starts[unit]; r1 = (int64_t)ends[unit]; }
    else { r0 = (int64_t)unit * chunk; r1 = r0 + chunk < n ? r0 + chunk : n; }
    __syncthreads();
    if (aligned) {
      constexpr int64_t step = (int64_t)T * 8;
      for (int64_t base = r0; base < r1; base += 2 * step) {
        Rows8 a, b;
        load_rows8(keys, mask, base + (int64_t)threadIdx.x * 8, r1, a);
        load_rows8(keys, mask, base + step + (int64_t)threadIdx.x * 8, r1, b);
        fold8(a);
        fold8(b);
      }
    } else {
      for (int64_t i = r0 + threadIdx.x; i < r1; i += T) {
        if (!valid1(mask, i)) { n_null++; continue; }
        const int32_t key = keys[i];
        const uint32_t h = PREHASHED ? (uint32_t)key : fold_hash((uint32_t)key);
        if (!ft.hit(h, ft.peek(h))) n_new += fold_slow(ft, h, t, arena, ctr);
      }
    }
    __syncthreads();
    // flush: one global update per distinct key of the unit, two first probes in flight per
    // thread; every flushed slot is handed back empty
    const unsigned n_live = s_live;
    for (unsigned i0 = 0; i0 < n_live; i0 += T * 2) {
      long long k[2];
      unsigned c[2];
      Probe<true> pr[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const unsigned i = i0 + j * T + threadIdx.x;
        c[j] = 0u;
        k[j] = 0;
        if (i < n_live) {
          const unsigned s = ft.live[i];
          c[j] = ft.cnt[s];
          k[j] = (long long)(int32_t)fold_unhash(ft.hk[s]);
          ft.hk[s] = kFoldEmpty;
          ft.cnt[s] = 0u;
          probe_first<true>(t, k[j], pr[j]);
        }
      }
#pragma unroll
      for (int j = 0; j < 2; ++j)
        if (c[j]) upsert_or_spill<true>(t, arena, ctr, k[j], (int64_t)c[j], pr[j], n_new);
    }
    __syncthreads();
    if (threadIdx.x == 0) s_live = 0u;
  }
  if (n_null) atomicAdd(&s_null, n_null);
  if (n_new) atomicAdd(&s_new, n_new);
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_null) atomicAdd(&ctr->size[0], (unsigned long long)s_null);
    if (s_new) atomicAdd(&ctr->n_unique, (unsigned long long)s_new);
  }
}

}  // namespace nvtb
