// bucketagg.cuh — the group-by of a staged batch of a sorted accumulator WITHOUT a sort:
// one order-free range partition + direct-address counting in shared memory.
// Included by sortacc.cu after partition.cuh.
//
// What it replaces: the LSD radix pipeline of sortagg.cuh (12-bit order-free pass + two STABLE
// 10-bit passes + run-length encode) moved every key through HBM three times and spent most of
// its time in the stable scatter, whose match.any ranking through shared memory keeps it far from
// HBM-bound.  Equal keys only have to MEET, and the result only has to come out in key order:
//
//   1. min / max of the valid keys (u = key ^ 2^31) -> lo, shift with (max - lo) >> shift < 2^13;
//      the staging copies (bk_stage_kernel) fold them, a batch grouped without staging has its own
//      pass (bk_minmax_kernel)
//   2. an order-free partition of v = u - lo by its top bits into 8192 buckets, in two levels so
//      that every write fills whole sectors: one histogram of the 8192 buckets (their starts are
//      the final layout), a scatter into 512 coarse ranges of 16 consecutive buckets (the partition
//      kernels of partition.cuh), then each range into its buckets (bk_refine_kernel)
//      — bucket b holds the keys of a window of 2^shift <= 2^19 consecutive values
//   3. one CTA per bucket: a PRESENCE BITMAP of the window in shared memory (<= 64 KB); a second
//      bitmap marks the values seen twice; only those get a counter (dense index = popcount
//      prefix of the second bitmap).  The bucket's keys are streamed, never stored: a bucket may
//      hold any number of rows and any number of distinct keys; only the number of DUPLICATED
//      values per window is bounded (14 336) — beyond that the caller falls back to the radix path.
//      The emit's shared memory is sized for the batch's window and its fullest bucket.
//   4. the distinct values are emitted in bitmap order = key order, as packed (key, count) pairs
// Buckets are consecutive key ranges, so the concatenation is the key-ordered accumulator.  Every
// key crosses HBM four times (two partition reads + writes) plus two L2-resident re-reads of its
// bucket.
#pragma once

namespace nvtb {

constexpr int kBkThreads = 1024;
constexpr int kBkLgParts = 13;                       // 8192 buckets
constexpr int kBkParts = 1 << kBkLgParts;
constexpr int kBkMaxShift = 32 - kBkLgParts;         // window of at most 2^19 values
constexpr int kBkWords = 1 << (kBkMaxShift - 5);     // 16384 bitmap words
constexpr int kBkDupCap = 14336;                     // counters per bucket
constexpr int kBkCountSmem = 4 * kBkWords;                                    // 64 KB

// partition policy: parameters live on the device (computed from the data, no host round trip)
struct PartRange {
  int lg;
  const uint32_t* par;     // [0] lo, [1] shift
  __device__ __forceinline__ uint32_t xform(uint32_t k) const { return (k ^ 0x80000000u) - par[0]; }
  __device__ __forceinline__ uint32_t bin(uint32_t v) const { return v >> par[1]; }
};

// min / max of u = key ^ 2^31 over the valid rows of one lane's group
__device__ __forceinline__ void bk_fold_minmax(const Rows8& r, uint32_t& lo, uint32_t& hi) {
#pragma unroll
  for (int k = 0; k < 8; ++k)
    if ((r.m >> k) & 1u) {
      const uint32_t u = (uint32_t)r.v[k] ^ 0x80000000u;
      lo = u < lo ? u : lo;
      hi = u > hi ? u : hi;
    }
}

// the lane's {lo, hi} into mm[0] = min, mm[1] = max (mm preset to {~0, 0})
__device__ __forceinline__ void bk_publish_minmax(uint32_t lo, uint32_t hi, uint32_t* mm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const uint32_t a = __shfl_down_sync(0xFFFFFFFFu, lo, o), b = __shfl_down_sync(0xFFFFFFFFu, hi, o);
    lo = a < lo ? a : lo;
    hi = b > hi ? b : hi;
  }
  if ((threadIdx.x & 31) == 0 && lo <= hi) { atomicMin(&mm[0], lo); atomicMax(&mm[1], hi); }
}

// the same order as PartRange, 16 times coarser: the first pass of the two-level partition
// (bk_refine_kernel splits each coarse range into its 16 buckets).  512 ranges: runs of ~32 keys
// (whole sectors) per tile and range, and at least as many ranges as part_scatter_kernel has threads
constexpr int kBkLgFine = 4;
constexpr int kBkFine = 1 << kBkLgFine;              // buckets per coarse range
constexpr int kBkCoarse = kBkParts / kBkFine;        // 512 coarse ranges
struct PartRangeCoarse {
  int lg;
  const uint32_t* par;     // [0] lo, [1] shift (of the fine buckets)
  __device__ __forceinline__ uint32_t xform(uint32_t k) const { return (k ^ 0x80000000u) - par[0]; }
  __device__ __forceinline__ uint32_t bin(uint32_t v) const { return v >> (par[1] + kBkLgFine); }
};

// write cursors of both partition passes from the bucket starts: fine[b] = starts[b],
// coarse[c] = starts[16 c]
static __global__ void bk_cursors_kernel(const uint32_t* __restrict__ starts, uint32_t* __restrict__ fine,
                                         uint32_t* __restrict__ coarse) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= kBkParts) return;
  const uint32_t v = starts[b];
  fine[b] = v;
  if ((b & (kBkFine - 1)) == 0) coarse[b / kBkFine] = v;
}

// second pass of the two-level partition: in[] holds the valid keys (v = u - lo) grouped by coarse
// range, range c at [starts[16 c], starts[16 c + 16]).  Tiles of kBkRefineTile keys never cross a
// range; each tile is binned by shared-memory counts into the range's 16 buckets, reserves one run per
// bucket at cursor[] (one global atomic per non-empty (tile, bucket)) and is written out of a
// shared-memory stage, so that runs are hundreds of keys long and every write fills whole sectors.
constexpr int kBkRefineVals = 16;                               // keys per thread and tile
constexpr int kBkRefineTile = kPartThreads * kBkRefineVals;     // 8192 keys: runs of ~256 per bucket
static __global__ void __launch_bounds__(kPartThreads, 2)
bk_refine_kernel(const uint32_t* __restrict__ in, const uint32_t* __restrict__ starts,
                 const uint32_t* __restrict__ n_valid, const uint32_t* __restrict__ par,
                 uint32_t* __restrict__ cursor, uint32_t* __restrict__ out) {
  __shared__ uint32_t bk_stage[kBkRefineTile];
  __shared__ uint32_t cs[kBkCoarse + 1];                  // range starts, cs[kBkCoarse] = end
  __shared__ uint32_t tp[kBkCoarse + 1];                  // first tile of each range
  __shared__ uint32_t cnt[kBkFine], delta[kBkFine];
  constexpr int kVals = kBkRefineVals;
  const uint32_t shift = par[1];
  const int lane = threadIdx.x & 31;
  for (int c = threadIdx.x; c <= kBkCoarse; c += kPartThreads) cs[c] = c < kBkCoarse ? starts[c * kBkFine] : *n_valid;
  __syncthreads();
  if (threadIdx.x < 32) {
    constexpr int kPer = kBkCoarse / 32;
    uint32_t t[kPer], loc = 0;
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int c = lane * kPer + j;
      t[j] = (cs[c + 1] - cs[c] + kBkRefineTile - 1) / kBkRefineTile;
      loc += t[j];
    }
    uint32_t incl = loc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
      if (lane >= o) incl += y;
    }
    uint32_t run = incl - loc;
#pragma unroll
    for (int j = 0; j < kPer; ++j) { tp[lane * kPer + j] = run; run += t[j]; }
    if (lane == 31) tp[kBkCoarse] = run;
  }
  __syncthreads();
  const uint32_t n_tiles = tp[kBkCoarse];
  for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    int c = 0;                                            // the last range whose first tile <= tile
    for (int step = kBkCoarse / 2; step > 0; step >>= 1)
      if (tp[c + step] <= tile) c += step;
    const uint32_t b0 = cs[c] + (tile - tp[c]) * kBkRefineTile;
    const uint32_t b1 = min(b0 + (uint32_t)kBkRefineTile, cs[c + 1]);
    if (threadIdx.x < kBkFine) cnt[threadIdx.x] = 0u;
    __syncthreads();
    uint32_t v[kVals];
#pragma unroll
    for (int j = 0; j < kVals; ++j) {
      const uint32_t i = b0 + j * kPartThreads + threadIdx.x;
      v[j] = i < b1 ? __ldg(in + i) : 0u;
    }
#pragma unroll
    for (int j = 0; j < kVals; ++j)
      if (b0 + j * kPartThreads + threadIdx.x < b1) atomicAdd(&cnt[(v[j] >> shift) & (kBkFine - 1)], 1u);
    __syncthreads();
    if (threadIdx.x < 32) {
      const uint32_t x = lane < kBkFine ? cnt[lane] : 0u;
      uint32_t incl = x;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
        if (lane >= o) incl += y;
      }
      const uint32_t off = incl - x;
      if (lane < kBkFine) {
        const uint32_t g0 = x ? atomicAdd(&cursor[c * kBkFine + lane], x) : 0u;
        delta[lane] = g0 - off;        // modulo 2^32: global index = delta + staged index
        cnt[lane] = off;               // running staged cursor
      }
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kVals; ++j)
      if (b0 + j * kPartThreads + threadIdx.x < b1) {
        const uint32_t p = atomicAdd(&cnt[(v[j] >> shift) & (kBkFine - 1)], 1u);
        bk_stage[p] = v[j];
      }
    __syncthreads();
    const uint32_t total = b1 - b0;
    for (uint32_t j = threadIdx.x; j < total; j += kPartThreads) {
      const uint32_t hv = bk_stage[j];
      out[delta[(hv >> shift) & (kBkFine - 1)] + j] = hv;
    }
    __syncthreads();
  }
}

// mm = {min, max} of u over the valid rows (a batch that is grouped without being staged)
static __global__ void __launch_bounds__(kPartThreads)
bk_minmax_kernel(const int32_t* __restrict__ keys, const uint8_t* __restrict__ mask, int64_t n,
                 uint32_t* __restrict__ mm, int aligned) {
  uint32_t lo = 0xFFFFFFFFu, hi = 0u;
  const int64_t n_tiles = (n + kPartTile - 1) / kPartTile;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    Rows8 r[kPartGroups];
#pragma unroll
    for (int g = 0; g < kPartGroups; ++g)
      load_rows8(keys, mask, tile * kPartTile + ((int64_t)g * kPartThreads + threadIdx.x) * 8, n, r[g], aligned != 0);
#pragma unroll
    for (int g = 0; g < kPartGroups; ++g) bk_fold_minmax(r[g], lo, hi);
  }
  bk_publish_minmax(lo, hi, mm);
}

// staging copy of a batch: keys to dk[0, n), validity bytes to dm[0, ceil(n / 8)) (all valid when
// mask is NULL), and the batch's {min, max} of u folded into mm, so that the flush of the staged
// rows needs no pass of its own to find them.  dk is 32-byte aligned.
static __global__ void __launch_bounds__(kPartThreads)
bk_stage_kernel(const int32_t* __restrict__ keys, const uint8_t* __restrict__ mask, int64_t n,
                int32_t* __restrict__ dk, uint8_t* __restrict__ dm, uint32_t* __restrict__ mm, int aligned) {
  uint32_t lo = 0xFFFFFFFFu, hi = 0u;
  const int64_t n_tiles = (n + kPartTile - 1) / kPartTile;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    Rows8 r[kPartGroups];
#pragma unroll
    for (int g = 0; g < kPartGroups; ++g)
      load_rows8(keys, mask, tile * kPartTile + ((int64_t)g * kPartThreads + threadIdx.x) * 8, n, r[g], aligned != 0);
#pragma unroll
    for (int g = 0; g < kPartGroups; ++g) {
      const int64_t i = tile * kPartTile + ((int64_t)g * kPartThreads + threadIdx.x) * 8;
      if (r[g].lv == 0xFFu) {
        st_rows8<int32_t>(dk + i, r[g].v);
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k)
          if ((r[g].lv >> k) & 1u) dk[i + k] = r[g].v[k];
      }
      if (r[g].lv) dm[i >> 3] = (uint8_t)r[g].m;
      bk_fold_minmax(r[g], lo, hi);
    }
  }
  bk_publish_minmax(lo, hi, mm);
}

// par = {lo, shift}: the smallest shift with (max - lo) >> shift < 2^kBkLgParts
static __global__ void bk_params_kernel(const uint32_t* __restrict__ mm, uint32_t* __restrict__ par) {
  uint32_t lo = mm[0], hi = mm[1];
  if (lo > hi) { lo = 0u; hi = 0u; }                     // no valid key at all
  const uint32_t range = hi - lo;
  const int bits = range ? 32 - __clz(range) : 0;
  par[0] = lo;
  par[1] = (uint32_t)(bits > kBkLgParts ? bits - kBkLgParts : 0);
}

__device__ __forceinline__ uint32_t bk_block_sum(uint32_t v, uint32_t* ws /*[32]*/) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, o);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = v;
  __syncthreads();
  uint32_t t = 0;
  if (threadIdx.x < 32) {
    t = ws[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_down_sync(0xFFFFFFFFu, t, o);
    if (threadIdx.x == 0) ws[0] = t;
  }
  __syncthreads();
  t = ws[0];
  __syncthreads();
  return t;
}

// exclusive prefix of one value per thread (1024 threads); *total = block sum
__device__ __forceinline__ uint32_t bk_block_excl(uint32_t v, uint32_t* ws /*[33]*/, uint32_t* total) {
  uint32_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if ((threadIdx.x & 31) >= o) incl += y;
  }
  if ((threadIdx.x & 31) == 31) ws[threadIdx.x >> 5] = incl;
  __syncthreads();
  if (threadIdx.x < 32) {
    const uint32_t w = ws[threadIdx.x];
    uint32_t wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, wi, o);
      if (threadIdx.x >= o) wi += y;
    }
    ws[threadIdx.x] = wi - w;
    if (threadIdx.x == 31) ws[32] = wi;
  }
  __syncthreads();
  const uint32_t ex = ws[threadIdx.x >> 5] + incl - v;
  *total = ws[32];
  __syncthreads();
  return ex;
}

// bucket keys each thread loads before it touches shared memory (independent loads in flight)
constexpr int kBkUnroll = 4;

// the keys buf[i] of a bucket [s, e): f(v) for each, kBkUnroll loads per thread issued together
template <typename F>
__device__ __forceinline__ void bk_stream(const uint32_t* __restrict__ buf, uint32_t s, uint32_t e, F f) {
  for (uint32_t i0 = s + threadIdx.x; i0 < e; i0 += kBkThreads * kBkUnroll) {
    uint32_t v[kBkUnroll];
#pragma unroll
    for (int j = 0; j < kBkUnroll; ++j) {
      const uint32_t i = i0 + j * kBkThreads;
      v[j] = i < e ? __ldg(buf + i) : 0u;
    }
#pragma unroll
    for (int j = 0; j < kBkUnroll; ++j)
      if (i0 + j * kBkThreads < e) f(v[j]);
  }
}

// distinct values per bucket (presence bitmap + popcount); *max_rows = the most rows of a bucket
static __global__ void __launch_bounds__(kBkThreads)
bk_count_kernel(const uint32_t* __restrict__ buf, const uint32_t* __restrict__ starts,
                const uint32_t* __restrict__ n_valid, const uint32_t* __restrict__ par,
                uint32_t* __restrict__ distinct, uint32_t* __restrict__ max_rows) {
  extern __shared__ __align__(16) uint32_t bk_smem[];
  __shared__ uint32_t ws[33];
  uint32_t* bm = bk_smem;
  const int b = blockIdx.x;
  const uint32_t s = starts[b], e = (b + 1 < kBkParts) ? starts[b + 1] : *n_valid;
  if (s >= e) { if (threadIdx.x == 0) distinct[b] = 0u; return; }
  if (threadIdx.x == 0) atomicMax(max_rows, e - s);
  const uint32_t shift = par[1];
  const uint32_t wmask = (1u << shift) - 1u;                // shift <= 19
  const int words = shift > 5 ? 1 << (shift - 5) : 1;
  for (int w = threadIdx.x; w < words; w += kBkThreads) bm[w] = 0u;
  __syncthreads();
  bk_stream(buf, s, e, [&](uint32_t v) {
    const uint32_t off = v & wmask;
    const uint32_t bit = 1u << (off & 31);
    if (!(bm[off >> 5] & bit)) atomicOr(&bm[off >> 5], bit);
  });
  __syncthreads();
  uint32_t c = 0;
  for (int w = threadIdx.x; w < words; w += kBkThreads) c += __popc(bm[w]);
  const uint32_t tot = bk_block_sum(c, ws);
  if (threadIdx.x == 0) distinct[b] = tot;
}

// shared memory of bk_emit_kernel for a window of 2^shift values and `cap` counters: presence and
// duplicate bitmaps, the uint16 prefix of the duplicate bitmap (padded to 4 bytes), the counters
__host__ __device__ constexpr int bk_emit_words(uint32_t shift) { return shift > 5 ? 1 << (shift - 5) : 1; }
__host__ __device__ constexpr int bk_emit_smem(uint32_t shift, int cap) {
  return 4 * (2 * bk_emit_words(shift) + (bk_emit_words(shift) + 1) / 2 + cap);
}
constexpr int kBkEmitSmem = bk_emit_smem(kBkMaxShift, kBkDupCap);   // 216 KB: the widest window

// packed pairs of every bucket, in key order, at out[out_base[b] ...).  The launch sizes the shared
// memory for the batch's window and for `cap` counters (cap <= kBkDupCap, and no bucket of the
// batch can hold more duplicated values than half its rows, which the caller bounds cap by).
// *flag is set when a bucket has more than cap duplicated values (the caller then redoes the batch
// with the radix pipeline).
static __global__ void __launch_bounds__(kBkThreads, 2)
bk_emit_kernel(const uint32_t* __restrict__ buf, const uint32_t* __restrict__ starts,
               const uint32_t* __restrict__ n_valid, const uint32_t* __restrict__ par,
               const uint32_t* __restrict__ out_base, uint64_t* __restrict__ out, uint32_t cap,
               unsigned int* __restrict__ flag, unsigned long long* __restrict__ max_count) {
  extern __shared__ __align__(16) uint32_t bk_smem[];
  __shared__ uint32_t ws[33];
  const int b = blockIdx.x;
  const uint32_t s = starts[b], e = (b + 1 < kBkParts) ? starts[b + 1] : *n_valid;
  if (s >= e) return;
  const uint32_t lo = par[0], shift = par[1];
  const uint32_t wmask = (1u << shift) - 1u;
  const int words = bk_emit_words(shift);
  uint32_t* bm = bk_smem;                                   // presence
  uint32_t* dup = bm + words;                               // seen at least twice
  uint16_t* pfx = reinterpret_cast<uint16_t*>(dup + words); // exclusive popcount prefix of dup
  uint32_t* cnt = dup + words + (words + 1) / 2;            // occurrences of the duplicated values
  const int per = (words + kBkThreads - 1) / kBkThreads;    // consecutive words per thread
  for (int w = threadIdx.x; w < words; w += kBkThreads) { bm[w] = 0u; dup[w] = 0u; }
  __syncthreads();
  bk_stream(buf, s, e, [&](uint32_t v) {
    const uint32_t off = v & wmask;
    const uint32_t bit = 1u << (off & 31), w = off >> 5;
    const uint32_t old = atomicOr(&bm[w], bit);
    if ((old & bit) && !(dup[w] & bit)) atomicOr(&dup[w], bit);
  });
  __syncthreads();
  // dense index of the duplicated values
  const int w0 = threadIdx.x * per;
  uint32_t c = 0;
  for (int j = 0; j < per; ++j) if (w0 + j < words) c += __popc(dup[w0 + j]);
  uint32_t n_dup;
  uint32_t run = bk_block_excl(c, ws, &n_dup);
  if (n_dup > cap) {
    if (threadIdx.x == 0) atomicOr(flag, 1u);
    return;
  }
  for (int j = 0; j < per; ++j)
    if (w0 + j < words) { pfx[w0 + j] = (uint16_t)run; run += __popc(dup[w0 + j]); }
  for (uint32_t i = threadIdx.x; i < n_dup; i += kBkThreads) cnt[i] = 0u;
  __syncthreads();
  if (n_dup) {
    bk_stream(buf, s, e, [&](uint32_t v) {
      const uint32_t off = v & wmask;
      const uint32_t bit = 1u << (off & 31), w = off >> 5;
      const uint32_t d = dup[w];
      if (d & bit) atomicAdd(&cnt[pfx[w] + __popc(d & (bit - 1u))], 1u);
    });
    __syncthreads();
  }
  // emit in bitmap order = key order.  Warp q owns words [q * span, (q + 1) * span); it walks them
  // 32 at a time, one word per lane, so that the lanes of a store write consecutive pairs.
  const int lane = threadIdx.x & 31;
  const int span = (words + 31) / 32;
  const int q0 = (threadIdx.x >> 5) * span, q1 = min(q0 + span, words);
  c = 0;
  for (int w = q0 + lane; w < q1; w += 32) c += __popc(bm[w]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xFFFFFFFFu, c, o);
  uint32_t n_out;
  uint32_t r = __shfl_sync(0xFFFFFFFFu, bk_block_excl(lane == 0 ? c : 0u, ws, &n_out), 0);
  uint64_t* o = out + out_base[b];
  const uint32_t vbase = lo + ((uint32_t)b << shift);      // u of the window's first value (no overflow: b << shift <= range)
  uint32_t mx = 1u;
  for (int w0q = q0; w0q < q1; w0q += 32) {
    const int w = w0q + lane;
    uint32_t bits = w < q1 ? bm[w] : 0u;
    const uint32_t n_bits = __popc(bits);
    uint32_t incl = n_bits;
#pragma unroll
    for (int o2 = 1; o2 < 32; o2 <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, o2);
      if (lane >= o2) incl += y;
    }
    uint32_t pos = r + incl - n_bits;
    r += __shfl_sync(0xFFFFFFFFu, incl, 31);
    if (bits) {
      const uint32_t d = dup[w];
      const uint32_t pd = pfx[w];
      while (bits) {
        const int k = __ffs(bits) - 1;
        bits &= bits - 1u;
        uint32_t n = 1u;
        if ((d >> k) & 1u) n = cnt[pd + __popc(d & ((1u << k) - 1u))];
        mx = n > mx ? n : mx;
        o[pos++] = ((uint64_t)(vbase + ((uint32_t)w << 5) + (uint32_t)k) << 32) | (uint64_t)n;
      }
    }
  }
#pragma unroll
  for (int o2 = 16; o2 > 0; o2 >>= 1) { const uint32_t y = __shfl_down_sync(0xFFFFFFFFu, mx, o2); mx = y > mx ? y : mx; }
  if (lane == 0) atomicMax(max_count, (unsigned long long)mx);
}

}  // namespace nvtb
