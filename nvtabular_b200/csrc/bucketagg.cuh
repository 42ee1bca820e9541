// bucketagg.cuh — the group-by of a staged batch of a sorted accumulator WITHOUT a sort:
// one order-free range partition + direct-address counting in shared memory.
// Included by sortacc.cu after partition.cuh.
//
// What it replaces: the LSD radix pipeline of sortagg.cuh (12-bit order-free pass + two STABLE
// 10-bit passes + run-length encode) moved every key through HBM three times and spent most of
// its time in the stable scatter, whose match.any ranking through shared memory keeps it far from
// HBM-bound.  Equal keys only have to MEET, and the result only has to come out in key order:
//
//   1. min / max of the valid keys (u = key ^ 2^31) -> lo, shift with (max - lo) >> shift < 2^13
//   2. ONE order-free partition of v = u - lo by its top bits into 8192 buckets (the partition
//      kernels of partition.cuh: shared-memory counts, one global reservation per tile and bucket)
//      — bucket b holds the keys of a window of 2^shift <= 2^19 consecutive values
//   3. one CTA per bucket: a PRESENCE BITMAP of the window in shared memory (64 KB); a second
//      bitmap marks the values seen twice; only those get a counter (dense index = popcount
//      prefix of the second bitmap).  The bucket's keys are streamed, never stored: a bucket may
//      hold any number of rows and any number of distinct keys; only the number of DUPLICATED
//      values per window is bounded (14 336) — beyond that the caller falls back to the radix path
//   4. the distinct values are emitted in bitmap order = key order, as packed (key, count) pairs
// Buckets are consecutive key ranges, so the concatenation is the key-ordered accumulator.  Every
// key crosses HBM twice (partition read + write) plus two L2-resident re-reads of its bucket.
#pragma once

namespace nvtb {

constexpr int kBkThreads = 1024;
constexpr int kBkLgParts = 13;                       // 8192 buckets
constexpr int kBkParts = 1 << kBkLgParts;
constexpr int kBkMaxShift = 32 - kBkLgParts;         // window of at most 2^19 values
constexpr int kBkWords = 1 << (kBkMaxShift - 5);     // 16384 bitmap words
constexpr int kBkDupCap = 14336;                     // counters per bucket
constexpr int kBkCountSmem = 4 * kBkWords;                                    // 64 KB
constexpr int kBkEmitSmem = 4 * kBkWords * 2 + 2 * kBkWords + 4 * kBkDupCap;   // 216 KB

// partition policy: parameters live on the device (computed from the data, no host round trip)
struct PartRange {
  int lg;
  const uint32_t* par;     // [0] lo, [1] shift
  __device__ __forceinline__ uint32_t xform(uint32_t k) const { return (k ^ 0x80000000u) - par[0]; }
  __device__ __forceinline__ uint32_t bin(uint32_t v) const { return v >> par[1]; }
};

// mm[0] = min, mm[1] = max of u = key ^ 2^31 over the valid rows (mm preset to {~0, 0})
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
    for (int g = 0; g < kPartGroups; ++g)
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if ((r[g].m >> k) & 1u) {
          const uint32_t u = (uint32_t)r[g].v[k] ^ 0x80000000u;
          lo = u < lo ? u : lo;
          hi = u > hi ? u : hi;
        }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const uint32_t a = __shfl_down_sync(0xFFFFFFFFu, lo, o), b = __shfl_down_sync(0xFFFFFFFFu, hi, o);
    lo = a < lo ? a : lo;
    hi = b > hi ? b : hi;
  }
  if ((threadIdx.x & 31) == 0 && lo <= hi) { atomicMin(&mm[0], lo); atomicMax(&mm[1], hi); }
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

// distinct values per bucket (presence bitmap + popcount)
static __global__ void __launch_bounds__(kBkThreads)
bk_count_kernel(const uint32_t* __restrict__ buf, const uint32_t* __restrict__ starts,
                const uint32_t* __restrict__ n_valid, const uint32_t* __restrict__ par,
                uint32_t* __restrict__ distinct) {
  extern __shared__ __align__(16) uint32_t bk_smem[];
  __shared__ uint32_t ws[33];
  uint32_t* bm = bk_smem;
  const int b = blockIdx.x;
  const uint32_t s = starts[b], e = (b + 1 < kBkParts) ? starts[b + 1] : *n_valid;
  if (s >= e) { if (threadIdx.x == 0) distinct[b] = 0u; return; }
  const uint32_t shift = par[1];
  const uint32_t wmask = (1u << shift) - 1u;                // shift <= 19
  const int words = shift > 5 ? 1 << (shift - 5) : 1;
  for (int w = threadIdx.x; w < words; w += kBkThreads) bm[w] = 0u;
  __syncthreads();
  for (uint32_t i = s + threadIdx.x; i < e; i += kBkThreads) {
    const uint32_t off = buf[i] & wmask;
    const uint32_t bit = 1u << (off & 31);
    if (!(bm[off >> 5] & bit)) atomicOr(&bm[off >> 5], bit);
  }
  __syncthreads();
  uint32_t c = 0;
  for (int w = threadIdx.x; w < words; w += kBkThreads) c += __popc(bm[w]);
  const uint32_t tot = bk_block_sum(c, ws);
  if (threadIdx.x == 0) distinct[b] = tot;
}

// packed pairs of every bucket, in key order, at out[out_base[b] ...).  *flag is set when a
// bucket has more than kBkDupCap duplicated values (the caller then redoes the batch with the
// radix pipeline).
static __global__ void __launch_bounds__(kBkThreads)
bk_emit_kernel(const uint32_t* __restrict__ buf, const uint32_t* __restrict__ starts,
               const uint32_t* __restrict__ n_valid, const uint32_t* __restrict__ par,
               const uint32_t* __restrict__ out_base, uint64_t* __restrict__ out,
               unsigned int* __restrict__ flag, unsigned long long* __restrict__ max_count) {
  extern __shared__ __align__(16) uint32_t bk_smem[];
  __shared__ uint32_t ws[33];
  uint32_t* bm = bk_smem;                                   // presence
  uint32_t* dup = bm + kBkWords;                            // seen at least twice
  uint16_t* pfx = reinterpret_cast<uint16_t*>(dup + kBkWords);   // exclusive popcount prefix of dup
  uint32_t* cnt = reinterpret_cast<uint32_t*>(pfx + kBkWords);   // occurrences of the duplicated values
  const int b = blockIdx.x;
  const uint32_t s = starts[b], e = (b + 1 < kBkParts) ? starts[b + 1] : *n_valid;
  if (s >= e) return;
  const uint32_t lo = par[0], shift = par[1];
  const uint32_t wmask = (1u << shift) - 1u;
  const int words = shift > 5 ? 1 << (shift - 5) : 1;
  const int per = (words + kBkThreads - 1) / kBkThreads;    // consecutive words per thread
  for (int w = threadIdx.x; w < words; w += kBkThreads) { bm[w] = 0u; dup[w] = 0u; }
  __syncthreads();
  for (uint32_t i = s + threadIdx.x; i < e; i += kBkThreads) {
    const uint32_t off = buf[i] & wmask;
    const uint32_t bit = 1u << (off & 31), w = off >> 5;
    const uint32_t old = atomicOr(&bm[w], bit);
    if ((old & bit) && !(dup[w] & bit)) atomicOr(&dup[w], bit);
  }
  __syncthreads();
  // dense index of the duplicated values
  const int w0 = threadIdx.x * per;
  uint32_t c = 0;
  for (int j = 0; j < per; ++j) if (w0 + j < words) c += __popc(dup[w0 + j]);
  uint32_t n_dup;
  uint32_t run = bk_block_excl(c, ws, &n_dup);
  if (n_dup > (uint32_t)kBkDupCap) {
    if (threadIdx.x == 0) atomicOr(flag, 1u);
    return;
  }
  for (int j = 0; j < per; ++j)
    if (w0 + j < words) { pfx[w0 + j] = (uint16_t)run; run += __popc(dup[w0 + j]); }
  for (uint32_t i = threadIdx.x; i < n_dup; i += kBkThreads) cnt[i] = 0u;
  __syncthreads();
  if (n_dup) {
    for (uint32_t i = s + threadIdx.x; i < e; i += kBkThreads) {
      const uint32_t off = buf[i] & wmask;
      const uint32_t bit = 1u << (off & 31), w = off >> 5;
      const uint32_t d = dup[w];
      if (d & bit) atomicAdd(&cnt[pfx[w] + __popc(d & (bit - 1u))], 1u);
    }
    __syncthreads();
  }
  // emit in bitmap order = key order
  c = 0;
  for (int j = 0; j < per; ++j) if (w0 + j < words) c += __popc(bm[w0 + j]);
  uint32_t n_out;
  uint32_t r = bk_block_excl(c, ws, &n_out);
  uint64_t* o = out + out_base[b];
  const uint32_t vbase = lo + ((uint32_t)b << shift);      // u of the window's first value (no overflow: b << shift <= range)
  uint32_t mx = 1u;
  for (int j = 0; j < per; ++j) {
    const int w = w0 + j;
    if (w >= words) break;
    uint32_t bits = bm[w];
    const uint32_t d = dup[w];
    const uint32_t pd = pfx[w];
    while (bits) {
      const int k = __ffs(bits) - 1;
      bits &= bits - 1u;
      uint32_t n = 1u;
      if ((d >> k) & 1u) n = cnt[pd + __popc(d & ((1u << k) - 1u))];
      mx = n > mx ? n : mx;
      o[r++] = ((uint64_t)(vbase + ((uint32_t)w << 5) + (uint32_t)k) << 32) | (uint64_t)n;
    }
  }
#pragma unroll
  for (int o2 = 16; o2 > 0; o2 >>= 1) { const uint32_t y = __shfl_down_sync(0xFFFFFFFFu, mx, o2); mx = y > mx ? y : mx; }
  if ((threadIdx.x & 31) == 0) atomicMax(max_count, (unsigned long long)mx);
}

}  // namespace nvtb
