// partition.cuh — order-free partition of the valid keys of an int32 column (hist -> scan ->
// scatter staged through shared memory), used with PartHashTop by the hash table's shared-memory
// fold (fold_i32.cuh), with PartKeyLow by the radix route (sortagg.cuh) and with PartRange by the
// bucket route (bucketagg.cuh) of the sorted accumulator.  Included after hashagg.cuh.
#pragma once

namespace nvtb {

constexpr int kPartThreads = 512;
constexpr int kPartGroups = 4;                                   // 8-row groups per thread per tile
constexpr int kPartTile = kPartThreads * 8 * kPartGroups;        // 16384 rows
constexpr int kMaxParts = 4096;

// rows [i, i+8) of an int32 column as one lane's group: values, valid bits, in-range bits
struct Rows8 { int32_t v[8]; unsigned m; unsigned lv; };

__device__ __forceinline__ void load_rows8(const int32_t* __restrict__ keys,
                                           const uint8_t* __restrict__ mask, int64_t i,
                                           int64_t end, Rows8& r, bool aligned = true) {
  if (i + 8 <= end && aligned) {
    ld_rows8<int32_t>(keys + i, r.v);
    r.lv = 0xFFu;
    r.m = valid8(mask, i);
  } else if (i < end) {
    r.lv = (end - i >= 8) ? 0xFFu : ((1u << (unsigned)(end - i)) - 1u);
    r.m = valid8(mask, i) & r.lv;
#pragma unroll
    for (int k = 0; k < 8; ++k) r.v[k] = (i + k < end) ? keys[i + k] : 0;
  } else {
    r.lv = 0u; r.m = 0u;
#pragma unroll
    for (int k = 0; k < 8; ++k) r.v[k] = 0;
  }
}

// What a key becomes in the partition buffer, and which partition it goes to:
//   PartHashTop  h = fold_hash(key), partition = top lg bits of h   (shared-memory fold)
//   PartKeyLow   u = key ^ 2^31 (unsigned order == signed order), partition = LOW lg bits
//                of u: the first, order-free pass of the LSD radix sort of sortagg.cuh
struct PartHashTop {
  int lg;
  __device__ __forceinline__ uint32_t xform(uint32_t k) const { return fold_hash(k); }
  __device__ __forceinline__ uint32_t bin(uint32_t v) const { return v >> (32 - lg); }
};
struct PartKeyLow {
  int lg;
  __device__ __forceinline__ uint32_t xform(uint32_t k) const { return k ^ 0x80000000u; }
  __device__ __forceinline__ uint32_t bin(uint32_t v) const { return v & ((1u << lg) - 1u); }
};

// (1) partition sizes; the nulls are counted here and dropped by the scatter
template <typename Pol>
__global__ void __launch_bounds__(kPartThreads)
part_hist_kernel(const int32_t* __restrict__ keys, const uint8_t* __restrict__ mask, int64_t n,
                 Pol pol, uint32_t* __restrict__ total, Counters* ctr, int aligned) {
  const int lg = pol.lg;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  uint32_t* cnt = reinterpret_cast<uint32_t*>(smem_raw);
  const int P = 1 << lg;
  for (int d = threadIdx.x; d < P; d += kPartThreads) cnt[d] = 0u;
  __shared__ unsigned int s_null;
  if (threadIdx.x == 0) s_null = 0u;
  __syncthreads();
  unsigned n_null = 0;
  const int64_t n_tiles = (n + kPartTile - 1) / kPartTile;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    Rows8 r[kPartGroups];
#pragma unroll
    for (int g = 0; g < kPartGroups; ++g)
      load_rows8(keys, mask, tile * kPartTile + ((int64_t)g * kPartThreads + threadIdx.x) * 8, n, r[g], aligned != 0);
#pragma unroll
    for (int g = 0; g < kPartGroups; ++g) {
      n_null += __popc(r[g].lv & ~r[g].m);
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if ((r[g].m >> k) & 1u) atomicAdd(&cnt[pol.bin(pol.xform((uint32_t)r[g].v[k]))], 1u);
    }
  }
  if (n_null) atomicAdd(&s_null, n_null);
  __syncthreads();
  for (int d = threadIdx.x; d < P; d += kPartThreads)
    if (cnt[d]) atomicAdd(&total[d], cnt[d]);
  if (threadIdx.x == 0 && s_null && ctr != nullptr) atomicAdd(&ctr->size[0], (unsigned long long)s_null);
}

// exclusive scan of `vals[0..P)` held in shared memory, P % T == 0; every value is first
// rounded up to a multiple of `round` (1 = none).  Result in out[0..P); returns nothing.
template <int T>
__device__ __forceinline__ void block_excl_scan(const uint32_t* vals, uint32_t* out, int P,
                                                uint32_t round, uint32_t* warp_sums /*[T/32]*/) {
  const int per = P / T;
  uint32_t local = 0;
  for (int j = 0; j < per; ++j) {
    const uint32_t v = vals[threadIdx.x * per + j];
    local += (v + round - 1) / round * round;
  }
  uint32_t incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if ((threadIdx.x & 31) >= o) incl += y;
  }
  if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = incl;
  __syncthreads();
  if (threadIdx.x < 32) {
    uint32_t w = threadIdx.x < T / 32 ? warp_sums[threadIdx.x] : 0u;
    uint32_t wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, wi, o);
      if (threadIdx.x >= o) wi += y;
    }
    if (threadIdx.x < T / 32) warp_sums[threadIdx.x] = wi - w;
  }
  __syncthreads();
  uint32_t run = warp_sums[threadIdx.x >> 5] + incl - local;
  for (int j = 0; j < per; ++j) {
    const uint32_t v = vals[threadIdx.x * per + j];
    out[threadIdx.x * per + j] = run;
    run += (v + round - 1) / round * round;
  }
  __syncthreads();
}

// (2) partition starts (rounded up to multiples of `round` rows: 8 rows = 32 bytes for the
// fold kernel's 256-bit loads, 1 = dense for the radix sort), write cursors = starts;
// n_total (may be NULL) receives the end of the last partition
static __global__ void __launch_bounds__(kPartThreads)
part_scan_kernel(const uint32_t* __restrict__ total, int lg, uint32_t* __restrict__ starts,
                 uint32_t* __restrict__ cursor, uint32_t round, uint32_t* __restrict__ n_total) {
  __shared__ uint32_t v[kMaxParts];
  __shared__ uint32_t o[kMaxParts];
  __shared__ uint32_t ws[kPartThreads / 32];
  const int P = 1 << lg;
  for (int d = threadIdx.x; d < P; d += kPartThreads) v[d] = total[d];
  __syncthreads();
  block_excl_scan<kPartThreads>(v, o, P, round, ws);
  for (int d = threadIdx.x; d < P; d += kPartThreads) { starts[d] = o[d]; cursor[d] = o[d]; }
  if (n_total != nullptr && threadIdx.x == 0) *n_total = o[P - 1] + (v[P - 1] + round - 1) / round * round;
}

// (3) scatter (the buffer receives pol.xform(key): h = fold_hash(key), which the fold kernel
// consumes as is, or the biased key).  Per tile of 16 384 rows: count per partition (shared RED),
// reserve the tile's run in every partition with ONE global atomic per non-empty (tile, partition),
// bin the keys in shared memory, then copy the staged tile out so that consecutive lanes
// write consecutive words of a run.  Order inside a partition is irrelevant (counting).
template <typename Pol>
__global__ void __launch_bounds__(kPartThreads, 2)
part_scatter_kernel(const int32_t* __restrict__ keys, const uint8_t* __restrict__ mask, int64_t n,
                    Pol pol, uint32_t* __restrict__ cursor, int32_t* __restrict__ out, int aligned) {
  const int lg = pol.lg;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int32_t* stage = reinterpret_cast<int32_t*>(smem_raw);                 // [kPartTile]
  uint32_t* cnt = reinterpret_cast<uint32_t*>(stage + kPartTile);        // [P] counts, then running cursors
  uint32_t* delta = cnt + (1 << lg);                                     // [P] global start - staged start
  __shared__ uint32_t ws[kPartThreads / 32];
  __shared__ uint32_t s_total;
  const int P = 1 << lg;
  const int64_t n_tiles = (n + kPartTile - 1) / kPartTile;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    for (int d = threadIdx.x; d < P; d += kPartThreads) cnt[d] = 0u;
    __syncthreads();
    Rows8 r[kPartGroups];
#pragma unroll
    for (int g = 0; g < kPartGroups; ++g)
      load_rows8(keys, mask, tile * kPartTile + ((int64_t)g * kPartThreads + threadIdx.x) * 8, n, r[g], aligned != 0);
#pragma unroll
    for (int g = 0; g < kPartGroups; ++g)
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        r[g].v[k] = (int32_t)pol.xform((uint32_t)r[g].v[k]);      // the buffer holds hashes / biased keys
        if ((r[g].m >> k) & 1u) atomicAdd(&cnt[pol.bin((uint32_t)r[g].v[k])], 1u);
      }
    __syncthreads();
    // staged offsets (exclusive scan of the counts, in place via `delta` as scratch)
    block_excl_scan<kPartThreads>(cnt, delta, P, 1u, ws);
    for (int d = threadIdx.x; d < P; d += kPartThreads) {
      const uint32_t c = cnt[d], off = delta[d];
      uint32_t g0 = 0;
      if (c) g0 = atomicAdd(&cursor[d], c);
      delta[d] = g0 - off;            // modulo 2^32: global index = delta + staged index
      cnt[d] = off;                   // running staged cursor
      if (d == P - 1) s_total = off + c;
    }
    __syncthreads();
#pragma unroll
    for (int g = 0; g < kPartGroups; ++g)
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if ((r[g].m >> k) & 1u) {
          const uint32_t p = atomicAdd(&cnt[pol.bin((uint32_t)r[g].v[k])], 1u);
          stage[p] = r[g].v[k];
        }
    __syncthreads();
    const uint32_t total = s_total;
    for (uint32_t j = threadIdx.x; j < total; j += kPartThreads) {
      const int32_t hv = stage[j];
      out[delta[pol.bin((uint32_t)hv)] + j] = hv;
    }
    __syncthreads();
  }
}

}  // namespace nvtb
