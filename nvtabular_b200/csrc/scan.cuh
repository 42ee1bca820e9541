// scan.cuh — the multi-CTA exclusive scan of int64 counts shared by the external-table join
// (join.cu, K9: the emit count of every left row) and the sub-list copy of the session ops
// (groupby.cu, nvtb_gb_list_rows: the length of every sub-list).
//
// In place over off[0..n): tile sums (2048 counts per CTA, 8 consecutive per lane), one CTA scans
// the tile sums, then every tile adds its base to its own exclusive scan; off[n] = the total.
// Three launches, O(n) reads and writes, and any n.  The kernels keep the join_ names they were
// written under, so join.cu compiles to the same SASS with or without the shared header.
#pragma once
#include "common.cuh"

namespace nvtb {
namespace {

constexpr int kScanTileThreads = 256;
constexpr int kScanTile = kScanTileThreads * kRows;    // 2048 counts per tile: 8 per lane
constexpr int kScanThreads = 1024;

template <int T>
__device__ __forceinline__ long long block_excl_scan_i64(long long v, long long* ws /*[T/32 + 1]*/, long long* total) {
  long long incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if ((threadIdx.x & 31) >= o) incl += y;
  }
  if ((threadIdx.x & 31) == 31) ws[threadIdx.x >> 5] = incl;
  __syncthreads();
  if (threadIdx.x < 32) {
    const long long w = threadIdx.x < T / 32 ? ws[threadIdx.x] : 0;
    long long wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xFFFFFFFFu, wi, o);
      if (threadIdx.x >= o) wi += y;
    }
    if (threadIdx.x < T / 32) ws[threadIdx.x] = wi - w;
    if (threadIdx.x == T / 32 - 1) ws[T / 32] = wi;
  }
  __syncthreads();
  const long long out = ws[threadIdx.x >> 5] + incl - v;
  *total = ws[T / 32];
  __syncthreads();
  return out;
}

__device__ __forceinline__ void load8_i64(const int64_t* __restrict__ p, int64_t i, int64_t n, int64_t (&v)[8]) {
  if (i + 8 <= n) {
    ld_rows8<int64_t>(p + i, v);
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = i + k < n ? p[i + k] : 0;
  }
}

__global__ void __launch_bounds__(kScanTileThreads)
join_tile_sums_kernel(const int64_t* __restrict__ counts, int64_t n, long long* __restrict__ tile_sum) {
  __shared__ long long ws[kScanTileThreads / 32 + 1];
  const int64_t i = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * 8;
  int64_t v[8];
  long long s = 0;
  if (i < n) {
    load8_i64(counts, i, n, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) s += v[k];
  }
  long long tot;
  block_excl_scan_i64<kScanTileThreads>(s, ws, &tot);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(kScanThreads)
join_tile_scan_kernel(long long* __restrict__ tile, int64_t ntiles, int64_t* __restrict__ off_end,
                      unsigned long long* __restrict__ total) {
  __shared__ long long ws[kScanThreads / 32 + 1];
  long long carry = 0;
  for (int64_t c0 = 0; c0 < ntiles; c0 += kScanThreads) {
    const int64_t i = c0 + threadIdx.x;
    const long long v = i < ntiles ? tile[i] : 0;
    long long tot;
    const long long ex = block_excl_scan_i64<kScanThreads>(v, ws, &tot);
    if (i < ntiles) tile[i] = carry + ex;
    carry += tot;
  }
  if (threadIdx.x == 0) { *off_end = carry; *total = (unsigned long long)carry; }
}

__global__ void __launch_bounds__(kScanTileThreads)
join_tile_apply_kernel(int64_t* __restrict__ off, int64_t n, const long long* __restrict__ tile_base) {
  __shared__ long long ws[kScanTileThreads / 32 + 1];
  const int64_t i = (int64_t)blockIdx.x * kScanTile + (int64_t)threadIdx.x * 8;
  int64_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  long long s = 0;
  if (i < n) {
    load8_i64(off, i, n, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) s += v[k];
  }
  long long tot;
  long long run = tile_base[blockIdx.x] + block_excl_scan_i64<kScanTileThreads>(s, ws, &tot);
  if (i >= n) return;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const long long c = v[k];
    v[k] = run;
    run += c;
  }
  if (i + 8 <= n) {
    st_rows8<int64_t>(off + i, v);
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) if (i + k < n) off[i + k] = v[k];
  }
}

// Exclusive scan of off[0..n) in place; off[n] and *total_host receive the total.  off must be
// 32-byte aligned and hold n + 1 int64.  Synchronises the stream.
inline int excl_scan_i64(int64_t* off, int64_t n, int64_t* total_host, cudaStream_t st) {
  const int64_t ntiles = (n + kScanTile - 1) / kScanTile;
  long long* tiles = nullptr;
  NVTB_CUDA_OK(cudaMallocAsync(&tiles, sizeof(long long) * (ntiles + 1), st));
  unsigned long long* total = reinterpret_cast<unsigned long long*>(tiles + ntiles);
  if (ntiles > 0) {
    join_tile_sums_kernel<<<(unsigned)ntiles, kScanTileThreads, 0, st>>>(off, n, tiles);
    NVTB_LAUNCH_OK();
  }
  join_tile_scan_kernel<<<1, kScanThreads, 0, st>>>(tiles, ntiles, off + n, total);
  NVTB_LAUNCH_OK();
  if (ntiles > 0) {
    join_tile_apply_kernel<<<(unsigned)ntiles, kScanTileThreads, 0, st>>>(off, n, tiles);
    NVTB_LAUNCH_OK();
  }
  unsigned long long h = 0;
  NVTB_CUDA_OK(cudaMemcpyAsync(&h, total, sizeof(h), cudaMemcpyDeviceToHost, st));
  NVTB_CUDA_OK(cudaFreeAsync(tiles, st));
  NVTB_CUDA_OK(cudaStreamSynchronize(st));
  *total_host = (int64_t)h;
  return NVTB_OK;
}

}  // namespace
}  // namespace nvtb
