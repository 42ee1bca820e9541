// exchange.cu — the cross-GPU owner exchange of the hash-table columns (nvtabular_b200/dist.py:
// global_merge, global_merge_many): every rank groups its exported (key, size [, payload]) rows
// by owner = mix(key) % W, so that one all-to-all hands each owner all partials of its keys.
//
// Stands in for the reference's split_out shuffle_group (nvtabular/ops/categorify.py:1036-1049).
// The owner is a pure function of the key; the row order inside an owner's segment is not.
#include "common.cuh"

namespace nvtb {

__device__ __forceinline__ int owner_of(int64_t key, int n_parts) {
  // bits disjoint from both the global and the smem slot bits
  return (int)((table_mix64((uint64_t)key) >> 52) % (uint64_t)n_parts);
}

__global__ void __launch_bounds__(kThreads)
owner_count_kernel(const int64_t* __restrict__ keys, int64_t n, int n_parts,
                   unsigned long long* counts) {
  __shared__ unsigned int sc[64];
  if (threadIdx.x < 64) sc[threadIdx.x] = 0;
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    atomicAdd(&sc[owner_of(keys[i], n_parts)], 1u);
  __syncthreads();
  if (threadIdx.x < n_parts && sc[threadIdx.x])
    atomicAdd(&counts[threadIdx.x], (unsigned long long)sc[threadIdx.x]);
}

// exclusive prefix of the per-owner counts -> write cursors (n_parts <= 64: one thread)
__global__ void owner_prefix_kernel(const unsigned long long* __restrict__ counts, int n_parts,
                                    unsigned long long* __restrict__ cursors) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    unsigned long long acc = 0;
    for (int p = 0; p < n_parts; ++p) { cursors[p] = acc; acc += counts[p]; }
  }
}

// scatter pass: each CTA ranks its chunk of rows per owner in shared memory and reserves
// ONE contiguous range per owner with a single global atomic, instead of one global
// atomic per row on only `n_parts` addresses (which serialised at ~1 row/ns).
__global__ void __launch_bounds__(kThreads)
owner_scatter_kernel(const int64_t* __restrict__ keys, int64_t n, int n_parts,
                     unsigned long long* cursors, int64_t* __restrict__ perm) {
  constexpr int kPer = 8;                       // rows per thread per chunk
  __shared__ unsigned int s_cnt[64];
  __shared__ unsigned long long s_base[64];
  const int64_t chunk = (int64_t)kThreads * kPer;
  const int64_t n_chunks = (n + chunk - 1) / chunk;
  for (int64_t c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    if (threadIdx.x < 64) s_cnt[threadIdx.x] = 0u;
    __syncthreads();
    int own[kPer];
    unsigned rank[kPer];
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int64_t i = c * chunk + (int64_t)j * kThreads + threadIdx.x;
      own[j] = -1;
      if (i < n) {
        own[j] = owner_of(keys[i], n_parts);
        rank[j] = atomicAdd(&s_cnt[own[j]], 1u);
      }
    }
    __syncthreads();
    if (threadIdx.x < n_parts && s_cnt[threadIdx.x])
      s_base[threadIdx.x] = atomicAdd(&cursors[threadIdx.x], (unsigned long long)s_cnt[threadIdx.x]);
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
      const int64_t i = c * chunk + (int64_t)j * kThreads + threadIdx.x;
      if (own[j] >= 0) perm[s_base[own[j]] + rank[j]] = i;
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kThreads)
gather_i64_kernel(const int64_t* __restrict__ src, const int64_t* __restrict__ perm,
                  int64_t n, int64_t* __restrict__ dst) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    dst[i] = src[perm[i]];
}

__global__ void __launch_bounds__(kThreads)
gather_f64_rows_kernel(const double* __restrict__ src, const int64_t* __restrict__ perm,
                       int64_t n, int w, double* __restrict__ dst) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t total = n * w;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
    const int64_t r = i / w, c = i - r * w;
    dst[i] = src[perm[r] * w + c];
  }
}

}  // namespace nvtb

using namespace nvtb;

extern "C" {

int nvtb_partition_by_owner_async(const int64_t* keys, int64_t n, int n_parts,
                                  int64_t* perm_out, int64_t* part_counts_dev, void* stream) {
  NVTB_REQUIRE(n >= 0 && n_parts >= 1 && n_parts <= 64, "n_parts must be in [1, 64]");
  NVTB_REQUIRE(part_counts_dev != nullptr, "part_counts_dev is NULL");
  cudaStream_t st = (cudaStream_t)stream;
  NVTB_CUDA_OK(cudaMemsetAsync(part_counts_dev, 0, sizeof(int64_t) * n_parts, st));
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(keys != nullptr && perm_out != nullptr, "NULL keys/perm");
  unsigned long long* d = nullptr;     // [64] write cursors
  NVTB_CUDA_OK(cudaMallocAsync(&d, sizeof(unsigned long long) * 64, st));
  const int grid = plain_grid(n);
  owner_count_kernel<<<grid, kThreads, 0, st>>>(keys, n, n_parts, reinterpret_cast<unsigned long long*>(part_counts_dev));
  NVTB_LAUNCH_OK();
  owner_prefix_kernel<<<1, 32, 0, st>>>(reinterpret_cast<const unsigned long long*>(part_counts_dev), n_parts, d);
  NVTB_LAUNCH_OK();
  owner_scatter_kernel<<<grid, kThreads, 0, st>>>(keys, n, n_parts, d, perm_out);
  NVTB_LAUNCH_OK();
  NVTB_CUDA_OK(cudaFreeAsync(d, st));
  return NVTB_OK;
}

int nvtb_gather_i64(const int64_t* src, const int64_t* perm, int64_t n, int64_t* dst, void* stream) {
  NVTB_REQUIRE(n >= 0, "n < 0");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(src && perm && dst, "NULL pointer");
  gather_i64_kernel<<<plain_grid(n), kThreads, 0, (cudaStream_t)stream>>>(src, perm, n, dst);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

int nvtb_gather_f64_rows(const double* src, const int64_t* perm, int64_t n, int row_width,
                         double* dst, void* stream) {
  NVTB_REQUIRE(n >= 0 && row_width >= 1, "bad n/row_width");
  if (n == 0) return NVTB_OK;
  NVTB_REQUIRE(src && perm && dst, "NULL pointer");
  gather_f64_rows_kernel<<<plain_grid(n * row_width), kThreads, 0, (cudaStream_t)stream>>>(src, perm, n, row_width, dst);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

}  // extern "C"
