// join.cu — K9: the external-table join of the JoinExternal operator, on sm_90a.
//
// Replaces, per partition, reference nvtabular/ops/join_external.py:148-164:
//   df[tmp] = arange(len(df)); df.merge(ext, left_on=on, right_on=on_ext, how=how)
//   .sort_values(tmp)
// i.e. a hash join followed by an O(n log n) sort back to row order.  Here the rows never leave
// left-row order, so there is no sort:
//   build   (once per operator, O(|ext|)) the ext rows are ordered by key with the stable K8
//           primitives (groupby.cu), so each distinct key is a run of ext rows in ext order; this
//           file keeps the runs (off), the ordered rows and a wide Lookup key -> run (lookup.cuh)
//   probe   one pass over the left key column: the first ext row of the key's run (or -1) and,
//           unless every key is unique and the join is a left join, the row's emit count,
//           scanned into int64 output offsets
//   expand  (duplicated keys / inner joins) per output row, its left row and ext row; balanced
//           over OUTPUT rows, so one key with 10^6 matches does not serialise on one thread
// The columns are then gathered at those rows by gather.cu (-1 = null).
// Int32 holds every count and group id: the ext table has fewer than 2^31 rows.
#include <cstring>
#include <new>

#include "common.cuh"
#include "lookup.cuh"

namespace nvtb {
namespace {

constexpr int kJoinThreads = 256;

// ---------------------------------------------------------------------------------------
// build: a wide table key -> run index g (keys are distinct: they come out of K8 segments)
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kJoinThreads)
join_table_init_kernel(int64_t* slots, int64_t capacity) {
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < capacity; s += (int64_t)gridDim.x * blockDim.x) {
    slots[2 * s] = kEmptyKey;
    slots[2 * s + 1] = INT64_MAX;
  }
}

// scal[0]: run index of the key INT64_MIN (the empty sentinel, which the table cannot hold) or -1;
// scal[1]: the longest run
__global__ void __launch_bounds__(kJoinThreads)
join_table_build_kernel(const int64_t* __restrict__ keys, const int64_t* __restrict__ off, int64_t n_groups,
                        int64_t* slots, int64_t capacity, long long* scal) {
  long long longest = 0;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < n_groups; g += (int64_t)gridDim.x * blockDim.x) {
    const long long k = keys[g];
    if (k == kEmptyKey) scal[0] = g;
    else wide_claim(slots, capacity, k, (long long)g);
    const long long len = off[g + 1] - off[g];
    longest = len > longest ? len : longest;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const long long y = __shfl_xor_sync(0xFFFFFFFFu, longest, o);
    longest = y > longest ? y : longest;
  }
  if ((threadIdx.x & 31) == 0 && longest) atomicMax(scal + 1, longest);
}

}  // namespace
}  // namespace nvtb

// Included after the build kernels, not at the top: the kernels are then emitted in the same
// order as when the scan lived in this file, and the file's SASS is byte-identical to that.
#include "scan.cuh"

namespace nvtb {
namespace {

// ---------------------------------------------------------------------------------------
// probe
// ---------------------------------------------------------------------------------------
// A null key joins the null run [null_lo, null_hi) (pandas and cuDF match null with null).
// counts == nullptr (left join on unique keys): ext_out[i] = the matching ext row or -1.
// Otherwise ext_out[i] = the position of the first match in key order (or -1) and counts[i] =
// the rows row i emits: its match count, at least 1 in a left join.
template <typename K>
__global__ void __launch_bounds__(kJoinThreads)
join_probe_kernel(const K* __restrict__ keys, const uint8_t* __restrict__ mask, int64_t n, Lookup t,
                  const int64_t* __restrict__ off, const int64_t* __restrict__ rows, int64_t null_lo,
                  int64_t null_hi, int left, int64_t* __restrict__ ext_out, int64_t* __restrict__ counts) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t pos = -1, cnt = 0;
    if (valid1(mask, i)) {
      const int64_t g = lookup_find(t, (int64_t)keys[i]);
      if (g >= 0) {
        pos = __ldg(off + g);
        cnt = __ldg(off + g + 1) - pos;
      }
    } else if (null_hi > null_lo) {
      pos = null_lo;
      cnt = null_hi - null_lo;
    }
    if (counts != nullptr) {
      ext_out[i] = pos;
      counts[i] = left && cnt == 0 ? 1 : cnt;
    } else {
      ext_out[i] = pos >= 0 ? __ldg(rows + pos) : -1;
    }
  }
}

// ---------------------------------------------------------------------------------------
// expand: every lane owns 8 consecutive output rows.  Two binary searches over off bound the left
// rows its outputs come from; each output then searches only that bracket.  The work per output
// row is the same whatever the match counts, so a key with 10^6 matches spreads over the grid.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ int64_t last_le(const int64_t* __restrict__ off, int64_t lo, int64_t hi, int64_t p) {
  // last i in [lo, hi) with off[i] <= p (off[lo] <= p is given)
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (__ldg(off + mid) <= p) lo = mid; else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(kJoinThreads)
join_expand_kernel(const int64_t* __restrict__ first, const int64_t* __restrict__ off, int64_t n, int64_t n_out,
                   const int64_t* __restrict__ rows, int64_t* __restrict__ left_rows, int64_t* __restrict__ ext_rows) {
  const int64_t nchunks = (n_out + 7) / 8;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < nchunks; c += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p0 = c * 8;
    const int64_t pe = p0 + 7 < n_out ? p0 + 7 : n_out - 1;
    const int64_t i0 = last_le(off, 0, n, p0);
    const int64_t i1 = last_le(off, i0, n, pe);
    int64_t lr[8], er[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int64_t p = p0 + k <= pe ? p0 + k : pe;
      const int64_t i = last_le(off, i0, i1 + 1, p);
      const int64_t f = __ldg(first + i);
      lr[k] = i;
      er[k] = f < 0 ? -1 : __ldg(rows + f + (p - __ldg(off + i)));
    }
    if (p0 + 8 <= n_out) {
      st_rows8<int64_t>(left_rows + p0, lr);
      st_rows8<int64_t>(ext_rows + p0, er);
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k)
        if (p0 + k < n_out) { left_rows[p0 + k] = lr[k]; ext_rows[p0 + k] = er[k]; }
    }
  }
}

}  // namespace
}  // namespace nvtb

struct nvtb_join {
  nvtb::Lookup t;
  int64_t* off;      // device [n_groups + 1]: run g is positions [off[g], off[g + 1])
  int64_t* rows;     // device [n_ext]: ext rows in key order (stable: ext order within a key)
  int64_t n_groups;
  int64_t n_ext;
  int64_t null_lo;   // the null-key run [null_lo, null_hi) of `rows`
  int64_t null_hi;
  int64_t max_group;
};

using namespace nvtb;

extern "C" {

int nvtb_join_create(nvtb_join_t** out, const int64_t* distinct_keys, int64_t n_groups, const int64_t* off,
                     const int64_t* ordered_rows, int64_t n_ext, int64_t null_lo, int64_t null_hi, void* stream) {
  NVTB_REQUIRE(out != nullptr && n_groups >= 0 && n_ext >= 0, "bad arguments");
  NVTB_REQUIRE(n_ext < ((int64_t)1 << 31), "the external table must have fewer than 2^31 rows");
  NVTB_REQUIRE(n_groups <= n_ext && 0 <= null_lo && null_lo <= null_hi && null_hi <= n_ext, "bad run bounds");
  NVTB_REQUIRE(n_groups == 0 || (distinct_keys && off), "NULL keys / offsets");
  NVTB_REQUIRE(n_ext == 0 || ordered_rows, "NULL ordered rows");
  cudaStream_t st = (cudaStream_t)stream;
  nvtb_join* j = new (std::nothrow) nvtb_join();
  NVTB_REQUIRE(j != nullptr, "host allocation failed");
  memset(j, 0, sizeof(*j));
  j->n_groups = n_groups; j->n_ext = n_ext; j->null_lo = null_lo; j->null_hi = null_hi;
  j->t.capacity = 16;
  while (j->t.capacity < 2 * n_groups) j->t.capacity <<= 1;
  j->t.min_key_pos = -1;
  j->t.narrow = 0;
  long long* scal = nullptr;
  long long h[2] = {-1, 0};
  int rc = NVTB_ECUDA;
  do {
    if (cudaMallocAsync(&j->off, sizeof(int64_t) * (n_groups + 1), st) != cudaSuccess) break;
    if (cudaMallocAsync(&j->rows, sizeof(int64_t) * (n_ext > 0 ? n_ext : 1), st) != cudaSuccess) break;
    if (cudaMallocAsync(&j->t.slots, sizeof(int64_t) * 2 * j->t.capacity, st) != cudaSuccess) break;
    if (cudaMallocAsync(&scal, sizeof(h), st) != cudaSuccess) break;
    if (cudaMemcpyAsync(scal, h, sizeof(h), cudaMemcpyHostToDevice, st) != cudaSuccess) break;
    if (n_groups > 0 && cudaMemcpyAsync(j->off, off, sizeof(int64_t) * (n_groups + 1), cudaMemcpyDeviceToDevice, st) != cudaSuccess) break;
    if (n_ext > 0 && cudaMemcpyAsync(j->rows, ordered_rows, sizeof(int64_t) * n_ext, cudaMemcpyDeviceToDevice, st) != cudaSuccess) break;
    join_table_init_kernel<<<plain_grid(j->t.capacity), kJoinThreads, 0, st>>>(j->t.slots, j->t.capacity);
    if (n_groups > 0)
      join_table_build_kernel<<<plain_grid(n_groups), kJoinThreads, 0, st>>>(distinct_keys, off, n_groups, j->t.slots,
                                                                             j->t.capacity, scal);
    if (cudaGetLastError() != cudaSuccess) break;
    if (cudaMemcpyAsync(h, scal, sizeof(h), cudaMemcpyDeviceToHost, st) != cudaSuccess) break;
    if (cudaFreeAsync(scal, st) != cudaSuccess) break;
    scal = nullptr;
    if (cudaStreamSynchronize(st) != cudaSuccess) break;
    rc = NVTB_OK;
  } while (false);
  if (rc != NVTB_OK) {
    set_error("nvtb_join_create: %s", cudaGetErrorString(cudaGetLastError()));
    if (scal) cudaFreeAsync(scal, st);
    nvtb_join_destroy(j);
    return rc;
  }
  j->t.min_key_pos = h[0];
  j->max_group = h[1] > null_hi - null_lo ? h[1] : null_hi - null_lo;
  *out = j;
  return NVTB_OK;
}

int nvtb_join_info(const nvtb_join_t* j, int64_t* n_groups, int64_t* max_group) {
  NVTB_REQUIRE(j != nullptr && n_groups != nullptr && max_group != nullptr, "NULL argument");
  *n_groups = j->n_groups;
  *max_group = j->max_group;
  return NVTB_OK;
}

int nvtb_join_destroy(nvtb_join_t* j) {
  if (j == nullptr) return NVTB_OK;
  if (j->t.slots) cudaFreeAsync(j->t.slots, 0);
  if (j->off) cudaFreeAsync(j->off, 0);
  if (j->rows) cudaFreeAsync(j->rows, 0);
  delete j;
  return NVTB_OK;
}

int nvtb_join_probe(const nvtb_join_t* j, const nvtb_col_t* key, int64_t n, int how, int64_t* ext_row_out,
                    int64_t* off_out, int64_t* n_out_host, void* stream) {
  NVTB_REQUIRE(j != nullptr && key != nullptr && n >= 0 && n_out_host != nullptr, "NULL argument or n < 0");
  NVTB_REQUIRE(how == 0 || how == 1, "how must be 0 (left) or 1 (inner)");
  NVTB_REQUIRE(key->dtype == NVTB_I32 || key->dtype == NVTB_I64, "key dtype must be int32 or int64");
  NVTB_REQUIRE(off_out == nullptr || is_aligned32(off_out), "off_out must be 32-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  *n_out_host = off_out == nullptr ? n : 0;
  if (off_out == nullptr && n == 0) return NVTB_OK;
  if (n > 0) {
    NVTB_REQUIRE(key->data != nullptr && ext_row_out != nullptr, "NULL key data / ext_row_out");
    const int grid = plain_grid(n);
    const int left = how == 0;
    if (key->dtype == NVTB_I32)
      join_probe_kernel<int32_t><<<grid, kJoinThreads, 0, st>>>((const int32_t*)key->data, key->validity, n, j->t, j->off,
                                                                j->rows, j->null_lo, j->null_hi, left, ext_row_out, off_out);
    else
      join_probe_kernel<int64_t><<<grid, kJoinThreads, 0, st>>>((const int64_t*)key->data, key->validity, n, j->t, j->off,
                                                                j->rows, j->null_lo, j->null_hi, left, ext_row_out, off_out);
    NVTB_LAUNCH_OK();
  }
  if (off_out == nullptr) return NVTB_OK;
  return excl_scan_i64(off_out, n, n_out_host, st);
}

int nvtb_join_expand(const nvtb_join_t* j, const int64_t* ext_row_first, const int64_t* off, int64_t n, int64_t n_out,
                     int64_t* left_rows, int64_t* ext_rows, void* stream) {
  NVTB_REQUIRE(j != nullptr && n >= 0 && n_out >= 0, "bad arguments");
  if (n_out == 0) return NVTB_OK;
  NVTB_REQUIRE(n > 0 && ext_row_first && off && left_rows && ext_rows, "NULL buffers");
  NVTB_REQUIRE(is_aligned32(left_rows) && is_aligned32(ext_rows), "outputs must be 32-byte aligned");
  join_expand_kernel<<<plain_grid((n_out + 7) / 8), kJoinThreads, 0, (cudaStream_t)stream>>>(
      ext_row_first, off, n, n_out, j->rows, left_rows, ext_rows);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

}  // extern "C"
