// gather.cu — the row gather of Groupby and shuffle_by_keys (K8), JoinExternal (K9) and Filter /
// Dropna (K11), on sm_90a.
//
// Every lane owns 8 consecutive output rows, i.e. one validity byte of every output, so the
// bitmasks are written without atomics; it works out the 8 source rows once and moves them for
// up to 16 columns per launch.  Full groups of 8 are stored as whole sectors (st_rows8).
#include "common.cuh"

namespace nvtb {
namespace {

constexpr int kMaxGatherCols = 16;

struct GatherCols {
  const void* src[kMaxGatherCols];
  const uint8_t* src_valid[kMaxGatherCols];
  void* out[kMaxGatherCols];
  uint8_t* out_valid[kMaxGatherCols];
  int32_t size[kMaxGatherCols];
  uint32_t canon_zero;   // bit j: column j is a float key, -0.0 is written as +0.0
  int32_t ncols;
};

template <typename T>
__device__ __forceinline__ void gather8(const GatherCols& c, int j, const int64_t (&r)[8], int64_t i, int64_t m) {
  const T* __restrict__ src = static_cast<const T*>(c.src[j]);
  const uint8_t* __restrict__ sv = c.src_valid[j];
  const bool canon = sizeof(T) >= 4 && ((c.canon_zero >> j) & 1u);
  T v[8];
  unsigned vb = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const bool ok = r[k] >= 0;
    v[k] = ok ? src[r[k]] : (T)0;
    // -0.0 is the bit pattern of the sign alone
    if (canon && v[k] == ((T)1 << (8 * sizeof(T) - 1))) v[k] = 0;
    if (ok && valid1(sv, r[k])) vb |= 1u << k;
  }
  T* out = static_cast<T*>(c.out[j]);
  if (i + 8 <= m) {
    st_rows8<T>(out + i, v);
  } else {
#pragma unroll
    for (int k = 0; k < 8; ++k) if (i + k < m) out[i + k] = v[k];
  }
  if (c.out_valid[j] != nullptr) c.out_valid[j][i >> 3] = (uint8_t)vb;
}

// vec_pos: which 0 with pos 32-byte aligned, so the 8 positions of a full group are one sector
__global__ void __launch_bounds__(kThreads)
gather_rows_kernel(nvtb_row_sel_t s, int64_t m, bool vec_pos, GatherCols c) {
  const int64_t nchunks = (m + 7) / 8;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < nchunks; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = g * 8;
    int64_t r[8];
    if (vec_pos && i + 8 <= m) {
      ld_rows8<int64_t>(s.pos + i, r);
#pragma unroll
      for (int k = 0; k < 8; ++k) r[k] = (int64_t)((uint64_t)r[k] & s.row_mask);
    } else {
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int64_t o = i + k;
        if (o >= m) { r[k] = -1; continue; }
        const int64_t p = s.which == 0 ? o : (s.which == 1 ? s.off[o] : s.off[o + 1] - 1);
        r[k] = s.pos != nullptr ? (int64_t)((uint64_t)s.pos[p] & s.row_mask) : p;
      }
    }
    for (int j = 0; j < c.ncols; ++j) {
      switch (c.size[j]) {
        case 1: gather8<uint8_t>(c, j, r, i, m); break;
        case 4: gather8<uint32_t>(c, j, r, i, m); break;
        default: gather8<uint64_t>(c, j, r, i, m); break;
      }
    }
  }
}

}  // namespace
}  // namespace nvtb

using namespace nvtb;

extern "C" {

int nvtb_gather_rows(const nvtb_col_t* cols, int ncols, const nvtb_row_sel_t* sel, int64_t m, void* const* outs,
                     uint8_t* const* valids, uint32_t canon_zero, void* stream) {
  NVTB_REQUIRE(cols != nullptr && sel != nullptr && outs != nullptr && m >= 0, "NULL argument or m < 0");
  NVTB_REQUIRE(ncols >= 1 && ncols <= kMaxGatherCols, "ncols must be in [1, 16]");
  NVTB_REQUIRE(sel->which >= 0 && sel->which <= 2, "which must be 0, 1 or 2");
  if (m == 0) return NVTB_OK;
  NVTB_REQUIRE(sel->which == 0 || sel->off != nullptr, "segment ends need offsets");
  GatherCols c;
  memset(&c, 0, sizeof(c));
  c.ncols = ncols;
  c.canon_zero = canon_zero;
  for (int k = 0; k < ncols; ++k) {
    const int sz = (int)dtype_size(cols[k].dtype);
    NVTB_REQUIRE(sz == 1 || sz == 4 || sz == 8, "unsupported column dtype");
    NVTB_REQUIRE(cols[k].data != nullptr && outs[k] != nullptr, "NULL column data / output");
    NVTB_REQUIRE(sz == 1 ? (reinterpret_cast<uintptr_t>(outs[k]) & 7u) == 0 : is_aligned32(outs[k]),
                 "outputs must be 32-byte aligned (uint8: 8-byte)");
    c.src[k] = cols[k].data;
    c.src_valid[k] = cols[k].validity;
    c.out[k] = outs[k];
    c.out_valid[k] = valids != nullptr ? valids[k] : nullptr;
    c.size[k] = sz;
  }
  const bool vec_pos = sel->which == 0 && sel->pos != nullptr && is_aligned32(sel->pos);
  gather_rows_kernel<<<plain_grid((m + 7) / 8), kThreads, 0, (cudaStream_t)stream>>>(*sel, m, vec_pos, c);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

}  // extern "C"
