// sortacc.cu — K3 for HIGH-CARDINALITY int32 key columns: the sorted accumulator a group-by handle
// becomes when its hash table would leave the L2 (hashagg.cu), and the packed-pair primitives of
// the cross-GPU vocabulary merge (nvtabular_b200/dist.py).  Staged batches are grouped by the
// bucket route (bucketagg.cuh) or, when a bucket holds too many duplicated values or
// NVTB_SORT_PATH=radix asks for it, the radix route (sortagg.cuh), then merged in.
#include <algorithm>
#include <new>

#include "hashagg.cuh"
#include "partition.cuh"
#include "sortagg.cuh"
#include "bucketagg.cuh"

namespace nvtb {

struct SortedAcc {
  uint64_t* acc[2] = {nullptr, nullptr};   // acc[cur] holds the u pairs, the other one takes the next merge
  int64_t acc_cap[2] = {0, 0};
  int cur = 0;
  // device uint32[8] of the batch being grouped: [1] valid keys, [2] distinct keys, [3] the most
  // rows of a bucket, [4] min and [5] max of u = key ^ 2^31 over the valid keys (folded by the
  // staging copies), [6] lo, [7] shift of the bucket partition.  [2, 8) is read back in one copy.
  uint32_t* d_n = nullptr;
  // staging: batches are only COPIED (keys + validity bytes) until NVTB_STAGE_ROWS rows are
  // waiting or somebody reads the handle; one group-by + merge then takes all of them (a merge
  // per batch re-reads and re-writes the whole accumulator, so its cost grows with every batch)
  int32_t* stage_keys = nullptr;
  uint8_t* stage_mask = nullptr;
  int64_t stage_cap = 0;     // rows
  int64_t stage_rows = 0;    // rows waiting (a multiple of 8 except after the last batch)
  int64_t stage_hint = 0;    // rows the previous fits staged: the buffer grows to hold one whole fit
  cudaEvent_t stage_ev = nullptr;
  cudaStream_t stage_last = nullptr;
};

static SharedScratch g_sort;      // the group-by routes and the merges

struct SortCarve {
  void* rx;                  // radix scratch; its first 256 B are kept at zero
  size_t rx_bytes;
  uint32_t* part_meta;       // total[P] | starts[P] | cursor[P]
  uint32_t* keys_a;
  uint32_t* keys_b;
  uint64_t* rle;             // [m + 1]
  uint32_t* tile_heads;      // [ceil(m / kRleTile)]
  uint2* splits;             // [MT + 1]
  uint32_t* tile_out;        // [MT]
};

static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

static int sort_scratch_acquire(int64_t m, int64_t n_pairs_sort, int64_t mt, cudaStream_t st, SortCarve* c) {
  const int P = 1 << kSortLowBits;
  const size_t rx_bytes = align_up(std::max(rx_scratch_bytes<uint32_t>(m), rx_scratch_bytes<uint64_t>(n_pairs_sort)), 256);
  // radix path: total[P] | starts[P] | cursor[P]; bucket path (bucketagg.cuh): the same three with
  // 8192 entries + distinct[8192] + {min, max, lo, shift, flag}
  const size_t meta_bytes = align_up(sizeof(uint32_t) * (size_t)std::max(3 * P, 4 * kBkParts + 64), 256);
  const size_t keys_bytes = align_up(sizeof(uint32_t) * (size_t)(m + 64), 256);
  const size_t rle_bytes = align_up(sizeof(uint64_t) * (size_t)(m + 2), 256);
  const size_t heads_bytes = align_up(sizeof(uint32_t) * (size_t)((m + kRleTile - 1) / kRleTile + 1), 256);
  const size_t splits_bytes = align_up(sizeof(uint2) * (size_t)(mt + 2), 256);
  const size_t out_bytes = align_up(sizeof(uint32_t) * (size_t)(mt + 2), 256);
  const size_t need = rx_bytes + meta_bytes + 2 * keys_bytes + rle_bytes + heads_bytes + splits_bytes + out_bytes;
  void* base = nullptr;
  bool grown = false;
  int rc = g_sort.acquire(need, need + need / 8, st, &base, &grown);
  if (rc) return rc;
  if (grown) NVTB_CUDA_OK(cudaMemsetAsync(base, 0, 256, st));
  char* p = reinterpret_cast<char*>(base);
  c->rx = p;                                         p += rx_bytes;
  c->rx_bytes = rx_bytes;
  c->part_meta = reinterpret_cast<uint32_t*>(p);     p += meta_bytes;
  c->keys_a = reinterpret_cast<uint32_t*>(p);        p += keys_bytes;
  c->keys_b = reinterpret_cast<uint32_t*>(p);        p += keys_bytes;
  c->rle = reinterpret_cast<uint64_t*>(p);           p += rle_bytes;
  c->tile_heads = reinterpret_cast<uint32_t*>(p);    p += heads_bytes;
  c->splits = reinterpret_cast<uint2*>(p);           p += splits_bytes;
  c->tile_out = reinterpret_cast<uint32_t*>(p);
  return NVTB_OK;
}

// make sure acc[which] can hold `pairs` packed pairs (contents are NOT preserved)
static int acc_reserve(SortedAcc* a, int which, int64_t pairs, cudaStream_t st) {
  if (a->acc_cap[which] >= pairs) return NVTB_OK;
  if (a->acc[which]) NVTB_CUDA_OK(cudaFreeAsync(a->acc[which], st));
  a->acc[which] = nullptr; a->acc_cap[which] = 0;
  const int64_t want = pairs + pairs / 8 + 1024;
  NVTB_CUDA_OK(cudaMallocAsync(&a->acc[which], sizeof(uint64_t) * (size_t)want, st));
  a->acc_cap[which] = want;
  return NVTB_OK;
}

// out = merge of the ua sorted pairs of A with B, counts of equal keys added.  B holds *ub_dev
// run heads of a sorted batch (B_PACKED = false) or packed pairs; mt merge tiles cover ua + *ub_dev.
// The merged count goes to *n_unique, the largest count to *max_count.
template <bool B_PACKED>
static int merge_pairs(const uint64_t* A, int64_t ua, const uint64_t* B, const uint32_t* ub_dev, int64_t mt,
                       uint64_t* out, unsigned long long* n_unique, unsigned long long* max_count, uint2* splits,
                       uint32_t* tile_out, cudaStream_t st) {
  static bool attrs = false;
  if (!attrs) {
    NVTB_CUDA_OK(cudaFuncSetAttribute(merge_write_kernel<B_PACKED>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(MergeSmem)));
    attrs = true;
  }
  merge_split_kernel<<<(int)((mt + 1 + 255) / 256), 256, 0, st>>>(A, (uint32_t)ua, B, ub_dev, (int)mt, splits);
  NVTB_LAUNCH_OK();
  merge_count_kernel<<<(int)mt, kRunThreads, 0, st>>>(A, B, splits, tile_out);
  NVTB_LAUNCH_OK();
  scan_tiles_kernel<<<1, kRunThreads, 0, st>>>(tile_out, (int)mt, nullptr, n_unique);
  NVTB_LAUNCH_OK();
  merge_write_kernel<B_PACKED><<<(int)mt, kRunThreads, sizeof(MergeSmem), st>>>(A, B, splits, tile_out, out, max_count);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

constexpr int kDnWords = 8;

// d_n[4, 6) = {~0, 0}: no valid key seen yet
static int minmax_reset(SortedAcc* a, cudaStream_t st) {
  NVTB_CUDA_OK(cudaMemsetAsync(a->d_n + 4, 0xFF, sizeof(uint32_t), st));
  NVTB_CUDA_OK(cudaMemsetAsync(a->d_n + 5, 0, sizeof(uint32_t), st));
  return NVTB_OK;
}

// bucket route (bucketagg.cuh): range partition + direct-address counting, no sort.  The batch's
// pairs go to acc[other] when the accumulator is empty, else to c.rle.  have_minmax: the staging
// copies have folded the batch's min / max into d_n[4, 6) already.  *ok = false: some window
// holds more than kBkDupCap duplicated values and the radix route has to redo the batch (the
// nulls are counted already).
static int bucket_route(SortedAcc* a, const int32_t* kp, const uint8_t* mp, int64_t m, int64_t ua, Counters* ctr,
                        bool have_minmax, const SortCarve& c, cudaStream_t st, bool* ok) {
  static bool attrs = false;
  constexpr int kBkScatterSmem = kPartTile * 4 + 2 * 4 * kBkCoarse;
  if (!attrs) {
    NVTB_CUDA_OK(cudaFuncSetAttribute(part_hist_kernel<PartRange>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * kBkParts));
    NVTB_CUDA_OK(cudaFuncSetAttribute(part_scatter_kernel<PartRangeCoarse>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kBkScatterSmem));
    NVTB_CUDA_OK(cudaFuncSetAttribute(bk_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kBkCountSmem));
    NVTB_CUDA_OK(cudaFuncSetAttribute(bk_emit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kBkEmitSmem));
    attrs = true;
  }
  const int sms = sm_count();
  const int aligned = is_aligned32(kp) ? 1 : 0;
  const int64_t tiles = (m + kPartTile - 1) / kPartTile;
  uint32_t* n_valid = a->d_n + 1;
  uint32_t* n_batch = a->d_n + 2;
  uint32_t* total = c.part_meta;                    // -> exclusive starts after the scan
  uint32_t* cursor = c.part_meta + kBkParts;
  uint32_t* distinct = c.part_meta + 2 * kBkParts;  // -> output offsets after the scan
  uint32_t* coarse = c.part_meta + 3 * kBkParts;    // cursors of the 512 coarse ranges
  unsigned int* flag = reinterpret_cast<unsigned int*>(c.part_meta + 4 * kBkParts);
  uint32_t* max_rows = a->d_n + 3;
  uint32_t* mm = a->d_n + 4;                        // {min, max}
  uint32_t* par = a->d_n + 6;                       // {lo, shift}
  NVTB_CUDA_OK(cudaMemsetAsync(flag, 0, sizeof(unsigned int), st));
  NVTB_CUDA_OK(cudaMemsetAsync(max_rows, 0, sizeof(uint32_t), st));
  NVTB_CUDA_OK(cudaMemsetAsync(total, 0, sizeof(uint32_t) * kBkParts, st));
  if (!have_minmax) {
    int rc = minmax_reset(a, st);
    if (rc) return rc;
    bk_minmax_kernel<<<(int)std::min<int64_t>(tiles, 4 * sms), kPartThreads, 0, st>>>(kp, mp, m, mm, aligned);
    NVTB_LAUNCH_OK();
  }
  bk_params_kernel<<<1, 1, 0, st>>>(mm, par);
  NVTB_LAUNCH_OK();
  part_hist_kernel<PartRange><<<(int)std::min<int64_t>(tiles, 3 * sms), kPartThreads, 4 * kBkParts, st>>>(
      kp, mp, m, PartRange{kBkLgParts, par}, total, ctr, aligned);
  NVTB_LAUNCH_OK();
  scan_tiles_kernel<<<1, kRunThreads, 0, st>>>(total, kBkParts, n_valid, nullptr);
  NVTB_LAUNCH_OK();
  // two-level partition: 512 coarse ranges (runs of ~32 keys per tile and range) into keys_b, then
  // each range into its 16 buckets (runs of hundreds of keys) at their final place in keys_a; the
  // single pass into 8192 buckets wrote runs of ~2 keys, a few bytes of a sector at a time
  bk_cursors_kernel<<<kBkParts / 256, 256, 0, st>>>(total, cursor, coarse);
  NVTB_LAUNCH_OK();
  part_scatter_kernel<PartRangeCoarse><<<(int)std::min<int64_t>(tiles, 2 * sms), kPartThreads, kBkScatterSmem, st>>>(
      kp, mp, m, PartRangeCoarse{kBkLgParts - kBkLgFine, par}, coarse, reinterpret_cast<int32_t*>(c.keys_b), aligned);
  NVTB_LAUNCH_OK();
  bk_refine_kernel<<<(int)std::min<int64_t>(m / kBkRefineTile + kBkCoarse, 2 * sms), kPartThreads, 0, st>>>(
      c.keys_b, total, n_valid, par, cursor, c.keys_a);
  NVTB_LAUNCH_OK();
  bk_count_kernel<<<kBkParts, kBkThreads, kBkCountSmem, st>>>(c.keys_a, total, n_valid, par, distinct, max_rows);
  NVTB_LAUNCH_OK();
  scan_tiles_kernel<<<1, kRunThreads, 0, st>>>(distinct, kBkParts, n_batch, ua == 0 ? &ctr->n_unique : nullptr);
  NVTB_LAUNCH_OK();
  // the accumulator is sized for what the batch really holds (its distinct keys are known now),
  // not for the worst case of all rows distinct; the emit's shared memory for the batch's window
  // and for at most half the rows of its fullest bucket as counters (a duplicated value takes two
  // rows), not for the widest window: two CTAs per SM fit up to shift 18
  uint32_t h[kDnWords - 2];          // d_n[2, 8)
  NVTB_CUDA_OK(cudaMemcpyAsync(h, n_batch, sizeof(h), cudaMemcpyDeviceToHost, st));
  NVTB_CUDA_OK(cudaStreamSynchronize(st));
  const uint32_t nb_h = h[0], shift_h = h[5];
  const int cap = (int)std::min<uint32_t>((uint32_t)kBkDupCap, h[1] / 2);
  int rc = acc_reserve(a, a->cur ^ 1, ua + (int64_t)nb_h, st);
  if (rc) return rc;
  uint64_t* B = (ua == 0) ? a->acc[a->cur ^ 1] : c.rle;
  bk_emit_kernel<<<kBkParts, kBkThreads, bk_emit_smem(shift_h, cap), st>>>(c.keys_a, total, n_valid, par, distinct,
                                                                            B, (uint32_t)cap, flag, &ctr->max_count);
  NVTB_LAUNCH_OK();
  unsigned int flag_h = 0;
  NVTB_CUDA_OK(cudaMemcpyAsync(&flag_h, flag, sizeof(flag_h), cudaMemcpyDeviceToHost, st));
  NVTB_CUDA_OK(cudaStreamSynchronize(st));
  *ok = (flag_h == 0);
  return NVTB_OK;
}

// radix route (sortagg.cuh): LSD radix sort of the valid keys (as key ^ 2^31), then the run heads
// of the sorted keys to c.rle.  null_ctr (may be NULL) receives the null count.
static int radix_route(SortedAcc* a, const int32_t* kp, const uint8_t* mp, int64_t m, int64_t ua, Counters* null_ctr,
                       const SortCarve& c, cudaStream_t st) {
  static bool attrs = false;
  constexpr int kScatterSmem = kPartTile * 4 + 2 * 4 * (1 << kSortLowBits);
  if (!attrs) {
    NVTB_CUDA_OK(cudaFuncSetAttribute(part_scatter_kernel<PartKeyLow>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, kScatterSmem));
    attrs = true;
  }
  const int sms = sm_count();
  const int P = 1 << kSortLowBits;
  const int aligned = is_aligned32(kp) ? 1 : 0;
  const int64_t tiles = (m + kPartTile - 1) / kPartTile;
  uint32_t* n_valid = a->d_n + 1;
  uint32_t* n_batch = a->d_n + 2;
  int rc = acc_reserve(a, a->cur ^ 1, ua + m, st);
  if (rc) return rc;
  NVTB_CUDA_OK(cudaMemsetAsync(c.part_meta, 0, sizeof(uint32_t) * P, st));
  part_hist_kernel<PartKeyLow><<<(int)std::min<int64_t>(tiles, 3 * sms), kPartThreads, 4 * P, st>>>(
      kp, mp, m, PartKeyLow{kSortLowBits}, c.part_meta, null_ctr, aligned);
  NVTB_LAUNCH_OK();
  part_scan_kernel<<<1, kPartThreads, 0, st>>>(c.part_meta, kSortLowBits, c.part_meta + P, c.part_meta + 2 * P, 1u, n_valid);
  NVTB_LAUNCH_OK();
  part_scatter_kernel<PartKeyLow><<<(int)std::min<int64_t>(tiles, 2 * sms), kPartThreads, kScatterSmem, st>>>(
      kp, mp, m, PartKeyLow{kSortLowBits}, c.part_meta + 2 * P, reinterpret_cast<int32_t*>(c.keys_a), aligned);
  NVTB_LAUNCH_OK();
  int in_b = 0;
  rc = rx_sort_bits<uint32_t>(nullptr, c.keys_a, c.keys_b, n_valid, m, kSortLowBits, 32, false, c.rx, c.rx_bytes, st,
                              &in_b);
  if (rc) return rc;
  const uint32_t* sorted = in_b ? c.keys_b : c.keys_a;
  const int rt = (int)((m + kRleTile - 1) / kRleTile);
  rle_count_kernel<<<rt, kRunThreads, 0, st>>>(sorted, n_valid, m, c.tile_heads);
  NVTB_LAUNCH_OK();
  scan_tiles_kernel<<<1, kRunThreads, 0, st>>>(c.tile_heads, rt, n_batch, nullptr);
  NVTB_LAUNCH_OK();
  rle_write_kernel<<<rt, kRunThreads, 0, st>>>(sorted, n_valid, m, c.tile_heads, n_batch, c.rle);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

// fold m rows of int32 keys into the accumulator, which holds ua pairs (have_minmax: see bucket_route)
static int insert_rows(SortedAcc* a, const int32_t* kp, const uint8_t* mp, int64_t m, int64_t ua, Counters* ctr,
                       bool have_minmax, cudaStream_t st) {
  const int64_t mt = (ua + m + kMergeTile - 1) / kMergeTile;
  SortCarve c;
  int rc = sort_scratch_acquire(m, 64, mt, st, &c);
  if (rc) return rc;
  const char* path_env = getenv("NVTB_SORT_PATH");
  const bool radix_only = path_env && strcmp(path_env, "radix") == 0;
  bool bucketed = false;
  if (!radix_only) {
    rc = bucket_route(a, kp, mp, m, ua, ctr, have_minmax, c, st, &bucketed);
    if (rc) return rc;
  }
  if (!bucketed) {
    rc = radix_route(a, kp, mp, m, ua, radix_only ? ctr : nullptr, c, st);
    if (rc) return rc;
  }
  const uint64_t* A = a->acc[a->cur];
  uint64_t* out = a->acc[a->cur ^ 1];
  uint32_t* n_batch = a->d_n + 2;
  if (!bucketed)
    rc = merge_pairs<false>(A, ua, c.rle, n_batch, mt, out, &ctr->n_unique, &ctr->max_count, c.splits, c.tile_out, st);
  else if (ua > 0)      // (into an empty accumulator the bucket route has emitted straight to `out`)
    rc = merge_pairs<true>(A, ua, c.rle, n_batch, mt, out, &ctr->n_unique, &ctr->max_count, c.splits, c.tile_out, st);
  if (rc) return rc;
  a->cur ^= 1;
  return g_sort.release(st);
}

int sortacc_insert(SortedAcc* a, const int32_t* kp, const uint8_t* mp, int64_t m, int64_t ua, Counters* ctr,
                   cudaStream_t st) {
  return insert_rows(a, kp, mp, m, ua, ctr, false, st);
}

// rows a sorted accumulator stages before it sorts (NVTB_STAGE_ROWS, default 2^28 = 1 GiB of keys)
static int64_t stage_cap_rows() {
  const char* e = getenv("NVTB_STAGE_ROWS");
  int64_t v = e ? atoll(e) : ((int64_t)1 << 28);
  if (v < 0) v = 0;
  if (v > (int64_t)0xF0000000ll) v = (int64_t)0xF0000000ll;
  return v / 64 * 64;
}

int sortacc_create(SortedAcc** out, int64_t u, cudaStream_t st, uint64_t** pairs) {
  SortedAcc* a = new (std::nothrow) SortedAcc();
  NVTB_REQUIRE(a != nullptr, "host allocation failed");
  *out = a;
  *pairs = nullptr;
  NVTB_CUDA_OK(cudaMalloc(&a->d_n, sizeof(uint32_t) * kDnWords));
  NVTB_CUDA_OK(cudaMemsetAsync(a->d_n, 0, sizeof(uint32_t) * kDnWords, st));
  if (u > 0) {
    int rc = acc_reserve(a, 0, u, st);
    if (rc) return rc;
    rc = acc_reserve(a, 1, u, st);
    if (rc) return rc;
    *pairs = a->acc[0];
  }
  return NVTB_OK;
}

int sortacc_sort_pairs(SortedAcc* a, int64_t u, cudaStream_t st) {
  if (u == 0) return NVTB_OK;
  SortCarve c;
  int rc = sort_scratch_acquire(64, u, 1, st, &c);
  if (rc) return rc;
  int in_b = 0;
  rc = rx_sort_bits<uint64_t>(nullptr, a->acc[0], a->acc[1], nullptr, u, 32, 64, false, c.rx, c.rx_bytes, st, &in_b);
  if (rc) return rc;
  a->cur = in_b;
  return g_sort.release(st);
}

bool sortacc_stages(const SortedAcc* a, int64_t m) {
  const int64_t cap = stage_cap_rows();
  return cap >= 64 && m <= cap && (a->stage_rows & 7) == 0;
}

bool sortacc_stage_full(const SortedAcc* a, int64_t m) {
  return a->stage_rows > 0 && a->stage_rows + m > a->stage_cap;
}

int64_t sortacc_staged_rows(const SortedAcc* a) { return a->stage_rows; }

// append one batch to the staging buffers (stage_rows % 8 == 0; the caller flushed when the
// batch does not fit behind the waiting rows)
int sortacc_stage(SortedAcc* a, const int32_t* kp, const uint8_t* mp, int64_t m, int64_t rows_total, cudaStream_t st) {
  if (a->stage_ev == nullptr) NVTB_CUDA_OK(cudaEventCreateWithFlags(&a->stage_ev, cudaEventDisableTiming));
  if (a->stage_last != nullptr && a->stage_last != st) NVTB_CUDA_OK(cudaStreamWaitEvent(st, a->stage_ev, 0));
  const int64_t cap_max = stage_cap_rows();
  const bool grow_for_fit = a->stage_rows == 0 && a->stage_cap < std::min<int64_t>(cap_max, a->stage_hint);
  if (a->stage_rows + m > a->stage_cap || grow_for_fit) {
    NVTB_REQUIRE(a->stage_rows == 0, "staging buffer resized while rows are waiting");
    if (a->stage_keys) NVTB_CUDA_OK(cudaFreeAsync(a->stage_keys, st));
    if (a->stage_mask) NVTB_CUDA_OK(cudaFreeAsync(a->stage_mask, st));
    a->stage_keys = nullptr; a->stage_mask = nullptr; a->stage_cap = 0;
    // sized for what the fit has shown so far (a small fit must not pay for 1 GiB), doubling
    int64_t want = (int64_t)1 << 22;
    while (want < 2 * (rows_total + m)) want <<= 1;
    want = std::max<int64_t>(want, (a->stage_hint + 63) / 64 * 64);      // one flush per fit from the second fit on
    want = std::max<int64_t>(std::min<int64_t>(want, cap_max), m);
    NVTB_CUDA_OK(cudaMallocAsync(&a->stage_keys, sizeof(int32_t) * (size_t)(want + 64), st));
    NVTB_CUDA_OK(cudaMallocAsync(&a->stage_mask, (size_t)(want / 8 + 64), st));
    a->stage_cap = want;
  }
  if (a->stage_rows == 0) {
    int rc = minmax_reset(a, st);
    if (rc) return rc;
  }
  const int64_t tiles = (m + kPartTile - 1) / kPartTile;
  bk_stage_kernel<<<(int)std::min<int64_t>(tiles, 4 * sm_count()), kPartThreads, 0, st>>>(
      kp, mp, m, a->stage_keys + a->stage_rows, a->stage_mask + (a->stage_rows >> 3), a->d_n + 4,
      is_aligned32(kp) ? 1 : 0);
  NVTB_LAUNCH_OK();
  a->stage_rows += m;
  NVTB_CUDA_OK(cudaEventRecord(a->stage_ev, st));
  a->stage_last = st;
  return NVTB_OK;
}

// group + merge everything that is staged
int sortacc_flush(SortedAcc* a, int64_t u, Counters* ctr, cudaStream_t st) {
  if (a->stage_rows == 0) return NVTB_OK;
  if (a->stage_last != st && a->stage_ev) NVTB_CUDA_OK(cudaStreamWaitEvent(st, a->stage_ev, 0));
  int rc = insert_rows(a, a->stage_keys, a->stage_mask, a->stage_rows, u, ctr, true, st);
  if (rc) return rc;
  a->stage_rows = 0;
  NVTB_CUDA_OK(cudaEventRecord(a->stage_ev, st));
  a->stage_last = st;
  return NVTB_OK;
}

void sortacc_reset(SortedAcc* a, int64_t rows_total) {
  a->stage_hint = std::max<int64_t>(a->stage_hint, rows_total);
  a->stage_rows = 0;          // batches still waiting belong to the fit that is being discarded
}

void sortacc_destroy(SortedAcc* a) {
  if (a->acc[0]) cudaFree(a->acc[0]);
  if (a->acc[1]) cudaFree(a->acc[1]);
  if (a->d_n) cudaFree(a->d_n);
  if (a->stage_keys) cudaFree(a->stage_keys);
  if (a->stage_mask) cudaFree(a->stage_mask);
  if (a->stage_ev) cudaEventDestroy(a->stage_ev);
  delete a;
}

const uint64_t* sortacc_pairs(const SortedAcc* a) { return a->acc[a->cur]; }

// int64 keys / sizes in key order (nvtb_hashagg_export of a sorted handle)
int sortacc_unpack(const SortedAcc* a, int64_t u, int64_t* keys, int64_t* sizes, cudaStream_t st) {
  runs_unpack_kernel<<<plain_grid(u), kThreads, 0, st>>>(a->acc[a->cur], u, keys, sizes);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

}  // namespace nvtb

using namespace nvtb;

extern "C" {

// Stable LSD radix sort of bits [lo_bit, hi_bit) (radix.cuh), exposed for tests and for
// callers that order their own device arrays.  The result ends in `data` or in `tmp`
// (*result_in_tmp_host).
static int radix_sort_entry(void* data, void* tmp, int64_t n, int elem_bytes, int lo_bit, int hi_bit,
                            int descending, int* result_in_tmp_host, void* stream) {
  NVTB_REQUIRE(n >= 0 && result_in_tmp_host != nullptr, "bad n / NULL result flag");
  NVTB_REQUIRE(lo_bit >= 0 && hi_bit <= 8 * elem_bytes && lo_bit <= hi_bit, "bad bit range");
  *result_in_tmp_host = 0;
  if (n == 0 || lo_bit == hi_bit) return NVTB_OK;
  NVTB_REQUIRE(data != nullptr && tmp != nullptr, "NULL data/tmp");
  NVTB_REQUIRE((reinterpret_cast<uintptr_t>(data) & 15u) == 0 && (reinterpret_cast<uintptr_t>(tmp) & 15u) == 0,
               "data/tmp must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  void* scratch = nullptr;
  const size_t bytes = elem_bytes == 4 ? rx_scratch_bytes<uint32_t>(n) : rx_scratch_bytes<uint64_t>(n);
  NVTB_CUDA_OK(cudaMallocAsync(&scratch, bytes, st));
  NVTB_CUDA_OK(cudaMemsetAsync(scratch, 0, 256, st));
  int rc;
  if (elem_bytes == 4)
    rc = rx_sort_bits<uint32_t>(nullptr, (uint32_t*)data, (uint32_t*)tmp, nullptr, n, lo_bit, hi_bit, descending != 0,
                                scratch, bytes, st, result_in_tmp_host);
  else
    rc = rx_sort_bits<uint64_t>(nullptr, (uint64_t*)data, (uint64_t*)tmp, nullptr, n, lo_bit, hi_bit, descending != 0,
                                scratch, bytes, st, result_in_tmp_host);
  NVTB_CUDA_OK(cudaFreeAsync(scratch, st));
  return rc;
}

int nvtb_radix_sort_u32(uint32_t* data, uint32_t* tmp, int64_t n, int lo_bit, int hi_bit, int descending,
                        int* result_in_tmp_host, void* stream) {
  return radix_sort_entry(data, tmp, n, 4, lo_bit, hi_bit, descending, result_in_tmp_host, stream);
}

int nvtb_radix_sort_u64(uint64_t* data, uint64_t* tmp, int64_t n, int lo_bit, int hi_bit, int descending,
                        int* result_in_tmp_host, void* stream) {
  return radix_sort_entry(data, tmp, n, 8, lo_bit, hi_bit, descending, result_in_tmp_host, stream);
}

// ---------------------------------------------------------------------------------------
// sorted-pair primitives of the cross-GPU vocabulary merge (nvtabular_b200/dist.py)
// ---------------------------------------------------------------------------------------
int nvtb_pairs_lower_bounds(const uint64_t* pairs, int64_t n, const uint32_t* bounds_dev, int m,
                            int64_t* out_dev, void* stream) {
  NVTB_REQUIRE(n >= 0 && m >= 0, "negative size");
  if (m == 0) return NVTB_OK;
  NVTB_REQUIRE(bounds_dev != nullptr && out_dev != nullptr && (n == 0 || pairs != nullptr), "NULL argument");
  pairs_lower_bound_kernel<<<(m + 127) / 128, 128, 0, (cudaStream_t)stream>>>(
      pairs, n, bounds_dev, m, reinterpret_cast<long long*>(out_dev));
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

// out = merge of two key-sorted, key-unique packed-pair arrays, counts of equal keys added.
// `out` must hold na + nb pairs; the merged length comes back on the host (one stream sync).
int nvtb_pairs_merge(const uint64_t* a, int64_t na, const uint64_t* b, int64_t nb, uint64_t* out,
                     int64_t* n_out_host, void* stream) {
  NVTB_REQUIRE(na >= 0 && nb >= 0 && n_out_host != nullptr, "bad sizes / NULL n_out");
  NVTB_REQUIRE(na + nb < (int64_t)0xFFFF0000ll, "more than 2^32 pairs in one merge");
  cudaStream_t st = (cudaStream_t)stream;
  *n_out_host = 0;
  if (na + nb == 0) return NVTB_OK;
  NVTB_REQUIRE(out != nullptr, "NULL out");
  if (na == 0 || nb == 0) {
    NVTB_CUDA_OK(cudaMemcpyAsync(out, na ? a : b, sizeof(uint64_t) * (size_t)(na + nb), cudaMemcpyDeviceToDevice, st));
    *n_out_host = na + nb;
    return NVTB_OK;
  }
  const int64_t mt = (na + nb + kMergeTile - 1) / kMergeTile;
  SortCarve c;
  int rc = sort_scratch_acquire(64, 64, mt, st, &c);
  if (rc) return rc;
  uint32_t* ub_dev = c.part_meta;                  // ub | n_unique | max_count
  unsigned long long* nu_dev = reinterpret_cast<unsigned long long*>(c.part_meta + 2);
  const uint32_t ub_h = (uint32_t)nb;
  NVTB_CUDA_OK(cudaMemsetAsync(ub_dev, 0, 64, st));
  NVTB_CUDA_OK(cudaMemcpyAsync(ub_dev, &ub_h, sizeof(ub_h), cudaMemcpyHostToDevice, st));
  rc = merge_pairs<true>(a, na, b, ub_dev, mt, out, nu_dev, nu_dev + 1, c.splits, c.tile_out, st);
  if (rc) return rc;
  unsigned long long nu_h = 0;
  NVTB_CUDA_OK(cudaMemcpyAsync(&nu_h, nu_dev, sizeof(nu_h), cudaMemcpyDeviceToHost, st));
  rc = g_sort.release(st);
  if (rc) return rc;
  NVTB_CUDA_OK(cudaStreamSynchronize(st));
  *n_out_host = (int64_t)nu_h;
  return NVTB_OK;
}

// contiguous segments of src to their destinations: seg_src[nseg + 1] ascending prefix (device),
// seg_dst[nseg] (device)
int nvtb_segment_copy_u64(const uint64_t* src, uint64_t* dst, const int64_t* seg_src_dev, const int64_t* seg_dst_dev,
                          int nseg, int64_t n, void* stream) {
  NVTB_REQUIRE(nseg >= 0 && n >= 0, "negative size");
  if (n == 0 || nseg == 0) return NVTB_OK;
  NVTB_REQUIRE(src && dst && seg_src_dev && seg_dst_dev, "NULL argument");
  segment_copy_kernel<<<plain_grid((n + 3) / 4), kThreads, 0, (cudaStream_t)stream>>>(
      src, dst, reinterpret_cast<const long long*>(seg_src_dev), reinterpret_cast<const long long*>(seg_dst_dev), nseg, n);
  NVTB_LAUNCH_OK();
  return NVTB_OK;
}

}  // extern "C"
