// hashagg.cuh — shared by the group-by handle (hashagg.cu), its sorted accumulator (sortacc.cu)
// and the vocabulary build (vocab.cu).
#pragma once

#include <mutex>

#include "common.cuh"

struct nvtb_hashagg;

namespace nvtb {

struct Counters {
  unsigned long long n_unique;   // distinct keys in the table
  unsigned long long size[2];    // special groups: [0] null key, [1] INT64_MIN key
  unsigned long long ovf_count;  // pairs refused into the arena by the pending launch
  unsigned long long max_count;  // sorted accumulator (sortagg.cuh): largest group size seen
};

// A grow-only device buffer shared by every handle of the process (a fresh cudaMallocAsync of
// hundreds of MB per column occasionally costs tens of ms when the pool has to map new memory).
// acquire orders `st` after the last release on another stream; growing (to `alloc` >= `need`
// bytes) synchronises the device and sets *grown.
struct SharedScratch {
  std::mutex mu;
  void* ptr = nullptr;
  size_t bytes = 0;
  cudaEvent_t ev = nullptr;
  cudaStream_t last = nullptr;
  bool used = false;
  int acquire(size_t need, size_t alloc, cudaStream_t st, void** out, bool* grown);
  int release(cudaStream_t st);
};

// Sorted accumulator (sortacc.cu): key-ordered packed pairs (key ^ 2^31) << 32 | count.  The
// handle owns the distinct count u (settled before every call that takes it) and the Counters
// that the calls update: n_unique, max_count and the null count size[0].
struct SortedAcc;
// from a hash table: a buffer for its u pairs in any order, which sortacc_sort_pairs then sorts
int sortacc_create(SortedAcc** out, int64_t u, cudaStream_t st, uint64_t** pairs);
int sortacc_sort_pairs(SortedAcc* a, int64_t u, cudaStream_t st);
// a batch is staged (copied) when sortacc_stages, after a flush when sortacc_stage_full; else
// the staged rows are flushed and the batch goes in through sortacc_insert
bool sortacc_stages(const SortedAcc* a, int64_t m);
bool sortacc_stage_full(const SortedAcc* a, int64_t m);
int64_t sortacc_staged_rows(const SortedAcc* a);
int sortacc_stage(SortedAcc* a, const int32_t* keys, const uint8_t* mask, int64_t m, int64_t rows_total,
                  cudaStream_t st);
int sortacc_flush(SortedAcc* a, int64_t u, Counters* ctr, cudaStream_t st);
int sortacc_insert(SortedAcc* a, const int32_t* keys, const uint8_t* mask, int64_t m, int64_t u, Counters* ctr,
                   cudaStream_t st);
void sortacc_reset(SortedAcc* a, int64_t rows_total);   // rows_total: the fit that ended
void sortacc_destroy(SortedAcc* a);                      // the device is idle
const uint64_t* sortacc_pairs(const SortedAcc* a);
int sortacc_unpack(const SortedAcc* a, int64_t u, int64_t* keys, int64_t* sizes, cudaStream_t st);

// view of a handle for nvtb_vocab_build_from_hashagg (vocab.cu): synchronises on the handle's
// pending launch.  *pairs == nullptr when the handle is a hash table (the caller exports).
int hashagg_sorted_view(nvtb_hashagg* h, const uint64_t** pairs, int64_t* n_unique, int64_t* null_size,
                        uint64_t* max_count, int* is_i32_table, cudaStream_t st);

}  // namespace nvtb
