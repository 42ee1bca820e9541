/*
 * nvtb200.h — C-ABI of libnvtb200.so, the H100 (sm_90a) engine behind the
 * nvtabular.ops operator API for the Categorify / Normalize / FillMissing /
 * HashBucket / JoinGroupby / TargetEncoding hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  The reference has no FFI on
 * this path: its operators call cuDF / pandas through merlin.core.dispatch
 * (reference nvtabular/dispatch.py:21).  Each entry point below replaces the
 * dataframe-library call(s) the reference makes at the cited file:line; the
 * Python operator classes in nvtabular_b200/ops bind these with ctypes
 * (see INTEGRATION.md for the binding a reference maintainer would add).
 *
 * Conventions
 *   - every function returns 0 on success or a negative nvtb_status_t;
 *     nvtb_last_error() gives a thread-local message.  No C++ exception ever
 *     crosses this boundary.
 *   - all data pointers are DEVICE pointers owned by the caller unless the
 *     parameter name ends in `_host`.
 *   - `stream` is a cudaStream_t passed as void*.  All kernels are stream
 *     ordered; only the functions documented as "synchronises" block the host.
 *   - a column is (data, validity, dtype).  `validity` is an Arrow-style
 *     bitmask: bit (i & 7) of byte (i >> 3) is 1 when row i is non-null;
 *     NULL means "no nulls".  Data pointers should be 32-byte aligned for
 *     the vectorised (256-bit) path; a scalar path is taken otherwise.
 *   - handles (nvtb_hashagg_t, nvtb_vocab_t, nvtb_groupstats_t) are created
 *     and destroyed explicitly; build-phase calls on one handle must not be
 *     issued concurrently; finalised vocab / groupstats handles are immutable
 *     and may be probed from any number of streams.
 *   - ONE device per process (the one-process-per-GPU model of SURVEY §8e): the
 *     hashagg build phase keeps grow-only scratch (two accumulator arenas, the
 *     partition buffer, the sort / bucket scratch) in process-global pools on the device
 *     that was current at the first call.  The pools are mutex-guarded and a use
 *     on another stream waits on an event of the previous one, so build calls
 *     of DIFFERENT handles may come from different streams of that device; a
 *     second device in the same process is not supported and not detected.
 */
#ifndef NVTB200_H
#define NVTB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  NVTB_OK = 0,
  NVTB_EINVAL = -1,  /* bad argument (dtype, null pointer, size)          */
  NVTB_ENOMEM = -2,  /* device allocation failed                          */
  NVTB_ECUDA = -3,   /* a CUDA runtime call or kernel launch failed       */
  NVTB_ESTATE = -4,  /* handle used in the wrong phase                    */
  NVTB_ENCCL = -5,   /* an NCCL call failed / NCCL is not loadable         */
  NVTB_EIO = -6      /* a file could not be written (the path is in the message) */
} nvtb_status_t;

typedef enum {
  NVTB_I32 = 0,
  NVTB_I64 = 1,
  NVTB_F32 = 2,
  NVTB_F64 = 3,
  NVTB_U8 = 4,  /* bool / fold ids */
  NVTB_H64 = 5  /* hash columns only: a precomputed 64-bit value hash (e.g. the
                   pandas string hash of a dictionary entry), used as-is   */
} nvtb_dtype_t;

typedef struct {
  const void* data;        /* device, n elements of `dtype`               */
  const uint8_t* validity; /* device bitmask or NULL                      */
  int32_t dtype;           /* nvtb_dtype_t                                */
  int32_t _pad;
} nvtb_col_t;

/* library identity ------------------------------------------------------- */
int nvtb_version(void);              /* 1000*major + minor                 */
const char* nvtb_last_error(void);   /* thread-local, never NULL           */
int nvtb_device_sm_count(int* out_host); /* SMs of the current device      */

/* ---- Normalize / NormalizeMinMax statistics ---------------------------
 * Replaces _chunkwise_moments (reference nvtabular/ops/moments.py:64-77:
 * count(), sum(), astype(f64).pow(2).sum() — three cuDF reductions per
 * column) and ddf.min()/ddf.max() (reference nvtabular/ops/normalize.py:
 * 166-170) with ONE fused scan over all columns.  FillMissing upstream
 * (reference nvtabular/ops/fill.py:49-57) is fused: when fill_vals_host[c]
 * is not NaN, null rows count as that value instead of being skipped.
 *
 * acc: device double[ncols * 5] = {count, sum, sumsq, min, max} per column.
 * The call ADDS this batch into acc (min/max: combines), so batches and the
 * tree reduction of moments.py:80-86 become repeated calls.  Initialise with
 * nvtb_moments_init.  Deterministic: fixed grid + ordered final reduction.
 */
int nvtb_moments_init(double* acc, int ncols, void* stream);
int nvtb_moments_accumulate(const nvtb_col_t* cols_host, int ncols, int64_t n,
                            const double* fill_vals_host, double* acc,
                            void* stream);
/* _finalize_moments (reference nvtabular/ops/moments.py:89-116), host math:
 * mean = sum/n; var = (sumsq - sum^2/n) / max(n-1,1), NaN when n-1 == 0;
 * std = sqrt(var).  acc_host is a HOST copy of acc.  out_host: double
 * [ncols*3] = {mean, var, std}. */
int nvtb_moments_finalize(const double* acc_host, int ncols, double* out_host);

/* ---- FillMissing / Normalize transforms --------------------------------
 * nvtb_fill_apply: FillMissing.transform (reference nvtabular/ops/fill.py:
 * 49-57, C++ twin cpp/nvtabular/inference/fill.cc:91-102): out = valid ? x :
 * (T)fill, dtype preserved; filled_out[c] (may be NULL) receives the
 * `<col>_filled` indicator as uint8 0/1.
 *
 * nvtb_normalize_apply: Normalize.transform (reference nvtabular/ops/
 * normalize.py:71-90) fused with an upstream FillMissing:
 * y = std>0 ? (x-mean)/std : (x-mean); float32 inputs are computed in float32
 * exactly like numpy does, everything else in float64; out_dtype F32|F64.
 * With fill NaN, null rows produce NaN (nulls propagate).
 *
 * nvtb_minmax_apply: NormalizeMinMax.transform (normalize.py:150-161):
 * (x-min)/(max-min) when max>min, x/(2x) when max==min.
 */
int nvtb_fill_apply(const nvtb_col_t* cols_host, int ncols, int64_t n,
                    const double* fill_vals_host, void* const* out_host,
                    uint8_t* const* filled_out_host, void* stream);
int nvtb_normalize_apply(const nvtb_col_t* cols_host, int ncols, int64_t n,
                         const double* fill_vals_host,
                         const double* means_host, const double* stds_host,
                         void* const* out_host, int out_dtype, void* stream);
int nvtb_minmax_apply(const nvtb_col_t* cols_host, int ncols, int64_t n,
                      const double* fill_vals_host, const double* mins_host,
                      const double* maxs_host, void* const* out_host,
                      int out_dtype, void* stream);

/* Clip (reference nvtabular/ops/clip.py:46-53) and Clip + LogOp (ops/logop.py:47-56) in one
 * pass, with an upstream FillMissing fused in (fill_vals[c] NaN = none): x = fill if null;
 * x = max(x, min_vals[c]); x = min(x, max_vals[c]) (NaN bound / NULL array = none);
 * take_log == 0: out[c] has the column's own dtype; take_log != 0: out[c] (out_dtype float32 |
 * float64) = log(x cast to out_dtype + 1).  Rows that stay null are written as 0 / NaN. */
int nvtb_cliplog_apply(const nvtb_col_t* cols, int ncols, int64_t n,
                       const double* fill_vals, const double* min_vals,
                       const double* max_vals, int take_log, void* const* out,
                       int out_dtype, void* stream);

/* ---- HashBucket ---------------------------------------------------------
 * dispatch.hash_series(col) % nb  (reference nvtabular/ops/hash_bucket.py:
 * 86-100, nvtabular/ops/categorify.py:1837-1852).  The hash is the value-only
 * pandas hash (pandas/core/util/hashing.py::_hash_ndarray): bits of the value
 * zero-extended to u64 by itemsize, then the splitmix64 finaliser.  ncols > 1
 * XORs the per-column hashes first (encode_type="combo", categorify.py:
 * 1847-1851; HashedCross).  out[i] = (int32)(h % nb) + add.  Null rows hash
 * the float64 NaN pattern (what the pandas path sees for a null).
 */
int nvtb_hash_bucket_apply(const nvtb_col_t* cols_host, int ncols, int64_t n,
                           uint64_t num_buckets, int64_t add, void* out,
                           int out_dtype, void* stream);
/* raw 64-bit hashes (testing / host-side composition) */
int nvtb_hash_values(const nvtb_col_t* col_host, int64_t n, uint64_t* out,
                     void* stream);

/* pack two key columns into one order-preserving int64 key:
 * (a << 32) | (b ^ 0x80000000), both I32.  Rows where BOTH are null become
 * null (validity_out bit cleared); a single null becomes INT32_MIN so the
 * tuple sorts first (categorify.py:1689-1692 all-null rule; KAT
 * tests/unit/ops/test_categorify.py:288-297). */
int nvtb_pack_keys2(const nvtb_col_t* a_host, const nvtb_col_t* b_host,
                    int64_t n, int64_t* keys_out, uint8_t* validity_out,
                    void* stream);

/* ---- hash aggregation: groupby(key, dropna=False).agg(size[,sum,...]) ----
 * Replaces _top_level_groupby / _mid_level_groupby / _bottom_level_groupby
 * (reference nvtabular/ops/categorify.py:955-1137): cuDF hash-groupby per
 * partition + tree of concat+groupby.  One handle per column group holds an
 * open-addressing device table {key:int64, size:int64 [, per cont col: sum,
 * sumsq, min, max : double]} that every batch is inserted into (block-level
 * shared-memory pre-aggregation, then global atomics).  The null key
 * (dropna=False) is kept out of the table in a dedicated group.
 *
 *   size  = rows in the group                       (agg "size", Categorify)
 *   count : the reference attaches agg "count" to the FIRST KEY column
 *           (categorify.py:989-999), so count == size when that key component
 *           is non-null and 0 otherwise — derived by the caller from the key,
 *           not stored.
 *   per cont column: sum / sumsq over non-null values, min, max
 *           (NaN when the group has no non-null value).
 *
 * n_agg = number of continuous columns (0 for Categorify).  capacity_hint =
 * expected number of distinct keys (0 = unknown: the first 2^20 rows are
 * inserted on their own and their exact distinct count sizes the table).
 * The hint only affects speed; results never depend on it.
 * key dtype I32 or I64 (multi-column keys are packed to I64 with
 * nvtb_pack_keys2 first).
 */
typedef struct nvtb_hashagg nvtb_hashagg_t;
int nvtb_hashagg_create(nvtb_hashagg_t** out, int n_agg,
                        int64_t capacity_hint);
int nvtb_hashagg_destroy(nvtb_hashagg_t* h);
/* empty the table but keep its capacity and cardinality estimate (a second fit
 * over similar data then needs neither growth nor the sampling pass) */
int nvtb_hashagg_reset(nvtb_hashagg_t* h, void* stream);
/* insert one batch of raw rows; agg_cols_host may be NULL when n_agg == 0.
 * int32 keys without payload are folded in SHARED memory (one kernel), after a
 * one-pass hash partition of the column (three more kernels) when the expected
 * number of distinct keys exceeds what one SM's shared memory holds
 * (csrc/fold_i32.cuh); other keys take one kernel that updates the table directly.  Waits for the handle's PREVIOUS launch (its counters are
 * read back), never for the one it enqueues. */
int nvtb_hashagg_insert(nvtb_hashagg_t* h, const nvtb_col_t* key_host,
                        const nvtb_col_t* agg_cols_host, int64_t n,
                        void* stream);
/* merge pre-aggregated partials (the cross-GPU unique-merge and the
 * _mid_level_groupby concat+groupby, categorify.py:1054-1070).  vals layout:
 * double[n * 4 * n_agg] row-major {sum,sumsq,min,max} per cont col, or NULL. */
int nvtb_hashagg_merge(nvtb_hashagg_t* h, const int64_t* keys,
                       const int64_t* sizes, const double* vals, int64_t n,
                       void* stream);
int nvtb_hashagg_add_null_group(nvtb_hashagg_t* h, int64_t size,
                                const double* vals_host);
/* synchronises; number of distinct non-null keys, and the null group's size */
int nvtb_hashagg_size(nvtb_hashagg_t* h, int64_t* n_unique_host,
                      int64_t* null_size_host, void* stream);
/* compact the table into caller arrays of length n_unique (unordered).
 * vals_out may be NULL when n_agg == 0.  null_vals_host: host double
 * [4*n_agg] for the null group, may be NULL. */
int nvtb_hashagg_export(nvtb_hashagg_t* h, int64_t* keys_out,
                        int64_t* sizes_out, double* vals_out,
                        double* null_vals_host, void* stream);

/* 0 = resident hash table, 1 = sorted accumulator.  int32 key columns whose expected number
 * of distinct keys exceeds NVTB_RUNS_MIN_KEYS (default 2^23: the table would leave the L2)
 * are accumulated as a key-ordered array of packed (key, count) pairs: every batch is
 * radix-sorted, run-length encoded and merged in (csrc/sortagg.cuh) — the streaming
 * replacement of the per-partition groupby + concat/groupby tree of reference
 * nvtabular/ops/categorify.py:955-1137 for the C20/C1/C22/C10 class of Criteo columns. */
int nvtb_hashagg_mode(nvtb_hashagg_t* h, int* mode_host);
/* A sorted accumulator only COPIES a batch (keys + validity bytes) into its staging buffer; the
 * sort + run-length encode + merge of everything staged runs when NVTB_STAGE_ROWS rows (default
 * 2^28) are waiting, when the handle is read (size / export / vocabulary build), or here. */
int nvtb_hashagg_flush(nvtb_hashagg_t* h, void* stream);

/* ---- sorted-pair primitives of the cross-GPU vocabulary merge (SURVEY.md 8e) --------------
 * A high-cardinality column is exchanged between GPUs as key-ordered packed pairs
 * word = (uint32)(key ^ 2^31) << 32 | (uint32)count (unsigned order of the word == key order),
 * split by KEY RANGE (the local accumulator is already grouped by owner: no partition pass),
 * merged by the owner, ordered by count on the owner, and the owners' count-ordered shards
 * are interleaved into the global (count desc, key asc) order group by group.  Replaces the
 * dask tree + shared-filesystem hop of reference nvtabular/ops/categorify.py:1036-1049,
 * 1399-1540.  The collectives themselves are issued by the host (torch.distributed / NCCL). */
/* make the handle a sorted accumulator (no-op if it is one); NVTB_ESTATE when the handle holds
 * int64 keys, payload columns or >= 2^32 rows */
int nvtb_hashagg_to_sorted(nvtb_hashagg_t* h, void* stream);
/* copy the packed pairs of a sorted accumulator (key order) to `out` (may be NULL: size query) */
int nvtb_hashagg_export_packed(nvtb_hashagg_t* h, uint64_t* out, int64_t* n_host, void* stream);
/* out_dev[j] = number of pairs whose unsigned key is < bounds_dev[j]  (the split points of the
 * key-range exchange) */
int nvtb_pairs_lower_bounds(const uint64_t* pairs, int64_t n, const uint32_t* bounds_dev, int m,
                            int64_t* out_dev, void* stream);
/* merge two key-sorted, key-unique pair arrays adding the counts of equal keys (the owner-side
 * _mid_level_groupby, categorify.py:1054-1070); out holds na + nb pairs; synchronises */
int nvtb_pairs_merge(const uint64_t* a, int64_t na, const uint64_t* b, int64_t nb, uint64_t* out,
                     int64_t* n_out_host, void* stream);
/* copy nseg contiguous segments [seg_src[s], seg_src[s+1]) of src to dst + seg_dst[s] */
int nvtb_segment_copy_u64(const uint64_t* src, uint64_t* dst, const int64_t* seg_src_dev,
                          const int64_t* seg_dst_dev, int nseg, int64_t n, void* stream);

/* Stable LSD radix sort of device arrays by bits [lo_bit, hi_bit) of every element
 * (csrc/radix.cuh; ascending, or descending on that bit field).  data/tmp: n elements
 * each, 16-byte aligned; the result ends in data (*result_in_tmp_host = 0) or tmp (= 1).
 * This is the ordering primitive behind sort_values in reference
 * nvtabular/ops/categorify.py:1300,1316. */
int nvtb_radix_sort_u32(uint32_t* data, uint32_t* tmp, int64_t n, int lo_bit, int hi_bit,
                        int descending, int* result_in_tmp_host, void* stream);
int nvtb_radix_sort_u64(uint64_t* data, uint64_t* tmp, int64_t n, int lo_bit, int hi_bit,
                        int descending, int* result_in_tmp_host, void* stream);

/* ---- cross-GPU exchange ---- */
/* owner = mix(key) % n_parts for the key-hash sharding of the hash-table
 * columns across GPUs (SURVEY.md §8e; the reference's split_out shuffle_group,
 * categorify.py:1036-1049).  perm_out receives a permutation that groups rows
 * by owner; part_counts_dev (device int64[n_parts]) the rows per owner.
 * Nothing synchronises, so the 26 columns of a Categorify fit are partitioned
 * back to back and their counts read with ONE copy (nvtabular_b200/dist.py
 * global_merge_many). */
int nvtb_partition_by_owner_async(const int64_t* keys, int64_t n, int n_parts,
                                  int64_t* perm_out, int64_t* part_counts_dev, void* stream);
int nvtb_gather_i64(const int64_t* src, const int64_t* perm, int64_t n,
                    int64_t* dst, void* stream);
int nvtb_gather_f64_rows(const double* src, const int64_t* perm, int64_t n,
                         int row_width, double* dst, void* stream);

/* ---- vocabulary: ordering, cut, lookup table, encode ----------------------
 * nvtb_vocab_build replaces _write_uniques + _save_encodings (reference
 * nvtabular/ops/categorify.py:1149-1337, 719-822): order the (key,size) rows
 * by (size desc, key asc), apply freq_threshold (keep size >= t) or max_size
 * (keep the first max_size - (num_buckets or 1) - 2), and build the
 * key -> position lookup used by the encode.  keys/sizes are device arrays of
 * length n (unordered, distinct keys, null group NOT included).
 *
 * nvtb_vocab_from_arrays: keys already in label order (user `vocabs=`,
 * categorify.py:421-454, or a unique.<col>.parquet read back); sizes may be
 * NULL.
 */
typedef struct nvtb_vocab nvtb_vocab_t;
typedef struct {
  int64_t n_kept;      /* rows written to unique.<col>.parquet            */
  int64_t n_total;     /* distinct non-null keys seen                     */
  int64_t null_size;   /* meta num_observed[null]                         */
  int64_t oov_size;    /* meta num_observed[oov]: rows of dropped keys    */
  int64_t unique_size; /* meta num_observed[unique]                       */
} nvtb_vocab_info_t;
/* key_bits: 32 when every key is known to be an int32 value (halves the radix passes),
 * else 0; size_bound: an upper bound on any size (e.g. rows seen), 0 = unknown.
 * Both are speed hints only.  The build is ENQUEUED: n_kept and the meta numbers are read
 * back by the first nvtb_vocab_info / export / encode call on the handle. */
int nvtb_vocab_build(nvtb_vocab_t** out, const int64_t* keys,
                     const int64_t* sizes, int64_t n, int64_t null_size,
                     int64_t freq_threshold, int64_t max_size,
                     int64_t num_buckets, int key_bits, int64_t size_bound,
                     void* stream);
/* the same straight from a group-by handle (single GPU: _write_uniques reads the result of
 * _bottom_level_groupby without leaving the device, categorify.py:1149-1337).  A handle
 * holding a sorted accumulator is already in key order, so the ordering is one stable
 * radix sort on the size bits in use; null_size comes from the handle. */
int nvtb_vocab_build_from_hashagg(nvtb_vocab_t** out, nvtb_hashagg_t* h,
                                  int64_t freq_threshold, int64_t max_size,
                                  int64_t num_buckets, int key_bits, int64_t size_bound,
                                  void* stream);
/* the same from packed pairs that are ALREADY in (count desc, key asc) order (assembled by the
 * cross-GPU merge); the array is copied */
int nvtb_vocab_build_from_pairs(nvtb_vocab_t** out, const uint64_t* ordered_pairs, int64_t n,
                                int64_t null_size, int64_t freq_threshold, int64_t max_size,
                                int64_t num_buckets, void* stream);
int nvtb_vocab_from_arrays(nvtb_vocab_t** out, const int64_t* keys,
                           const int64_t* sizes, int64_t n, void* stream);
int nvtb_vocab_destroy(nvtb_vocab_t* v);
int nvtb_vocab_info(const nvtb_vocab_t* v, nvtb_vocab_info_t* info_host);
/* copy the kept keys / sizes in label order into caller device arrays */
int nvtb_vocab_export(const nvtb_vocab_t* v, int64_t* keys_out,
                      int64_t* sizes_out, void* stream);

/* ---- Categorify artefact files (csrc/artifacts.cu, host only) ---------------------------
 * meta.<col>.parquet and unique.<col>.parquet (reference nvtabular/ops/categorify.py:731-822)
 * written by library threads instead of pandas / pyarrow calls under the GIL.  The files are
 * what DataFrame.to_parquet(compression=None) writes, reduced to what pandas needs to read them
 * back: one row group, PLAIN, uncompressed v1 data pages of about 1 MiB per OPTIONAL column (no
 * dictionary pages, no statistics), and the `pandas` schema metadata, which carries the RangeIndex of the
 * labels.  Column types: INT32, INT64, FLOAT, DOUBLE, and BYTE_ARRAY + UTF8 for the meta
 * file's `kind` column.
 *
 * nvtb_parquet_write: host arrays -> one file.  cols_host[c].data holds n values of dtype
 * I32 | I64 | F32 | F64.  pandas_meta: the JSON stored under the `pandas` key (may be NULL).
 * page_rows: values per data page, 0 = pages of about 1 MiB. */
typedef struct {
  const char* name;
  const void* data;   /* host */
  int32_t dtype;      /* nvtb_dtype_t */
  int32_t _pad;
} nvtb_pq_col_t;
int nvtb_parquet_write(const char* path, const nvtb_pq_col_t* cols_host, int ncols, int64_t n,
                       const char* pandas_meta, int64_t page_rows);
/* meta.<col>.parquet of a vocabulary from its (host) info: kind = pad, null, oov, unique;
 * offset = 0, 1, 2, 2 + oov_count; num_indices = 1, 1, oov_count, n_kept; with_observed != 0
 * adds num_observed = 0, null_size, oov_size, unique_size.  oov_count = num_buckets or 1. */
int nvtb_parquet_write_meta(const char* path, int64_t oov_count, const nvtb_vocab_info_t* info_host,
                            int with_observed, const char* pandas_meta);
/* An asynchronous batch of vocabulary files.  begin starts `threads` writer threads (>= 1).
 * submit_vocab returns at once and never waits for the device.  Jobs run as their vocabularies'
 * builds finish (the event the enqueued build records, or, for a handle without one, an event
 * recorded here on `stream`), not in submission order: a writer thread takes the first queued
 * job whose event has fired, reads the vocabulary's scalars, copies the kept keys / sizes to the host
 * through library-owned pinned memory on a stream of its own, decodes the keys and writes
 *   meta_path    kind (pad, null, oov, unique), offset, num_indices [, num_observed when
 *                size_name != NULL]; meta_pandas is its `pandas` metadata;
 *   unique_path  (may be NULL) key_name [, size_name] with the kept rows, when the handle saw at
 *                least one key and unique_max_rows < 0 or n_kept <= unique_max_rows; its
 *                `pandas` metadata is unique_pandas_head + decimal(index_start + n_kept) +
 *                unique_pandas_tail (the stop of the RangeIndex is only known then).
 * key_dtype is the dtype of the written keys: I32 | I64 (int keys, written as they are) or
 * F32 | F64 (float keys: the order-preserving int64 image of a float64, k >= 0 ? k :
 * k ^ INT64_MAX, turned back into the float64 and cast).  oov_count = num_buckets or 1.
 * join waits for every job, stops the threads, frees the handle, and returns the status of the
 * first submitted job that failed (nvtb_last_error() names its path).  The vocabulary handles
 * must outlive the join. */
typedef struct nvtb_artifacts nvtb_artifacts_t;
int nvtb_artifacts_begin(nvtb_artifacts_t** out, int threads);
int nvtb_artifacts_submit_vocab(nvtb_artifacts_t* h, const nvtb_vocab_t* v, const char* meta_path,
                                const char* meta_pandas, const char* unique_path,
                                int64_t unique_max_rows, const char* key_name, int key_dtype,
                                const char* size_name, int64_t index_start, int64_t oov_count,
                                const char* unique_pandas_head, const char* unique_pandas_tail,
                                void* stream);
int nvtb_artifacts_join(nvtb_artifacts_t* h);

/* _encode (reference nvtabular/ops/categorify.py:1558-1807), without the
 * join + sort: label = null_label for null rows; first_label + position for
 * keys in the vocab; otherwise oov_label (+ hash(key) % num_buckets when
 * num_buckets > 1, categorify.py:1709-1715).  For the default layout
 * null_label=1, oov_label=2, first_label=2+(num_buckets or 1); single_table
 * shifts all three (categorify.py:1683-1685).  hash_cols_host: the original
 * column(s) to hash for OOV (NULL = hash `key` itself); out_dtype I32|I64. */
int nvtb_encode_apply(const nvtb_vocab_t* v, const nvtb_col_t* key_host,
                      int64_t n, int64_t null_label, int64_t oov_label,
                      int64_t first_label, uint64_t num_buckets,
                      const nvtb_col_t* hash_cols_host, int n_hash_cols,
                      void* out, int out_dtype, void* stream);

/* ---- group statistics gather: JoinGroupby / TargetEncoding transforms -----
 * Replaces the left-merge + sort_values("__tmp__") of reference
 * nvtabular/ops/join_groupby.py:200-215 and target_encoding.py:357-384.
 * The handle maps key -> row of a caller-provided stats matrix (device,
 * row-major double[n_groups][width]); nvtb_groupstats_gather writes, for
 * column j of the matrix, out[j][i] = stats[row(key_i)][j] cast to
 * out_dtypes[j] (I32|I64|F32|F64), or miss_vals[j] (NaN == null; the global
 * mean for TargetEncoding, target_encoding.py:378-380) when the key is
 * absent.  valid_out (NULL, or one entry per output column, each NULL or a
 * device bitmask of ceil(n / 32) 4-byte-aligned words): bit i set (Arrow
 * layout, LSB first) when key i has a row and that value is not NaN.  An
 * integer output holds 0 where the bit is clear. */
typedef struct nvtb_groupstats nvtb_groupstats_t;
/* null_row: row of `stats` that null keys join to (pandas/cuDF merge matches
 * null with null, and dropna=False makes the null key a group), or -1. */
int nvtb_groupstats_create(nvtb_groupstats_t** out, const int64_t* keys,
                           int64_t n_groups, const double* stats, int width,
                           int64_t null_row, void* stream);
int nvtb_groupstats_destroy(nvtb_groupstats_t* g);
int nvtb_groupstats_gather(const nvtb_groupstats_t* g,
                           const nvtb_col_t* key_host, int64_t n,
                           const int* cols_host, int ncols_out,
                           const double* miss_vals_host,
                           void* const* out_host, const int* out_dtypes_host,
                           uint8_t* const* valid_out_host, void* stream);

/* ---- row gather: the columns of Groupby, shuffle_by_keys, JoinExternal and Filter (csrc/gather.cu)
 * Output i (i < m) reads position p = i (which 0), off[i] (1, a segment's first position) or
 * off[i + 1] - 1 (2, its last), and row = pos ? pos[p] & row_mask : p.  A negative row (pos[p] = -1
 * under an all-ones mask: an unmatched join row) writes 0 and a null.  Group-by callers pass the
 * rows their ordered elements carry, row_mask = 2^row_bits - 1. */
typedef struct {
  const int64_t* pos;      /* may be NULL */
  uint64_t row_mask;
  const int64_t* off;      /* segment offsets; needed for which 1 and 2 */
  int32_t which;
  int32_t _pad;
} nvtb_row_sel_t;
/* For k < ncols (<= 16) fixed-width columns (1, 4 or 8 bytes), outs[k][i] = cols[k][row(i)], exact
 * for every width.  valids (NULL, or per column NULL or ceil(m/8) bitmask bytes, overwritten)
 * receive the output validity: bit i set when row(i) >= 0 and the source is valid there.  Bit k of
 * canon_zero: column k is a float key, -0.0 is written as +0.0.  The 4/8-byte outputs 32-byte
 * aligned, 1-byte outputs 8-byte aligned; pos has no alignment requirement. */
int nvtb_gather_rows(const nvtb_col_t* cols, int ncols, const nvtb_row_sel_t* sel, int64_t m,
                     void* const* outs, uint8_t* const* valids, uint32_t canon_zero, void* stream);

/* ---- session group-by: Groupby operator and Dataset.shuffle_by_keys (csrc/groupby.cu, K8) ----
 * Per partition, replaces the cuDF / pandas calls of reference nvtabular/ops/groupby.py:
 * df.sort_values(sort_cols, ascending) (groupby.py:118-120), df.groupby(groupby_cols).agg(...)
 * (groupby.py:222-227) and _first_or_last's list.get(0) / list.get(-1) (groupby.py:290-313).
 *
 * nvtb_gb_order_codes: one pass over a column -> codes_out[i], a uint64 whose unsigned order is
 * the column's order (int: sign bit flipped; float: order-preserving image with -0.0 made +0.0;
 * uint8: the value; a string column passes its int32 dictionary codes), valid_out (bitmask,
 * ceil(n/8) bytes: clear for a null or NaN row), and stats_dev[3] = {min, max, n_valid} of the
 * valid codes.  key_valid (may be NULL) receives the bitmask too, ANDed into it when
 * and_key_valid != 0 (the "every key is valid" mask of a multi-column key).  codes_out 32-byte
 * aligned. */
int nvtb_gb_order_codes(const nvtb_col_t* col, int64_t n, uint64_t* codes_out, uint8_t* valid_out,
                        uint8_t* key_valid, int and_key_valid, uint64_t* stats_dev, void* stream);
/* One chunk of one field of a row-ordering round.  A field's value for a row:
 *   mode 0  codes[row] - min                          (a group key; null-key rows are flagged)
 *   mode 1  valid ? codes[row] - min : span + 1        (ascending, nulls last)
 *   mode 2  valid ? span - (codes[row] - min) : span + 1  (descending, nulls last)
 *   mode 3  valid ? 0 : 1                              (a null flag)
 * and the chunk takes bits [lo, lo + nbits) of it. */
typedef struct {
  const uint64_t* codes;
  const uint8_t* valid;
  uint64_t min;
  uint64_t span;
  int32_t mode;
  int32_t lo;
  int32_t nbits;
  int32_t _pad;
} nvtb_gb_chunk_t;
/* Order rows 0..n-1 by fields F1 > F2 > ...: elements (packed fields << row_bits) | row are
 * sorted by LSD rounds; round k packs round_sizes_host[k] consecutive chunks of chunks_host
 * (least significant first, at most 64 - row_bits bits) and sorts those bits with the stable
 * radix primitive (radix.cuh).  Later rounds rewrite the high bits in place from the row, so
 * stability carries the earlier rounds.  The round plan comes from the host
 * (nvtabular_b200/ops/groupby.py plan_rounds).  No rounds: elements are the rows in order.
 * The result ends in elems (*result_in_tmp_host = 0) or tmp (1).  n < 2^32. */
int nvtb_gb_order_rows(const nvtb_gb_chunk_t* chunks_host, const int* round_sizes_host, int n_rounds,
                       int64_t n, int row_bits, uint64_t* elems, uint64_t* tmp,
                       int* result_in_tmp_host, void* stream);
/* Segments of the ordered rows: a position starts a group when its row's keys are all valid
 * (key_valid, NULL = all) and one of the n_keys key codes differs from the previous position's.
 * flags: ceil(n/8) bytes; tile_scan: ceil(n/2048) uint32.  counts_host = {groups, rows with valid
 * keys}.  Synchronises.  nvtb_gb_segments_write then writes off_out[groups + 1] (int64). */
int nvtb_gb_segments_count(const uint64_t* order, int64_t n, int row_bits,
                           const uint64_t* const* key_codes_host, int n_keys,
                           const uint8_t* key_valid, uint8_t* flags, uint32_t* tile_scan,
                           int64_t* counts_host, void* stream);
int nvtb_gb_segments_write(const uint8_t* flags, const uint32_t* tile_scan, int64_t n,
                           int64_t n_groups, int64_t n_kept, int64_t* off_out, void* stream);
/* gid_out[p] = g for off[g] <= p < off[g + 1], p < n */
int nvtb_gb_segment_ids(const int64_t* off, int64_t n_groups, int64_t n, uint64_t* gid_out,
                        void* stream);
/* Per segment [off[g], off[g+1]) of a column in group order, over its valid non-NaN values, in
 * fp64 and a fixed order: outs_host[7] = {count int32, sum f32, mean f32, var f32, std f32
 * (ddof 1, two passes), min, max (the column's dtype)}; NULL entries are skipped.  sum of no
 * values is 0; mean / min / max of none are NaN; var / std of fewer than 2 are NaN.  valid_host
 * (NULL or 2 zeroed bitmasks, 4-byte aligned): bit g set when the integer min / max of g exists. */
int nvtb_gb_reduce(const nvtb_col_t* col, const int64_t* off, int64_t n_groups,
                   void* const* outs_host, uint8_t* const* valid_host, void* stream);
/* median (f32; the fp64 mean of the two middle values at an even count) and nunique (int32) per
 * segment, from positions `order` sorted by (group, value code) with null values last in a group
 * (nvtb_gb_order_rows), codes / codes_valid from nvtb_gb_order_codes of col.  Either output may
 * be NULL. */
int nvtb_gb_rank_stats(const nvtb_col_t* col, const uint64_t* codes, const uint8_t* codes_valid,
                       const uint64_t* order, uint64_t row_mask, const int64_t* off,
                       int64_t n_groups, float* median_out, int32_t* nunique_out, void* stream);

/* Sub-lists [lo[g], hi[g]) of a list column's leaves, concatenated (first / last of a list input
 * column, reference test_groupby_list_first_last; the unpadded ListSlice).  Called twice: with
 * out == NULL it writes off_out[m + 1] and *total_host (a multi-CTA scan; synchronises); then with
 * out (total_host leaves of the leaf dtype) and out_valid (NULL, or ceil(total_host / 8) bitmask
 * bytes, which it overwrites) it copies the leaves, balanced over output elements. */
int nvtb_gb_list_rows(const nvtb_col_t* leaves, const int64_t* lo, const int64_t* hi, int64_t m,
                      int64_t* off_out, void* out, uint8_t* out_valid, int64_t* total_host,
                      void* stream);

/* ---- session operators: ListSlice and DifferenceLag (csrc/session.cu, K10) -----------------
 * nvtb_list_slice_bounds (reference nvtabular/ops/list_slice.py:78-144 and its GPU kernel
 * _calculate_row_sizes, list_slice.py:180-198): for every row i of a list column with offsets[n + 1],
 * [lo_out[i], hi_out[i]) is the absolute leaf range of Python's row[start:end]: a negative index
 * counts from the row end, both ends are clamped to [0, len] and hi >= lo.  nvtb_gb_list_rows over
 * these bounds is the unpadded slice. */
int nvtb_list_slice_bounds(const int64_t* offsets, int64_t n, int64_t start, int64_t end,
                           int64_t* lo_out, int64_t* hi_out, void* stream);
/* nvtb_list_slice_pad (list_slice.py:78-144 with pad=True, and _slice_rows, list_slice.py:201-228):
 * the dense n x L slice: out[i * L + k] = row i's k-th element of row[start:end] for k below its
 * length, else the pad value (pad_bits: the value's bit pattern in the leaf dtype, low bytes),
 * which is valid.  Copied elements carry the leaf validity (out_valid: NULL when the leaves have
 * none, else ceil(n * L / 8) bytes).  off_out[n + 1] = i * L.  out 32-byte aligned (1-byte
 * leaves: 8-byte).  No scan and no host read. */
int nvtb_list_slice_pad(const nvtb_col_t* leaves, const int64_t* offsets, int64_t n, int64_t start,
                        int64_t end, int64_t L, uint64_t pad_bits, void* out, uint8_t* out_valid,
                        int64_t* off_out, void* stream);
/* nvtb_lag_same_key (reference nvtabular/ops/difference_lag.py:65-75, the partition mask): bit i of
 * same_out (ceil(n/8) bytes) is set when 0 <= i - shift < n and every one of the n_keys (<= 8) key
 * columns is valid and equal at i and i - shift.  Floats compare with IEEE == (-0.0 == +0.0, NaN
 * equals nothing); integers, uint8 and string codes compare by value. */
int nvtb_lag_same_key(const nvtb_col_t* keys, int n_keys, int64_t n, int64_t shift, uint8_t* same_out,
                      void* stream);
/* nvtb_difference_lag (difference_lag.py:76-80): for k < ncols (<= 16) value columns (int32, int64,
 * uint8, float32, float64), outs[k][i] = x[i] - x[i - shift] as float32 where bit i of `same`
 * (nvtb_lag_same_key with the same n and shift) is set and both values are valid; otherwise 0 and
 * a cleared bit of out_valids[k] (ceil(n/8) bytes each).  Integers subtract in int64 (wrapping)
 * and round once; float32 subtracts in float32; float64 in float64, then rounds once.  Outputs
 * 32-byte aligned. */
int nvtb_difference_lag(const nvtb_col_t* cols, int ncols, int64_t n, int64_t shift, const uint8_t* same,
                        float* const* outs, uint8_t* const* out_valids, void* stream);

/* ---- row selection: Filter and Dropna (csrc/filter.cu, K11) ---------------------------------
 * A mask is a bitmask in the validity layout: bit (i & 7) of byte (i >> 3) is row i, and it is
 * padded to whole 32-byte blocks like pack_validity: ((ceil(n / 8) + 31) / 32) * 32 bytes.  The
 * mask writers fill every byte of that padding and leave the bits at rows >= n zero.  Every entry
 * point returns NVTB_OK for n = 0 without touching its outputs. */
typedef enum {
  NVTB_CMP_EQ = 0,
  NVTB_CMP_NE = 1,
  NVTB_CMP_LT = 2,
  NVTB_CMP_LE = 3,
  NVTB_CMP_GT = 4,
  NVTB_CMP_GE = 5
} nvtb_cmp_op_t;
typedef enum { NVTB_MASK_AND = 0, NVTB_MASK_OR = 1, NVTB_MASK_XOR = 2, NVTB_MASK_NOT = 3 } nvtb_mask_op_t;
/* nvtb_mask_compare (reference nvtabular/ops/filter.py:51-55, the comparisons f(df) makes, i.e.
 * pandas `df[c] op x`): bit i = a[i] op (b ? b[i] : scalar).  Both operands are converted to
 * cmp_type (NVTB_I64, NVTB_F32 or NVTB_F64; I64 only when neither operand is a float), and
 * scalar_bits is the scalar's bit pattern in cmp_type (low bytes).  A null operand, like a NaN,
 * gives true for NVTB_CMP_NE and false for every other op.  a and b: int32, int64, float32,
 * float64 or uint8 columns of n rows. */
int nvtb_mask_compare(const nvtb_col_t* a, const nvtb_col_t* b, int op, int cmp_type, uint64_t scalar_bits,
                      int64_t n, uint8_t* mask_out, void* stream);
/* nvtb_mask_notnull (reference nvtabular/ops/dropna.py:33-37, df.dropna(subset=cols); pandas
 * notnull): bit i is set when each of the ncols (<= 16) columns is valid at row i and, if it is a
 * float, not NaN there. */
int nvtb_mask_notnull(const nvtb_col_t* cols, int ncols, int64_t n, uint8_t* mask_out, void* stream);
/* nvtb_mask_logic (filter.py:51-55, pandas & | ^ ~ of bool Series): out = a op b, or ~a for
 * NVTB_MASK_NOT (b unused).  Masks 16-byte aligned; out aliases neither input. */
int nvtb_mask_logic(const uint8_t* a, const uint8_t* b, int64_t n, int op, uint8_t* out, void* stream);
/* nvtb_mask_count (filter.py:56-60 and dropna.py:35, the length of the indexed frame): tile_off
 * (ceil(n / 2048) + 1 int64, 32-byte aligned) receives the exclusive scan of the set bits of every
 * 2048-row tile and *n_kept_host their total.  Bits at rows >= n are ignored.  Mask 8-byte
 * aligned.  Synchronises the stream. */
int nvtb_mask_count(const uint8_t* mask, int64_t n, int64_t* tile_off, int64_t* n_kept_host, void* stream);
/* nvtb_mask_select (pandas boolean indexing, df[mask], then reset_index(drop=True)): rows_out
 * (n_kept int64) receives the rows whose bit is set, in ascending order, from nvtb_mask_count's
 * tile_off.  No atomics: the output is deterministic.  Moving the columns to those rows is
 * nvtb_gather_rows (fixed width) and nvtb_gb_list_rows (lists). */
int nvtb_mask_select(const uint8_t* mask, int64_t n, const int64_t* tile_off, int64_t* rows_out, void* stream);

/* ---- external-table join: JoinExternal operator (csrc/join.cu, K9) -------------------------
 * Replaces, per partition, reference nvtabular/ops/join_external.py:148-164: df.merge(ext,
 * left_on=on, right_on=on_ext, how=how) followed by sort_values("__tmp__") back to row order.
 * Output rows follow left-row order, and the matches of one left row follow ext-table order.
 *
 * nvtb_join_create (join_external.py:148-164, the build side of the merge; once per operator):
 * distinct_keys[n_groups] (int64) are the distinct valid ext keys, and run g of the ext rows in
 * key order is ordered_rows[off[g] .. off[g + 1]) (off: n_groups + 1 int64), as the K8 calls
 * nvtb_gb_order_codes / nvtb_gb_order_rows / nvtb_gb_segments leave them (stable: ext order
 * within a key).  ordered_rows[null_lo .. null_hi) are the null-key ext rows, which null left
 * keys join.  The handle copies off and ordered_rows and builds a wide table key -> run.
 * n_ext < 2^31 (NVTB_EINVAL otherwise).  Synchronises. */
typedef struct nvtb_join nvtb_join_t;
int nvtb_join_create(nvtb_join_t** out, const int64_t* distinct_keys, int64_t n_groups,
                     const int64_t* off, const int64_t* ordered_rows, int64_t n_ext,
                     int64_t null_lo, int64_t null_hi, void* stream);
/* n_groups and the largest run (null run included): 1 or less means every ext key is unique */
int nvtb_join_info(const nvtb_join_t* j, int64_t* n_groups, int64_t* max_group);
int nvtb_join_destroy(nvtb_join_t* j);
/* Probe (join_external.py:148-164, the probe side of the merge): one pass over key (int32 or
 * int64; a null row joins the null run).  how 0 = left, 1 = inner.
 *   off_out == NULL: ext_row_out[i] = the ext row matching row i, or -1; *n_out_host = n.  This is
 *     the whole join for a left join whose ext keys are unique.
 *   otherwise: ext_row_out[i] = the position of row i's first match in key order, or -1, and
 *     off_out[n + 1] (int64, 32-byte aligned) the exclusive scan of the rows each left row emits
 *     (its match count; at least 1 in a left join); *n_out_host = off_out[n].  Synchronises. */
int nvtb_join_probe(const nvtb_join_t* j, const nvtb_col_t* key, int64_t n, int how,
                    int64_t* ext_row_out, int64_t* off_out, int64_t* n_out_host, void* stream);
/* Expand (join_external.py:148-164, the rows the merge emits, already in left-row order): for
 * every output row p < n_out, left_rows[p] = its left row and ext_rows[p] = its ext row (-1 for
 * the unmatched row of a left join), from the probe's ext_row_first and off.  Balanced over
 * output rows.  Outputs 32-byte aligned. */
int nvtb_join_expand(const nvtb_join_t* j, const int64_t* ext_row_first, const int64_t* off,
                     int64_t n, int64_t n_out, int64_t* left_rows, int64_t* ext_rows, void* stream);
/* The merged columns (join_external.py:148-164) are nvtb_gather_rows of the left columns at
 * left_rows and of the ext columns at ext_rows (pos = the rows, an all-ones row_mask), and
 * nvtb_gb_list_rows over the gathered offsets of a list column. */

/* ---- cross-GPU collectives of the fit path (SURVEY.md 8e) ---------------------------------
 * nvtb_comm_t wraps an ncclComm_t: created here (rank 0 makes a unique id, the host runtime
 * hands it to every rank — torch.distributed broadcast, MPI, a file) or provided by the caller.
 * These are all the exchanges the path has: moments all-reduce, variable-block all-to-all of
 * group-by partials, all-gather of vocabulary shards.  They replace the dask tree reduction and
 * the shared-filesystem broadcast of reference nvtabular/ops/categorify.py:1399-1540, 1627-1643
 * and ops/moments.py:34-57.  Stream-ordered; NVTB_ENCCL on failure. */
typedef struct nvtb_comm nvtb_comm_t;
int nvtb_comm_available(void);
int nvtb_comm_unique_id(uint8_t* id_out128);
int nvtb_comm_create(nvtb_comm_t** out, const uint8_t* id128, int rank, int world);
int nvtb_comm_wrap(nvtb_comm_t** out, void* nccl_comm, int rank, int world);
int nvtb_comm_destroy(nvtb_comm_t* c);
int nvtb_comm_rank(const nvtb_comm_t* c, int* rank, int* world);
/* in place; op: 0 sum, 1 min, 2 max */
int nvtb_comm_allreduce_f64(nvtb_comm_t* c, double* buf_dev, int64_t n, int op, void* stream);
int nvtb_comm_allreduce_i64(nvtb_comm_t* c, int64_t* buf_dev, int64_t n, int op, void* stream);
/* acc_dev: [ncols][5] = {count, sum, sumsq, min, max} (nvtb_moments_accumulate's accumulator) */
int nvtb_moments_allreduce(nvtb_comm_t* c, double* acc_dev, int ncols, void* stream);
/* recv holds world blocks of `bytes` bytes in rank order */
int nvtb_comm_allgather(nvtb_comm_t* c, const void* send_dev, void* recv_dev, int64_t bytes, void* stream);
/* send_counts_host[r] elements (elem_bytes each, consecutive in send) go to rank r;
 * recv_counts_host[r] arrive from rank r (consecutive in recv) */
int nvtb_comm_alltoallv(nvtb_comm_t* c, const void* send_dev, const int64_t* send_counts_host,
                        void* recv_dev, const int64_t* recv_counts_host, int elem_bytes, void* stream);

/* ---- inference-time transforms on HOST arrays --------------------------------------------
 * The twin of the reference's pybind11 module nvtabular_cpp.inference
 * (cpp/nvtabular/inference/categorify.cc:31-347, fill.cc:32-124; bound at
 * nvtabular/ops/categorify.py:602-609, ops/fill.py:59-65): dict-of-numpy requests of a serving
 * process are encoded by probing a host table of the kept keys (built once from the device
 * vocabulary) with a few host threads — a serving batch is too small to pay for a PCIe round
 * trip.  Labels are identical to nvtb_encode_apply's. */
typedef struct nvtb_infer_vocab nvtb_infer_vocab_t;
/* label = first_label + position of the key in keys_host */
int nvtb_infer_vocab_create(nvtb_infer_vocab_t** out, const int64_t* keys_host, int64_t n);
int nvtb_infer_vocab_from_device(nvtb_infer_vocab_t** out, const nvtb_vocab_t* v, void* stream);
int nvtb_infer_vocab_destroy(nvtb_infer_vocab_t* v);
/* keys_host: int32 | int64 [n]; validity_host: Arrow bitmask or NULL; labels_out_host: int32 |
 * int64 [n]; n_threads <= 0: hardware concurrency (one thread per 16 Ki rows at most) */
int nvtb_infer_categorify_host(const nvtb_infer_vocab_t* v, const void* keys_host, int key_dtype,
                               const uint8_t* validity_host, int64_t n, int64_t null_label,
                               int64_t oov_label, int64_t first_label, uint64_t num_buckets,
                               void* labels_out_host, int out_dtype, int n_threads);
/* FillMissing in place on a host float32 / float64 array (NaN -> fill); integer arrays pass */
int nvtb_infer_fill_host(void* data_host, int dtype, int64_t n, double fill);

#ifdef __cplusplus
}
#endif
#endif /* NVTB200_H */
