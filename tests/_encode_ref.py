"""Exact reference of the vocabulary encode (K5) and the group-statistics gather (K7), and numpy
replicas of the engine's table hashes, used to BUILD keys that reach given probe branches.

Reference (independent of the engine):

* label of a row = `null_label` when the row is null; else `first_label + pos` when the key is
  at position `pos` of the exported vocabulary (a repeated key: its smallest position); else
  `oov_label + h % num_buckets` when `num_buckets > 1`, else `oov_label`.
* `h` = the pandas value hash of the key (`oracle.hashing.hash_values`: the key's bits in its
  own width, zero-extended), or with hash columns the XOR over the columns of that hash, where a
  null hashes as the float64 NaN bits and an H64 column already is a hash.

Replicas (uint32 / uint64 numpy arithmetic, wrapping on purpose):

* `table_mix32` / `table_mix64`: murmur3 fmix32 / fmix64 (csrc/common.cuh `table_mix32`,
  `table_mix64`: constants 0x85EBCA6B, 0xC2B2AE35 / 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53),
  and their inverses (an xor-shift by s >= half the width is its own inverse; a shorter one is
  undone by repeating it; a multiplication by the odd constant's inverse mod 2^w).
* `fold_hash` / `fold_unhash`: csrc/common.cuh (kFoldC1 = 0x9E3779B1, kFoldC2 = 0x85EBCA6B,
  kFoldEmpty = 0xFFFFFFFF is the one h never stored in shared memory).
* home buckets: narrow = table_mix32(key) & (nbuckets - 1), wide = table_mix64(key) & (cap - 1)
  (csrc/lookup.cuh `lookup_home`); shared-memory bucket = umulhi(fold_hash(key), 7168)
  (csrc/vocab.cu kEncSmemBuckets); `narrow_slice_buckets` (csrc/lookup.cuh, kSliceBuckets =
  kSliceParts = 8192).

tests/test_encode_replicas.py compares every replica with the header compiled on the host.
"""
import numpy as np

from oracle.hashing import NAN_BITS, _mix, hash_values

M32 = (1 << 32) - 1
M64 = (1 << 64) - 1

TM32_C1, TM32_C2 = 0x85EBCA6B, 0xC2B2AE35                       # common.cuh table_mix32
TM64_C1, TM64_C2 = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53       # common.cuh table_mix64
FOLD_C1, FOLD_C2 = 0x9E3779B1, 0x85EBCA6B                       # common.cuh kFoldC1, kFoldC2
FOLD_EMPTY = 0xFFFFFFFF                                         # common.cuh kFoldEmpty
SMEM_BUCKETS = 7168                                             # vocab.cu kEncSmemBuckets
SMEM_MAX_KEYS = 2 * SMEM_BUCKETS                                # vocab.cu kEncSmemMaxKeys
SLICE_BUCKETS = 8192                                            # lookup.cuh kSliceBuckets
SLICE_PARTS = 8192                                              # lookup.cuh kSliceParts


def _u32(x):
    return np.asarray(x).astype(np.int64).astype(np.uint32) if np.asarray(x).dtype.kind == "i" \
        else np.asarray(x, dtype=np.uint32)


def _u64(x):
    a = np.asarray(x)
    return a.astype(np.int64).view(np.uint64) if a.dtype.kind == "i" else a.astype(np.uint64)


def _inv(c, bits):
    return pow(c, -1, 1 << bits)


# ------------------------------------------------------------------ 32-bit mixers
def table_mix32(k):
    h = _u32(k).copy()
    with np.errstate(over="ignore"):
        h ^= h >> np.uint32(16)
        h *= np.uint32(TM32_C1)
        h ^= h >> np.uint32(13)
        h *= np.uint32(TM32_C2)
        h ^= h >> np.uint32(16)
    return h


def table_unmix32(h):
    k = _u32(h).copy()
    with np.errstate(over="ignore"):
        k ^= k >> np.uint32(16)
        k *= np.uint32(_inv(TM32_C2, 32))
        k ^= (k >> np.uint32(13)) ^ (k >> np.uint32(26))
        k *= np.uint32(_inv(TM32_C1, 32))
        k ^= k >> np.uint32(16)
    return k


def fold_hash(k):
    h = _u32(k).copy()
    with np.errstate(over="ignore"):
        h *= np.uint32(FOLD_C1)
        h ^= h >> np.uint32(15)
        h *= np.uint32(FOLD_C2)
    return h


def fold_unhash(h):
    k = _u32(h).copy()
    with np.errstate(over="ignore"):
        k *= np.uint32(_inv(FOLD_C2, 32))
        k ^= k >> np.uint32(15)
        k ^= k >> np.uint32(30)
        k *= np.uint32(_inv(FOLD_C1, 32))
    return k


def smem_bucket(k):
    """shared-memory bucket of int32 key k: __umulhi(fold_hash(k), 7168)"""
    return ((fold_hash(k).astype(np.uint64) * np.uint64(SMEM_BUCKETS)) >> np.uint64(32)).astype(np.int64)


# ------------------------------------------------------------------ 64-bit mixer
def table_mix64(k):
    h = _u64(k).copy()
    with np.errstate(over="ignore"):
        h ^= h >> np.uint64(33)
        h *= np.uint64(TM64_C1)
        h ^= h >> np.uint64(33)
        h *= np.uint64(TM64_C2)
        h ^= h >> np.uint64(33)
    return h


def table_unmix64(h):
    k = _u64(h).copy()
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(33)
        k *= np.uint64(_inv(TM64_C2, 64))
        k ^= k >> np.uint64(33)
        k *= np.uint64(_inv(TM64_C1, 64))
        k ^= k >> np.uint64(33)
    return k


# ------------------------------------------------------------------ table geometry
def narrow_slice_buckets(nbuckets: int) -> int:
    s = max(nbuckets // SLICE_PARTS, SLICE_BUCKETS)
    return min(s, nbuckets)


def narrow_next(b: int, nbuckets: int) -> int:
    sm = narrow_slice_buckets(nbuckets) - 1
    return (b & ~sm) | ((b + 1) & sm)


def narrow_home(k, nbuckets: int):
    return (table_mix32(k) & np.uint32(nbuckets - 1)).astype(np.int64)


def wide_home(k, cap: int):
    return (table_mix64(k) & np.uint64(cap - 1)).astype(np.int64)


# ------------------------------------------------------------------ adversarial keys
def narrow_chain(rng, low_bits: int, pattern: int, count: int):
    """`count` distinct int32 keys whose table_mix32 has `pattern` in its low `low_bits` bits:
    one home bucket in every narrow table of at most 2^low_bits buckets"""
    hi = rng.choice(1 << (32 - low_bits), count, replace=False).astype(np.uint64)
    h = ((hi << np.uint64(low_bits)) | np.uint64(pattern)).astype(np.uint32)
    return table_unmix32(h).view(np.int32)


def wide_chain(rng, low_bits: int, pattern: int, count: int):
    """`count` distinct int64 keys with one home slot in every wide table of <= 2^low_bits slots"""
    hi = rng.integers(1, 1 << 62, count, dtype=np.int64).astype(np.uint64)
    h = (hi << np.uint64(low_bits)) | np.uint64(pattern)
    return np.unique(table_unmix64(h).view(np.int64))[:count]


def smem_bucket_keys(bucket: int, count: int):
    """`count` int32 keys of shared-memory bucket `bucket` (consecutive h at the bucket's start)"""
    h0 = -((-bucket << 32) // SMEM_BUCKETS)                  # ceil(bucket * 2^32 / 7168)
    h = np.arange(h0, h0 + count, dtype=np.uint64).astype(np.uint32)
    keys = fold_unhash(h).view(np.int32)
    assert (smem_bucket(keys) == bucket).all()
    return keys


# ------------------------------------------------------------------ reference
def col_hash(values, null=None, prehashed=False):
    """uint64 hash of one hash column: pandas value hash, a null = the float64 NaN bits"""
    values = np.asarray(values)
    if prehashed:
        h = values.view(np.uint64).copy()
        if null is not None:
            h[null] = _mix(np.array([NAN_BITS]))[0]
        return h
    return hash_values(values, null)


def ref_labels(keys, null, vocab_keys, null_label, oov_label, first_label, num_buckets, hashes=None):
    """exact labels (int64) of `keys` (int32 / int64, `null`: True = null row) for a vocabulary
    whose exported keys are `vocab_keys` in label order; `hashes`: the XOR of the hash columns
    (None: the key's own value hash)"""
    keys = np.asarray(keys)
    k64 = keys.astype(np.int64)
    vk = np.asarray(vocab_keys, dtype=np.int64)
    uk, first = np.unique(vk, return_index=True)             # a repeated key: its first position
    idx_c = np.minimum(np.searchsorted(uk, k64), len(uk) - 1)   # the vocabulary is not empty
    found = uk[idx_c] == k64
    out = np.full(len(keys), oov_label, dtype=np.int64)
    if num_buckets and num_buckets > 1:
        h = hash_values(keys) if hashes is None else hashes
        out += (h % np.uint64(num_buckets)).astype(np.int64)
    out[found] = first_label + first[idx_c[found]]
    if null is not None:
        out[np.asarray(null, bool)] = null_label
    return out


def ref_rows(keys, null, group_keys, null_row):
    """stats row of every key: its group's row, `null_row` for a null key, -1 for none"""
    gk = np.asarray(group_keys, np.int64)                   # distinct, at least one
    order = np.argsort(gk)
    sk = gk[order]
    k64 = np.asarray(keys).astype(np.int64)
    idx = np.minimum(np.searchsorted(sk, k64), len(sk) - 1)
    row = np.where(sk[idx] == k64, order[idx], -1)
    if null is not None:
        row = np.where(null, null_row, row)
    return row


def ref_gather(row, stats, col, miss, out_dtype):
    """(values, valid) of one gathered output: column `col` of the stats row, `miss` where there is
    no row; integer outputs truncate toward zero and hold 0 for NaN; valid = there is a row and the
    value is not NaN"""
    v = np.where(row >= 0, stats[np.maximum(row, 0), col], miss)
    valid = (row >= 0) & ~np.isnan(v)
    dt = np.dtype(out_dtype)
    if dt.kind == "i":
        out = np.where(np.isnan(v), 0.0, np.trunc(v)).astype(dt)
    else:
        with np.errstate(over="ignore"):                        # beyond float32: inf
            out = v.astype(dt)
    return out, valid
