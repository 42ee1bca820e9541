"""Thin, typed Python face of the C-ABI (include/nvtb200.h): every function
here is one or two calls into libnvtb200.so on Column buffers.  The operator
classes in nvtabular_b200/ops are written against this module only.

No arithmetic happens in Python on row data; torch is used to allocate output
buffers and to read back O(#columns) scalars.
"""
import ctypes
import os
from ctypes import byref, c_int, c_int64, c_void_p
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _lib
from .column import Column

_CODE2TORCH = {_lib.I32: torch.int32, _lib.I64: torch.int64, _lib.F32: torch.float32,
               _lib.F64: torch.float64, _lib.U8: torch.uint8}
_NP2CODE = {np.dtype("int32"): _lib.I32, np.dtype("int64"): _lib.I64,
            np.dtype("float32"): _lib.F32, np.dtype("float64"): _lib.F64,
            np.dtype("uint8"): _lib.U8, np.dtype("bool"): _lib.U8}
NAN = float("nan")
kernel_launches = 0  # counted for bench.py's "gpu_launches"


def _count(n=1):
    global kernel_launches
    kernel_launches += n


# --- optional per-kernel-family device timing (bench.py's roofline object) -----
# When `profile` is a list, every wrapper below brackets its launch with CUDA
# events on the launching stream and appends (family, start, end, algorithmic
# bytes).  Events are only read after the timed region has been synchronised.
profile = None


class _timed:
    def __init__(self, family: str, nbytes: float):
        self.family, self.nbytes = family, nbytes

    def __enter__(self):
        if profile is not None:
            self.s = torch.cuda.Event(enable_timing=True)
            self.e = torch.cuda.Event(enable_timing=True)
            self.s.record()
        return self

    def __exit__(self, *exc):
        if profile is not None:
            self.e.record()
            profile.append((self.family, self.s, self.e, self.nbytes))
        return False


def _in_bytes(cols) -> float:
    """algorithmic read bytes: data + 1 validity bit per row (SURVEY.md §8d)."""
    return float(sum(c.data.numel() * (c.data.element_size() + 0.125) for c in cols))


def dtype_code(dt) -> int:
    if isinstance(dt, torch.dtype):
        return {v: k for k, v in _CODE2TORCH.items()}[dt]
    return _NP2CODE[np.dtype(dt)]


def _ptr(t: Optional[torch.Tensor]):
    return c_void_p(t.data_ptr()) if t is not None and t.numel() else None


def _fills(cols: Sequence[Column]):
    return _lib.double_array([NAN if c.fill is None else float(c.fill) for c in cols])


def _descs(cols: Sequence[Column]):
    return _lib.col_array([c.desc() for c in cols])


def _check_same_len(cols: Sequence[Column]) -> int:
    n = cols[0].data.numel()
    for c in cols:
        if c.data.numel() != n:
            raise ValueError("columns of one call must have the same length")
    return n


# ----------------------------------------------------------------- moments
class Moments:
    """Running {count, sum, sumsq, min, max} per column on the device
    (nvtb_moments_*; replaces nvtabular/ops/moments.py:28-116)."""

    def __init__(self, ncols: int, device=None):
        _lib.require_cuda()
        self.lib = _lib.load()
        self.ncols = ncols
        self.acc = torch.empty(ncols * 5, dtype=torch.float64, device=device or "cuda")
        _lib.check(self.lib.nvtb_moments_init(_ptr(self.acc), ncols, _lib.stream_ptr()))
        _count()

    def accumulate(self, cols: Sequence[Column]):
        assert len(cols) == self.ncols
        n = _check_same_len(cols)
        with _timed("moments", _in_bytes(cols)):
            _lib.check(self.lib.nvtb_moments_accumulate(
                _descs(cols), self.ncols, n, _fills(cols), _ptr(self.acc), _lib.stream_ptr()))
        _count(2)

    def allreduce(self):
        """Cross-GPU merge: one NCCL all-reduce of 3 sums + min + max per column
        (SURVEY.md §8e; replaces the dask tree of moments.py:45-55)."""
        import torch.distributed as dist
        from .dist import native_comm, world
        if world()[0] <= 1:
            return
        nc = native_comm()
        if nc is not None and self.acc.is_cuda:            # the library's own communicator (csrc/comm.cu)
            _lib.check(nc[0].nvtb_moments_allreduce(nc[1], _ptr(self.acc), self.ncols, _lib.stream_ptr()))
            _count()
            return
        a = self.acc.view(self.ncols, 5)
        sums = a[:, 0:3].contiguous()
        mn = a[:, 3].contiguous()
        mx = a[:, 4].contiguous()
        dist.all_reduce(sums, op=dist.ReduceOp.SUM)
        dist.all_reduce(mn, op=dist.ReduceOp.MIN)
        dist.all_reduce(mx, op=dist.ReduceOp.MAX)
        a[:, 0:3] = sums
        a[:, 3] = mn
        a[:, 4] = mx

    def result(self):
        """-> dict of numpy arrays: count,sum,sumsq,min,max,mean,var,std."""
        acc = self.acc.cpu().numpy().astype(np.float64)
        out = np.zeros(self.ncols * 3, dtype=np.float64)
        _lib.check(self.lib.nvtb_moments_finalize(
            acc.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), self.ncols,
            out.ctypes.data_as(ctypes.POINTER(ctypes.c_double))))
        a = acc.reshape(self.ncols, 5)
        o = out.reshape(self.ncols, 3)
        return {"count": a[:, 0], "sum": a[:, 1], "sumsq": a[:, 2], "min": a[:, 3], "max": a[:, 4],
                "mean": o[:, 0], "var": o[:, 1], "std": o[:, 2]}


# ------------------------------------------------------------- transforms
def _alloc_like(cols: Sequence[Column], dtype: torch.dtype) -> List[torch.Tensor]:
    return [torch.empty(c.data.numel(), dtype=dtype, device=c.data.device) for c in cols]


def fill_apply(cols: Sequence[Column], fill_vals: Sequence[float], add_binary_cols=False):
    """FillMissing (nvtb_fill_apply).  Returns (filled columns, indicator columns|None)."""
    _lib.require_cuda()
    lib = _lib.load()
    n = _check_same_len(cols)
    outs = [torch.empty_like(c.data) for c in cols]
    flags = [torch.empty(n, dtype=torch.uint8, device=c.data.device) for c in cols] if add_binary_cols else None
    _lib.check(lib.nvtb_fill_apply(
        _descs(cols), len(cols), n, _lib.double_array(fill_vals),
        _lib.ptr_array([o.data_ptr() for o in outs]),
        _lib.ptr_array([f.data_ptr() for f in flags]) if flags else None, _lib.stream_ptr()))
    _count()
    out_cols = [Column(o, None, c.offsets, None, None, c.is_bool) for o, c in zip(outs, cols)]
    flag_cols = [Column(f, None, c.offsets, is_bool=True) for f, c in zip(flags, cols)] if flags else None
    return out_cols, flag_cols


def normalize_apply(cols: Sequence[Column], means, stds, out_dtype=np.float64):
    _lib.require_cuda()
    lib = _lib.load()
    n = _check_same_len(cols)
    code = dtype_code(out_dtype)
    outs = _alloc_like(cols, _CODE2TORCH[code])
    with _timed("normalize", _in_bytes(cols) + sum(o.numel() * o.element_size() for o in outs)):
        _lib.check(lib.nvtb_normalize_apply(
            _descs(cols), len(cols), n, _fills(cols), _lib.double_array(means), _lib.double_array(stds),
            _lib.ptr_array([o.data_ptr() for o in outs]), code, _lib.stream_ptr()))
    _count()
    return [Column(o, None if c.fill is not None else c.validity, c.offsets) for o, c in zip(outs, cols)]


def minmax_apply(cols: Sequence[Column], mins, maxs, out_dtype=np.float64):
    _lib.require_cuda()
    lib = _lib.load()
    n = _check_same_len(cols)
    code = dtype_code(out_dtype)
    outs = _alloc_like(cols, _CODE2TORCH[code])
    _lib.check(lib.nvtb_minmax_apply(
        _descs(cols), len(cols), n, _fills(cols), _lib.double_array(mins), _lib.double_array(maxs),
        _lib.ptr_array([o.data_ptr() for o in outs]), code, _lib.stream_ptr()))
    _count()
    return [Column(o, None if c.fill is not None else c.validity, c.offsets) for o, c in zip(outs, cols)]


def cliplog_apply(cols: Sequence[Column], min_value=None, max_value=None, take_log=False, out_dtype=np.float32):
    """Clip (+ LogOp) with an upstream FillMissing fused in (nvtb_cliplog_apply).  take_log=False
    keeps every column's dtype; nulls that are not filled stay nulls."""
    _lib.require_cuda()
    lib = _lib.load()
    n = _check_same_len(cols)
    code = dtype_code(out_dtype) if take_log else 0
    outs = _alloc_like(cols, _CODE2TORCH[code]) if take_log else [torch.empty_like(c.data) for c in cols]
    lo = _lib.double_array([NAN if min_value is None else float(min_value)] * len(cols))
    hi = _lib.double_array([NAN if max_value is None else float(max_value)] * len(cols))
    with _timed("cliplog", _in_bytes(cols) + sum(o.numel() * o.element_size() for o in outs)):
        _lib.check(lib.nvtb_cliplog_apply(_descs(cols), len(cols), n, _fills(cols), lo, hi, 1 if take_log else 0,
                                          _lib.ptr_array([o.data_ptr() for o in outs]), code, _lib.stream_ptr()))
    _count()
    return [Column(o, None if c.fill is not None else c.validity, c.offsets, None, None, c.is_bool and not take_log)
            for o, c in zip(outs, cols)]


def hash_bucket(cols: Sequence[Column], num_buckets: int, add: int = 0, out_dtype=np.int32) -> torch.Tensor:
    """hash(cols...) % num_buckets + add (nvtb_hash_bucket_apply)."""
    _lib.require_cuda()
    lib = _lib.load()
    n = _check_same_len(cols)
    code = dtype_code(out_dtype)
    out = torch.empty(n, dtype=_CODE2TORCH[code], device=cols[0].data.device)
    with _timed("hash_bucket", _in_bytes(cols) + out.numel() * out.element_size()):
        _lib.check(lib.nvtb_hash_bucket_apply(_descs(cols), len(cols), n, int(num_buckets), int(add),
                                              _ptr(out), code, _lib.stream_ptr()))
    _count()
    return out


def hash_values(col: Column) -> torch.Tensor:
    """raw uint64 value hashes as an int64 tensor (bit pattern)."""
    _lib.require_cuda()
    lib = _lib.load()
    n = col.data.numel()
    out = torch.empty(n, dtype=torch.int64, device=col.data.device)
    _lib.check(lib.nvtb_hash_values(_descs([col]), n, _ptr(out), _lib.stream_ptr()))
    _count()
    return out


def pack_keys2(a: Column, b: Column) -> Column:
    """(a, b) int32 pair -> one order-preserving int64 key column."""
    _lib.require_cuda()
    lib = _lib.load()
    n = _check_same_len([a, b])
    keys = torch.empty(n, dtype=torch.int64, device=a.data.device)
    need_mask = a.validity is not None and b.validity is not None
    nbytes = (((n + 7) // 8 + 31) // 32) * 32
    mask = torch.zeros(nbytes, dtype=torch.uint8, device=a.data.device) if need_mask else None
    _lib.check(lib.nvtb_pack_keys2(_descs([a]), _descs([b]), n, _ptr(keys), _ptr(mask), _lib.stream_ptr()))
    _count()
    return Column(keys, mask)


def unpack_keys2(keys: np.ndarray):
    """host inverse of pack_keys2: int64 -> (a int32, b int32); INT32_MIN marks a null component."""
    k = keys.astype(np.int64)
    a = (k >> 32).astype(np.int32)
    b = ((k & 0xFFFFFFFF).astype(np.uint32) ^ np.uint32(0x80000000)).astype(np.uint32).view(np.int32)
    return a, b


# ------------------------------------------------------------- hash aggregation
class HashAgg:
    """groupby(key, dropna=False) -> size [, sum/sumsq/min/max per cont col]
    (nvtb_hashagg_*; replaces nvtabular/ops/categorify.py:955-1137)."""

    def __init__(self, n_agg: int = 0, capacity_hint: int = 0):
        _lib.require_cuda()
        self.lib = _lib.load()
        self.n_agg = n_agg
        self.h = c_void_p()
        _lib.check(self.lib.nvtb_hashagg_create(byref(self.h), n_agg, int(capacity_hint)))

    def __del__(self):
        try:
            if getattr(self, "h", None) is not None and self.h.value:
                self.lib.nvtb_hashagg_destroy(self.h)
                self.h = c_void_p()
        except Exception:
            pass

    def reset(self):
        _lib.check(self.lib.nvtb_hashagg_reset(self.h, _lib.stream_ptr()))
        _count(2)

    @property
    def mode(self) -> int:
        """0 = resident hash table, 1 = sorted accumulator (csrc/sortagg.cuh)"""
        m = c_int(0)
        _lib.check(self.lib.nvtb_hashagg_mode(self.h, byref(m)))
        return m.value

    def flush(self):
        """fold in whatever a sorted accumulator has staged (timed with the inserts: it is their cost)"""
        with _timed("hashagg_insert", 0.0):
            _lib.check(self.lib.nvtb_hashagg_flush(self.h, _lib.stream_ptr()))
        _count(12)

    def to_sorted(self):
        """make the handle a sorted accumulator (key-ordered packed pairs), see csrc/sortagg.cuh"""
        _lib.check(self.lib.nvtb_hashagg_to_sorted(self.h, _lib.stream_ptr()))
        _count(3)

    def export_packed(self, device="cuda") -> torch.Tensor:
        """packed pairs (key ^ 2^31) << 32 | count of a sorted accumulator, key order, as the bit
        pattern of an int64 tensor"""
        n = c_int64(0)
        _lib.check(self.lib.nvtb_hashagg_export_packed(self.h, None, byref(n), _lib.stream_ptr()))
        out = torch.empty(n.value, dtype=torch.int64, device=device)
        if n.value:
            _lib.check(self.lib.nvtb_hashagg_export_packed(self.h, _ptr(out), byref(n), _lib.stream_ptr()))
        return out

    def insert(self, key: Column, agg_cols: Sequence[Column] = ()):
        n = key.data.numel()
        assert len(agg_cols) == self.n_agg
        for c in agg_cols:
            assert c.data.numel() == n
        with _timed("hashagg_insert", _in_bytes([key]) + _in_bytes(agg_cols)):
            _lib.check(self.lib.nvtb_hashagg_insert(
                self.h, _descs([key]), _descs(agg_cols) if self.n_agg else None, n, _lib.stream_ptr()))
        _count(1)

    def merge(self, keys: torch.Tensor, sizes: torch.Tensor, vals: Optional[torch.Tensor] = None):
        n = keys.numel()
        _lib.check(self.lib.nvtb_hashagg_merge(self.h, _ptr(keys), _ptr(sizes), _ptr(vals), n, _lib.stream_ptr()))
        _count(1 if n else 0)

    def add_null_group(self, size: int, vals: Optional[np.ndarray] = None):
        arr = _lib.double_array(list(vals)) if vals is not None and self.n_agg else None
        _lib.check(self.lib.nvtb_hashagg_add_null_group(self.h, int(size), arr))

    def size(self):
        nu, ns = c_int64(0), c_int64(0)
        _lib.check(self.lib.nvtb_hashagg_size(self.h, byref(nu), byref(ns), _lib.stream_ptr()))
        return nu.value, ns.value

    def export(self, device="cuda"):
        """-> (keys int64[U], sizes int64[U], vals float64[U, n_agg, 4] | None,
                null_size, null_vals ndarray[n_agg,4] | None), unordered."""
        nu, ns = self.size()
        keys = torch.empty(nu, dtype=torch.int64, device=device)
        sizes = torch.empty(nu, dtype=torch.int64, device=device)
        vals = torch.empty((nu, self.n_agg, 4), dtype=torch.float64, device=device) if self.n_agg else None
        null_vals = (ctypes.c_double * (4 * max(self.n_agg, 1)))()
        with _timed("hashagg_export", float(nu * 16)):
            _lib.check(self.lib.nvtb_hashagg_export(self.h, _ptr(keys), _ptr(sizes), _ptr(vals),
                                                    null_vals if self.n_agg else None, _lib.stream_ptr()))
        _count()
        nv = np.array(list(null_vals), dtype=np.float64).reshape(-1, 4)[: self.n_agg] if self.n_agg else None
        return keys, sizes, vals, ns, nv


def partition_by_owner(keys: torch.Tensor, n_parts: int):
    """-> (perm int64[n], counts list[int]) grouping rows by hash-owner."""
    lib = _lib.load()
    n = keys.numel()
    perm = torch.empty(n, dtype=torch.int64, device=keys.device)
    counts = (c_int64 * n_parts)()
    _lib.check(lib.nvtb_partition_by_owner(_ptr(keys), n, n_parts, _ptr(perm), counts, _lib.stream_ptr()))
    _count(2)
    return perm, [int(c) for c in counts]


def partition_by_owner_async(keys: torch.Tensor, n_parts: int, counts_out: torch.Tensor):
    """-> perm int64[n]; the per-owner row counts go to `counts_out` (device int64[n_parts])
    without a host round trip."""
    lib = _lib.load()
    n = keys.numel()
    perm = torch.empty(n, dtype=torch.int64, device=keys.device)
    _lib.check(lib.nvtb_partition_by_owner_async(_ptr(keys), n, n_parts, _ptr(perm), _ptr(counts_out),
                                                 _lib.stream_ptr()))
    _count(3)
    return perm


def gather_i64(src: torch.Tensor, perm: torch.Tensor) -> torch.Tensor:
    lib = _lib.load()
    out = torch.empty(perm.numel(), dtype=torch.int64, device=src.device)
    _lib.check(lib.nvtb_gather_i64(_ptr(src), _ptr(perm), perm.numel(), _ptr(out), _lib.stream_ptr()))
    _count()
    return out


def gather_f64_rows(src: torch.Tensor, perm: torch.Tensor, width: int) -> torch.Tensor:
    lib = _lib.load()
    out = torch.empty((perm.numel(), width), dtype=torch.float64, device=src.device)
    _lib.check(lib.nvtb_gather_f64_rows(_ptr(src), _ptr(perm), perm.numel(), width, _ptr(out), _lib.stream_ptr()))
    _count()
    return out


# ------------------------------------------------------------------ vocabulary
class Vocab:
    """Ordered vocabulary + device lookup (nvtb_vocab_*; replaces
    _write_uniques/_save_encodings/_encode, categorify.py:1149-1337,719-822,1558-1807)."""

    def __init__(self, handle, lib, n_total=None):
        self.h = handle
        self.lib = lib
        self._info = None
        self._n_total = n_total

    def _load(self):
        """nvtb_vocab_build only ENQUEUES the build; the scalars come back through a pinned
        mailbox and are read (one event wait) the first time anything asks for them."""
        if self._info is None:
            info = _lib.nvtb_vocab_info_t()
            _lib.check(self.lib.nvtb_vocab_info(self.h, byref(info)))
            self._info = info
        return self._info

    n_kept = property(lambda self: self._load().n_kept)
    null_size = property(lambda self: self._load().null_size)
    oov_size = property(lambda self: self._load().oov_size)
    unique_size = property(lambda self: self._load().unique_size)

    @property
    def n_total(self):
        return self._n_total if self._n_total is not None else self._load().n_total

    @classmethod
    def build(cls, keys: torch.Tensor, sizes: torch.Tensor, null_size=0, freq_threshold=0,
              max_size=0, num_buckets=0, key_bits=0, size_bound=0):
        _lib.require_cuda()
        lib = _lib.load()
        h = c_void_p()
        with _timed("vocab_build", float(keys.numel() * 16)):
            _lib.check(lib.nvtb_vocab_build(byref(h), _ptr(keys), _ptr(sizes), keys.numel(), int(null_size),
                                            int(freq_threshold or 0), int(max_size or 0), int(num_buckets or 0),
                                            int(key_bits), int(size_bound), _lib.stream_ptr()))
        _count(8)
        return cls(h, lib, n_total=keys.numel())

    @classmethod
    def build_from_agg(cls, agg: "HashAgg", freq_threshold=0, max_size=0, num_buckets=0, key_bits=0,
                       size_bound=0):
        """vocabulary straight from a group-by handle (single GPU): no int64 export round
        trip; a sorted accumulator only needs one stable sort on the size bits."""
        _lib.require_cuda()
        lib = _lib.load()
        h = c_void_p()
        with _timed("vocab_build", 0.0):
            _lib.check(lib.nvtb_vocab_build_from_hashagg(byref(h), agg.h, int(freq_threshold or 0), int(max_size or 0),
                                                         int(num_buckets or 0), int(key_bits), int(size_bound),
                                                         _lib.stream_ptr()))
        _count(8)
        return cls(h, lib)

    @classmethod
    def build_from_pairs(cls, ordered_pairs: torch.Tensor, null_size=0, freq_threshold=0, max_size=0, num_buckets=0):
        """vocabulary from packed pairs already in (count desc, key asc) order (cross-GPU merge)"""
        _lib.require_cuda()
        lib = _lib.load()
        h = c_void_p()
        with _timed("vocab_build", float(ordered_pairs.numel() * 16)):
            _lib.check(lib.nvtb_vocab_build_from_pairs(byref(h), _ptr(ordered_pairs), ordered_pairs.numel(),
                                                       int(null_size), int(freq_threshold or 0), int(max_size or 0),
                                                       int(num_buckets or 0), _lib.stream_ptr()))
        _count(4)
        return cls(h, lib, n_total=ordered_pairs.numel())

    @classmethod
    def from_arrays(cls, keys: torch.Tensor, sizes: Optional[torch.Tensor] = None):
        _lib.require_cuda()
        lib = _lib.load()
        h = c_void_p()
        _lib.check(lib.nvtb_vocab_from_arrays(byref(h), _ptr(keys), _ptr(sizes), keys.numel(), _lib.stream_ptr()))
        _count(2)
        return cls(h, lib)

    def __del__(self):
        try:
            if getattr(self, "h", None) is not None and self.h.value:
                self.lib.nvtb_vocab_destroy(self.h)
                self.h = c_void_p()
        except Exception:
            pass

    def export(self, device="cuda", with_sizes=True):
        keys = torch.empty(self.n_kept, dtype=torch.int64, device=device)
        sizes = torch.empty(self.n_kept, dtype=torch.int64, device=device) if with_sizes else None
        _lib.check(self.lib.nvtb_vocab_export(self.h, _ptr(keys), _ptr(sizes), _lib.stream_ptr()))
        return keys, sizes

    def encode(self, key: Column, null_label=1, oov_label=2, first_label=3, num_buckets=0,
               hash_cols: Sequence[Column] = (), out_dtype=np.int64) -> torch.Tensor:
        n = key.data.numel()
        code = dtype_code(out_dtype)
        out = torch.empty(n, dtype=_CODE2TORCH[code], device=key.data.device)
        with _timed("encode", _in_bytes([key]) + out.numel() * out.element_size()):
            _lib.check(self.lib.nvtb_encode_apply(
                self.h, _descs([key]), n, int(null_label), int(oov_label), int(first_label),
                int(num_buckets or 0), _descs(hash_cols) if hash_cols else None, len(hash_cols),
                _ptr(out), code, _lib.stream_ptr()))
        _count()
        return out


# ------------------------------------------------------------ artefact files
def _path(p) -> bytes:
    return os.fsencode(str(p))


def parquet_write(path, columns, pandas_meta: Optional[bytes] = None, page_rows: int = 0):
    """[(name, 1-d numpy array of int32 | int64 | float32 | float64)] of one length -> a parquet
    file (nvtb_parquet_write: PLAIN, uncompressed pages of `page_rows` values, 0 = about 1 MiB;
    host only, no device)"""
    lib = _lib.load()
    arrays = [(name, np.ascontiguousarray(a)) for name, a in columns]
    n = len(arrays[0][1]) if arrays else 0
    cols = (_lib.nvtb_pq_col_t * max(len(arrays), 1))()
    for i, (name, a) in enumerate(arrays):
        if a.dtype not in _NP2CODE or a.dtype in (np.dtype("uint8"), np.dtype("bool")) or a.ndim != 1 or len(a) != n:
            raise TypeError(f"parquet_write: column {name!r} must be a 1-d int32/int64/float32/float64 "
                            f"array of {n} values, got {a.dtype} {a.shape}")
        cols[i].name = str(name).encode()
        cols[i].data = a.ctypes.data if n else None
        cols[i].dtype = _NP2CODE[a.dtype]
    _lib.check(lib.nvtb_parquet_write(_path(path), cols, len(arrays), n, pandas_meta, int(page_rows)))


def parquet_write_meta(path, oov_count: int, n_kept: int, null_size=0, oov_size=0, unique_size=0,
                       with_observed=True, pandas_meta: bytes = b""):
    """meta.<col>.parquet of a vocabulary (nvtb_parquet_write_meta; host only)"""
    lib = _lib.load()
    info = _lib.nvtb_vocab_info_t(int(n_kept), 0, int(null_size), int(oov_size), int(unique_size))
    _lib.check(lib.nvtb_parquet_write_meta(_path(path), int(oov_count), byref(info), 1 if with_observed else 0,
                                           pandas_meta))


class ArtifactWriter:
    """A batch of vocabulary files written by library threads (nvtb_artifacts_*).  submit_vocab
    returns without waiting for the device; join() waits for every file, stops the threads and
    raises NvtbError (naming the path) if a write failed."""

    def __init__(self, threads: int = 4):
        self.lib = _lib.load()
        self.h = c_void_p()
        _lib.check(self.lib.nvtb_artifacts_begin(byref(self.h), int(threads)))
        self._vocabs = []            # the handles must outlive the join

    def submit_vocab(self, vocab: "Vocab", meta_path, meta_pandas: bytes, unique_path, unique_max_rows: int,
                     key_name: str, key_dtype, size_name: Optional[str], index_start: int, oov_count: int,
                     unique_pandas_head: bytes, unique_pandas_tail: bytes):
        self._vocabs.append(vocab)
        _lib.check(self.lib.nvtb_artifacts_submit_vocab(
            self.h, vocab.h, _path(meta_path), meta_pandas, _path(unique_path) if unique_path else None,
            int(unique_max_rows), key_name.encode(), dtype_code(key_dtype),
            size_name.encode() if size_name is not None else None, int(index_start), int(oov_count),
            unique_pandas_head, unique_pandas_tail, _lib.stream_ptr()))

    def join(self):
        h, self.h = self.h, c_void_p()
        if h.value:
            rc = self.lib.nvtb_artifacts_join(h)
            self._vocabs = []
            _lib.check(rc)

    def __del__(self):
        try:
            if getattr(self, "h", None) is not None and self.h.value:
                self.lib.nvtb_artifacts_join(self.h)
        except Exception:
            pass


def pairs_lower_bounds(pairs: torch.Tensor, bounds: torch.Tensor) -> torch.Tensor:
    """number of key-sorted packed pairs whose unsigned key is below each of `bounds` (int64
    tensor of values in [0, 2^32]; 2^32 = "everything") -> int64 tensor on the device"""
    lib = _lib.load()
    n = pairs.numel()
    full = bounds >= (1 << 32)
    b = torch.where(full, torch.zeros_like(bounds), bounds)
    b32 = torch.where(b >= (1 << 31), b - (1 << 32), b).to(torch.int32).contiguous()
    out = torch.empty(bounds.numel(), dtype=torch.int64, device=pairs.device)
    _lib.check(lib.nvtb_pairs_lower_bounds(_ptr(pairs), n, _ptr(b32), b32.numel(), _ptr(out), _lib.stream_ptr()))
    _count()
    return torch.where(full, torch.full_like(out, n), out)


def pairs_merge(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """merge of two key-sorted, key-unique packed-pair arrays, counts of equal keys added"""
    lib = _lib.load()
    out = torch.empty(a.numel() + b.numel(), dtype=torch.int64, device=a.device)
    n = c_int64(0)
    _lib.check(lib.nvtb_pairs_merge(_ptr(a), a.numel(), _ptr(b), b.numel(), _ptr(out), byref(n), _lib.stream_ptr()))
    _count(4)
    return out[: n.value]


def segment_copy(src: torch.Tensor, dst: torch.Tensor, seg_src: torch.Tensor, seg_dst: torch.Tensor):
    """dst[seg_dst[s] + k] = src[seg_src[s] + k] for every segment s (seg_src: nseg + 1 ascending
    offsets ending at src.numel(); seg_dst < 0 skips a segment)"""
    lib = _lib.load()
    _lib.check(lib.nvtb_segment_copy_u64(_ptr(src), _ptr(dst), _ptr(seg_src), _ptr(seg_dst), seg_dst.numel(),
                                         src.numel(), _lib.stream_ptr()))
    _count()


def radix_sort(data: torch.Tensor, lo_bit: int = 0, hi_bit: Optional[int] = None, descending=False) -> torch.Tensor:
    """stable LSD radix sort of an int32/int64 tensor by bits [lo_bit, hi_bit) of its
    elements viewed as unsigned (nvtb_radix_sort_u32/u64); returns the sorted tensor"""
    _lib.require_cuda()
    lib = _lib.load()
    assert data.dtype in (torch.int32, torch.int64) and data.is_contiguous()
    bits = 8 * data.element_size()
    hi_bit = bits if hi_bit is None else hi_bit
    a = data.clone()
    b = torch.empty_like(a)
    flag = c_int(0)
    fn = lib.nvtb_radix_sort_u32 if bits == 32 else lib.nvtb_radix_sort_u64
    _lib.check(fn(_ptr(a), _ptr(b), a.numel(), int(lo_bit), int(hi_bit), 1 if descending else 0, byref(flag),
                  _lib.stream_ptr()))
    _count(3)
    return b if flag.value else a


class GroupStats:
    """key -> row of a stats matrix, gathered per row (nvtb_groupstats_*)."""

    def __init__(self, keys: torch.Tensor, stats: torch.Tensor, null_row: int = -1):
        _lib.require_cuda()
        self.lib = _lib.load()
        self.h = c_void_p()
        stats = stats.contiguous().to(torch.float64)
        self.width = int(stats.shape[1])
        _lib.check(self.lib.nvtb_groupstats_create(byref(self.h), _ptr(keys), keys.numel(), _ptr(stats),
                                                   self.width, int(null_row), _lib.stream_ptr()))
        _count(2)

    def __del__(self):
        try:
            if getattr(self, "h", None) is not None and self.h.value:
                self.lib.nvtb_groupstats_destroy(self.h)
                self.h = c_void_p()
        except Exception:
            pass

    MAX_COLS = 16   # output columns of one nvtb_groupstats_gather launch (kMaxGatherCols, csrc/vocab.cu)

    def gather(self, key: Column, cols: Sequence[int], miss_vals: Sequence[float], out_dtypes) -> List[torch.Tensor]:
        """one output tensor per entry of `cols`; more than MAX_COLS take several launches"""
        return [c.data for c in self.gather_columns(key, cols, miss_vals, out_dtypes)]

    def gather_columns(self, key: Column, cols: Sequence[int], miss_vals: Sequence[float], out_dtypes,
                       masked: Sequence[bool] = ()) -> List[Column]:
        """as gather(), as Columns; output j with masked[j] gets a validity bitmask that is clear
        where the key has no row or the statistic is NaN (an integer output holds 0 there)"""
        n = key.data.numel()
        dev = key.data.device
        codes = [dtype_code(d) for d in out_dtypes]
        outs = [torch.empty(n, dtype=_CODE2TORCH[c], device=dev) for c in codes]
        nbytes = (((n + 7) // 8 + 31) // 32) * 32          # pack_validity's padding (>= ceil(n/32) words)
        valid = [torch.zeros(nbytes, dtype=torch.uint8, device=dev) if j < len(masked) and masked[j] else None
                 for j in range(len(cols))]
        for s in range(0, len(cols), self.MAX_COLS):
            e = s + self.MAX_COLS
            vptrs = [v.data_ptr() if v is not None else None for v in valid[s:e]]
            _lib.check(self.lib.nvtb_groupstats_gather(
                self.h, _descs([key]), n, _lib.int_array(cols[s:e]), len(cols[s:e]), _lib.double_array(miss_vals[s:e]),
                _lib.ptr_array([o.data_ptr() for o in outs[s:e]]), _lib.int_array(codes[s:e]),
                _lib.ptr_array(vptrs) if any(vptrs) else None, _lib.stream_ptr()))
            _count()
        return [Column(o, v) for o, v in zip(outs, valid)]


# ------------------------------------------------------------- session group-by (K8, csrc/groupby.cu)
def _bitmask(n: int, device) -> torch.Tensor:
    """a zeroed validity bitmask of n bits in pack_validity's padding (whole 32-byte blocks)"""
    return torch.zeros((((n + 7) // 8 + 31) // 32) * 32, dtype=torch.uint8, device=device)


def gb_order_codes(col: Column, stats: torch.Tensor, key_valid: Optional[torch.Tensor] = None, and_key_valid=False):
    """-> (codes uint64-as-int64[n], validity bitmask); stats (device int64[3]) receives
    {min, max, n_valid} of the valid codes as unsigned bit patterns (nvtb_gb_order_codes)"""
    lib = _lib.load()
    n = col.data.numel()
    codes = torch.empty(max(n, 1), dtype=torch.int64, device=col.data.device)
    valid = _bitmask(n, col.data.device)
    with _timed("groupby_codes", _in_bytes([col]) + n * 8.125):
        _lib.check(lib.nvtb_gb_order_codes(_descs([col]), n, _ptr(codes), _ptr(valid), _ptr(key_valid),
                                           1 if and_key_valid else 0, _ptr(stats), _lib.stream_ptr()))
    _count(3)
    return codes, valid


def gb_order_rows(chunks, round_sizes: Sequence[int], n: int, row_bits: int, device) -> torch.Tensor:
    """rows 0..n-1 ordered by the packed fields of `chunks` (nvtb_gb_order_rows): -> the sorted
    elements (int64 bit patterns; row = element & (2^row_bits - 1))"""
    lib = _lib.load()
    a = torch.empty(max(n, 1), dtype=torch.int64, device=device)
    b = torch.empty(max(n, 1), dtype=torch.int64, device=device) if round_sizes else a
    arr = (_lib.nvtb_gb_chunk_t * max(len(chunks), 1))()
    for i, (codes, valid, mn, span, mode, lo, nbits) in enumerate(chunks):
        arr[i].codes = codes.data_ptr()
        arr[i].valid = valid.data_ptr() if valid is not None else None
        arr[i].min, arr[i].span, arr[i].mode, arr[i].lo, arr[i].nbits = mn, span, mode, lo, nbits
    flag = c_int(0)
    with _timed("groupby_sort", 0.0):
        _lib.check(lib.nvtb_gb_order_rows(arr, _lib.int_array(round_sizes), len(round_sizes), n, int(row_bits),
                                          _ptr(a), _ptr(b), byref(flag), _lib.stream_ptr()))
    _count(1 + 4 * len(round_sizes))
    return (b if flag.value else a)[:n]


def gb_segments(order: torch.Tensor, row_bits: int, key_codes: Sequence[torch.Tensor],
                key_valid: Optional[torch.Tensor]):
    """-> (offsets int64[G + 1], G, rows with valid keys); one host read (nvtb_gb_segments_*)"""
    lib = _lib.load()
    n = order.numel()
    dev = order.device
    flags = torch.empty(max((n + 7) // 8, 1), dtype=torch.uint8, device=dev)
    tiles = torch.empty(max((n + 2047) // 2048, 1), dtype=torch.int32, device=dev)
    counts = (c_int64 * 2)()
    with _timed("groupby_segments", n * (8.0 + 8 * len(key_codes))):
        _lib.check(lib.nvtb_gb_segments_count(_ptr(order), n, int(row_bits),
                                              _lib.ptr_array([k.data_ptr() for k in key_codes]), len(key_codes),
                                              _ptr(key_valid), _ptr(flags), _ptr(tiles), counts, _lib.stream_ptr()))
        g, kept = int(counts[0]), int(counts[1])
        off = torch.empty(g + 1, dtype=torch.int64, device=dev)
        _lib.check(lib.nvtb_gb_segments_write(_ptr(flags), _ptr(tiles), n, g, kept, _ptr(off), _lib.stream_ptr()))
    _count(3)
    return off, g, kept


def gb_segment_ids(off: torch.Tensor, n_groups: int, n: int) -> torch.Tensor:
    lib = _lib.load()
    gid = torch.empty(max(n, 1), dtype=torch.int64, device=off.device)
    _lib.check(lib.nvtb_gb_segment_ids(_ptr(off), n_groups, n, _ptr(gid), _lib.stream_ptr()))
    _count()
    return gid


def gb_gather(col: Column, order: Optional[torch.Tensor], row_bits: int, m: int, which: int = 0,
              off: Optional[torch.Tensor] = None) -> Column:
    """data + validity of `col` at row(i) (which 0), at the first (1) or last (2) position of every
    segment; row(p) = order[p] & (2^row_bits - 1), or p without an order (nvtb_gb_gather)"""
    lib = _lib.load()
    dev = col.data.device
    out = torch.empty(m, dtype=col.data.dtype, device=dev)
    valid = _bitmask(m, dev) if col.validity is not None else None
    with _timed("groupby_gather", m * (col.data.element_size() * 2 + (8 if order is not None else 0))):
        _lib.check(lib.nvtb_gb_gather(_descs([col]), _ptr(order), (1 << row_bits) - 1, _ptr(off), m, which,
                                      _ptr(out), _ptr(valid), _lib.stream_ptr()))
    _count()
    return Column(out, valid, None, col.dictionary, None, col.is_bool)


def gb_reduce(col: Column, off: torch.Tensor, n_groups: int, aggs: Sequence[str]):
    """{agg: Column} for the aggs of {count, sum, mean, var, std, min, max} over every segment of a
    column in group order (nvtb_gb_reduce: fp64, fixed order)"""
    lib = _lib.load()
    dev = col.data.device
    names = ("count", "sum", "mean", "var", "std", "min", "max")
    outs, ptrs = {}, []
    for a in names:
        if a in aggs:
            dt = torch.int32 if a == "count" else (col.data.dtype if a in ("min", "max") else torch.float32)
            outs[a] = torch.empty(max(n_groups, 1), dtype=dt, device=dev)
            ptrs.append(outs[a].data_ptr())
        else:
            ptrs.append(None)
    is_int = not col.data.dtype.is_floating_point
    valid = {a: _bitmask(n_groups, dev) for a in ("min", "max") if a in aggs and is_int}
    vptrs = _lib.ptr_array([valid[a].data_ptr() if a in valid else None for a in ("min", "max")]) if valid else None
    with _timed("groupby_reduce", _in_bytes([col]) + n_groups * (8 + 4 * len(outs))):
        _lib.check(lib.nvtb_gb_reduce(_descs([col]), _ptr(off), n_groups, _lib.ptr_array(ptrs), vptrs,
                                      _lib.stream_ptr()))
    _count(2)
    res = {}
    for a, t in outs.items():
        if a in ("min", "max"):
            res[a] = Column(t[:n_groups], valid.get(a), None, col.dictionary, None, col.is_bool)
        else:
            res[a] = Column(t[:n_groups])
    return res


def gb_rank_stats(col: Column, codes: torch.Tensor, codes_valid: torch.Tensor, order: torch.Tensor, row_bits: int,
                  off: torch.Tensor, n_groups: int, median: bool, nunique: bool):
    """-> (median float32[G] | None, nunique int32[G] | None) (nvtb_gb_rank_stats)"""
    lib = _lib.load()
    dev = col.data.device
    med = torch.empty(max(n_groups, 1), dtype=torch.float32, device=dev) if median else None
    nun = torch.empty(max(n_groups, 1), dtype=torch.int32, device=dev) if nunique else None
    with _timed("groupby_rank", order.numel() * 16.0):
        _lib.check(lib.nvtb_gb_rank_stats(_descs([col]), _ptr(codes), _ptr(codes_valid), _ptr(order),
                                          (1 << row_bits) - 1, _ptr(off), n_groups, _ptr(med), _ptr(nun),
                                          _lib.stream_ptr()))
    _count()
    return (med[:n_groups] if med is not None else None), (nun[:n_groups] if nun is not None else None)


def gb_list_rows(leaves: Column, lo: torch.Tensor, hi: torch.Tensor) -> Column:
    """a list column whose row g holds leaves[lo[g]:hi[g]] (nvtb_gb_list_rows)"""
    lib = _lib.load()
    m = lo.numel()
    dev = leaves.data.device
    off = torch.empty(m + 1, dtype=torch.int64, device=dev)
    total = c_int64(0)
    _lib.check(lib.nvtb_gb_list_rows(_descs([leaves]), _ptr(lo), _ptr(hi), m, _ptr(off), None, None, byref(total),
                                     _lib.stream_ptr()))
    out = torch.empty(total.value, dtype=leaves.data.dtype, device=dev)
    valid = _bitmask(total.value, dev) if leaves.validity is not None else None
    _lib.check(lib.nvtb_gb_list_rows(_descs([leaves]), _ptr(lo), _ptr(hi), m, _ptr(off), _ptr(out), _ptr(valid),
                                     byref(total), _lib.stream_ptr()))
    _count(2)
    return Column(out, valid, off, leaves.dictionary, None, leaves.is_bool)


# ------------------------------------------------------------- session operators (K10, csrc/session.cu)
LAG_MAX_KEYS = 8    # partition columns of one nvtb_lag_same_key launch (kMaxLagKeys, csrc/session.cu)
LAG_MAX_COLS = 16   # value columns of one nvtb_difference_lag launch (kMaxLagCols)


def list_slice(col: Column, start: int, end: int) -> Column:
    """row[start:end] of every row of a list column: the leaf bounds (nvtb_list_slice_bounds), then
    the sub-list copy (nvtb_gb_list_rows).  The input is only read."""
    lib = _lib.load()
    n = col.nrows
    dev = col.data.device
    lo = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
    hi = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
    with _timed("list_slice_bounds", n * 24.0):
        _lib.check(lib.nvtb_list_slice_bounds(_ptr(col.offsets), n, int(start), int(end), _ptr(lo), _ptr(hi),
                                              _lib.stream_ptr()))
    _count()
    return gb_list_rows(col.leaves(), lo[:n], hi[:n])


def list_slice_pad(col: Column, start: int, end: int, width: int, pad_bits: int) -> Column:
    """the dense n x width slice of a list column, padded with the value whose bit pattern in the
    leaf dtype is pad_bits (nvtb_list_slice_pad)"""
    lib = _lib.load()
    leaves = col.leaves()
    n = col.nrows
    m = n * width
    dev = col.data.device
    out = torch.empty(max(m, 1), dtype=leaves.data.dtype, device=dev)
    valid = _bitmask(m, dev) if leaves.validity is not None else None
    off = torch.empty(n + 1, dtype=torch.int64, device=dev)
    with _timed("list_slice_pad", n * 16.0 + m * (leaves.data.element_size() * 2.0 + 0.25)):
        _lib.check(lib.nvtb_list_slice_pad(_descs([leaves]), _ptr(col.offsets), n, int(start), int(end), int(width),
                                           int(pad_bits), _ptr(out), _ptr(valid), _ptr(off), _lib.stream_ptr()))
    _count()
    return Column(out[:m], valid, off, leaves.dictionary, None, leaves.is_bool)


def lag_same_key(keys: Sequence[Column], n: int, shift: int) -> torch.Tensor:
    """bitmask: bit i set when row i - shift is in the frame and every key is valid and equal at i
    and i - shift (nvtb_lag_same_key)"""
    lib = _lib.load()
    if len(keys) > LAG_MAX_KEYS:
        raise ValueError(f"at most {LAG_MAX_KEYS} partition columns, got {len(keys)}")
    same = _bitmask(n, keys[0].data.device)
    shift = max(-n, min(n, int(shift)))
    with _timed("lag_same_key", _in_bytes(keys) + n / 8.0):
        _lib.check(lib.nvtb_lag_same_key(_descs(keys), len(keys), n, shift, _ptr(same), _lib.stream_ptr()))
    _count()
    return same


def difference_lag(cols: Sequence[Column], same: torch.Tensor, shift: int) -> List[Column]:
    """float32 x[i] - x[i - shift] of every column where `same` (lag_same_key with this shift) has
    bit i and both values are valid, else null (nvtb_difference_lag)"""
    lib = _lib.load()
    n = _check_same_len(cols)
    dev = cols[0].data.device
    shift = max(-n, min(n, int(shift)))
    outs = [torch.empty(max(n, 1), dtype=torch.float32, device=dev) for _ in cols]
    valids = [_bitmask(n, dev) for _ in cols]
    for s in range(0, len(cols), LAG_MAX_COLS):
        e = s + LAG_MAX_COLS
        with _timed("difference_lag", _in_bytes(cols[s:e]) + n * (4.125 * len(cols[s:e]) + 0.125)):
            _lib.check(lib.nvtb_difference_lag(_descs(cols[s:e]), len(cols[s:e]), n, shift, _ptr(same),
                                               _lib.ptr_array([o.data_ptr() for o in outs[s:e]]),
                                               _lib.ptr_array([v.data_ptr() for v in valids[s:e]]),
                                               _lib.stream_ptr()))
        _count()
    return [Column(o[:n], v) for o, v in zip(outs, valids)]


# ------------------------------------------------------------- external-table join (K9, csrc/join.cu)
class JoinTable:
    """The build side of JoinExternal on the device: ext rows in key order, the run of every
    distinct key and a table key -> run (nvtb_join_create)."""

    def __init__(self, distinct_keys: torch.Tensor, off: torch.Tensor, ordered_rows: torch.Tensor,
                 null_lo: int, null_hi: int):
        _lib.require_cuda()
        self.lib = _lib.load()
        self.h = c_void_p()
        keys = distinct_keys.to(torch.int64).contiguous()
        rows = ordered_rows.to(torch.int64).contiguous()
        _lib.check(self.lib.nvtb_join_create(byref(self.h), _ptr(keys), keys.numel(), _ptr(off), _ptr(rows),
                                             rows.numel(), int(null_lo), int(null_hi), _lib.stream_ptr()))
        _count(2)
        g, mx = c_int64(0), c_int64(0)
        _lib.check(self.lib.nvtb_join_info(self.h, byref(g), byref(mx)))
        self.n_groups, self.max_group = g.value, mx.value

    def __del__(self):
        try:
            if getattr(self, "h", None) is not None and self.h.value:
                self.lib.nvtb_join_destroy(self.h)
                self.h = c_void_p()
        except Exception:
            pass

    def probe(self, key: Column, how: str, scan: bool):
        """-> (ext int64[n], off int64[n + 1] | None, n_out).  Without `scan`: the ext row of every
        left row (-1 = no match).  With it: the first match's position in key order and the output
        offsets (nvtb_join_probe; one host read)."""
        n = key.data.numel()
        dev = key.data.device
        ext = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
        off = torch.empty(n + 1, dtype=torch.int64, device=dev) if scan else None
        n_out = c_int64(0)
        with _timed("join_probe", _in_bytes([key]) + n * (16.0 if scan else 8.0)):
            _lib.check(self.lib.nvtb_join_probe(self.h, _descs([key]), n, 0 if how == "left" else 1, _ptr(ext),
                                                _ptr(off), byref(n_out), _lib.stream_ptr()))
        _count(4 if scan else 1)
        return ext[:n], off, n_out.value

    def expand(self, first: torch.Tensor, off: torch.Tensor, n_out: int):
        """-> (left rows, ext rows) int64[n_out] of every output row (nvtb_join_expand)"""
        dev = first.device
        left = torch.empty(max(n_out, 1), dtype=torch.int64, device=dev)
        ext = torch.empty(max(n_out, 1), dtype=torch.int64, device=dev)
        with _timed("join_expand", n_out * 16.0 + first.numel() * 8.0):
            _lib.check(self.lib.nvtb_join_expand(self.h, _ptr(first), _ptr(off), first.numel(), n_out, _ptr(left),
                                                 _ptr(ext), _lib.stream_ptr()))
        _count()
        return left[:n_out], ext[:n_out]


JOIN_GATHER_MAX_COLS = 16   # columns of one nvtb_join_gather launch (kMaxJoinCols, csrc/join.cu)


def join_gather(cols: Sequence[Column], rows: torch.Tensor, masked: Sequence[bool]) -> List[Column]:
    """flat columns at int64 `rows` (-1 = null) -> Columns with the sources' dtype, dictionary and
    bool flag; output k gets a validity bitmask when masked[k] or its source has one
    (nvtb_join_gather)"""
    lib = _lib.load()
    m = rows.numel()
    dev = rows.device
    # an empty source (an empty ext table) is only ever read at row -1: give the kernel one row
    cols = [c if c.data.numel() else Column(torch.zeros(1, dtype=c.data.dtype, device=dev), None, None,
                                            c.dictionary, None, c.is_bool) for c in cols]
    outs = [torch.empty(max(m, 1), dtype=c.data.dtype, device=dev) for c in cols]
    valids = [_bitmask(m, dev) if (mk or c.validity is not None) else None for c, mk in zip(cols, masked)]
    for s in range(0, len(cols), JOIN_GATHER_MAX_COLS):
        e = s + JOIN_GATHER_MAX_COLS
        nbytes = m * 8.0 + sum(m * (c.data.element_size() + 0.125) for c in cols[s:e])
        with _timed("join_gather", nbytes):
            _lib.check(lib.nvtb_join_gather(_descs(cols[s:e]), len(cols[s:e]), _ptr(rows), m,
                                            _lib.ptr_array([o.data_ptr() for o in outs[s:e]]),
                                            _lib.ptr_array([v.data_ptr() if v is not None else None
                                                            for v in valids[s:e]]), _lib.stream_ptr()))
        _count()
    return [Column(o[:m], v, None, c.dictionary, None, c.is_bool) for o, v, c in zip(outs, valids, cols)]


def take_rows(cols, rows: torch.Tensor, masked: bool = False):
    """{name: Column} at int64 `rows`, in the same order; a fixed-width column through
    nvtb_join_gather, a list column through nvtb_gb_list_rows over its gathered offsets.  With
    `masked`, row -1 is null (an empty list for a list column)."""
    flat = [n for n, c in cols.items() if not c.is_list]
    res = dict(zip(flat, join_gather([cols[n] for n in flat], rows, [masked] * len(flat)))) if flat else {}
    for n, c in cols.items():
        if c.is_list:
            lo, hi = join_gather([Column(c.offsets[:-1]), Column(c.offsets[1:])], rows, [False, False])
            res[n] = gb_list_rows(c.leaves(), lo.data, hi.data)
    return {n: res[n] for n in cols}


# ------------------------------------------------------------- row selection (K11, csrc/filter.cu)
CMP_EQ, CMP_NE, CMP_LT, CMP_LE, CMP_GT, CMP_GE = range(6)    # nvtb_cmp_op_t
MASK_AND, MASK_OR, MASK_XOR, MASK_NOT = range(4)            # nvtb_mask_op_t
NOTNULL_MAX_COLS = 16   # columns of one nvtb_mask_notnull launch (kMaxNotnullCols, csrc/filter.cu)
MASK_TILE = 2048        # rows per tile of nvtb_mask_count / nvtb_mask_select (kScanTile, csrc/scan.cuh)


def mask_nbytes(n: int) -> int:
    """bytes of a row mask of n rows: pack_validity's padding, which the mask kernels fill"""
    return (((n + 7) // 8 + 31) // 32) * 32


def mask_compare(a: Column, b: Optional[Column], op: int, cmp_type: int, scalar_bits: int, n: int) -> torch.Tensor:
    """row mask of a op (b, or the scalar whose bit pattern in cmp_type is scalar_bits); a null
    operand is true for CMP_NE only (nvtb_mask_compare)"""
    lib = _lib.load()
    out = torch.empty(mask_nbytes(n), dtype=torch.uint8, device=a.data.device)
    with _timed("mask", _in_bytes([a] if b is None else [a, b]) + n / 8.0):
        _lib.check(lib.nvtb_mask_compare(_descs([a]), _descs([b]) if b is not None else None, int(op), int(cmp_type),
                                         int(scalar_bits), n, _ptr(out), _lib.stream_ptr()))
    _count()
    return out


def mask_logic(a: torch.Tensor, b: Optional[torch.Tensor], n: int, op: int) -> torch.Tensor:
    """a & b, a | b, a ^ b or ~a of two row masks of n rows (nvtb_mask_logic)"""
    lib = _lib.load()
    out = torch.empty_like(a)
    with _timed("mask", n / 8.0 * (2 if b is None else 3)):
        _lib.check(lib.nvtb_mask_logic(_ptr(a), _ptr(b), n, int(op), _ptr(out), _lib.stream_ptr()))
    _count()
    return out


def mask_notnull(cols: Sequence[Column], n: int) -> torch.Tensor:
    """row mask: every column valid and, if a float, not NaN (nvtb_mask_notnull; more than
    NOTNULL_MAX_COLS columns are ANDed)"""
    lib = _lib.load()
    out = None
    for s in range(0, len(cols), NOTNULL_MAX_COLS):
        part = cols[s:s + NOTNULL_MAX_COLS]
        m = torch.empty(mask_nbytes(n), dtype=torch.uint8, device=part[0].data.device)
        with _timed("mask", _in_bytes(part) + n / 8.0):
            _lib.check(lib.nvtb_mask_notnull(_descs(part), len(part), n, _ptr(m), _lib.stream_ptr()))
        _count()
        out = m if out is None else mask_logic(out, m, n, MASK_AND)
    return out


def mask_count(mask: torch.Tensor, n: int):
    """-> (kept rows, tile offsets for mask_select); one host read (nvtb_mask_count)"""
    lib = _lib.load()
    tile_off = torch.empty((n + MASK_TILE - 1) // MASK_TILE + 1, dtype=torch.int64, device=mask.device)
    kept = c_int64(0)
    with _timed("count", n / 8.0 + tile_off.numel() * 16.0):
        _lib.check(lib.nvtb_mask_count(_ptr(mask), n, _ptr(tile_off), byref(kept), _lib.stream_ptr()))
    _count(4 if n else 0)
    return kept.value, tile_off


def mask_select(mask: torch.Tensor, n: int, tile_off: torch.Tensor, n_kept: int) -> torch.Tensor:
    """the int64 ids of the n_kept rows whose bit is set, ascending (nvtb_mask_select)"""
    lib = _lib.load()
    rows = torch.empty(max(n_kept, 1), dtype=torch.int64, device=mask.device)
    with _timed("select", n / 8.0 + tile_off.numel() * 8.0 + n_kept * 8.0):
        _lib.check(lib.nvtb_mask_select(_ptr(mask), n, _ptr(tile_off), _ptr(rows), _lib.stream_ptr()))
    _count()
    return rows[:n_kept]
