"""Filter (reference nvtabular/ops/filter.py:28-62): keep the rows of every partition that a
user predicate selects, on the GPU (csrc/filter.cu, family K11).

`f` is called with a predicate view of the partition (`FrameView`), not with the DeviceFrame
itself: `df["a"]` and `df.a` are `ColumnView`s, whose comparisons with a scalar or with another
column of the frame, and isnull / isna / notnull / notna, each run as one mask kernel and return a
`Mask`; masks combine with & | ^ ~ (one kernel each), and `df[mask]` is the filtered view.  What
`f` returns decides the result:
- a Mask, or a bool column (a null counts as false): the rows it selects;
- a view (`df[mask]`, or `df` itself) or a DeviceFrame: that frame, as the reference takes any frame;
- anything else: ValueError, as the reference raises (filter.py:56-60).
Selecting rows reads the kept count once (one stream synchronise per partition), then writes the
kept row ids and gathers every column at them (engine.take_rows).  If every row is kept the
partition passes through untouched, with the same buffers; if none is, the result has 0 rows and
the same dtypes and dictionaries.  Partitions may shrink or become empty; they are not rebalanced.

Comparison rules, pinned against pandas by tests/test_filter_host.py (`scalar_compare_type`,
`column_compare_type`):
- a null behaves like NaN in pandas' float image of the column: every op is false but !=, which is
  true, so ~(x > 0) is true at a null;
- an integer, bool or uint8 column against a Python int compares exactly in int64, whatever the
  column's width (int32 < 2**40 holds for every valid row); an int outside int64 raises
  OverflowError;
- an integer column against a float compares in float64, like numpy (int64 2**53 + 1 > 2.0**53 is
  false);
- a float32 column against a Python int or float casts the scalar to float32 (beyond its range:
  +-inf) and compares in float32; a float64 column compares in float64;
- a numpy scalar, or another column, compares in numpy's result type of the pair;
- a string column compares == and != with a str through its dictionary (a string that is not in
  it matches no row); comparing two string columns, an ordering comparison of a string column, a
  comparison of a list column or with None raises TypeError.
An integer column with nulls is float64 in pandas' image, so pandas would compare values beyond
2**53 after rounding them; this operator compares them exactly.

Filter has no fit state, serving hook or collective: on several GPUs each rank filters its own
partitions.  Workflow.save records `f` by module and qualified name (a lambda or a function
defined in __main__ cannot be saved).  A graph that adds a Filter branch to an unfiltered one
(`filtered + other`) merges frames of different lengths: the reference silently misaligns their
rows, and Workflow raises ValueError instead.
"""
import numbers

import numpy as np
import torch

from .. import _lib, engine
from ..column import Column, DeviceFrame
from ..graph import ColumnSelector
from .base import Operator

INT64_MIN = int(np.iinfo(np.int64).min)
INT64_MAX = int(np.iinfo(np.int64).max)
_OPS = {"==": engine.CMP_EQ, "!=": engine.CMP_NE, "<": engine.CMP_LT, "<=": engine.CMP_LE,
        ">": engine.CMP_GT, ">=": engine.CMP_GE}


# ------------------------------------------------------------------------------ comparison rules
def _type_code(dt: np.dtype) -> int:
    if dt.kind in "biu":
        return _lib.I64
    if dt.kind == "f":
        return _lib.F32 if dt.itemsize == 4 else _lib.F64
    raise TypeError(f"Filter: cannot compare values of dtype {dt}")


def _bits(cmp_type: int, value) -> int:
    """the bit pattern of `value` in cmp_type, as nvtb_mask_compare's scalar_bits"""
    if cmp_type == _lib.I64:
        return int(value) & 0xFFFFFFFFFFFFFFFF
    if cmp_type == _lib.F32:
        return int(np.array(value, dtype=np.float32).view(np.uint32))
    return int(np.array(value, dtype=np.float64).view(np.uint64))


def column_compare_type(a: np.dtype, b: np.dtype) -> int:
    """the type a column-against-column comparison runs in: numpy's result type of the pair"""
    return _type_code(np.result_type(np.dtype(a), np.dtype(b)))


def scalar_compare_type(dtype: np.dtype, x):
    """-> (cmp_type, scalar_bits) of a column of `dtype` compared with the scalar x"""
    dtype = np.dtype(dtype)
    if dtype.kind not in "biuf":
        raise TypeError(f"Filter: cannot compare a {dtype} column with {x!r}")
    if isinstance(x, np.generic) and not isinstance(x, np.bool_):
        if x.dtype.kind not in "iuf":
            raise TypeError(f"Filter: cannot compare a {dtype} column with {x!r}")
        t = _type_code(np.result_type(dtype, x.dtype))
        if t == _lib.I64:
            return t, _bits(t, _int64(int(x)))
        return t, _bits(t, float(x) if t == _lib.F64 else np.float32(x))
    if isinstance(x, (bool, np.bool_)):
        x = int(x)
    if isinstance(x, numbers.Integral):
        x = int(x)
        if dtype.kind in "biu":
            return _lib.I64, _bits(_lib.I64, _int64(x))
    elif isinstance(x, numbers.Real):
        x = float(x)
    else:
        raise TypeError(f"Filter: cannot compare a {dtype} column with {x!r}")
    if dtype.kind == "f" and dtype.itemsize == 4:
        with np.errstate(over="ignore"):
            return _lib.F32, _bits(_lib.F32, np.float32(float(x)))
    return _lib.F64, _bits(_lib.F64, float(x))


def _int64(x: int) -> int:
    if not INT64_MIN <= x <= INT64_MAX:
        raise OverflowError(f"Filter: {x} is outside the int64 range")
    return x


def string_code(dictionary: np.ndarray, s: str) -> int:
    """the code of s in a column's sorted dictionary, or -1 (which no row holds)"""
    i = int(np.searchsorted(dictionary, s)) if len(dictionary) else 0
    return i if i < len(dictionary) and dictionary[i] == s else -1


# ----------------------------------------------------------------------------- predicate view
class Mask:
    """A row predicate on the device: a bitmask of n rows in the validity layout."""

    __slots__ = ("bits", "n")

    def __init__(self, bits: torch.Tensor, n: int):
        self.bits, self.n = bits, n

    def _logic(self, other, op):
        other = _as_mask(other)
        if other.n != self.n:
            raise ValueError(f"Filter: masks of {self.n} and {other.n} rows cannot be combined")
        return Mask(engine.mask_logic(self.bits, other.bits, self.n, op), self.n)

    def __and__(self, other):
        return self._logic(other, engine.MASK_AND)

    def __or__(self, other):
        return self._logic(other, engine.MASK_OR)

    def __xor__(self, other):
        return self._logic(other, engine.MASK_XOR)

    __rand__, __ror__, __rxor__ = __and__, __or__, __xor__

    def __invert__(self):
        return Mask(engine.mask_logic(self.bits, None, self.n, engine.MASK_NOT), self.n)

    def __len__(self):
        return self.n

    def __bool__(self):
        raise ValueError("The truth value of a row mask is ambiguous; combine masks with & | ~, not and / or / not")


class ColumnView:
    """One column of a FrameView: comparisons and null tests return a Mask."""

    __array_ufunc__ = None      # a numpy scalar on the left defers to the reflected comparison
    __hash__ = None

    def __init__(self, col: Column, name: str):
        self.col, self.name = col, name

    def __len__(self):
        return self.col.nrows

    def __bool__(self):
        raise ValueError(f"The truth value of the column {self.name!r} is ambiguous; compare it to get a mask")

    @property
    def dtype(self):
        return self.col.np_dtype

    def _compare(self, other, sym):
        op = _OPS[sym]
        a, n = self.col, self.col.nrows
        if a.is_list or (isinstance(other, ColumnView) and other.col.is_list):
            raise TypeError(f"Filter: {self.name!r} {sym} ...: list columns cannot be compared")
        if isinstance(other, ColumnView):
            b = other.col
            if b.nrows != n:
                raise ValueError(f"Filter: columns {self.name!r} and {other.name!r} differ in length")
            if a.is_string or b.is_string:
                raise TypeError(f"Filter: {self.name!r} {sym} {other.name!r}: string columns can only be compared "
                                "with a str")
            return Mask(engine.mask_compare(a, b, op, column_compare_type(a.np_dtype, b.np_dtype), 0, n), n)
        if other is None:
            raise TypeError(f"Filter: {self.name!r} {sym} None; use isnull() / notnull()")
        if a.is_string:
            if not isinstance(other, str):
                raise TypeError(f"Filter: the string column {self.name!r} can only be compared with a str")
            if op not in (engine.CMP_EQ, engine.CMP_NE):
                raise TypeError(f"Filter: {self.name!r} {sym} {other!r}: string columns support only == and !=")
            code = string_code(a.dictionary, other)
            return Mask(engine.mask_compare(a, None, op, _lib.I64, _bits(_lib.I64, code), n), n)
        if isinstance(other, str):
            raise TypeError(f"Filter: the {a.np_dtype} column {self.name!r} cannot be compared with a str")
        t, bits = scalar_compare_type(a.np_dtype, other)
        return Mask(engine.mask_compare(a, None, op, t, bits, n), n)

    def __eq__(self, other):
        return self._compare(other, "==")

    def __ne__(self, other):
        return self._compare(other, "!=")

    def __lt__(self, other):
        return self._compare(other, "<")

    def __le__(self, other):
        return self._compare(other, "<=")

    def __gt__(self, other):
        return self._compare(other, ">")

    def __ge__(self, other):
        return self._compare(other, ">=")

    def notnull(self) -> Mask:
        n = self.col.nrows
        if self.col.is_list:          # a list row is never NA (a null row is an empty list)
            zero = torch.zeros(engine.mask_nbytes(n), dtype=torch.uint8, device=self.col.data.device)
            return ~Mask(zero, n)
        return Mask(engine.mask_notnull([self.col], n), n)

    def isnull(self) -> Mask:
        return ~self.notnull()

    notna, isna = notnull, isnull

    def __and__(self, other):
        return _as_mask(self) & other

    def __or__(self, other):
        return _as_mask(self) | other

    def __xor__(self, other):
        return _as_mask(self) ^ other

    __rand__, __ror__, __rxor__ = __and__, __or__, __xor__

    def __invert__(self):
        return ~_as_mask(self)


def _as_mask(x) -> Mask:
    """a Mask, or a bool column as one (a null is false)"""
    if isinstance(x, Mask):
        return x
    if isinstance(x, ColumnView) and x.col.is_bool and not x.col.is_list:
        n = x.col.nrows
        return Mask(engine.mask_compare(x.col, None, engine.CMP_GT, _lib.I64, 0, n), n)
    raise TypeError(f"Filter: {type(x).__name__} is not a row mask or a bool column")


class FrameView:
    """The frame a Filter predicate receives: columns by `df[name]` or `df.name`, and `df[mask]`,
    the frame's rows that a Mask (or a bool column) selects."""

    def __init__(self, df: DeviceFrame):
        self._df = df

    @property
    def frame(self) -> DeviceFrame:
        return self._df

    @property
    def columns(self):
        return self._df.columns

    def __len__(self):
        return len(self._df)

    def __contains__(self, name):
        return name in self._df

    def __getitem__(self, key):
        if isinstance(key, str):
            return ColumnView(self._df[key], key)
        if isinstance(key, (Mask, ColumnView)):
            return FrameView(compact(self._df, _as_mask(key)))
        if isinstance(key, (list, tuple)):
            return FrameView(self._df[list(key)])
        raise TypeError(f"Filter: cannot index a frame with {type(key).__name__}")

    def __getattr__(self, name):
        if not name.startswith("_") and name in self._df:
            return ColumnView(self._df[name], name)
        raise AttributeError(name)


def compact(df: DeviceFrame, mask: Mask) -> DeviceFrame:
    """the rows of df that `mask` selects, in order; df itself when it selects every row"""
    from .fill import materialize
    n = len(df)
    if mask.n != n:
        raise ValueError(f"Filter: a mask of {mask.n} rows cannot select from a frame of {n} rows")
    kept, tile_off = engine.mask_count(mask.bits, n)
    if kept == n:
        return df
    rows = engine.mask_select(mask.bits, n, tile_off, kept)
    return DeviceFrame(engine.take_rows({k: materialize(c) for k, c in df.items()}, rows))


class Filter(Operator):
    """Keep the rows that f selects.

    f takes the partition's predicate view and returns a row mask, a bool column or a frame, e.g.
    ``Filter(f=lambda df: df["a"] >= 0)`` or ``Filter(f=lambda df: df[df.x.notnull()])``.  See the
    module docstring for what a predicate can do and the comparison rules."""

    def __init__(self, f):
        super().__init__()
        if f is None:
            raise ValueError("f cannot be None. Filter op applies f to dataframe")
        self.f = f

    def transform(self, col_selector: ColumnSelector, df: DeviceFrame) -> DeviceFrame:
        df = DeviceFrame({n: self._get(df, n) for n in col_selector.names})
        res = self.f(FrameView(df))
        if isinstance(res, FrameView):
            return res.frame
        if isinstance(res, DeviceFrame):
            return res
        if isinstance(res, Mask) or (isinstance(res, ColumnView) and res.col.is_bool and not res.col.is_list):
            return compact(df, _as_mask(res))
        raise ValueError(f"Invalid output from filter op: f returned {type(res).__name__}; it must return a "
                         "row mask, a bool column or a frame")
