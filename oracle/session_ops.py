"""pandas / numpy restatements of the session operators, with the rules the reference leaves open
pinned as nvtabular_b200/ops/list_slice.py and ops/difference_lag.py state them.

ListSlice (reference nvtabular/ops/list_slice.py:58-75, the argument normalisation, and :88-102,
the CPU branch): Python's row[start:end], padded at the end with pad_value up to max_elements.
Leaf nulls stay in the list (the reference's GPU branch drops them); a null row is an empty list,
as Column.from_arrow reads it.

DifferenceLag (reference nvtabular/ops/difference_lag.py:65-80): the reference's CPU code,
`mask[mask == False] = None` on a bool Series, raises TypeError on pandas 3, so its intent is
restated as (x - x.shift(s)).where(mask).astype("float32"), with
- mask: every partition column valid and equal at i and i - s, compared by pandas == on exact
  (nullable) dtypes, so a null or NaN key never matches and -0.0 == +0.0;
- integer columns subtracted in int64, wrapping, and rounded once to float32 (the reference's GPU
  branch, cuDF's int64 arithmetic; pandas would first turn both operands into float64);
- float32 subtracted in float32, float64 in float64 and then rounded to float32.
"""
from typing import List, Sequence

import numpy as np
import pandas as pd

INT64_MAX = int(np.iinfo(np.int64).max)


def normalise(start, end=None):
    """-> (start, end, max_elements), list_slice.py:65-75"""
    if start > 0 and end is None:
        start, end = 0, start
    if end is None:
        end = INT64_MAX
    if start < 0:
        max_elements = -(start if end > 0 else start - end)
    else:
        max_elements = end - start
    return start, end, max_elements


def list_slice(rows: Sequence, start, end=None, pad=False, pad_value=0.0) -> List[list]:
    """list_slice.py:88-102 on a sequence of rows (None = an empty row)"""
    s, e, width = normalise(start, end)
    out = []
    for r in rows:
        v = [] if r is None else list(r)[s:e]
        if pad and len(v) < width:
            v = v + [pad_value] * (width - len(v))
        out.append(v)
    return out


def _exact(s: pd.Series) -> pd.Series:
    """a dtype whose shift keeps every value exact and marks the shifted-in rows null"""
    if s.dtype.kind in "iu":
        return s.astype("Int64")
    if s.dtype.kind == "b":
        return s.astype("boolean")
    return s


def same_key(df: pd.DataFrame, partition_cols: Sequence[str], shift: int) -> np.ndarray:
    """difference_lag.py:71-74: True where every partition column is valid and equal at i and
    i - shift"""
    mask = np.ones(len(df), dtype=bool)
    for p in partition_cols:
        a = _exact(df[p])
        eq = (a == a.shift(shift))
        mask &= np.asarray(eq.fillna(False), dtype=bool) & a.notna().to_numpy() & a.shift(shift).notna().to_numpy()
    return mask


def lag(x: pd.Series, mask: np.ndarray, shift: int) -> np.ndarray:
    """difference_lag.py:76-79 for one value column: float32, NaN where there is no lag"""
    n = len(x)
    i = np.arange(n)
    j = i - shift
    inside = (j >= 0) & (j < n)
    j = np.clip(j, 0, max(n - 1, 0))
    valid = x.notna().to_numpy()
    ok = mask & inside & valid & valid[j]
    kind = x.dtype.kind if not isinstance(x.dtype, pd.api.extensions.ExtensionDtype) else \
        ("i" if pd.api.types.is_integer_dtype(x.dtype) else "f")
    if kind in "iu":
        v = x.to_numpy(dtype=np.int64, na_value=0)
        with np.errstate(over="ignore"):
            d = (v - v[j]).astype(np.float32)
    elif x.dtype == np.float32:
        v = x.to_numpy(dtype=np.float32, na_value=np.nan)
        d = v - v[j]
    else:
        v = x.to_numpy(dtype=np.float64, na_value=np.nan)
        d = (v - v[j]).astype(np.float32)
    return np.where(ok, d, np.float32(np.nan)).astype(np.float32)


def difference_lag(df: pd.DataFrame, cols: Sequence[str], partition_cols, shift=1) -> pd.DataFrame:
    """DifferenceLag on ONE partition: {col}_difference_lag_{s} for every col and shift, in the
    reference's column_mapping order (difference_lag.py:88-94)"""
    partition_cols = [partition_cols] if isinstance(partition_cols, str) else list(partition_cols)
    shifts = [shift] if isinstance(shift, int) else list(shift)
    masks = {s: same_key(df, partition_cols, s) for s in shifts}
    out = {}
    for c in cols:
        for s in shifts:
            out[f"{c}_difference_lag_{s}"] = lag(df[c], masks[s], s)
    return pd.DataFrame(out, index=range(len(df)))
