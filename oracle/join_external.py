"""pandas restatement of JoinExternal (reference nvtabular/ops/join_external.py:97-164), with the
points the reference leaves to cuDF / pandas pinned:

- rows follow left-row order, and the matches of one left row follow ext-table order (the
  reference's sort on __tmp__ is unstable; here the sort is on (left row, ext row));
- null / NaN keys match each other; -0.0 == +0.0; int and float keys compare by value;
- an unmatched row of a left join has a null in every ext column, and an EMPTY list in an ext list
  column (the engine's list columns have no row validity);
- a non-key ext column named like a left column raises ValueError.
"""
from typing import List, Optional

import numpy as np
import pandas as pd


def _as_list(x):
    return [x] if isinstance(x, str) else list(x)


def ext_table(df_ext: pd.DataFrame, columns_ext: Optional[List[str]] = None, drop_duplicates_ext=False):
    """join_external.py:116-146: the column subset, then drop_duplicates(ignore_index=True)"""
    ext = df_ext[list(columns_ext)] if columns_ext else df_ext
    if drop_duplicates_ext:
        ext = ext.drop_duplicates(ignore_index=True)
    return ext.reset_index(drop=True)


def join_external(df: pd.DataFrame, df_ext: pd.DataFrame, on, how="left", on_ext=None, columns_ext=None,
                  drop_duplicates_ext=False) -> pd.DataFrame:
    """join_external.py:148-164 on one partition `df` (its columns are the selected ones)"""
    on = _as_list(on)
    on_ext = _as_list(on_ext) if on_ext is not None else list(on)
    if how not in ("left", "inner"):
        raise ValueError("Only left join is currently supported.")
    ext = ext_table(df_ext, columns_ext, drop_duplicates_ext)
    shared = {o for o, e in zip(on, on_ext) if o == e}
    clash = [c for c in ext.columns if c in df.columns and c not in shared]
    if clash:
        raise ValueError(f"ext columns {clash} have the names of left columns")
    left = df.reset_index(drop=True).assign(__tmp__=np.arange(len(df)))
    right = ext.assign(__ext_tmp__=np.arange(len(ext)))
    for o, e in zip(on, on_ext):      # -0.0 and +0.0 are one key
        if left[o].dtype.kind == "f":
            left[o] = left[o] + 0.0
        if right[e].dtype.kind == "f":
            right[e] = right[e] + 0.0
    if len(right) == 0 and how == "left":
        # pandas keeps the ext dtypes of an empty right side; every ext value is null
        out = left.copy()
        for c in ext.columns:
            if c not in out.columns:
                out[c] = pd.Series([None] * len(left), dtype=object) if ext[c].dtype == object else np.nan
    else:
        merged_left = left.copy()
        out = merged_left.merge(right, left_on=on, right_on=on_ext, how=how, sort=False)
        # with on == on_ext the key is one column holding the left values
        for o, e in zip(on, on_ext):
            if o == e:
                out[o] = left[o].to_numpy()[out["__tmp__"].to_numpy()]
        out = out.sort_values(["__tmp__", "__ext_tmp__"], kind="stable", na_position="last")
    out = out.drop(columns=[c for c in ("__tmp__", "__ext_tmp__") if c in out.columns]).reset_index(drop=True)
    for c in ext.columns:
        if c in out.columns and len(ext) and ext[c].map(lambda v: isinstance(v, (list, tuple, np.ndarray))).any():
            out[c] = [v if isinstance(v, (list, tuple, np.ndarray)) else [] for v in out[c]]
    names = list(dict.fromkeys(list(df.columns) + list(ext.columns)))
    return out[names]
