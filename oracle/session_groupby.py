"""Oracle for the Groupby operator — TEST INFRASTRUCTURE.

Restates reference nvtabular/ops/groupby.py on pandas, with the rules the engine pins
(nvtabular_b200/ops/groupby.py):
  sort          Groupby.transform: df.sort_values(sort_cols, ascending)        groupby.py:118-120,
                here kind="stable", na_position="last" (ties keep input order: a documented
                deviation, like kind="stable" of the Categorify oracle)
  groups        _apply_aggs: df.groupby(groupby_cols).agg(conv_aggs)           groupby.py:222-227,
                sort=True, dropna=True; a NaN key is null; -0.0 and +0.0 are one key (+0.0)
  aggs          _get_agg_dicts / _ensure_agg_dict: "__all__" = every non-key   groupby.py:262-276
  first / last  _first_or_last: ends of the "list" aggregation, swapped when
                ascending=False                                                 groupby.py:290-313
  dtypes        by the aggregation requested (count / nunique int32; sum, mean, var, std, median
                float32), not by the regex on the name of groupby.py:255-259
Results are python values per group (None = null), so int64 extremes and the nulls of integer
outputs compare exactly.
"""
import math
from typing import Dict, List

import numpy as np
import pandas as pd

AGGS = ("count", "sum", "mean", "var", "std", "median", "nunique", "min", "max", "first", "last", "list")


def _norm_aggs(aggs) -> Dict[str, List[str]]:
    """Groupby.__init__'s normalisation (groupby.py:86-107): str / list -> "__all__"."""
    if isinstance(aggs, (str, list)) or aggs is list:
        aggs = {"__all__": aggs}
    out = {}
    for col, v in aggs.items():
        vals = v if isinstance(v, (list, tuple)) else [v]
        out[col] = list(dict.fromkeys("list" if a is list else a for a in vals))
    return out


def _isnull(v) -> bool:
    return v is None or v is pd.NA or (isinstance(v, float) and math.isnan(v))


def session_groupby(df: pd.DataFrame, groupby_cols, sort_cols=None, aggs="list", name_sep="_",
                    ascending=True, columns=None):
    """-> {output name: list of per-group python values} (None = null), groups in key order.
    A value of a `list` output is a python list (None for a null leaf)."""
    keys = [groupby_cols] if isinstance(groupby_cols, str) else list(groupby_cols)
    sorts = [sort_cols] if isinstance(sort_cols, str) else list(sort_cols or [])
    columns = list(columns) if columns is not None else list(df.columns)
    aggd = _norm_aggs(aggs)
    allowed = [c for c in columns if c not in keys]                       # groupby.py:262-268
    aggd = {c: aggd["__all__"] for c in allowed} if "__all__" in aggd else \
        {c: a for c, a in aggd.items() if c in allowed}                   # groupby.py:271-276
    d = df.reset_index(drop=True).copy()
    for k in keys:
        if pd.api.types.is_float_dtype(d[k].dtype):
            d[k] = d[k] + 0.0                                             # -0.0 -> +0.0
    if sorts:
        d = d.sort_values(sorts, ascending=ascending, kind="stable", na_position="last")   # groupby.py:118-120
    out: Dict[str, list] = {}
    grouped = d.groupby(keys[0] if len(keys) == 1 else keys, sort=True, dropna=True)   # groupby.py:222-227
    groups = list(grouped.groups.keys()) if len(d) else []
    index = [grouped.indices[g] for g in groups]
    for k_i, k in enumerate(keys):
        if k in columns:
            out[k] = [(g if len(keys) == 1 else g[k_i]) for g in groups]
            out[k] = [None if _isnull(v) else v for v in out[k]]
    for col, col_aggs in aggd.items():
        vals = d[col].tolist()
        for a in col_aggs:
            res = []
            for idx in index:
                seg = [vals[i] for i in idx]
                res.append(_agg(seg, a, ascending))
            out[f"{col}{name_sep}{a}"] = res
    return out


def _agg(seg, a, ascending):
    """one aggregation of one group's values in sorted order"""
    if a == "list":
        return [None if _isnull(v) else v for v in seg]
    if a in ("first", "last"):                                            # groupby.py:290-313
        pick_first = (a == "first") == ascending
        v = seg[0] if pick_first else seg[-1]
        if isinstance(v, (list, np.ndarray)):
            return list(v)
        return None if _isnull(v) else v
    valid = [v for v in seg if not _isnull(v)]
    if a == "count":
        return len(valid)
    if a == "nunique":
        return len({(v + 0.0) if isinstance(v, float) else v for v in valid})
    if a in ("min", "max"):
        if not valid:
            return None
        return min(valid) if a == "min" else max(valid)
    x = np.asarray(valid, dtype=np.float64)
    if a == "sum":
        return float(np.float32(math.fsum(x))) if len(x) else 0.0
    if a == "mean":
        return float(np.float32(math.fsum(x) / len(x))) if len(x) else float("nan")
    if a in ("var", "std"):
        if len(x) < 2:
            return float("nan")
        var = float(np.var(x, ddof=1))
        return float(np.float32(var if a == "var" else math.sqrt(var)))
    if a == "median":
        return float(np.float32(np.median(x))) if len(x) else float("nan")
    raise ValueError(a)
