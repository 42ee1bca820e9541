"""pandas restatements of the row-selection operators (nvtabular_b200/ops/filter.py, ops/dropna.py).

Filter (reference nvtabular/ops/filter.py:51-62): f(df); a DataFrame result is the output, a bool
Series indexes the frame (pandas boolean indexing), anything else raises ValueError; then
reset_index(drop=True).  A bool Series holding nulls (a nullable boolean) counts a null as false.

Dropna (reference nvtabular/ops/dropna.py:33-37): df.dropna(subset=<selected columns>), then
reset_index(drop=True).  A list cell is never NA here: the engine reads a null list row as an
empty list, so list columns are left out of the subset.
"""
from typing import Callable, Optional, Sequence

import numpy as np
import pandas as pd


def filter_frame(df: pd.DataFrame, f: Callable) -> pd.DataFrame:
    """reference filter.py:51-62"""
    res = f(df)
    if isinstance(res, pd.DataFrame):
        out = res
    elif isinstance(res, pd.Series) and (res.dtype == bool or pd.api.types.is_bool_dtype(res.dtype)):
        out = df[res.fillna(False).astype(bool)]
    else:
        raise ValueError(f"Invalid output from filter op: f{res.__class__}")
    return out.reset_index(drop=True)


def _is_list_column(s: pd.Series) -> bool:
    return s.dtype == object and any(isinstance(v, (list, tuple, np.ndarray)) for v in s)


def dropna_frame(df: pd.DataFrame, subset: Optional[Sequence[str]] = None) -> pd.DataFrame:
    """reference dropna.py:33-37"""
    cols = [c for c in (subset or list(df.columns)) if not _is_list_column(df[c])]
    out = df.dropna(subset=cols) if cols else df
    return out.reset_index(drop=True)
