"""Dropna (reference nvtabular/ops/dropna.py:33-37): df.dropna(subset=<selected columns>) on every
partition, on the GPU (csrc/filter.cu, family K11): one mask pass over the selected columns, then
the row selection of ops/filter.py.

- A row is dropped when any selected column is null there or is a float holding NaN there, including
  a NaN a kernel wrote under a set validity bit (LogOp of a negative value, for example).
- A list row is never NA: Column.from_arrow already reads a null list row as an empty one, so list
  columns never drop a row.
- When no selected column has a validity bitmask and none is a float, the partition is returned
  without launching anything.
The operator returns every selected column, has no fit state, serving hook or collective, and
partitions may shrink or become empty.  Branches of different lengths cannot be merged: where the
reference silently misaligns `(cols >> Dropna()) + other`, Workflow raises ValueError.
"""
from .. import engine
from ..column import DeviceFrame
from ..graph import ColumnSelector
from .base import Operator
from .filter import Mask, compact


class Dropna(Operator):
    """Drop the rows in which any selected column is null (or NaN)."""

    def transform(self, col_selector: ColumnSelector, df: DeviceFrame) -> DeviceFrame:
        df = DeviceFrame({n: self._get(df, n) for n in col_selector.names})
        check = [c for _, c in df.items()
                 if not c.is_list and (c.validity is not None or c.data.is_floating_point())]
        if not check:
            return df
        n = len(df)
        return compact(df, Mask(engine.mask_notnull(check, n), n))
