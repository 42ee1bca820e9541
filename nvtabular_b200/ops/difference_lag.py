"""DifferenceLag (reference nvtabular/ops/difference_lag.py:23-105): for every shift s and value
column x, the float32 column x[i] - x[i - s], null where row i - s belongs to another partition key
(the lag within a user's or session's events), on the GPU (csrc/session.cu, family K10): one pass
over the partition columns writes a same-key bitmask, one pass over up to 16 value columns writes
the lags.

The frame must already be ordered by (partition columns, time) within each Dataset partition, as
the reference requires; the operator does not sort, and a lag never crosses a Dataset partition
(the reference's map_partitions).  Rules (tests/test_session_ops_host.py):
- row i has a lag when 0 <= i - s < len(partition) and every partition column is valid and equal
  at i and i - s: a null or NaN key never matches, -0.0 matches +0.0, shift=0 gives 0 and a shift
  beyond the partition gives nulls;
- integer columns subtract in int64, wrapping like cuDF, and round once to float32 (the
  reference's GPU branch; pandas' float64 operands differ above 2^53); float32 subtracts in
  float32; float64 subtracts in float64 and rounds to float32; a NaN operand gives NaN;
- bool, string and list value columns raise TypeError, as does a shift that is not an int;
  at most 8 partition columns (ValueError).
The reference's literal CPU code (`mask[mask == False] = None` on a bool Series) raises TypeError
on current pandas; oracle/session_ops.py restates its intent.  There is no fit state and no
collective; Workflow.save raises for this operator, as the reference has no serializer for it.
"""
import numpy as np

from .. import engine
from ..column import DeviceFrame
from ..graph import ColumnSelector, Tags
from .base import Operator


def _is_int(x):
    return isinstance(x, (int, np.integer)) and not isinstance(x, (bool, np.bool_))


class DifferenceLag(Operator):
    """Difference between a row and the row `shift` rows before it (after it for a negative shift)
    when both rows share every partition column; output columns {col}_difference_lag_{shift}."""

    def __init__(self, partition_cols, shift=1):
        super().__init__()
        if isinstance(partition_cols, str):
            partition_cols = [partition_cols]
        self.partition_cols = list(partition_cols)
        if not self.partition_cols:
            raise ValueError("DifferenceLag needs at least one partition column")
        shifts = [shift] if _is_int(shift) else shift
        if not isinstance(shifts, (list, tuple)) or not shifts or not all(_is_int(s) for s in shifts):
            raise TypeError(f"DifferenceLag: shift must be an int or a list of ints, got {shift!r}")
        self.shifts = [int(s) for s in shifts]

    @property
    def dependencies(self):
        return self.partition_cols

    def column_mapping(self, col_selector: ColumnSelector):
        return {self._column_name(col, s): [col] for col in col_selector.names for s in self.shifts}

    @property
    def output_tags(self):
        return [Tags.CONTINUOUS]

    @property
    def output_dtype(self):
        return np.float32

    def _compute_dtype(self, col_schema, input_schema):
        return super()._compute_dtype(col_schema, input_schema).with_dtype(np.dtype(np.float32), False, False)

    def _column_name(self, col, shift):
        return f"{col}_difference_lag_{shift}"

    def _partition_names(self):
        names = []
        for p in self.partition_cols:
            for n in ([p] if isinstance(p, str) else p.output_columns.names):
                if n not in names:
                    names.append(n)
        return names

    def transform(self, col_selector: ColumnSelector, df: DeviceFrame) -> DeviceFrame:
        key_names = self._partition_names()
        if len(key_names) > engine.LAG_MAX_KEYS:
            raise ValueError(f"DifferenceLag: at most {engine.LAG_MAX_KEYS} partition columns, got {len(key_names)}")
        keys = [self._get(df, k) for k in key_names]
        for k, c in zip(key_names, keys):
            if c.is_list:
                raise ValueError(f"DifferenceLag: the list column {k!r} cannot be a partition column")
        names = list(col_selector.names)
        vals = [self._get(df, c) for c in names]
        for name, c in zip(names, vals):
            kind = "list" if c.is_list else ("string" if c.is_string else ("bool" if c.is_bool else None))
            if kind is not None:
                raise TypeError(f"DifferenceLag: the {kind} column {name!r} has no difference")
        if not vals:
            return DeviceFrame()
        n = len(df)
        out = {}
        for s in self.shifts:
            same = engine.lag_same_key(keys, n, s)
            for name, col in zip(names, engine.difference_lag(vals, same, s)):
                out[self._column_name(name, s)] = col
        return DeviceFrame({k: out[k] for k in self.column_mapping(col_selector)})
