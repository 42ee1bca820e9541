"""ListSlice (reference nvtabular/ops/list_slice.py:29-177): every row of a list column sliced like
Python's row[start:end], and with pad=True padded at the end with pad_value up to max_elements, on
the GPU (csrc/session.cu, family K10).  Without pad the leaf bounds of every row are one pass and
the copy is nvtb_gb_list_rows, balanced over output elements; with pad the output is dense (n x
max_elements) and written in one pass, with no scan and no host read.

Rules the reference leaves open and this operator pins (tests/test_session_ops_host.py):
- slicing is Python's row[start:end], the reference's CPU branch; start / end / max_elements are
  normalised as the reference does (list_slice.py:58-75);
- leaf nulls inside a list are kept.  DEVIATION: the reference's GPU branch drops them (it copies
  elements.values);
- the input must be a list column (ValueError); it is never written, since a Groupby list output
  shares its leaf buffer with the other aggregations of the column;
- pad=True with an unbounded slice (ListSlice(0, pad=True)) or with max_elements <= 0
  (ListSlice(1, -1, pad=True)) raises ValueError in __init__;
- pad_value is converted to the leaf dtype: an integer or bool leaf takes it only when the value
  survives the conversion exactly (1.5 or NaN raise ValueError), a float leaf takes the nearest
  value of its width (a finite value that overflows raises ValueError); pad=True on a string-leaf
  column raises TypeError.
The operator has no fit state and works on one partition at a time.
"""
import math

import numpy as np

from .. import engine
from ..column import Column, DeviceFrame
from ..graph import ColumnSelector, Tags
from .base import Operator

INT64_MAX = int(np.iinfo(np.int64).max)
INT64_MIN = int(np.iinfo(np.int64).min)


def _as_index(name, v):
    if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, np.integer)):
        raise TypeError(f"ListSlice: {name} must be an int, got {type(v).__name__}")
    return int(v)


def pad_bits(value, col: Column) -> int:
    """the bit pattern of pad_value in the leaf dtype of `col` (low bytes of a uint64)"""
    if col.is_string:
        raise TypeError("ListSlice: pad=True on a list of strings; a string leaf has no pad value")
    x = value.item() if isinstance(value, np.generic) else value
    if isinstance(x, bool):
        x = int(x)
    if not isinstance(x, (int, float)):
        raise ValueError(f"ListSlice: pad_value {value!r} is not a number")
    dt = np.dtype(str(col.data.dtype).replace("torch.", ""))
    if dt.kind in "iu":
        if isinstance(x, float) and not (math.isfinite(x) and x == int(x)):
            raise ValueError(f"ListSlice: pad_value {value!r} is not a value of the {col.np_dtype} leaves")
        info = (0, 1) if col.is_bool else (int(np.iinfo(dt).min), int(np.iinfo(dt).max))
        if not info[0] <= int(x) <= info[1]:
            raise ValueError(f"ListSlice: pad_value {value!r} is not a value of the {col.np_dtype} leaves")
        conv = np.array(int(x), dtype=dt)
    else:
        with np.errstate(over="ignore"):
            conv = np.array(x, dtype=dt)
        if math.isfinite(x) and not np.isfinite(conv):
            raise ValueError(f"ListSlice: pad_value {value!r} overflows the {dt} leaves")
    return int.from_bytes(conv.tobytes(), "little")


class ListSlice(Operator):
    """Slice every row of a list column.

    ListSlice(10) keeps the first 10 elements, ListSlice(1, 11) the 10 after the first and
    ListSlice(-10) the last 10.  pad=True pads every row at the end with pad_value to
    max_elements elements, which makes the column fixed-length."""

    def __init__(self, start, end=None, pad=False, pad_value=0.0):
        super().__init__()
        start = _as_index("start", start)
        end = None if end is None else _as_index("end", end)
        self.pad = bool(pad)
        self.pad_value = pad_value
        # the reference's normalisation (list_slice.py:65-75)
        if start > 0 and end is None:
            start, end = 0, start
        if end is None:
            end = INT64_MAX
        self.start, self.end = start, end
        if start < 0:
            self.max_elements = -(start if end > 0 else start - end)
        else:
            self.max_elements = end - start
        if self.pad:
            if start >= 0 and end >= INT64_MAX:
                raise ValueError(f"ListSlice: pad=True needs a bounded slice; ListSlice({start}, pad=True) keeps "
                                 "every element of a row, so there is no length to pad to")
            if self.max_elements <= 0:
                raise ValueError(f"ListSlice: pad=True with start={start}, end={end} gives max_elements "
                                 f"{self.max_elements}; it must be positive")

    @property
    def output_tags(self):
        return [Tags.LIST]

    def _compute_dtype(self, col_schema, input_schema):
        cs = super()._compute_dtype(col_schema, input_schema)
        return cs.with_dtype(cs.dtype, True, not self.pad)

    def _compute_properties(self, col_schema, input_schema):
        cs = super()._compute_properties(col_schema, input_schema)
        value_count = {"min": 0, "max": None}
        if self.max_elements != INT64_MAX:
            value_count["max"] = self.max_elements
            if self.pad:
                value_count["min"] = self.max_elements
        return cs.with_properties({"value_count": value_count})

    def transform(self, col_selector: ColumnSelector, df: DeviceFrame) -> DeviceFrame:
        cols = {name: self._get(df, name) for name in col_selector.names}
        bits = {}
        for name, c in cols.items():
            if not c.is_list:
                raise ValueError(f"ListSlice: the column {name!r} is not a list column")
            if self.pad:
                bits[name] = pad_bits(self.pad_value, c)
        # Python's slice semantics are unchanged by clamping the bounds to int64
        start = max(INT64_MIN, min(INT64_MAX, self.start))
        end = max(INT64_MIN, min(INT64_MAX, self.end))
        out = DeviceFrame()
        for name, c in cols.items():
            if self.pad:
                out[name] = engine.list_slice_pad(c, start, end, self.max_elements, bits[name])
            else:
                out[name] = engine.list_slice(c, start, end)
        return out
