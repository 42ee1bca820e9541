"""Groupby (reference nvtabular/ops/groupby.py:25-313): per partition,

    df.sort_values(sort_cols, ascending=ascending, kind="stable", na_position="last")
      .groupby(groupby_cols, sort=True, dropna=True).agg(...)

on the GPU (csrc/groupby.cu, family K8).  Rows are ordered by (group keys ascending, sort
columns) with the engine's own stable radix rounds, every group is a contiguous segment, and
each value column is gathered once into group order: that buffer is the `list` output, `first` /
`last` read its segment ends, and the reductions run over its segments in a fixed order, so the
outputs are bit-identical from run to run.

Rules the reference leaves to cuDF / pandas and this operator pins (tests/test_groupby_host.py):
- a row with a null (or NaN) group key is dropped; -0.0 and +0.0 are one key, written +0.0;
- nulls and NaN of a sort column come last in both directions; ties keep input order;
- `first` / `last` are positional (the ends of the `list`, nulls included), and with
  ascending=False `first` is the last element and `last` the first (groupby.py:290-297);
- output dtypes follow the aggregation, not the column name (the reference casts by a regex on
  the name, groupby.py:255-259).
"""
from typing import Dict, List, Tuple

import numpy as np
import torch

from .. import engine
from ..column import Column, DeviceFrame
from ..graph import ColumnSelector
from .base import Operator

AGGS = ("count", "sum", "mean", "var", "std", "median", "nunique", "min", "max", "first", "last", "list")
_REDUCE = ("count", "sum", "mean", "var", "std", "min", "max")
_NUMERIC_ONLY = ("sum", "mean", "var", "std", "median")
_AGG_DTYPES = {"count": np.dtype("int32"), "nunique": np.dtype("int32"), "sum": np.dtype("float32"),
               "mean": np.dtype("float32"), "var": np.dtype("float32"), "std": np.dtype("float32"),
               "median": np.dtype("float32")}
MAX_ROWS = 1 << 32          # row ids are 32-bit


def _bitlen(x: int) -> int:
    return int(x).bit_length()


def plan_rounds(widths: List[int], n: int) -> Tuple[int, List[List[Tuple[int, int, int]]]]:
    """The LSD round plan of "order rows by fields F1 > F2 > ...".

    widths: the bit width of every field, most significant first.  Elements are
    (packed fields << r) | row with r = bitlen(n - 1), so a round holds at most 64 - r field bits.
    Returns (r, rounds): rounds run least significant first; a round is a list of chunks
    (field index, lowest bit of the field, bits), least significant first.  Fields are packed
    greedily from the least significant one; a field wider than what is left of a round is split,
    its low chunk going to the earlier round."""
    r = _bitlen(max(n - 1, 0))
    cap = 64 - r
    rounds: List[List[Tuple[int, int, int]]] = []
    cur: List[Tuple[int, int, int]] = []
    used = 0
    for f in reversed(range(len(widths))):
        lo, w = 0, int(widths[f])
        while lo < w:
            take = min(w - lo, cap - used)
            if take == 0:
                rounds.append(cur)
                cur, used = [], 0
                continue
            cur.append((f, lo, take))
            used += take
            lo += take
    if cur:
        rounds.append(cur)
    return r, rounds


def _norm_agg(a) -> str:
    if a is list:
        return "list"
    if not isinstance(a, str) or a not in AGGS:
        raise ValueError(f"Groupby does not support the aggregation {a!r}; supported: {', '.join(AGGS)}")
    return a


def _as_list(x):
    if x is None:
        return []
    if isinstance(x, str):
        return [x]
    return list(x)


class Groupby(Operator):
    """Group each partition by `groupby_cols` and aggregate the other selected columns.

    The partition must already hold every row of a key (see `Dataset.shuffle_by_keys`): like the
    reference, this operator does not move rows between partitions."""

    def __init__(self, groupby_cols=None, sort_cols=None, aggs="list", name_sep="_", ascending=True):
        super().__init__()
        self.groupby_cols = _as_list(groupby_cols)
        self.sort_cols = _as_list(sort_cols)
        self.name_sep = name_sep
        self.ascending = bool(ascending)
        if isinstance(aggs, (str, list)) or aggs is list:
            aggs = {"__all__": aggs}
        if not isinstance(aggs, dict):
            raise ValueError(f"Groupby aggs must be a str, a list or a dict, got {type(aggs).__name__}")
        self.aggs: Dict[str, List[str]] = {}
        for col, v in aggs.items():
            vals = v if isinstance(v, (list, tuple)) else [v]
            self.aggs[col] = list(dict.fromkeys(_norm_agg(a) for a in vals))

    @property
    def dependencies(self):
        return list(self.groupby_cols) or None

    def _agg_dict(self, names) -> Dict[str, List[str]]:
        allowed = [c for c in names if c not in self.groupby_cols]
        if "__all__" in self.aggs:
            return {c: self.aggs["__all__"] for c in allowed}
        return {c: a for c, a in self.aggs.items() if c in allowed}

    def _outputs(self, names) -> Dict[str, Tuple[str, str]]:
        """output name -> (source column, agg); agg None for a group-by column"""
        out: Dict[str, Tuple[str, str]] = {}
        for k in self.groupby_cols:
            if k in names:
                out[k] = (k, None)
        for col, aggs in self._agg_dict(names).items():
            for a in aggs:
                out[f"{col}{self.name_sep}{a}"] = (col, a)
        return out

    def column_mapping(self, col_selector: ColumnSelector):
        return {name: [src] for name, (src, _) in self._outputs(col_selector.names).items()}

    def compute_output_schema(self, input_schema, col_selector):
        self._schema_outputs = self._outputs(col_selector.names)
        return super().compute_output_schema(input_schema, col_selector)

    def _compute_dtype(self, col_schema, input_schema):
        cs = super()._compute_dtype(col_schema, input_schema)
        agg = getattr(self, "_schema_outputs", {}).get(cs.name, (None, None))[1]
        if agg in _AGG_DTYPES:
            return cs.with_dtype(_AGG_DTYPES[agg], False, False)
        if agg == "list":
            return cs.with_dtype(cs.dtype, True, True)
        return cs

    # ------------------------------------------------------------------------------ transform
    def transform(self, col_selector: ColumnSelector, df: DeviceFrame) -> DeviceFrame:
        outputs = self._outputs(col_selector.names)
        cols = {name: self._get(df, name) for name in dict.fromkeys(
            [s for s, _ in outputs.values()] + self.groupby_cols + self.sort_cols)}
        for name, (src, agg) in outputs.items():
            c = cols[src]
            if agg is None:
                continue
            if c.is_list and agg == "list":
                raise ValueError(f"Groupby: a list of the list column {src!r} (nested lists) is not supported")
            if c.is_list and agg not in ("first", "last"):
                raise ValueError(f"Groupby: {agg!r} of the list column {src!r} is not supported")
            if c.is_string and agg in _NUMERIC_ONLY:
                raise TypeError(f"Groupby: {agg!r} of the string column {src!r}")
        for k in self.groupby_cols + self.sort_cols:
            if cols[k].is_list:
                raise ValueError(f"Groupby: the list column {k!r} cannot be a group-by or sort column")
        n = len(df)
        if n >= MAX_ROWS:
            raise ValueError(f"Groupby: a partition of {n} rows; row ids are 32-bit, so at most 2^32 - 1")
        if not self.groupby_cols:
            raise ValueError("Groupby needs groupby_cols")
        if n == 0:
            return self._empty(outputs, cols)
        dev = cols[self.groupby_cols[0]].data.device

        # 1. order codes of the keys and sort columns; ONE host read of their {min, max, n_valid}
        keys = [cols[k] for k in self.groupby_cols]
        sorts = [cols[s] for s in self.sort_cols]
        stats = torch.empty((len(keys) + len(sorts), 3), dtype=torch.int64, device=dev)
        key_valid = engine._bitmask(n, dev)
        kc, sc = [], []
        for i, c in enumerate(keys):
            kc.append(engine.gb_order_codes(c, stats[i], key_valid, and_key_valid=i > 0))
        for j, c in enumerate(sorts):
            sc.append(engine.gb_order_codes(c, stats[len(keys) + j]))
        st = stats.cpu().numpy().view(np.uint64)
        if any(int(st[i, 2]) == 0 for i in range(len(keys))):
            return self._empty(outputs, cols)
        null_keys = any(int(st[i, 2]) < n for i in range(len(keys)))

        # 2. order rows by (null-key flag, keys ascending, sort columns)
        fields = []            # (codes, valid, min, span, mode, width), most significant first
        if null_keys:
            fields.append((kc[0][0], key_valid, 0, 0, 3, 1))
        for i, (codes, _) in enumerate(kc):
            mn, mx = int(st[i, 0]), int(st[i, 1])
            fields.append((codes, None, mn, mx - mn, 0, _bitlen(mx - mn)))
        for j, (codes, valid) in enumerate(sc):
            fields += _sort_fields(codes, valid, st[len(keys) + j], n, self.ascending)
        order, r = _order_rows(fields, n, dev)

        # 3. segments: the second host read
        off, g, kept = engine.gb_segments(order, r, [c for c, _ in kc], key_valid if null_keys else None)
        if g == 0:
            return self._empty(outputs, cols)

        # 4-6. values: the keys at every group's first row, the value columns in group order
        key_out = {name: cols[src] for name, (src, agg) in outputs.items() if agg is None}
        out = dict(zip(key_out, engine.gather(list(key_out.values()), engine.order_sel(order, r, 1, off), g,
                                              canon_zero=[c.data.dtype.is_floating_point for c in key_out.values()])))
        srcs = list(dict.fromkeys(s for s, a in outputs.values() if a is not None and not cols[s].is_list))
        bufs = dict(zip(srcs, engine.gather([cols[s] for s in srcs], engine.order_sel(order, r), kept)))
        for end in (1, 2):
            ends = {name: src for name, (src, agg) in outputs.items()
                    if agg in ("first", "last") and self._end(agg) == end}
            flat = {name: bufs[src] for name, src in ends.items() if not cols[src].is_list}
            lists = {name: cols[src] for name, src in ends.items() if cols[src].is_list}
            out.update(engine.take_rows(flat, engine.RowSel(off=off, which=end), g))
            out.update(engine.take_rows(lists, engine.order_sel(order, r, end, off), g))
        rank_cols = {}
        for name, (src, agg) in outputs.items():
            if agg == "list":
                buf = bufs[src]
                out[name] = Column(buf.data, buf.validity, off, buf.dictionary, None, buf.is_bool)
            elif agg in ("median", "nunique"):
                rank_cols.setdefault(src, set()).add(agg)
        reduced = {}
        for src in bufs:
            want = [a for s, a in outputs.values() if s == src and a in _REDUCE]
            if want:
                reduced[src] = engine.gb_reduce(bufs[src], off, g, want)
        ranked = _rank_stats({s: bufs[s] for s in rank_cols}, rank_cols, off, g, kept, dev)
        for name, (src, agg) in outputs.items():
            if agg in _REDUCE:
                out[name] = reduced[src][agg]
            elif agg in ("median", "nunique"):
                out[name] = ranked[(src, agg)]
        return DeviceFrame({name: out[name] for name in outputs})

    def _end(self, agg) -> int:
        """gather mode of `first` / `last`: 1 = segment start, 2 = segment end; swapped when
        descending, as the reference's _first_or_last does"""
        first = (agg == "first") == self.ascending
        return 1 if first else 2

    def _empty(self, outputs, cols) -> DeviceFrame:
        out = DeviceFrame()
        for name, (src, agg) in outputs.items():
            c = cols[src]
            dev = c.data.device
            if agg in _AGG_DTYPES:
                dt = torch.int32 if _AGG_DTYPES[agg].kind == "i" else torch.float32
                out[name] = Column(torch.empty(0, dtype=dt, device=dev))
            elif agg == "list" or (c.is_list and agg in ("first", "last")):
                out[name] = Column(torch.empty(0, dtype=c.data.dtype, device=dev), None,
                                   torch.zeros(1, dtype=torch.int64, device=dev), c.dictionary, None, c.is_bool)
            else:
                out[name] = Column(torch.empty(0, dtype=c.data.dtype, device=dev), None, None, c.dictionary, None,
                                   c.is_bool)
        return out


def _sort_fields(codes, valid, st, n, ascending):
    """the fields of one sort column: nulls and NaN in a last slot after the largest value, in both
    directions; a descending column is complemented within its width"""
    nv, mn, mx = int(st[2]), int(st[0]), int(st[1])
    if nv == 0:
        return []                       # all null: every row ties
    span = mx - mn
    mode = 1 if ascending else 2
    if nv == n:
        return [(codes, valid, mn, span, mode, _bitlen(span))]
    if span == (1 << 64) - 1:           # no free slot above the full 64-bit range: a null flag first
        return [(codes, valid, 0, 0, 3, 1), (codes, valid, mn, span, mode, 64)]
    return [(codes, valid, mn, span, mode, _bitlen(span + 1))]


def _order_rows(fields, n, dev):
    r, rounds = plan_rounds([f[5] for f in fields], n)
    chunks, sizes = [], []
    for rnd in rounds:
        for f, lo, bits in rnd:
            codes, valid, mn, span, mode, _ = fields[f]
            chunks.append((codes, valid, mn, span, mode, lo, bits))
        sizes.append(len(rnd))
    return engine.gb_order_rows(chunks, sizes, n, r, dev), r


def _rank_stats(bufs, wanted, off, g, kept, dev):
    """median / nunique: the group-ordered values ordered again by (group, value), nulls last in
    a group, with the same row-ordering primitive; one host read for every column's code range"""
    if not bufs:
        return {}
    stats = torch.empty((len(bufs), 3), dtype=torch.int64, device=dev)
    codes = {s: engine.gb_order_codes(b, stats[i]) for i, (s, b) in enumerate(bufs.items())}
    st = stats.cpu().numpy().view(np.uint64)
    gid = engine.gb_segment_ids(off, g, kept)
    res = {}
    for i, (s, b) in enumerate(bufs.items()):
        c, v = codes[s]
        fields = [(gid, None, 0, g - 1, 0, _bitlen(g - 1))] + _sort_fields(c, v, st[i], kept, True)
        order, r = _order_rows(fields, kept, dev)
        med, nun = engine.gb_rank_stats(b, c, v, order, r, off, g, "median" in wanted[s], "nunique" in wanted[s])
        if med is not None:
            res[(s, "median")] = Column(med)
        if nun is not None:
            res[(s, "nunique")] = Column(nun)
    return res

