"""JoinGroupby (reference nvtabular/ops/join_groupby.py:37-283; statistics by
nvtabular/ops/categorify.py:955-1137 with agg columns).

fit        one resident device hash table per key group carrying
           {size, sum, sumsq, min, max} per continuous column (K3 with payload)
transform  one probe + gather pass per group (K7) — no merge, no sort by __tmp__.
"""
import os
from typing import Dict, List

import numpy as np
import pandas as pd
import torch

from .. import engine
from ..column import Column, DeviceFrame
from ..dist import global_merge
from ..graph import ColumnSelector, Node
from .base import StatOperator
from .keyspace import ComboKeySpace, KeySpace, _leaf

AGG_DTYPES = {"count": np.int32, "std": np.float32, "var": np.float32, "mean": np.float32}  # join_groupby.py:29-34
# sum / min / max keep the dtype the statistics file holds instead of float64 (only AGG_DTYPES are
# recast, join_groupby.py:211-214, 252-261): pandas / cuDF reduce a float32 column in float32, keep
# min / max of an int column in its dtype, and sum an int column into int64 (pandas keeps int32 for
# an int32 sum that fits, and widens one that does not).  The engine sums in fp64: an int64 sum is
# exact while |sum| < 2^53.
_TYPED_STATS = ("sum", "min", "max")
_KEEP_DTYPES = (np.dtype(np.float32), np.dtype(np.int32), np.dtype(np.int64))


def _kept_dtype(dt, stat="min"):
    """the dtype of statistic `stat` (sum/min/max) of a column of dtype `dt`, or None (float64)"""
    try:
        dt = np.dtype(getattr(dt, "numpy_dtype", dt)) if dt is not None else None
    except TypeError:
        return None
    if dt not in _KEEP_DTYPES:
        return None
    return np.dtype(np.int64) if stat == "sum" and dt.kind == "i" else dt


def _make_name(*args, sep="_"):
    return sep.join(args)


class GroupTable:
    """`cat_stats.<name>.parquet` of the reference + the device gather handle."""

    def __init__(self, name, key_names, space, keys, stat_names, stats, null_row, first_null):
        self.name = name
        self.key_names = key_names
        self.space = space
        self.keys = keys                  # device int64 [U]
        self.stat_names = stat_names      # column names of the stats matrix
        self.stats = stats                # device float64 [U (+1 null row), len(stat_names)]
        self.null_row = null_row
        self.first_null = first_null
        self.handle = engine.GroupStats(keys, stats, null_row)
        self.path = None

    @classmethod
    def from_parquet(cls, name, path, sep="_") -> "GroupTable":
        """rebuild the device table from a cat_stats.<name>.parquet file (this engine's or the
        reference's, categorify.py:1073-1137): key columns = everything that is not a
        `<name>_...` statistic; the row with a null key becomes the null group"""
        from ._tables import keys_from_frame
        df = pd.read_parquet(path)
        stat_names = [c for c in df.columns if c.startswith(name + sep)]
        key_names = [c for c in df.columns if c not in stat_names]
        space, keys, isnull = keys_from_frame(df, key_names)
        mat = torch.from_numpy(df[stat_names].to_numpy(dtype=np.float64, na_value=np.nan)).to(keys.device) \
            if stat_names else \
            torch.zeros((len(df), 1), dtype=torch.float64, device=keys.device)
        null_idx = torch.nonzero(isnull).flatten()
        keep = ~isnull
        null_row = -1
        stats = mat[keep]
        if null_idx.numel():
            stats = torch.cat([stats, mat[null_idx[:1]]], dim=0)
            null_row = int(keep.sum().item())
        t = cls(name, key_names, space, keys[keep].contiguous(), stat_names, stats.contiguous(), null_row, None)
        t.stat_dtypes = {c: _kept_dtype(df[c].dtype) for c in stat_names
                         if c.rsplit(sep, 1)[-1] in _TYPED_STATS and _kept_dtype(df[c].dtype) is not None}
        t.path = path
        return t

    def frame(self) -> pd.DataFrame:
        from ._tables import key_columns
        k = self.keys.cpu().numpy()
        st = self.stats.cpu().numpy()
        data = key_columns(self.space, self.key_names, k, with_null_row=self.null_row >= 0)
        rows = len(k) + (1 if self.null_row >= 0 else 0)
        typed = getattr(self, "stat_dtypes", {})
        for j, sn in enumerate(self.stat_names):
            col = st[:rows, j]
            if sn.endswith("_count"):                  # the reference's file holds integer counts
                col = col.astype(np.int64)
            elif sn in typed and (typed[sn].kind == "f" or not np.isnan(col).any()):
                col = col.astype(typed[sn])            # ... and sum/min/max in the column's dtype
            elif sn in typed:                          # an int min/max of a group without values
                col = pd.array(np.where(np.isnan(col), 0, col).astype(typed[sn]), dtype=f"Int{typed[sn].itemsize * 8}")
                col[np.isnan(st[:rows, j])] = pd.NA
            data[sn] = col
        return pd.DataFrame(data)

    def write(self, base, force=True):
        """cat_stats.<name>.parquet (categorify.py:1500-1503).  Tables above 2^20 groups are written
        when their path is first read (`op.categories[name]`, Workflow.save): decoding tens of
        millions of group keys on the host is seconds of pandas work the transform never needs —
        the same rule as Categorify's large vocabulary files."""
        os.makedirs(base, exist_ok=True)
        self.path = os.path.join(base, f"cat_stats.{self.name}.parquet")
        lazy = os.environ.get("NVTB_ARTIFACTS", "eager").lower() == "lazy"
        if force or (not lazy and self.keys.numel() <= (1 << 20)):
            self.frame().to_parquet(self.path)
            self._written = True
        else:
            self._written = False
        return self.path

    def ensure_written(self):
        if self.path is not None and not getattr(self, "_written", True):
            self.write(os.path.dirname(self.path), force=True)


class _StatPaths(dict):
    """group name -> cat_stats path; reading a path makes sure a deferred file exists"""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.tables = {}

    def __getitem__(self, key):
        t = self.tables.get(key)
        if t is not None:
            t.ensure_written()
        return super().__getitem__(key)


def build_group_table(name, key_names, space, agg: engine.HashAgg, cont_names, stats, sep="_") -> GroupTable:
    """_bottom_level_groupby (categorify.py:1073-1137) on the merged table, on device."""
    keys, sizes, vals, null_size, null_vals = global_merge(agg)
    dev = keys.device
    U = keys.numel()
    has_null = null_size > 0
    sizes_f = sizes.to(torch.float64)
    # "count" is pandas count() of the FIRST key column (categorify.py:989-999):
    # == size when that component is non-null, 0 otherwise
    if isinstance(space, ComboKeySpace):
        fn = space.first_component_null_t(keys) if U else \
            torch.zeros(0, dtype=torch.bool, device=dev)
        count = torch.where(fn, torch.zeros_like(sizes_f), sizes_f)
    else:
        count = sizes_f.clone()
    if has_null:
        count = torch.cat([count, torch.zeros(1, dtype=torch.float64, device=dev)])
        if vals is not None:
            nv = torch.tensor(null_vals, dtype=torch.float64, device=dev).reshape(1, -1, 4)
            vals = torch.cat([vals, nv], dim=0)
    cols, names = [], []
    prefix = name
    if "count" in stats:
        names.append(_make_name(prefix, "count", sep=sep))
        cols.append(count)
    for j, cont in enumerate(cont_names):
        s, s2, mn, mx = vals[:, j, 0], vals[:, j, 1], vals[:, j, 2], vals[:, j, 3]
        if "sum" in stats:
            names.append(_make_name(prefix, cont, "sum", sep=sep)); cols.append(s)
        if "mean" in stats:
            names.append(_make_name(prefix, cont, "mean", sep=sep)); cols.append(s / count)
        if "min" in stats:
            names.append(_make_name(prefix, cont, "min", sep=sep)); cols.append(mn)
        if "max" in stats:
            names.append(_make_name(prefix, cont, "max", sep=sep)); cols.append(mx)
        if "var" in stats or "std" in stats:
            result = s2 - s * s / count                      # categorify.py:1114-1118
            div = torch.clamp(count - 1, min=1.0)
            result = result / div
            result = torch.where((count - 1) == 0, torch.full_like(result, float("nan")), result)
            if "var" in stats:
                names.append(_make_name(prefix, cont, "var", sep=sep)); cols.append(result)
            if "std" in stats:
                names.append(_make_name(prefix, cont, "std", sep=sep)); cols.append(torch.sqrt(result))
    mat = torch.stack(cols, dim=1) if cols else torch.zeros((U + int(has_null), 1), dtype=torch.float64, device=dev)
    return GroupTable(name, key_names, space, keys, names, mat, U if has_null else -1, None)


class JoinGroupby(StatOperator):
    def __init__(self, cont_cols=None, stats=("count",), tree_width=None, split_out=None, split_every=None,
                 cat_cache="host", out_path=None, on_host=True, name_sep="_"):
        super().__init__()
        self.storage_name = {}
        self.name_sep = name_sep
        self.stats = list(stats)
        self.split_out = split_out
        self.split_every = split_every
        self.out_path = out_path or "./"
        self.on_host = on_host
        self.cat_cache = cat_cache
        self.categories: Dict[str, str] = _StatPaths()
        self.tables: Dict[str, GroupTable] = {}
        self._cont_names = None
        if isinstance(cont_cols, Node):
            self.cont_cols = cont_cols
        elif isinstance(cont_cols, ColumnSelector):
            self.cont_cols = self._cont_names = cont_cols
        else:
            self.cont_cols = self._cont_names = ColumnSelector(cont_cols or [])
        supported_ops = ["count", "sum", "mean", "std", "var", "min", "max"]
        for op in self.stats:
            if op not in supported_ops:
                raise ValueError(op + " operation is not supported.")      # join_groupby.py:123-126

    @property
    def cont_names(self):
        if self._cont_names is not None:
            return self._cont_names
        return self.cont_cols.output_columns

    @property
    def dependencies(self):
        return self.cont_cols if isinstance(self.cont_cols, Node) else (
            Node(self.cont_cols) if self.cont_cols else None)

    def _groups(self, col_selector):
        out = []
        for g in col_selector.grouped_names:
            names = list(g) if isinstance(g, tuple) else [g]
            out.append((_make_name(*names, sep=self.name_sep), names))
        return out

    def fit(self, col_selector: ColumnSelector, ddf):
        parts = list(ddf)
        cont = self.cont_names.names
        tables = {}
        for name, names in self._groups(col_selector):
            tables[name] = fit_group_table(name, names, parts, cont, self.stats, self.name_sep)
        return tables

    def fit_finalize(self, tables):
        base = os.path.join(self.out_path, "categories")
        for name, t in tables.items():
            self.tables[name] = t
            self.categories[name] = t.write(base, force=False)
            if isinstance(self.categories, _StatPaths):
                self.categories.tables[name] = t

    def transform(self, col_selector: ColumnSelector, df: DeviceFrame) -> DeviceFrame:
        new_df = DeviceFrame()
        for name, names in self._groups(col_selector):
            if not all(n in df for n in names):
                continue
            t = self._table(name)
            key = t.space.keys_for([df[n] for n in names]) if isinstance(t.space, ComboKeySpace) \
                else t.space.keys_for(df[names[0]])
            idx, dts, out_names = [], [], []
            for j, sn in enumerate(t.stat_names):
                if sn in new_df:
                    continue
                dt = getattr(t, "stat_dtypes", {}).get(sn, np.float64)
                for agg, d in AGG_DTYPES.items():
                    if sn.endswith(f"{self.name_sep}{agg}"):
                        dt = d
                idx.append(j); dts.append(dt); out_names.append(sn)
            if not idx:
                continue
            # an integer output is null where the key has no group (a key the fit never saw, or a null
            # key when the fit had none) or the statistic is NaN: the reference's left merge leaves
            # those rows missing, it must not read as 0
            masked = [np.dtype(d).kind != "f" for d in dts]
            outs = t.handle.gather_columns(key, idx, [float("nan")] * len(idx), dts, masked)
            for sn, o in zip(out_names, outs):
                new_df[sn] = o
        return new_df

    def _table(self, name) -> GroupTable:
        t = self.tables.get(name)
        if t is None:                       # a workflow reloaded from disk: read the stat file
            path = self.categories.get(self.storage_name.get(name, name))
            if path is None:
                raise KeyError(name)
            t = self.tables[name] = GroupTable.from_parquet(name, path, self.name_sep)
        return t

    def column_mapping(self, col_selector):
        column_mapping = {}
        for group in col_selector.grouped_names:
            if isinstance(group, (tuple, list)):
                name = _make_name(*group, sep=self.name_sep)
                group = [*group]
            else:
                name = group
                group = [group]
            for cont in self.cont_names.names:
                for stat in self.stats:
                    if stat == "count":
                        column_mapping[f"{name}_{stat}"] = [*group]
                    else:
                        column_mapping[f"{name}_{cont}_{stat}"] = [cont, *group]
            if not self.cont_names.names and "count" in self.stats:
                column_mapping[f"{name}_count"] = [*group]
        return column_mapping

    def _compute_dtype(self, col_schema, input_schema):
        new_schema = super()._compute_dtype(col_schema, input_schema)
        dtype = np.float64
        for agg, d in AGG_DTYPES.items():
            if new_schema.name.endswith(f"{self.name_sep}{agg}"):
                dtype = d
                break
        else:   # sum / min / max: from the dtype of the continuous column (the first source)
            stat = new_schema.name.rsplit(self.name_sep, 1)[-1]
            if stat in _TYPED_STATS:
                dtype = _kept_dtype(new_schema.dtype, stat) or dtype
        return new_schema.with_dtype(dtype, False, False)

    def export_tables(self, new_path) -> Dict[str, str]:
        """write every group table under new_path/categories WITHOUT re-pointing this op
        (Workflow.save); -> {group name: path}"""
        base = os.path.join(new_path, "categories")
        os.makedirs(base, exist_ok=True)
        out = {}
        for name in list(self.categories):
            t = self._table(name)
            p = os.path.join(base, f"cat_stats.{name}.parquet")
            t.frame().to_parquet(p)
            out[name] = p
        return out

    def set_storage_path(self, new_path, copy=False):
        for name, t in self.tables.items():
            if copy:
                self.categories[name] = t.write(os.path.join(new_path, "categories"))
        self.out_path = new_path

    def clear(self):
        self.categories = _StatPaths()
        self.tables = {}
        self.storage_name = {}


def fit_group_table(name, names, parts, cont, stats, sep="_") -> GroupTable:
    """_category_stats with agg columns (categorify.py:1543-1555) for one key group."""
    if len(names) > 1:
        space = ComboKeySpace.fit([[_leaf(df[n]) for n in names] for df in parts])
    else:
        space = KeySpace.for_columns([_leaf(df[names[0]]) for df in parts])
    agg = engine.HashAgg(len(cont))
    for df in parts:
        key = space.keys_for([df[n] for n in names]) if len(names) > 1 else space.keys_for(df[names[0]])
        agg.insert(key, [_leaf(df[c]) for c in cont])
    t = build_group_table(name, names, space, agg, cont, stats, sep)
    # sum / min / max in the dtype the reference's stat file holds (see _kept_dtype; join_groupby.py
    # :200-215 reads it back unchanged), decided by the column's dtype alone so that it matches the
    # output schema.  Rows without a value are nulls of the integer outputs (transform).
    t.stat_dtypes = {}
    for c in cont:
        src = str(_leaf(parts[0][c]).data.dtype).replace("torch.", "") if parts else None
        for a in _TYPED_STATS:
            dt = _kept_dtype(src, a)
            if dt is not None:
                t.stat_dtypes[_make_name(name, c, a, sep=sep)] = dt
    return t
