"""JoinExternal (reference nvtabular/ops/join_external.py:35-206): join every partition to an
external table,

    df.assign(__tmp__=arange(len(df))).merge(ext, left_on=on, right_on=on_ext, how=how)
      .sort_values("__tmp__").drop(columns="__tmp__").reset_index(drop=True)

on the GPU (csrc/join.cu, family K9) without the merge's sort: the ext table is ordered by key
once per operator (the K8 row-ordering primitives) and indexed by a device table key -> run of
ext rows; every partition is then one probe pass, and, unless the ext keys are unique and the
join is a left join, a scan, an output-balanced expand and a gather.  Left-join-on-unique-keys
(the MovieLens `movies` table) passes the left columns through untouched and gathers the ext
columns at the probed rows.

Rules the reference leaves to cuDF / pandas and this operator pins (tests/test_join_external_host.py):
- rows follow left-row order; the matches of one left row follow ext-table order;
- a null or NaN key matches a null or NaN ext key; -0.0 and +0.0 are one key;
- int keys of any width and float keys compare by value (float image of both sides); a string key
  against a numeric one raises ValueError, as pandas does;
- in a left join every ext column of an unmatched row is null (int columns stay int with a
  cleared validity bit; to_pandas makes them float64 / NaN as pandas does).  DEVIATION: list
  columns have no row validity in this engine (Column.from_arrow maps a null list row to an empty
  one), so the ext list column of an unmatched row is an EMPTY list, where pandas has NaN;
- a non-key ext column named like a selected left column raises ValueError (pandas would add
  _x / _y suffixes, and the reference's column_mapping would name a column that does not exist);
  with on == on_ext the key appears once with the left values, otherwise both key columns appear.

The ext table is loaded, deduplicated (drop_duplicates_ext: pandas drop_duplicates semantics, on
the host, once) and indexed on the first transform and kept on the device, whatever `cache` says.
Every rank of a torch.distributed job builds its own copy and runs no collective.  Workflow.save
raises for a workflow holding this operator, as the reference's serializer does.
"""
import os
from typing import Dict, List

import numpy as np
import torch

from .. import engine
from ..column import Column, DeviceFrame
from ..graph import ColumnSchema, ColumnSelector, Schema
from .base import Operator
from .groupby import _order_rows, _sort_fields
from .keyspace import ComboKeySpace, KeySpace, _float_to_key

# the reference's merlin.core.dispatch.ExtData members
EXT_KINDS = ("dataset", "arrow", "cudf", "pandas", "dask_cudf", "dask_pandas", "parquet", "csv")


def _as_list(x):
    if x is None:
        return None
    return [x] if isinstance(x, str) else list(x)


def _norm_kind(kind):
    name = getattr(kind, "name", kind)
    if isinstance(name, str) and name.lower() in EXT_KINDS:
        return name.lower()
    raise ValueError("kind_ext option not recognized.")


def _paths(src):
    if isinstance(src, (str, os.PathLike)):
        return [os.fspath(src)]
    if isinstance(src, (list, tuple)) and src and all(isinstance(s, (str, os.PathLike)) for s in src):
        return [os.fspath(s) for s in src]
    return None


def _files(paths, suffix):
    out = []
    for p in paths:
        if os.path.isdir(p):
            out += sorted(os.path.join(p, f) for f in os.listdir(p) if f.endswith(suffix))
        else:
            out.append(p)
    return out


def _detect(df_ext, kind_ext):
    """-> (source kind, normalised source): pandas | arrow | dataset | parquet | csv"""
    import pandas as pd
    import pyarrow as pa
    from ..dataset import Dataset
    if isinstance(df_ext, pd.DataFrame):
        return "pandas", df_ext
    if isinstance(df_ext, pa.Table):
        return "arrow", df_ext
    if isinstance(df_ext, Dataset):
        return "dataset", df_ext
    paths = _paths(df_ext)
    if paths is not None:
        if kind_ext == "csv" or (kind_ext is None and all(p.endswith(".csv") for p in paths)):
            return "csv", _files(paths, ".csv")
        return "parquet", paths
    raise ValueError(f"JoinExternal: df_ext of type {type(df_ext).__name__} is not supported; give a pandas "
                     "DataFrame, a pyarrow.Table, a Dataset, or parquet / CSV path(s)")


def _arrow_column_schema(name, t) -> ColumnSchema:
    """the engine column an arrow field becomes (Column.from_arrow's type rules)"""
    import pyarrow as pa
    is_list = pa.types.is_list(t) or pa.types.is_large_list(t)
    if is_list:
        t = t.value_type
    if pa.types.is_dictionary(t):
        t = t.value_type
    if pa.types.is_string(t) or pa.types.is_large_string(t):
        dt = np.dtype("object")
    elif pa.types.is_boolean(t):
        dt = np.dtype("bool")
    else:
        dt = np.dtype(t.to_pandas_dtype())
        if dt.kind in "iu" and dt not in (np.dtype("int32"), np.dtype("int64")):
            dt = np.dtype("int32" if dt.itemsize < 4 else "int64")
        elif dt.kind == "f" and dt.itemsize < 4:
            dt = np.dtype("float32")
    return ColumnSchema(name, dtype=dt, is_list=is_list, is_ragged=is_list)


def _join_kind(left: Column, ext: Column, lname: str, ename: str) -> str:
    if left.is_list or ext.is_list:
        raise ValueError(f"JoinExternal: the list column {lname if left.is_list else ename!r} cannot be a join key")
    if left.is_string != ext.is_string:
        raise ValueError(f"JoinExternal: cannot join the {'string' if left.is_string else 'numeric'} key {lname!r} "
                         f"with the {'string' if ext.is_string else 'numeric'} ext key {ename!r}")
    if left.is_string:
        return "str"
    if left.data.is_floating_point() or ext.data.is_floating_point():
        return "float"
    return "int"


def _image(col: Column, kind: str, space) -> Column:
    """the int32 / int64 key column both sides of one key component are compared by"""
    if kind == "str":
        return space.keys_for(col)
    if kind == "float":
        return _float_to_key(col)          # by value: never KeySpace.keys_for of a float column
    if col.data.dtype == torch.uint8:
        return Column(col.data.to(torch.int32), col.validity)
    return Column(col.data, col.validity)


class _Table:
    """the ext table of one key-kind combination on the device: its columns, the key mapping of
    each side and the K9 join handle"""

    def __init__(self, ext: DeviceFrame, on_ext: List[str], kinds):
        self.ext = ext
        self.kinds = kinds
        keys = [ext[c] for c in on_ext]
        self.spaces = [KeySpace.for_columns([k], sync=False) if kind == "str" else None
                       for k, kind in zip(keys, kinds)]
        self.combo = None
        imgs = [_image(k, kind, s) for k, kind, s in zip(keys, kinds, self.spaces)]
        if len(imgs) > 1:
            # int64 components: the ranked path of ComboKeySpace, never its direct two-int32 pack
            # (a left component of another width could not be packed alike)
            imgs = [Column(c.data.to(torch.int64), c.validity) for c in imgs]
            self.combo = ComboKeySpace.fit([imgs], ncomp=len(imgs), sync=False)
            key = self.combo.keys_for(imgs)
        else:
            key = imgs[0]
        self.join = self._build(key, len(ext))

    def left_key(self, cols: List[Column]) -> Column:
        imgs = [_image(c, kind, s) for c, kind, s in zip(cols, self.kinds, self.spaces)]
        if self.combo is None:
            return imgs[0]
        return self.combo.keys_for([Column(c.data.to(torch.int64), c.validity) for c in imgs])

    @staticmethod
    def _build(key: Column, n: int) -> engine.JoinTable:
        """ext rows ordered by key, stable, null keys last (K8), cut into one run per key"""
        dev = key.data.device
        if n == 0:
            z = torch.zeros(1, dtype=torch.int64, device=dev)
            return engine.JoinTable(z[:0], z, z[:0], 0, 0)
        stats = torch.empty((1, 3), dtype=torch.int64, device=dev)
        codes, valid = engine.gb_order_codes(key, stats[0])
        st = stats.cpu().numpy().view(np.uint64)
        fields = _sort_fields(codes, valid, st[0], n, True)
        if not fields:                                  # every ext key is null: one null run
            return engine.JoinTable(torch.empty(0, dtype=torch.int64, device=dev),
                                    torch.zeros(1, dtype=torch.int64, device=dev),
                                    torch.arange(n, dtype=torch.int64, device=dev), 0, n)
        order, r = _order_rows(fields, n, dev)
        off, g, kept = engine.gb_segments(order, r, [codes], valid)
        distinct = engine.gb_gather(Column(key.data, None), order, r, g, 1, off).data
        rows = order & ((1 << r) - 1)
        return engine.JoinTable(distinct, off, rows, kept, n)


class JoinExternal(Operator):
    """Join each partition to an external table (left or inner join), keeping left-row order.

    df_ext: a pandas DataFrame, a pyarrow.Table, a Dataset (its partitions are concatenated), a
    parquet file / directory / list of files, or a CSV path.  The table is replicated on every
    GPU (the reference's broadcast merge).  See the module docstring for the pinned rules and the
    one deviation (an unmatched ext list row is an empty list)."""

    def __init__(self, df_ext, on, how="left", on_ext=None, columns_ext=None, drop_duplicates_ext=None,
                 kind_ext=None, cache="host", **kwargs):
        super().__init__()
        if how not in ("left", "inner"):
            raise ValueError("Only left join is currently supported.")
        self.kind_ext = _norm_kind(kind_ext) if kind_ext is not None else None
        self._source_kind, self._source = _detect(df_ext, self.kind_ext)
        if self.kind_ext is None:
            self.kind_ext = self._source_kind
        self.df_ext = df_ext
        self.on = _as_list(on)
        self.on_ext = _as_list(on_ext) or list(self.on)
        if not self.on or len(self.on) != len(self.on_ext):
            raise ValueError(f"JoinExternal: on {self.on} and on_ext {self.on_ext} must name as many columns")
        self.how = how
        self.columns_ext = list(columns_ext) if columns_ext else None
        self.drop_duplicates_ext = drop_duplicates_ext
        self.cache = cache
        self.kwargs = kwargs
        self._schema = None
        self._frame = None
        self._tables: Dict[tuple, _Table] = {}

    # ---------------------------------------------------------------- ext table metadata
    @property
    def ext_schema(self) -> Schema:
        """the ext columns (after columns_ext) from the table's metadata: no data is loaded for a
        frame, a table or a parquet file"""
        if self._schema is None:
            import pyarrow as pa
            kind, src = self._source_kind, self._source
            if kind == "dataset":
                full = src.schema
            else:
                if kind == "pandas":
                    sch = pa.Schema.from_pandas(src, preserve_index=False)
                elif kind == "arrow":
                    sch = src.schema
                elif kind == "parquet":
                    import pyarrow.parquet as pq
                    sch = pq.read_schema(_files(src, ".parquet")[0])
                else:
                    import pyarrow.csv as pcsv
                    with pcsv.open_csv(src[0]) as reader:
                        sch = reader.schema
                full = Schema([_arrow_column_schema(f.name, f.type) for f in sch])
            names = self.columns_ext if self.columns_ext else full.column_names
            missing = [c for c in names if c not in full]
            if missing:
                raise ValueError(f"JoinExternal: columns {missing} are not in the external table")
            self._schema = Schema([full[c] for c in names])
        return self._schema

    def _ext_names(self) -> List[str]:
        return self.ext_schema.column_names

    def _check(self, names: List[str]):
        ext = self._ext_names()
        missing = [o for o in self.on if o not in names]
        if missing:
            raise ValueError(f"JoinExternal: the join keys {missing} are not among the selected columns {names}")
        missing = [o for o in self.on_ext if o not in ext]
        if missing:
            raise ValueError(f"JoinExternal: the ext join keys {missing} are not among the ext columns {ext}")
        shared = {o for o, e in zip(self.on, self.on_ext) if o == e}
        clash = [c for c in ext if c in names and c not in shared]
        if clash:
            raise ValueError(f"JoinExternal: the ext columns {clash} have the names of selected columns; "
                             "rename them (columns_ext) or drop them from the selection")

    # ----------------------------------------------------------------------- graph hooks
    def column_mapping(self, col_selector: ColumnSelector):
        names = list(dict.fromkeys(list(col_selector.names) + self._ext_names()))
        return {n: [n] for n in names}

    def compute_output_schema(self, input_schema: Schema, col_selector: ColumnSelector) -> Schema:
        # left columns keep their dtype, ext columns take the ext table's; no tags or properties
        # (reference join_external.py:195-206)
        ext = self.ext_schema
        out = []
        for name in self.column_mapping(col_selector):
            src = input_schema[name] if name in col_selector.names and name in input_schema else \
                (ext[name] if name in ext else ColumnSchema(name))
            out.append(ColumnSchema(name, dtype=src.dtype, is_list=src.is_list, is_ragged=src.is_ragged))
        return Schema(out)

    # ------------------------------------------------------------------------ ext table
    def _load_frame(self, device) -> DeviceFrame:
        """the ext table on the device, loaded once: columns_ext, then drop_duplicates_ext"""
        if self._frame is None:
            import pyarrow as pa
            kind, src = self._source_kind, self._source
            if kind == "pandas":
                tab = pa.Table.from_pandas(src, preserve_index=False)
            elif kind == "arrow":
                tab = src
            elif kind == "csv":
                import pyarrow.csv as pcsv
                tab = pa.concat_tables([pcsv.read_csv(p) for p in src], promote_options="default")
            else:
                from ..dataset import Dataset
                ds = src if kind == "dataset" else Dataset(_files(src, ".parquet"))
                parts = [p.to_arrow() for p in ds.partitions()]
                tab = pa.concat_tables(parts, promote_options="default") if parts else \
                    pa.schema([]).empty_table()
            tab = tab.select(self._ext_names())
            if self.drop_duplicates_ext:
                # pandas drop_duplicates(ignore_index=True): first occurrence kept, NaN == NaN, and
                # a list column raises TypeError (unhashable)
                dup = tab.to_pandas().duplicated().to_numpy()
                tab = tab.filter(pa.array(~dup))
            self._frame = DeviceFrame.from_arrow(tab, device)
        return self._frame

    def _table(self, left_keys: List[Column], device) -> _Table:
        ext = self._load_frame(device)
        kinds = tuple(_join_kind(c, ext[e], o, e) for c, o, e in zip(left_keys, self.on, self.on_ext))
        t = self._tables.get(kinds)
        if t is None:
            t = self._tables[kinds] = _Table(ext, self.on_ext, kinds)
        return t

    # ------------------------------------------------------------------------- transform
    def transform(self, col_selector: ColumnSelector, df: DeviceFrame) -> DeviceFrame:
        names = list(col_selector.names)
        self._check(names)
        left = {n: self._get(df, n) for n in names}
        dev = next(iter(left.values())).data.device
        t = self._table([left[o] for o in self.on], dev)
        if len(t.ext) >= (1 << 31):
            raise ValueError(f"JoinExternal: an external table of {len(t.ext)} rows; at most 2^31 - 1")
        key = t.left_key([left[o] for o in self.on])
        ext_names = [c for c in self._ext_names() if c not in left]
        ext_cols = {c: t.ext[c] for c in ext_names}
        if self.how == "left" and t.join.max_group <= 1:
            # unique ext keys: exactly one output row per left row, in order
            ext_rows, _, _ = t.join.probe(key, "left", scan=False)
            out = dict(left)
            out.update(engine.take_rows(ext_cols, ext_rows, masked=True))
        else:
            first, off, n_out = t.join.probe(key, self.how, scan=True)
            left_rows, ext_rows = t.join.expand(first, off, n_out)
            out = engine.take_rows(left, left_rows)
            out.update(engine.take_rows(ext_cols, ext_rows, masked=self.how == "left"))
        return DeviceFrame({n: out[n] for n in self.column_mapping(col_selector)})

