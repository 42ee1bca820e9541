"""Categorify (reference nvtabular/ops/categorify.py:58-613, helpers to :1897).

Same constructor, label space, artefacts and error behaviour as the reference;
everything underneath is different (SURVEY.md §8a A1-A14):

  fit        per partition, every column group is folded into a resident
             device hash table (K3, engine.HashAgg) — no per-partition
             groupby frames, no tree of concat+groupby, no host spill;
             across GPUs the partial tables are exchanged by key-hash owner
             (all-to-all), merged, all-gathered, and every rank builds the
             identical vocabulary (K4: (size desc, key asc) ordering,
             freq_threshold / max_size cut) and lookup table (K5).
  transform  one in-order probe pass per column (K5) — no merge, no sort back.
"""
import os
import warnings
from copy import deepcopy
from typing import Dict, List, Optional

import numpy as np
import pandas as pd
import torch

from .. import engine
from ..column import Column, DeviceFrame
from ..graph import ColumnSelector, Tags
from .base import StatOperator
from .hash_bucket import emb_sz_rule
from .keyspace import ComboKeySpace, KeySpace, _leaf

PAD_OFFSET, NULL_OFFSET, OOV_OFFSET = 0, 1, 2   # categorify.py:51-55
EAGER_ARTIFACT_ROWS = 1 << 20                   # larger vocabularies are written lazily
WRITER_THREADS = 4                              # library threads writing the artefact files of a fit


def _artifacts_mode() -> str:
    """NVTB_ARTIFACTS = eager (default) | lazy.

    eager  every meta.<col>.parquet and the unique.<col>.parquet of every vocabulary up to
           2^20 keys is written DURING fit, like the reference (whose only fitted state IS those
           files).  The small vocabularies are built first; library threads
           (engine.ArtifactWriter) copy their keys / sizes to the host and write the files while
           the GPU goes on with the builds of the large columns, and fit_finalize joins those
           threads before it returns.
           Larger vocabulary files are written when their path is first read
           (`op.categories[name]`, `Workflow.save`, `set_storage_path`).
    lazy   nothing until a path is read."""
    m = os.environ.get("NVTB_ARTIFACTS", "eager").lower()
    return "eager" if m == "sync" else m


def _artifacts_lazy() -> bool:
    return _artifacts_mode() == "lazy"


def _pandas_meta(columns, index_start, n):
    """the b"pandas" schema metadata pandas.DataFrame.to_parquet would write for a frame with
    these (name, numpy dtype | "object") columns and RangeIndex(index_start, index_start + n)"""
    import json
    import pyarrow as pa
    cols = []
    for name, dt in columns:
        if dt == "object":
            cols.append({"name": name, "field_name": name, "pandas_type": "unicode", "numpy_type": "object",
                         "metadata": None})
        else:
            cols.append({"name": name, "field_name": name, "pandas_type": str(np.dtype(dt)),
                         "numpy_type": str(np.dtype(dt)), "metadata": None})
    return json.dumps({
        "index_columns": [{"kind": "range", "name": None, "start": int(index_start), "stop": int(index_start + n),
                           "step": 1}],
        "column_indexes": [{"name": None, "field_name": None, "pandas_type": "unicode", "numpy_type": "object",
                            "metadata": {"encoding": "UTF-8"}}],
        "columns": cols, "attributes": {}, "creator": {"library": "pyarrow", "version": pa.__version__},
        "pandas_version": pd.__version__}).encode()


def _pandas_meta_parts(columns, index_start):
    """_pandas_meta cut around the stop of the RangeIndex -> (head, tail), for a writer that only
    learns the row count later: the metadata is head + str(index_start + n) + tail"""
    text = _pandas_meta(columns, index_start, 0)
    stop = b'"stop": %d' % int(index_start)
    head, tail = text.split(stop)           # column names are escaped: they cannot hold this
    return head + b'"stop": ', tail


def _write_numeric_parquet(path, arrays, index_start):
    """{name: numpy array} -> parquet that pandas reads back as a frame with
    RangeIndex(index_start, ...): what df.to_parquet(compression=None) writes, minus the pandas
    conversion and the dictionary pages.  Written by the library (engine.parquet_write)."""
    n = len(next(iter(arrays.values()))) if arrays else 0
    engine.parquet_write(path, list(arrays.items()),
                         _pandas_meta([(k, v.dtype) for k, v in arrays.items()], index_start, n))


def _make_name(*args, sep="_"):
    return sep.join(args)


def _resolve(opt, name, default=None):
    if isinstance(opt, dict):
        return opt.get(name, default)
    return opt if opt is not None else default


class FittedVocab:
    """What the reference keeps as `unique.<name>.parquet` + `meta.<name>.parquet`
    (categorify.py:719-822): device lookup handle + host metadata; the parquet
    files are (re)written from it."""

    def __init__(self, name, key_names, space, vocab: engine.Vocab, num_buckets=None,
                 has_sizes=True, index_start=None):
        self.name = name
        self.key_names = list(key_names)      # column names inside the parquet file
        self.space = space                    # KeySpace | ComboKeySpace
        self.vocab = vocab
        self.num_buckets = num_buckets
        self.has_sizes = has_sizes
        oov_count = num_buckets or 1
        self.index_start = OOV_OFFSET + oov_count if index_start is None else index_start
        self.path = None
        self._written = False
        self._queued = None        # (base_path, force) of files queued on an ArtifactWriter

    @property
    def n_kept(self):
        return self.vocab.n_kept

    @property
    def file_rows(self):
        """rows of unique.<name>.parquet (an empty input writes one null row)"""
        return 1 if self.vocab.n_total == 0 else self.vocab.n_kept

    def _host_arrays(self):
        keys, sizes = self.vocab.export(with_sizes=self.has_sizes)
        return keys.cpu().numpy(), (sizes.cpu().numpy() if sizes is not None else None)

    def unique_frame(self) -> pd.DataFrame:
        k, sz = self._host_arrays()
        if isinstance(self.space, ComboKeySpace):
            comps = self.space.decode(k)
            data = {n: pd.Series(v, dtype=object) for n, v in zip(self.key_names, comps)}
        else:
            data = {self.key_names[0]: self.space.decode(k)}
        df = pd.DataFrame(data)
        if self.has_sizes:
            df[f"{self.name}_size"] = sz
        df.index = pd.RangeIndex(self.index_start, self.index_start + len(df))
        return df

    def _meta_columns(self):
        """(name, dtype) of meta.<name>.parquet (categorify.py:801-822: kind = pad, null, oov,
        unique; offset = PAD_OFFSET, NULL_OFFSET, OOV_OFFSET, first label; num_indices
        [; num_observed]), for its pandas metadata"""
        cols = [("kind", "object"), ("offset", np.int64), ("num_indices", np.int64)]
        return cols + ([("num_observed", np.int64)] if self.has_sizes else [])

    def _paths(self, base_path):
        return ("/".join([str(base_path), f"meta.{self.name}.parquet"]),
                "/".join([str(base_path), f"unique.{self.name}.parquet"]))

    @property
    def native_files(self) -> bool:
        """int and float key spaces: both files are written by the library (engine.ArtifactWriter)"""
        return isinstance(self.space, KeySpace) and self.space.kind in ("int", "float")

    def write(self, base_path, force=False, writer=None):
        """categorify.py:731-822: unique.<name>.parquet (index = label) + meta.<name>.parquet.
        With `writer` (an engine.ArtifactWriter) the files of an int / float key space are only
        queued; finish_write() completes them after writer.join()."""
        self.path = "/".join([str(base_path), f"unique.{self.name}.parquet"])
        if not force and _artifacts_lazy():
            self._written = False
            return self.path
        os.makedirs(base_path, exist_ok=True)
        if writer is not None and self.native_files:
            self._submit(writer, base_path, force)
        else:
            self._write_now(base_path, force)
        return self.path

    def _submit(self, writer, base_path, force):
        """queue meta + unique files on the library's writer threads: no wait for the device here"""
        meta_path, upath = self._paths(base_path)
        key = self.key_names[0]
        key_dtype = np.dtype(self.space.np_dtype or (np.int64 if self.space.kind == "int" else np.float64))
        size_name = f"{self.name}_size" if self.has_sizes else None
        head, tail = _pandas_meta_parts([(key, key_dtype)] + ([(size_name, np.int64)] if size_name else []),
                                        self.index_start)
        writer.submit_vocab(self.vocab, meta_path, _pandas_meta(self._meta_columns(), 0, 4), upath,
                            -1 if force else EAGER_ARTIFACT_ROWS, key, key_dtype, size_name, self.index_start,
                            self.num_buckets or 1, head, tail)
        self._queued = (base_path, force)

    def finish_write(self):
        """after the ArtifactWriter of a write(..., writer=) joined: the file the library leaves to
        pandas (an empty input's single null row) and the written flag"""
        if self._queued is None:
            return
        base_path, force = self._queued
        self._queued = None
        if force or self.vocab.n_kept <= EAGER_ARTIFACT_ROWS:
            _, upath = self._paths(base_path)
            if self.vocab.n_total == 0:
                self._empty_unique_frame().to_parquet(upath, compression=None)
            if self.path is None or os.path.abspath(upath) == os.path.abspath(self.path):
                self._written = True

    def _empty_unique_frame(self):
        """categorify.py:1318-1324: empty input -> a single null row"""
        return pd.DataFrame({n: pd.Series([None], dtype=object) for n in self.key_names})

    def _write_now(self, base_path, force):
        if self.native_files:
            writer = engine.ArtifactWriter(1)
            try:
                self._submit(writer, base_path, force)
            finally:
                writer.join()
            self.finish_write()
            return
        # string and combination key spaces: the meta file from the library, the vocabulary from pandas
        meta_path, upath = self._paths(base_path)
        v = self.vocab
        engine.parquet_write_meta(meta_path, self.num_buckets or 1, v.n_kept, v.null_size, v.oov_size, v.unique_size,
                                  self.has_sizes, _pandas_meta(self._meta_columns(), 0, 4))
        if force or self.vocab.n_kept <= EAGER_ARTIFACT_ROWS:
            df = self._empty_unique_frame() if self.vocab.n_total == 0 else self.unique_frame()
            df.to_parquet(upath, compression=None)
            if self.path is None or os.path.abspath(upath) == os.path.abspath(self.path):
                self._written = True

    def wait(self):
        """kept for callers of the earlier threaded writer: writes are complete when write()
        returns, or, with a writer, after its join() and finish_write()"""
        return None

    def ensure_written(self):
        if self.path is not None and not self._written:
            self.write(os.path.dirname(self.path), force=True)


class _Categories(dict):
    """storage name -> parquet path, like the reference's `Categorify.categories`.
    Reading a path makes sure a lazily written (very large) vocabulary file exists."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.fitted: Dict[str, FittedVocab] = {}

    def __getitem__(self, key):
        fv = self.fitted.get(key)
        if fv is not None:
            fv.ensure_written()
        return super().__getitem__(key)


class Categorify(StatOperator):
    def __init__(self, freq_threshold=0, out_path=None, cat_cache="host", dtype=None, on_host=True,
                 encode_type="joint", name_sep="_", search_sorted=False, num_buckets=None, vocabs=None,
                 max_size=0, single_table=False, cardinality_memory_limit=None, tree_width=None,
                 split_out=1, split_every=8, **kwargs):
        # categorify.py:226-241
        if "start_index" in kwargs:
            raise ValueError(
                "start_index is now deprecated. `Categorify` will always reserve index `0` for "
                "user-specific purposes, and will use index `1` for null values.")
        if "na_sentinel" in kwargs:
            raise ValueError(
                "na_sentinel is now deprecated. `Categorify` will always reserve index `1` for null "
                "values, and the following `num_buckets` indices for out-of-vocabulary values "
                "(or just index `2` if `num_buckets is None`).")
        if kwargs:
            raise ValueError(f"Unrecognized key-word arguments: {kwargs}")
        if num_buckets and not (max_size or freq_threshold):   # :246-251
            warnings.warn(
                "You are setting num_buckets without using max_size or freq_threshold to restrict "
                "the number of distinct categories. Are you sure this is what you want?")
        self.name_sep = name_sep
        self.storage_name = {}
        if encode_type not in ("joint", "combo"):               # :287-290
            raise ValueError(f"encode_type={encode_type} not supported.")
        if encode_type == "combo" and vocabs is not None:
            raise ValueError("Passing in vocabs is not supported with a combo encoding.")
        super().__init__()
        self.single_table = single_table
        self.freq_threshold = freq_threshold or 0
        self.out_path = out_path or "./"
        self.dtype = dtype
        self.on_host = on_host            # accepted, meaningless here: nothing spills to host
        self.cat_cache = cat_cache        # accepted: the lookup table always lives in HBM
        self.encode_type = encode_type
        self.search_sorted = search_sorted
        self.cardinality_memory_limit = cardinality_memory_limit
        self.split_every = split_every    # accepted: there is no reduction tree
        self.split_out = split_out        # accepted: sharding is by key-hash owner across GPUs
        if tree_width is not None:        # :1900-1907
            warnings.warn("The tree_width argument is now deprecated, and will be ignored. "
                          "Please use split_out and split_every.", FutureWarning)
        if self.search_sorted and self.freq_threshold:           # :307-310
            raise ValueError("cannot use search_sorted=True with anything else than the default freq_threshold")
        if num_buckets == 0:                                     # :311-322
            raise ValueError("For hashing num_buckets should be an int > 1, otherwise set num_buckets=None.")
        elif isinstance(num_buckets, dict) or isinstance(num_buckets, int) or num_buckets is None:
            self.num_buckets = num_buckets
        else:
            raise ValueError(f"`num_buckets` must be dict or int, got type {type(num_buckets)}")
        if isinstance(max_size, dict) or isinstance(max_size, int) or max_size is None:
            self.max_size = max_size
        else:
            raise ValueError(f"max_size must be dict or int, got type {type(max_size)}")
        if freq_threshold and max_size:                          # :329-330
            raise ValueError("cannot use freq_threshold param together with max_size param")
        if self.num_buckets is not None:                         # :332-338
            warnings.warn("Performing a hash-based transformation. Do not expect Categorify to be "
                          "consistent on GPU and CPU with this num_buckets setting!")
        self._user_vocabs = vocabs
        self._aggs = {}      # storage name -> engine.HashAgg, reused (reset) across fits
        self._rows_seen = {}
        self._rows_bound_global = 0
        self._owner_pool = []   # per-column owner tables of the cross-GPU merge, reused across fits
        self.vocabs = {}
        self.categories = _Categories()
        if vocabs is not None:
            self._check_vocabs(vocabs)

    # ------------------------------------------------------------------ vocabs=
    def _check_vocabs(self, vocabs):
        ok_series = isinstance(vocabs, dict) and all(isinstance(v, pd.Series) for v in vocabs.values())
        ok_paths = isinstance(vocabs, dict) and all(isinstance(v, str) for v in vocabs.values())
        if not (ok_series or ok_paths):
            raise ValueError("Unrecognized vocab type, please provide either a dictionary with paths "
                             "to parquet files or a dictionary with pandas Series objects.")

    def _nb(self, name):
        nb = _resolve(self.num_buckets, name)
        return nb or None

    def _vocab_from_values(self, col_name, values: pd.Series, sizes=None, index_start=None) -> FittedVocab:
        """process_vocabs (categorify.py:421-454): labels are 2 + B + position after dropna()."""
        values = values.dropna().reset_index(drop=True)
        if values.dtype == object or str(values.dtype) in ("str", "string"):
            space = KeySpace("str", np.array(sorted(set(values.tolist())), dtype=object))
        elif np.issubdtype(values.dtype, np.floating):
            space = KeySpace("float", None, values.dtype)
        else:
            space = KeySpace("int", None, np.dtype("int64") if values.dtype.itemsize == 8 else np.dtype("int32"))
        keys = torch.from_numpy(space.encode_values(values).astype(np.int64)).cuda()
        szt = torch.from_numpy(np.array(sizes, dtype=np.int64, copy=True)).cuda() if sizes is not None else None
        vocab = engine.Vocab.from_arrays(keys, szt)
        return FittedVocab(col_name, [col_name], space, vocab, self._nb(col_name),
                           has_sizes=sizes is not None, index_start=index_start)

    def _load_user_vocabs(self):
        if not self._user_vocabs or self.vocabs:
            return
        base = os.path.join(self.out_path, "categories")
        for col, v in self._user_vocabs.items():
            name = _make_name(*col, sep=self.name_sep) if isinstance(col, tuple) else col
            if isinstance(v, str):
                fv = self._vocab_from_parquet(name, v)
                fv.path, fv._written = v, True
            else:
                fv = self._vocab_from_values(name, v)
                fv.write(base, force=True)
            self.vocabs[name] = fv
        for name, fv in self.vocabs.items():
            self.categories[name] = fv.path
            self.categories.fitted[name] = fv

    def _vocab_from_parquet(self, name, path) -> FittedVocab:
        """A vocabulary file (this engine's or the reference's, categorify.py:731-822) -> device
        lookup.  Multi-column files (encode_type="combo") rebuild the combination key space
        from all of their key columns."""
        df = pd.read_parquet(path)
        size_col = f"{name}_size"
        key_cols = [c for c in df.columns if c != size_col]
        start = int(df.index[0]) if len(df) and isinstance(df.index, pd.RangeIndex) else None
        if len(key_cols) == 1:
            keep = ~df[key_cols[0]].isna()
            sizes = df[size_col] if size_col in df.columns else None
            fv = self._vocab_from_values(name, df[key_cols[0]][keep], sizes[keep] if sizes is not None else None,
                                         index_start=start)
            fv.key_names = [key_cols[0]]
            return fv
        from ._tables import keys_from_frame
        space, keys, isnull = keys_from_frame(df, key_cols)
        keep = ~isnull
        szt = None
        if size_col in df.columns:
            szt = torch.from_numpy(df[size_col].to_numpy(dtype=np.int64)).to(keys.device)[keep]
        vocab = engine.Vocab.from_arrays(keys[keep].contiguous(), szt)
        return FittedVocab(name, key_cols, space, vocab, self._nb(name), has_sizes=szt is not None,
                           index_start=start)

    # ----------------------------------------------------------------------- fit
    def _groups(self, col_selector: ColumnSelector):
        """[(storage name, [column names])] for every column group to fit."""
        out = []
        for g in col_selector.grouped_names:
            names = list(g) if isinstance(g, tuple) else [g]
            out.append((_make_name(*names, sep=self.name_sep), names))
        return out

    def fit(self, col_selector: ColumnSelector, ddf):
        # categorify.py:350-357
        columns_all = col_selector.names
        if len(columns_all) != len(set(columns_all)) and self.encode_type == "joint":
            raise ValueError("Same column name included in multiple groups.")
        for group in col_selector.subgroups:
            if len(group.names) > 1:
                name = _make_name(*group.names, sep=self.name_sep)
                for col in group.names:
                    self.storage_name[col] = name
        self._load_user_vocabs()
        groups = [(s, n) for s, n in self._groups(col_selector) if s not in self.vocabs]
        if not groups:
            return {}
        it = iter(ddf)
        first = next(it, None)
        # Every rank must issue the SAME sequence of collectives, so the path is agreed on
        # first: a rank whose shard is empty (or whose first partition is not streamable while
        # the others' are) follows the majority instead of picking a path from local data.
        from ..dist import all_gather_object, world
        mode = "empty" if first is None else ("stream" if self._streamable(first, groups) else "general")
        wide = {}
        if first is not None and mode == "stream":
            wide = {storage: any(_leaf(first[n]).data.dtype == torch.int64 for n in names)
                    for storage, names in groups}
        if world()[0] > 1:
            seen = all_gather_object((mode, wide))
            live = [m for m, _ in seen if m != "empty"]
            mode = "empty" if not live else ("stream" if all(m == "stream" for m in live) else "general")
            wide = {storage: any(w.get(storage, False) for _, w in seen) for storage, _ in groups}
        if mode == "empty":
            return {storage: self._fit_group(storage, names, []) for storage, names in groups}
        if mode == "stream":
            # numeric keys: ONE streaming pass — partition i is folded into the tables while
            # partition i+1 is still being uploaded (Dataset.partitions prefetches one ahead)
            state = {storage: self._open_group(storage, names, first, wide.get(storage, False))
                     for storage, names in groups}
            part = first
            while part is not None:
                for storage, names in groups:
                    space, agg = state[storage]
                    for n in names:
                        self._insert(storage, agg, space.keys_for(part[n]))
                part = next(it, None)
            for storage, _ in groups:                       # staged batches of the sorted accumulators
                flush = getattr(state[storage][1], "flush", None)
                if flush is not None:
                    flush()
            if world()[0] == 1:
                # single GPU: every vocabulary is built straight from its handle — the small ones
                # first, so that their artefact files can be written (fit_finalize) while the
                # builds of the sorted accumulators (large) still run
                return self._close_in_order(groups, state, {storage: "direct" for storage, _ in groups})
            from ..dist import global_merge_many, global_merge_sorted
            self._rows_bound_global = _global_rows(max(self._rows_seen.values(), default=0))
            # a column that ANY rank accumulated as a sorted array of packed pairs (high
            # cardinality, csrc/sortagg.cuh) takes the key-range exchange on every rank; the
            # others travel together through the key-hash owner exchange
            aggs = [state[storage][1] for storage, _ in groups]
            modes = [getattr(a, "mode", 0) for a in aggs]
            seen = all_gather_object(modes)
            use_sorted = [any(m[i] == 1 for m in seen) and not wide.get(groups[i][0], False)
                          and self._rows_bound_global < 0xFFFFFFF0 for i in range(len(groups))]
            for a, srt in zip(aggs, use_sorted):
                if srt:
                    a.to_sorted()
            hashed = [i for i, srt in enumerate(use_sorted) if not srt]
            ranged = [i for i, srt in enumerate(use_sorted) if srt]
            merged = [None] * len(groups)
            for i, m in zip(hashed, global_merge_many([aggs[i] for i in hashed], owner_pool=self._owner_pool)
                            if hashed else []):
                merged[i] = m
            for i, m in zip(ranged, global_merge_sorted([aggs[i] for i in ranged])):
                merged[i] = ("pairs",) + tuple(m)
            return self._close_in_order(groups, state, {storage: m for (storage, _), m in zip(groups, merged)})
        parts = ([first] if first is not None else []) + list(it)   # strings / general combos: dictionary pre-pass
        fitted = {}
        for storage, names in groups:
            fitted[storage] = self._fit_group(storage, names, parts)
        return fitted

    def _close_in_order(self, groups, state, merged):
        def large(storage):
            m = merged[storage]
            return getattr(state[storage][1], "mode", 0) == 1 or (isinstance(m, tuple) and m and m[0] == "pairs")
        fitted = {}
        small = [g for g in groups if not large(g[0])]
        for storage, _ in small:
            fitted[storage] = self._close_group(storage, [storage], state[storage][0], state[storage][1], merged[storage])
        for storage, _ in groups:
            if storage not in fitted:
                fitted[storage] = self._close_group(storage, [storage], state[storage][0], state[storage][1],
                                                    merged[storage])
        return {storage: fitted[storage] for storage, _ in groups}

    def _streamable(self, df, groups) -> bool:
        for _, names in groups:
            if self.encode_type == "combo" and len(names) > 1:
                return False
            if any(df[n].is_string for n in names):
                return False
        return True

    def _get_agg(self, storage):
        agg = self._aggs.get(storage)
        if agg is None:
            agg = self._aggs[storage] = engine.HashAgg(0)
        else:
            agg.reset()
        self._rows_seen[storage] = 0
        return agg

    def _insert(self, storage, agg, key):
        agg.insert(key)
        self._rows_seen[storage] += key.data.numel()

    def _size_bound(self, storage) -> int:
        """upper bound on any group's size (speed hint for the radix sort); unknown across GPUs"""
        from ..dist import world
        if world()[0] == 1:
            return self._rows_seen.get(storage, 0)
        return self._rows_bound_global            # 0 = unknown

    def _open_group(self, storage, names, df, wide=False):
        """streaming path: numeric keys only; `wide` (agreed across ranks) = some rank holds int64"""
        if df is None:
            space = KeySpace("int", None, np.dtype("int64") if wide else np.dtype("int32"))
        else:
            space = KeySpace.for_columns([_leaf(df[n]) for n in names], sync=False)
            if space.kind == "int" and wide:
                space.np_dtype = np.dtype("int64")
        return space, self._get_agg(storage)

    def _close_group(self, storage, key_names, space, agg, merged=None) -> FittedVocab:
        direct = isinstance(merged, str)
        pairs = isinstance(merged, tuple) and len(merged) == 3 and isinstance(merged[0], str)
        if pairs:
            _, ordered_pairs, null_size = merged
        elif not direct:
            keys, sizes, null_size = merged if merged is not None else _global_unique_merge(agg)
        ft = _resolve(self.freq_threshold, storage, 0) or 0
        ms = _resolve(self.max_size, storage, 0) or 0
        nb = self._nb(storage)
        try:
            key_bits = 32 if isinstance(space, KeySpace) and (space.kind == "str" or (
                space.kind == "int" and space.np_dtype == np.dtype("int32"))) else 0
            if direct:
                vocab = engine.Vocab.build_from_agg(agg, ft, ms, nb or 0, key_bits, self._size_bound(storage))
            elif pairs:
                vocab = engine.Vocab.build_from_pairs(ordered_pairs, null_size, ft, ms, nb or 0)
            else:
                vocab = engine.Vocab.build(keys, sizes, null_size, ft, ms, nb or 0, key_bits,
                                           self._size_bound(storage))
        except Exception as e:
            if "max_size" in str(e):     # categorify.py:1206-1211
                raise ValueError(
                    "`max_size` can never be less than the maximum of `num_buckets + 2` and `3`, because "
                    "we must always reserve pad, null and at least 1 oov-bucket index.") from e
            raise
        limit = self.cardinality_memory_limit
        if limit:
            limit = _parse_bytes(limit)
            nbytes = vocab.n_total * 16
            if nbytes > limit:           # categorify.py:1285-1294
                warnings.warn(f"Category DataFrame (with columns: {key_names}) is {nbytes} bytes in size. "
                              f"This is large compared to the suggested upper limit of {limit} bytes!"
                              f"(12.5% of the total memory by default)")
        return FittedVocab(storage, key_names, space, vocab, nb)

    def _fit_group(self, storage, names, parts) -> FittedVocab:
        combo = self.encode_type == "combo" and len(names) > 1
        if combo:
            comp_parts = [[_leaf(df[n]) for n in names] for df in parts]
            if any(c.is_list for df in parts for c in (df[n] for n in names)):
                raise ValueError("Can't categorical encode multiple list columns")
            space = ComboKeySpace.fit(comp_parts, ncomp=len(names))
            key_names = names
        else:
            cols_all = [df[n] for df in parts for n in names]
            space = KeySpace.for_columns([_leaf(c) for c in cols_all])
            key_names = [storage]
        agg = self._get_agg(storage)
        for df in parts:
            if combo:
                self._insert(storage, agg, space.keys_for([df[n] for n in names]))
            else:
                for n in names:          # joint encoding: every column feeds the SAME table
                    self._insert(storage, agg, space.keys_for(df[n]))
        merged = _global_unique_merge(agg)
        self._rows_bound_global = _global_rows(self._rows_seen.get(storage, 0))
        return self._close_group(storage, key_names, space, agg, merged)

    def fit_finalize(self, categories):
        base = os.path.join(self.out_path, "categories")
        idx_count = 0
        merged = dict(self.vocabs)
        merged.update(categories)
        # the int / float vocabularies' files are written by library threads, each as soon as its
        # vocabulary is built; they are all joined here, so every eager file exists on return
        writer = None
        if not _artifacts_lazy() and any(fv.native_files for fv in merged.values()):
            writer = engine.ArtifactWriter(WRITER_THREADS)
        try:
            for name, fv in merged.items():
                if self.single_table:                      # categorify.py:410-415, 1884-1897
                    fv.index_start = fv.index_start + idx_count
                    idx_count += fv.file_rows
                    fv._written = False
                if name in categories or self.single_table:
                    fv.write(base, writer=writer)
                self.categories[name] = fv.path
                self.categories.fitted[name] = fv
        finally:
            if writer is not None:
                writer.join()
        for fv in merged.values():
            fv.finish_write()

    def clear(self):
        self.categories = _Categories()
        for name, fv in self.vocabs.items():
            self.categories[name] = fv.path
            self.categories.fitted[name] = fv

    def export_artifacts(self, new_path) -> Dict[str, str]:
        """write unique.<name>.parquet / meta.<name>.parquet of every vocabulary under
        new_path/categories WITHOUT re-pointing this op (Workflow.save); -> {storage name: path}"""
        base = os.path.join(new_path, "categories")
        os.makedirs(base, exist_ok=True)
        out = {}
        for name in list(self.categories):
            fv = self._fitted(name)
            fv._write_now(base, True)
            out[name] = "/".join([base, f"unique.{fv.name}.parquet"])
        return out

    def set_storage_path(self, new_path, copy=False):
        for name, fv in self.categories.fitted.items():
            if copy:
                fv.write(os.path.join(new_path, "categories"), force=True)
            else:
                fv.path = fv.path.replace(str(self.out_path), str(new_path))
            dict.__setitem__(self.categories, name, fv.path)
        self.out_path = new_path

    # ----------------------------------------------------------------- transform
    def _fitted(self, storage) -> FittedVocab:
        fv = self.categories.fitted.get(storage)
        if fv is None:
            path = dict.get(self.categories, storage)
            if path is None:
                raise KeyError(storage)
            fv = self._vocab_from_parquet(storage, path)    # a workflow reloaded from disk
            fv.path, fv._written = path, True
            self.categories.fitted[storage] = fv
        return fv

    def transform(self, col_selector: ColumnSelector, df: DeviceFrame) -> DeviceFrame:
        new_df = df.copy()
        if isinstance(self.freq_threshold, dict):
            assert all(x in self.freq_threshold for x in col_selector.names)
        column_mapping = self.column_mapping(col_selector)
        for name, use in column_mapping.items():
            try:
                use_name = use[0] if len(use) == 1 else list(use)
                if use_name != name or self.encode_type == "joint":
                    storage = self.storage_name.get(name, name)     # categorify.py:501-504
                else:
                    storage = name
                new_df[name] = self._encode(name, use_name, storage, df)
            except Exception as e:
                raise RuntimeError(f"Failed to categorical encode column {name}") from e
        return new_df

    def _encode(self, name, use_name, storage, df) -> Column:
        fv = self._fitted(storage)
        # categorify.py:1607-1619: an int num_buckets is keyed by OUTPUT column name
        buckets = self.num_buckets
        if isinstance(buckets, int):
            buckets = {n: buckets for n in self.column_mapping_names}
        nb = buckets[storage] if buckets and storage in buckets else 0
        num_oov = nb or 1
        if self.single_table:                                       # :1683-1685
            null_label = fv.index_start
        else:
            null_label = NULL_OFFSET
        oov_label = null_label + 1
        first_label = fv.index_start if self.single_table else oov_label + num_oov
        if isinstance(use_name, list):
            cols = [df[c] for c in use_name]
            key = fv.space.keys_for(cols)
            hash_cols = []
            if nb:
                for s, c in zip(fv.space.spaces, cols):
                    hc = s.hash_column(c)
                    hash_cols.append(hc if hc is not None else _leaf(c))
            src = cols[0]
            offsets = None
        else:
            src = df[use_name]
            key = fv.space.keys_for(src)
            hc = fv.space.hash_column(src) if nb else None
            hash_cols = [hc] if hc is not None else ([_leaf(src)] if nb else [])
            offsets = src.offsets
        labels = fv.vocab.encode(key, null_label, oov_label, first_label, nb, hash_cols,
                                 np.dtype(self.output_dtype))
        return Column(labels, None, offsets)

    @property
    def column_mapping_names(self):
        return self._mapping_names

    def column_mapping(self, col_selector):
        column_mapping = {}
        if self.encode_type == "combo":                              # categorify.py:539-553
            for group in col_selector.grouped_names:
                if isinstance(group, (tuple, list)):
                    name = _make_name(*group, sep=self.name_sep)
                    group = [*group]
                else:
                    name = group
                    group = [group]
                column_mapping[name] = group
        else:
            column_mapping = super().column_mapping(col_selector)
        self._mapping_names = list(column_mapping.keys())
        return column_mapping

    # -------------------------------------------------------------------- schema
    def get_embedding_sizes(self, columns):
        """_get_embeddings_dask (categorify.py:666-684)."""
        buckets = self.num_buckets
        if isinstance(buckets, int):
            buckets = {name: buckets for name in columns}
        out = {}
        for col in columns:
            num_rows = OOV_OFFSET
            fv = self.categories.fitted.get(col)
            if fv is None and dict.get(self.categories, col) is not None:
                fv = self._fitted(col)          # a workflow reloaded from disk: read the file
            if fv is not None:
                num_rows += fv.file_rows
            if isinstance(buckets, dict):
                bucket_size = buckets.get(col, 0)
            else:
                bucket_size = 1
            out[col] = emb_sz_rule(num_rows + bucket_size)
        return out

    def _compute_properties(self, col_schema, input_schema):
        new_schema = super()._compute_properties(col_schema, input_schema)
        col_name = col_schema.name
        category_name = self.storage_name.get(col_name, col_name)
        target_category_path = dict.get(self.categories, category_name, None)
        cardinality, dimensions = self.get_embedding_sizes([category_name])[category_name]
        to_add = {
            "num_buckets": _resolve(self.num_buckets, col_name),
            "freq_threshold": _resolve(self.freq_threshold, col_name),
            "max_size": _resolve(self.max_size, col_name),
            "cat_path": target_category_path,
            "domain": {"min": 0, "max": cardinality - 1, "name": category_name},
            "embedding_sizes": {"cardinality": cardinality, "dimension": dimensions},
        }
        return col_schema.with_properties({**new_schema.properties, **to_add})

    @property
    def output_tags(self):
        return [Tags.CATEGORICAL]

    @property
    def output_dtype(self):
        return self.dtype or np.int64

    def inference_initialize(self, columns, inference_config):
        """categorify.py:602-609: the dict-of-arrays transform for serving (no 'combo' support)"""
        if self.encode_type == "combo":
            warnings.warn("Falling back to unoptimized inference path for encode_type 'combo' ")
            return None
        from ..inference import CategorifyTransform
        return CategorifyTransform(self)

    @property
    def supported_formats(self):
        from ..inference import DataFormats
        return (DataFormats.PANDAS_DATAFRAME | DataFormats.CUDF_DATAFRAME | DataFormats.NUMPY_DICT_ARRAY
                | DataFormats.CUPY_DICT_ARRAY)


def _global_rows(local_rows: int) -> int:
    """sum over ranks of the rows a rank folded in: an upper bound on any group's global size"""
    from ..dist import world
    if world()[0] == 1:
        return int(local_rows)
    import torch.distributed as dist
    dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() and \
        dist.get_backend() == "nccl" else torch.device("cpu")
    t = torch.tensor([int(local_rows)], dtype=torch.int64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return int(t.item())


def _parse_bytes(v):
    if isinstance(v, (int, float)):
        return int(v)
    s = str(v).strip().upper()
    units = {"KB": 10**3, "MB": 10**6, "GB": 10**9, "TB": 10**12, "KIB": 2**10, "MIB": 2**20,
             "GIB": 2**30, "B": 1}
    for u in sorted(units, key=len, reverse=True):
        if s.endswith(u):
            return int(float(s[: -len(u)]) * units[u])
    return int(float(s))


def _global_unique_merge(agg: engine.HashAgg):
    """Local table -> globally merged (keys, sizes, null_size), identical on every
    rank (single GPU: a plain export).  See nvtabular_b200/dist.py."""
    from ..dist import global_merge
    keys, sizes, _, null_size, _ = global_merge(agg)
    return keys, sizes, null_size
