"""The library's Parquet writer for the Categorify artefact files (csrc/artifacts.cu).

pandas must read every file back exactly as it reads what DataFrame.to_parquet writes for the
same frame: values, column dtypes, and the RangeIndex whose start carries the labels.  The host
writer runs without a device; the fit path (library threads that copy a vocabulary off the
device and decode its keys) is checked on the GPU against the pandas path it replaced."""
import os

import numpy as np
import pandas as pd
import pyarrow.parquet as pq
import pytest

from nvtabular_b200 import engine
from nvtabular_b200._lib import NvtbError
from nvtabular_b200.ops.categorify import _pandas_meta, _pandas_meta_parts, _write_numeric_parquet

KEY_DTYPES = [np.int32, np.int64, np.float64, np.float32]


def _keys(dtype, n, seed):
    rng = np.random.default_rng(seed)
    if np.issubdtype(dtype, np.integer):
        info = np.iinfo(dtype)
        k = rng.integers(info.min, info.max, n, dtype=dtype, endpoint=True)
        k[: min(n, 2)] = [info.min, info.max][: min(n, 2)]
        return k
    k = rng.standard_normal(n).astype(dtype) * 1e6
    special = np.array([np.nan, 0.0, -0.0, np.inf, -np.inf], dtype=dtype)
    k[: min(n, 5)] = special[: min(n, 5)]
    return k


def _same_as_pandas(path, frame, tmp_path):
    ref_path = tmp_path / "ref.parquet"
    frame.to_parquet(ref_path, compression=None)
    got = pd.read_parquet(path)
    pd.testing.assert_frame_equal(got, pd.read_parquet(ref_path))
    pd.testing.assert_frame_equal(got, frame)
    assert isinstance(got.index, pd.RangeIndex) and got.index.start == frame.index.start
    md = pq.read_metadata(path)
    assert md.num_rows == len(frame) and md.num_columns == len(frame.columns)


@pytest.mark.parametrize("n", [0, 1, 7, (1 << 20) + 3])
@pytest.mark.parametrize("key_dtype", KEY_DTYPES)
@pytest.mark.parametrize("with_sizes", [False, True])
def test_vocabulary_file_reads_back_like_to_parquet(tmp_path, n, key_dtype, with_sizes):
    keys = _keys(key_dtype, n, n)
    arrays = {"C1": keys}
    if with_sizes:
        arrays["C1_size"] = np.random.default_rng(n + 1).integers(1, 1 << 40, n).astype(np.int64)
    path = tmp_path / "unique.C1.parquet"
    _write_numeric_parquet(str(path), arrays, index_start=3)
    exp = pd.DataFrame(arrays)
    exp.index = pd.RangeIndex(3, 3 + n)
    _same_as_pandas(path, exp, tmp_path)
    got = pd.read_parquet(path)["C1"].to_numpy()
    # bit-exact keys: NaN stays NaN, -0.0 keeps its sign
    np.testing.assert_array_equal(got.view(f"u{got.itemsize}"), keys.view(f"u{keys.itemsize}"))


@pytest.mark.parametrize("page_rows", [1, 7, 64])
@pytest.mark.parametrize("n", [0, 1, 7, 50, 449])
@pytest.mark.parametrize("key_dtype", KEY_DTYPES)
def test_columns_cut_into_pages_read_back_like_to_parquet(tmp_path, page_rows, n, key_dtype):
    """a column is written as several data pages (each page's sizes are int32 in its header): every
    page must carry its own value count and definition levels"""
    keys = _keys(key_dtype, n, n + page_rows)
    sizes = np.arange(n, dtype=np.int64) * 3 + 1
    path = tmp_path / "unique.C1.parquet"
    engine.parquet_write(str(path), [("C1", keys), ("C1_size", sizes)],
                         _pandas_meta([("C1", keys.dtype), ("C1_size", sizes.dtype)], 5, n), page_rows=page_rows)
    exp = pd.DataFrame({"C1": keys, "C1_size": sizes})
    exp.index = pd.RangeIndex(5, 5 + n)
    _same_as_pandas(path, exp, tmp_path)
    rg = pq.read_metadata(path).row_group(0)
    assert rg.column(0).num_values == n and rg.column(1).num_values == n


@pytest.mark.parametrize("oov_count", [1, 5])
@pytest.mark.parametrize("with_observed", [False, True])
def test_meta_file_reads_back_like_to_parquet(tmp_path, oov_count, with_observed):
    n_kept, null_size, oov_size, unique_size = 123, 4, 17, 1 << 33
    cols = [("kind", "object"), ("offset", np.int64), ("num_indices", np.int64)]
    cols += [("num_observed", np.int64)] if with_observed else []
    path = tmp_path / "meta.C1.parquet"
    engine.parquet_write_meta(str(path), oov_count, n_kept, null_size, oov_size, unique_size, with_observed,
                              _pandas_meta(cols, 0, 4))
    meta = {"kind": ["pad", "null", "oov", "unique"], "offset": [0, 1, 2, 2 + oov_count],
            "num_indices": [1, 1, oov_count, n_kept]}
    if with_observed:
        meta["num_observed"] = [0, null_size, oov_size, unique_size]
    _same_as_pandas(path, pd.DataFrame(meta), tmp_path)


def test_pandas_metadata_is_completed_with_the_row_count():
    cols = [("C1", np.dtype("int32")), ("C1_size", np.dtype("int64"))]
    head, tail = _pandas_meta_parts(cols, 7)
    assert head + b"12" + tail == _pandas_meta(cols, 7, 5)


def test_unwritable_path_raises_naming_it(tmp_path):
    path = str(tmp_path / "missing-dir" / "unique.C1.parquet")
    with pytest.raises(NvtbError, match="missing-dir/unique.C1.parquet"):
        _write_numeric_parquet(path, {"C1": np.arange(3, dtype=np.int32)}, index_start=3)
    with pytest.raises(NvtbError, match="missing-dir/meta.C1.parquet"):
        engine.parquet_write_meta(str(tmp_path / "missing-dir" / "meta.C1.parquet"), 1, 3,
                                  pandas_meta=_pandas_meta([("kind", "object")], 0, 4))


# ---------------------------------------------------------------- the fit path, on the GPU
def _frame(n, seed):
    rng = np.random.default_rng(seed)
    i32 = rng.integers(-50, 50, n).astype(np.int32)
    i32[:3] = np.iinfo(np.int32).min
    i64 = rng.integers(-(1 << 40), 1 << 40, n)
    i64[:40] = np.iinfo(np.int64).min + rng.integers(0, 4, 40)
    f64 = np.round(rng.standard_normal(n), 1)
    f64[:5] = [np.nan, 0.0, -0.0, np.inf, -np.inf]
    f32 = (np.round(rng.standard_normal(n), 2)).astype(np.float32)
    f32[:3] = [-0.0, np.nan, 0.0]
    return pd.DataFrame({"a": i32, "b": i64, "c": f64, "d": f32})


def _pandas_files(fv):
    """what the pandas path writes for a fitted vocabulary (KeySpace.decode of the kept keys)"""
    meta = {"kind": ["pad", "null", "oov", "unique"],
            "offset": [0, 1, 2, 2 + (fv.num_buckets or 1)],
            "num_indices": [1, 1, fv.num_buckets or 1, fv.vocab.n_kept]}
    if fv.has_sizes:
        meta["num_observed"] = [0, fv.vocab.null_size, fv.vocab.oov_size, fv.vocab.unique_size]
    return pd.DataFrame(meta), fv.unique_frame()


@pytest.mark.gpu
@pytest.mark.parametrize("kw", [{}, {"freq_threshold": 2}, {"max_size": 20, "num_buckets": 4}])
def test_fit_files_match_the_pandas_path(tmp_path, kw):
    import nvtabular as nvt
    df = _frame(5000, 3)
    op = nvt.ops.Categorify(out_path=str(tmp_path), **kw)
    nvt.Workflow(list(df.columns) >> op).fit(nvt.Dataset(df))
    base = tmp_path / "categories"
    for name in df.columns:
        fv = op.categories.fitted[name]
        meta, uniq = _pandas_files(fv)
        pd.testing.assert_frame_equal(pd.read_parquet(base / f"meta.{name}.parquet"), meta)
        got = pd.read_parquet(base / f"unique.{name}.parquet")
        pd.testing.assert_frame_equal(got, uniq)
        key = got[name].to_numpy()
        np.testing.assert_array_equal(key.view(f"u{key.itemsize}"), uniq[name].to_numpy().view(f"u{key.itemsize}"))
        assert key.dtype == df[name].dtype


@pytest.mark.gpu
def test_fit_file_error_names_the_path_and_leaves_no_thread(tmp_path):
    import nvtabular as nvt
    df = _frame(1000, 4)

    def fit():
        nvt.Workflow(list(df.columns) >> nvt.ops.Categorify(out_path=str(tmp_path))).fit(nvt.Dataset(df))

    fit()
    tasks = len(os.listdir("/proc/self/task"))
    fit()
    assert len(os.listdir("/proc/self/task")) == tasks
    bad = tmp_path / "categories" / "meta.c.parquet"
    bad.unlink()
    bad.mkdir()                        # a directory where the file goes: the write must fail
    with pytest.raises(NvtbError, match="categories/meta.c.parquet"):
        fit()
    assert len(os.listdir("/proc/self/task")) == tasks
