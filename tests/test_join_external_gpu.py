"""JoinExternal on the GPU (csrc/join.cu, K9) against the pandas oracle (oracle/join_external.py):
every key kind, both join kinds, unique and duplicated ext keys, nulls on both sides, every ext
column kind, the edge cases and the workflow-level paths."""
import numpy as np
import pandas as pd
import pytest

import nvtabular as nvt
from nvtabular import ops
from oracle.join_external import join_external as oracle_join

pytestmark = pytest.mark.gpu


def _is_list(v):
    return isinstance(v, (list, tuple, np.ndarray))


def _same(got: pd.DataFrame, want: pd.DataFrame):
    assert list(got.columns) == list(want.columns)
    assert len(got) == len(want), (len(got), len(want))
    for c in want.columns:
        g, w = got[c].tolist(), want[c].tolist()
        if any(_is_list(v) for v in w) or any(_is_list(v) for v in g):
            assert [list(x) for x in g] == [list(x) for x in w], c
            continue
        if want[c].dtype.kind in "iu" and got[c].dtype.kind in "iu":
            assert np.array_equal(got[c].to_numpy(np.int64), want[c].to_numpy(np.int64)), c
            continue
        if want[c].dtype.kind in "fiub" and got[c].dtype.kind in "fiub":
            a = got[c].to_numpy(dtype=np.float64, na_value=np.nan)
            b = want[c].to_numpy(dtype=np.float64, na_value=np.nan)
            assert np.array_equal(a, b, equal_nan=True), (c, a, b)
            continue
        norm = [None if (v is None or (isinstance(v, float) and np.isnan(v))) else v for v in g]
        wnorm = [None if (v is None or (isinstance(v, float) and np.isnan(v))) else v for v in w]
        assert norm == wnorm, c


def _run(left, ext, on, how="left", select=None, **kw):
    select = select or list(left.columns)
    wf = nvt.Workflow(select >> ops.JoinExternal(ext, on=on, how=how, **kw))
    wf.fit(nvt.Dataset(left[select]))
    return wf.transform(left[select])


def _check(left, ext, on, how="left", **kw):
    got = _run(left, ext, on, how, **kw)
    want = oracle_join(left, ext, on, how=how, on_ext=kw.get("on_ext"), columns_ext=kw.get("columns_ext"),
                       drop_duplicates_ext=kw.get("drop_duplicates_ext", False))
    _same(got, want)
    return got


def _keys(kind, vals, rng):
    if kind == "int32":
        return pd.Series(vals, dtype="int32")
    if kind == "int64":
        return pd.Series(np.asarray(vals, dtype=np.int64) * 1_000_000_007)
    if kind == "float":
        return pd.Series(np.asarray(vals, dtype=np.float64) / 4.0)
    if kind == "string":
        return pd.Series([f"k{v}" for v in vals], dtype=object)
    raise AssertionError(kind)


def _ext_payload(n, rng):
    genres = ["Drama", "Comedy", "Action", "Horror", "Sci-Fi"]
    i = pd.Series(rng.integers(-5, 5, n), dtype="Int64")
    i[rng.random(n) < 0.2] = pd.NA
    f = pd.Series(rng.random(n))
    f[rng.random(n) < 0.2] = np.nan
    s = pd.Series([f"s{v}" for v in rng.integers(0, 7, n)], dtype=object)
    s[rng.random(n) < 0.2] = None
    return pd.DataFrame({"e_i32": rng.integers(0, 100, n).astype("int32"), "e_int": i, "e_f": f,
                         "e_b": rng.random(n) < 0.5, "e_s": s,
                         "e_l": [list(rng.choice(genres, rng.integers(1, 4), replace=False)) for _ in range(n)]})


@pytest.mark.parametrize("how", ["left", "inner"])
@pytest.mark.parametrize("kind", ["int32", "int64", "float", "string"])
@pytest.mark.parametrize("dup", [False, True])
def test_parity_single_key(how, kind, dup):
    rng = np.random.default_rng(hash((how, kind, dup)) % 2**32)
    ext_vals = np.arange(0, 40) if not dup else rng.integers(0, 30, 80)
    ext = pd.concat([pd.DataFrame({"k": _keys(kind, ext_vals, rng)}), _ext_payload(len(ext_vals), rng)], axis=1)
    left = pd.DataFrame({"k": _keys(kind, rng.integers(-5, 45, 500), rng), "x": rng.random(500)})
    # null keys on both sides (NaN for floats), and -0.0 against +0.0
    if kind == "float":
        left.loc[::17, "k"] = np.nan
        left.loc[3, "k"] = -0.0
        ext.loc[5, "k"] = np.nan
    elif kind == "string":
        left.loc[::17, "k"] = None
        ext.loc[5, "k"] = None
    else:
        left["k"] = left["k"].astype("Int64" if kind == "int64" else "Int32")
        left.loc[::17, "k"] = pd.NA
        ext["k"] = ext["k"].astype("Int64" if kind == "int64" else "Int32")
        ext.loc[5, "k"] = pd.NA
    _check(left, ext, "k", how)


@pytest.mark.parametrize("how", ["left", "inner"])
def test_parity_int32_against_int64_and_int_against_float(how):
    rng = np.random.default_rng(7)
    ext = pd.DataFrame({"k": np.arange(0, 50, dtype=np.int64), "v": rng.random(50)})
    left = pd.DataFrame({"k": rng.integers(-3, 60, 300).astype(np.int32)})
    _check(left, ext, "k", how)
    ext_f = pd.DataFrame({"kf": np.arange(0, 50, dtype=np.float64) / 2.0, "v": rng.random(50)})
    _check(left, ext_f, "k", how, on_ext="kf")
    left_f = pd.DataFrame({"k": rng.integers(-3, 60, 300) / 2.0})
    _check(left_f, ext, "k", how)


@pytest.mark.parametrize("how", ["left", "inner"])
@pytest.mark.parametrize("ncols", [2, 3])
@pytest.mark.parametrize("dup", [False, True])
def test_parity_multi_column_keys(how, ncols, dup):
    rng = np.random.default_rng(ncols * 10 + dup)
    n_ext = 60
    cols = {"a": rng.integers(0, 4, n_ext).astype(np.int32), "b": rng.integers(0, 5, n_ext).astype(np.int64),
            "c": [f"c{v}" for v in rng.integers(0, 3, n_ext)]}
    ext = pd.DataFrame({f"{k}_e": v for k, v in list(cols.items())[:ncols]})
    if not dup:
        ext = ext.drop_duplicates(ignore_index=True)
    ext["payload"] = np.arange(len(ext), dtype=np.int64) * (2**40 + 1)          # above 2^53 after the scale
    ext["payload"] *= 4099
    ext.loc[0, "a_e"] = 0
    left = pd.DataFrame({"a": rng.integers(0, 5, 400).astype(np.int64), "b": rng.integers(0, 6, 400).astype(np.int32),
                         "c": [f"c{v}" for v in rng.integers(0, 4, 400)]})
    on = ["a", "b", "c"][:ncols]
    left = left[on]
    left.loc[::13, "a"] = -1
    _check(left, ext, on, how, on_ext=[f"{k}_e" for k in on])


def test_multi_column_null_components_match():
    ext = pd.DataFrame({"a": [1.0, np.nan, np.nan, 2.0], "b": ["x", "y", None, None], "v": [10, 20, 30, 40]})
    left = pd.DataFrame({"a": [np.nan, np.nan, 1.0, 2.0, 2.0], "b": ["y", None, "x", None, "z"]})
    for how in ("left", "inner"):
        _check(left, ext, ["a", "b"], how)


@pytest.mark.parametrize("how", ["left", "inner"])
def test_columns_ext_and_drop_duplicates(how):
    rng = np.random.default_rng(3)
    ext = pd.DataFrame({"k": rng.integers(0, 20, 100), "v": rng.integers(0, 3, 100), "w": rng.random(100)})
    left = pd.DataFrame({"k": rng.integers(0, 25, 200)})
    for dd in (False, True):
        _check(left, ext, "k", how, columns_ext=["k", "v"], drop_duplicates_ext=dd)


def test_int64_payload_is_exact():
    big = np.array([2**62 + 1, -(2**61) - 3, 2**53 + 1], dtype=np.int64)
    ext = pd.DataFrame({"k": [1, 2, 3], "big": big})
    got = _check(pd.DataFrame({"k": [3, 1, 2, 3]}), ext, "k")
    assert got["big"].tolist() == [big[2], big[0], big[1], big[2]]


def test_edge_cases():
    ext = pd.DataFrame({"k": [1, 2, 2], "v": [1.0, 2.0, 3.0], "g": [["a"], ["b", "c"], []]})
    left = pd.DataFrame({"k": [5, 2, 1]})
    for how in ("left", "inner"):
        _check(left, ext.iloc[:0][["k", "v"]], "k", how)           # empty ext table
        _check(left.iloc[:0], ext, "k", how)                       # empty partition
        _check(pd.DataFrame({"k": [7, 8, 9]}), ext, "k", how)      # no key matches
        _check(left, ext, "k", how)


def test_one_key_matching_many_rows():
    n = 200_000
    ext = pd.DataFrame({"k": np.r_[np.full(n, 7), np.arange(100, 120)], "v": np.arange(n + 20, dtype=np.int64)})
    left = pd.DataFrame({"k": [7, 3, 105, 7], "x": [0.5, 1.5, 2.5, 3.5]})
    for how in ("left", "inner"):
        got = _check(left, ext, "k", how)
        assert len(got) == 2 * n + 1 + (how == "left")


def test_left_list_columns_pass_through_and_expand():
    left = pd.DataFrame({"k": [1, 2, 3], "tags": [["a", "b"], [], ["c"]]})
    for ext in (pd.DataFrame({"k": [1, 2], "v": [10, 20]}), pd.DataFrame({"k": [1, 1, 3], "v": [10, 11, 30]})):
        for how in ("left", "inner"):
            _check(left, ext, "k", how)


def _movielens(n_ratings=5000, n_movies=300, seed=0):
    rng = np.random.default_rng(seed)
    names = ["Action", "Adventure", "Animation", "Children", "Comedy", "Crime", "Documentary", "Drama", "Fantasy",
             "Film-Noir", "Horror", "Musical", "Mystery", "Romance", "Sci-Fi", "Thriller", "War", "Western"]
    movies = pd.DataFrame({"movieId": np.arange(1, n_movies + 1),
                           "genres": [list(rng.choice(names, rng.integers(1, 7), replace=False))
                                      for _ in range(n_movies)]})
    ratings = pd.DataFrame({"userId": rng.integers(1, 400, n_ratings), "movieId": rng.integers(1, n_movies + 1, n_ratings),
                            "rating": rng.integers(1, 11, n_ratings) / 2.0})
    return movies, ratings


def test_workflow_multi_partition_and_each_source_kind(tmp_path):
    import pyarrow as pa
    import pyarrow.parquet as pq
    movies, ratings = _movielens()
    movies["year"] = (1950 + movies["movieId"] % 70).astype("int32")
    want = oracle_join(ratings[["movieId", "userId"]], movies, "movieId")
    pq.write_table(pa.Table.from_pandas(movies.iloc[:150], preserve_index=False), tmp_path / "m0.parquet")
    pq.write_table(pa.Table.from_pandas(movies.iloc[150:], preserve_index=False), tmp_path / "m1.parquet")
    movies.drop(columns="genres").to_csv(tmp_path / "m.csv", index=False)
    sources = {"pandas": movies, "arrow": pa.Table.from_pandas(movies, preserve_index=False),
               "dataset": nvt.Dataset(movies, npartitions=3), "parquet_dir": str(tmp_path),
               "parquet_files": [str(tmp_path / "m0.parquet"), str(tmp_path / "m1.parquet")],
               "parquet_file": str(tmp_path / "m0.parquet")}
    for name, src in sources.items():
        wf = nvt.Workflow(["movieId", "userId"] >> ops.JoinExternal(src, on="movieId"))
        ds = nvt.Dataset(ratings, npartitions=4)
        got = wf.fit_transform(ds).to_ddf().compute()
        exp = want if name != "parquet_file" else oracle_join(ratings[["movieId", "userId"]], movies.iloc[:150], "movieId")
        _same(got.reset_index(drop=True), exp)
        assert [c.name for c in wf.output_schema] == ["movieId", "userId", "genres", "year"]
    wf = nvt.Workflow(["movieId"] >> ops.JoinExternal(str(tmp_path / "m.csv"), on="movieId", how="inner"))
    got = wf.fit_transform(nvt.Dataset(ratings, npartitions=2)).to_ddf().compute()
    _same(got.reset_index(drop=True), oracle_join(ratings[["movieId"]], movies.drop(columns="genres"), "movieId",
                                                  how="inner"))


def test_movielens_example_pipeline():
    """examples/02-Advanced-NVTabular-workflow.ipynb of the reference, on synthetic frames"""
    from oracle.categorify import categorify_encode, categorify_fit
    movies, ratings = _movielens(20000, 500, seed=5)
    joined = ["movieId"] >> ops.JoinExternal(movies, on="movieId", columns_ext=["movieId", "genres"])
    output = (joined >> ops.Categorify(freq_threshold=10)) + ["userId", "rating"]
    wf = nvt.Workflow(output)
    got = wf.fit_transform(nvt.Dataset(ratings, npartitions=3)).to_ddf().compute()
    j = oracle_join(ratings[["movieId"]], movies, "movieId", columns_ext=["movieId", "genres"])
    vocabs = categorify_fit(j, ["movieId", "genres"], freq_threshold=10)
    for col in ("movieId", "genres"):
        enc = categorify_encode(j, col, vocabs[col])
        g = got[col].tolist()
        if col == "genres":
            assert [list(x) for x in g] == [list(x) for x in enc]
        else:
            assert np.array_equal(np.asarray(g, dtype=np.int64), np.asarray(enc, dtype=np.int64))
    assert np.array_equal(got["userId"].to_numpy(), ratings["userId"].to_numpy())


def test_workflow_save_raises(tmp_path):
    movies, ratings = _movielens(100, 20)
    wf = nvt.Workflow(["movieId"] >> ops.JoinExternal(movies, on="movieId"))
    wf.fit(nvt.Dataset(ratings))
    with pytest.raises(Exception, match="JoinExternal"):
        wf.save(str(tmp_path / "wf"))
