"""CPU tests of JoinExternal: the pandas oracle (oracle/join_external.py) against the reference's
test_join_external and the rules it pins, the constructor's argument errors, and the
column_mapping / output schema of every kind of external table, read from metadata only."""
import numpy as np
import pandas as pd
import pytest

from oracle.join_external import join_external


def _frame(n=200, seed=0):
    rng = np.random.default_rng(seed)
    return pd.DataFrame({"name-cat": rng.choice(["Alice", "Bob", "Dan"], n), "x": rng.random(n),
                         "id": rng.integers(900, 1100, n)})


@pytest.mark.parametrize("how", ["left", "inner"])
@pytest.mark.parametrize("drop_duplicates", [True, False])
def test_oracle_matches_reference_test_join_external(how, drop_duplicates):
    """reference tests/unit/ops/test_join.py::test_join_external, re-typed for pandas"""
    df = _frame()
    shift = 100
    df_ext = df[["id"]].copy().sort_values("id")
    df_ext["new_col"] = df_ext["id"] + shift
    df_ext["new_col_2"] = "keep"
    df_ext["new_col_3"] = "ignore"
    columns_ext = ["id", "new_col", "new_col_2"]
    check = df_ext[columns_ext]
    if drop_duplicates:
        check = check.drop_duplicates(ignore_index=True)
    out = join_external(df, df_ext, "id", how=how, columns_ext=columns_ext, drop_duplicates_ext=drop_duplicates)
    assert len(out) == len(df.merge(check, how=how, on="id"))
    assert (out["id"] + shift == out["new_col"]).all()
    assert "new_col_2" in out.columns and "new_col_3" not in out.columns
    assert list(out.columns) == list(df.columns) + ["new_col", "new_col_2"]
    # rows follow left-row order (x is unique per left row)
    xs = out["x"].tolist()
    runs = [x for i, x in enumerate(xs) if i == 0 or xs[i - 1] != x]
    emitted = df["x"].tolist() if how == "left" else df.loc[df["id"].isin(check["id"]), "x"].tolist()
    assert runs == emitted


def test_oracle_row_order_and_ext_order_within_a_key():
    ext = pd.DataFrame({"k": [2, 1, 2, 2], "v": [10, 20, 30, 40]})
    left = pd.DataFrame({"k": [2, 3, 1, 2]})
    out = join_external(left, ext, "k", how="left")
    assert out["k"].tolist() == [2, 2, 2, 3, 1, 2, 2, 2]
    assert out["v"].tolist()[:3] == [10, 30, 40] and np.isnan(out["v"][3]) and out["v"].tolist()[4:] == [20, 10, 30, 40]
    inner = join_external(left, ext, "k", how="inner")
    assert inner["v"].tolist() == [10, 30, 40, 20, 10, 30, 40]


def test_oracle_nulls_nan_and_signed_zero():
    ext = pd.DataFrame({"k": [np.nan, 0.0, 1.5], "v": [1, 2, 3]})
    left = pd.DataFrame({"k": [np.nan, -0.0, 1.5, 2.0]})
    out = join_external(left, ext, "k", how="inner")
    assert out["v"].tolist() == [1, 2, 3]
    ext_i = pd.DataFrame({"k": pd.array([None, 1], dtype="Int64"), "v": [5, 6]})
    left_i = pd.DataFrame({"k": pd.array([1, None], dtype="Int64")})
    assert join_external(left_i, ext_i, "k", how="inner")["v"].tolist() == [6, 5]


def test_oracle_int_float_and_widths_compare_by_value():
    ext = pd.DataFrame({"k": np.array([1, 2, 3], dtype=np.int64), "v": [1, 2, 3]})
    left = pd.DataFrame({"k": np.array([3, 1], dtype=np.int32)})
    assert join_external(left, ext, "k", how="inner")["v"].tolist() == [3, 1]
    left_f = pd.DataFrame({"k": [3.0, 1.5]})
    assert join_external(left_f, ext, "k", how="inner")["v"].tolist() == [3]


def test_oracle_string_against_numeric_raises():
    with pytest.raises(ValueError):
        join_external(pd.DataFrame({"k": ["a"]}), pd.DataFrame({"k": [1], "v": [2]}), "k")


def test_oracle_unmatched_list_row_is_empty_and_name_clash_raises():
    ext = pd.DataFrame({"k": [1], "g": [["a", "b"]]})
    out = join_external(pd.DataFrame({"k": [1, 2]}), ext, "k")
    assert [list(x) for x in out["g"]] == [["a", "b"], []]
    with pytest.raises(ValueError, match="v"):
        join_external(pd.DataFrame({"k": [1], "v": [0]}), pd.DataFrame({"k": [1], "v": [2]}), "k")
    both = join_external(pd.DataFrame({"a": [1]}), pd.DataFrame({"b": [1], "v": [2]}), "a", on_ext="b")
    assert list(both.columns) == ["a", "b", "v"]


def test_oracle_multi_column_keys_and_drop_duplicates():
    ext = pd.DataFrame({"a": [1, 1, 2, 1], "b": ["x", "y", "x", "x"], "v": [1, 2, 3, 1]})
    left = pd.DataFrame({"a": [1, 2], "b": ["x", "x"]})
    assert join_external(left, ext, ["a", "b"], how="inner")["v"].tolist() == [1, 1, 3]
    assert join_external(left, ext, ["a", "b"], how="inner", drop_duplicates_ext=True)["v"].tolist() == [1, 3]
    with pytest.raises(TypeError):
        join_external(left, pd.DataFrame({"a": [1], "g": [["x"]]}), "a", drop_duplicates_ext=True)


# ------------------------------------------------------------------------------- the operator
def test_constructor_errors():
    from nvtabular import ops
    ext = pd.DataFrame({"k": [1], "v": [2]})
    with pytest.raises(ValueError, match="Only left join"):
        ops.JoinExternal(ext, on="k", how="outer")
    with pytest.raises(ValueError, match="kind_ext"):
        ops.JoinExternal(ext, on="k", kind_ext="feather")
    with pytest.raises(ValueError):
        ops.JoinExternal(object(), on="k")
    with pytest.raises(ValueError):
        ops.JoinExternal(ext, on=["k", "v"], on_ext="k")
    op = ops.JoinExternal(ext, on="k", kind_ext="PANDAS")
    assert op.kind_ext == "pandas" and op.on_ext == ["k"]


def test_key_and_name_errors_are_raised_before_any_data():
    import nvtabular as nvt
    from nvtabular import ColumnSelector, ops
    ext = pd.DataFrame({"k": [1], "v": [2]})
    op = ops.JoinExternal(ext, on="k")
    with pytest.raises(ValueError, match="'k'"):
        op._check(["x"])
    with pytest.raises(ValueError, match="'v'"):
        op._check(["k", "v"])
    with pytest.raises(ValueError, match="columns"):
        ops.JoinExternal(ext, on="k", columns_ext=["k", "nope"]).column_mapping(ColumnSelector(["k"]))
    assert not isinstance(op, ops.StatOperator)
    del nvt


def _schema_of(op, names, dtypes):
    import nvtabular as nvt
    from nvtabular_b200.graph import ColumnSchema, Schema
    wf = nvt.Workflow(names >> op)
    wf.fit_schema(Schema([ColumnSchema(n, dtype=np.dtype(d)) for n, d in zip(names, dtypes)]))
    return [(c.name, np.dtype(c.dtype), c.is_list) for c in wf.output_schema]


def test_column_mapping_and_schema_of_every_source_kind(tmp_path):
    import pyarrow as pa
    import pyarrow.parquet as pq
    from nvtabular import ops
    movies = pd.DataFrame({"movieId": np.arange(1, 4, dtype=np.int64), "genres": [["a"], ["b", "c"], []],
                           "year": np.array([1990, 1991, 1992], dtype=np.int32), "title": ["x", "y", "z"]})
    table = pa.Table.from_pandas(movies, preserve_index=False)
    pq.write_table(table, tmp_path / "movies.parquet")
    movies.drop(columns="genres").to_csv(tmp_path / "movies.csv", index=False)
    want = [("movieId", np.dtype("int64"), False), ("userId", np.dtype("int64"), False),
            ("genres", np.dtype("object"), True), ("year", np.dtype("int32"), False)]
    for src in (movies, table, str(tmp_path / "movies.parquet"), str(tmp_path), [str(tmp_path / "movies.parquet")]):
        op = ops.JoinExternal(src, on="movieId", columns_ext=["movieId", "genres", "year"])
        assert _schema_of(op, ["movieId", "userId"], ["int64", "int64"]) == want
        assert op._frame is None                    # the graph loaded no data
    op = ops.JoinExternal(str(tmp_path / "movies.csv"), on="movieId")
    got = _schema_of(op, ["movieId"], ["int64"])
    assert [n for n, _, _ in got] == ["movieId", "year", "title"]
    assert op.kind_ext == "csv" and op._frame is None


def test_distinct_key_names_keep_both_key_columns():
    from nvtabular import ColumnSelector, ops
    op = ops.JoinExternal(pd.DataFrame({"mid": [1], "v": [2.0]}), on="movieId", on_ext="mid")
    assert list(op.column_mapping(ColumnSelector(["movieId", "u"]))) == ["movieId", "u", "mid", "v"]
