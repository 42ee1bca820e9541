"""Groupby and Dataset.shuffle_by_keys on the GPU against oracle/session_groupby.py.

Exactness: integer outputs and the float32 outputs of exactly representable inputs (values
k * 2^-e with |k| < 2^15, the tests/_exact_stats.py convention) are bit-exact, except var / std,
whose mean is rounded in fp64 and which are checked within 1 float32 ulp like every output of
general float64 inputs.  NaN matches NaN; a null matches a cleared validity bit."""
import math

import numpy as np
import pandas as pd
import pytest
import torch

import nvtabular_b200 as nvt
from nvtabular_b200.column import DeviceFrame
from oracle.session_groupby import session_groupby

pytestmark = pytest.mark.gpu
NaN = float("nan")
ALL = ["count", "sum", "mean", "var", "std", "median", "nunique", "min", "max", "first", "last", "list"]


def _values(col):
    """a device output column -> python values (None = null), lists for list columns"""
    vals, mask = col.to_numpy()
    if col.dictionary is not None:
        d = col.dictionary
        vals = np.array([d[v] if 0 <= v < len(d) else None for v in vals], dtype=object)
    out = [None if (mask is not None and mask[i]) else vals[i].item() if hasattr(vals[i], "item") else vals[i]
           for i in range(len(vals))]
    if col.offsets is not None:
        off = col.offsets.cpu().numpy()
        return [out[off[i]:off[i + 1]] for i in range(len(off) - 1)]
    return out


def _close(a, b, ulps):
    if a is None or b is None or (isinstance(a, float) and math.isnan(a)) or (isinstance(b, float) and math.isnan(b)):
        na = a is None or (isinstance(a, float) and math.isnan(a))
        nb = b is None or (isinstance(b, float) and math.isnan(b))
        return na and nb
    if isinstance(a, float) or isinstance(b, float):
        if ulps == 0 or math.isinf(a) or math.isinf(b):
            return float(a) == float(b)
        fa, fb = np.float32(a), np.float32(b)
        return abs(int(fa.view(np.int32)) - int(fb.view(np.int32))) <= ulps if np.sign(fa) == np.sign(fb) else fa == fb
    return a == b


def _run(df, groupby_cols, sort_cols=None, aggs="list", ascending=True, columns=None, ulps=0, loose=("var", "std")):
    columns = list(columns or df.columns)
    op = nvt.ops.Groupby(groupby_cols=groupby_cols, sort_cols=sort_cols, aggs=aggs, ascending=ascending)
    wf = nvt.Workflow(columns >> op)
    frame = DeviceFrame.from_pandas(df)
    wf.fit_schema(nvt.Dataset(frame).schema)
    out = wf.transform(frame)
    exp = session_groupby(df, groupby_cols, sort_cols, aggs, ascending=ascending, columns=columns)
    assert out.columns == list(exp), (out.columns, list(exp))
    for name, want in exp.items():
        got = _values(out[name])
        assert len(got) == len(want), name
        tol = max(ulps, 1 if name.rsplit("_", 1)[-1] in loose else 0)
        for i, (g, w) in enumerate(zip(got, want)):
            if isinstance(w, list):
                assert len(g) == len(w) and all(_close(x, y, 0) for x, y in zip(g, w)), (name, i, g, w)
            else:
                assert _close(g, w, tol), (name, i, g, w)
    for name, sch in wf.output_schema.column_schemas.items():
        c = out[name]
        assert c.is_list == bool(sch.is_list), name
        if not c.is_string:
            assert c.np_dtype == np.dtype(sch.dtype), (name, c.np_dtype, sch.dtype)
    return out


def _exact_values(rng, n, dtype):
    v = rng.integers(-(1 << 14), 1 << 14, n)
    if np.dtype(dtype).kind == "f":
        return v.astype(dtype) * np.asarray(2.0 ** -4, dtype=dtype)
    return v.astype(dtype)


def _with_nulls(arr, mask, dtype):
    ext = {"int32": "Int32", "int64": "Int64", "float32": "Float32", "float64": "Float64"}[dtype]
    return pd.array([None if m else x for x, m in zip(arr.tolist(), mask)], dtype=ext)


@pytest.mark.parametrize("dtype", ["int32", "int64", "float32", "float64"])
def test_every_agg_on_values_with_nulls_and_all_null_groups(dtype):
    rng = np.random.default_rng(3)
    n = 20000
    k = rng.integers(0, 1500, n)
    v = _exact_values(rng, n, dtype)
    v[rng.random(n) < 0.2] = 0            # ties for median / nunique (and -0.0 below)
    if np.dtype(dtype).kind == "f":
        v[rng.random(n) < 0.05] = -0.0
    mask = (rng.random(n) < 0.15) | (k % 97 == 0)           # groups 0, 97, ... are all null
    df = pd.DataFrame({"k": k, "v": _with_nulls(v, mask, dtype), "ts": rng.permutation(n)})
    _run(df, "k", "ts", {"v": ALL}, columns=["k", "v", "ts"])


def test_general_float64_values_within_one_ulp():
    rng = np.random.default_rng(5)
    n = 30000
    df = pd.DataFrame({"k": rng.integers(0, 800, n), "v": rng.standard_normal(n) * 1e3})
    _run(df, "k", None, {"v": ["sum", "mean", "var", "std", "median", "min", "max"]}, ulps=1)


def test_var_of_timestamps_does_not_cancel():
    rng = np.random.default_rng(7)
    n = 50000
    k = rng.integers(0, 300, n)
    ts = 1.7e9 + rng.integers(0, 1000, n).astype(np.float64) * 0.25
    df = pd.DataFrame({"k": k, "ts": ts})
    out = _run(df, "k", None, {"ts": ["var", "std", "mean"]}, ulps=1)
    assert np.all(np.isfinite(_values(out["ts_var"])))


@pytest.mark.parametrize("kind", ["int32", "int64_extremes", "float64_special", "string", "bool"])
def test_key_kinds(kind):
    rng = np.random.default_rng(11)
    n = 5000
    if kind == "int32":
        key = pd.array(rng.integers(-50, 50, n), dtype="Int32")
        key[rng.random(n) < 0.1] = None
    elif kind == "int64_extremes":
        pool = np.array([np.iinfo(np.int64).min, np.iinfo(np.int64).max, 0, -1, 1, 1 << 40], dtype=np.int64)
        key = pool[rng.integers(0, len(pool), n)]
    elif kind == "float64_special":
        pool = np.array([0.0, -0.0, NaN, np.inf, -np.inf, 1.5, -2.25, 1e300])
        key = pool[rng.integers(0, len(pool), n)]
    elif kind == "string":
        pool = np.array(["b", "a", "zz", "", "ab", None], dtype=object)
        key = pool[rng.integers(0, len(pool), n)]
    else:
        key = rng.random(n) < 0.3
    df = pd.DataFrame({"key": key, "x": rng.integers(0, 1000, n).astype(np.int32), "ts": rng.integers(0, 50, n)})
    _run(df, "key", "ts", {"x": ["list", "count", "first", "last", "min"]})


def test_two_and_three_column_keys_with_null_keys():
    rng = np.random.default_rng(13)
    n = 8000
    a = pd.array(rng.integers(0, 5, n), dtype="Int64")
    a[rng.random(n) < 0.05] = None
    b = np.array(["x", "y", None], dtype=object)[rng.integers(0, 3, n)]
    c = rng.integers(-3, 3, n).astype(np.float32)
    df = pd.DataFrame({"a": a, "b": b, "c": c, "v": rng.integers(0, 100, n)})
    _run(df, ["a", "b"], None, {"v": ["list", "sum"]})
    _run(df, ["a", "b", "c"], None, {"v": ["list", "max"]})


@pytest.mark.parametrize("ascending", [True, False])
def test_sort_columns(ascending):
    rng = np.random.default_rng(17)
    n = 6000
    ts = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, dtype=np.int64)   # full range: split field
    ts[rng.random(n) < 0.3] = ts[0]                                                        # ties
    f = rng.standard_normal(n)
    f[rng.random(n) < 0.1] = NaN
    s = np.array(["p", "q", "r", None], dtype=object)[rng.integers(0, 4, n)]
    df = pd.DataFrame({"k": rng.integers(0, 40, n), "ts": ts, "f": f, "s": s, "row": np.arange(n)})
    _run(df, "k", "ts", {"row": ["list", "first", "last"]}, ascending=ascending)
    _run(df, "k", ["f", "ts"], {"row": ["list", "first", "last"]}, ascending=ascending)
    _run(df, "k", ["s", "f"], {"row": ["list", "first", "last"]}, ascending=ascending)


def test_list_null_leaves_and_list_input_first_last():
    df = pd.DataFrame({"k": [1, 2, 1, 2, 1], "ts": [3, 1, 2, 5, 1],
                       "v": pd.array([1.5, None, None, 4.0, 2.0], dtype="Float64"),
                       "l": [[1, 2], [3], [], [4, 5, 6], [7]]})
    out = _run(df, "k", "ts", {"v": ["list", "first", "last"]}, columns=["k", "ts", "v"])
    assert _values(out["v_list"]) == [[2.0, None, 1.5], [None, 4.0]]
    op = nvt.ops.Groupby(groupby_cols="k", sort_cols="ts", aggs={"l": ["first", "last"]})
    res = nvt.Workflow(["k", "ts", "l"] >> op).transform(DeviceFrame.from_pandas(df))
    assert _values(res["l_first"]) == [[7], [3]]
    assert _values(res["l_last"]) == [[1, 2], [4, 5, 6]]
    with pytest.raises(ValueError):
        nvt.Workflow(["k", "l"] >> nvt.ops.Groupby(groupby_cols="k", aggs="list")).transform(DeviceFrame.from_pandas(df))
    with pytest.raises(TypeError):
        nvt.Workflow(["k", "s"] >> nvt.ops.Groupby(groupby_cols="k", aggs="mean")).transform(
            DeviceFrame.from_pandas(pd.DataFrame({"k": [1], "s": ["a"]})))


def test_empty_and_all_null_key_partitions():
    df = pd.DataFrame({"k": pd.array([None, None, None], dtype="Int64"), "v": [1.0, 2.0, 3.0]})
    for frame in (df, df.iloc[:0]):
        out = _run(frame, "k", None, {"v": ["list", "count", "mean", "min", "first"]})
        assert len(out["v_count"]) == 0 and out["v_mean"].data.dtype == torch.float32
        assert out["v_min"].data.dtype == torch.float64 and out["v_list"].is_list


def test_deterministic():
    rng = np.random.default_rng(19)
    n = 200000
    df = pd.DataFrame({"k": rng.integers(0, 3000, n), "v": rng.standard_normal(n), "ts": rng.random(n)})
    frame = DeviceFrame.from_pandas(df)
    wf = nvt.Workflow(["k", "v", "ts"] >> nvt.ops.Groupby("k", "ts", {"v": ["sum", "mean", "var", "median", "list"]}))
    a, b = wf.transform(frame), wf.transform(frame)
    for name in a.columns:
        assert torch.equal(a[name].data.view(torch.uint8), b[name].data.view(torch.uint8)), name


def _segment_check(df, key, out, vcol):
    """vectorised oracle for the large shapes: count, mean (fp64 -> f32), first by input order"""
    g = df.groupby(key, sort=True)
    np.testing.assert_array_equal(out[key].data.cpu().numpy(), np.asarray(list(g.groups.keys())))
    np.testing.assert_array_equal(out[f"{vcol}_count"].data.cpu().numpy(), g[vcol].count().to_numpy())
    mean = (g[vcol].sum() / g[vcol].count()).to_numpy().astype(np.float32)
    got = out[f"{vcol}_mean"].data.cpu().numpy()
    assert np.max(np.abs(got.view(np.int32).astype(np.int64) - mean.view(np.int32).astype(np.int64))) <= 1
    np.testing.assert_array_equal(out[f"{vcol}_first"].data.cpu().numpy(), g[vcol].first().to_numpy())


def test_one_giant_group_beside_a_million_singletons():
    n = 1 << 24
    rng = np.random.default_rng(23)
    k = np.arange(n, dtype=np.int64)
    big = rng.random(n) < 0.6
    k[big] = -1
    df = pd.DataFrame({"k": k, "v": rng.integers(0, 1 << 10, n).astype(np.float64)})
    op = nvt.ops.Groupby("k", None, {"v": ["count", "mean", "first", "var"]})
    out = nvt.Workflow(["k", "v"] >> op).transform(DeviceFrame.from_pandas(df))
    _segment_check(df, "k", out, "v")
    v0 = df.v[big].to_numpy()
    assert abs(float(out["v_var"].data[0]) - np.float32(np.var(v0, ddof=1))) <= 1e-6 * np.var(v0)


def test_power_law_session_table():
    from nvtabular_b200.synth import session_frame
    n = 1 << 25
    frame, _ = session_frame(n, seed=29, device="cuda")
    op = nvt.ops.Groupby("session_id", "ts", {"item_id": ["list", "count", "first", "last"], "price": "mean"})
    out = nvt.Workflow(["session_id", "item_id", "ts", "price"] >> op).transform(frame)
    sid = frame["session_id"].data.cpu().numpy()
    ts = frame["ts"].data.cpu().numpy()
    item = frame["item_id"].data.cpu().numpy()
    order = np.lexsort((ts, sid))
    s_sorted = sid[order]
    starts = np.flatnonzero(np.r_[True, s_sorted[1:] != s_sorted[:-1]])
    np.testing.assert_array_equal(out["session_id"].data.cpu().numpy(), s_sorted[starts])
    np.testing.assert_array_equal(out["item_id_first"].data.cpu().numpy(), item[order][starts])
    ends = np.r_[starts[1:], n] - 1
    np.testing.assert_array_equal(out["item_id_last"].data.cpu().numpy(), item[order][ends])
    np.testing.assert_array_equal(out["item_id_count"].data.cpu().numpy(), np.diff(np.r_[starts, n]))
    np.testing.assert_array_equal(out["item_id_list"].data.cpu().numpy(), item[order])


def test_shuffle_by_keys_properties():
    rng = np.random.default_rng(31)
    n = 30000
    df = pd.DataFrame({"a": rng.integers(0, 400, n), "b": np.array(["u", "v", "w", None], dtype=object)[rng.integers(0, 4, n)],
                       "f": np.where(rng.random(n) < 0.5, 0.0, -0.0), "row": np.arange(n)})
    ds = nvt.Dataset(df, npartitions=4).shuffle_by_keys(["a", "b", "f"], npartitions=5)
    parts = [p.to_pandas() for p in ds.partitions()]
    assert len(parts) == 5
    seen = {}
    for i, p in enumerate(parts):
        assert list(p["row"]) == sorted(p["row"])                              # input order kept
        for key in set(zip(p["a"], p["b"].fillna("<null>"), p["f"] + 0.0)):
            assert seen.setdefault(key, i) == i                                # one partition per key
    allrows = pd.concat(parts, ignore_index=True).sort_values("row", ignore_index=True)
    pd.testing.assert_frame_equal(allrows[["a", "b", "row"]], df[["a", "b", "row"]], check_dtype=False)
    dicts = {tuple(p["b"].dictionary) for p in ds.partitions()}
    assert dicts == {("u", "v", "w")}                                           # unified dictionaries


def test_end_to_end_after_shuffle_and_with_categorify():
    rng = np.random.default_rng(37)
    n = 20000
    df = pd.DataFrame({"session_id": rng.integers(0, 2000, n), "item_id": rng.integers(0, 300, n),
                       "ts": rng.integers(0, 10 ** 6, n), "price": _exact_values(rng, n, "float64")})
    ds = nvt.Dataset(df, npartitions=3).shuffle_by_keys(["session_id"])
    feats = ["session_id", "item_id", "ts", "price"] >> nvt.ops.Groupby(
        groupby_cols=["session_id"], sort_cols=["ts"],
        aggs={"item_id": ["list", "count"], "ts": ["first", "last"], "price": "mean"})
    out = nvt.Workflow(feats).fit_transform(ds).to_ddf().compute().sort_values("session_id", ignore_index=True)
    exp = session_groupby(df, "session_id", "ts", {"item_id": ["list", "count"], "ts": ["first", "last"],
                                                   "price": "mean"})
    assert out["session_id"].tolist() == exp["session_id"]
    assert [list(x) for x in out["item_id_list"]] == exp["item_id_list"]
    assert out["ts_first"].tolist() == exp["ts_first"] and out["ts_last"].tolist() == exp["ts_last"]
    assert out["price_mean"].tolist() == exp["price_mean"]

    cat = ["item_id"] >> nvt.ops.Categorify(out_path="/tmp/nvtb_gb_cat")
    wf = nvt.Workflow((cat + ["session_id", "ts"]) >> nvt.ops.Groupby("session_id", "ts", {"item_id": "list"}))
    res = wf.fit_transform(nvt.Dataset(df)).to_ddf().compute()
    assert len(res) == df.session_id.nunique() and res["item_id_list"].map(len).sum() == n

    wf2 = nvt.Workflow(["session_id", "item_id", "ts"] >> nvt.ops.Groupby("session_id", "ts", {"item_id": "list"})
                       >> nvt.ops.Categorify(out_path="/tmp/nvtb_gb_cat2"))
    res2 = wf2.fit_transform(nvt.Dataset(df)).to_ddf().compute()
    assert res2["item_id_list"].map(len).sum() == n
