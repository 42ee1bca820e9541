"""Filter and Dropna on the GPU (csrc/filter.cu, K11, with the gather of csrc/join.cu and the
sub-list copy of csrc/groupby.cu) against the oracle (oracle/filter.py) applied to to_pandas() of
the same frame with the same predicate, exactly: every comparison over every column kind with nulls
and NaNs, every mask size class and pattern, 2^31 + 65 rows, pass-through without a copy or a
launch, every column kind compacted, the reference's scenarios, fit through a filter that empties a
partition, save / load in a fresh process, and run-to-run bit identity."""
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest
import torch

import nvtabular as nvt
from nvtabular import ColumnSelector, ops
from nvtabular_b200 import engine
from nvtabular_b200.column import Column, DeviceFrame
from nvtabular_b200.graph import Node
from oracle.categorify import CategorifyOracle
from oracle.filter import dropna_frame, filter_frame
from oracle.normalize import normalize_fit

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SYMS = ["==", "!=", "<", "<=", ">", ">="]
CMP = {"==": lambda a, b: a == b, "!=": lambda a, b: a != b, "<": lambda a, b: a < b,
       "<=": lambda a, b: a <= b, ">": lambda a, b: a > b, ">=": lambda a, b: a >= b}


def keep_small(df):
    """a module-level predicate, so that a workflow holding it can be saved and loaded"""
    return (df["a"] < 40) | df["b"].isnull()


# ---------------------------------------------------------------------------------- helpers
def _eq(a, b):
    if a is None or b is None or (isinstance(a, float) and np.isnan(a)):
        return (a is None or (isinstance(a, float) and np.isnan(a))) and \
            (b is None or (isinstance(b, float) and np.isnan(b)))
    return a == b


def _cells(s: pd.Series):
    out = []
    for v in s.tolist():
        if isinstance(v, (list, np.ndarray)):
            out.append([None if x is None or (isinstance(x, float) and np.isnan(x)) else
                        (x.item() if isinstance(x, np.generic) else x) for x in list(v)])
        else:
            out.append(None if v is None or (isinstance(v, float) and np.isnan(v)) else
                       (v.item() if isinstance(v, np.generic) else v))
    return out


def _same(got: pd.DataFrame, want: pd.DataFrame, ctx="", rtol=0.0):
    assert list(got.columns) == list(want.columns), ctx
    assert len(got) == len(want), (ctx, len(got), len(want))
    for c in want.columns:
        a, b = got[c].to_numpy(), want[c].to_numpy()
        if a.dtype != object and b.dtype != object:
            if a.dtype != b.dtype:        # an int column whose nulls were all dropped: pandas' float image
                a, b = a.astype(np.float64), b.astype(np.float64)
            if rtol and a.dtype.kind == "f":
                np.testing.assert_allclose(a, b, rtol=rtol, err_msg=f"{ctx} {c}")
            else:
                np.testing.assert_array_equal(a, b, err_msg=f"{ctx} {c}")
            continue
        g, w = _cells(got[c]), _cells(want[c])
        assert all(_eq(x, y) if not isinstance(y, list) else (len(x) == len(y) and all(map(_eq, x, y)))
                   for x, y in zip(g, w)), (ctx, c)


def _filter(frame: DeviceFrame, f):
    return ops.Filter(f).transform(ColumnSelector(frame.columns), frame)


def _check_filter(frame: DeviceFrame, f, ctx=""):
    got = _filter(frame, f)
    _same(got.to_pandas(), filter_frame(frame.to_pandas(), f), ctx)
    return got


def _numeric_frame(n, seed):
    """int32 / int64 / float32 / float64 / bool columns with nulls, NaNs, and values on both
    sides of every scalar the comparisons use"""
    rng = np.random.default_rng(seed)
    null = lambda p=0.1: rng.random(n) < p  # noqa: E731
    ints = rng.integers(-6, 7, n)
    f32 = rng.choice(np.array([-2.5, 0.0, 2.5, 3.0, 0.1, np.nan], np.float32), n)
    f64 = rng.choice(np.array([-2.5, 0.0, 2.5, 3.0, 0.1, np.nan, 2.0 ** 53]), n)
    cols = {
        "i32": pa.array(ints.astype(np.int32), mask=null()),
        "i64": pa.array(ints.astype(np.int64) * 3, mask=null()),
        "big": pa.array(np.array([2 ** 53 + 1, 2 ** 53, 2 ** 40, -3], np.int64)[rng.integers(0, 4, n)]),
        "f32": pa.array(f32, mask=null()),
        "f64": pa.array(f64, mask=null()),
        "bool": pa.array(rng.random(n) < 0.5, mask=null()),
        "flag": pa.array(rng.random(n) < 0.5),
        "u8": pa.array(rng.integers(0, 256, n).astype(np.uint8)),
    }
    return DeviceFrame.from_arrow(pa.table(cols))


def _kinds_frame(n, seed, lists=True):
    """every column kind, with and without validity"""
    rng = np.random.default_rng(seed)
    cols = {
        "i32": pa.array(rng.integers(-1000, 1000, n).astype(np.int32)),
        "i64n": pa.array(rng.integers(-2 ** 40, 2 ** 40, n), mask=rng.random(n) < 0.2),
        "f32n": pa.array(rng.normal(size=n).astype(np.float32), mask=rng.random(n) < 0.2),
        "f64": pa.array(rng.normal(size=n)),
        "bool": pa.array(rng.random(n) < 0.5, mask=rng.random(n) < 0.1),
        "u8": pa.array(rng.integers(0, 256, n).astype(np.uint8)),
        "s": pa.array([None if rng.random() < 0.1 else f"s{rng.integers(0, 30)}" for _ in range(n)], pa.string()),
    }
    if lists:
        cols["l"] = pa.array([None if rng.random() < 0.05 else
                              [None if rng.random() < 0.1 else int(rng.integers(0, 99))
                               for _ in range(int(rng.integers(0, 5)))] for _ in range(n)],
                             type=pa.list_(pa.int64()))
        cols["ls"] = pa.array([[f"t{rng.integers(0, 9)}" for _ in range(int(rng.integers(0, 3)))]
                               for _ in range(n)], type=pa.list_(pa.string()))
    return DeviceFrame.from_arrow(pa.table(cols))


# ------------------------------------------------------------------------------ comparisons
@pytest.mark.parametrize("col", ["i32", "i64", "big", "f32", "f64", "bool", "u8"])
@pytest.mark.parametrize("scalar", [3, 2.5, True, 2 ** 40, 2 ** 53 + 1, -(2 ** 40), float("nan"), np.float32(0.1)],
                         ids=["int", "float", "bool", "2^40", "2^53+1", "-2^40", "nan", "np.float32"])
def test_compare_with_scalar(col, scalar):
    frame = _numeric_frame(3001, 1)
    for sym in SYMS:
        _check_filter(frame, lambda d, s=sym: CMP[s](d[col], scalar), f"{col} {sym} {scalar!r}")
        _check_filter(frame, lambda d, s=sym: CMP[s](scalar, d[col]), f"{scalar!r} {sym} {col}")


@pytest.mark.parametrize("a, b", [("i32", "i64"), ("i32", "f32"), ("i64", "f64"), ("f32", "f64"), ("f32", "f32"),
                                  ("bool", "i32"), ("bool", "f32"), ("u8", "i64"), ("big", "f64")])
def test_compare_columns(a, b):
    frame = _numeric_frame(2049, 2)
    for sym in SYMS:
        _check_filter(frame, lambda d, s=sym: CMP[s](d[a], d[b]), f"{a} {sym} {b}")


def test_compare_strings():
    rng = np.random.default_rng(3)
    vals = [None if rng.random() < 0.1 else f"k{rng.integers(0, 12)}" for _ in range(1000)]
    frame = DeviceFrame.from_arrow(pa.table({"s": pa.array(vals), "x": pa.array(np.arange(1000))}))
    for s in ["k3", "k0", "k11", "absent", ""]:
        _check_filter(frame, lambda d: d["s"] == s, f"== {s}")
        _check_filter(frame, lambda d: d["s"] != s, f"!= {s}")
        _check_filter(frame, lambda d: s == d.s, f"{s} ==")
    for bad in [lambda d: d["s"] < "k3", lambda d: d["s"] == d["s"], lambda d: d["s"] == 3,
                lambda d: d["x"] == "k3"]:
        with pytest.raises(TypeError):
            _filter(frame, bad)


def test_compare_list_raises():
    frame = _kinds_frame(64, 4)
    with pytest.raises(TypeError):
        _filter(frame, lambda d: d["l"] == 1)
    with pytest.raises(OverflowError):
        _filter(frame, lambda d: d["i32"] < 2 ** 64)


def test_null_tests_and_mask_logic():
    frame = _numeric_frame(5000, 5)
    preds = [
        lambda d: d["f32"].isnull(), lambda d: d.f64.isna(), lambda d: d["i32"].notnull(), lambda d: d.bool.notna(),
        lambda d: (d["i32"] > 0) & (d["f32"] < 2.5), lambda d: (d["i32"] > 0) | d["f64"].isnull(),
        lambda d: (d["i64"] == 3) ^ (d["f32"] != 0.0), lambda d: ~(d["i32"] > 0), lambda d: ~d["f32"].isnull(),
        lambda d: d["flag"], lambda d: d["flag"] & (d["i32"] < 0), lambda d: ~d["flag"], lambda d: d.flag ^ d.flag,
        lambda d: d[d["i32"] >= 2], lambda d: d[d["flag"]], lambda d: d, lambda d: d[["i32", "f32"]],
        lambda d: d[d["i32"] > 0][["f32", "i32"]],
    ]
    for k, p in enumerate(preds):
        _check_filter(frame, p, f"pred {k}")
    # a bool column with nulls selects its true rows: a null counts as false
    got = _filter(frame, lambda d: d["bool"]).to_pandas()
    _same(got, filter_frame(frame.to_pandas(), lambda d: d["bool"] == 1), "bool column with nulls")
    with pytest.raises(ValueError):
        _filter(frame, lambda d: d["i32"])
    with pytest.raises(ValueError):
        _filter(frame, lambda d: 3)


# ---------------------------------------------------------------------------- sizes, kinds
SIZES = [0, 1, 7, 8, 9, 63, 64, 65, 2047, 2048, 2049, 10 ** 6 + 3]


def _pattern(kind, n, rng):
    if kind == "all":
        return np.ones(n, bool)
    if kind == "none":
        return np.zeros(n, bool)
    if kind == "alternating":
        return np.arange(n) % 2 == 0
    if kind == "random":
        return rng.random(n) < 0.5
    runs = np.repeat(rng.random(n // 500 + 1) < 0.5, 500)[:n]        # long runs
    return runs


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("pattern", ["all", "none", "alternating", "random", "runs"])
def test_sizes_and_patterns(n, pattern):
    rng = np.random.default_rng(n + len(pattern))
    frame = _kinds_frame(n, n, lists=n <= 2049)
    frame["p"] = Column.from_numpy(_pattern(pattern, n, rng), device="cuda")
    got = _check_filter(frame, lambda d: d["p"], f"{n} {pattern}")
    if pattern == "all":
        assert all(got[c] is frame[c] for c in frame.columns)
    if pattern == "none":
        assert len(got) == 0
        for c in frame.columns:
            assert got[c].data.dtype == frame[c].data.dtype and got[c].is_bool == frame[c].is_bool
            assert (got[c].dictionary is None) == (frame[c].dictionary is None)
            if frame[c].is_list:
                assert got[c].offsets.tolist() == [0]
    _check_filter(frame, lambda d: d["i32"] > 0, f"{n} i32 > 0")


def test_mask_rows_of_2_31_plus_65():
    n = (1 << 31) + 65
    hits = [0, 5, (1 << 31) - 1, 1 << 31, (1 << 31) + 64]
    data = torch.zeros(n, dtype=torch.uint8, device="cuda")
    data[torch.tensor(hits, device="cuda")] = torch.tensor([1, 2, 3, 4, 5], dtype=torch.uint8, device="cuda")
    col = Column(data)
    mask = engine.mask_compare(col, None, engine.CMP_GT, 1, 0, n)
    kept, tile_off = engine.mask_count(mask, n)
    assert kept == len(hits)
    assert engine.mask_select(mask, n, tile_off, kept).tolist() == hits
    del mask, tile_off
    out = _filter(DeviceFrame({"u": col}), lambda d: d["u"] > 0)
    assert out["u"].data.tolist() == [1, 2, 3, 4, 5]


# ------------------------------------------------------------------------ pass-through
def test_keep_all_passes_the_buffers_through():
    frame = _kinds_frame(4000, 6)
    out = _filter(frame, lambda d: d["i32"] > -10 ** 6)
    for c in frame.columns:
        assert out[c].data.data_ptr() == frame[c].data.data_ptr()
        if frame[c].validity is not None:
            assert out[c].validity.data_ptr() == frame[c].validity.data_ptr()
    out = ops.Dropna().transform(ColumnSelector(["f64", "i32"]), frame)
    assert out["f64"].data.data_ptr() == frame["f64"].data.data_ptr()


def test_dropna_without_nulls_launches_nothing():
    frame = DeviceFrame.from_pandas(pd.DataFrame({"a": np.arange(100), "b": np.arange(100, dtype=np.int32)}))
    before = engine.kernel_launches
    out = ops.Dropna().transform(ColumnSelector(["a", "b"]), frame)
    assert engine.kernel_launches == before
    assert out["a"] is frame["a"] and out["b"] is frame["b"]


# --------------------------------------------------------------------------------- Dropna
@pytest.mark.parametrize("subset", [["i64n"], ["f32n", "f64"], ["s", "bool"], ["i32", "u8", "l", "ls"],
                                    ["i64n", "f32n", "bool", "s", "l"]])
def test_dropna_subsets(subset):
    frame = _kinds_frame(3000, 7)
    got = ops.Dropna().transform(ColumnSelector(subset), frame).to_pandas()
    _same(got, dropna_frame(frame.to_pandas()[subset], subset), str(subset))


def test_dropna_many_columns_and_lists_never_drop():
    rng = np.random.default_rng(8)
    n = 1000
    cols = {f"c{k}": pa.array(rng.normal(size=n), mask=rng.random(n) < 0.01) for k in range(20)}
    cols["l"] = pa.array([None if k % 3 == 0 else [k] for k in range(n)], type=pa.list_(pa.int64()))
    frame = DeviceFrame.from_arrow(pa.table(cols))
    got = ops.Dropna().transform(ColumnSelector(list(cols)), frame).to_pandas()
    _same(got, dropna_frame(frame.to_pandas()), "20 columns")
    only_list = ops.Dropna().transform(ColumnSelector(["l"]), frame)
    assert len(only_list) == n


def test_dropna_drops_a_device_made_nan():
    df = pd.DataFrame({"x": np.array([1.0, -2.0, 3.0, -2.0, 0.5] * 20, dtype=np.float32)})
    logged = nvt.Workflow(["x"] >> ops.LogOp())
    want = dropna_frame(logged.fit_transform(nvt.Dataset(df)).to_ddf().compute())
    wf = nvt.Workflow(["x"] >> ops.LogOp() >> ops.Dropna())
    got = wf.fit_transform(nvt.Dataset(df)).to_ddf().compute()
    assert len(got) == 60
    _same(got, want, "LogOp of -2")


# ------------------------------------------------------------------- reference scenarios
def test_reference_test_filter():
    """reference tests/unit/ops/test_ops.py::test_filter"""
    rng = np.random.default_rng(9)
    df = pd.DataFrame({"x": rng.normal(size=2000), "y": rng.random(2000), "id": np.arange(2000)})
    ds = nvt.Dataset(df, npartitions=3)
    for f in [lambda d: d[d["y"] > 0.5], lambda d: d["y"] > 0.5]:
        got = nvt.Workflow(["x", "y"] >> ops.Filter(f=f)).fit_transform(ds).to_ddf().compute()
        _same(got.reset_index(drop=True), filter_frame(df[["x", "y"]], f), "y > 0.5")
    df.loc[df.index[::5], "x"] = np.nan
    ds = nvt.Dataset(df, npartitions=3)
    for f in [lambda d: d[d.x.isnull()], lambda d: d.x.isnull()]:
        got = nvt.Workflow(["x", "y"] >> ops.Filter(f=f)).fit_transform(ds).to_ddf().compute()
        _same(got.reset_index(drop=True), filter_frame(df[["x", "y"]], f), "isnull")
        assert 0 < len(got) < len(df)
    wf = nvt.Workflow(["x", "y"] >> ops.Filter(f=lambda d: "some invalid value"))
    wf.fit(ds)
    with pytest.raises(ValueError):
        wf.transform(ds).to_ddf().compute()


def test_reference_test_filtered_partition(tmp_path):
    """reference tests/unit/test_dask_nvt.py::test_filtered_partition: the last partitions empty"""
    df = pd.DataFrame({"col": range(100)})
    wf = nvt.Workflow(["col"] >> ops.Filter(lambda d: d["col"] < 55))
    out = wf.transform(nvt.Dataset(df, npartitions=5))
    lens = [len(p) for p in out.partitions()]
    assert lens == [20, 20, 15, 0, 0]
    out.to_parquet(str(tmp_path / "out"))
    back = pd.read_parquet(str(tmp_path / "out"))
    assert back["col"].tolist() == list(range(55))


def test_transformers4rec_session_filter():
    """the reference's Transformers4Rec ETL (tests/unit/test_tf4rec.py): Groupby, ListSlice, then
    Filter(item_id_count >= 2)"""
    rng = np.random.default_rng(10)
    n = 20_000
    df = pd.DataFrame({"session_id": rng.integers(0, 6000, n), "item_id": rng.integers(0, 500, n).astype(np.int32),
                       "ts": rng.integers(0, 1 << 30, n)})
    groups = ["session_id", "item_id", "ts"] >> ops.Groupby("session_id", sort_cols="ts",
                                                            aggs={"item_id": ["list", "count"]})
    trim = groups["item_id_list"] >> ops.ListSlice(-5)
    selected = groups[["session_id", "item_id_count"]] + trim
    wf = nvt.Workflow(selected >> ops.Filter(f=lambda d: d["item_id_count"] >= 2))
    got = wf.fit_transform(nvt.Dataset(df)).to_ddf().compute()
    unf = nvt.Workflow(selected).fit_transform(nvt.Dataset(df)).to_ddf().compute()
    want = filter_frame(unf, lambda d: d["item_id_count"] >= 2)
    _same(got, want, "tf4rec")
    assert len(want) < len(unf) and (got["item_id_count"] >= 2).all()
    assert wf.output_schema["item_id_list"].properties["value_count"] == {"min": 0, "max": 5}


# -------------------------------------------------------------------- fit through a filter
def _fit_frame():
    rng = np.random.default_rng(11)
    n = 4000
    return pd.DataFrame({"a": rng.integers(0, 50, n), "b": rng.normal(size=n), "x": rng.normal(size=n),
                         "t": rng.integers(0, 2, n).astype(np.float64), "k": rng.integers(0, 30, n)})


def _pred(d):
    return (d["a"] < 40) & (d["k"] < 1000)


def _emptied(df):
    """4 partitions; the predicate also empties the third one"""
    parts = [df.iloc[i:i + 1000].reset_index(drop=True) for i in range(0, 4000, 1000)]
    parts[2] = parts[2].assign(a=parts[2]["a"] + 100)
    return parts


def _compare_fit(make, cols, tmp_path, rtol=0.0):
    """fit `make(cols >> Filter(_pred))` on partitions the filter shrinks and empties, and the same
    graph without the filter on the partitions filtered by the oracle: the fitted state shows in
    every transformed partition.  rtol: statistics summed in fp64 by the group-by, whose order of
    additions differs between the two fits"""
    df = _fit_frame()
    parts = _emptied(df)
    filt = cols >> ops.Filter(f=_pred)
    wf = nvt.Workflow(make(filt, str(tmp_path / "a")))
    wf.fit(nvt.Dataset(parts))
    pre = [filter_frame(p[cols], _pred) for p in parts]
    assert len(pre[2]) == 0
    ref = nvt.Workflow(make(Node.construct_from(cols), str(tmp_path / "b")))
    ref.fit(nvt.Dataset([p for p in pre if len(p)]))
    for p, q in zip(parts, pre):
        got = wf.transform(DeviceFrame.from_pandas(p)).to_pandas()
        want = ref.transform(DeviceFrame.from_pandas(q)).to_pandas() if len(q) else None
        if want is None:
            assert len(got) == 0
        else:
            _same(got, want, "fit through filter", rtol)
    return wf, pd.concat(pre, ignore_index=True)


def test_fit_categorify_through_filter(tmp_path):
    wf, pre = _compare_fit(lambda n, p: n[["a", "k"]] >> ops.Categorify(out_path=p), ["a", "k", "b"], tmp_path)
    out = wf.transform(nvt.Dataset(_emptied(_fit_frame()))).to_ddf().compute()
    want = CategorifyOracle(["a", "k"]).fit(pre).transform(pre)
    for c in ["a", "k"]:
        np.testing.assert_array_equal(out[c].to_numpy(), want[c].to_numpy())


def test_fit_normalize_through_filter(tmp_path):
    wf, pre = _compare_fit(lambda n, p: n[["b", "x"]] >> ops.Normalize(), ["a", "k", "b", "x"], tmp_path)
    op = [n.op for n in wf.output_node.topo_order() if n.kind == "op" and isinstance(n.op, ops.Normalize)][0]
    means, stds = normalize_fit(pre, ["b", "x"])
    for c in ["b", "x"]:
        np.testing.assert_allclose(op.means[c], means[c], rtol=1e-12)
        np.testing.assert_allclose(op.stds[c], stds[c], rtol=1e-12)


def test_fit_join_groupby_and_target_encoding_through_filter(tmp_path):
    _compare_fit(lambda n, p: n[["a"]] >> ops.JoinGroupby(cont_cols=n[["x"]], stats=["count", "sum"], out_path=p),
                 ["a", "k", "x"], tmp_path / "jg", rtol=1e-12)
    _compare_fit(lambda n, p: n[["a"]] >> ops.TargetEncoding(n[["t"]], p_smooth=5, out_path=p),
                 ["a", "k", "t"], tmp_path / "te", rtol=1e-12)


def test_join_external_through_filter_and_groupby_keys_from_the_dataset(tmp_path):
    # Groupby reads its keys as a dependency from the dataset: after a Filter they have other rows
    wf = nvt.Workflow(["a", "x"] >> ops.Filter(f=lambda d: d["a"] < 40) >> ops.Groupby("a", aggs={"x": ["sum"]}))
    with pytest.raises(ValueError, match="different row counts"):
        wf.fit_transform(nvt.Dataset(_fit_frame())).to_ddf().compute()
    ext = pd.DataFrame({"k": np.arange(0, 30, 2), "label": np.arange(15) * 1.5})
    _compare_fit(lambda n, p: n >> ops.JoinExternal(ext, on="k", how="inner"), ["a", "k"], tmp_path / "je")


# -------------------------------------------------------------------------- save / load
def test_save_load_in_a_fresh_process(tmp_path):
    df = pd.DataFrame({"a": np.arange(200) % 70, "b": np.where(np.arange(200) % 7 == 0, np.nan, 1.5)})
    wf = nvt.Workflow((["a", "b"] >> ops.Filter(f=keep_small)) >> ops.Dropna())
    wf.fit(nvt.Dataset(df))
    wf.save(str(tmp_path / "wf"))
    want = wf.transform(nvt.Dataset(df)).to_ddf().compute()
    df.to_parquet(tmp_path / "in.parquet")
    code = (f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]\n"
            "import nvtabular as nvt, pandas as pd\n"
            f"wf = nvt.Workflow.load({str(tmp_path / 'wf')!r})\n"
            f"out = wf.transform(nvt.Dataset(pd.read_parquet({str(tmp_path / 'in.parquet')!r}))).to_ddf().compute()\n"
            f"out.to_parquet({str(tmp_path / 'out.parquet')!r})\n")
    subprocess.run([sys.executable, "-c", code], check=True, cwd=str(tmp_path))
    got = pd.read_parquet(tmp_path / "out.parquet")
    assert 0 < len(want) < len(df)
    pd.testing.assert_frame_equal(got.reset_index(drop=True), want.reset_index(drop=True), check_exact=True)


def test_bit_identical_from_run_to_run():
    frame = _kinds_frame(100_003, 12)

    def run():
        out = _filter(frame, lambda d: (d["i32"] > 0) | d["f32n"].isnull())
        out2 = ops.Dropna().transform(ColumnSelector(frame.columns), frame)
        bufs = []
        for o in (out, out2):
            for c in o.columns:
                bufs += [t.clone() for t in (o[c].data, o[c].validity, o[c].offsets) if t is not None]
        return bufs

    first = run()
    for _ in range(2):
        again = run()
        assert len(again) == len(first)
        assert all(torch.equal(x, y) for x, y in zip(first, again))
