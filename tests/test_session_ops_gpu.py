"""ListSlice and DifferenceLag on the GPU (csrc/session.cu, K10, and the sub-list copy of
csrc/groupby.cu) against the oracle (oracle/session_ops.py), exactly: every leaf dtype with leaf
nulls, empty lists and null list rows, a start / end grid with and without pad, n = 0, one list
longer than 2^16 among a million short ones, every value and key kind over several shifts and
partitions, int64 values above 2^53, the session pipeline end to end, and run-to-run bit identity."""
import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.parquet as pq
import pytest
import torch

import nvtabular as nvt
from nvtabular import ColumnSelector, ops
from nvtabular_b200.column import Column, DeviceFrame, pack_validity, unpack_validity
from oracle.categorify import CategorifyOracle
from oracle.session_ops import difference_lag as oracle_lag
from oracle.session_ops import list_slice as oracle_slice

pytestmark = pytest.mark.gpu

LEAF_TYPES = {"int32": pa.int32(), "int64": pa.int64(), "float32": pa.float32(), "float64": pa.float64(),
              "bool": pa.bool_(), "string": pa.string()}
PAD = {"int32": -1, "int64": -(2 ** 40), "float32": -1.5, "float64": 2.25, "bool": True, "string": 0}
STARTS = [-15, -5, -1, 0, 1, 3, 20]
ENDS = [None, -7, -1, 0, 2, 5, 30]
SHIFTS = [1, -1, 3, -7, 1000]


# --------------------------------------------------------------------------------- helpers
def _py(v):
    return v.item() if isinstance(v, np.generic) else v


def _rows(col: Column):
    """the exact host rows of a list Column (None = a null leaf)"""
    vals, mask = col.to_numpy()
    if col.dictionary is not None:
        vals = np.array([col.dictionary[v] for v in vals], dtype=object) if len(vals) else vals
    off = col.offsets.cpu().numpy()
    return [[None if mask is not None and mask[k] else _py(vals[k]) for k in range(off[i], off[i + 1])]
            for i in range(len(off) - 1)]


def _eq(a, b):
    if a is None or b is None:
        return a is None and b is None
    if isinstance(a, float) and isinstance(b, float) and np.isnan(a):
        return bool(np.isnan(b))
    return a == b


def _same_rows(got, want, ctx):
    assert len(got) == len(want), ctx
    for i, (g, w) in enumerate(zip(got, want)):
        assert len(g) == len(w) and all(_eq(a, b) for a, b in zip(g, w)), (ctx, i, g, w)


def _leaf(kind, rng):
    if kind in ("int32", "int64"):
        return int(rng.integers(-1000, 1000))
    if kind in ("float32", "float64"):
        if rng.random() < 0.05:
            return float("nan")
        v = float(rng.normal())
        return float(np.float32(v)) if kind == "float32" else v
    if kind == "bool":
        return bool(rng.random() < 0.5)
    return f"s{rng.integers(0, 20)}"


def _list_rows(kind, n, seed):
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(n):
        if rng.random() < 0.05:
            rows.append(None)
            continue
        rows.append([None if rng.random() < 0.1 else _leaf(kind, rng) for _ in range(int(rng.integers(0, 13)))])
    return rows


@pytest.fixture(scope="module")
def list_tables():
    return {kind: _list_rows(kind, 300, 7 + i) for i, kind in enumerate(LEAF_TYPES)}


def _frame(rows, kind):
    return DeviceFrame.from_arrow(pa.table({"x": pa.array(rows, type=pa.list_(LEAF_TYPES[kind]))}))


def _snapshot(col):
    return [t.clone() for t in (col.data, col.offsets, col.validity) if t is not None]


def _same_bits(a, b):
    """bitwise equality (torch.equal says NaN != NaN)"""
    return torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


# ------------------------------------------------------------------------------- ListSlice
@pytest.mark.parametrize("kind", list(LEAF_TYPES))
def test_list_slice_grid_matches_oracle(list_tables, kind):
    rows = list_tables[kind]
    frame = _frame(rows, kind)
    col = frame["x"]
    before = _snapshot(col)
    for start in STARTS:
        for end in ENDS:
            for pad in (False, True):
                if pad and kind == "string":
                    continue
                try:
                    op = ops.ListSlice(start, end, pad=pad, pad_value=PAD[kind])
                except ValueError:
                    assert pad
                    continue
                got = op.transform(ColumnSelector(["x"]), frame)["x"]
                assert got.data.dtype == col.data.dtype and got.is_bool == col.is_bool
                if pad:
                    L = op.max_elements
                    assert got.offsets.cpu().tolist() == [i * L for i in range(len(rows) + 1)]
                want = oracle_slice(rows, start, end, pad=pad, pad_value=PAD[kind])
                _same_rows(_rows(got), want, (kind, start, end, pad))
    # the operator never writes its input
    assert all(_same_bits(a, b) for a, b in zip(before, _snapshot(col)))


def test_list_slice_string_leaves_through_workflow():
    rows = _list_rows("string", 500, 3)
    df = pa.table({"x": pa.array(rows, type=pa.list_(pa.string()))}).to_pandas()
    wf = nvt.Workflow(["x"] >> ops.ListSlice(-3))
    wf.fit(nvt.Dataset(df))
    got = wf.transform(DeviceFrame.from_arrow(pa.table({"x": pa.array(rows, type=pa.list_(pa.string()))})))
    _same_rows(_rows(got["x"]), oracle_slice(rows, -3), "string")


@pytest.mark.parametrize("kind", ["int64", "float32", "bool", "string"])
def test_list_slice_empty_frames_and_all_empty_rows(kind):
    for rows in ([], [[], None, []]):
        frame = _frame(rows, kind)
        for op in (ops.ListSlice(-2), ops.ListSlice(1, 3)) + (
                () if kind == "string" else (ops.ListSlice(2, pad=True, pad_value=PAD[kind]),)):
            got = op.transform(ColumnSelector(["x"]), frame)["x"]
            assert got.nrows == len(rows)
            _same_rows(_rows(got), oracle_slice(rows, op.start, op.end, op.pad, PAD[kind]), (kind, len(rows)))


def test_list_slice_null_rows_from_parquet(tmp_path):
    rows = _list_rows("int64", 2000, 11)
    pq.write_table(pa.table({"x": pa.array(rows, type=pa.list_(pa.int64()))}), tmp_path / "l.parquet",
                   row_group_size=700)
    for op in (ops.ListSlice(-4, pad=True, pad_value=-1), ops.ListSlice(2, -1)):
        wf = nvt.Workflow(["x"] >> op)
        ds = nvt.Dataset(str(tmp_path / "l.parquet"))
        wf.fit(ds)
        got = []
        for part in ds.partitions():
            got += _rows(wf.transform(part)["x"])
        _same_rows(got, oracle_slice(rows, op.start, op.end, op.pad, -1), str(op.start))


def _np_slice(off, start, end, pad, L):
    """vectorised restatement of row[start:end] (+ pad) over offsets: -> (leaf index, keep, offsets)"""
    lens = np.diff(off)
    s = np.minimum(np.maximum(start + lens if start < 0 else np.full_like(lens, start), 0), lens)
    e = np.minimum(np.maximum(end + lens if end < 0 else np.full_like(lens, end), 0), lens)
    e = np.maximum(e, s)
    lo, cnt = off[:-1] + s, e - s
    if not pad:
        new_off = np.concatenate([[0], np.cumsum(cnt)])
        idx = np.repeat(lo - new_off[:-1], cnt) + np.arange(new_off[-1])
        return idx, np.ones(len(idx), dtype=bool), new_off
    n = len(lens)
    r = np.repeat(np.arange(n), L)
    k = np.tile(np.arange(L), n)
    keep = k < cnt[r]
    return np.where(keep, lo[r] + k, 0), keep, np.arange(n + 1) * L


def test_list_slice_one_long_list_among_a_million():
    n = 1_000_000
    g = torch.Generator(device="cuda")
    g.manual_seed(5)
    lens = torch.randint(0, 6, (n,), generator=g, device="cuda", dtype=torch.int64)
    lens[n // 2] = 70_000                                        # one list longer than 2^16
    off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    off[1:] = torch.cumsum(lens, 0)
    total = int(off[-1].item())
    leaves = torch.randint(-(1 << 40), 1 << 40, (total,), generator=g, device="cuda", dtype=torch.int64)
    valid = torch.rand(total, generator=g, device="cuda") < 0.9
    for validity in (None, pack_validity(valid)):
        col = Column(leaves, validity, off)
        frame = DeviceFrame({"x": col})
        off_h, leaves_h = off.cpu().numpy(), leaves.cpu().numpy()
        valid_h = valid.cpu().numpy() if validity is not None else np.ones(total, dtype=bool)
        for start, end, pad in [(-20, None, True), (-20, None, False), (3, 69_990, False), (0, 8, True),
                                (-70_005, -3, False)]:
            op = ops.ListSlice(start, end, pad=pad, pad_value=-7)
            got = op.transform(ColumnSelector(["x"]), frame)["x"]
            idx, keep, new_off = _np_slice(off_h, op.start, op.end, pad, op.max_elements)
            assert np.array_equal(got.offsets.cpu().numpy(), new_off)
            want = np.where(keep, leaves_h[idx], -7)
            assert np.array_equal(got.data.cpu().numpy(), want), (start, end, pad)
            want_valid = np.where(keep, valid_h[idx], True)
            got_valid = unpack_validity(got.validity, got.data.numel()).cpu().numpy() \
                if got.validity is not None else np.ones(len(want), dtype=bool)
            assert np.array_equal(got_valid, want_valid), (start, end, pad)
            if validity is None:
                assert got.validity is None
            # the vectorised restatement is the oracle on the long row and its neighbours
            sub = [list(leaves_h[off_h[i]:off_h[i + 1]]) for i in range(n // 2 - 3, n // 2 + 3)]
            got_sub = [list(got.data[new_off[i]:new_off[i + 1]].cpu().numpy()) for i in range(n // 2 - 3, n // 2 + 3)]
            assert got_sub == oracle_slice(sub, op.start, op.end, pad, -7)


# --------------------------------------------------------------------------- DifferenceLag
def _lag_frame(n, seed):
    rng = np.random.default_rng(seed)
    k = np.sort(rng.integers(0, max(n // 6, 1), n))
    kf = (k % 5).astype(np.float64)
    kf[(kf == 0) & (rng.random(n) < 0.5)] = -0.0
    kf[rng.random(n) < 0.02] = np.nan
    ks = pd.Series([f"u{v % 7}" for v in k], dtype=object)
    ks[rng.random(n) < 0.02] = None
    ki = pd.Series(k, dtype="Int64")
    ki[rng.random(n) < 0.02] = pd.NA
    v_null = pd.Series(rng.integers(-1000, 1000, n), dtype="Int64")
    v_null[rng.random(n) < 0.1] = pd.NA
    f32 = rng.normal(size=n).astype(np.float32)
    f32[rng.random(n) < 0.05] = np.nan
    f64 = rng.normal(size=n) * 1e6
    f64[rng.random(n) < 0.05] = np.nan
    f64[rng.random(n) < 0.05] = -0.0
    return pd.DataFrame({
        "k": k.astype(np.int64), "kf": kf, "ks": ks, "ki": ki, "kb": (k % 3) == 0, "k32": (k % 4).astype(np.int32),
        "v_i32": rng.integers(-(1 << 30), 1 << 30, n).astype(np.int32),
        "v_i64": rng.integers(-(1 << 62), 1 << 62, n).astype(np.int64),
        "v_u8": rng.integers(0, 256, n).astype(np.uint8),
        "v_f32": f32, "v_f64": f64, "v_null": v_null,
    })


VALUES = ["v_i32", "v_i64", "v_u8", "v_f32", "v_f64", "v_null"]


def _same_f32(a, b, ctx):
    a = np.asarray(a, dtype=np.float32)
    b = np.asarray(b, dtype=np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    assert np.array_equal(na, nb), ctx
    assert np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32)), ctx


@pytest.mark.parametrize("keys", [["k"], ["ki"], ["kf"], ["ks"], ["kb"], ["ki", "ks"], ["k32", "kf", "ks", "kb"]])
def test_difference_lag_matches_oracle_over_partitions(keys):
    df = _lag_frame(20_000, 13)
    nparts = 3
    wf = nvt.Workflow(VALUES >> ops.DifferenceLag(keys, shift=SHIFTS))
    ds = nvt.Dataset(df, npartitions=nparts)
    wf.fit(ds)
    got = wf.transform(ds).to_ddf().compute()
    chunk = -(-len(df) // nparts)
    want = pd.concat([oracle_lag(df.iloc[s:s + chunk].reset_index(drop=True), VALUES, keys, SHIFTS)
                      for s in range(0, len(df), chunk)], ignore_index=True)
    assert list(got.columns) == list(want.columns)
    for c in want.columns:
        assert got[c].dtype == np.float32
        _same_f32(got[c].to_numpy(dtype=np.float32, na_value=np.nan), want[c].to_numpy(), (keys, c))


def test_difference_lag_int64_above_2_53_and_edge_cases():
    df = pd.DataFrame({"k": [1, 1, 1, 2, 2], "x": np.array([2 ** 60 + 1, 2 ** 60 + 3, -(2 ** 62), 7, np.iinfo(np.int64).max],
                                                             dtype=np.int64)})
    wf = nvt.Workflow(["x"] >> ops.DifferenceLag("k", shift=[1, 0, -1, 1000, -1000]))
    wf.fit(nvt.Dataset(df))
    got = wf.transform(df)
    want = oracle_lag(df, ["x"], "k", [1, 0, -1, 1000, -1000])
    assert got["x_difference_lag_1"][1] == 2.0
    for c in want.columns:
        _same_f32(got[c].to_numpy(dtype=np.float32, na_value=np.nan), want[c].to_numpy(), c)
    empty = df.iloc[:0]
    out = ops.DifferenceLag("k", shift=[1, -1]).transform(ColumnSelector(["x"]), DeviceFrame.from_pandas(empty))
    assert [len(out[c]) for c in out.columns] == [0, 0]


def test_difference_lag_reference_example():
    """reference tests/unit/ops/test_ops.py::test_difference_lag on the GPU"""
    df = pd.DataFrame({"userid": [0, 0, 0, 1, 1, 2], "timestamp": [1000, 1005, 1100, 2000, 2001, 3000]})
    wf = nvt.Workflow(["timestamp"] >> ops.DifferenceLag(partition_cols=["userid"], shift=[1, -1]))
    out = wf.fit_transform(nvt.Dataset(df)).to_ddf().compute()
    want = oracle_lag(df, ["timestamp"], ["userid"], [1, -1])
    for c in want.columns:
        _same_f32(out[c].to_numpy(dtype=np.float32, na_value=np.nan), want[c].to_numpy(), c)


# ------------------------------------------------------------------------- the pipeline
def _sessions(n, seed):
    rng = np.random.default_rng(seed)
    sid = np.sort(rng.integers(0, n // 8, n)).astype(np.int64)
    ts = rng.integers(1_700_000_000, 1_700_000_000 + (1 << 20), n).astype(np.int64)
    df = pd.DataFrame({"session_id": sid, "item_id": rng.integers(0, 500, n).astype(np.int32), "ts": ts})
    return df.sort_values(["session_id", "ts"], kind="stable").reset_index(drop=True)


def test_reference_session_snippet_through_fit_transform():
    df = _sessions(30_000, 17)
    lags = ["ts"] >> ops.DifferenceLag("session_id", shift=[1, -1])
    seqs = ["session_id", "item_id", "ts"] >> ops.Groupby("session_id", sort_cols="ts",
                                                          aggs={"item_id": ["list", "count"]})
    trunc = seqs["item_id_list"] >> ops.ListSlice(-20, pad=True)
    got_lags = nvt.Workflow(lags).fit_transform(nvt.Dataset(df)).to_ddf().compute()
    want = oracle_lag(df, ["ts"], "session_id", [1, -1])
    for c in want.columns:
        _same_f32(got_lags[c].to_numpy(dtype=np.float32, na_value=np.nan), want[c].to_numpy(), c)
    wf = nvt.Workflow(trunc)
    out = wf.fit_transform(nvt.Dataset(df)).to_ddf().compute()
    got = [[int(v) for v in r] for r in out["item_id_list"]]
    lists = [g["item_id"].tolist() for _, g in df.groupby("session_id", sort=True)]
    _same_rows(got, oracle_slice(lists, -20, pad=True), "snippet")
    assert wf.output_schema["item_id_list"].properties["value_count"] == {"min": 20, "max": 20}


def test_chain_shuffle_lag_groupby_slice_categorify():
    df = _sessions(40_000, 23)
    ds = nvt.Dataset(df, npartitions=2).shuffle_by_keys("session_id", npartitions=3)
    lags = ["ts"] >> ops.DifferenceLag("session_id", shift=1)
    feats = (["session_id", "item_id", "ts"] + lags) >> ops.Groupby(
        "session_id", sort_cols="ts", aggs={"item_id": ["list"], "ts_difference_lag_1": ["list"]})
    k = 6
    out = feats["item_id_list"] >> ops.ListSlice(-k, pad=True) >> ops.Categorify()
    wf = nvt.Workflow(out + feats["ts_difference_lag_1_list"])
    wf.fit(ds)
    got_items, got_lags, parts = [], [], []
    for part in ds.partitions():
        res = wf.transform(part)
        got_items += _rows(res["item_id_list"])
        got_lags += _rows(res["ts_difference_lag_1_list"])
        p = part.to_pandas()
        lag = oracle_lag(p, ["ts"], "session_id", 1)["ts_difference_lag_1"].to_numpy()
        p = p.assign(lag=lag)
        groups = [g for _, g in p.groupby("session_id", sort=True)]
        parts.append(pd.DataFrame({"item_id_list": oracle_slice([g.sort_values("ts", kind="stable")["item_id"].tolist()
                                                                 for g in groups], -k, pad=True)}))
        want_lags = [[None if np.isnan(v) else float(v) for v in g.sort_values("ts", kind="stable")["lag"]]
                     for g in groups]
        _same_rows(_rows(res["ts_difference_lag_1_list"]), want_lags, "lag lists")
    cat = CategorifyOracle(["item_id_list"]).fit(parts)
    want_items = []
    for p in parts:
        want_items += [list(map(int, r)) for r in cat.transform(p)["item_id_list"]]
    _same_rows(got_items, want_items, "categorified")
    assert all(len(r) == k for r in got_items)
    sizes = nvt.ops.get_embedding_sizes(wf)
    assert isinstance(sizes, dict) and "item_id_list" in sizes       # fixed-length: not multi-hot


def test_bit_identical_from_run_to_run():
    df = _lag_frame(50_000, 29)
    frame = DeviceFrame.from_pandas(df)
    rows = _list_rows("float64", 5000, 31)
    lists = _frame(rows, "float64")

    def run():
        lag = ops.DifferenceLag(["ki", "ks"], shift=[1, -3]).transform(ColumnSelector(VALUES), frame)
        a = ops.ListSlice(-4, pad=True, pad_value=0.5).transform(ColumnSelector(["x"]), lists)["x"]
        b = ops.ListSlice(1, -1).transform(ColumnSelector(["x"]), lists)["x"]
        bufs = [lag[c].data for c in lag.columns] + [lag[c].validity for c in lag.columns]
        return [t.clone() for t in bufs + [a.data, a.validity, a.offsets, b.data, b.validity, b.offsets]]

    first = run()
    for _ in range(2):
        assert all(_same_bits(x, y) for x, y in zip(first, run()))
