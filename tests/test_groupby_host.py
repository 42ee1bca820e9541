"""Groupby without a GPU: the oracle's rules on hand-computed answers, the output schema, the
argument errors, the LSD round planner and a save / load round trip."""
import json
import math
import os

import numpy as np
import pandas as pd
import pytest

import nvtabular_b200 as nvt
from nvtabular_b200.graph import ColumnSchema, Schema, Tags
from nvtabular_b200.ops.groupby import plan_rounds
from oracle.session_groupby import session_groupby

NaN = float("nan")


def _eq(a, b):
    if isinstance(a, float) and isinstance(b, float) and math.isnan(a) and math.isnan(b):
        return True
    return a == b


def test_oracle_groups_sort_and_first_last():
    df = pd.DataFrame({"s": [2, 1, 2, 1, 2, None, 1],
                       "ts": [30.0, 5.0, 10.0, NaN, 20.0, 1.0, 5.0],
                       "x": [1, 2, 3, 4, 5, 6, 7]})
    df["s"] = df["s"].astype("Int64")
    up = session_groupby(df, "s", "ts", {"x": ["list", "first", "last"]})
    assert up["s"] == [1, 2]                                   # null key dropped, keys ascending
    assert up["x_list"] == [[2, 7, 4], [3, 5, 1]]              # NaN ts last, tie 5.0 keeps input order
    assert up["x_first"] == [2, 3] and up["x_last"] == [4, 1]
    down = session_groupby(df, "s", "ts", {"x": ["list", "first", "last"]}, ascending=False)
    assert down["s"] == [1, 2]                                 # ascending never reverses the groups
    assert down["x_list"] == [[2, 7, 4], [1, 5, 3]]            # NaN still last; ties keep input order
    # the reference's swap: with ascending=False `first` is the LAST element of the list
    assert down["x_first"] == [4, 3] and down["x_last"] == [2, 1]


def test_oracle_no_sort_cols_keeps_input_order_and_zero_keys():
    df = pd.DataFrame({"k": [0.0, -0.0, NaN, 1.0, -0.0], "v": [1, 2, 3, 4, 5]})
    out = session_groupby(df, ["k"], None, {"v": ["list", "count"]})
    assert out["k"] == [0.0, 1.0] and all(math.copysign(1, k) == 1 for k in out["k"])
    assert out["v_list"] == [[1, 2, 5], [4]]
    assert out["v_count"] == [3, 1]


def test_oracle_null_rules():
    df = pd.DataFrame({"k": [1, 1, 1, 2, 2, 3],
                       "v": pd.array([None, None, None, 4.0, 4.0, 7.0], dtype="Float64")})
    out = session_groupby(df, "k", None, {"v": ["count", "sum", "mean", "min", "max", "var", "std",
                                                "median", "nunique", "list", "first"]})
    assert out["v_count"] == [0, 2, 1]
    assert out["v_sum"] == [0.0, 8.0, 7.0]                     # sum of an all-null group is 0
    assert math.isnan(out["v_mean"][0]) and out["v_mean"][1:] == [4.0, 7.0]
    assert out["v_min"] == [None, 4.0, 7.0] and out["v_max"] == [None, 4.0, 7.0]
    assert math.isnan(out["v_var"][0]) and out["v_var"][1] == 0.0 and math.isnan(out["v_var"][2])
    assert math.isnan(out["v_std"][2])                          # var / std of one value: NaN
    assert math.isnan(out["v_median"][0]) and out["v_median"][1:] == [4.0, 7.0]
    assert out["v_nunique"] == [0, 1, 1]
    assert out["v_list"][0] == [None, None, None]
    assert out["v_first"] == [None, 4.0, 7.0]                  # positional: a null first element stays


def test_oracle_median_nunique_and_zero_values():
    df = pd.DataFrame({"k": [1, 1, 1, 1, 2, 2, 2], "v": [3.0, 1.0, -0.0, 0.0, 5.0, 1.0, 2.0]})
    out = session_groupby(df, "k", None, {"v": ["median", "nunique"]})
    assert out["v_median"] == [0.5, 2.0]                       # even: mean of the two middle values
    assert out["v_nunique"] == [3, 3]                          # -0.0 and +0.0 are one value


def _fit_schema(op, cols, dtypes, tags=None):
    wf = nvt.Workflow(cols >> op)
    schema = Schema([ColumnSchema(c, np.dtype(dtypes[c]), tags=(tags or {}).get(c, []),
                                  properties={"p": c}) for c in dtypes])
    wf.fit_schema(schema)
    return wf.output_schema


def test_schema_dtypes_lists_and_tags():
    dtypes = {"s": "int64", "item": "int32", "ts": "int64", "price": "float64", "x_counting": "float64"}
    op = nvt.ops.Groupby(groupby_cols=["s"], sort_cols="ts",
                         aggs={"item": ["list", "count", "first"], "ts": ["first", "last"],
                               "price": ["mean", "sum", "median", "nunique", "min"], "x_counting": "mean"})
    sch = _fit_schema(op, ["s", "item", "ts", "price", "x_counting"], dtypes, {"item": [Tags.CATEGORICAL, "custom_tag"]})
    assert sch.column_names == ["s", "item_list", "item_count", "item_first", "ts_first", "ts_last",
                                "price_mean", "price_sum", "price_median", "price_nunique", "price_min",
                                "x_counting_mean"]
    assert sch["s"].dtype == np.dtype("int64")
    assert sch["item_list"].dtype == np.dtype("int32") and sch["item_list"].is_list and sch["item_list"].is_ragged
    assert sch["item_count"].dtype == np.dtype("int32") and not sch["item_count"].is_list
    assert sch["item_first"].dtype == np.dtype("int32") and not sch["item_first"].is_list
    assert sch["ts_last"].dtype == np.dtype("int64")
    for c in ("price_mean", "price_sum", "price_median", "x_counting_mean"):
        assert sch[c].dtype == np.dtype("float32"), c          # the agg decides, not the name
    assert sch["price_nunique"].dtype == np.dtype("int32")
    assert sch["price_min"].dtype == np.dtype("float64")
    assert "custom_tag" in sch["item_list"].tags and Tags.CATEGORICAL in sch["item_first"].tags
    assert sch["price_mean"].properties["p"] == "price"


def test_schema_selector_without_groupby_cols():
    op = nvt.ops.Groupby(groupby_cols="s", aggs=["count", list])
    sch = _fit_schema(op, ["x"], {"s": "int64", "x": "float32"})
    assert sch.column_names == ["x_count", "x_list"]           # the key is not in the selector
    assert op.dependencies == ["s"]


def test_argument_errors():
    with pytest.raises(ValueError, match="cumprod"):
        nvt.ops.Groupby(groupby_cols="s", aggs="cumprod")
    with pytest.raises(ValueError):
        nvt.ops.Groupby(groupby_cols="s", aggs={"x": [np.sum]})
    with pytest.raises(ValueError):
        nvt.ops.Groupby(groupby_cols="s", aggs=lambda x: x)


@pytest.mark.parametrize("n,r", [(1, 0), (2, 1), (1 << 10, 10), ((1 << 10) + 1, 11), (1 << 20, 20),
                                 ((1 << 20) + 1, 21)])
def test_plan_rounds_row_bits(n, r):
    assert plan_rounds([5], n)[0] == r


def _check_plan(widths, n):
    r, rounds = plan_rounds(widths, n)
    cap = 64 - r
    got = {f: [] for f in range(len(widths))}
    for rnd in rounds:
        assert 0 < sum(b for _, _, b in rnd) <= cap
        for f, lo, b in rnd:
            got[f].append((lo, b))
    for f, w in enumerate(widths):
        lo = 0
        for clo, b in got[f]:                                 # low chunk first, contiguous
            assert clo == lo
            lo += b
        assert lo == w
    # greedy: every round but the last is full
    for rnd in rounds[:-1]:
        assert sum(b for _, _, b in rnd) == cap
    # significance: reading the rounds from last to first gives the fields most significant first
    order = [f for rnd in reversed(rounds) for f, _, _ in reversed(rnd)]
    assert order == sorted(order)
    return r, rounds


def test_plan_rounds_split_and_pack():
    r, rounds = _check_plan([1, 20, 64], 1 << 20)             # a 64-bit field is split
    assert r == 20 and len(rounds) == 2
    assert rounds[0] == [(2, 0, 44)] and rounds[1][0] == (2, 44, 20)
    _check_plan([3, 7, 11, 13], 100)                          # small fields share one round
    assert len(plan_rounds([3, 7, 11, 13], 100)[1]) == 1
    _check_plan([64, 64, 64], 1 << 25)
    _check_plan([33, 1, 0, 40, 2], 5)
    assert plan_rounds([0, 0], 10)[1] == []                   # nothing to sort


def test_groupby_graph_json_round_trip(tmp_path):
    op = nvt.ops.Groupby(groupby_cols=["s"], sort_cols=["ts"], aggs={"x": ["list", "first"], "ts": "max"},
                         name_sep="-", ascending=False)
    wf = nvt.Workflow(["s", "ts", "x"] >> op)
    wf.fit_schema(Schema([ColumnSchema("s", np.dtype("int64")), ColumnSchema("ts", np.dtype("int64")),
                          ColumnSchema("x", np.dtype("float32"))]))
    wf.save(str(tmp_path / "wf"))
    with open(os.path.join(tmp_path, "wf", "graph.json")) as f:
        graph = json.load(f)
    rec = [r for r in graph["nodes"] if r["op_class"] == "nvtabular.ops.groupby.Groupby"]
    assert len(rec) == 1 and rec[0]["op_params"]["aggs"] == {"x": ["list", "first"], "ts": ["max"]}
    wf2 = nvt.Workflow.load(str(tmp_path / "wf"))
    op2 = [n.op for n in wf2.output_node.topo_order() if n.kind == "op"][0]
    assert isinstance(op2, nvt.ops.Groupby)
    assert (op2.groupby_cols, op2.sort_cols, op2.aggs, op2.name_sep, op2.ascending) == \
        (["s"], ["ts"], {"x": ["list", "first"], "ts": ["max"]}, "-", False)
    assert wf2.output_schema.column_names == ["s", "x-list", "x-first", "ts-max"]
