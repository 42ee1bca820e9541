"""CPU tests of ListSlice and DifferenceLag: the oracle (oracle/session_ops.py) against the
reference's known answers and the pinned rules, the argument normalisation and every argument /
type error (all raised before any kernel), the output schema, and the graph.json round trip."""
import json

import numpy as np
import pandas as pd
import pytest
import torch

from oracle.session_ops import INT64_MAX, difference_lag, list_slice, normalise

ROWS = [[0, 1, 2, 2, 767], [1, 2, 2, 3], [1, 223, 4]]


# ------------------------------------------------------------------------------- the oracle
@pytest.mark.parametrize("args, want", [
    ((0, 2), [[0, 1], [1, 2], [1, 223]]),
    ((3, 5), [[2, 767], [3], []]),
    ((4, 10), [[767], [], []]),
    ((100, 20000), [[], [], []]),
    ((-4,), [[1, 2, 2, 767], [1, 2, 2, 3], [1, 223, 4]]),
    ((-3, -1), [[2, 2], [2, 2], [1, 223]]),
])
def test_oracle_matches_reference_test_list_slice(args, want):
    """reference tests/unit/ops/test_list_slice.py::test_list_slice (every case)"""
    assert list_slice(ROWS, *args) == want


@pytest.mark.parametrize("args, kw, want", [
    ((5,), {}, [[0, 1, 2, 2, 767], [1, 2, 2, 3, 0], [1, 223, 4, 0, 0]]),
    ((1, 6), {"pad_value": 123}, [[1, 2, 2, 767, 123], [2, 2, 3, 123, 123], [223, 4, 123, 123, 123]]),
    ((-4,), {"pad_value": -1}, [[1, 2, 2, 767], [1, 2, 2, 3], [1, 223, 4, -1]]),
    ((-4, -1), {"pad_value": -1}, [[1, 2, 2], [1, 2, 2], [1, 223, -1]]),
])
def test_oracle_matches_reference_test_list_slice_pad(args, kw, want):
    """reference tests/unit/ops/test_list_slice.py::test_list_slice_pad (every case)"""
    assert list_slice(ROWS, *args, pad=True, **kw) == want


def test_oracle_keeps_leaf_nulls_and_reads_a_null_row_as_empty():
    assert list_slice([[1, None, 3], None], -2) == [[None, 3], []]
    assert list_slice([[1, None, 3], None], 2, pad=True, pad_value=9) == [[1, None], [9, 9]]


def test_oracle_matches_reference_test_difference_lag():
    """reference tests/unit/ops/test_ops.py::test_difference_lag"""
    df = pd.DataFrame({"userid": [0, 0, 0, 1, 1, 2], "timestamp": [1000, 1005, 1100, 2000, 2001, 3000]})
    out = difference_lag(df, ["timestamp"], ["userid"], shift=[1, -1])
    assert list(out.columns) == ["timestamp_difference_lag_1", "timestamp_difference_lag_-1"]
    lag, lead = out["timestamp_difference_lag_1"], out["timestamp_difference_lag_-1"]
    assert lag.dtype == np.float32 and lead.dtype == np.float32
    assert lag[1] == 5 and lag[2] == 95 and np.isnan(lag[0]) and np.isnan(lag[3])
    assert lead[0] == -5 and lead[1] == -95 and lead[3] == -1 and np.isnan(lead[2]) and np.isnan(lead[5])


def test_oracle_key_rules():
    # a null or NaN key never matches, -0.0 matches +0.0, shift 0 gives 0, a long shift gives nulls
    df = pd.DataFrame({"k": [np.nan, np.nan, -0.0, 0.0, 1.0], "x": [1, 2, 3, 5, 9]})
    lag = difference_lag(df, ["x"], "k", 1)["x_difference_lag_1"].to_numpy()
    assert np.isnan(lag[:3]).all() and lag[3] == 2.0 and np.isnan(lag[4])
    zero = difference_lag(df, ["x"], "k", 0)["x_difference_lag_0"].to_numpy()
    assert np.isnan(zero[:2]).all() and (zero[2:] == 0).all()
    assert np.isnan(difference_lag(df, ["x"], "k", 1000)["x_difference_lag_1000"].to_numpy()).all()
    ki = pd.DataFrame({"k": pd.array([None, None, 7], dtype="Int64"), "s": ["a", None, None], "x": [1, 2, 3]})
    assert np.isnan(difference_lag(ki, ["x"], "k", 1)["x_difference_lag_1"][1])
    assert np.isnan(difference_lag(ki, ["x"], "s", 1)["x_difference_lag_1"][2])


def test_oracle_value_rules():
    # int64 subtracts exactly (wrapping), then rounds once; pandas' float64 operands would give 0.0
    big = pd.DataFrame({"k": [1, 1], "x": np.array([2 ** 60 + 1, 2 ** 60 + 3], dtype=np.int64)})
    assert difference_lag(big, ["x"], "k", 1)["x_difference_lag_1"][1] == 2.0
    wrap = pd.DataFrame({"k": [1, 1], "x": np.array([np.iinfo(np.int64).max, np.iinfo(np.int64).min])})
    assert difference_lag(wrap, ["x"], "k", 1)["x_difference_lag_1"][1] == 1.0
    f32 = pd.DataFrame({"k": [1, 1], "x": np.array([1.0, 1.0 + 2 ** -23], dtype=np.float32)})
    assert difference_lag(f32, ["x"], "k", 1)["x_difference_lag_1"][1] == np.float32(2 ** -23)
    f64 = pd.DataFrame({"k": [1, 1], "x": [0.1, 0.3]})
    assert difference_lag(f64, ["x"], "k", 1)["x_difference_lag_1"][1] == np.float32(0.3 - 0.1)
    nan = pd.DataFrame({"k": [1, 1, 1], "x": [1.0, np.nan, 2.0]})
    assert np.isnan(difference_lag(nan, ["x"], "k", 1)["x_difference_lag_1"][1:]).all()


# ------------------------------------------------------------------------------ ListSlice
def test_list_slice_argument_normalisation():
    from nvtabular import ops
    for args, want in [((5,), (0, 5, 5)), ((1, 6), (1, 6, 5)), ((-4,), (-4, INT64_MAX, 4)), ((-4, -1), (-4, -1, 3)),
                       ((-3, 5), (-3, 5, 3)), ((0,), (0, INT64_MAX, INT64_MAX)), ((2, 2), (2, 2, 0))]:
        op = ops.ListSlice(*args)
        assert (op.start, op.end, op.max_elements) == want == normalise(*args), args


def test_list_slice_constructor_errors():
    from nvtabular import ops
    with pytest.raises(ValueError, match="bounded"):
        ops.ListSlice(0, pad=True)
    with pytest.raises(ValueError, match="bounded"):
        ops.ListSlice(3, INT64_MAX, pad=True)
    with pytest.raises(ValueError, match="max_elements"):
        ops.ListSlice(1, -1, pad=True)
    with pytest.raises(ValueError, match="max_elements"):
        ops.ListSlice(4, 4, pad=True)
    with pytest.raises(TypeError):
        ops.ListSlice("1")
    with pytest.raises(TypeError):
        ops.ListSlice(1, 2.0)
    ops.ListSlice(1, -1)                     # without pad the same slice is fine
    ops.ListSlice(-3, pad=True)


def _cpu_list(values, dtype, validity=None, dictionary=None, is_bool=False):
    from nvtabular_b200.column import Column
    c = Column(torch.tensor(values, dtype=dtype), validity, torch.tensor([0, len(values)]), dictionary, None, is_bool)
    return c


def test_pad_value_conversion():
    from nvtabular_b200.ops.list_slice import pad_bits
    assert pad_bits(-1, _cpu_list([1], torch.int32)) == 0xFFFFFFFF
    assert pad_bits(7.0, _cpu_list([1], torch.int64)) == 7
    assert pad_bits(0.1, _cpu_list([1.0], torch.float32)) == int(np.array(0.1, np.float32).view(np.uint32))
    assert pad_bits(0.1, _cpu_list([1.0], torch.float64)) == int(np.array(0.1).view(np.uint64))
    assert pad_bits(float("nan"), _cpu_list([1.0], torch.float32)) == int(np.array(np.nan, np.float32).view(np.uint32))
    assert pad_bits(True, _cpu_list([1], torch.uint8, is_bool=True)) == 1
    assert pad_bits(np.int64(5), _cpu_list([1], torch.uint8)) == 5
    for v, dt in [(1.5, torch.int64), (float("nan"), torch.int32), (2 ** 31, torch.int32), (-1, torch.uint8),
                  (2, None), (1e300, torch.float32), ("x", torch.int64), (None, torch.int64)]:
        col = _cpu_list([1], torch.uint8, is_bool=True) if dt is None else \
            _cpu_list([1.0] if dt.is_floating_point else [1], dt)
        with pytest.raises(ValueError):
            pad_bits(v, col)
    with pytest.raises(TypeError):
        pad_bits(0, _cpu_list([0], torch.int32, dictionary=np.array(["a"], dtype=object)))


def test_list_slice_transform_errors_come_before_any_kernel():
    from nvtabular import ColumnSelector, ops
    from nvtabular_b200.column import Column, DeviceFrame
    flat = DeviceFrame({"x": Column(torch.tensor([1, 2, 3]))})
    with pytest.raises(ValueError, match="not a list column"):
        ops.ListSlice(0, 2).transform(ColumnSelector(["x"]), flat)
    strings = DeviceFrame({"s": _cpu_list([0, 1], torch.int32, dictionary=np.array(["a", "b"], dtype=object))})
    with pytest.raises(TypeError, match="string"):
        ops.ListSlice(0, 2, pad=True).transform(ColumnSelector(["s"]), strings)
    ints = DeviceFrame({"y": _cpu_list([1, 2], torch.int64)})
    with pytest.raises(ValueError, match="pad_value"):
        ops.ListSlice(0, 2, pad=True, pad_value=0.5).transform(ColumnSelector(["y"]), ints)


def _fit_schema(node, cols):
    import nvtabular as nvt
    wf = nvt.Workflow(node)
    wf.fit_schema(nvt.Schema(cols))
    return wf


def test_list_slice_schema_and_embedding_sizes():
    import nvtabular as nvt
    from nvtabular import ops
    from nvtabular_b200.graph import ColumnSchema, Tags
    src = [ColumnSchema("items", dtype=np.dtype("int64"), is_list=True, is_ragged=True)]
    for op, ragged, vc in [(ops.ListSlice(-20, pad=True), False, {"min": 20, "max": 20}),
                           (ops.ListSlice(-20), True, {"min": 0, "max": 20}),
                           (ops.ListSlice(2, 5), True, {"min": 0, "max": 3}),
                           (ops.ListSlice(0), True, {"min": 0, "max": None})]:
        cs = _fit_schema(["items"] >> op, src).output_schema["items"]
        assert cs.dtype == np.dtype("int64") and cs.is_list and cs.is_ragged == ragged
        assert cs.properties["value_count"] == vc and Tags.LIST in cs.tags
    padded = _fit_schema(["items"] >> ops.Categorify() >> ops.ListSlice(-20, pad=True), src)
    ragged = _fit_schema(["items"] >> ops.Categorify() >> ops.ListSlice(-20), src)
    sizes = nvt.ops.get_embedding_sizes(padded)
    assert isinstance(sizes, dict) and "items" in sizes          # fixed-length: not multi-hot
    single, multi = nvt.ops.get_embedding_sizes(ragged)
    assert "items" in multi and "items" not in single
    assert Tags.CATEGORICAL in padded.output_schema["items"].tags


def test_difference_lag_schema_names_and_dependencies():
    from nvtabular import ColumnSelector, ops
    from nvtabular_b200.graph import ColumnSchema, Tags
    op = ops.DifferenceLag("userid", shift=[1, -1])
    assert op.dependencies == ["userid"] and op.shifts == [1, -1]
    assert op.column_mapping(ColumnSelector(["ts", "price"])) == {
        "ts_difference_lag_1": ["ts"], "ts_difference_lag_-1": ["ts"],
        "price_difference_lag_1": ["price"], "price_difference_lag_-1": ["price"]}
    node = ["ts"] >> op
    wf = _fit_schema(node, [ColumnSchema("ts", dtype=np.dtype("int64")), ColumnSchema("userid", dtype=np.dtype("int64"))])
    assert wf.output_schema.column_names == ["ts_difference_lag_1", "ts_difference_lag_-1"]
    for cs in wf.output_schema:
        assert cs.dtype == np.dtype("float32") and Tags.CONTINUOUS in cs.tags and not cs.is_list
    assert sorted(wf.input_schema.column_names) == ["ts", "userid"]
    assert ops.DifferenceLag(["a", "b"], 3).dependencies == ["a", "b"]


def test_difference_lag_errors():
    from nvtabular import ColumnSelector, ops
    from nvtabular_b200.column import Column, DeviceFrame
    for bad in (1.5, "1", [1, 2.0], True, None, []):
        with pytest.raises(TypeError):
            ops.DifferenceLag("k", shift=bad)
    assert ops.DifferenceLag("k", shift=np.int64(2)).shifts == [2]
    k = Column(torch.tensor([1, 1, 2]))
    frames = {"bool": Column(torch.tensor([True, False, True])),
              "string": Column(torch.tensor([0, 1, 0], dtype=torch.int32), None, None, np.array(["a", "b"], dtype=object)),
              "list": _cpu_list([1, 2, 3], torch.int64)}
    for kind, col in frames.items():
        with pytest.raises(TypeError, match=kind):
            ops.DifferenceLag("k").transform(ColumnSelector(["v"]), DeviceFrame({"k": k, "v": col}))
    with pytest.raises(ValueError, match="partition"):
        ops.DifferenceLag([f"k{i}" for i in range(9)]).transform(
            ColumnSelector(["v"]), DeviceFrame({**{f"k{i}": k for i in range(9)}, "v": k}))
    assert not isinstance(ops.DifferenceLag("k"), ops.StatOperator)
    assert not isinstance(ops.ListSlice(2), ops.StatOperator)


# ------------------------------------------------------------------------------ save / load
def test_list_slice_graph_json_round_trip(tmp_path):
    import nvtabular as nvt
    from nvtabular import ops
    from nvtabular_b200.graph import ColumnSchema
    cases = [ops.ListSlice(5), ops.ListSlice(-4, pad=True, pad_value=-1), ops.ListSlice(1, 6, pad=True, pad_value=2.5),
             ops.ListSlice(-3, -1)]
    for i, op in enumerate(cases):
        wf = _fit_schema(["items"] >> op, [ColumnSchema("items", dtype=np.dtype("float32"), is_list=True, is_ragged=True)])
        path = tmp_path / f"wf{i}"
        wf.save(str(path))
        graph = json.loads((path / "graph.json").read_text())
        rec = [r for r in graph["nodes"] if r["op_class"] == "nvtabular.ops.list_slice.ListSlice"]
        assert len(rec) == 1
        assert rec[0]["op_params"] == {"start": op.start, "end": op.end, "pad": op.pad, "pad_value": op.pad_value}
        back = nvt.Workflow.load(str(path))
        got = [n.op for n in back.output_node.topo_order() if n.kind == "op"][0]
        assert isinstance(got, ops.ListSlice)
        assert (got.start, got.end, got.pad, got.pad_value, got.max_elements) == \
            (op.start, op.end, op.pad, op.pad_value, op.max_elements)
        assert back.output_schema["items"].properties["value_count"] == wf.output_schema["items"].properties["value_count"]


def test_saving_difference_lag_raises(tmp_path):
    from nvtabular import ops
    from nvtabular_b200.graph import ColumnSchema
    from nvtabular_b200.serialize import WorkflowSerializationError
    wf = _fit_schema(["ts"] >> ops.DifferenceLag("u"), [ColumnSchema("ts", dtype=np.dtype("int64")),
                                                        ColumnSchema("u", dtype=np.dtype("int64"))])
    with pytest.raises(WorkflowSerializationError, match="DifferenceLag"):
        wf.save(str(tmp_path / "wf"))
