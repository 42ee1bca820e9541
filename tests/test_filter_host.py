"""CPU tests of Filter and Dropna: the oracle (oracle/filter.py) against the reference's known
answers, every comparison rule of ops/filter.py pinned against pandas through the host function
that picks the comparison type and scalar bits, the save / load parameters, and the workflow's
guard against merging frames of different lengths."""
import json

import numpy as np
import pandas as pd
import pytest
import torch

from nvtabular_b200 import _lib
from nvtabular_b200.column import Column, DeviceFrame
from nvtabular_b200.graph import ColumnSelector
from nvtabular_b200.ops.base import Operator
from nvtabular_b200.ops.filter import column_compare_type, scalar_compare_type, string_code
from oracle.filter import dropna_frame, filter_frame

OPS = {"==": np.equal, "!=": np.not_equal, "<": np.less, "<=": np.less_equal, ">": np.greater,
       ">=": np.greater_equal}
_NP = {_lib.I64: np.int64, _lib.F32: np.float32, _lib.F64: np.float64}


def select_even(df):
    """a module-level predicate: importable, so a workflow holding it can be saved"""
    return df["a"] % 2 == 0


# ------------------------------------------------------------------------------- the oracle
def _ref_frame():
    rng = np.random.default_rng(0)
    return pd.DataFrame({"x": rng.normal(size=200), "y": rng.random(200)})


def test_oracle_matches_reference_test_filter():
    """reference tests/unit/ops/test_ops.py::test_filter: a frame result, a bool Series result,
    isnull, and an invalid return value"""
    df = _ref_frame()
    out = filter_frame(df, lambda d: d[d["y"] > 0.5])
    want = df[df["y"] > 0.5].reset_index(drop=True)
    pd.testing.assert_frame_equal(out, want)
    assert list(out.index) == list(range(len(out)))
    df.loc[df.index[::5], "x"] = np.nan
    by_frame = filter_frame(df, lambda d: d[d.x.isnull()])
    by_series = filter_frame(df, lambda d: d.x.isnull())
    pd.testing.assert_frame_equal(by_frame, by_series)
    assert 0 < len(by_series) < len(df)
    with pytest.raises(ValueError):
        filter_frame(df, lambda d: "some invalid value")


def test_oracle_matches_reference_test_filtered_partition():
    """reference tests/unit/test_dask_nvt.py::test_filtered_partition: 5 partitions of 20 rows,
    col < 75 leaves the last one empty"""
    df = pd.DataFrame({"col": range(100)})
    parts = [filter_frame(df.iloc[i:i + 20].reset_index(drop=True), lambda d: d["col"] < 75)
             for i in range(0, 100, 20)]
    assert [len(p) for p in parts] == [20, 20, 20, 15, 0]
    assert pd.concat(parts)["col"].tolist() == list(range(75))


def test_oracle_matches_reference_test_dropna_and_chaining():
    """reference tests/unit/ops/test_ops.py::test_dropna and the Dropna branch of
    tests/unit/workflow/test_workflow_chaining.py::test_chaining_3"""
    df = pd.DataFrame({"ad_id": [1, 2, 2, 6, 6, 8, 3, 3], "platform": [1, 2, np.nan, 2, 1, 3, 3, 1]})
    out = dropna_frame(df[["platform"]], ["platform"])
    assert out["platform"].tolist() == [1, 2, 2, 1, 3, 3, 1]
    assert not out.isnull().any().any()
    both = dropna_frame(pd.DataFrame({"a": [1.0, None, 3.0], "b": ["x", "y", None]}))
    assert both["a"].tolist() == [1.0]
    # a list column never drops a row
    lists = pd.DataFrame({"l": [[1], [], [2, 3]], "v": [1.0, 2.0, np.nan]})
    assert dropna_frame(lists)["l"].tolist() == [[1], []]


# ------------------------------------------------------------------------ comparison rules
def _emulate(vals: np.ndarray, cmp_type: int, bits: int, op: str) -> np.ndarray:
    """what nvtb_mask_compare computes: both operands converted to cmp_type"""
    t = _NP[cmp_type]
    if cmp_type == _lib.I64:
        s = np.array(bits, dtype=np.uint64).view(np.int64)
    elif cmp_type == _lib.F32:
        s = np.array(bits & 0xFFFFFFFF, dtype=np.uint32).view(np.float32)
    else:
        s = np.array(bits, dtype=np.uint64).view(np.float64)
    return OPS[op](vals.astype(t), s)


# (column dtype, column values, scalar): every op is checked against pandas
RULES = [
    ("int32", [1, -5, 2 ** 31 - 1, -2 ** 31], 2 ** 40),                 # exact in int64 beyond int32
    ("int32", [1, -5, 2 ** 31 - 1, -2 ** 31], -2 ** 40),
    ("int32", [1, -5, 7, 0], 7),
    ("int32", [1, -5, 7, 0], 2.5),                                        # int vs float: float64
    ("int64", [2 ** 53 + 1, 2 ** 53, -3, 2 ** 62], float(2 ** 53)),       # 2**53 + 1 > 2.0**53 is false
    ("int64", [2 ** 53 + 1, 2 ** 53, -3, 2 ** 62], 2 ** 53 + 1),          # exact in int64
    ("int64", [2 ** 63 - 1, -2 ** 63, 0, 5], 2 ** 63 - 1),
    ("int64", [1, 2, 3, 4], True),
    ("float32", [0.1, 16777216.0, -1.5, np.inf], 0.1),                    # the scalar becomes float32
    ("float32", [0.1, 16777216.0, -1.5, np.inf], 16777217),
    ("float32", [0.1, 16777216.0, -1.5, -np.inf], 1e300),                 # beyond float32: +inf
    ("float32", [0.1, 16777216.0, -1.5, -np.inf], -1e300),
    ("float32", [0.1, 2.0, -1.5, np.nan], float("nan")),
    ("float32", [0.1, 2.0, -1.5, 3.0], np.float64(0.1)),                  # a numpy scalar: result type
    ("float64", [0.1, 2.0, np.nan, -0.0], 0.0),
    ("float64", [0.1, 2.0, 2 ** 53, -7.0], 2 ** 53 + 1),
    ("float64", [0.1, 2.0, 2 ** 53, -7.0], np.float32(0.1)),
    ("bool", [True, False, True, False], True),
    ("bool", [True, False, True, False], 0),
    ("bool", [True, False, True, False], 0.5),
    ("uint8", [0, 1, 200, 255], 100),
    ("uint8", [0, 1, 200, 255], -1),
    ("uint8", [0, 1, 200, 255], 254.5),
    ("int32", [1, 2, 3, -4], np.int64(3)),
    ("int32", [1, 2, 3, -4], np.float32(1.5)),
    ("int64", [1, 2, 3, -4], np.uint8(3)),
]


@pytest.mark.parametrize("dtype, values, scalar", RULES, ids=[f"{d}-{s!r}" for d, _, s in RULES])
def test_scalar_rules_match_pandas(dtype, values, scalar):
    vals = np.array(values, dtype=dtype)
    cmp_type, bits = scalar_compare_type(np.dtype(dtype), scalar)
    for op in OPS:
        with np.errstate(over="ignore", invalid="ignore"):
            want = OPS[op](pd.Series(vals), scalar).to_numpy(dtype=bool)
        got = _emulate(vals, cmp_type, bits, op)
        np.testing.assert_array_equal(got, want, err_msg=f"{dtype} {op} {scalar!r}")


@pytest.mark.parametrize("dtype, scalar, cmp_type", [
    ("int32", 2 ** 40, _lib.I64), ("int64", 2.5, _lib.F64), ("bool", 1, _lib.I64), ("uint8", 3, _lib.I64),
    ("float32", 3, _lib.F32), ("float32", 0.1, _lib.F32), ("float64", 3, _lib.F64),
    ("float32", np.float64(0.1), _lib.F64), ("int32", np.float32(1.5), _lib.F64),
])
def test_scalar_compare_type(dtype, scalar, cmp_type):
    assert scalar_compare_type(np.dtype(dtype), scalar)[0] == cmp_type


def test_scalar_rules_named_in_the_docs():
    i64 = np.array([2 ** 53 + 1], dtype=np.int64)
    assert not _emulate(i64, *scalar_compare_type(np.dtype("int64"), float(2 ** 53)), ">")[0]
    f32 = np.array([0.1, 16777216], dtype=np.float32)
    assert not _emulate(f32, *scalar_compare_type(np.dtype("float32"), 0.1), ">")[0]
    assert _emulate(f32, *scalar_compare_type(np.dtype("float32"), 16777217), "==")[1]
    assert _emulate(np.array([-2 ** 31], np.int32), *scalar_compare_type(np.dtype("int32"), 2 ** 40), "<")[0]
    t, bits = scalar_compare_type(np.dtype("float32"), 1e300)
    assert t == _lib.F32 and np.array(bits, np.uint32).view(np.float32) == np.inf


@pytest.mark.parametrize("scalar", [2 ** 63, -2 ** 63 - 1, 2 ** 70])
@pytest.mark.parametrize("dtype", ["int32", "int64", "bool", "uint8"])
def test_int_outside_int64_raises(dtype, scalar):
    with pytest.raises(OverflowError):
        scalar_compare_type(np.dtype(dtype), scalar)


@pytest.mark.parametrize("dtype", ["int32", "float64", "bool"])
@pytest.mark.parametrize("scalar", ["a", None, [1], object()])
def test_non_numeric_scalar_raises(dtype, scalar):
    with pytest.raises(TypeError):
        scalar_compare_type(np.dtype(dtype), scalar)


PAIRS = ["int32", "int64", "float32", "float64", "bool", "uint8"]


@pytest.mark.parametrize("da", PAIRS)
@pytest.mark.parametrize("db", PAIRS)
def test_column_rules_match_pandas(da, db):
    rng = np.random.default_rng(len(da) * 7 + len(db))
    raw_a = rng.integers(-3, 4, 64)
    raw_b = rng.integers(-3, 4, 64)
    a = (raw_a > 0) if da == "bool" else (raw_a % 256 if da == "uint8" else raw_a).astype(da)
    b = (raw_b > 0) if db == "bool" else (raw_b % 256 if db == "uint8" else raw_b).astype(db)
    if da.startswith("float"):
        a = a + np.array(0.1, dtype=da) * (raw_b > 1)
    t = column_compare_type(np.dtype(da), np.dtype(db))
    for op in OPS:
        want = OPS[op](pd.Series(a), pd.Series(b)).to_numpy(dtype=bool)
        np.testing.assert_array_equal(OPS[op](a.astype(_NP[t]), b.astype(_NP[t])), want, err_msg=f"{da} {op} {db}")


def test_string_codes():
    d = np.array(["a", "bb", "c"], dtype=object)
    assert [string_code(d, s) for s in ["a", "bb", "c", "b", "zz", ""]] == [0, 1, 2, -1, -1, -1]
    assert string_code(np.array([], dtype=object), "a") == -1


# --------------------------------------------------------------------------- operators
def test_filter_needs_a_function():
    from nvtabular_b200 import ops
    with pytest.raises(ValueError):
        ops.Filter(None)
    with pytest.raises(ValueError):
        ops.Filter(f=None)


def _saved_graph(tmp_path, op):
    import nvtabular_b200 as nvt
    from nvtabular_b200.graph import Schema, ColumnSchema
    wf = nvt.Workflow(["a", "b"] >> op)
    wf.fit_schema(Schema([ColumnSchema("a", np.dtype("int64")), ColumnSchema("b", np.dtype("float64"))]))
    wf.save(str(tmp_path / "wf"))
    return wf, json.load(open(tmp_path / "wf" / "graph.json"))


def test_save_load_module_level_function(tmp_path):
    import nvtabular_b200 as nvt
    from nvtabular_b200 import ops
    _, graph = _saved_graph(tmp_path, ops.Filter(f=select_even))
    node = [r for r in graph["nodes"] if r["op_class"] == "nvtabular.ops.filter.Filter"]
    assert node and node[0]["op_params"] == {"f": {"module": __name__, "qualname": "select_even"}}
    loaded = nvt.Workflow.load(str(tmp_path / "wf"))
    ops_ = [n.op for n in loaded.output_node.topo_order() if n.kind == "op"]
    assert isinstance(ops_[0], ops.Filter) and ops_[0].f is select_even


def test_save_load_dropna(tmp_path):
    import nvtabular_b200 as nvt
    from nvtabular_b200 import ops
    _, graph = _saved_graph(tmp_path, ops.Dropna())
    node = [r for r in graph["nodes"] if r["op_class"] == "nvtabular.ops.dropna.Dropna"]
    assert node and node[0]["op_params"] == {} and node[0]["op_state"] == {}
    loaded = nvt.Workflow.load(str(tmp_path / "wf"))
    assert any(isinstance(n.op, ops.Dropna) for n in loaded.output_node.topo_order() if n.kind == "op")


def test_save_rejects_lambda_main_and_local_functions(tmp_path):
    from nvtabular_b200 import ops
    from nvtabular_b200.serialize import WorkflowSerializationError

    def local(df):
        return df["a"] > 0

    main_fn = lambda df: df["a"] > 0  # noqa: E731
    with pytest.raises(WorkflowSerializationError, match="lambda"):
        _saved_graph(tmp_path / "l", ops.Filter(f=main_fn))
    in_main = (lambda df: df).__class__(select_even.__code__, {"__name__": "__main__"}, "in_main")
    in_main.__module__ = "__main__"
    with pytest.raises(WorkflowSerializationError, match="__main__"):
        _saved_graph(tmp_path / "m", ops.Filter(f=in_main))
    with pytest.raises(WorkflowSerializationError):
        _saved_graph(tmp_path / "x", ops.Filter(f=local))


# ------------------------------------------------------------------------------ merge guard
class _Head(Operator):
    """keeps the first k rows (host tensors; no device needed)"""

    def __init__(self, k):
        super().__init__()
        self.k = k

    def transform(self, col_selector, df):
        return DeviceFrame({n: Column(df[n].data[:self.k]) for n in col_selector.names})


def _host_frame(n=10):
    return DeviceFrame({"a": Column(torch.arange(n)), "b": Column(torch.arange(n) * 2.0),
                        "c": Column(torch.arange(n, dtype=torch.int32))})


@pytest.mark.parametrize("graph", ["concat", "op_input"])
def test_merge_of_unequal_row_counts_raises(graph):
    from nvtabular_b200.graph import Node
    from nvtabular_b200.workflow import _execute_node
    short = ["a"] >> _Head(4)
    node = short + ["b"] if graph == "concat" else (short + ["b"]) >> _Head(10)
    with pytest.raises(ValueError, match=r"\['a'\] have 4 rows.*\['b'\] have 10 rows"):
        _execute_node(Node.construct_from(node), _host_frame(), {})


def test_merge_of_equal_row_counts_passes():
    from nvtabular_b200.graph import Node
    from nvtabular_b200.workflow import _execute_node
    out = _execute_node(Node.construct_from((["a"] >> _Head(10)) + ["b", "c"]), _host_frame(), {})
    assert out.columns == ["a", "b", "c"] and len(out) == 10
    out = _execute_node(Node.construct_from((["a"] >> _Head(3)) + (["b"] >> _Head(3))), _host_frame(), {})
    assert len(out) == 3
