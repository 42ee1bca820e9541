"""GPU parity tests at the operator/Workflow boundary: the reference's own
known-answer tests (tests/unit/ops/test_{categorify,normalize,fill,join,
target_encode,hash_bucket}.py, tests/unit/workflow/test_cpu_workflow.py)
re-typed against `import nvtabular as nvt` — same user code, H100 engine
underneath — plus randomised comparisons with the CPU oracle."""
import math
import os

import numpy as np
import pandas as pd
import pytest

import oracle
from oracle.categorify import CategorifyOracle
from oracle.groupby import groupby_stats, join_groupby_transform, target_encoding

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nvt():
    import nvtabular
    return nvtabular


@pytest.fixture(scope="module")
def ops(nvt):
    return nvt.ops


def _run(nvt, node, df, **ds_kw):
    wf = nvt.Workflow(node)
    out = wf.fit_transform(nvt.Dataset(df, **ds_kw)).to_ddf().compute()
    return wf, out


# reference tests/unit/ops/test_categorify.py:124-157
@pytest.mark.parametrize("freq_threshold", [0, 1, 2])
@pytest.mark.parametrize("dtype", [None, np.int32, np.int64])
@pytest.mark.parametrize("use_vocab", [False, True])
def test_categorify_lists(nvt, ops, tmp_path, freq_threshold, dtype, use_vocab):
    df = pd.DataFrame({
        "Authors": [["User_A"], ["User_A", "User_E"], ["User_B", "User_C"], ["User_C"]],
        "Engaging User": ["User_B", "User_B", "User_A", "User_D"],
        "Post": [1, 2, 3, 4],
    })
    vocabs = {"Authors": pd.Series([f"User_{x}" for x in "ACBE"])} if use_vocab else None
    cats = ["Authors", "Engaging User"] >> ops.Categorify(
        out_path=str(tmp_path), freq_threshold=freq_threshold, dtype=dtype, vocabs=vocabs)
    _, out = _run(nvt, cats + ["Post"], df)
    assert out["Authors"][0].dtype == (np.dtype(dtype) if dtype else np.dtype("int64"))
    compare = [list(r) for r in out["Authors"].tolist()]
    if freq_threshold < 2 or use_vocab:
        assert compare == [[3], [3, 6], [5, 4], [4]]
    else:
        assert compare == [[3], [3, 2], [2, 4], [4]]


# reference tests/unit/ops/test_categorify.py:160-216
@pytest.mark.parametrize("cat_names", [[["Author", "Engaging User"]], ["Author", "Engaging User"]])
@pytest.mark.parametrize("kind", ["joint", "combo"])
def test_categorify_multi(nvt, ops, tmp_path, cat_names, kind):
    df = pd.DataFrame({
        "Author": ["User_A", "User_E", "User_B", "User_C"],
        "Engaging User": ["User_B", "User_B", "User_A", "User_D"],
        "Post": [1, 2, 3, 4],
    })
    cats = cat_names >> ops.Categorify(out_path=str(tmp_path), encode_type=kind)
    _, out = _run(nvt, cats + ["Post"], df)
    if len(cat_names) == 1:
        if kind == "joint":
            assert out["Author"].tolist() == [4, 7, 3, 5]
            assert out["Engaging User"].tolist() == [3, 3, 4, 6]
        else:
            assert out["Author_Engaging User"].tolist() == [3, 6, 4, 5]
    else:
        assert out["Author"].tolist() == [3, 6, 4, 5]
        assert out["Engaging User"].tolist() == [3, 3, 4, 5]


_COMBO_CASES = [
    ({"Author": ["User_B", "User_E", "User_B", "User_C"], "Engaging User": ["User_C", "User_B", "User_A", "User_D"]},
     [3, 5, 3, 4], [5, 4, 3, 6], [4, 6, 3, 5]),
    ({"Author": ["User_A", "User_E", "User_B", "User_C"], "Engaging User": ["User_B", "User_B", "User_A", "User_D"]},
     [3, 6, 4, 5], [3, 3, 4, 5], [3, 6, 4, 5]),
    ({"Author": ["User_C", "User_E", "User_B", "User_C"], "Engaging User": ["User_B", "User_B", "User_A", "User_D"]},
     [3, 5, 4, 3], [3, 3, 4, 5], [4, 6, 3, 5]),
    ({"Author": ["User_A", "User_B", "User_C", "User_C"], "Engaging User": ["User_A", "User_B", "User_C", "User_C"]},
     [4, 5, 3, 3], [4, 5, 3, 3], [4, 5, 3, 3]),
    ({"Author": ["User_C", "User_E", "User_B", "User_A"], "Engaging User": ["User_C", "User_B", "User_A", "User_D"]},
     [5, 6, 4, 3], [5, 4, 3, 6], [5, 6, 4, 3]),
    ({"Author": [np.nan, "User_E", "User_B", "User_A"], "Engaging User": ["User_C", "User_B", "User_A", "User_D"]},
     [1, 5, 4, 3], [5, 4, 3, 6], [3, 6, 5, 4]),
]


# reference tests/unit/ops/test_categorify.py:219-323
@pytest.mark.parametrize("case", _COMBO_CASES)
@pytest.mark.parametrize("cat_names", [
    [["Author", "Engaging User"], ["Author"], ["Engaging User"]],
    [["Author", "Engaging User"], "Author", "Engaging User"],
])
def test_categorify_multi_combo(nvt, ops, tmp_path, case, cat_names):
    data, exp_a, exp_e, exp_ae = case
    df = pd.DataFrame({**data, "Post": [1, 2, 3, 4]})
    cats = cat_names >> ops.Categorify(out_path=str(tmp_path), encode_type="combo")
    _, out = _run(nvt, cats + ["Post"], df)
    assert out["Author"].tolist() == exp_a
    assert out["Engaging User"].tolist() == exp_e
    assert out["Author_Engaging User"].tolist() == exp_ae


# reference tests/unit/ops/test_categorify.py:99-121
def test_na_value_count(nvt, ops, tmp_path):
    df = pd.DataFrame({
        "productID": ["B00406YHLI"] * 5 + ["B002YXS8E6"] * 5 + ["B00011KM38"] * 2 + [np.nan] * 3,
        "brand": ["Coby"] * 5 + [np.nan] * 5 + ["Cooler Master"] * 2 + ["Asus"] * 3,
    })
    cats = ["brand", "productID"] >> ops.Categorify(out_path=str(tmp_path))
    wf = nvt.Workflow(cats)
    wf.fit(nvt.Dataset(df))
    wf.transform(nvt.Dataset(df)).to_ddf().compute()
    m1 = pd.read_parquet(tmp_path / "categories" / "meta.brand.parquet")
    m2 = pd.read_parquet(tmp_path / "categories" / "meta.productID.parquet")
    assert m1["kind"].iloc[1] == "null" and m1["num_observed"].iloc[1] == 5
    assert m2["kind"].iloc[1] == "null" and m2["num_observed"].iloc[1] == 3


# reference tests/unit/ops/test_categorify.py:38-96
@pytest.mark.parametrize("include_nulls", [True, False])
@pytest.mark.parametrize("cardinality_memory_limit", [None, "24B"])
def test_categorify_size(nvt, ops, tmp_path, include_nulls, cardinality_memory_limit):
    rng = np.random.RandomState(0)
    ids = list(range(10)) + ([None] if include_nulls else [])
    df = pd.DataFrame({"session_id": [ids[i] for i in rng.randint(0, len(ids), 50)]})
    cats = ["session_id"] >> ops.Categorify(out_path=str(tmp_path), cardinality_memory_limit=cardinality_memory_limit)
    wf = nvt.Workflow(cats)
    if cardinality_memory_limit:
        with pytest.warns(UserWarning):
            wf.fit_transform(nvt.Dataset(df)).to_ddf().compute()
    else:
        wf.fit_transform(nvt.Dataset(df)).to_ddf().compute()
    vals = df["session_id"].value_counts()
    vocab = pd.read_parquet(tmp_path / "categories" / "unique.session_id.parquet")
    computed = {k: s for k, s in zip(vocab["session_id"], vocab["session_id_size"]) if s}
    assert computed == dict(zip(vals.index, vals))


# reference tests/unit/ops/test_categorify.py:326-421 (the merge path)
@pytest.mark.parametrize("freq_limit", [{"Author": 3, "Engaging User": 4}])
@pytest.mark.parametrize("buckets", [None, 10, {"Author": 10, "Engaging User": 20}])
def test_categorify_freq_limit(nvt, ops, tmp_path, freq_limit, buckets):
    df = pd.DataFrame({
        "Author": ["User_A", "User_E", "User_B", "User_C", "User_A", "User_E", "User_B", "User_C", "User_B", "User_C"],
        "Engaging User": ["User_B", "User_B", "User_A", "User_D", "User_B", "User_c", "User_A", "User_D", "User_D", "User_D"],
    })
    cats = ["Author", "Engaging User"] >> ops.Categorify(
        freq_threshold=freq_limit, out_path=str(tmp_path), num_buckets=buckets)
    _, out = _run(nvt, cats, df)
    for col in ["Author", "Engaging User"]:
        meta = pd.read_parquet(tmp_path / "categories" / f"meta.{col}.parquet")
        assert meta["num_observed"].sum() == len(df)
    freq_limited = {"Author": 2, "Engaging User": 1}
    if not buckets:
        assert out["Author"].max() == 1 + 1 + freq_limited["Author"]
        assert out["Engaging User"].max() == 1 + 1 + freq_limited["Engaging User"]
    else:
        b = buckets if isinstance(buckets, dict) else {"Author": buckets, "Engaging User": buckets}
        assert out["Author"].max() <= 1 + freq_limited["Author"] + b["Author"]
        assert out["Engaging User"].max() <= 1 + freq_limited["Engaging User"] + b["Engaging User"]
        # string OOV buckets follow pandas' own string hash (hash_series CPU branch)
        oov = df["Author"].isin(["User_A", "User_E"])
        exp = 2 + pd.util.hash_array(df["Author"].to_numpy(dtype=object)) % np.uint64(b["Author"])
        np.testing.assert_array_equal(out["Author"][oov].to_numpy(), exp[oov.to_numpy()].astype(np.int64))


# reference tests/unit/ops/test_categorify.py:424-447
def test_categorify_hash_bucket_only(nvt, ops, tmp_path):
    df = pd.DataFrame({"Authors": ["User_A", "User_A", "User_E", "User_B", "User_C"],
                       "Engaging_User": ["User_B", "User_B", "User_A", "User_D", "User_D"], "Post": [1, 2, 3, 4, 5]})
    buckets = 10
    max_size = buckets + 2
    feats = ["Authors", "Engaging_User"] >> ops.Categorify(num_buckets=buckets, max_size=max_size, out_path=str(tmp_path))
    wf = nvt.Workflow(feats)
    wf.fit(nvt.Dataset(df))
    out = wf.transform(nvt.Dataset(df)).to_ddf().compute()
    assert out["Authors"].max() <= max_size and out["Engaging_User"].max() <= max_size
    assert nvt.ops.get_embedding_sizes(wf)["Authors"][0] == max_size
    assert nvt.ops.get_embedding_sizes(wf)["Engaging_User"][0] == max_size


# reference tests/unit/ops/test_categorify.py:450-506
@pytest.mark.parametrize("max_emb_size", [6, {"Author": 8, "Engaging_User": 7}])
def test_categorify_max_size(nvt, ops, tmp_path, max_emb_size):
    df = pd.DataFrame({"Author": [f"User_{c}" for c in "AEBCAEBCDFF"],
                       "Engaging_User": [f"User_{c}" for c in "BBADBMADNFE"]})
    feats = ["Author", "Engaging_User"] >> ops.Categorify(max_size=max_emb_size, num_buckets=3, out_path=str(tmp_path))
    wf = nvt.Workflow(feats)
    wf.fit(nvt.Dataset(df))
    out = wf.transform(nvt.Dataset(df)).to_ddf().compute()
    if isinstance(max_emb_size, int):
        max_emb_size = {n: max_emb_size for n in ["Author", "Engaging_User"]}
    sizes = nvt.ops.get_embedding_sizes(wf)
    for n in ["Author", "Engaging_User"]:
        assert out[n].max() <= max_emb_size[n] + 1
        assert sizes[n][0] <= max_emb_size[n] + 1


# reference tests/unit/ops/test_categorify.py:509-529
def test_categorify_single_table(nvt, ops, tmp_path):
    df = pd.DataFrame({"Authors": [None, "User_A", "User_A", "User_E", "User_B", "User_C"],
                       "Engaging_User": [None, "User_B", "User_B", "User_A", "User_D", "User_D"],
                       "Post": [1, 2, 3, 4, None, 5]})
    feats = ["Authors", "Engaging_User"] >> ops.Categorify(single_table=True, out_path=str(tmp_path))
    _, out = _run(nvt, feats, df)
    old_max = 1
    for name in ["Authors", "Engaging_User"]:
        assert old_max <= out[name].min()
        old_max += out[name].max()
    o = CategorifyOracle(["Authors", "Engaging_User"], single_table=True).fit(df)
    exp = o.transform(df)
    for name in ["Authors", "Engaging_User"]:
        assert out[name].tolist() == exp[name].tolist()


# reference tests/unit/ops/test_categorify.py:543-556, 615-633
def test_categorify_null_meta(nvt, ops, tmp_path):
    df = pd.DataFrame({"user_id": [1, 2, 3, 4, 6, 8, 5, 3] * 10, "item_id": [2, 4, 4, 7, 5, 2, 5, 2] * 10})
    nvt.Workflow(["user_id", "item_id"] >> ops.Categorify(out_path=str(tmp_path))).fit(nvt.Dataset(df))
    meta = pd.read_parquet(tmp_path / "categories" / "meta.user_id.parquet")
    assert meta["kind"].iloc[1] == "null" and meta["num_observed"].iloc[1] == 0
    df = pd.DataFrame({"C1": [1, np.nan, 3, 4, 3] * 5, "C2": [1, 1, 2, 3, 6] * 5})
    wf = nvt.Workflow(["C1", "C2"] >> ops.Categorify(max_size=4, out_path=str(tmp_path)))
    wf.fit(nvt.Dataset(df))
    out = wf.transform(nvt.Dataset(df)).to_ddf().compute()
    assert pd.read_parquet(tmp_path / "categories" / "meta.C1.parquet")["num_observed"].iloc[1] == 5
    assert pd.read_parquet(tmp_path / "categories" / "meta.C2.parquet")["num_observed"].iloc[1] == 0
    exp = CategorifyOracle(["C1", "C2"], max_size=4).fit(df).transform(df)
    assert out["C1"].tolist() == exp["C1"].tolist() and out["C2"].tolist() == exp["C2"].tolist()


# reference tests/unit/ops/test_categorify.py:636-665
def test_categorify_joint_list(nvt, ops, tmp_path):
    df = pd.DataFrame({"Author": ["User_A", "User_E", "User_B", "User_C"],
                       "Engaging User": [["User_B", "User_C"], [], ["User_A", "User_D"], ["User_A"]],
                       "Post": [1, 2, 3, 4]})
    cats = ["Post", ["Author", "Engaging User"]] >> ops.Categorify(encode_type="joint", out_path=str(tmp_path))
    _, out = _run(nvt, cats, df)
    assert out["Author"].tolist() == [3, 7, 4, 5]
    assert [x for r in out["Engaging User"] for x in r] == [4, 5, 3, 6, 3]


# reference tests/unit/ops/test_categorify.py:559-612
@pytest.mark.parametrize("cat_names", [[["Author", "Engaging User"]], ["Author", "Engaging User"]])
@pytest.mark.parametrize("kind", ["joint", "combo"])
def test_categorify_domain_name(nvt, ops, tmp_path, cat_names, kind):
    df = pd.DataFrame({"Author": ["User_A", "User_E", "User_B", "User_C"],
                       "Engaging User": ["User_B", "User_B", "User_A", "User_D"], "Post": [1, 2, 3, 4]})
    cats = cat_names >> ops.Categorify(out_path=str(tmp_path), encode_type=kind)
    wf, _ = _run(nvt, cats, df)
    domain_names = [wf.output_schema[c].properties["domain"]["name"] for c in wf.output_schema.column_names]
    if len(cat_names) == 1 and kind == "combo":
        assert domain_names == ["Author_Engaging User"]
    elif len(cat_names) == 1 and kind == "joint":
        assert len(set(domain_names)) == 1
    else:
        assert len(set(domain_names)) > 1
    for c in wf.output_schema.column_names:
        assert wf.output_schema[c].properties["domain"]["max"] > 0


def test_categorify_errors(nvt, ops):
    with pytest.raises(ValueError):
        ops.Categorify(start_index=1)
    with pytest.raises(ValueError):
        ops.Categorify(freq_threshold=2, max_size=10)
    with pytest.raises(ValueError):
        ops.Categorify(encode_type="nope")
    with pytest.raises(ValueError):
        ops.Categorify(num_buckets=0)
    with pytest.warns(FutureWarning):
        ops.Categorify(tree_width=8)
    df = pd.DataFrame({"a": [1, 2, 3]})
    with pytest.raises(ValueError):   # max_size < num_buckets + 2 (categorify.py:1206-1211)
        nvt.Workflow(["a"] >> ops.Categorify(max_size=3, num_buckets=5)).fit(nvt.Dataset(df))


@pytest.mark.parametrize("nparts", [1, 3])
@pytest.mark.parametrize("kw", [{}, {"freq_threshold": 3}, {"max_size": 40}, {"max_size": 40, "num_buckets": 7},
                                {"num_buckets": 5, "freq_threshold": 2}, {"dtype": np.int32}])
def test_categorify_random_vs_oracle(nvt, ops, tmp_path, nparts, kw):
    """integer keys, nulls, Zipf skew, several partitions: labels and vocab files bit-exact."""
    rng = np.random.default_rng(123)
    n = 20000
    a = (rng.zipf(1.3, n) % 500 * 104729 % 100003).astype("int32")
    b = rng.integers(-50, 50, n).astype("int64")
    df = pd.DataFrame({"a": pd.array(a, dtype="Int32"), "b": b})
    df.loc[rng.random(n) < 0.05, "a"] = pd.NA
    cats = ["a", "b"] >> ops.Categorify(out_path=str(tmp_path), **kw)
    wf, out = _run(nvt, cats, df, npartitions=nparts)
    dfo = pd.DataFrame({"a": df["a"].astype("float64"), "b": b})
    o = CategorifyOracle(["a", "b"], **kw).fit(dfo)
    # OOV hash parity is defined on the integer column (oracle/hashing.py): give the oracle
    # the int values and re-impose the nulls
    dfi = pd.DataFrame({"a": df["a"].fillna(0).astype("int32"), "b": b})
    exp = o.transform(dfi)
    exp_a = exp["a"].to_numpy().copy()
    exp_a[df["a"].isna().to_numpy()] = 1
    np.testing.assert_array_equal(out["a"].to_numpy(), exp_a)
    np.testing.assert_array_equal(out["b"].to_numpy(), exp["b"].to_numpy())
    for c in ["a", "b"]:
        got = pd.read_parquet(tmp_path / "categories" / f"unique.{c}.parquet")
        ov = o.categories[c].unique
        np.testing.assert_array_equal(got.index.to_numpy(), ov.index.to_numpy())
        np.testing.assert_array_equal(got[c].to_numpy().astype("int64"), ov[c].to_numpy().astype("int64"))
        np.testing.assert_array_equal(got[f"{c}_size"].to_numpy(), ov[f"{c}_size"].to_numpy())
        meta = pd.read_parquet(tmp_path / "categories" / f"meta.{c}.parquet")
        assert meta["num_observed"].tolist() == [int(x) for x in o.categories[c].meta["num_observed"]]


# reference tests/unit/ops/test_normalize.py:60-84, 87-117, 120-139; test_fill.py:61-85
def test_fill_normalize_workflow(nvt, ops):
    rng = np.random.default_rng(5)
    n = 30000
    df = pd.DataFrame({"x": rng.standard_normal(n) * 3 + 1, "y": rng.integers(-5, 1000, n).astype("float64"),
                       "z": rng.integers(0, 9, n)})
    df.loc[rng.random(n) < 0.2, "x"] = np.nan
    df.loc[rng.random(n) < 0.3, "y"] = np.nan
    conts = ["x", "y", "z"] >> ops.FillMissing() >> ops.Normalize()
    wf, out = _run(nvt, conts, df, npartitions=3)
    filled = oracle.fill_missing(df, ["x", "y", "z"], 0)
    parts = [filled.iloc[i:i + 10000] for i in range(0, n, 10000)]
    means, stds = oracle.normalize_fit(parts, ["x", "y", "z"])
    op = wf.output_node.op
    for c in ["x", "y", "z"]:
        assert math.isclose(op.means[c], means[c], rel_tol=1e-9)
        assert math.isclose(op.stds[c], stds[c], rel_tol=1e-9)
        assert math.isclose(filled[c].mean(), op.means[c], rel_tol=1e-4)   # the reference's own bar
        assert math.isclose(filled[c].std(), op.stds[c], rel_tol=1e-4)
    exp = oracle.normalize_transform(filled, ["x", "y", "z"], op.means, op.stds)
    for c in ["x", "y", "z"]:
        np.testing.assert_array_equal(out[c].to_numpy(), exp[c].to_numpy())
        assert out[c].dtype == np.float64
    # std == 0 -> all zeros (test_normalize.py:110-117)
    _, r = _run(nvt, ["a"] >> ops.Normalize(), pd.DataFrame({"a": 7 * [10]}))
    assert (r["a"] == 0).all()
    # values up to 1.6e19 need fp64 (test_normalize.py:120-139)
    big = pd.DataFrame({"x": [1.9e10, 2.3e16, 3.4e18, 1.6e19]})
    w, r = _run(nvt, ["x"] >> ops.Normalize(), big)
    assert math.isclose(big["x"].mean(), w.output_node.op.means["x"], rel_tol=1e-4)
    assert math.isclose(big["x"].std(), w.output_node.op.stds["x"], rel_tol=1e-4)
    # list column (test_normalize.py:87-107)
    ldf = pd.DataFrame({"vals": [[0.0, 1.0, 2.0], [3.0, 4.0], [5.0]]})
    _, r = _run(nvt, ["vals"] >> ops.Normalize(), ldf)
    flat = pd.Series([0.0, 1.0, 2.0, 3.0, 4.0, 5.0])
    np.testing.assert_allclose(np.concatenate(r["vals"].tolist()), ((flat - flat.mean()) / flat.std()).to_numpy(), rtol=1e-12)


@pytest.mark.parametrize("add_binary_cols", [True, False])
def test_fill_missing(nvt, ops, add_binary_cols):
    rng = np.random.default_rng(6)
    df = pd.DataFrame({"x": rng.random(1000), "y": rng.random(1000)})
    df.loc[rng.choice(1000, 200), "x"] = None
    df.loc[rng.choice(1000, 200), "y"] = None
    feats = ["x", "y"] >> ops.FillMissing(fill_val=42, add_binary_cols=add_binary_cols)
    _, out = _run(nvt, feats, df)
    exp = oracle.fill_missing(df, ["x", "y"], 42, add_binary_cols)
    for c in ["x", "y"]:
        np.testing.assert_array_equal(out[c].to_numpy(), exp[c].to_numpy())
        assert out[c].isna().sum() == 0
        assert (f"{c}_filled" in out) == add_binary_cols
        if add_binary_cols:
            assert df[c].isna().sum() == out[f"{c}_filled"].sum()
            assert out[f"{c}_filled"].dtype == bool


def test_normalize_minmax(nvt, ops):
    rng = np.random.default_rng(7)
    df = pd.DataFrame({"x": rng.random(5000), "y": rng.integers(0, 100, 5000)})
    wf, out = _run(nvt, ["x", "y"] >> ops.NormalizeMinMax(), df)
    mins, maxs = oracle.minmax_fit(df, ["x", "y"])
    exp = oracle.minmax_transform(df, ["x", "y"], mins, maxs)
    for c in ["x", "y"]:
        assert wf.output_node.op.mins[c] == mins[c] and wf.output_node.op.maxs[c] == maxs[c]
        np.testing.assert_array_equal(out[c].to_numpy(), exp[c].to_numpy())


# reference tests/unit/ops/test_hash_bucket.py:50-56 (+ bit-exact vs the pandas hash)
def test_hash_bucket(nvt, ops):
    rng = np.random.default_rng(8)
    df = pd.DataFrame({"a": rng.integers(0, 1 << 40, 10000), "b": rng.integers(0, 1000, 10000).astype("int32")})
    _, out = _run(nvt, ["a", "b"] >> ops.HashBucket({"a": 10, "b": 1 << 20}), df)
    np.testing.assert_array_equal(out["a"].to_numpy(), oracle.hash_bucket(df["a"].to_numpy(), 10))
    np.testing.assert_array_equal(out["b"].to_numpy(), oracle.hash_bucket(df["b"].to_numpy(), 1 << 20))
    assert out["a"].dtype == np.int32 and out["a"].min() >= 0 and out["a"].max() <= 9


# reference tests/unit/ops/test_join.py:32-92
def test_joingroupby(nvt, ops, tmp_path):
    df = pd.DataFrame({"Author": ["User_A", "User_A", "User_A", "User_B"],
                       "Engaging-User": ["User_B", "User_B", "User_C", "User_C"],
                       "Cost": [100.0, 200.0, 300.0, 400.0], "Post": [1, 2, 3, 4]})
    g = [["Author", "Engaging-User"]] >> ops.JoinGroupby(out_path=str(tmp_path), stats=["sum"], cont_cols=["Cost"])
    _, out = _run(nvt, g + "Post", df)
    assert out["Author_Engaging-User_Cost_sum"].tolist() == [300.0, 300.0, 300.0, 400.0]
    g = "Author" >> ops.JoinGroupby(out_path=str(tmp_path), stats=["sum"], cont_cols=["Cost"])
    _, out = _run(nvt, g + "Post", df)
    assert out["Author_Cost_sum"].tolist() == [600.0, 600.0, 600.0, 400.0]
    # dependency on an upstream node (test_join.py:32-57)
    df = pd.DataFrame({"Author": ["User_A"] * 3 + ["User_B"] * 2, "Cost": [100.0, 200.0, 300.0, 400.0, 400.0]})
    normalized = ["Cost"] >> ops.NormalizeMinMax()
    g = ["Author"] >> ops.JoinGroupby(out_path=str(tmp_path), stats=["sum"], cont_cols=normalized)
    _, out = _run(nvt, g, df)
    assert out["Author_Cost_sum"].tolist() == [1.0, 1.0, 1.0, 2.0, 2.0]


def test_joingroupby_random_vs_oracle(nvt, ops, tmp_path):
    rng = np.random.default_rng(9)
    n = 20000
    df = pd.DataFrame({"u": rng.integers(0, 300, n).astype("int32"), "m": rng.integers(0, 50, n).astype("int32"),
                       "r": rng.integers(1, 11, n) / 2.0})
    df.loc[rng.random(n) < 0.05, "r"] = np.nan
    stats = ["count", "sum", "mean", "std", "var", "min", "max"]
    g = ["u", ["u", "m"]] >> ops.JoinGroupby(out_path=str(tmp_path), stats=stats, cont_cols=["r"])
    _, out = _run(nvt, g, df, npartitions=2)
    tabs = {"u": groupby_stats(df, ["u"], ["r"], stats), "u_m": groupby_stats(df, ["u", "m"], ["r"], stats)}
    exp = join_groupby_transform(df, ["u", ["u", "m"]], tabs)
    # column order follows column_mapping (the user's `stats` order), as the reference's
    # executor selects node.output_columns after op.transform
    assert sorted(out.columns) == sorted(exp.columns)
    assert list(out.columns)[:4] == ["u_count", "u_r_sum", "u_r_mean", "u_r_std"]
    for c in exp.columns:
        assert out[c].dtype == exp[c].dtype, c
        np.testing.assert_allclose(out[c].to_numpy(), exp[c].to_numpy(), rtol=2e-6, equal_nan=True, err_msg=c)
        if c.endswith("count") or c.endswith("min") or c.endswith("max") or c.endswith("sum"):
            np.testing.assert_array_equal(out[c].to_numpy(), exp[c].to_numpy())


def test_joingroupby_int_columns_on_unseen_and_null_keys_vs_oracle(nvt, ops, tmp_path):
    """Fit on one frame, transform it and a second frame whose keys the fit never saw, with null
    keys the fit had no group for.  Integer statistics: sum int64 (exact beyond 2^31, where an
    int32 sum would overflow), min/max in the column's dtype, and missing where the reference's
    left merge finds no group, never 0."""
    rng = np.random.default_rng(19)
    n = 30_000
    train = pd.DataFrame({"u": rng.integers(0, 300, n).astype("int32"), "m": rng.integers(0, 20, n).astype("int32"),
                          "big": rng.integers(1 << 29, (1 << 31) - 1, n).astype("int32"),   # group sums > 2^31
                          "small": rng.integers(-50, 50, n).astype("int32"),
                          "w": rng.integers(-(1 << 40), 1 << 40, n).astype("int64"),
                          "r": rng.normal(0, 1, n)})
    m = 4000
    test = pd.DataFrame({"u": pd.array(rng.integers(0, 400, m), dtype="Int32"),     # 1/4 unseen keys
                         "m": rng.integers(0, 25, m).astype("int32")})
    test.loc[rng.random(m) < 0.05, "u"] = pd.NA                                     # no null group in the fit
    for c in ("big", "small", "w", "r"):
        test[c] = train[c].iloc[:m].to_numpy()
    conts, groups = ["big", "small", "w", "r"], ["u", ["u", "m"]]
    stats = ["sum", "min", "max", "mean"]    # "count" of a missing key cannot be cast to int32 by the reference
    wf = nvt.Workflow(groups >> ops.JoinGroupby(out_path=str(tmp_path), stats=stats, cont_cols=conts))
    wf.fit(nvt.Dataset(train))
    tabs = {"u": groupby_stats(train, ["u"], conts, stats), "u_m": groupby_stats(train, ["u", "m"], conts, stats)}
    assert tabs["u"]["u_big_sum"].max() > (1 << 31)
    schema = {c: np.dtype(wf.output_schema[c].dtype) for c in wf.output_schema.column_names}
    for frame, unseen in ((train, False), (test, True)):
        out = wf.transform(nvt.Dataset(frame)).to_ddf().compute()
        exp = join_groupby_transform(frame, groups, tabs)
        assert sorted(out.columns) == sorted(exp.columns)
        for c in exp.columns:
            stat, src = c.rsplit("_", 1)[-1], c.split("_")[-2]
            want = np.dtype("int64") if stat == "sum" and src != "r" else schema[c]
            if not unseen:
                # pandas keeps int32 for an int32 sum that fits; the engine always sums ints into int64
                assert schema[c] == want and out[c].dtype == want, (c, out[c].dtype, want)
            else:
                # rows without a group: missing, so pandas and the engine both hold float64 NaN
                assert out[c].dtype == exp[c].dtype, (c, out[c].dtype, exp[c].dtype)
                if np.dtype(schema[c]).kind == "i":
                    assert out[c].isna().to_numpy().sum() > m // 5, c
            if c.endswith("_mean") or src == "r":
                np.testing.assert_allclose(out[c].to_numpy(dtype=np.float64), exp[c].to_numpy(dtype=np.float64),
                                           rtol=1e-6, equal_nan=True, err_msg=c)
            else:
                np.testing.assert_array_equal(out[c].to_numpy(dtype=np.float64), exp[c].to_numpy(dtype=np.float64),
                                              err_msg=c)


# reference tests/unit/ops/test_target_encode.py:38-84, 111-147
@pytest.mark.parametrize("kfold", [1, 3])
@pytest.mark.parametrize("npartitions", [1, 2])
def test_target_encode_vs_oracle(nvt, ops, tmp_path, kfold, npartitions):
    cat_1 = np.asarray(["baaaa"] * 12)
    cat_2 = np.asarray(["baaaa"] * 6 + ["bbaaa"] * 3 + ["bcaaa"] * 3)
    num_1 = np.asarray([1, 1, 2, 2, 2, 1, 1, 5, 4, 4, 4, 4])
    df = pd.DataFrame({"cat": cat_1, "cat2": cat_2, "num": num_1, "num_2": num_1 * 2})
    groups = ["cat", "cat2", ["cat", "cat2"]]
    te = groups >> ops.TargetEncoding(["num", "num_2"], out_path=str(tmp_path), kfold=kfold, p_smooth=5,
                                      out_dtype="float32")
    _, out = _run(nvt, te, df, npartitions=npartitions)
    chunk = -(-12 // npartitions)
    parts = [df.iloc[i:i + chunk] for i in range(0, 12, chunk)]
    exp = pd.concat(target_encoding(parts, groups, ["num", "num_2"], kfold=kfold, p_smooth=5, out_dtype="float32")[0],
                    ignore_index=True)
    for c in exp.columns:
        np.testing.assert_allclose(out[c].to_numpy(), exp[c].to_numpy(), rtol=1e-6, err_msg=c)
        assert out[c].dtype == np.float32
    if kfold == 1:
        np.testing.assert_array_equal(out["TE_cat2_num"].values, out["TE_cat_cat2_num"].values)
        assert math.isclose(out["TE_cat_num"].iloc[0], num_1.mean(), abs_tol=1e-4)


# reference tests/unit/workflow/test_cpu_workflow.py:16-81 (Categorify + FillMissing + Normalize end to end)
def test_criteo_shape_workflow_vs_oracle(nvt, ops, tmp_path):
    rng = np.random.default_rng(10)
    n = 50000
    conts = [f"I{i}" for i in range(1, 4)]
    cats = [f"C{i}" for i in range(1, 5)]
    data = {"label": rng.integers(0, 2, n).astype("int32")}
    for i, c in enumerate(conts):
        v = np.floor(np.exp(rng.normal(2, 2, n))).clip(0, 2**31 - 1).astype("float64")
        v[rng.random(n) < 0.1 * (i + 1)] = np.nan
        data[c] = pd.array(v, dtype="Int32")
    for i, c in enumerate(cats):
        k = [3, 1000, 50000, 7][i]
        v = ((rng.random(n) ** (1 / 0.9) * k).astype("int64") * 2654435761 % (2**31 - 1)).astype("float64")
        v[rng.random(n) < 0.03 * i] = np.nan
        data[c] = pd.array(v, dtype="Int32")
    df = pd.DataFrame(data)
    cat_f = cats >> ops.Categorify(out_path=str(tmp_path))
    cont_f = conts >> ops.FillMissing() >> ops.Normalize()
    wf = nvt.Workflow(cat_f + cont_f + ["label"])
    out = wf.fit_transform(nvt.Dataset(df, npartitions=4)).to_ddf().compute()
    assert list(out.columns) == cats + conts + ["label"]
    dfo = pd.DataFrame({c: df[c].astype("float64") for c in conts + cats})
    o = CategorifyOracle(cats).fit(dfo)
    exp_c = o.transform(dfo)
    filled = oracle.fill_missing(dfo, conts, 0)
    means, stds = oracle.normalize_fit(filled, conts)
    exp_n = oracle.normalize_transform(filled, conts, means, stds)
    for c in cats:
        np.testing.assert_array_equal(out[c].to_numpy(), exp_c[c].to_numpy())
        assert out[c].dtype == np.int64
    for c in conts:
        got, exp = out[c].to_numpy(), exp_n[c].to_numpy()
        np.testing.assert_allclose(got, exp, rtol=1e-9, atol=1e-12)   # stats agree to ~1e-12 => outputs too
        assert out[c].dtype == np.float64
    np.testing.assert_array_equal(out["label"].to_numpy(), df["label"].to_numpy())
    # a second, unseen frame: OOV -> 2, null -> 1
    df2 = pd.DataFrame({c: pd.array(rng.integers(0, 2**31 - 1, 1000), dtype="Int32") for c in cats})
    df2.loc[:10, "C1"] = pd.NA
    for c in conts:
        df2[c] = pd.array(rng.integers(0, 100, 1000), dtype="Int32")
    df2["label"] = 0
    out2 = wf.transform(df2)
    exp2 = o.transform(pd.DataFrame({c: df2[c].astype("float64") for c in cats}))
    for c in cats:
        np.testing.assert_array_equal(out2[c].to_numpy(), exp2[c].to_numpy())


def test_full_size_properties(nvt, ops, tmp_path):
    """Size-independent properties at a bench-scale table (2^24 rows x 39 columns), where the
    CPU oracle would take minutes: meta counts add up to the row count, labels stay inside
    [1, cardinality), nulls map to 1, fit is idempotent (second fit == first), transform of the
    kept keys is a bijection onto [first_label, first_label + n_kept), normalised columns have
    mean 0 / std 1, and a 1/64 sample agrees bit-exactly with the oracle run on that sample's
    rows against the same vocabulary."""
    import torch
    from nvtabular_b200.column import unpack_validity
    from nvtabular_b200.synth import CAT_NAMES, CONT_NAMES, criteo_frame
    rows = 1 << 24
    frame = criteo_frame(rows, total_rows=rows, device="cuda")
    cats = CAT_NAMES >> ops.Categorify(out_path=str(tmp_path))
    conts = CONT_NAMES >> ops.FillMissing() >> ops.Normalize()
    wf = nvt.Workflow(cats + conts + ["label"])
    ds = nvt.Dataset(frame)
    wf.fit(ds)
    out = next(iter(wf.transform(ds).partitions()))
    cat_op = cats.op
    first = {}
    for c in CAT_NAMES:
        fv = cat_op.categories.fitted[c]
        v = fv.vocab
        col = frame[c]
        nulls = rows - int(unpack_validity(col.validity, rows).sum().item()) if col.validity is not None else 0
        assert v.null_size == nulls
        assert v.null_size + v.oov_size + v.unique_size == rows       # num_observed sums to len(df)
        lab = out[c].data
        assert lab.dtype == torch.int64 and int(lab.min()) >= 1 and int(lab.max()) == 2 + v.n_kept
        if col.validity is not None:
            assert bool((lab[~unpack_validity(col.validity, rows)] == 1).all())
        # every kept key encodes to its own position: a bijection onto [3, 3 + n_kept)
        keys, sizes = v.export()
        kc = nvt.Column(keys.to(torch.int32))
        enc = v.encode(kc, 1, 2, 3)
        assert torch.equal(enc, torch.arange(3, 3 + v.n_kept, device="cuda"))
        # (size desc, key asc)
        assert bool((sizes[:-1] >= sizes[1:]).all())
        ties = sizes[:-1] == sizes[1:]
        assert bool((keys[:-1][ties] < keys[1:][ties]).all())
        first[c] = (keys.clone(), sizes.clone())
    for c in CONT_NAMES:
        x = out[c].data
        assert x.dtype == torch.float64 and abs(float(x.mean())) < 1e-9 and abs(float(x.std()) - 1) < 1e-6
    # idempotence: a second fit over the same data reproduces the vocabularies exactly
    wf.fit(ds)
    for c in CAT_NAMES:
        keys, sizes = cat_op.categories.fitted[c].vocab.export()
        assert torch.equal(keys, first[c][0]) and torch.equal(sizes, first[c][1])
    # 1/64 sample vs the oracle's encode against the SAME vocabulary
    from oracle.categorify import Vocab as OVocab, categorify_encode
    idx = torch.arange(0, rows, 64, device="cuda")
    for c in ["C1", "C6", "C20", "C23"]:
        keys, sizes = first[c]
        uniq = pd.DataFrame({c: keys.cpu().numpy(), f"{c}_size": sizes.cpu().numpy()})
        uniq.index = pd.RangeIndex(3, 3 + len(uniq))
        ov = OVocab(c, [c], uniq, pd.DataFrame())
        vals = frame[c].data[idx].cpu().numpy()
        valid = unpack_validity(frame[c].validity, rows)[idx].cpu().numpy() if frame[c].validity is not None \
            else np.ones(len(vals), bool)
        exp = categorify_encode(pd.DataFrame({c: vals}), c, ov)
        exp[~valid] = 1
        np.testing.assert_array_equal(out[c].data[idx].cpu().numpy(), exp)
