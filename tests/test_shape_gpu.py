"""GPU parity tests AT SHAPE for BASELINE.json configs C4 (MovieLens JoinGroupby +
TargetEncoding), C5 (HashBucket over int64 key columns) and for the fit paths the
Criteo-1TB profile reaches (partitioned fold at >= 4 M keys, sorted accumulator beyond).

Reference behaviour: tests/unit/ops/test_target_encode.py:38-147, tests/unit/ops/test_join.py:32-92,
tests/unit/ops/test_hash_bucket.py:50-56, tests/unit/test_dask_nvt.py:143-181; operators
nvtabular/ops/{join_groupby.py:140-217, target_encoding.py:171-439, hash_bucket.py:86-100,
categorify.py:955-1337}.  Integer results bit-exact; float32 statistics within the tolerance
stated in each test."""
import numpy as np
import pandas as pd
import pytest

from oracle.groupby import groupby_stats, join_groupby_transform, target_encoding
from oracle.hashing import hash_bucket as oracle_hash_bucket

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nvt():
    import nvtabular
    return nvtabular


@pytest.fixture(scope="module")
def ops(nvt):
    return nvt.ops


def _movielens_pandas(rows, seed, n_user, n_movie):
    rng = np.random.default_rng(seed)
    # power-law ids (nvtabular/tools/data_gen.py:55-66 form), scattered so key order != frequency order
    def ids(k, alpha):
        g = 1.0 - alpha
        x = np.power(rng.random(rows) * (float(k) ** g - 1.0) + 1.0, 1.0 / g)
        return ((np.clip(x.astype(np.int64), 1, k) * 2654435761) & 0x7FFFFFFF).astype(np.int32)
    return pd.DataFrame({"userId": ids(n_user, 0.1), "movieId": ids(n_movie, 0.5),
                         "rating": (rng.integers(1, 11, rows) * 0.5).astype(np.float32)})


# C4: the fused three-group workflow of SURVEY.md 8(d) at MovieLens cardinalities
def test_movielens_shape_joingroupby_targetencoding_vs_oracle(nvt, ops, tmp_path):
    rows = 1_000_000
    df = _movielens_pandas(rows, 11, 160_000, 60_000)
    groups = ["userId", "movieId", ["userId", "movieId"]]
    stats = ["count", "sum", "mean", "std"]
    jg = groups >> ops.JoinGroupby(out_path=str(tmp_path), cont_cols=["rating"], stats=stats)
    te = groups >> ops.TargetEncoding("rating", kfold=5, p_smooth=20, out_path=str(tmp_path))
    wf = nvt.Workflow(jg + te)
    out = wf.fit_transform(nvt.Dataset(df, npartitions=2)).to_ddf().compute()

    chunk = -(-rows // 2)
    parts = [df.iloc[i:i + chunk].reset_index(drop=True) for i in range(0, rows, chunk)]
    tabs = {"userId": groupby_stats(parts, ["userId"], ["rating"], stats),
            "movieId": groupby_stats(parts, ["movieId"], ["rating"], stats),
            "userId_movieId": groupby_stats(parts, ["userId", "movieId"], ["rating"], stats)}
    exp_j = join_groupby_transform(df, groups, tabs)
    for c in exp_j.columns:
        assert out[c].dtype == exp_j[c].dtype, c
        if c.endswith("count"):
            np.testing.assert_array_equal(out[c].to_numpy(), exp_j[c].to_numpy(), err_msg=c)
        else:       # float32 outputs; pandas accumulates a float32 column IN float32, the engine in fp64:
            # a few float32 ulps of the partial sums (ratings are multiples of 0.5, so most are exact)
            np.testing.assert_allclose(out[c].to_numpy(), exp_j[c].to_numpy(), rtol=2e-5, atol=1e-5,
                                       equal_nan=True, err_msg=c)
    exp_t = pd.concat(target_encoding(parts, groups, ["rating"], kfold=5, p_smooth=20)[0], ignore_index=True)
    for c in exp_t.columns:
        assert out[c].dtype == np.float32, c
        np.testing.assert_allclose(out[c].to_numpy(), exp_t[c].to_numpy(), rtol=2e-6, err_msg=c)


# One 5e6-row partition: with no hint and no estimate the operator's first insert is the blind
# 2^20-row sample (4 M-slot table), from which ~2e6 keys are estimated, and prepare() then grows
# the table before the rest of the rows: the payload goes through rehash_kernel.  TargetEncoding's
# packed (fold, group) keys are int64, so the wide table with payload grows the same way.
def test_groupby_stats_through_table_growth_vs_oracle(nvt, ops, tmp_path):
    rows = 5_000_000
    rng = np.random.default_rng(12)
    x = rng.normal(3.0, 2.0, rows)
    x[rng.random(rows) < 0.05] = np.nan
    df = pd.DataFrame({
        "g": ((rng.integers(0, 2_000_000, rows) * 2654435761) % (1 << 31)).astype(np.int32),
        "h": rng.integers(0, 4, rows).astype(np.int32),
        "x": x,                                                           # float64 with NaN
        "i": rng.integers(-1000, 1000, rows).astype(np.int32),            # int32, no nulls
        "f": (rng.integers(1, 11, rows) * 0.5).astype(np.float32)})      # float32
    groups = ["g", ["g", "h"]]
    stats = ["count", "sum", "mean", "std", "var", "min", "max"]
    jg = groups >> ops.JoinGroupby(out_path=str(tmp_path), cont_cols=["x", "i", "f"], stats=stats)
    te = groups >> ops.TargetEncoding(["f", "i"], kfold=3, p_smooth=20, out_path=str(tmp_path))
    wf = nvt.Workflow(jg + te)
    out = wf.fit_transform(nvt.Dataset(df, npartitions=1)).to_ddf().compute()

    tabs = {"g": groupby_stats([df], ["g"], ["x", "i", "f"], stats),
            "g_h": groupby_stats([df], ["g", "h"], ["x", "i", "f"], stats)}
    exp_j = join_groupby_transform(df, groups, tabs)
    assert sorted(c for c in out.columns if not c.startswith("TE_")) == sorted(exp_j.columns)
    for c in exp_j.columns:
        # the sum of an int column is int64 (exact); pandas keeps int32 for an int32 sum that fits
        want = np.dtype("int64") if c.endswith("_i_sum") else exp_j[c].dtype
        assert out[c].dtype == want, (c, out[c].dtype, exp_j[c].dtype)
        if c.endswith("count") or np.issubdtype(exp_j[c].dtype, np.integer):
            np.testing.assert_array_equal(out[c].to_numpy(), exp_j[c].to_numpy(), err_msg=c)
        else:
            np.testing.assert_allclose(out[c].to_numpy(), exp_j[c].to_numpy(), rtol=2e-5, atol=1e-5,
                                       equal_nan=True, err_msg=c)
    exp_t = pd.concat(target_encoding([df], groups, ["f", "i"], kfold=3, p_smooth=20)[0], ignore_index=True)
    assert sorted(c for c in out.columns if c.startswith("TE_")) == sorted(exp_t.columns)
    for c in exp_t.columns:
        assert out[c].dtype == exp_t[c].dtype == np.float32, c
        np.testing.assert_allclose(out[c].to_numpy(), exp_t[c].to_numpy(), rtol=2e-6, err_msg=c)


# TargetEncoding, random frame, every fold count the reference's tests use
@pytest.mark.parametrize("kfold", [1, 3, 5])
@pytest.mark.parametrize("npartitions", [1, 3])
def test_target_encoding_random_vs_oracle(nvt, ops, tmp_path, kfold, npartitions):
    rows = 100_000
    rng = np.random.default_rng(100 + kfold)
    df = pd.DataFrame({"a": rng.integers(0, 2000, rows).astype(np.int32),
                       "b": rng.integers(0, 37, rows).astype(np.int64),
                       "y": rng.normal(3.0, 2.0, rows), "z": rng.integers(0, 2, rows).astype(np.float32)})
    groups = ["a", "b", ["a", "b"]]
    te = groups >> ops.TargetEncoding(["y", "z"], kfold=kfold, p_smooth=10, fold_seed=7, out_path=str(tmp_path),
                                      out_dtype="float64")
    out = nvt.Workflow(te).fit_transform(nvt.Dataset(df, npartitions=npartitions)).to_ddf().compute()
    chunk = -(-rows // npartitions)
    parts = [df.iloc[i:i + chunk].reset_index(drop=True) for i in range(0, rows, chunk)]
    exp = pd.concat(target_encoding(parts, groups, ["y", "z"], kfold=kfold, p_smooth=10, fold_seed=7,
                                    out_dtype="float64")[0], ignore_index=True)
    assert sorted(out.columns) == sorted(exp.columns)
    for c in exp.columns:
        assert out[c].dtype == np.float64
        # `z` is a float32 column: pandas reduces it (target mean, group sums) in float32, the engine
        # in fp64 -> a float32 ulp of the mean (3e-8 relative); the float64 target agrees to 1e-9
        np.testing.assert_allclose(out[c].to_numpy(), exp[c].to_numpy(), rtol=1e-6 if c.endswith("_z") else 1e-9,
                                   err_msg=c)


# C5: HashBucket(2^20) over 40 int64 key columns, keys uniform over 1e8 ids through a 64-bit bijection
def test_hashbucket_c5_shape_vs_oracle(nvt, ops):
    import torch
    from nvtabular_b200.synth import hashbucket_frame
    rows, ncols = 10_000_000, 40
    frame = hashbucket_frame(rows, ncols, device="cuda")
    names = list(frame.columns)
    wf = nvt.Workflow(names >> ops.HashBucket(1 << 20))
    out = next(iter(wf.transform(nvt.Dataset(frame)).partitions()))
    for j, c in enumerate(names):
        lab = out[c].data
        assert lab.dtype == torch.int32 and lab.numel() == rows
        if j % 5 == 0:          # 8 of the 40 columns in full against the numpy oracle
            exp = oracle_hash_bucket(frame[c].data.cpu().numpy(), 1 << 20)
            np.testing.assert_array_equal(lab.cpu().numpy(), exp, err_msg=c)
        else:                   # the others on a strided 1/16 sample
            idx = torch.arange(j % 16, rows, 16, device="cuda")
            exp = oracle_hash_bucket(frame[c].data[idx].cpu().numpy(), 1 << 20)
            np.testing.assert_array_equal(lab[idx].cpu().numpy(), exp, err_msg=c)


# Categorify fit at 2^24 rows against pandas value_counts: the partitioned fold (4.45 M keys,
# DRAM-resident table) and the sorted accumulator (>= 8 M expected keys), one and three batches
@pytest.mark.parametrize("card,nparts", [(4_450_000, 1), (4_450_000, 3), (20_000_000, 1), (20_000_000, 4)])
def test_fit_large_cardinality_vs_value_counts(nvt, ops, tmp_path, card, nparts):
    import torch
    from nvtabular_b200.column import Column, DeviceFrame, pack_validity
    from nvtabular_b200.synth import power_law_ids, scatter_ids
    rows = 1 << 24
    g = torch.Generator(device="cuda").manual_seed(card % 1000 + nparts)
    keys = scatter_ids(power_law_ids(rows, card, g, "cuda"))
    valid = torch.rand(rows, generator=g, device="cuda") >= 0.04
    frame = DeviceFrame({"C": Column(keys, pack_validity(valid))})
    chunk = ((rows + nparts - 1) // nparts + 63) // 64 * 64
    parts = [frame.slice_rows(s, min(rows, s + chunk)) for s in range(0, rows, chunk)]
    op = ops.Categorify(out_path=str(tmp_path))
    wf = nvt.Workflow(["C"] >> op)
    wf.fit(nvt.Dataset(parts))
    fv = op.categories.fitted["C"]
    got_k, got_s = fv.vocab.export()
    ser = pd.Series(keys.cpu().numpy()[valid.cpu().numpy()])
    vc = ser.value_counts(sort=False)
    exp = pd.DataFrame({"k": vc.index.to_numpy(), "s": vc.to_numpy()}).sort_values(
        ["s", "k"], ascending=[False, True], kind="stable")
    np.testing.assert_array_equal(got_k.cpu().numpy(), exp["k"].to_numpy().astype(np.int64))
    np.testing.assert_array_equal(got_s.cpu().numpy(), exp["s"].to_numpy().astype(np.int64))
    assert fv.vocab.null_size == int((~valid).sum().item())
    # labels of a sample: position in that order + 3, nulls -> 1
    out = next(iter(wf.transform(nvt.Dataset(parts[0])).partitions()))
    n0 = len(parts[0])
    idx = np.arange(0, n0, 97)
    pos = pd.Series(np.arange(len(exp), dtype=np.int64) + 3, index=exp["k"].to_numpy())
    k_host = keys[:n0].cpu().numpy()[idx]
    v_host = valid[:n0].cpu().numpy()[idx]
    exp_lab = np.where(v_host, pos.reindex(k_host).to_numpy(), 1)
    np.testing.assert_array_equal(out["C"].data.cpu().numpy()[idx], exp_lab)
