"""CPU tests of the exact group-statistics reference (tests/_exact_stats.py) that the payload
group-by kernels are checked against: it must agree with pandas groupby(dropna=False), give
exactly the rational sums on columns of the exact kind, and its checker must reject a one-ulp
error on an exact column."""
import math
from fractions import Fraction

import numpy as np
import pandas as pd
import pytest

from _exact_stats import assert_stats_close, group_stats

I64_MIN = np.iinfo(np.int64).min


def _frame(seed, n, n_keys):
    rng = np.random.default_rng(seed)
    keys = rng.integers(-n_keys, n_keys, n).astype(np.int64) * (1 << 33)
    keys[rng.random(n) < 0.1] = I64_MIN
    key_null = rng.random(n) < 0.08
    a = rng.integers(-2 ** 15 + 1, 2 ** 15, n).astype(np.int32)                     # exact, e = 0
    b = (rng.integers(-2 ** 15 + 1, 2 ** 15, n) * 2.0 ** -7).astype(np.float32)     # exact, e = 7
    b_null = rng.random(n) < 0.2
    c = rng.normal(0, 1e3, n) + 1e6                                                   # general
    c[rng.random(n) < 0.1] = np.nan
    c[rng.integers(0, n, 3)] = -0.0
    d = rng.integers(0, 256, n).astype(np.uint8)                                      # exact, e = 0
    d_null = np.isin(keys, keys[:3]) | key_null             # null in every row of some groups
    return keys, key_null, [a, b, c, d], [None, b_null, None, d_null], [0, 7, None, 0]


@pytest.mark.parametrize("seed,n,n_keys", [(1, 1, 1), (2, 50, 3), (3, 2000, 40), (4, 5000, 2000)])
def test_exact_stats_agree_with_pandas(seed, n, n_keys):
    keys, key_null, cols, nulls, exps = _frame(seed, n, n_keys)
    ref = group_stats(keys, key_null, cols, nulls, exps)
    df = pd.DataFrame({"k": pd.array(np.where(key_null, 0, keys), dtype="Int64")})
    df.loc[key_null, "k"] = pd.NA
    agg = {}
    for j, (c, m) in enumerate(zip(cols, nulls)):
        x = c.astype(np.float64)
        if m is not None:
            x = np.where(m, np.nan, x)
        df[f"x{j}"] = x
        df[f"q{j}"] = x * x
        agg.update({f"s{j}": (f"x{j}", "sum"), f"s2{j}": (f"q{j}", "sum"),
                    f"mn{j}": (f"x{j}", "min"), f"mx{j}": (f"x{j}", "max")})
    g = df.groupby("k", dropna=False).agg(size=("k", "size"), **agg)
    isnull = g.index.isna()
    gv = g[~isnull].sort_index()
    np.testing.assert_array_equal(ref.keys, gv.index.to_numpy(dtype=np.int64))
    np.testing.assert_array_equal(ref.sizes, gv["size"].to_numpy())
    assert ref.null_size == (int(g[isnull]["size"].iloc[0]) if isnull.any() else 0)
    for j in range(len(cols)):
        for q, name in enumerate(("s", "s2", "mn", "mx")):
            exp = gv[f"{name}{j}"].to_numpy(dtype=np.float64)
            got = ref.stats[:, j, q]
            if q < 2:
                np.testing.assert_allclose(got, exp, rtol=1e-12, atol=0, err_msg=f"{name}{j}")
            else:
                np.testing.assert_array_equal(got, exp, err_msg=f"{name}{j}")
            if isnull.any():
                e0 = float(g[isnull][f"{name}{j}"].iloc[0])
                got0 = ref.null_stats[j, q]
                assert (math.isnan(e0) and math.isnan(got0)) or got0 == pytest.approx(e0, rel=1e-12), (name, j)
    # the all-null groups of column 3 have NaN min/max and zero sums
    allnull = np.isin(ref.keys, keys[:3][~key_null[:3]])
    assert np.isnan(ref.stats[allnull, 3, 2:]).all() and (ref.stats[allnull, 3, :2] == 0).all()


def test_exact_stats_sums_are_the_rational_sums():
    keys, key_null, cols, nulls, exps = _frame(5, 3000, 30)
    ref = group_stats(keys, key_null, cols, nulls, exps)
    for j, e in enumerate(exps):
        if e is None:
            continue
        x = cols[j].astype(np.float64)
        m = np.zeros(len(x), bool) if nulls[j] is None else nulls[j]
        for gi, k in enumerate(ref.keys[:40].tolist() + [None]):
            rows = np.flatnonzero(key_null) if k is None else np.flatnonzero((keys == k) & ~key_null)
            vals = [Fraction(float(v)) for v in x[rows][~m[rows]]]
            s, s2 = sum(vals, Fraction(0)), sum((v * v for v in vals), Fraction(0))
            got = ref.null_stats[j] if k is None else ref.stats[gi, j]
            assert Fraction(float(got[0])) == s and Fraction(float(got[1])) == s2, (j, k)


def test_exact_stats_general_column_edges():
    # +inf and -inf in one group: NaN sum; one infinity: that infinity; -0.0 and NaN holes
    keys = np.array([1, 1, 1, 2, 2, 3, 3, 4], dtype=np.int64)
    x = np.array([np.inf, -np.inf, 5.0, np.inf, 1.0, -0.0, np.nan, np.nan])
    ref = group_stats(keys, None, [x], [None], [None])
    s = ref.stats[:, 0]
    assert math.isnan(s[0, 0]) and s[0, 1] == np.inf and s[0, 2] == -np.inf and s[0, 3] == np.inf
    assert s[1, 0] == np.inf and s[1, 2] == 1.0
    assert s[2, 0] == 0.0 and s[2, 2] == 0.0 and s[2, 3] == 0.0
    assert s[3, 0] == 0.0 and np.isnan(s[3, 2:]).all()
    # large cancellations: the reference is the correctly rounded sum
    y = np.array([1e16, 1.0, -1e16, 1.0, 3.0, 2.0 ** -30], dtype=np.float64)
    ref = group_stats(np.zeros(6, np.int64), None, [y], [None], [None])
    assert ref.stats[0, 0, 0] == math.fsum(y)


def test_exact_stats_checker_rejects_one_ulp():
    keys, key_null, cols, nulls, exps = _frame(6, 4000, 50)
    ref = group_stats(keys, key_null, cols, nulls, exps)
    assert_stats_close(ref.stats, ref.stats, ref.bound, exps)
    for j, q in [(0, 0), (1, 1), (3, 0), (2, 2)]:       # exact sums, exact sumsq, general min
        bad = ref.stats.copy()
        g = int(np.flatnonzero(np.isfinite(bad[:, j, q]) & (bad[:, j, q] != 0))[0])
        bad[g, j, q] = np.nextafter(bad[g, j, q], np.inf)
        with pytest.raises(AssertionError):
            assert_stats_close(bad, ref.stats, ref.bound, exps)
    # a general sum off by much more than the rounding bound
    bad = ref.stats.copy()
    g = int(np.argmax(ref.sizes))
    bad[g, 2, 0] += 1e-3 * abs(bad[g, 2, 0])
    with pytest.raises(AssertionError):
        assert_stats_close(bad, ref.stats, ref.bound, exps)
