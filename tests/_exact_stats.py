"""Exact per-group payload statistics: the reference the group-by kernels are compared with.

`group_stats` computes, for every non-null key (INT64_MIN is an ordinary key here) and for the
null-key group, the size and per payload column {sum, sumsq, min, max} as csrc/hashagg.cu defines
them: x is the value cast to float64 (`load_agg`), sum = Σ x, sumsq = Σ fl(x·x), NaN or a masked
row is null, and min/max of a group without a single value are NaN.

Two kinds of column, because fp64 atomics add in any order:

* exact columns (`exps[j]` = e): every value is k·2^-e with |k| < 2^15, and no group has more
  than 2^22 rows, so Σk < 2^37 and Σk² < 2^52.  Every partial sum of x and of x² is then a
  representable double: any summation order gives the same bits.  The sums are computed on int64
  integers and scaled once, so the kernel must match them bit for bit.
* general float64 columns (`exps[j]` is None): sums are `math.fsum` of the finite values, with
  +inf / -inf / NaN(+inf and -inf) decided from the infinities of the group.  `bound[..., 0:2]`
  holds gamma_{n_g - 1}·Σ|x| + ulp(ref) for sum and sumsq (gamma_k = k·2^-53 / (1 - k·2^-53)),
  which bounds the rounding error of any summation order; min and max stay exact.
"""
import math
from typing import List, NamedTuple, Optional, Sequence

import numpy as np


class GroupStats(NamedTuple):
    keys: np.ndarray        # int64[G], ascending
    sizes: np.ndarray       # int64[G]
    stats: np.ndarray       # float64[G, m, 4]  {sum, sumsq, min, max}
    bound: np.ndarray       # float64[G, m, 2]  allowed |got - ref| of sum, sumsq (0 for exact columns)
    null_size: int
    null_stats: np.ndarray  # float64[m, 4]
    null_bound: np.ndarray  # float64[m, 2]


def _seg_sum_i64(v: np.ndarray, starts: np.ndarray, ends: np.ndarray) -> np.ndarray:
    c = np.concatenate([[0], np.cumsum(v, dtype=np.int64)])
    return c[ends] - c[starts]


def _seg_reduce(ufunc, v: np.ndarray, starts: np.ndarray, ends: np.ndarray, empty: float) -> np.ndarray:
    out = np.full(len(starts), empty, dtype=np.float64)
    ne = ends > starts
    if ne.any() and len(v):
        out[ne] = ufunc.reduceat(v, starts[ne])
    return out


def _fsum_segments(v: np.ndarray, starts: np.ndarray, ends: np.ndarray) -> np.ndarray:
    """correctly rounded sum of each segment (a segment of <= 2 values needs one rounding only)"""
    lens = ends - starts
    out = np.zeros(len(starts), dtype=np.float64)
    one = lens == 1
    out[one] = v[starts[one]]
    two = lens == 2
    out[two] = v[starts[two]] + v[starts[two] + 1]
    for g in np.flatnonzero(lens > 2):
        out[g] = math.fsum(v[starts[g]:ends[g]])
    return out


def group_stats(keys: np.ndarray, key_null: Optional[np.ndarray], cols: Sequence[np.ndarray],
                col_nulls: Sequence[Optional[np.ndarray]], exps: Sequence[Optional[int]]) -> GroupStats:
    keys = np.asarray(keys, dtype=np.int64)
    n = len(keys)
    key_null = np.zeros(n, dtype=bool) if key_null is None else np.asarray(key_null, dtype=bool)
    m = len(cols)
    # rows ordered by key, the null-key rows last: one segment per group, the last one = null group
    valid_rows = np.flatnonzero(~key_null)
    order = valid_rows[np.argsort(keys[valid_rows], kind="stable")]
    ks = keys[order]
    heads = np.flatnonzero(np.r_[True, ks[1:] != ks[:-1]]) if len(ks) else np.zeros(0, dtype=np.int64)
    uniq = ks[heads]
    rows = np.concatenate([order, np.flatnonzero(key_null)])
    starts = np.concatenate([heads, [len(order)]]).astype(np.int64)
    ends = np.concatenate([heads[1:], [len(order)], [n]]).astype(np.int64)
    G = len(uniq)
    stats = np.zeros((G + 1, m, 4), dtype=np.float64)
    bound = np.zeros((G + 1, m, 2), dtype=np.float64)
    for j, (col, null, e) in enumerate(zip(cols, col_nulls, exps)):
        raw = np.asarray(col)[rows]
        x = raw.astype(np.float64)
        isnull = np.isnan(x)
        if null is not None:
            isnull |= np.asarray(null, dtype=bool)[rows]
        ok = ~isnull
        cnt = _seg_sum_i64(ok.astype(np.int64), starts, ends)
        xv = np.where(ok, x, 0.0)
        stats[:, j, 2] = _seg_reduce(np.minimum, np.where(ok, x, np.inf), starts, ends, np.inf)
        stats[:, j, 3] = _seg_reduce(np.maximum, np.where(ok, x, -np.inf), starts, ends, -np.inf)
        stats[cnt == 0, j, 2:] = np.nan
        if e is not None:
            k = np.where(ok, raw, 0).astype(np.int64) if raw.dtype.kind in "iu" else None
            if k is None or e != 0:
                k = xv * (2.0 ** e)
                assert np.all(k == np.round(k)) and np.all(np.abs(k) < 2 ** 15), f"column {j} is not k*2^-{e}"
                k = k.astype(np.int64)
            assert np.all(np.abs(k) < 2 ** 15), f"column {j}: |k| >= 2^15"
            s = _seg_sum_i64(k, starts, ends)
            s2 = _seg_sum_i64(k * k, starts, ends)
            assert np.all(s2 < 2 ** 52), f"column {j}: a group's sum of squares is not exact"
            stats[:, j, 0] = s.astype(np.float64) * 2.0 ** -e
            stats[:, j, 1] = s2.astype(np.float64) * 2.0 ** (-2 * e)
            continue
        fin = ok & np.isfinite(x)
        xf = np.where(fin, x, 0.0)
        sq = xf * xf
        n_fin = _seg_sum_i64(fin.astype(np.int64), starts, ends)
        n_pos = _seg_sum_i64((ok & (x == np.inf)).astype(np.int64), starts, ends)
        n_neg = _seg_sum_i64((ok & (x == -np.inf)).astype(np.int64), starts, ends)
        # the finite values of each group, contiguous: sort rows by (segment, not finite)
        seg = np.repeat(np.arange(G + 1), ends - starts)
        fo = np.lexsort((~fin, seg))
        fstarts = starts
        fends = starts + n_fin
        s = _fsum_segments(xf[fo], fstarts, fends)
        s2 = _fsum_segments(sq[fo], fstarts, fends)
        abs_s = _seg_reduce(np.add, np.abs(xf[fo]), fstarts, fends, 0.0)
        abs_s2 = _seg_reduce(np.add, sq[fo], fstarts, fends, 0.0)
        # any order of n additions is within gamma_{n-1}·Σ|x| of the exact sum, gamma_k = k·u / (1 - k·u);
        # abs_s is itself a float sum of non-negative terms, at most a factor (1 - gamma) below Σ|x|,
        # and (1 + 2^-50) covers the roundings of this line.  ulp(ref) covers ref's own rounding.
        ku = np.maximum(n_fin - 1, 0) * 2.0 ** -53
        gamma = ku / (1 - ku)
        slack = gamma / (1 - gamma) * (1 + 2.0 ** -50)
        bound[:, j, 0] = slack * abs_s + np.spacing(np.abs(s))
        bound[:, j, 1] = slack * abs_s2 + np.spacing(np.abs(s2))
        s = np.where(n_pos > 0, np.inf, s)
        s = np.where(n_neg > 0, -np.inf, s)
        s = np.where((n_pos > 0) & (n_neg > 0), np.nan, s)
        s2 = np.where(n_pos + n_neg > 0, np.inf, s2)
        stats[:, j, 0] = s
        stats[:, j, 1] = s2
    sizes = (ends - starts)[:G].astype(np.int64)
    return GroupStats(uniq, sizes, stats[:G], bound[:G], int(key_null.sum()), stats[G], bound[G])


def assert_stats_close(got: np.ndarray, ref: np.ndarray, bound: np.ndarray, exps: Sequence[Optional[int]],
                       what: str = ""):
    """got/ref float64[..., m, 4], bound float64[..., m, 2]: exact columns bit for bit (NaN == NaN),
    general columns' sums within the bound (non-finite sums exactly), min/max exact.
    The sign of a zero min/max is not checked: assert_array_equal treats -0.0 == 0.0."""
    for j, e in enumerate(exps):
        names = ("sum", "sumsq", "min", "max")
        for q in range(4):
            g, r = got[..., j, q], ref[..., j, q]
            msg = f"{what} column {j} {names[q]}"
            if e is not None or q >= 2:
                np.testing.assert_array_equal(g, r, err_msg=msg)
                continue
            fin = np.isfinite(r)
            np.testing.assert_array_equal(g[~fin], r[~fin], err_msg=msg + " (non-finite)")
            err = np.abs(g[fin] - r[fin])
            b = bound[..., j, q][fin]
            bad = ~(err <= b)
            assert not bad.any(), (f"{msg}: {int(bad.sum())} groups outside the bound, e.g. got {g[fin][bad][:3]} "
                                   f"ref {r[fin][bad][:3]} bound {b[bad][:3]}")


def check_export(ref: GroupStats, keys, sizes, vals, null_size, null_vals, exps, what: str = ""):
    """compare a HashAgg export (any row order) with the reference"""
    k = np.asarray(keys)
    order = np.argsort(k, kind="stable")
    np.testing.assert_array_equal(k[order], ref.keys, err_msg=f"{what} keys")
    np.testing.assert_array_equal(np.asarray(sizes)[order], ref.sizes, err_msg=f"{what} sizes")
    assert null_size == ref.null_size, (what, null_size, ref.null_size)
    assert_stats_close(np.asarray(vals)[order], ref.stats, ref.bound, exps, what)
    assert_stats_close(np.asarray(null_vals)[None], ref.null_stats[None], ref.null_bound[None], exps, f"{what} null group")
