"""Group-by payload statistics (HashAgg with n_agg > 0, csrc/hashagg.cu) on every table route,
against the exact reference of tests/_exact_stats.py.

One handle layout for every case, n_agg = 8 (kMaxAgg):
  0 int32    exact, k                      4 float64 exact, k·2^-20, validity mask
  1 int64    exact, c·2^25 (up to 2^40)    5 float64 general: N(1e6, 1e3), NaN holes, ±inf, -0.0
  2 uint8    exact, 0..255                 6 int32   exact, k, validity mask
  3 float32  exact, k·2^-8                 7 float32 exact, k·2^-8, null in every row of 1/8 of
                                             the groups, of the null-key group and of INT64_MIN
with |k|, |c| < 2^15.  Exact columns must match bit for bit whatever order the fp64 atomics
add in; the general column's sums must lie within the rounding bound of any summation order.
Keys and sizes are exact.  Group sizes are skewed (zipf), so the head slots take 1e4 to 1e6
atomics.  Each case says which route of insert / settle / merge it reaches and why, from the
sizing rules of predict(), prepare() and settle()."""
import numpy as np
import pytest
import torch

from _exact_stats import check_export, group_stats

pytestmark = pytest.mark.gpu

I64_MIN = np.iinfo(np.int64).min
EXPS = [0, -25, 0, 8, 20, None, 0, 8]
SAMPLE = 1 << 20                      # kSampleRows


@pytest.fixture(scope="module")
def eng():
    from nvtabular_b200 import engine
    return engine


def _col(arr, null=None):
    from nvtabular_b200.column import Column
    return Column.from_numpy(np.asarray(arr), null, device="cuda")


def _zipf_ids(rng, n, n_ids, zipf_frac):
    """ids in [0, n_ids): a zipf(1.2) head on `zipf_frac` of the rows, uniform on the rest"""
    z = (rng.zipf(1.2, n) - 1) % n_ids
    return np.where(rng.random(n) < zipf_frac, z, rng.integers(0, n_ids, n))


def _i32_keys(ids):
    return ((ids.astype(np.int64) * 2654435761) % (1 << 32)).astype(np.uint32).view(np.int32)   # negative too


def _i64_keys(ids):
    return (ids.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)).view(np.int64)            # beyond int32


def _allnull_groups(keys):
    return ((keys.astype(np.int64).view(np.uint64) * np.uint64(0xD6E8FEB86659FD93)) >> np.uint64(61)) == 0


class Data:
    """keys (+ null mask) and the 8 payload columns (+ null masks) of one case"""

    def __init__(self, rng, keys, key_null):
        n = len(keys)
        self.keys, self.key_null = keys, key_null
        k15 = lambda: rng.integers(-2 ** 15 + 1, 2 ** 15, n)   # noqa: E731
        c5 = rng.normal(0, 1e3, n) + 1e6
        c5[rng.random(n) < 0.05] = np.nan
        spots = rng.choice(n, 12, replace=False)
        c5[spots[:4]] = np.inf
        c5[spots[4:8]] = -np.inf
        c5[spots[8:]] = -0.0
        # one group holds both +inf and -inf: its sum is NaN
        same = np.flatnonzero(keys == keys[spots[0]])
        c5[same[-1] if same[-1] != spots[0] else spots[4]] = -np.inf
        self.cols = [k15().astype(np.int32), k15().astype(np.int64) << 25, rng.integers(0, 256, n).astype(np.uint8),
                     (k15() * 2.0 ** -8).astype(np.float32), k15() * 2.0 ** -20, c5, k15().astype(np.int32),
                     (k15() * 2.0 ** -8).astype(np.float32)]
        null7 = _allnull_groups(keys) | (keys == I64_MIN)
        if key_null is not None:
            null7 |= key_null
        self.nulls = [None, None, None, None, rng.random(n) < 0.1, None, rng.random(n) < 0.2, null7]

    def __len__(self):
        return len(self.keys)

    def ref(self):
        return group_stats(self.keys, self.key_null, self.cols, self.nulls, EXPS)

    def columns(self, s=0, e=None):
        """device key column and payload columns of rows [s, e) (s a multiple of 64)"""
        e = len(self) if e is None else e
        kn = self.key_null[s:e] if self.key_null is not None else None
        return _col(self.keys[s:e], kn), [_col(c[s:e], m[s:e] if m is not None else None)
                                            for c, m in zip(self.cols, self.nulls)]


def _export(h):
    k, s, v, ns, nv = h.export()
    return k.cpu().numpy(), s.cpu().numpy(), v.cpu().numpy(), ns, nv


def _check(h, ref, what):
    k, s, v, ns, nv = _export(h)
    check_export(ref, k, s, v, ns, nv, EXPS, what)
    return k, s, v, ns, nv


def _insert(eng, d, hint=0):
    h = eng.HashAgg(8, capacity_hint=hint) if hint else eng.HashAgg(8)
    kc, cs = d.columns()
    h.insert(kc, cs)
    return h


def test_payload_sized(eng):
    """200 k rows, 5 k int32 keys, 2 % null keys.  One insert of <= 4·2^20 rows takes no sample;
    with no hint and no estimate predict() assumes every row is a new key, so the table is
    next_pow2(2.5·200 k) = 512 K slots: nothing is refused and nothing grows."""
    rng = np.random.default_rng(101)
    n = 200_000
    d = Data(rng, _i32_keys(_zipf_ids(rng, n, 5000, 0.5)), rng.random(n) < 0.02)
    _check(_insert(eng, d), d.ref(), "sized")


def test_payload_blind_sample_then_growth(eng):
    """One insert of 6e6 rows over 3e6 int32 keys (10 % of the rows zipf).  With no hint and no
    estimate, an insert of more than 4·2^20 rows first takes the 2^20-row sample, for which
    predict() assumes 2^20 new keys: a table of next_pow2(2.5·2^20) = 4 M slots.  The sample shows
    817 k distinct keys, which inverts to K ≈ 2.08e6; for the remaining rows prepare() then
    predicts K(1 - exp(-6e6/K)) ≈ 1.96e6 keys and grows the table to 8 M slots, so rehash_kernel
    copies the payload of every live slot."""
    rng = np.random.default_rng(102)
    n = 6_000_000
    d = Data(rng, _i32_keys(_zipf_ids(rng, n, 3_000_000, 0.1)), rng.random(n) < 0.01)
    _check(_insert(eng, d), d.ref(), "blind sample + growth")


def test_payload_hint_far_too_low_uses_arena(eng):
    """HashAgg(8, capacity_hint=1000) and 1e6 distinct int32 keys in 2e6 rows.  The hint sizes the
    table to kMinCapacity = 65 536 slots and predict() keeps trusting it (predicted = hint), so
    the table fills and probes give up after 128 buckets: most rows go to the arena with their
    raw payload (the arena branch of insert_agg_kernel).  settle() then grows the table to
    next_pow2(4·(u + refused)) and folds the arena back in through merge_kernel."""
    rng = np.random.default_rng(103)
    n_keys, n = 1_000_000, 2_000_000
    ids = np.concatenate([np.arange(n_keys), _zipf_ids(rng, n - n_keys, n_keys, 0.5)])
    ids = ids[rng.permutation(n)]
    d = Data(rng, _i32_keys(ids), rng.random(n) < 0.01)
    _check(_insert(eng, d, hint=1000), d.ref(), "hint far too low")


def test_payload_adversarial_order_growth_and_arena(eng):
    """The first 2^20 + 4096 rows are ONE key, the remaining 6e6 rows all distinct.  The 2^20-row
    sample builds a 4 M-slot table and estimates K = 1, so prepare() does not grow it for the
    rest; the 6e6 distinct keys overflow it, refused rows go to the arena, and settle() grows the
    table (rehash_kernel copies the payload) and merges the arena (merge_kernel with payload).
    The single head key takes more than 1e6 atomics on one slot."""
    rng = np.random.default_rng(104)
    n_head, n_tail = SAMPLE + 4096, 6_000_000
    ids = np.concatenate([np.full(n_head, 7), np.arange(8, 8 + n_tail)])
    key_null = np.zeros(n_head + n_tail, dtype=bool)
    key_null[n_head:] = rng.random(n_tail) < 0.01      # nulls only after the sample
    d = Data(rng, _i32_keys(ids), key_null)
    _check(_insert(eng, d), d.ref(), "adversarial order")


def _i64_data(seed, n=1_000_000):
    rng = np.random.default_rng(seed)
    keys = _i64_keys(_zipf_ids(rng, n, 300_000, 0.5))
    keys[rng.random(n) < 0.1] = I64_MIN                 # the wide table's empty sentinel, frequent
    return Data(rng, keys, rng.random(n) < 0.03)


def test_payload_int64_keys_and_int64_min(eng):
    """int64 keys beyond int32, 3 % null keys, 10 % INT64_MIN keys (column 7 is null in all of
    those rows).  1e6 rows take no sample; the table is sized for 1e6 keys (4 M slots).  Null
    keys and INT64_MIN live in special_vals; export appends the INT64_MIN group last and hands
    the null group back on the host."""
    d = _i64_data(105)
    ref = d.ref()
    assert I64_MIN in ref.keys
    k, _, v, _, nv = _check(_insert(eng, d), ref, "int64 keys")
    assert k[-1] == I64_MIN                                            # appended last
    assert np.isnan(v[-1, 7, 2:]).all() and np.isnan(nv[7, 2:]).all()  # all-null payload: NaN min/max


def test_payload_batches_and_reuse(eng):
    """Three inserts of the rows [0, 192 064), [192 064, 960 000) and [960 000, 1.5e6), each a
    Column of its own (the kernel's own row offset into a column is reached by the sample of the
    blind-sample cases, off = 2^20), then reset() and the same three again through the same handle.  The first batch (192 k rows, 151 k keys) sizes a 512 K-slot
    table for the worst case; the second is sized from the estimate of the first (K ≈ 4.1e5, so
    about 3.7e5 keys expected after it), which grows the table to 1 M slots: rehash_kernel copies
    the payload.  reset() keeps the capacity and turns the seen key count into the hint: the
    second fit neither samples nor grows."""
    rng = np.random.default_rng(106)
    n = 1_500_000
    d = Data(rng, _i32_keys(_zipf_ids(rng, n, 600_000, 0.1)), rng.random(n) < 0.02)
    ref = d.ref()
    bounds = [0, 64 * 3001, 64 * 15000, n]
    h = eng.HashAgg(8)
    for rnd in range(2):
        if rnd:
            h.reset()
        for s, e in zip(bounds[:-1], bounds[1:]):
            kc, cs = d.columns(s, e)
            h.insert(kc, cs)
        _check(h, ref, f"batches, fit {rnd}")


def _split_exports(eng, d, K):
    bounds = [(len(d) * i // K) // 64 * 64 for i in range(K)] + [len(d)]
    outs = []
    for s, e in zip(bounds[:-1], bounds[1:]):
        h = eng.HashAgg(8)
        kc, cs = d.columns(s, e)
        h.insert(kc, cs)
        outs.append(h.export())
    return outs, bounds


def _merge_data():
    d = _i64_data(107)
    # column 6 is null in every row of 1/4 of the groups INSIDE the first partial only: that
    # partial exports NaN min/max for them, which the merge must skip, not propagate
    first = np.zeros(len(d), dtype=bool)
    first[: (len(d) // 4) // 64 * 64] = True
    cls = ((d.keys.view(np.uint64) * np.uint64(0xC2B2AE3D27D4EB4F)) >> np.uint64(62)) == 1
    d.nulls[6] = d.nulls[6] | (first & cls)
    return d


def test_payload_merge_of_partials(eng):
    """K = 4 partial handles, exported, then merge() + add_null_group() into one handle (the tree
    merge).  Every partial holds the INT64_MIN key (merge_kernel routes it to special_vals); the
    null-key group's min/max are merged on the host (enc_ordered).  The result equals the single
    handle and the reference."""
    d = _merge_data()
    ref = d.ref()
    single = _check(_insert(eng, d), ref, "single handle")
    outs, _ = _split_exports(eng, d, 4)
    hm = eng.HashAgg(8)
    for pk, ps, pv, pn, pnv in outs:
        assert (pk.cpu().numpy() == I64_MIN).any()
        hm.merge(pk, ps, pv.reshape(-1))
        hm.add_null_group(pn, pnv.reshape(-1))
    k, s, v, ns, nv = _check(hm, ref, "merged")
    o1, o2 = np.argsort(single[0]), np.argsort(k)
    np.testing.assert_array_equal(k[o2], single[0][o1])
    np.testing.assert_array_equal(s[o2], single[1][o1])
    assert ns == single[3]


@pytest.mark.parametrize("W", [2, 3, 8])
def test_payload_simulated_owners(eng, W):
    """The owner-side merge of the multi-GPU fit, on one GPU: the exports of 4 partials are
    concatenated (a key appears in several partials), partition_by_owner groups the rows by
    owner, gather_i64 / gather_f64_rows(width = 4·n_agg) reorder them, and each owner merges
    its segment into its own handle.  Every key must land in exactly one owner and the union
    of the owners must equal the single table."""
    d = _merge_data()
    ref = d.ref()
    outs, _ = _split_exports(eng, d, 4)
    ak = torch.cat([o[0] for o in outs])
    asz = torch.cat([o[1] for o in outs])
    av = torch.cat([o[2] for o in outs]).reshape(-1, 32)
    perm, counts = eng.partition_by_owner(ak, W)
    assert sum(counts) == ak.numel()
    gk, gs = eng.gather_i64(ak, perm), eng.gather_i64(asz, perm)
    gv = eng.gather_f64_rows(av, perm, 32)
    p = perm.cpu().numpy()
    np.testing.assert_array_equal(gv.cpu().numpy(), av.cpu().numpy()[p])
    np.testing.assert_array_equal(gk.cpu().numpy(), ak.cpu().numpy()[p])
    ks, ss, vs, owner_of = [], [], [], {}
    off = 0
    for w, c in enumerate(counts):
        h = eng.HashAgg(8, capacity_hint=max(c, 1))
        h.merge(gk[off:off + c], gs[off:off + c], gv[off:off + c].reshape(-1))
        off += c
        k, s, v, ns, _ = _export(h)
        assert ns == 0
        for key in np.unique(k).tolist():
            assert owner_of.setdefault(key, w) == w, f"key {key} in owners {owner_of[key]} and {w}"
        ks.append(k); ss.append(s); vs.append(v)
    k, s, v = np.concatenate(ks), np.concatenate(ss), np.concatenate(vs)
    assert len(np.unique(k)) == len(k)
    # the null-key group does not travel between owners (test_payload_merge_of_partials checks it)
    check_export(ref, k, s, v, ref.null_size, ref.null_stats, EXPS, f"owners W={W}")


@pytest.mark.parametrize("width", [1, 4, 32])
@pytest.mark.parametrize("n", [0, 1, 1000, 300_007])
def test_gather_f64_rows(eng, width, n):
    rng = np.random.default_rng(width * 1000 + n)
    rows = n + 17
    src = torch.tensor(rng.standard_normal((rows, width)), device="cuda")
    perm = torch.tensor(rng.integers(0, rows, n), dtype=torch.int64, device="cuda")
    out = eng.gather_f64_rows(src, perm, width)
    assert out.shape == (n, width)
    np.testing.assert_array_equal(out.cpu().numpy(), src.cpu().numpy()[perm.cpu().numpy()])


def test_groupstats_gather_more_than_one_launch_of_columns(eng):
    """JoinGroupby gathers every statistic of a group in one call (7 stats of 3 columns = 19
    columns); one launch holds 16 output columns, so the call takes several.  Outputs asked for
    with a validity bitmask are valid exactly where the key has a row and the value is not NaN;
    an integer output holds 0 elsewhere."""
    from nvtabular_b200.column import unpack_validity
    rng = np.random.default_rng(71)
    keys = torch.tensor(rng.permutation(5000)[:2000].astype("int64") * 7, device="cuda")
    width = 40
    st = rng.standard_normal((2001, width)) * 1e3                              # row 2000 = null group
    st[rng.random(st.shape) < 0.05] = np.nan
    stats = torch.tensor(st, device="cuda")
    dts = ["float64", "float32", "int64", "int32"] * 10
    cols = [int(c) for c in rng.permutation(width)[:37]]
    for null_row in (2000, -1):
        g = eng.GroupStats(keys, stats, null_row=null_row)
        for n in (0, 1, 33, 50_001):
            data = rng.integers(0, 35000, n)
            mask = rng.random(n) < 0.05
            masked = [j % 3 != 1 for j in range(37)]
            outs = g.gather_columns(_col(data, mask), cols, [float(-c) for c in cols], dts[:37], masked)
            lut = {int(k): i for i, k in enumerate(keys.cpu().numpy())}
            rows = np.array([null_row if m else lut.get(int(d), -1) for d, m in zip(data, mask)], dtype=np.int64)
            for j, c in enumerate(cols):
                v = np.where(rows >= 0, st[np.maximum(rows, 0), c], -c)
                ok = (rows >= 0) & ~np.isnan(v)
                exp = np.where(np.isnan(v), 0, v).astype(dts[j]) if dts[j].startswith("int") else v.astype(dts[j])
                o = outs[j]
                assert o.data.dtype == getattr(torch, dts[j]) and o.data.numel() == n
                np.testing.assert_array_equal(o.data.cpu().numpy(), exp, err_msg=f"output {j}, n={n}")
                if masked[j]:
                    got_ok = unpack_validity(o.validity, n).cpu().numpy() if n else np.zeros(0, bool)
                    np.testing.assert_array_equal(got_ok, ok, err_msg=f"validity {j}, n={n}")
                    tail = o.validity.cpu().numpy()
                    assert not (np.unpackbits(tail, bitorder="little")[n:]).any(), "bits past the last row"
                else:
                    assert o.validity is None
            plain = g.gather(_col(data, mask), cols[:3], [float(-c) for c in cols[:3]], dts[:3])
            for j in range(3):
                np.testing.assert_array_equal(plain[j].cpu().numpy(), outs[j].data.cpu().numpy())
