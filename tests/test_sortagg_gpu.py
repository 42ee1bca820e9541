"""GPU parity tests of the radix-sort primitive (csrc/radix.cuh) and the sort-based
group-by for high-cardinality int32 columns (csrc/sortagg.cuh) through the C-ABI, against
torch.sort / torch.unique (independent implementations of the pandas semantics the
oracle restates: value_counts, sort_values — reference nvtabular/ops/categorify.py:1018,
1300, 1316)."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _engine():
    from nvtabular_b200 import engine
    from nvtabular_b200.column import Column, pack_validity
    return engine, Column, pack_validity


@pytest.mark.parametrize("n", [1, 100, 8192, 8193, 100_000, 3_000_001])
def test_radix_sort_u32_full(n):
    engine, _, _ = _engine()
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randint(-2**31, 2**31 - 1, (n,), generator=g, device="cuda", dtype=torch.int64).to(torch.int32)
    got = engine.radix_sort(x)                                   # unsigned order of the bit pattern
    exp = torch.sort(x.to(torch.int64) & 0xFFFFFFFF).values
    assert torch.equal(got.to(torch.int64) & 0xFFFFFFFF, exp)


@pytest.mark.parametrize("lo,hi", [(0, 8), (12, 32), (0, 20), (5, 16)])
def test_radix_sort_u32_bit_range_is_stable(lo, hi):
    engine, _, _ = _engine()
    n = 777_777
    g = torch.Generator(device="cuda").manual_seed(lo * 100 + hi)
    x = torch.randint(0, 2**31 - 1, (n,), generator=g, device="cuda", dtype=torch.int64).to(torch.int32)
    got = engine.radix_sort(x, lo, hi)
    field = (x.to(torch.int64) >> lo) & ((1 << (hi - lo)) - 1)
    order = torch.sort(field, stable=True).indices
    assert torch.equal(got, x[order])


@pytest.mark.parametrize("n,bits", [(5, 3), (50_000, 10), (2_000_003, 17), (400_000, 32)])
def test_radix_sort_u64_low_bits_descending_stable(n, bits):
    """the vocabulary ordering: packed (key << 32 | size) sorted by size DESC keeps key order"""
    engine, _, _ = _engine()
    g = torch.Generator(device="cuda").manual_seed(n)
    size = torch.randint(0, 2**min(bits, 31), (n,), generator=g, device="cuda", dtype=torch.int64)
    key = torch.arange(n, device="cuda", dtype=torch.int64)
    packed = (key << 32) | size
    got = engine.radix_sort(packed, 0, bits, descending=True)
    order = torch.sort(size, stable=True, descending=True).indices
    assert torch.equal(got, packed[order])


def test_radix_sort_u64_high_bits():
    engine, _, _ = _engine()
    n = 1_234_567
    g = torch.Generator(device="cuda").manual_seed(7)
    hi = torch.randint(0, 2**32 - 1, (n,), generator=g, device="cuda", dtype=torch.int64)
    lo = torch.arange(n, device="cuda", dtype=torch.int64)
    packed = ((hi << 32) | lo)
    got = engine.radix_sort(packed, 32, 64)
    order = torch.sort(hi, stable=True).indices
    assert torch.equal(got, packed[order])


def _ref_counts(keys, valid):
    k = keys[valid] if valid is not None else keys
    u, c = torch.unique(k.to(torch.int64), return_counts=True)
    return u, c


def _insert_batches(engine, Column, pack_validity, keys, valid, cuts, agg=None):
    agg = agg or engine.HashAgg(0)
    for a, b in zip(cuts[:-1], cuts[1:]):
        v = pack_validity(valid[a:b]) if valid is not None else None
        agg.insert(Column(keys[a:b].contiguous(), v))
    return agg


@pytest.mark.parametrize("card,n", [(50_000_000, 2_000_000), (300_000, 1_500_000), (7, 600_000)])
@pytest.mark.parametrize("with_nulls", [False, True])
@pytest.mark.parametrize("ragged", [False, True])
def test_sorted_accumulator_counts(monkeypatch, card, n, with_nulls, ragged):
    """every batch grouped and merged: exact value_counts incl. nulls.  ragged: the first batch is not
    a multiple of 8 rows long, so the batch after it bypasses the staging buffer (the staged rows are
    flushed and it goes in on its own)."""
    engine, Column, pack_validity = _engine()
    monkeypatch.setenv("NVTB_RUNS_MIN_KEYS", "1")
    g = torch.Generator(device="cuda").manual_seed(card % 1000 + n % 97)
    keys = (torch.randint(0, card, (n,), generator=g, device="cuda", dtype=torch.int64) * 2654435761 % (2**32) - 2**31).to(torch.int32)
    valid = (torch.rand(n, generator=g, device="cuda") > 0.07) if with_nulls else None
    cuts = [0, 64 * 4000, 64 * 4000 + 64 * 9001, n]              # three uneven batches (64-row aligned cuts)
    if ragged:
        cuts = [0, 64 * 4000 + 3, 64 * 4000 + 64 * 9001, n]
    agg = _insert_batches(engine, Column, pack_validity, keys, valid, cuts)
    assert agg.mode == 1
    k, s, _, null_size, _ = agg.export()
    u, c = _ref_counts(keys, valid)
    assert torch.equal(k, u)                                     # a sorted accumulator exports in key order
    assert torch.equal(s, c)
    assert null_size == (0 if valid is None else int((~valid).sum()))
    # reset keeps the mode; a second fit over the same data gives the same answer
    agg.reset()
    agg = _insert_batches(engine, Column, pack_validity, keys, valid, [0, n], agg)
    assert agg.mode == 1
    k2, s2, _, ns2, _ = agg.export()
    assert torch.equal(k2, u) and torch.equal(s2, c) and ns2 == null_size


def test_table_converts_to_sorted_accumulator(monkeypatch):
    """a handle that starts as a hash table (blind sample) and crosses the threshold later"""
    engine, Column, pack_validity = _engine()
    monkeypatch.setenv("NVTB_RUNS_MIN_KEYS", str(1 << 40))
    n = 3_000_000
    g = torch.Generator(device="cuda").manual_seed(5)
    keys = torch.randint(-2**31, 2**31 - 1, (n,), generator=g, device="cuda", dtype=torch.int64).to(torch.int32)
    agg = engine.HashAgg(0)
    agg.insert(Column(keys[: 64 * 10000].contiguous()))
    assert agg.mode == 0
    monkeypatch.setenv("NVTB_RUNS_MIN_KEYS", "1000")
    agg.insert(Column(keys[64 * 10000:].contiguous()))
    assert agg.mode == 1
    k, s, _, ns, _ = agg.export()
    u, c = _ref_counts(keys, None)
    assert torch.equal(k, u) and torch.equal(s, c) and ns == 0


def test_unaligned_batch_into_sorted_accumulator(monkeypatch):
    engine, Column, pack_validity = _engine()
    monkeypatch.setenv("NVTB_RUNS_MIN_KEYS", "1")
    n = 500_003
    g = torch.Generator(device="cuda").manual_seed(11)
    base = torch.randint(0, 1000, (n + 1,), generator=g, device="cuda", dtype=torch.int64).to(torch.int32)
    keys = base[1:]                                              # 4-byte aligned only
    agg = engine.HashAgg(0)
    agg.insert(Column(keys))
    assert agg.mode == 1
    k, s, _, _, _ = agg.export()
    u, c = _ref_counts(keys, None)
    assert torch.equal(k, u) and torch.equal(s, c)


@pytest.mark.parametrize("cut", ["none", "freq", "max_size"])
def test_vocab_from_sorted_accumulator(monkeypatch, cut):
    """(size desc, key asc) + cut + meta + labels, straight from the handle"""
    engine, Column, pack_validity = _engine()
    monkeypatch.setenv("NVTB_RUNS_MIN_KEYS", "1")
    n = 2_500_000
    g = torch.Generator(device="cuda").manual_seed(23)
    # power-law-ish counts: many keys with 1-3 rows, a few with thousands
    ids = (torch.rand(n, generator=g, device="cuda", dtype=torch.float64) ** 6 * 400_000).to(torch.int64)
    keys = ((ids * 2654435761) % (2**31)).to(torch.int32)
    valid = torch.rand(n, generator=g, device="cuda") > 0.03
    agg = _insert_batches(engine, Column, pack_validity, keys, valid, [0, 64 * 20000, n])
    assert agg.mode == 1
    ft, ms = (3, 0) if cut == "freq" else ((0, 5000) if cut == "max_size" else (0, 0))
    vocab = engine.Vocab.build_from_agg(agg, ft, ms, 0, 32, n)
    u, c = _ref_counts(keys, valid)
    order = torch.sort(c, stable=True, descending=True).indices      # u is key-ascending
    u, c = u[order], c[order]
    if cut == "freq":
        keep = int((c >= 3).sum())
    elif cut == "max_size":
        keep = min(len(u), 5000 - 3)
    else:
        keep = len(u)
    assert vocab.n_kept == keep and vocab.n_total == len(order)
    k, s = vocab.export()
    assert torch.equal(k, u[:keep]) and torch.equal(s, c[:keep])
    assert vocab.null_size == int((~valid).sum())
    assert vocab.unique_size == int(c[:keep].sum()) and vocab.oov_size == int(c[keep:].sum())
    labels = vocab.encode(Column(keys, pack_validity(valid)), 1, 2, 3, 0, (), np.int64)
    pos = torch.full((int(u.max()) + 2,), -1, dtype=torch.int64, device="cuda") if False else None
    # reference labels through a sorted search on the kept keys
    kk, perm = torch.sort(u[:keep])
    idx = torch.searchsorted(kk, keys.to(torch.int64)).clamp_(max=max(keep - 1, 0))
    hit = (kk[idx] == keys.to(torch.int64)) if keep else torch.zeros(n, dtype=torch.bool, device="cuda")
    exp = torch.where(hit, perm[idx] + 3, torch.full_like(idx, 2))
    exp = torch.where(valid, exp, torch.ones_like(exp))
    assert torch.equal(labels, exp)


@pytest.mark.parametrize("shape", ["uniform32", "dense_small_range", "heavy_hitters", "cluster_fallback"])
@pytest.mark.parametrize("stage_rows", [None, 64 * 20000, 0])
def test_bucket_groupby_paths_agree(monkeypatch, shape, stage_rows):
    """The staged batches of a sorted accumulator are grouped by ONE range partition + direct-address
    counting in shared memory (csrc/bucketagg.cuh); the radix pipeline (NVTB_SORT_PATH=radix) is the
    fallback when a window holds more duplicated values than the counters a CTA has.  Both must give
    torch.unique's answer for: keys over the whole int32 range; a dense small range (the window
    shrinks to a few values); a few values with millions of rows each; and a dense cluster inside a
    wide range (more than 14 336 duplicated values in one 2^18 window: the fallback fires).
    stage_rows: one flush per fit (None); a stage smaller than the fit (64 * 20000: the second batch
    flushes the first, the third flushes the second into a non-empty accumulator and then goes in
    on its own); or no staging, one group-by + merge per batch (0)."""
    engine, Column, pack_validity = _engine()
    monkeypatch.setenv("NVTB_RUNS_MIN_KEYS", "1")
    if stage_rows is not None:
        monkeypatch.setenv("NVTB_STAGE_ROWS", str(stage_rows))
    n = 4_000_000
    g = torch.Generator(device="cuda").manual_seed(len(shape))
    if shape == "uniform32":
        keys = torch.randint(-2**31, 2**31 - 1, (n,), generator=g, device="cuda", dtype=torch.int64)
    elif shape == "dense_small_range":
        keys = torch.randint(-500, 70_000, (n,), generator=g, device="cuda", dtype=torch.int64)
    elif shape == "heavy_hitters":
        keys = torch.randint(-2**31, 2**31 - 1, (n,), generator=g, device="cuda", dtype=torch.int64)
        hot = torch.rand(n, generator=g, device="cuda") < 0.6
        keys = torch.where(hot, torch.randint(0, 5, (n,), generator=g, device="cuda", dtype=torch.int64) * 123_456_789, keys)
    else:
        wide = torch.randint(-2**31, 2**31 - 1, (n,), generator=g, device="cuda", dtype=torch.int64)
        dense = 1_000 + torch.randint(0, 100_000, (n,), generator=g, device="cuda", dtype=torch.int64)
        keys = torch.where(torch.rand(n, generator=g, device="cuda") < 0.5, dense, wide)
    keys = keys.to(torch.int32)
    valid = torch.rand(n, generator=g, device="cuda") > 0.02
    u, c = _ref_counts(keys, valid)
    cuts = [0, 64 * 11000, 64 * 30000, n]
    for path in ("", "radix"):
        if path:
            monkeypatch.setenv("NVTB_SORT_PATH", path)
        else:
            monkeypatch.delenv("NVTB_SORT_PATH", raising=False)
        agg = _insert_batches(engine, Column, pack_validity, keys, valid, cuts)
        assert agg.mode == 1
        k, s, _, null_size, _ = agg.export()
        assert torch.equal(k, u) and torch.equal(s, c), (shape, path)
        assert null_size == int((~valid).sum())


def test_small_staging_buffer_merges_flushes(monkeypatch):
    """NVTB_STAGE_ROWS below the fit size: several flushes, each merged into the accumulator"""
    engine, Column, pack_validity = _engine()
    monkeypatch.setenv("NVTB_RUNS_MIN_KEYS", "1")
    monkeypatch.setenv("NVTB_STAGE_ROWS", str(64 * 9000))
    n = 3_000_000
    g = torch.Generator(device="cuda").manual_seed(77)
    keys = (torch.randint(0, 900_000, (n,), generator=g, device="cuda", dtype=torch.int64) * 2654435761 % (2**32) - 2**31).to(torch.int32)
    valid = torch.rand(n, generator=g, device="cuda") > 0.05
    cuts = list(range(0, n, 64 * 5000)) + [n]
    agg = _insert_batches(engine, Column, pack_validity, keys, valid, cuts)
    k, s, _, null_size, _ = agg.export()
    u, c = _ref_counts(keys, valid)
    assert torch.equal(k, u) and torch.equal(s, c) and null_size == int((~valid).sum())


def _unique_packed(g, n, lo, hi):
    """n distinct int32 keys in [lo, hi) with counts in [1, 1000], as key-ordered packed pairs"""
    keys = torch.unique(torch.randint(lo, hi, (n,), generator=g, device="cuda", dtype=torch.int64))
    counts = torch.randint(1, 1001, (keys.numel(),), generator=g, device="cuda", dtype=torch.int64)
    return keys, counts, ((keys + 2**31) << 32) | counts


@pytest.mark.parametrize("case", ["a_empty", "b_empty", "disjoint", "identical", "overlap"])
def test_pairs_merge(case):
    """nvtb_pairs_merge (the cross-GPU shard merge) against a torch reference: the merged pairs stay
    key-ordered and key-unique, and the counts of a key present on both sides are added"""
    engine, _, _ = _engine()
    g = torch.Generator(device="cuda").manual_seed(len(case))
    if case == "disjoint":
        ka, ca, a = _unique_packed(g, 30_000, -2**31, 0)
        kb, cb, b = _unique_packed(g, 20_000, 0, 2**31 - 1)
    elif case == "identical":
        ka, ca, a = _unique_packed(g, 50_000, -2**31, 2**31 - 1)
        kb, cb, b = ka, ca * 3, ((ka + 2**31) << 32) | (ca * 3)
    else:   # overlap: far more than one 4096-element merge tile, keys drawn from a shared range
        ka, ca, a = _unique_packed(g, 700_000, -3_000_000, 3_000_000)
        kb, cb, b = _unique_packed(g, 500_000, -3_000_000, 3_000_000)
    if case == "a_empty":
        ka, ca, a = ka[:0], ca[:0], a[:0]
    elif case == "b_empty":
        kb, cb, b = kb[:0], cb[:0], b[:0]
    got = engine.pairs_merge(a.contiguous(), b.contiguous())
    k = torch.cat([ka, kb])
    u, inv = torch.unique(k, return_inverse=True)
    c = torch.zeros_like(u).index_add_(0, inv, torch.cat([ca, cb]))
    assert torch.equal(got, ((u + 2**31) << 32) | c)
