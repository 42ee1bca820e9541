"""GPU tests of the large-vocabulary build (K4, csrc/vocab.cu): vocabularies of more than 5.2e6
kept keys, whose lookup is built slice by slice, checked against an independent reference of
the value_counts order with the stable tie rule (count desc, key asc; reference
nvtabular/ops/categorify.py:1300,1316): exported keys and sizes, meta sums, and the labels of
present, dropped, absent and null keys through the encode."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

INT32_MIN, INT32_MAX = -2**31, 2**31 - 1
# below this many kept keys the lookup is 2^23 slots or fewer and is built directly; above it the
# table has 512 slices of 8192 buckets or more and is built one slice per CTA
SLICED_FROM = 5_242_881


def _engine():
    from nvtabular_b200 import engine
    from nvtabular_b200.column import Column, pack_validity
    return engine, Column, pack_validity


def _distinct_keys(n, seed, extremes=True):
    """n distinct int32 values (int64 tensor, random order); INT32_MIN and INT32_MAX among them"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    k = torch.unique(torch.randint(INT32_MIN + 1, INT32_MAX, (n + n // 8 + 16,), generator=g, device="cuda",
                                   dtype=torch.int64))
    k = k[torch.randperm(k.numel(), generator=g, device="cuda")[:n]]
    if extremes:
        k[0], k[n // 2] = INT32_MIN, INT32_MAX
    return k


def _reference(keys, counts, freq_threshold=0, max_keep=-1):
    """(count desc, key asc) order and the number of kept rows"""
    o = torch.sort(keys, stable=True).indices
    keys, counts = keys[o], counts[o]
    o = torch.sort(counts, stable=True, descending=True).indices
    keys, counts = keys[o], counts[o]
    if freq_threshold > 0:
        keep = int((counts >= freq_threshold).sum())
    elif max_keep >= 0:
        keep = min(keys.numel(), max_keep)
    else:
        keep = keys.numel()
    return keys, counts, keep


def _check(vocab, keys, counts, keep, seed):
    engine, Column, pack_validity = _engine()
    assert vocab.n_kept == keep
    k, s = vocab.export()
    assert torch.equal(k, keys[:keep]) and torch.equal(s, counts[:keep])
    assert vocab.unique_size == int(counts[:keep].sum())
    assert vocab.oov_size == int(counts[keep:].sum())
    # queries: every key of the accumulator (kept or dropped), keys it never saw, and nulls
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    absent = torch.randint(INT32_MIN, INT32_MAX, (1 << 20,), generator=g, device="cuda", dtype=torch.int64)
    absent = absent[~torch.isin(absent, keys)]
    q = torch.cat([keys, absent])
    q = q[torch.randperm(q.numel(), generator=g, device="cuda")]
    q = q[: q.numel() // 64 * 64]
    valid = torch.rand(q.numel(), generator=g, device="cuda") > 0.05
    labels = vocab.encode(Column(q.to(torch.int32), pack_validity(valid)), 1, 2, 3, 0, (), np.int64)
    kk, perm = torch.sort(keys[:keep])
    idx = torch.searchsorted(kk, q).clamp_(max=max(keep - 1, 0))
    hit = kk[idx] == q
    exp = torch.where(hit, perm[idx] + 3, torch.full_like(idx, 2))
    exp = torch.where(valid, exp, torch.ones_like(exp))
    assert torch.equal(labels, exp)


def _accumulator(monkeypatch, keys, counts):
    """a sorted accumulator holding `counts[i]` rows of `keys[i]`, inserted in two batches"""
    engine, Column, _ = _engine()
    monkeypatch.setenv("NVTB_RUNS_MIN_KEYS", "1")
    rows = torch.repeat_interleave(keys, counts).to(torch.int32)
    g = torch.Generator(device="cuda").manual_seed(int(counts.numel()))
    rows = rows[torch.randperm(rows.numel(), generator=g, device="cuda")]
    cut = rows.numel() // 2 // 64 * 64
    agg = engine.HashAgg(0)
    agg.insert(Column(rows[:cut].contiguous()))
    agg.insert(Column(rows[cut:].contiguous()))
    agg.flush()
    assert agg.mode == 1
    return agg, rows.numel()


@pytest.mark.parametrize("case", ["counts_1", "counts_2_pass", "freq_threshold", "max_size"])
def test_vocab_from_large_accumulator(monkeypatch, case):
    engine, _, _ = _engine()
    n = 6_000_000
    keys = _distinct_keys(n, 31)
    g = torch.Generator(device="cuda").manual_seed(32)
    if case == "counts_1":
        counts = torch.ones(n, dtype=torch.int64, device="cuda")
    else:
        counts = torch.randint(1, 11, (n,), generator=g, device="cuda", dtype=torch.int64)
        if case == "counts_2_pass":       # counts of 11-12 bits: the count ordering takes two passes
            counts[torch.randint(0, n, (300,), generator=g, device="cuda")] = torch.randint(
                1024, 4000, (300,), generator=g, device="cuda", dtype=torch.int64)
    ft, ms = {"freq_threshold": (2, 0), "max_size": (0, 5_500_003)}.get(case, (0, 0))
    agg, rows = _accumulator(monkeypatch, keys, counts)
    vocab = engine.Vocab.build_from_agg(agg, ft, ms, 0, 32, rows)
    ref_k, ref_c, keep = _reference(keys, counts, ft, ms - 3 if ms else -1)
    if case in ("freq_threshold", "max_size"):
        assert SLICED_FROM <= keep < n
    _check(vocab, ref_k, ref_c, keep, 33)


@pytest.mark.parametrize("n", [SLICED_FROM - 1, SLICED_FROM, 6_300_000])
def test_vocab_from_ordered_pairs_around_the_sliced_build(n):
    """build_from_pairs (the multi-GPU tail) on both sides of the first sliced table size"""
    engine, _, _ = _engine()
    keys = _distinct_keys(n, n % 1000)
    g = torch.Generator(device="cuda").manual_seed(n % 977)
    counts = torch.randint(1, 50, (n,), generator=g, device="cuda", dtype=torch.int64)
    ref_k, ref_c, keep = _reference(keys, counts)
    # packed pairs (key ^ 2^31) << 32 | count, as int64 bit patterns (little-endian words)
    hi = ref_k.to(torch.int32) ^ torch.tensor(INT32_MIN, dtype=torch.int32, device="cuda")
    pairs = torch.stack([ref_c.to(torch.int32), hi], dim=1).contiguous().view(torch.int64).reshape(-1)
    vocab = engine.Vocab.build_from_pairs(pairs, 0)
    _check(vocab, ref_k, ref_c, keep, n % 1000)


def test_vocab_from_large_rows():
    """(key, size) rows in any order (nvtb_vocab_build, int32 keys): key passes, then count passes"""
    engine, _, _ = _engine()
    n = 5_600_000
    keys = _distinct_keys(n, 41)
    g = torch.Generator(device="cuda").manual_seed(42)
    counts = torch.randint(1, 3000, (n,), generator=g, device="cuda", dtype=torch.int64)
    vocab = engine.Vocab.build(keys.contiguous(), counts.contiguous(), 0, 0, 0, 0, 32, 3000)
    ref_k, ref_c, keep = _reference(keys, counts)
    _check(vocab, ref_k, ref_c, keep, 43)
