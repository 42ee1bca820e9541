"""GPU tests of the flush of a sorted accumulator (csrc/sortacc.cu, csrc/bucketagg.cuh): the staging
copies fold the min / max of the keys, the bucket route sizes its emit for the batch's real window,
and the result must still be exactly torch.unique's counts and the radix route's
(NVTB_SORT_PATH=radix) packed pairs, null count and largest count, at the shapes that stress each of
those choices."""
import pytest
import torch

pytestmark = pytest.mark.gpu

I32_MIN, I32_MAX = -2**31, 2**31 - 1


def _fit(monkeypatch, keys, valid, cuts, path):
    from nvtabular_b200 import engine
    from nvtabular_b200.column import Column, pack_validity
    if path:
        monkeypatch.setenv("NVTB_SORT_PATH", path)
    else:
        monkeypatch.delenv("NVTB_SORT_PATH", raising=False)
    agg = engine.HashAgg(0)
    for a, b in zip(cuts[:-1], cuts[1:]):
        v = pack_validity(valid[a:b]) if valid is not None else None
        agg.insert(Column(keys[a:b].contiguous(), v))
    assert agg.mode == 1
    packed = agg.export_packed()
    k, s, _, null_size, _ = agg.export()
    vocab = engine.Vocab.build_from_agg(agg, 0, 0, 0, 32, keys.numel()) if k.numel() else None
    return packed, k, s, null_size, vocab


def _check(monkeypatch, keys, valid, cuts, stage_rows=None):
    monkeypatch.setenv("NVTB_RUNS_MIN_KEYS", "1")
    if stage_rows is not None:
        monkeypatch.setenv("NVTB_STAGE_ROWS", str(stage_rows))
    kv = keys[valid] if valid is not None else keys
    u, c = torch.unique(kv.to(torch.int64), return_counts=True)
    nulls = 0 if valid is None else int((~valid).sum())
    bucket = _fit(monkeypatch, keys, valid, cuts, "")
    radix = _fit(monkeypatch, keys, valid, cuts, "radix")
    for packed, k, s, null_size, vocab in (bucket, radix):
        assert torch.equal(k, u) and torch.equal(s, c)
        assert null_size == nulls
        if u.numel():
            order = torch.sort(c, stable=True, descending=True).indices     # u is key-ascending
            vk, vs = vocab.export()
            assert torch.equal(vk, u[order]) and torch.equal(vs, c[order])
            assert vocab.null_size == nulls and vocab.n_total == u.numel()
    assert torch.equal(bucket[0], radix[0])


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _cuts(n, parts=4):
    step = (n // parts + 63) // 64 * 64
    return list(range(0, n, step)) + [n]


def test_flush_criteo_c20_shape(monkeypatch):
    """2^27 staged rows shaped like Criteo's C20 (power-law ids scattered over the int32 range,
    7.6 % nulls) in 4 batches: one flush into an empty accumulator"""
    from nvtabular_b200.synth import power_law_ids, scatter_ids
    n = 1 << 27
    g = _gen(19)
    keys = scatter_ids(power_law_ids(n, 290_000_000, g, "cuda"))
    valid = torch.rand(n, generator=g, device="cuda") >= 0.076
    _check(monkeypatch, keys, valid, _cuts(n))


def test_flush_full_int32_range(monkeypatch):
    """INT32_MIN and INT32_MAX both present: the range is 2^32 - 1, shift 19, the widest window"""
    n = 4_000_000
    g = _gen(3)
    keys = torch.randint(I32_MIN, I32_MAX, (n,), generator=g, device="cuda", dtype=torch.int64)
    keys[::1000] = I32_MIN
    keys[7::1000] = I32_MAX
    valid = torch.rand(n, generator=g, device="cuda") > 0.05
    valid[:16] = True
    _check(monkeypatch, keys.to(torch.int32), valid, _cuts(n))


def test_flush_single_value(monkeypatch):
    n = 1_000_000
    keys = torch.full((n,), -123_457, dtype=torch.int32, device="cuda")
    valid = torch.rand(n, generator=_gen(5), device="cuda") > 0.3
    _check(monkeypatch, keys, valid, _cuts(n))


def test_flush_all_null_batch(monkeypatch):
    """one batch of nothing but nulls among valid ones, then a fit of nothing but nulls"""
    n = 1_000_000
    g = _gen(6)
    keys = torch.randint(I32_MIN, I32_MAX, (n,), generator=g, device="cuda", dtype=torch.int64).to(torch.int32)
    valid = torch.ones(n, dtype=torch.bool, device="cuda")
    cuts = _cuts(n)
    valid[cuts[1]:cuts[2]] = False
    _check(monkeypatch, keys, valid, cuts)
    _check(monkeypatch, keys, torch.zeros(n, dtype=torch.bool, device="cuda"), cuts)


def test_flush_narrow_range_few_buckets(monkeypatch):
    """four clusters of 50 values, 2^20 apart: every row lands in one of four buckets"""
    n = 4_000_000
    g = _gen(7)
    keys = (5_000_000 + torch.randint(0, 4, (n,), generator=g, device="cuda", dtype=torch.int64) * (1 << 20)
            + torch.randint(0, 50, (n,), generator=g, device="cuda", dtype=torch.int64))
    valid = torch.rand(n, generator=g, device="cuda") > 0.02
    _check(monkeypatch, keys.to(torch.int32), valid, _cuts(n))


def test_flush_one_heavy_bucket(monkeypatch):
    """keys over the whole range, plus 30 % of the rows on 10 000 values inside one window: that
    bucket holds ~100 times the rows of the others, and its duplicated values still fit"""
    n = 4_000_000
    g = _gen(8)
    wide = torch.randint(I32_MIN, I32_MAX, (n,), generator=g, device="cuda", dtype=torch.int64)
    dense = 77_000_000 + torch.randint(0, 10_000, (n,), generator=g, device="cuda", dtype=torch.int64)
    keys = torch.where(torch.rand(n, generator=g, device="cuda") < 0.3, dense, wide)
    valid = torch.rand(n, generator=g, device="cuda") > 0.02
    _check(monkeypatch, keys.to(torch.int32), valid, _cuts(n))


@pytest.mark.parametrize("stage_rows", [None, 64 * 9000])
def test_flush_ragged_and_small_stage(monkeypatch, stage_rows):
    """a first batch that is not a multiple of 8 rows (the next batch bypasses the staging copies and
    finds its own min / max), with the default stage or one that several flushes go through"""
    n = 3_000_000
    g = _gen(9)
    keys = (torch.randint(0, 900_000, (n,), generator=g, device="cuda", dtype=torch.int64) * 2654435761 % (2**32)
            - 2**31).to(torch.int32)
    valid = torch.rand(n, generator=g, device="cuda") > 0.05
    cuts = [0, 64 * 3000 + 5] + list(range(64 * 8000, n, 64 * 5000)) + [n]
    _check(monkeypatch, keys, valid, cuts, stage_rows)
