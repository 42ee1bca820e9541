"""The Categorify encode (K5, `Vocab.encode` -> nvtb_encode_apply), the group-statistics gather
(K7, `GroupStats.gather_columns`) and the host serving encode (csrc/infer.cu) against the exact
reference of tests/_encode_ref.py, with keys built from the table-hash replicas so that every
probe branch is reached on purpose (tests/test_encode_replicas.py checks the replicas against the
headers).

Every encode case records its kernels with torch.profiler and asserts the ROUTE it targets, and
checks int32 and int64 labels, with num_buckets 0 and NB = 7 (hashed OOV), label for label.

  case                          route                     branch reached, and why
  test_encode_smem              encode_smem_kernel        1 <= n_kept <= 14 336, int32 keys, n >= 2^18,
    [n_kept 1 / 700 / 14 336,                             aligned buffers (vocab.cu nvtb_encode_apply);
     n 2^18, 2^18+5, 2^20+3]                              n = 2^18 + 5: the scalar tail of the last thread
                                encode_kernel<.., true>   n_kept = 14 337, n = 2^18 - 1 or a key view one
    [n_kept 14 337, n 2^18-1,                             element off 32-byte alignment: the global route
     unaligned view]
      fold_unhash(0xFFFFFFFF)   h == kFoldEmpty: never stored in shared memory; its bucket (7167)
                                has free slots, whose word IS kFoldEmpty, so only the h test stops a
                                false match.  Present (served by the global lookup) and absent.
      7 keys of bucket 1234     4 slots per shared bucket: 3 spill at build time and must be
                                found through the global lookup; 3 more keys of that bucket are
                                absent queries that meet the full bucket
      nulls none / some / all, and two hash columns (int32, float64 with nulls) under nb = 7
  test_encode_narrow            encode_kernel<.., true>   40 000 int32 keys: a 16 384-bucket table of two
                                                          8 192-bucket slices
      chains of 12 / 9 / 6 / 5 keys on one home bucket (table_mix32 low bits fixed): at the end of
      slice 0 (bucket 8191, wraps to 0), at the end of the table (wraps to 8192), in the middle,
      and one at 8190 that spills into 8191; 4 absent keys per chain walk it to a free slot
      keys 0, -1, INT32_MIN, INT32_MAX present or absent (0 against free slots, whose word is 0)
      int64 queries k +- 2^32 of present keys: OOV through the range guard (nb = 0: decided in
      the fast path; nb = 7: encode_slow), INT64_MIN / INT64_MAX
      n = 200 003 (not a multiple of the 4096-row tile), and an unaligned view (per-row path)
  test_encode_wide              encode_kernel<.., false>  Vocab.from_arrays (int64 keys beyond int32)
      chains from the table_mix64 inverse: 12 keys on the last slot (linear probing wraps to 0),
      8 in the middle; INT64_MIN (the empty-slot sentinel, kept in min_key_pos) present three
      times or absent; 100 repeated keys (the smallest position wins); int32 and int64 queries
  test_encode_hash_cols         encode_kernel, both       1 .. 8 hash columns cycling int32, int64,
                                                          float32 (-0.0), float64, uint8, bool, H64,
                                                          float32, with nulls; odd counts on a narrow
                                                          table, even counts on a wide one.  A float
                                                          NaN is a null, as Column.from_pandas makes
                                                          it.  Up to 6 columns the OOV buckets also
                                                          equal oracle.categorify.hash_bucket_oov on
                                                          the pandas frame.
  test_encode_labels            encode_kernel<.., true>   Categorify (1, 2, 3 + nb), single table
                                                          (null = first = 5), TargetEncoding (n_groups,
                                                          -2, 0), the key-space codes (0, INT32_MIN + 1, 1)
  test_gather                   gather_stats_kernel       n in {1, 31, 32, 33, 257, 2^21 + 17} (a partial
                                                          last bitmask word; more rows than one grid
                                                          stride), int32 / int64 query keys, null_row
                                                          -1 or the extra row, 20 outputs (two launches
                                                          of 16 + 4) of all four dtypes, masked or not
  test_host_*                   csrc/infer.cu             the host table against the device encode and
                                                          the reference; 1, 3 and all threads

Gather statistics hold NaN, +-inf, -0.0, values that need int64 and fractions (integer outputs
truncate toward zero).  Integer outputs only read columns whose values fit their type: a double
out of the integer range has no defined conversion."""
import types

import numpy as np
import pandas as pd
import pytest
import torch

import _encode_ref as R
from oracle.categorify import hash_bucket_oov

pytestmark = pytest.mark.gpu

I32_MIN, I32_MAX = np.iinfo(np.int32).min, np.iinfo(np.int32).max
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
NB = 7
OUT = (np.int32, np.int64)
SPECIAL32 = np.array([0, -1, I32_MIN, I32_MAX], dtype=np.int32)
K_EMPTY = R.fold_unhash(np.uint32(R.FOLD_EMPTY)).astype(np.uint32).view(np.int32).reshape(1)   # h == kFoldEmpty
FULL = R.smem_bucket_keys(1234, 10)           # one shared bucket: 7 in the vocabulary, 3 absent


@pytest.fixture(scope="module")
def eng():
    from nvtabular_b200 import engine
    return engine


def _col(arr, null=None, offset=0, prehashed=False):
    """device column of `arr` (True in `null` = null row); `offset` > 0: a view that starts that many
    elements into its allocation, with the validity packed for the view"""
    from nvtabular_b200.column import Column, pack_validity
    arr = np.ascontiguousarray(arr)
    if arr.dtype == bool:
        arr = arr.astype(np.uint8)
    full = np.concatenate([np.zeros(offset, arr.dtype), arr])
    data = torch.from_numpy(full).cuda()[offset:]
    valid = pack_validity(torch.from_numpy(~np.asarray(null, bool)).cuda()) if null is not None else None
    c = Column(data, valid)
    c.prehashed = prehashed
    return c


def _nulls(rng, n, kind):
    return {"none": None, "some": rng.random(n) < 0.1, "all": np.ones(n, bool)}[kind]


def _draw(rng, n, pools, weights):
    """n keys drawn from the pools with the given weights"""
    which = rng.choice(len(pools), n, p=np.asarray(weights) / np.sum(weights))
    out = np.empty(n, dtype=np.result_type(*pools))
    for j, p in enumerate(pools):
        sel = which == j
        out[sel] = p[rng.integers(0, len(p), sel.sum())]
    return out


def _random_i32(rng, n, exclude):
    k = np.unique(rng.integers(I32_MIN, I32_MAX, 2 * n + 16, endpoint=True).astype(np.int32))
    k = np.setdiff1d(k, np.asarray(exclude, np.int32))
    return rng.permutation(k)[:n]


def _build(eng, keys, rng):
    """Vocab.build of distinct int32-valued keys with random counts; the exported keys must be in
    (count desc, key asc) order"""
    keys = np.asarray(keys, np.int64)
    sizes = rng.integers(1, 1000, len(keys))
    v = eng.Vocab.build(torch.from_numpy(keys).cuda(), torch.from_numpy(sizes).cuda(), key_bits=32,
                        size_bound=int(sizes.sum()))
    vk = v.export(with_sizes=False)[0].cpu().numpy()
    order = np.lexsort((keys, -sizes))
    np.testing.assert_array_equal(vk, keys[order])
    assert v.n_kept == len(keys)
    return v, vk


def _route(name):
    base = name.split("(")[0].rstrip()
    if "encode_smem_kernel" in base:
        return "smem"
    if "encode_kernel" in base:
        if base.endswith("true>") or "Lb1E" in base:
            return "narrow"
        if base.endswith("false>") or "Lb0E" in base:
            return "wide"
    return None


def _eq(got, exp, keys, what):
    bad = np.flatnonzero(got != exp)
    assert bad.size == 0, (f"{what}: {bad.size} of {len(exp)} labels differ; first rows "
                           f"{bad[:5].tolist()}, keys {np.asarray(keys)[bad[:5]].tolist()}, "
                           f"got {got[bad[:5]].tolist()}, expected {exp[bad[:5]].tolist()}")


def _check_encode(vocab, vk, keys, null, route, labels=(1, 2, 3 + NB), hash_cols=None, offset=0, host=True):
    """device labels of every (num_buckets, out dtype) against the reference, and the route that
    ran; `hash_cols`: [(values, null, prehashed)] for nb = NB; `host`: the serving encode too"""
    from torch.profiler import ProfilerActivity, profile
    nl, ol, fl = labels
    key = _col(keys, null, offset)
    hcols = [_col(v, m, prehashed=p) for v, m, p in hash_cols] if hash_cols else []
    hashes = None
    if hash_cols:
        hashes = np.zeros(len(keys), np.uint64)
        for v, m, p in hash_cols:
            hashes ^= R.col_hash(v, m, p)
    # Now and then a profiling session records no device activity at all (2 sessions of about 200
    # in one run on an H100 with torch 2.11), so a session without a single kernel is repeated, at
    # most twice.  A session that recorded kernels is always judged.
    for _ in range(3):
        got = {}
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for nb in (0, NB):
                for od in OUT:
                    got[nb, od] = vocab.encode(key, nl, ol, fl, nb, hcols if nb else (), od)
            torch.cuda.synchronize()
        names = [ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA]
        if names:
            break
    routes = {_route(name) for name in names}
    routes.discard(None)
    assert routes == {route}, routes
    for (nb, od), t in got.items():
        exp = R.ref_labels(keys, null, vk, nl, ol, fl, nb, hashes if nb else None)
        lab = t.cpu().numpy()
        assert lab.dtype == od
        _eq(lab, exp.astype(od), keys, f"device nb={nb} out={np.dtype(od)}")
    if host and not hash_cols:
        hv = _host(vocab)
        valid = None if null is None else ~null
        for nb in (0, NB):
            for od in OUT:
                exp = R.ref_labels(keys, null, vk, nl, ol, fl, nb)
                _eq(hv.encode(keys, valid, nl, ol, fl, nb, od), exp.astype(od), keys, f"host nb={nb} out={np.dtype(od)}")
    return got


def _host(vocab):
    from nvtabular_b200.inference import _HostVocab
    return _HostVocab(types.SimpleNamespace(vocab=vocab))


# --------------------------------------------------------------------------------- shared memory
def _smem_vocab_keys(rng, n_kept, empty_in):
    if n_kept == 1:
        return K_EMPTY if empty_in else FULL[:1]
    adv = [FULL[:7], SPECIAL32, R.narrow_chain(rng, 14, 8191, 12), R.narrow_chain(rng, 20, (1 << 20) - 1, 9)]
    if empty_in:
        adv.append(K_EMPTY)
    adv = np.concatenate(adv)
    rest = _random_i32(rng, n_kept - len(adv), np.concatenate([adv, FULL, K_EMPTY]))
    return rng.permutation(np.concatenate([adv, rest]))


SMEM_CASES = [   # n_kept, n, nulls, fold-empty key in the vocabulary, hash columns, view offset
    (1, 1 << 18, "none", True, False, 0),
    (1, (1 << 18) + 5, "some", False, False, 0),
    (700, (1 << 18) + 5, "all", True, False, 0),
    (700, (1 << 20) + 3, "some", True, True, 0),
    (14336, 1 << 18, "none", True, False, 0),
    (14336, (1 << 18) + 5, "some", False, True, 0),
    (14336, (1 << 20) + 3, "some", True, False, 0),
    (14336, (1 << 18) - 1, "some", True, False, 0),
    (14336, (1 << 18) + 5, "some", True, False, 1),
    (14337, 1 << 18, "some", False, False, 0),
]


@pytest.mark.parametrize("n_kept,n,nulls,empty_in,with_hash,offset", SMEM_CASES)
def test_encode_smem(eng, n_kept, n, nulls, empty_in, with_hash, offset):
    rng = np.random.default_rng(n_kept * 31 + n + offset)
    vocab, vk = _build(eng, _smem_vocab_keys(rng, n_kept, empty_in), rng)
    vk32 = vk.astype(np.int32)
    absent = _random_i32(rng, 1000, vk32)
    adv = np.concatenate([FULL, K_EMPTY, SPECIAL32])
    keys = _draw(rng, n, [vk32, absent, adv], [0.6, 0.3, 0.1])
    null = _nulls(rng, n, nulls)
    hash_cols = None
    if with_hash:
        f = rng.normal(0, 1e3, n)
        hash_cols = [(rng.integers(-50, 50, n).astype(np.int32), rng.random(n) < 0.2, False),
                     (f, rng.random(n) < 0.2, False)]
    smem = 1 <= n_kept <= R.SMEM_MAX_KEYS and n >= (1 << 18) and offset == 0
    _check_encode(vocab, vk, keys, null, "smem" if smem else "narrow", hash_cols=hash_cols, offset=offset)


# --------------------------------------------------------------------------------- narrow, global
NARROW_CASES = [   # specials in the vocabulary, query dtype, n, view offset
    (True, np.int32, 200_003, 0),
    (False, np.int32, 200_003, 1),
    (True, np.int64, 200_003, 0),
    (False, np.int64, 65_536 + 77, 1),
]


@pytest.mark.parametrize("specials_in,qdt,n,offset", NARROW_CASES)
def test_encode_narrow(eng, specials_in, qdt, n, offset):
    rng = np.random.default_rng(7 + n + offset + int(specials_in))
    chains = [(R.narrow_chain(rng, 14, 8191, 16), 12),              # end of slice 0 of 16 384 buckets
              (R.narrow_chain(rng, 20, (1 << 20) - 1, 13), 9),      # end of the table
              (R.narrow_chain(rng, 20, 12345, 10), 6),
              (R.narrow_chain(rng, 20, 8190, 9), 5)]
    present = np.concatenate([c[:k] for c, k in chains] + ([SPECIAL32] if specials_in else []))
    chain_absent = np.concatenate([c[k:] for c, k in chains])
    reserved = np.concatenate([present, chain_absent, SPECIAL32])
    keys_v = rng.permutation(np.concatenate([present, _random_i32(rng, 40_000 - len(present), reserved)]))
    vocab, vk = _build(eng, keys_v, rng)
    vk32 = vk.astype(np.int32)
    pools = [vk32, np.concatenate([c for c, _ in chains]), SPECIAL32, _random_i32(rng, 2000, reserved)]
    weights = [0.5, 0.2, 0.05, 0.15]
    if qdt == np.int64:
        s = vk[rng.integers(0, len(vk), 1000)]
        shifted = np.concatenate([s + (1 << 32), s - (1 << 32), SPECIAL32.astype(np.int64) + (1 << 32),
                                  SPECIAL32.astype(np.int64) - (1 << 32), [I64_MIN, I64_MAX]])
        pools = [p.astype(np.int64) for p in pools] + [shifted]
        weights.append(0.1)
    keys = _draw(rng, n, pools, weights).astype(qdt)
    _check_encode(vocab, vk, keys, rng.random(n) < 0.05, "narrow", offset=offset)


# --------------------------------------------------------------------------------- wide
@pytest.mark.parametrize("min_in", [True, False])
@pytest.mark.parametrize("qdt", [np.int64, np.int32])
def test_encode_wide(eng, min_in, qdt):
    rng = np.random.default_rng(11 + int(min_in) + 2 * (qdt == np.int32))
    chains = [(R.wide_chain(rng, 24, (1 << 24) - 1, 16), 12), (R.wide_chain(rng, 24, 777, 12), 8)]
    big = rng.integers(1 << 33, 1 << 62, 30_000) * rng.choice([-1, 1], 30_000)
    small = _random_i32(rng, 2000, SPECIAL32).astype(np.int64)
    base = np.concatenate([c[:k] for c, k in chains] + [big, small, SPECIAL32.astype(np.int64)[:2]])
    base = np.setdiff1d(base, np.concatenate([c[k:] for c, k in chains] + [[I64_MIN]]))   # distinct
    keys_v = np.concatenate([base, base[rng.integers(0, len(base), 100)]] + ([np.full(3, I64_MIN)] if min_in else []))
    keys_v = rng.permutation(keys_v)
    vocab = eng.Vocab.from_arrays(torch.from_numpy(keys_v).cuda())
    vk = vocab.export(with_sizes=False)[0].cpu().numpy()
    np.testing.assert_array_equal(vk, keys_v)
    n = 300_001
    if qdt == np.int64:
        pools = [keys_v, np.concatenate([c for c, _ in chains]), rng.integers(I64_MIN, I64_MAX, 3000),
                 np.array([I64_MIN, I64_MAX, 0, -1, I32_MIN, I32_MAX], np.int64)]
        keys = _draw(rng, n, pools, [0.5, 0.15, 0.25, 0.1])
    else:
        pools = [small.astype(np.int32), _random_i32(rng, 3000, small), SPECIAL32]
        keys = _draw(rng, n, pools, [0.5, 0.4, 0.1]).astype(np.int32)
    _check_encode(vocab, vk, keys, rng.random(n) < 0.05, "wide")


# --------------------------------------------------------------------------------- hash columns
HASH_DTYPES = ["int32", "int64", "float32", "float64", "uint8", "bool", "h64", "float32"]


def _hash_column(rng, dt, n):
    """(values, null, prehashed, pandas Series or None) of one hash column"""
    null = rng.random(n) < 0.15
    if dt == "bool":
        v = rng.random(n) < 0.5
        return v, None, False, pd.Series(v)                       # a null bool has no pandas twin here
    if dt == "h64":
        return rng.integers(I64_MIN, I64_MAX, n), null, True, None
    if dt.startswith("float"):
        v = (rng.normal(0, 10, n) * 4).round().astype(dt) / 4     # repeats, -0.0 among them
        v[rng.random(n) < 0.05] = -0.0
        v[rng.random(n) < 0.05] = np.nan
        null = null | np.isnan(v)                                 # a NaN is a null (Column.from_pandas)
        return v, null, False, pd.Series(np.where(null, np.nan, v).astype(dt))
    if dt == "uint8":
        v = rng.integers(0, 256, n).astype(np.uint8)
        return v, null, False, pd.Series(pd.array(v, dtype="UInt8")).mask(null)
    info = np.iinfo(dt)
    v = rng.integers(info.min, info.max, n, endpoint=True).astype(dt)
    return v, null, False, pd.Series(pd.array(v, dtype=dt.capitalize())).mask(null)


@pytest.mark.parametrize("ncols", range(1, 9))
def test_encode_hash_cols(eng, ncols):
    rng = np.random.default_rng(100 + ncols)
    n = 50_003
    cols = [_hash_column(rng, dt, n) for dt in HASH_DTYPES[:ncols]]
    if ncols % 2:
        vocab, vk = _build(eng, _random_i32(rng, 500, []), rng)
        keys = _draw(rng, n, [vk.astype(np.int32), _random_i32(rng, 2000, vk)], [0.5, 0.5])
        route = "narrow"
    else:
        vk = rng.integers(I64_MIN, I64_MAX, 500)
        vocab = eng.Vocab.from_arrays(torch.from_numpy(vk).cuda())
        keys = _draw(rng, n, [vk, rng.integers(I64_MIN, I64_MAX, 2000)], [0.5, 0.5])
        route = "wide"
    null = rng.random(n) < 0.05
    got = _check_encode(vocab, vk, keys, null, route, hash_cols=[c[:3] for c in cols])
    if all(c[3] is not None for c in cols):
        df = pd.DataFrame({f"c{j}": c[3] for j, c in enumerate(cols)})
        exp = hash_bucket_oov(df, NB, list(df.columns), encode_type="combo").astype(np.int64)
        miss = ~null & ~np.isin(keys, vk)
        for od in OUT:
            lab = got[NB, od].cpu().numpy().astype(np.int64)
            _eq(lab[miss] - 2, exp[miss], keys[miss], f"pandas frame out={np.dtype(od)}")


# --------------------------------------------------------------------------------- label layouts
@pytest.mark.parametrize("labels", [(1, 2, 3 + NB), (5, 6, 5), (1000, -2, 0), (0, I32_MIN + 1, 1)],
                         ids=["categorify", "single_table", "target_encoding", "keyspace"])
def test_encode_labels(eng, labels):
    rng = np.random.default_rng(200 + labels[0])
    vocab, vk = _build(eng, _random_i32(rng, 30_000, []), rng)
    n = 100_003
    keys = _draw(rng, n, [vk.astype(np.int32), _random_i32(rng, 2000, vk), SPECIAL32], [0.6, 0.35, 0.05])
    _check_encode(vocab, vk, keys, rng.random(n) < 0.1, "narrow", labels=labels)


# --------------------------------------------------------------------------------- serving encode
@pytest.mark.parametrize("threads", [1, 3, 0])
def test_host_threads(eng, threads):
    """n > 3 * 2^14 rows: run_threads splits the request; every split gives the reference"""
    rng = np.random.default_rng(300 + threads)
    vocab, vk = _build(eng, np.concatenate([SPECIAL32, _random_i32(rng, 20_000, SPECIAL32)]), rng)
    hv = _host(vocab)
    n = 200_001
    keys = _draw(rng, n, [vk.astype(np.int32), _random_i32(rng, 3000, vk)], [0.5, 0.5])
    null = rng.random(n) < 0.1
    for kd in (np.int32, np.int64):
        k = keys.astype(kd)
        for od in OUT:
            exp = R.ref_labels(k, null, vk, 1, 2, 3 + NB, NB).astype(od)
            _eq(hv.encode(k, ~null, 1, 2, 3 + NB, NB, od, threads=threads), exp, k, f"host {np.dtype(kd)}")
            dev = vocab.encode(_col(k, null), 1, 2, 3 + NB, NB, (), od).cpu().numpy()
            _eq(dev, exp, k, f"device {np.dtype(kd)}")


def test_host_workflow_end_to_end(tmp_path):
    """a fitted Categorify with OOV buckets: a numpy request, a CUDA tensor request and
    Workflow.transform give the same labels, and those of the reference"""
    import nvtabular_b200 as nvt
    rng = np.random.default_rng(400)
    pool = np.concatenate([rng.integers(-(1 << 40), 1 << 40, 3000), [I64_MIN, -1, 0, I32_MIN]])
    fit = pd.DataFrame({"a": pool[rng.integers(0, len(pool), 40_000)]})
    unseen = rng.integers(I64_MIN, I64_MAX, 500)
    req = pd.DataFrame({"a": np.concatenate([pool, unseen])[rng.permutation(len(pool) + 500)]})
    op = nvt.ops.Categorify(out_path=str(tmp_path), num_buckets=NB)
    wf = nvt.Workflow(["a"] >> op)
    wf.fit(nvt.Dataset(fit))
    exp = wf.transform(nvt.Dataset(req)).to_ddf().compute()["a"].to_numpy()
    sel = nvt.ColumnSelector(["a"])
    inf = op.inference_initialize(sel, {})
    a = req["a"].to_numpy()
    got_np = np.asarray(inf.transform(sel, {"a": a})["a"])
    got_dev = inf.transform(sel, {"a": torch.from_numpy(a).cuda()})["a"].cpu().numpy()
    np.testing.assert_array_equal(got_np, exp)
    np.testing.assert_array_equal(got_dev, exp)
    vk = op._fitted("a").vocab.export(with_sizes=False)[0].cpu().numpy()
    np.testing.assert_array_equal(exp, R.ref_labels(a, None, vk, 1, 2, 2 + NB, NB).astype(exp.dtype))


# --------------------------------------------------------------------------------- gather
N_GROUPS = 3000
GATHER_OUT = [np.int32, np.int64, np.float32, np.float64]


def _group_table(rng):
    """distinct int64 group keys and a stats matrix of N_GROUPS + 1 rows (the last: the null group)
    with columns 0: fits int32 (fractions, NaN, -0.0); 1: fits int64 (up to 2^62, fractions, NaN);
    2, 3: any double (NaN, +-inf, -0.0, beyond float32)"""
    keys = np.setdiff1d(np.concatenate([
        [I64_MAX, -1, 0, I32_MIN, I32_MAX, 1 << 32, -(1 << 32)],
        rng.integers(I32_MIN, I32_MAX, 1000),
        rng.integers(1 << 33, 1 << 62, 1000) * rng.choice([-1, 1], 1000),
        rng.integers(-5000, 5000, 2000)]), [I64_MIN, -7])
    keys = rng.permutation(np.concatenate([[I64_MIN, -7], rng.permutation(keys)[:N_GROUPS - 2]]))
    m = N_GROUPS + 1
    s = np.zeros((m, 4))
    s[:, 0] = rng.integers(-(1 << 31) + 1, 1 << 31, m) + rng.choice([0, 0.25, 0.5, 0.75, -0.75], m)
    s[:, 0] = np.clip(s[:, 0], -(2.0 ** 31) + 1, 2.0 ** 31 - 1)
    s[:, 1] = rng.integers(-(1 << 52), 1 << 52, m) * rng.choice([1, 1024], m) + rng.choice([0, 0.5, -0.25], m) * \
        (rng.random(m) < 0.3)
    s[:, 2] = rng.normal(0, 1e6, m)
    s[:, 3] = rng.normal(0, 1, m) * 10.0 ** rng.integers(-320, 300, m)
    for j in range(4):
        s[rng.random(m) < 0.1, j] = np.nan
        s[rng.random(m) < 0.05, j] = -0.0
    s[rng.random(m) < 0.05, 2] = np.inf
    s[rng.random(m) < 0.05, 3] = -np.inf
    s[-1] = [-2.5, -(2.0 ** 62), np.nan, -0.0]
    return keys, s


def _gather_outputs():
    """20 outputs (cols, miss, dtypes, masked): every dtype, NaN and finite misses, masks mixed in
    both launches"""
    cols, miss, dts, masked = [], [], [], []
    for j in range(20):
        dt = GATHER_OUT[j % 4]
        dts.append(dt)
        cols.append({np.int32: 0, np.int64: (1, 0)[j // 4 % 2], np.float32: 2 + j // 4 % 2, np.float64: (3, 2, 1, 0)[j // 4 % 4]}[dt])
        miss.append(np.nan if j % 3 == 0 else {np.int32: -3.75, np.int64: 2.0 ** 40 + 0.25}.get(dt, 1e300))
        masked.append(j % 5 != 1)
    return cols, miss, dts, masked


@pytest.fixture(scope="module")
def group_table():
    return _group_table(np.random.default_rng(500))


@pytest.mark.parametrize("n", [1, 31, 32, 33, 257, (1 << 21) + 17])
@pytest.mark.parametrize("qdt", [np.int64, np.int32])
@pytest.mark.parametrize("null_row", [-1, N_GROUPS])
def test_gather(eng, group_table, n, qdt, null_row):
    gk, stats = group_table
    rng = np.random.default_rng(n + 2 * (qdt == np.int32) + null_row)
    gs = eng.GroupStats(torch.from_numpy(gk).cuda(), torch.from_numpy(stats if null_row >= 0 else stats[:-1]).cuda(),
                        null_row=null_row)
    if qdt == np.int64:
        pools = [gk, rng.integers(I64_MIN, I64_MAX, 1000), np.array([I64_MIN, I64_MAX, 0, -1, -7], np.int64)]
    else:
        fit = gk[(gk >= I32_MIN) & (gk <= I32_MAX)]
        pools = [fit, rng.integers(I32_MIN, I32_MAX, 1000), np.array([I32_MIN, I32_MAX, 0, -1, -7], np.int64)]
    keys = _draw(rng, n, pools, [0.6, 0.3, 0.1]).astype(qdt)
    null = rng.random(n) < 0.1
    cols, miss, dts, masked = _gather_outputs()
    got = gs.gather_columns(_col(keys, null), cols, miss, dts, masked)
    row = R.ref_rows(keys, null, gk, null_row)
    for j, c in enumerate(got):
        what = f"output {j} ({np.dtype(dts[j])}, col {cols[j]}, miss {miss[j]})"
        exp, valid = R.ref_gather(row, stats, cols[j], miss[j], dts[j])
        v = c.data.cpu().numpy()
        assert v.dtype == dts[j], what
        if np.dtype(dts[j]).kind == "f":
            nan = np.isnan(v)
            np.testing.assert_array_equal(nan, np.isnan(exp), err_msg=what)
            ui = "u4" if dts[j] == np.float32 else "u8"
            np.testing.assert_array_equal(v[~nan].view(ui), exp[~nan].view(ui), err_msg=what)   # -0.0 too
        else:
            _eq(v, exp, keys, what)
        if not masked[j]:
            assert c.validity is None, what
            continue
        bits = c.validity.cpu().numpy()
        ref = np.zeros(len(bits), np.uint8)
        packed = np.packbits(valid, bitorder="little")
        ref[:len(packed)] = packed
        np.testing.assert_array_equal(bits, ref, err_msg=what + ": validity bitmask (bits >= n must be 0)")
