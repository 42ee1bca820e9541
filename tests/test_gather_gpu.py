"""The row gather (csrc/gather.cu: engine.gather and engine.take_rows) against torch indexing:
every column kind with and without validity, row -1 with and without `masked`, the group-by row
selections (order & row_mask at which 0, 1 and 2; offsets without an order), an unaligned
selection, sizes around the 8-row groups, more than one launch of columns, an empty source, -0.0
canonicalisation and list columns."""
import numpy as np
import pytest
import torch

from nvtabular_b200 import engine
from nvtabular_b200.column import Column, pack_validity, unpack_validity

pytestmark = pytest.mark.gpu

KINDS = ["bool", "uint8", "int32", "int64", "float32", "float64", "string"]
WORDS = np.array(["ant", "bee", "cat", "dog", "eel", "fox", "gnu"], dtype=object)


def _column(kind, n, g, with_validity):
    if kind == "bool":
        data = torch.randint(0, 2, (n,), generator=g, device="cuda").to(torch.uint8)
    elif kind == "uint8":
        data = torch.randint(0, 256, (n,), generator=g, device="cuda").to(torch.uint8)
    elif kind == "int32":
        data = torch.randint(-2**31, 2**31, (n,), generator=g, device="cuda", dtype=torch.int64).to(torch.int32)
    elif kind == "int64":
        data = torch.randint(-2**62, 2**62, (n,), generator=g, device="cuda", dtype=torch.int64)
    elif kind == "float32":
        data = torch.randn(n, generator=g, device="cuda")
    elif kind == "float64":
        data = torch.randn(n, generator=g, device="cuda", dtype=torch.float64)
    else:
        data = torch.randint(0, len(WORDS), (n,), generator=g, device="cuda").to(torch.int32)
    valid = pack_validity(torch.rand(n, generator=g, device="cuda") > 0.3) if with_validity else None
    return Column(data, valid, None, WORDS if kind == "string" else None, None, kind == "bool")


def _rows(sel, m):
    """the row every output reads, from the rule of nvtb_row_sel_t"""
    p = torch.arange(m, device="cuda")
    if sel.which == 1:
        p = sel.off[:m]
    elif sel.which == 2:
        p = sel.off[1:m + 1] - 1
    if sel.pos is None:
        return p
    r = sel.pos[p]
    return r if sel.row_mask == engine.ALL_ROWS else r & sel.row_mask


def _check(out, src, rows, masked):
    """out == src at rows, row -1 null with data 0; a bitmask exactly when src has one or masked"""
    m = rows.numel()
    hit = rows >= 0
    at = rows.clamp(min=0)
    want = torch.where(hit, src.data[at] if src.data.numel() else torch.zeros_like(at, dtype=src.data.dtype),
                       torch.zeros((), dtype=src.data.dtype, device="cuda"))
    assert out.data.dtype == src.data.dtype and out.data.numel() == m
    assert torch.equal(out.data.view(torch.uint8), want.contiguous().view(torch.uint8))
    assert out.dictionary is src.dictionary and out.is_bool == src.is_bool and out.offsets is None
    if src.validity is None and not masked:
        assert out.validity is None
        return
    src_valid = unpack_validity(src.validity, src.data.numel(), "cuda") if src.validity is not None else None
    want_valid = hit & (src_valid[at] if src_valid is not None else True)
    assert out.validity is not None and out.validity.numel() == engine.mask_nbytes(m)
    assert torch.equal(unpack_validity(out.validity, m, "cuda"), want_valid)


def _ids(n, m, g, nulls=True):
    rows = torch.randint(0, n, (m,), generator=g, device="cuda")
    if nulls:
        rows[torch.rand(m, generator=g, device="cuda") < 0.2] = -1
    return rows


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("with_validity", [False, True])
@pytest.mark.parametrize("masked", [False, True])
def test_gather_at_rows(kind, with_validity, masked):
    g = torch.Generator(device="cuda")
    g.manual_seed(11)
    src = _column(kind, 50_000, g, with_validity)
    rows = _ids(50_000, 100_003, g)
    (out,) = engine.gather([src], rows, rows.numel(), masked=masked)
    _check(out, src, rows, masked)


@pytest.mark.parametrize("m", [0, 1, 7, 8, 9, 1_000_003])
def test_gather_sizes(m):
    g = torch.Generator(device="cuda")
    g.manual_seed(m)
    cols = [_column(k, 4096, g, True) for k in KINDS]
    rows = _ids(4096, m, g)
    for masked in (False, True):
        for out, src in zip(engine.gather(cols, rows, m, masked=masked), cols):
            _check(out, src, rows, masked)


@pytest.mark.parametrize("which", [0, 1, 2])
def test_gather_group_selections(which):
    """ordered elements (fields << r) | row read at i, at segment starts and at segment ends"""
    g = torch.Generator(device="cuda")
    g.manual_seed(5 + which)
    n = 200_001
    r = int(n - 1).bit_length()
    row = torch.randperm(n, generator=g, device="cuda")
    order = (torch.randint(0, 2**20, (n,), generator=g, device="cuda") << r) | row
    cut = torch.unique(torch.randint(1, n, (20_000,), generator=g, device="cuda"))
    off = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), cut,
                     torch.full((1,), n, dtype=torch.int64, device="cuda")])
    m = n if which == 0 else off.numel() - 1
    cols = [_column(k, n, g, v) for k in KINDS for v in (False, True)]
    for sel in (engine.order_sel(order, r, which, off), engine.RowSel(off=off, which=which)):
        rows = _rows(sel, m)
        assert bool((rows >= 0).all())
        for out, src in zip(engine.gather(cols, sel, m), cols):
            _check(out, src, rows, False)


def test_gather_unaligned_selection():
    """a slice of the row ids that starts off a 32-byte boundary, as shuffle_by_keys passes"""
    g = torch.Generator(device="cuda")
    g.manual_seed(3)
    n = 70_000
    r = int(n - 1).bit_length()
    order = (torch.randint(0, 2**16, (n,), generator=g, device="cuda") << r) | torch.randperm(n, generator=g,
                                                                                             device="cuda")
    cols = [_column(k, n, g, True) for k in KINDS]
    for start in (1, 3, 5, 13):
        piece = order[start: start + 40_009]
        assert piece.data_ptr() % 32
        sel = engine.order_sel(piece, r)
        rows = _rows(sel, piece.numel())
        for out, src in zip(engine.gather(cols, sel, piece.numel()), cols):
            _check(out, src, rows, False)
        ids = _ids(n, n, g)[start: start + 40_009]
        for out, src in zip(engine.gather(cols, ids, ids.numel(), masked=True), cols):
            _check(out, src, ids, True)


@pytest.mark.parametrize("ncols", [17, 33])
def test_gather_many_columns(ncols):
    g = torch.Generator(device="cuda")
    g.manual_seed(ncols)
    cols = [_column(KINDS[k % len(KINDS)], 30_000, g, k % 3 == 0) for k in range(ncols)]
    rows = _ids(30_000, 50_001, g)
    outs = engine.gather(cols, rows, rows.numel(), masked=False)
    assert len(outs) == ncols
    for out, src in zip(outs, cols):
        _check(out, src, rows, False)


def test_gather_empty_source_at_null_rows():
    """an empty external table: every row reads -1"""
    cols = [Column(torch.empty(0, dtype=dt, device="cuda")) for dt in (torch.uint8, torch.int32, torch.float64)]
    rows = torch.full((1001,), -1, dtype=torch.int64, device="cuda")
    for masked in (False, True):
        for out, src in zip(engine.gather(cols, rows, rows.numel(), masked=masked), cols):
            _check(out, src, rows, masked)


def test_gather_canonicalises_negative_zero_only_where_asked():
    vals = [0.0, -0.0, 1.5, -2.0]
    n = 1000
    f32 = torch.tensor(vals * (n // 4), dtype=torch.float32, device="cuda")
    f64 = torch.tensor(vals * (n // 4), dtype=torch.float64, device="cuda")
    i32 = torch.full((n,), -2**31, dtype=torch.int32, device="cuda")
    i64 = torch.full((n,), -2**63, dtype=torch.int64, device="cuda")
    cols = [Column(t) for t in (f32, f64, f32, f64, i32, i64)]
    rows = torch.arange(n, device="cuda").flip(0)
    outs = engine.gather(cols, rows, n, canon_zero=[True, True, False, False])
    neg = torch.tensor([v == 0 and np.signbit(v) for v in vals] * (n // 4), device="cuda").flip(0)
    for k, (out, src) in enumerate(zip(outs, cols)):
        want = src.data.flip(0)
        if k < 2:
            assert not bool(torch.signbit(out.data[neg]).any())
            want = torch.where(neg, torch.zeros_like(want), want)
        assert torch.equal(out.data.view(torch.uint8), want.contiguous().view(torch.uint8))


def _list_column(n, g, kind, with_validity):
    lens = torch.randint(0, 6, (n,), generator=g, device="cuda")
    off = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    off[1:] = torch.cumsum(lens, 0)
    leaves = _column(kind, int(off[-1]), g, with_validity)
    return Column(leaves.data, leaves.validity, off, leaves.dictionary, None, leaves.is_bool)


def _lists(c):
    off = c.offsets.cpu().tolist()
    data = c.data.cpu().tolist()
    valid = unpack_validity(c.validity, c.data.numel(), "cuda").cpu().tolist() if c.validity is not None else None
    return [[(data[k], valid[k] if valid else True) for k in range(off[i], off[i + 1])] for i in range(len(off) - 1)]


def test_take_rows_lists_at_rows_first_and_last():
    g = torch.Generator(device="cuda")
    g.manual_seed(17)
    n = 20_000
    cols = {"a": _list_column(n, g, "int64", True), "b": _list_column(n, g, "float32", False),
            "c": _column("int32", n, g, True), "d": _list_column(n, g, "string", False)}
    want = {k: _lists(c) for k, c in cols.items() if c.is_list}
    rows = _ids(n, 30_001, g)
    r = int(n - 1).bit_length()
    order = (torch.randint(0, 2**10, (n,), generator=g, device="cuda") << r) | torch.randperm(n, generator=g,
                                                                                            device="cuda")
    cut = torch.unique(torch.randint(1, n, (3000,), generator=g, device="cuda"))
    off = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), cut,
                     torch.full((1,), n, dtype=torch.int64, device="cuda")])
    cases = [(rows, None, False), (rows, None, True)]
    cases += [(engine.order_sel(order, r, w, off), off.numel() - 1, False) for w in (1, 2)]
    for sel, m, masked in cases:
        got = engine.take_rows(cols, sel, m, masked=masked)
        assert list(got) == list(cols)
        at = (sel if m is None else _rows(sel, m)).cpu().tolist()
        for k, c in cols.items():
            if not c.is_list:
                _check(got[k], c, sel if m is None else _rows(sel, m), masked)
                continue
            assert got[k].dictionary is c.dictionary and got[k].is_bool == c.is_bool
            assert (got[k].validity is None) == (c.validity is None)
            assert _lists(got[k]) == [want[k][i] if i >= 0 else [] for i in at]
