"""Measure the row-selection operators (Filter and Dropna, K11) on one GPU.

    python tools/bench_filter.py [--rows 100000000] [--steps 5] [--warmup 2]

Three workloads, all device-resident, built from synth.session_frame(rows) (session_id int64,
item_id int32, ts int64, price float32 uniform in [0, 100)):
  filter_price   Filter(lambda df: df["price"] > 50) over the four fixed-width columns: keeps about
                 half the rows
  dropna         Dropna() of the same four columns with about 5 % nulls injected into price
  t4rec          the Transformers4Rec step: the Groupby("session_id") output (item_id list + count,
                 about rows / 10 sessions) -> Filter(item_id_count >= 2), list column included.
                 Every session of session_frame has at least 2 rows, so this step keeps every row
                 and passes the frame through; t4rec_ge5 (item_id_count >= 5) keeps about 45 % and
                 measures the compaction of the list column
Every workload reports the whole operator call and its families, each timed alone with CUDA events
(median of `steps` after `warmup`): mask (nvtb_mask_compare / nvtb_mask_notnull), count
(nvtb_mask_count, with its host read), select (nvtb_mask_select), gather (nvtb_gather_rows of the
fixed-width columns) and list_copy (the list column's offsets gather and nvtb_gb_list_rows).
Bytes are the algorithmic minimum computed here (every input read once, every output written once,
row ids read once per gather launch) over the measured time, against 3.35 TB/s (H100 SXM HBM3).
Parity: both operators against oracle/filter.py on a seeded 1e5-row sample.  Prints ONE JSON line
with the card's name and power limit, read in the same run.  Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM_BPS = 3.35e12


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        name, power = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return name, power
    except Exception:
        return None, None


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ms.append(s.elapsed_time(e))
    return float(np.median(ms))


def _family(ms, nbytes):
    bps = nbytes / (ms * 1e-3)
    return {"ms": round(ms, 3), "bytes": int(nbytes), "bytes_per_s": bps, "of_hbm_peak": round(bps / HBM_BPS, 4)}


def _measure(name, frame, make_mask, run_op, steps, warmup, in_bytes):
    """families of one workload: make_mask() -> mask; run_op() is the whole operator"""
    from nvtabular_b200 import engine
    n = len(frame)
    mask = make_mask()
    kept, tile_off = engine.mask_count(mask, n)
    rows = engine.mask_select(mask, n, tile_off, kept)
    flat = {k: c for k, c in frame.items() if not c.is_list}
    lists = {k: c for k, c in frame.items() if c.is_list}
    ntiles = tile_off.numel() - 1
    out = {"rows": n, "kept": kept}
    out["mask"] = _family(_time(make_mask, steps, warmup), in_bytes + n / 8)
    out["count"] = _family(_time(lambda: engine.mask_count(mask, n), steps, warmup), n / 8 + ntiles * 16)
    out["select"] = _family(_time(lambda: engine.mask_select(mask, n, tile_off, kept), steps, warmup),
                            n / 8 + ntiles * 8 + kept * 8)
    fb = sum(kept * (c.data.element_size() * 2 + (0.25 if c.validity is not None else 0)) for c in flat.values())
    launches = -(-len(flat) // engine.GATHER_MAX_COLS)
    out["gather"] = _family(_time(lambda: engine.take_rows(flat, rows), steps, warmup), kept * 8 * launches + fb)
    if lists:
        res = engine.take_rows(lists, rows)
        lb = 0
        for k, c in lists.items():
            leaves = res[k].data.numel()
            lb += kept * 8 * 2 + kept * 8 * 2 + (kept + 1) * 8 + leaves * c.data.element_size() * 2
        out["list_copy"] = _family(_time(lambda: engine.take_rows(lists, rows), steps, warmup), lb)
    total_bytes = in_bytes + n / 8 + fb + sum(v["bytes"] for k, v in out.items() if k == "list_copy")
    out["operator"] = _family(_time(run_op, steps, warmup), total_bytes)
    return name, out


def _parity(seed=7):
    """exact parity of Filter and Dropna with oracle/filter.py on a 1e5-row sample"""
    import pandas as pd
    from nvtabular import ColumnSelector, ops
    from nvtabular_b200.column import Column, pack_validity
    from nvtabular_b200.synth import session_frame
    from oracle.filter import dropna_frame, filter_frame
    frame, _ = session_frame(100_000, seed=seed)
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    price = frame["price"]
    frame["price"] = Column(price.data, pack_validity(torch.rand(len(frame), generator=g, device="cuda") > 0.05))
    names = frame.columns
    pdf = frame.to_pandas()
    f = lambda d: d["price"] > 50  # noqa: E731
    got = ops.Filter(f).transform(ColumnSelector(names), frame).to_pandas()
    ok_f = got.equals(filter_frame(pdf, f)) or np.array_equal(got.to_numpy(float), filter_frame(pdf, f).to_numpy(float),
                                                             equal_nan=True)
    got = ops.Dropna().transform(ColumnSelector(names), frame).to_pandas()
    want = dropna_frame(pdf)
    ok_d = len(got) == len(want) and all(np.array_equal(got[c].to_numpy(float), want[c].to_numpy(float))
                                         for c in names)
    return {"rows": len(pdf), "filter_exact": bool(ok_f), "dropna_exact": bool(ok_d), "pandas": pd.__version__}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=float, default=1e8)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_filter.py needs a CUDA device")
    name, power = _card()
    from nvtabular import ColumnSelector, ops
    from nvtabular_b200 import engine
    from nvtabular_b200.column import Column, pack_validity
    from nvtabular_b200.ops.filter import scalar_compare_type
    from nvtabular_b200.synth import session_frame
    rows = int(args.rows)
    frame, _ = session_frame(rows)
    names = frame.columns
    res = {}

    # 1. Filter(price > 50)
    t, bits = scalar_compare_type(np.dtype("float32"), 50)
    price = frame["price"]
    op = ops.Filter(lambda df: df["price"] > 50)
    k, v = _measure("filter_price", frame, lambda: engine.mask_compare(price, None, engine.CMP_GT, t, bits, rows),
                    lambda: op.transform(ColumnSelector(names), frame), args.steps, args.warmup, rows * 4.0)
    res[k] = v

    # 2. Dropna with ~5 % nulls in price
    g = torch.Generator(device="cuda")
    g.manual_seed(5)
    nulled = frame.copy()
    nulled["price"] = Column(price.data, pack_validity(torch.rand(rows, generator=g, device="cuda") > 0.05))
    drop = ops.Dropna()
    k, v = _measure("dropna", nulled, lambda: engine.mask_notnull([nulled["price"]], rows),
                    lambda: drop.transform(ColumnSelector(names), nulled), args.steps, args.warmup, rows * 4.125)
    res[k] = v
    del nulled

    # 3. the Transformers4Rec step: Groupby output (item_id list + count) -> Filter(count >= 2)
    gb = ops.Groupby("session_id", aggs={"item_id": ["list", "count"]})
    sessions = gb.transform(ColumnSelector(["session_id", "item_id"]), frame)
    del frame
    sessions = sessions[["item_id_list", "item_id_count"]]
    cnt = sessions["item_id_count"]
    ns = len(sessions)
    for key, least in (("t4rec", 2), ("t4rec_ge5", 5)):
        t, bits = scalar_compare_type(cnt.np_dtype, least)
        op = ops.Filter(lambda df, m=least: df["item_id_count"] >= m)
        k, v = _measure(key, sessions, lambda: engine.mask_compare(cnt, None, engine.CMP_GE, t, bits, ns),
                        lambda: op.transform(ColumnSelector(sessions.columns), sessions), args.steps, args.warmup,
                        ns * float(cnt.data.element_size()))
        v["sessions"] = ns
        res[k] = v

    print(json.dumps({"tool": "bench_filter", "gpu": name, "power_limit": power, "rows": rows,
                      "steps": args.steps, "warmup": args.warmup, "hbm_peak_bps": HBM_BPS, "workloads": res,
                      "parity": _parity()}))


if __name__ == "__main__":
    main()
