"""Measure the flush of the high-cardinality sorted accumulators (K3b) on one GPU.

    python tools/bench_flush.py [--rows 100000000] [--steps 7] [--warmup 2] [--profile DIR]

Input: the five columns that the Criteo step groups with a sorted accumulator (C20, C1, C22, C10,
C21), generated exactly as synth.criteo_frame(rows, total_rows=4.37e9) generates them (same seeds,
same nulls), device-resident.  Each column has its own HashAgg; one fit (4 batches through
HashAgg.insert, then HashAgg.flush) warms it up, then per step: reset(), the 4 inserts (they only
stage), the flush.  Staging and flush are timed apart with CUDA events; medians of `steps`.

--profile DIR: instead of timing, one step of every column under torch.profiler (CUDA activities),
the kernel times summed by name, and the trace written to DIR.

Bytes come from the shapes (n staged rows, v valid rows, d distinct keys per column):
  staging          keys and validity bytes read and written: 8.25 n (+ the min/max fold)
  bk_minmax        4.125 n read (a build whose staging copies do not fold the min / max)
  part_hist        4.125 n read
  part_scatter     4.125 n read + 4 v written (into 512 coarse ranges)
  bk_refine        4 v read + 4 v written (each range into its 16 buckets)
  bk_count         4 v read
  bk_emit          4 v read (the second stream of a bucket hits L2) + 8 d written
Achieved GB/s = bytes / time, against 3.35 TB/s (H100 SXM HBM3).  Prints ONE JSON line with the
card's name and power limit, read in the same run.  Writes nothing to the tree."""
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
COLUMNS = ["C20", "C1", "C22", "C10", "C21"]
BATCHES = 4


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        name, power, sm, sm_max = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception:
        return {"gpu": None, "power_limit": None}


def criteo_column(name, rows, total_rows, seed=1234):
    """column `name` of synth.criteo_frame(rows, total_rows, seed) without the other 39"""
    from nvtabular_b200 import synth
    from nvtabular_b200.column import Column
    j = synth.CAT_NAMES.index(name)
    g = synth._gen(seed + 100 + j, "cuda")
    k = synth.scaled_cardinality(name, total_rows)
    keys = synth.scatter_ids(synth.power_law_ids(rows, k, g, "cuda"))
    return Column(keys, synth._null_mask(rows, 0.10 * j / 25.0, g, "cuda"))


def _batches(col, n):
    from nvtabular_b200.column import Column
    step = (n // BATCHES + 63) // 64 * 64
    out = []
    for a in range(0, n, step):
        b = min(a + step, n)
        v = col.validity[a // 8:(b + 7) // 8] if col.validity is not None else None
        out.append(Column(col.data[a:b], v))
    return out


def _model(n, v, d, parent_minmax):
    """bytes each step of a flush moves, from the shapes"""
    kb = 4.125 * n
    m = {"staging": 8.25 * n, "part_hist": kb, "part_scatter": kb + 4.0 * v, "bk_refine": 8.0 * v,
         "bk_count": 4.0 * v, "bk_emit": 4.0 * v + 8.0 * d}
    if parent_minmax:
        m["bk_minmax"] = kb
    return m


def _rate(ms, nbytes):
    bps = nbytes / (ms * 1e-3) if ms > 0 else 0.0
    return {"ms": round(ms, 3), "bytes": int(nbytes), "GB_per_s": round(bps / 1e9, 1),
            "of_hbm_peak": round(bps / HBM_BPS, 3)}


def _step(agg, batches):
    agg.reset()
    s0, s1, s2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
    s0.record()
    for b in batches:
        agg.insert(b)
    s1.record()
    agg.flush()
    s2.record()
    return s0, s1, s2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--total-rows", type=int, default=4_370_000_000)
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile", default="", metavar="DIR", help="per-kernel times from torch.profiler instead")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_flush.py needs a CUDA device")
    from nvtabular_b200 import engine

    res = {"workload": "k3b_flush", **_card(), "rows": args.rows, "batches": BATCHES,
           "stage_rows_env": os.environ.get("NVTB_STAGE_ROWS")}
    cols, aggs, shapes = {}, {}, {}
    for name in COLUMNS:
        col = criteo_column(name, args.rows, args.total_rows)
        cols[name] = _batches(col, args.rows)
        agg = engine.HashAgg(0)
        for b in cols[name]:
            agg.insert(b)
        agg.flush()
        assert agg.mode == 1, f"{name} did not become a sorted accumulator"
        k, s, _, nulls, _ = agg.export()
        shapes[name] = {"n": args.rows, "valid": args.rows - int(nulls), "distinct": int(k.numel()),
                        "max_count": int(s.max().item()) if s.numel() else 0}
        aggs[name] = agg
        del col, k, s
    torch.cuda.synchronize()
    res["shapes"] = shapes

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(args.profile, exist_ok=True)
        for name in COLUMNS:
            _step(aggs[name], cols[name])
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for name in COLUMNS:
                _step(aggs[name], cols[name])
            torch.cuda.synchronize()
        prof.export_chrome_trace(os.path.join(args.profile, "bench_flush.pt.trace.json"))
        kern = {}
        for ev in prof.events():
            if ev.device_type.name != "CUDA":
                continue
            key = ev.name.split("(")[0].split("<")[0].replace("void ", "").replace("nvtb::", "").strip()
            t = kern.setdefault(key, [0.0, 0])
            t[0] += ev.device_time / 1e3
            t[1] += 1
        n = sum(s["n"] for s in shapes.values())
        v = sum(s["valid"] for s in shapes.values())
        d = sum(s["distinct"] for s in shapes.values())
        model = _model(n, v, d, parent_minmax=any(k.startswith("bk_minmax") for k in kern))
        out = {}
        for key, (ms, calls) in sorted(kern.items(), key=lambda kv: -kv[1][0]):
            e = {"ms": round(ms, 3), "calls": calls}
            for mk, mb in model.items():
                if key.startswith(mk):
                    e.update(_rate(ms, mb))
            out[key] = e
        res["kernels_all_five"] = out
        print(json.dumps(res))
        return

    for _ in range(args.warmup):
        for name in COLUMNS:
            _step(aggs[name], cols[name])
    torch.cuda.synchronize()
    stage_ms = {c: [] for c in COLUMNS}
    flush_ms = {c: [] for c in COLUMNS}
    for _ in range(args.steps):
        for name in COLUMNS:
            s0, s1, s2 = _step(aggs[name], cols[name])
            torch.cuda.synchronize()
            stage_ms[name].append(s0.elapsed_time(s1))
            flush_ms[name].append(s1.elapsed_time(s2))
    # every step's result must still be the warm-up fit's
    for name in COLUMNS:
        k, s, _, nulls, _ = aggs[name].export()
        assert int(k.numel()) == shapes[name]["distinct"] and args.rows - int(nulls) == shapes[name]["valid"]
    per_col = {}
    tot_ms, tot_bytes, flush_tot, flush_bytes = 0.0, 0.0, 0.0, 0.0
    for name in COLUMNS:
        sh = shapes[name]
        m = _model(sh["n"], sh["valid"], sh["distinct"], parent_minmax=False)
        st, fl = float(np.median(stage_ms[name])), float(np.median(flush_ms[name]))
        fb = sum(b for k, b in m.items() if k != "staging")
        per_col[name] = {"stage": _rate(st, m["staging"]), "flush": _rate(fl, fb),
                         "flush_ms_all": [round(x, 3) for x in flush_ms[name]]}
        tot_ms += st + fl
        tot_bytes += m["staging"] + fb
        flush_tot += fl
        flush_bytes += fb
    res["columns"] = per_col
    res["flush_five"] = _rate(flush_tot, flush_bytes)
    res["stage_and_flush_five"] = _rate(tot_ms, tot_bytes)
    res["bytes_note"] = "bytes of the byte model of this build's passes (docstring)"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
