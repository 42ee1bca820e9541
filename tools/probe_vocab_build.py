"""Where the time of the high-cardinality vocabulary builds (K4) goes, at the bench's sizes.

    python tools/probe_vocab_build.py [--rows 100000000] [--reps 3] [--out DIR]

Builds the columns C20, C1, C22, C10 and C21 of `synth.criteo_frame` (1e8 rows, full-profile
cardinalities, the bench's 4 partitions) into sorted accumulators, then times
  - Vocab.build_from_agg  (the single-GPU fit: count ordering + cut + lookup), and
  - Vocab.build_from_pairs (the multi-GPU tail: pairs already in label order)
with CUDA events, and in a separate run lists the device time of every kernel name with
torch.profiler (CUDA activities).  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nvtabular_b200 import engine  # noqa: E402
from nvtabular_b200.column import Column  # noqa: E402
from nvtabular_b200.synth import (CAT_NAMES, CRITEO_ROWS, _gen, _null_mask, power_law_ids,  # noqa: E402
                                  scaled_cardinality, scatter_ids)

COLUMNS = ["C20", "C1", "C22", "C10", "C21"]


def card():
    try:
        q = "name,power.limit,clocks.max.sm"
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:          # noqa: BLE001
        return f"unknown ({exc!r})"


def column(name, rows, parts):
    """the same keys and nulls as synth.criteo_frame(rows, total_rows=CRITEO_ROWS), cut like bench.py"""
    j = CAT_NAMES.index(name)
    g = _gen(1234 + 100 + j, "cuda")
    keys = scatter_ids(power_law_ids(rows, scaled_cardinality(name, CRITEO_ROWS), g, "cuda"))
    mask = _null_mask(rows, 0.10 * j / 25.0, g, "cuda")
    step = (rows // parts) // 64 * 64
    out = []
    for p in range(parts):
        lo, hi = p * step, (rows if p == parts - 1 else (p + 1) * step)
        out.append(Column(keys[lo:hi], None if mask is None else mask[lo // 8:(hi + 7) // 8]))
    return out


def timed(fn, reps):
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        v = fn()
        e1.record()
        v.n_kept                      # the build's scalars: waits for it
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
        del v
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--parts", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = {"card": card(), "rows": a.rows, "columns": {}}
    aggs, pairs = {}, {}
    for name in COLUMNS:
        agg = engine.HashAgg(0)
        for c in column(name, a.rows, a.parts):
            agg.insert(c)
        agg.flush()
        v = engine.Vocab.build_from_agg(agg, key_bits=32, size_bound=a.rows)
        k, s = v.export()
        pairs[name] = (((k & 0xFFFFFFFF) ^ 0x80000000) << 32) | s
        aggs[name] = agg
        res["columns"][name] = {"distinct": int(v.n_kept)}
        del v, k, s
    torch.cuda.synchronize()

    # end to end per build (CUDA events), after one warm-up build of each
    for name in COLUMNS:
        agg, p = aggs[name], pairs[name]
        r = res["columns"][name]
        timed(lambda: engine.Vocab.build_from_agg(agg, key_bits=32, size_bound=a.rows), 1)
        r["from_agg_ms"] = timed(lambda: engine.Vocab.build_from_agg(agg, key_bits=32, size_bound=a.rows), a.reps)
        timed(lambda: engine.Vocab.build_from_pairs(p, 0), 1)
        r["from_pairs_ms"] = timed(lambda: engine.Vocab.build_from_pairs(p, 0), a.reps)
        print(name, json.dumps(r), flush=True)
    res["from_agg_total_ms"] = sum(min(r["from_agg_ms"]) for r in res["columns"].values())
    res["from_pairs_total_ms"] = sum(min(r["from_pairs_ms"]) for r in res["columns"].values())

    # per kernel name, one build of each column and kind, in a run of its own
    from torch.profiler import ProfilerActivity, profile
    per = {}
    for kind in ("from_agg", "from_pairs"):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for name in COLUMNS:
                if kind == "from_agg":
                    v = engine.Vocab.build_from_agg(aggs[name], key_bits=32, size_bound=a.rows)
                else:
                    v = engine.Vocab.build_from_pairs(pairs[name], 0)
                v.n_kept
                del v
            torch.cuda.synchronize()
        tot = defaultdict(lambda: [0.0, 0])
        for ev in prof.events():
            if ev.device_type == torch.autograd.DeviceType.CUDA:
                key = ev.name.split("(")[0].split("<")[0].replace("void ", "").replace("nvtb::", "")
                tot[key][0] += ev.device_time_total / 1e3
                tot[key][1] += 1
        per[kind] = {k: {"ms": round(v[0], 3), "calls": v[1]} for k, v in sorted(tot.items(), key=lambda kv: -kv[1][0])}
        print(f"{kind}: kernels over the five builds (ms, calls)", flush=True)
        for k, v in per[kind].items():
            print(f"  {v['ms']:9.3f}  {v['calls']:4d}  {k}", flush=True)
    res["kernels"] = per
    res["card_after"] = card()
    print(json.dumps({k: res[k] for k in ("card", "from_agg_total_ms", "from_pairs_total_ms")}), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "probe_vocab_build.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
