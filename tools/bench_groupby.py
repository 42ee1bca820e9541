"""Measure the session group-by (Groupby, K8) and Dataset.shuffle_by_keys on one GPU.

    python tools/bench_groupby.py [--rows 100000000] [--steps 3] [--warmup 1]

Workload: a device-resident synthetic session table (nvtabular_b200.synth.session_frame:
power-law session lengths, about rows / 10 sessions, rows shuffled) grouped by session_id,
sorted by ts, with item_id list + count + first / last and price mean -- the input stage of a
sequential recommender.  Prints ONE JSON line: Groupby rows/s, shuffle_by_keys rows/s (3 input
partitions -> 3 output partitions), per-stage device times from CUDA events, a parity flag
against oracle/session_groupby.py on a seeded sample, and the card name and power limit read in
the same run.  Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        name, power = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return name, power
    except Exception:
        return None, None


def _op():
    import nvtabular_b200 as nvt
    return nvt.ops.Groupby(groupby_cols=["session_id"], sort_cols=["ts"],
                           aggs={"item_id": ["list", "count", "first", "last"], "price": "mean"})


def _parity(seed):
    """the same transform on a 100k-row sample against the pandas oracle"""
    import pandas as pd
    import nvtabular_b200 as nvt
    from nvtabular_b200.synth import session_frame
    from oracle.session_groupby import session_groupby
    frame, _ = session_frame(100_000, seed=seed, device="cuda")
    out = nvt.Workflow(["session_id", "item_id", "ts", "price"] >> _op()).transform(frame)
    df = pd.DataFrame({k: frame[k].data.cpu().numpy() for k in frame.columns})
    exp = session_groupby(df, "session_id", "ts", {"item_id": ["list", "count", "first", "last"], "price": "mean"})
    ok = out["session_id"].data.cpu().tolist() == exp["session_id"]
    off = out["item_id_list"].offsets.cpu().numpy()
    leaves = out["item_id_list"].data.cpu().numpy()
    ok &= [leaves[off[i]:off[i + 1]].tolist() for i in range(len(off) - 1)] == exp["item_id_list"]
    for a in ("count", "first", "last"):
        ok &= out[f"item_id_{a}"].data.cpu().tolist() == exp[f"item_id_{a}"]
    ok &= np.array_equal(out["price_mean"].data.cpu().numpy(), np.asarray(exp["price_mean"], dtype=np.float32))
    return bool(ok)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=1234)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_groupby.py needs a CUDA device")
    import nvtabular_b200 as nvt
    from nvtabular_b200 import engine
    from nvtabular_b200.column import DeviceFrame
    from nvtabular_b200.synth import session_frame

    name, power = _card()
    frame, n_sess = session_frame(args.rows, seed=args.seed, device="cuda")
    wf = nvt.Workflow(["session_id", "item_id", "ts", "price"] >> _op())
    for _ in range(args.warmup):
        wf.transform(frame)
    torch.cuda.synchronize()
    times = []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        out = wf.transform(frame)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    groups = len(out["session_id"])
    del out

    # per-stage device times: one more transform with CUDA events around every launch family
    engine.profile = []
    wf.transform(frame)
    torch.cuda.synchronize()
    stages = {}
    for fam, s, e, _ in engine.profile:
        stages[fam] = stages.get(fam, 0.0) + s.elapsed_time(e)
    engine.profile = None

    # shuffle_by_keys: 3 input partitions -> 3 output partitions, all in HBM
    n = args.rows
    cut = [0, n // 3 // 64 * 64, 2 * n // 3 // 64 * 64, n]
    parts = [frame.slice_rows(cut[i], cut[i + 1]) for i in range(3)]
    ds = nvt.Dataset(parts)
    ds.shuffle_by_keys(["session_id"], npartitions=3)      # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    shuffled = ds.shuffle_by_keys(["session_id"], npartitions=3)
    list(shuffled.partitions())
    torch.cuda.synchronize()
    t_shuffle = time.perf_counter() - t0
    del shuffled, ds, parts

    t = float(np.median(times))
    print(json.dumps({
        "workload": "session_groupby",
        "rows": n, "sessions_generated": n_sess, "groups": groups,
        "aggs": "item_id list+count+first+last, price mean; sort by ts",
        "groupby_rows_per_s": n / t, "groupby_s_median": t, "groupby_s_all": times,
        "shuffle_by_keys_rows_per_s": n / t_shuffle, "shuffle_by_keys_s": t_shuffle,
        "stage_ms": {k: round(v, 3) for k, v in sorted(stages.items())},
        "parity_vs_oracle": _parity(args.seed + 1),
        "gpu": name, "power_limit": power,
    }))


if __name__ == "__main__":
    main()
