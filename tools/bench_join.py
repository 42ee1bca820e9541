"""Measure the external-table join (JoinExternal, K9) on one GPU.

    python tools/bench_join.py [--steps 3] [--warmup 1]

Two workloads, device-resident:
  movielens  synth.movielens_frame(2.5e7) left-joined on movieId to synth.movies_frame (the same
             6e4 scattered ids, a genres list of 1-6 of 18 names, an int32 year): unique ext keys,
             so the probe is the whole join (the fast path)
  expand     1e8 left int32 keys inner-joined to a 1e7-row ext table with about two rows per key
             and 10 % of the left keys missing, carrying int64 and float32 ext columns: probe,
             scan, expand and gather; the key table (16 B slots, 2^24 of them) does not fit in L2
Prints ONE JSON line: per workload rows/s, output rows/s, per-family CUDA-event times (join_probe,
join_expand, and gather: nvtb_gather_rows of the left and ext columns and list offsets), achieved
bytes/s of each family against 3.35 TB/s (H100 SXM HBM3) with what bounds it, a parity flag
against oracle/join_external.py on a seeded 1e5-row sample, and the card name and power limit
read in the same run.  Writes nothing to the tree."""
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

HBM_BPS = 3.35e12
BOUNDS = {"join_probe": "one dependent random 16 B table slot per row (latency of L2 / HBM sectors)",
          "join_expand": "two binary searches over the output offsets per 8 output rows",
          "gather": "random ext-row reads at the gathered rows (32 B sectors for 4-8 B values)"}


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        name, power = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return name, power
    except Exception:
        return None, None


def _expand_tables(n_left, n_ext, seed):
    from nvtabular_b200.column import Column, DeviceFrame
    from nvtabular_b200.synth import scatter_ids
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    n_keys = n_ext // 2
    k = torch.arange(n_keys, device="cuda", dtype=torch.int64).repeat(2)
    k = k[torch.randperm(n_ext, generator=g, device="cuda")]
    ext = DeviceFrame({"key": Column(scatter_ids(k)),
                       "amount": Column(torch.randint(-2**40, 2**40, (n_ext,), generator=g, device="cuda")),
                       "score": Column(torch.rand(n_ext, generator=g, device="cuda"))})
    lk = torch.randint(0, int(n_keys / 0.9), (n_left,), generator=g, device="cuda")
    left = DeviceFrame({"key": Column(scatter_ids(lk))})
    return left, ext


def _to_pandas(frame):
    import pandas as pd
    return pd.DataFrame({k: frame[k].to_pandas(k) for k in frame.columns})


def _parity(op_args, ext_pd, left_frame, select, seed):
    """the same join on a seeded 1e5-row sample of the left table against the pandas oracle"""
    import nvtabular_b200 as nvt
    from nvtabular_b200.column import DeviceFrame
    from oracle.join_external import join_external
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    n = len(left_frame)
    idx = torch.randint(0, n, (100_000,), generator=g, device="cuda")
    sample = DeviceFrame({k: type(left_frame[k])(left_frame[k].data[idx], None, None, left_frame[k].dictionary,
                                                  None, left_frame[k].is_bool) for k in select})
    out = nvt.Workflow(select >> nvt.ops.JoinExternal(ext_pd, **op_args)).transform(sample).to_pandas()
    exp = join_external(_to_pandas(sample), ext_pd, op_args["on"], how=op_args.get("how", "left"))
    if list(out.columns) != list(exp.columns) or len(out) != len(exp):
        return False
    for c in exp.columns:
        a, b = out[c].tolist(), exp[c].tolist()
        if a and isinstance(b[0], (list, np.ndarray)):
            if [list(x) for x in a] != [list(x) for x in b]:
                return False
        elif not np.array_equal(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64), equal_nan=True):
            return False
    return True


def _measure(wf, frame, steps, warmup):
    from nvtabular_b200 import engine
    for _ in range(warmup):
        wf.transform(frame)
    torch.cuda.synchronize()
    times = []
    for _ in range(steps):
        t0 = time.perf_counter()
        out = wf.transform(frame)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    n_out = len(out)
    del out
    engine.profile = []
    wf.transform(frame)
    torch.cuda.synchronize()
    fam = {}
    for f, s, e, nbytes in engine.profile:
        if f in BOUNDS:
            ms, b = fam.get(f, (0.0, 0.0))
            fam[f] = (ms + s.elapsed_time(e), b + nbytes)
    engine.profile = None
    t = float(np.median(times))
    n = len(frame)
    return {"rows": n, "output_rows": n_out, "rows_per_s": n / t, "output_rows_per_s": n_out / t,
            "transform_s_median": t, "transform_s_all": times,
            "families": {f: {"ms": round(ms, 3), "bytes": b, "bytes_per_s": b / (ms * 1e-3),
                             "of_hbm_peak": round(b / (ms * 1e-3) / HBM_BPS, 4), "bound": BOUNDS.get(f)}
                         for f, (ms, b) in sorted(fam.items())}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ratings", type=int, default=25_000_000)
    ap.add_argument("--left", type=int, default=100_000_000)
    ap.add_argument("--ext", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=1234)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_join.py needs a CUDA device")
    import nvtabular_b200 as nvt
    from nvtabular_b200.synth import movielens_frame, movies_frame

    name, power = _card()
    res = {"gpu": name, "power_limit": power}

    ratings = movielens_frame(args.ratings, seed=args.seed)
    movies = _to_pandas(movies_frame(seed=args.seed + 1))
    sel = ["movieId", "userId", "rating"]
    ml = {"on": "movieId", "how": "left"}
    wf = nvt.Workflow(sel >> nvt.ops.JoinExternal(movies, **ml))
    res["movielens"] = _measure(wf, ratings, args.steps, args.warmup)
    res["movielens"]["parity"] = _parity(ml, movies, ratings, sel, args.seed + 2)
    del wf, ratings

    left, ext = _expand_tables(args.left, args.ext, args.seed + 3)
    ext_pd = _to_pandas(ext)
    ex = {"on": "key", "how": "inner"}
    wf = nvt.Workflow(["key"] >> nvt.ops.JoinExternal(ext_pd, **ex))
    res["expand"] = _measure(wf, left, args.steps, args.warmup)
    res["expand"]["parity"] = _parity(ex, ext_pd, left, ["key"], args.seed + 4)
    res["parity"] = bool(res["movielens"]["parity"] and res["expand"]["parity"])
    print(json.dumps({"workload": "join_external", **res}))


if __name__ == "__main__":
    main()
