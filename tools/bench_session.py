"""Measure the session operators (ListSlice and DifferenceLag, K10) on one GPU.

    python tools/bench_session.py [--rows 100000000] [--steps 5] [--warmup 2] [--baseline-lib PATH]

Input: synth.session_frame(rows), about rows / 10 power-law sessions, device-resident.  The frame
comes out shuffled, so it is ordered once by (session_id, ts) before anything is timed, as the
operators require.  Timed with CUDA events, median of `steps` after `warmup`:
  difference_lag   DifferenceLag("session_id", shift=[1, -1]) of ts (int64)
  list_slice       ListSlice(-20) of the Groupby item_id list (int32 leaves)
  list_slice_pad   ListSlice(-20, pad=True) of the same list
  list_rows        nvtb_gb_list_rows over every sub-list of that column (the Groupby first /
                   last-of-list path); with --baseline-lib, the same call through another build of
                   libnvtb200.so (for instance the parent commit's), alternating call by call
Bytes are the algorithmic minimum (every input read once, every output written once) over the
measured time, against 3.35 TB/s (H100 SXM HBM3).  Parity: both operators against
oracle/session_ops.py on a seeded 1e5-row sample of the ordered frame.  Prints ONE JSON line with
the card's name and power limit, read in the same run.  Writes nothing to the tree."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
from ctypes import byref, c_int64

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
    return float(np.median(ms)), ms


def _family(ms, nbytes, note=None):
    bps = nbytes / (ms * 1e-3)
    out = {"ms": round(ms, 3), "bytes": nbytes, "bytes_per_s": bps, "of_hbm_peak": round(bps / HBM_BPS, 4)}
    if note:
        out["note"] = note
    return out


def _ordered(frame):
    """the frame ordered by (session_id, ts): one torch sort of a packed key (bench set-up only)"""
    from nvtabular_b200.column import Column, DeviceFrame
    sid, ts = frame["session_id"].data, frame["ts"].data
    key = sid * (1 << 25) + (ts - int(ts.min().item()))
    perm = torch.sort(key, stable=True).indices
    return DeviceFrame({k: Column(c.data[perm].contiguous()) for k, c in frame.items()})


def _list_rows_with(lib, leaves, lo, hi):
    """engine.gb_list_rows through the library handle `lib`"""
    from nvtabular_b200 import _lib
    from nvtabular_b200.engine import _descs, _ptr
    m = lo.numel()
    off = torch.empty(m + 1, dtype=torch.int64, device=lo.device)
    total = c_int64(0)
    _lib.check(lib.nvtb_gb_list_rows(_descs([leaves]), _ptr(lo), _ptr(hi), m, _ptr(off), None, None, byref(total),
                                     _lib.stream_ptr()))
    out = torch.empty(total.value, dtype=leaves.data.dtype, device=lo.device)
    _lib.check(lib.nvtb_gb_list_rows(_descs([leaves]), _ptr(lo), _ptr(hi), m, _ptr(off), _ptr(out), None,
                                     byref(total), _lib.stream_ptr()))
    return out, off


def _parity(frame, seed):
    """both operators on a seeded 1e5-row slice of the ordered frame against the oracle"""
    import nvtabular_b200 as nvt
    from nvtabular_b200.column import DeviceFrame
    from nvtabular_b200.graph import ColumnSelector
    from oracle.session_ops import difference_lag, list_slice
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    n = len(frame)
    s0 = int(torch.randint(0, max(n - 100_000, 1), (1,), generator=g).item())
    sample = DeviceFrame({k: frame[k].__class__(frame[k].data[s0:s0 + 100_000].contiguous())
                          for k in ("session_id", "item_id", "ts")})
    pdf = sample.to_pandas()
    got = nvt.ops.DifferenceLag("session_id", shift=[1, -1]).transform(ColumnSelector(["ts"]), sample).to_pandas()
    want = difference_lag(pdf, ["ts"], "session_id", [1, -1])
    ok = all(np.array_equal(got[c].to_numpy(np.float32), want[c].to_numpy(), equal_nan=True) for c in want.columns)
    gb = nvt.ops.Groupby("session_id", sort_cols="ts", aggs={"item_id": ["list"]})
    lists = gb.transform(ColumnSelector(["session_id", "item_id", "ts"]), sample)
    rows = [[int(v) for v in r] for r in lists["item_id_list"].to_pandas()]
    for pad in (False, True):
        out = nvt.ops.ListSlice(-20, pad=pad).transform(ColumnSelector(["item_id_list"]), lists)["item_id_list"]
        ok = ok and [[int(v) for v in r] for r in out.to_pandas()] == list_slice(rows, -20, pad=pad)
    return bool(ok)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1234)
    ap.add_argument("--baseline-lib", default=None, help="another libnvtb200.so to time nvtb_gb_list_rows against")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_session.py needs a CUDA device")
    import nvtabular_b200 as nvt
    from nvtabular_b200 import _lib
    from nvtabular_b200.graph import ColumnSelector
    from nvtabular_b200.synth import session_frame

    name, power = _card()
    res = {"workload": "session_ops", "gpu": name, "power_limit": power, "rows": args.rows}
    raw, n_sess = session_frame(args.rows, seed=args.seed)
    frame = _ordered(raw)
    del raw
    n = len(frame)
    res["sessions"] = n_sess

    lag = nvt.ops.DifferenceLag("session_id", shift=[1, -1])
    ms, _ = _time(lambda: lag.transform(ColumnSelector(["ts"]), frame), args.steps, args.warmup)
    # per shift: session_id and ts read, a float32 value and a validity bit written
    res["difference_lag"] = _family(ms, 2 * n * (8 + 8 + 4 + 0.125))

    gb = nvt.ops.Groupby("session_id", sort_cols="ts", aggs={"item_id": ["list"]})
    lists = gb.transform(ColumnSelector(["session_id", "item_id", "ts"]), frame)
    col = lists["item_id_list"]
    m, leaves_n = col.nrows, col.data.numel()
    lens = col.offsets[1:] - col.offsets[:-1]
    kept = int(torch.clamp(lens, max=20).sum().item())
    res["lists"] = {"rows": m, "leaves": leaves_n, "kept_by_slice": kept}
    sl = nvt.ops.ListSlice(-20)
    ms, _ = _time(lambda: sl.transform(ColumnSelector(["item_id_list"]), lists), args.steps, args.warmup)
    res["list_slice"] = _family(ms, m * 16.0 + kept * 8.0,
                                "offsets read and written, kept leaves read and written; includes one host read "
                                "of the output length")
    sp = nvt.ops.ListSlice(-20, pad=True)
    ms, _ = _time(lambda: sp.transform(ColumnSelector(["item_id_list"]), lists), args.steps, args.warmup)
    res["list_slice_pad"] = _family(ms, m * 16.0 + kept * 4.0 + m * 20 * 4.0,
                                    "offsets read and written, kept leaves read, n x 20 leaves written")

    # the Groupby first / last-of-list path: every sub-list copied, this build against the baseline
    leaves = col.leaves()
    lo, hi = col.offsets[:-1].contiguous(), col.offsets[1:].contiguous()
    libs = {"this": _lib.load()}
    if args.baseline_lib:
        libs["baseline"] = ctypes.CDLL(os.path.abspath(args.baseline_lib))
        libs["baseline"].nvtb_gb_list_rows.argtypes = _lib._SIGNATURES["nvtb_gb_list_rows"][1]
        libs["baseline"].nvtb_last_error.restype = ctypes.c_char_p
    for fn in libs.values():
        _list_rows_with(fn, leaves, lo, hi)
    ref_out, ref_off = _list_rows_with(libs["this"], leaves, lo, hi)
    same = True
    times = {k: [] for k in libs}
    for _ in range(args.steps):
        for k, fn in libs.items():
            t, _ = _time(lambda: _list_rows_with(fn, leaves, lo, hi), 1, 0)
            times[k].append(t)
    for k, fn in libs.items():
        out, off = _list_rows_with(fn, leaves, lo, hi)
        same = same and torch.equal(out, ref_out) and torch.equal(off, ref_off)
    res["list_rows"] = {k: _family(float(np.median(v)), m * 24.0 + leaves_n * 8.0,
                                   "lo / hi read, offsets written, every leaf read and written")
                        for k, v in times.items()}
    res["list_rows"]["outputs_identical"] = bool(same)
    res["parity"] = _parity(frame, args.seed + 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
