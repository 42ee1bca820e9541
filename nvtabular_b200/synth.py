"""Deterministic synthetic tables in the shapes BASELINE.json names (SURVEY.md
§8d), generated directly in device memory with torch (data generation is not
part of any measured region).

Criteo-shape: `label:int32`, `I1..I13:int32` (nullable), `C1..C26:int32`
(nullable) — column names per reference bench/examples/
dask-nvtabular-criteo-benchmark.py:135-141.  Categorical ids follow the
reference's own power-law inverse CDF (nvtabular/tools/data_gen.py:55-66,
alpha=0.1) and are scattered over the int32 range with a multiplicative
permutation so key order != frequency order.
"""
from typing import Dict, List, Optional

import numpy as np
import torch

from .column import Column, DeviceFrame, pack_validity

CONT_NAMES = [f"I{i}" for i in range(1, 14)]
CAT_NAMES = [f"C{i}" for i in range(1, 27)]
# distinct-value profile of the public Criteo-1TB categorical features; the four raw
# high-cardinality columns are the reference's own list (benchmark.py:361: C20,C1,C22,C10)
CRITEO_CARDINALITY = {
    "C1": 230_000_000, "C2": 39_043, "C3": 17_289, "C4": 7_420, "C5": 20_263, "C6": 3, "C7": 7_120,
    "C8": 1_543, "C9": 63, "C10": 130_000_000, "C11": 2_953_546, "C12": 403_346, "C13": 10,
    "C14": 2_208, "C15": 11_938, "C16": 155, "C17": 4, "C18": 976, "C19": 14, "C20": 290_000_000,
    "C21": 40_000_000, "C22": 190_000_000, "C23": 585_935, "C24": 12_972, "C25": 108, "C26": 36,
}
CRITEO_ROWS = 4_370_000_000


def scaled_cardinality(name: str, total_rows: int) -> int:
    """Low-cardinality features saturate; high-cardinality ones grow with the row count."""
    k = CRITEO_CARDINALITY[name]
    if k <= 100_000:
        return k
    s = min(1.0, total_rows / CRITEO_ROWS)
    return max(100_000, int(round(k * s)))


def _gen(seed: int, device) -> torch.Generator:
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    return g


def _null_mask(n, frac, g, device) -> Optional[torch.Tensor]:
    if frac <= 0:
        return None
    valid = torch.rand(n, generator=g, device=device) >= frac
    return pack_validity(valid)


def power_law_ids(n: int, k: int, g, device, alpha: float = 0.1) -> torch.Tensor:
    """data_gen.py:55-66 with min_val=1, max_val=k: x = (u*(k^g - 1) + 1)^(1/g), g = 1-alpha."""
    gamma = 1.0 - alpha
    u = torch.rand(n, generator=g, device=device, dtype=torch.float64)
    x = torch.pow(u * (float(k) ** gamma - 1.0) + 1.0, 1.0 / gamma)
    return torch.clamp(x.to(torch.int64), 1, k)


def scatter_ids(ids: torch.Tensor) -> torch.Tensor:
    """bijection on [0, 2^31): key = id * 2654435761 mod 2^31 (odd multiplier)."""
    return ((ids * 2654435761) & 0x7FFFFFFF).to(torch.int32)


def criteo_frame(rows: int, total_rows: Optional[int] = None, seed: int = 1234, device="cuda",
                 alpha: float = 0.1, rank: int = 0) -> DeviceFrame:
    """One device-resident shard of `rows` rows of a `total_rows`-row Criteo-shape table."""
    total_rows = total_rows or rows
    cols: Dict[str, Column] = {}
    g = _gen(seed + 10_000 * rank, device)
    cols["label"] = Column((torch.rand(rows, generator=g, device=device) < 0.03).to(torch.int32))
    for j, name in enumerate(CONT_NAMES):
        g = _gen(seed + 1 + j + 10_000 * rank, device)
        z = torch.randn(rows, generator=g, device=device, dtype=torch.float32) * 2.0 + 2.0
        v = torch.floor(torch.exp(z.to(torch.float64))).clamp_(0, 2**31 - 1).to(torch.int32)
        neg = torch.rand(rows, generator=g, device=device) < 0.10            # ~10 % are -1..-3
        v = torch.where(neg, -(torch.randint(1, 4, (rows,), generator=g, device=device, dtype=torch.int32)), v)
        cols[name] = Column(v, _null_mask(rows, 0.45 * j / 12.0, g, device))
    for j, name in enumerate(CAT_NAMES):
        g = _gen(seed + 100 + j + 10_000 * rank, device)
        k = scaled_cardinality(name, total_rows)
        keys = scatter_ids(power_law_ids(rows, k, g, device, alpha))
        cols[name] = Column(keys, _null_mask(rows, 0.10 * j / 25.0, g, device))
    return DeviceFrame(cols)


def frame_to_pandas_nullable(frame: DeviceFrame, rows: Optional[int] = None):
    """Host copy of (a prefix of) a frame as pandas nullable-int columns (for the CPU oracle)."""
    import pandas as pd
    from .column import unpack_validity
    out = {}
    for name, c in frame.items():
        n = c.data.numel() if rows is None else min(rows, c.data.numel())
        vals = c.data[:n].cpu().numpy()
        if c.validity is not None:
            valid = unpack_validity(c.validity, c.data.numel())[:n].cpu().numpy()
            arr = pd.array(vals, dtype="Int32")
            arr[~valid] = pd.NA
            out[name] = arr
        else:
            out[name] = vals
    return pd.DataFrame(out)


def movielens_frame(rows: int, seed: int = 4321, device="cuda", rank: int = 0) -> DeviceFrame:
    """MovieLens-25M-shaped ratings: userId (K=1.6e5), movieId (K=6e4, power-law), rating 0.5..5.0."""
    g = _gen(seed + 10_000 * rank, device)
    user = scatter_ids(power_law_ids(rows, 160_000, g, device, 0.1))
    movie = scatter_ids(power_law_ids(rows, 60_000, g, device, 0.5))
    rating = (torch.randint(1, 11, (rows,), generator=g, device=device).to(torch.float32)) * 0.5
    return DeviceFrame({"userId": Column(user), "movieId": Column(movie), "rating": Column(rating)})


def hashbucket_frame(rows: int, ncols: int = 40, n_ids: int = 100_000_000, seed: int = 777, device="cuda",
                     rank: int = 0) -> DeviceFrame:
    """BASELINE.json configs[4] (SURVEY.md 8d C5): `ncols` int64 key columns, keys uniform over
    `n_ids` ids mixed through a 64-bit bijection (odd multiply, xor-shift, odd multiply — wrapping
    int64 arithmetic), no nulls.  Input of HashBucket(num_buckets=2**20)."""
    cols: Dict[str, Column] = {}
    m1, m2 = -7046029254386353131, -4658895280553007687      # 0x9E3779B97F4A7C15, 0xBF58476D1CE4E5B9 as int64
    for j in range(ncols):
        g = _gen(seed + j + 10_000 * rank, device)
        k = torch.randint(0, n_ids, (rows,), generator=g, device=device, dtype=torch.int64)
        k.mul_(m1)
        k.bitwise_xor_((k >> 29) & ((1 << 35) - 1))       # logical shift: a bijection
        k.mul_(m2)
        cols[f"K{j + 1}"] = Column(k)
    return DeviceFrame(cols)


def session_frame(rows: int, seed: int = 1234, device="cuda", mean_length: float = 10.0):
    """A synthetic session table of `rows` rows, grouped by nothing: session_id (int64, lengths
    drawn from a Zipf-like power law with about rows / mean_length sessions, rows shuffled),
    item_id (int32), ts (int64 seconds near 1.7e9), price (float32).  -> (DeviceFrame, sessions)."""
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    n_sess = max(1, int(rows / mean_length))
    # power-law lengths: a Pareto tail, scaled to the row count
    u = torch.rand(n_sess, generator=g, device=device, dtype=torch.float64)
    w = u.clamp_min(1e-12).pow(-1.0 / 1.2)
    lens = torch.floor(w / w.sum() * (rows - n_sess)).to(torch.int64) + 1
    lens[0] += rows - int(lens.sum().item())
    sid = torch.repeat_interleave(torch.arange(n_sess, dtype=torch.int64, device=device), lens)
    perm = torch.randperm(rows, generator=g, device=device)
    sid = sid[perm].contiguous()
    item = torch.randint(0, 1 << 20, (rows,), generator=g, device=device, dtype=torch.int32)
    ts = 1_700_000_000 + torch.randint(0, 1 << 24, (rows,), generator=g, device=device, dtype=torch.int64)
    price = torch.rand(rows, generator=g, device=device, dtype=torch.float32) * 100
    return DeviceFrame({"session_id": Column(sid), "item_id": Column(item), "ts": Column(ts),
                        "price": Column(price)}), n_sess
