"""world_size-2 gloo worker for tests/test_dist_cpu.py: runs the product's exchange
code (nvtabular_b200.dist.global_merge, engine.Moments.allreduce arithmetic) with a
numpy stand-in for the CUDA kernels, and writes each rank's result to disk."""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _mix(k):
    k = np.asarray(k).astype(np.uint64)
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(33); k *= np.uint64(0xFF51AFD7ED558CCD)
        k ^= k >> np.uint64(33); k *= np.uint64(0xC4CEB9FE1A85EC53)
        k ^= k >> np.uint64(33)
    return k


class FakeAgg:
    """host stand-in for engine.HashAgg (TEST ONLY)."""

    def __init__(self, n_agg=0, capacity_hint=0):
        self.n_agg = n_agg
        self.table = {}
        self.null_size = 0
        self.null_vals = np.tile(np.array([0.0, 0.0, np.nan, np.nan]), (max(n_agg, 1), 1))[:n_agg] if n_agg else None

    def merge(self, keys, sizes, vals=None):
        v = vals.reshape(-1, self.n_agg, 4).numpy() if vals is not None else None
        for i, (k, s) in enumerate(zip(keys.tolist(), sizes.tolist())):
            cur = self.table.get(k)
            if cur is None:
                self.table[k] = [s, v[i].copy() if v is not None else None]
            else:
                cur[0] += s
                if v is not None:
                    cur[1][:, 0:2] += v[i][:, 0:2]
                    cur[1][:, 2] = np.fmin(cur[1][:, 2], v[i][:, 2])
                    cur[1][:, 3] = np.fmax(cur[1][:, 3], v[i][:, 3])

    def export(self):
        keys = torch.tensor(list(self.table.keys()), dtype=torch.int64)
        sizes = torch.tensor([v[0] for v in self.table.values()], dtype=torch.int64)
        vals = torch.tensor(np.stack([v[1] for v in self.table.values()]), dtype=torch.float64) \
            if self.n_agg and self.table else (torch.zeros((0, self.n_agg, 4), dtype=torch.float64) if self.n_agg else None)
        return keys, sizes, vals, self.null_size, self.null_vals


class FakeEngine:
    HashAgg = FakeAgg

    @staticmethod
    def partition_by_owner(keys, n_parts):
        owner = ((_mix(keys.numpy()) >> np.uint64(52)) % np.uint64(n_parts)).astype(np.int64)
        perm = np.argsort(owner, kind="stable")
        return torch.from_numpy(perm), [int((owner == p).sum()) for p in range(n_parts)]

    @staticmethod
    def partition_by_owner_async(keys, n_parts, counts_out):
        perm, cnt = FakeEngine.partition_by_owner(keys, n_parts)
        counts_out.copy_(torch.tensor(cnt, dtype=torch.int64))
        return perm

    @staticmethod
    def gather_i64(src, perm):
        return src[perm]

    @staticmethod
    def gather_f64_rows(src, perm, width):
        return src[perm]


def main():
    out_dir = sys.argv[1]
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    from nvtabular_b200.dist import allgather_var, global_merge
    rng = np.random.default_rng(100 + rank)
    # each rank saw different rows: overlapping key sets, different counts
    keys = rng.integers(0, 500, 3000)
    x = rng.standard_normal(3000)
    agg = FakeAgg(1)
    for k, v in zip(keys.tolist(), x.tolist()):
        agg.merge(torch.tensor([k]), torch.tensor([1]), torch.tensor([[v, v * v, v, v]], dtype=torch.float64))
    agg.null_size = 7 + rank
    agg.null_vals = np.array([[1.0 + rank, 2.0, -3.0 - rank, 4.0 + rank]])
    k, s, v, ns, nv = global_merge(agg, engine=FakeEngine)
    order = np.argsort(k.numpy())
    res = {"keys": k.numpy()[order].tolist(), "sizes": s.numpy()[order].tolist(),
           "vals": v.numpy()[order].reshape(len(order), -1).tolist(), "null_size": ns, "null_vals": nv.tolist(),
           "local_keys": keys.tolist(), "local_x": x.tolist()}
    # many keys-only tables at once (the Categorify path)
    from nvtabular_b200.dist import global_merge_many
    many = []
    local_cols = []
    for c in range(5):
        kk = rng.integers(0, 50 * (c + 1), 2000)
        a = FakeAgg(0)
        for key in kk.tolist():
            a.merge(torch.tensor([key]), torch.tensor([1]))
        a.null_size = c + rank
        many.append(a)
        local_cols.append(kk.tolist())
    merged = global_merge_many(many, engine=FakeEngine)
    res["many"] = []
    for (mk, ms, mns) in merged:
        o = np.argsort(mk.numpy())
        res["many"].append({"keys": mk.numpy()[o].tolist(), "sizes": ms.numpy()[o].tolist(), "null": mns})
    res["many_local"] = local_cols
    # high-cardinality path: key-range exchange of sorted packed pairs (dist.global_merge_sorted)
    # with numpy stand-ins for the device primitives
    from nvtabular_b200.dist import global_merge_sorted

    class PackedAgg:
        def __init__(self, keys_i32, nulls):
            u, c = np.unique(keys_i32.astype(np.int64), return_counts=True)
            uk = (u + (1 << 31)).astype(np.uint64)                     # key ^ 2^31 == key + 2^31 for int32
            self.pairs = torch.from_numpy(((uk << np.uint64(32)) | c.astype(np.uint64)).view(np.int64))
            self.nulls = nulls

        def size(self):
            return self.pairs.numel(), self.nulls

        def export_packed(self, device=None):
            return self.pairs.clone()

    def _u(t):
        return t.numpy().view(np.uint64)

    class SortedEngine:
        @staticmethod
        def pairs_lower_bounds(pairs, bounds):
            k = _u(pairs) >> np.uint64(32)
            return torch.from_numpy(np.searchsorted(k, bounds.numpy().astype(np.uint64), side="left").astype(np.int64))

        @staticmethod
        def pairs_merge(a, b):
            w = np.concatenate([_u(a), _u(b)])
            k, c = w >> np.uint64(32), w & np.uint64(0xFFFFFFFF)
            uk, inv = np.unique(k, return_inverse=True)
            cs = np.zeros(len(uk), dtype=np.uint64)
            np.add.at(cs, inv, c)
            return torch.from_numpy(((uk << np.uint64(32)) | cs).view(np.int64))

        @staticmethod
        def radix_sort(data, lo_bit=0, hi_bit=None, descending=False):
            w = _u(data)
            f = (w >> np.uint64(lo_bit)) & np.uint64((1 << (hi_bit - lo_bit)) - 1)
            order = np.argsort(-f.astype(np.int64) if descending else f.astype(np.int64), kind="stable")
            return torch.from_numpy(w[order].view(np.int64))

        @staticmethod
        def segment_copy(src, dst, seg_src, seg_dst):
            ss, sd = seg_src.tolist(), seg_dst.tolist()
            for j in range(len(sd)):
                if sd[j] >= 0:
                    n = ss[j + 1] - ss[j]
                    dst[sd[j]: sd[j] + n] = src[ss[j]: ss[j + 1]]

    big_local = []
    big = []
    for c in range(2):
        kk = (rng.integers(0, 4000 * (c + 1), 9000 + 1000 * rank) * 2654435761 % (1 << 31) - (1 << 30) * c).astype(np.int32)
        big_local.append(kk.tolist())
        big.append(PackedAgg(kk, 3 + c + rank))
    res["sorted"] = []
    for ordered, nsz in global_merge_sorted(big, engine=SortedEngine, device=torch.device("cpu")):
        w = _u(ordered)
        res["sorted"].append({"keys": ((w >> np.uint64(32)).astype(np.int64) - (1 << 31)).tolist(),
                              "sizes": (w & np.uint64(0xFFFFFFFF)).astype(np.int64).tolist(), "null": nsz})
    res["sorted_local"] = big_local
    t = allgather_var(torch.arange(rank + 2, dtype=torch.int64))
    res["allgather_var"] = t.tolist()
    with open(os.path.join(out_dir, f"rank{rank}.json"), "w") as f:
        json.dump(res, f)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
