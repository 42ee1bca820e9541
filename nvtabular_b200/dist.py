"""Cross-GPU exchange for the fit statistics (SURVEY.md §8e).

One process per GPU (torch.distributed, NCCL over NVLink/NVSwitch).  Rows are
data-parallel; the only exchanges are
  * moments: one all-reduce of 5 doubles per column (engine.Moments.allreduce)
  * group-by tables: (key, size[, payload]) rows are routed to owner =
    mix(key) % world with ONE all-to-all per table, merged by the owner (exact
    global aggregates over disjoint keys), and the merged shards are
    all-gathered so every rank builds the identical vocabulary / stats table.
This replaces the reference's dask tree reduction over TCP/UCX and its shared
-filesystem "broadcast" (nvtabular/ops/categorify.py:1399-1540, 1627-1643).
On CPU test runs the same code path is exercised with the gloo backend
(tests/test_dist_cpu.py) with torch ops standing in for the device kernels.
"""
from typing import Optional

import numpy as np
import torch


def world():
    import os
    import torch.distributed as dist
    if os.environ.get("NVTB_DISABLE_DIST"):      # single-process reference fits inside a rank
        return 1, 0
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(), dist.get_rank()
    return 1, 0


def all_gather_object(obj):
    """[obj of rank 0, obj of rank 1, ...] on every rank (host metadata only: fit modes,
    string dictionaries — never row data)."""
    import torch.distributed as dist
    w, _ = world()
    if w == 1:
        return [obj]
    out = [None] * w
    dist.all_gather_object(out, obj)
    return out


# ---------------------------------------------------------------------------------------
# transport: the library's own NCCL communicator (csrc/comm.cu, nvtb_comm_t) when the process
# group runs on NCCL — torch.distributed then only carries the 128-byte unique id and host
# metadata; gloo (CPU tests) and NVTB_COMM=torch go through torch.distributed's collectives
# ---------------------------------------------------------------------------------------
_NATIVE = {"comm": None, "tried": False}


def native_comm():
    """-> ctypes handle of this process group's nvtb_comm_t, or None"""
    import ctypes
    import os
    import torch.distributed as dist
    if _NATIVE["tried"]:
        return _NATIVE["comm"]
    _NATIVE["tried"] = True
    w, rank = world()
    if w <= 1 or os.environ.get("NVTB_COMM", "native").lower() == "torch" or not dist.is_initialized() \
            or dist.get_backend() != "nccl" or not torch.cuda.is_available():
        return None
    from . import _lib
    lib = _lib.load()
    if not lib.nvtb_comm_available():
        return None
    buf = (ctypes.c_uint8 * 128)()
    if rank == 0:
        _lib.check(lib.nvtb_comm_unique_id(buf))
    box = [bytes(buf)]
    dist.broadcast_object_list(box, src=0)
    buf = (ctypes.c_uint8 * 128).from_buffer_copy(box[0])
    h = ctypes.c_void_p()
    _lib.check(lib.nvtb_comm_create(ctypes.byref(h), buf, rank, w))
    _NATIVE["comm"] = (lib, h)
    return _NATIVE["comm"]


def reset_native_comm():
    nc = _NATIVE["comm"]
    if nc is not None:
        nc[0].nvtb_comm_destroy(nc[1])
    _NATIVE["comm"], _NATIVE["tried"] = None, False


def alltoallv(send: torch.Tensor, send_counts, recv_counts) -> torch.Tensor:
    """variable-block all-to-all of a 1-D tensor: send_counts[r] elements go to rank r"""
    import ctypes
    import torch.distributed as dist
    from . import _lib
    recv = torch.empty(sum(recv_counts), dtype=send.dtype, device=send.device)
    nc = native_comm()
    if nc is not None and send.is_cuda:
        lib, h = nc
        sc = (ctypes.c_int64 * len(send_counts))(*[int(x) for x in send_counts])
        rc = (ctypes.c_int64 * len(recv_counts))(*[int(x) for x in recv_counts])
        send = send.contiguous()
        _lib.check(lib.nvtb_comm_alltoallv(h, ctypes.c_void_p(send.data_ptr()), sc, ctypes.c_void_p(recv.data_ptr()), rc,
                                           send.element_size(), _lib.stream_ptr()))
        return recv
    dist.all_to_all_single(recv, send.contiguous(), output_split_sizes=[int(x) for x in recv_counts],
                           input_split_sizes=[int(x) for x in send_counts])
    return recv


def allgather_equal(t: torch.Tensor) -> torch.Tensor:
    """all-gather of equal-sized 1-D blocks -> [world * n] in rank order"""
    import ctypes
    import torch.distributed as dist
    from . import _lib
    w, _ = world()
    t = t.contiguous()
    out = torch.empty(w * t.numel(), dtype=t.dtype, device=t.device)
    nc = native_comm()
    if nc is not None and t.is_cuda:
        lib, h = nc
        _lib.check(lib.nvtb_comm_allgather(h, ctypes.c_void_p(t.data_ptr()), ctypes.c_void_p(out.data_ptr()),
                                           t.numel() * t.element_size(), _lib.stream_ptr()))
        return out
    dist.all_gather_into_tensor(out, t)
    return out


def allreduce_sum_i64(t: torch.Tensor) -> torch.Tensor:
    import ctypes
    import torch.distributed as dist
    from . import _lib
    nc = native_comm()
    if nc is not None and t.is_cuda:
        lib, h = nc
        _lib.check(lib.nvtb_comm_allreduce_i64(h, ctypes.c_void_p(t.data_ptr()), t.numel(), 0, _lib.stream_ptr()))
        return t
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t


def exchange_by_owner(keys, sizes, vals, counts):
    """all-to-all of rows already grouped by owner (counts from
    engine.partition_by_owner).  Returns the rows this rank owns."""
    import torch.distributed as dist
    dev = keys.device
    send_counts = torch.tensor(counts, dtype=torch.int64, device=dev)
    recv_counts = torch.empty_like(send_counts)
    dist.all_to_all_single(recv_counts, send_counts)
    rc = [int(x) for x in recv_counts.cpu().tolist()]
    total = sum(rc)

    def a2a(t, width=1):
        out = torch.empty((total,) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)
        dist.all_to_all_single(out, t.contiguous(),
                               output_split_sizes=rc, input_split_sizes=list(counts))
        return out

    rk = a2a(keys)
    rs = a2a(sizes)
    rv = a2a(vals) if vals is not None else None
    return rk, rs, rv


def allgather_var(t: torch.Tensor):
    """all-gather of a variable-length (dim 0) tensor -> concatenation in rank order."""
    import torch.distributed as dist
    w, _ = world()
    dev = t.device
    n_local = torch.tensor([t.shape[0]], dtype=torch.int64, device=dev)
    n_all = [torch.empty_like(n_local) for _ in range(w)]
    dist.all_gather(n_all, n_local)
    n_all = [int(x.item()) for x in n_all]
    mx = max(max(n_all), 1)
    pad = torch.zeros((mx,) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)
    pad[: t.shape[0]] = t
    out = torch.empty((w * mx,) + tuple(t.shape[1:]), dtype=t.dtype, device=dev)
    dist.all_gather_into_tensor(out, pad)
    return torch.cat([out[r * mx: r * mx + n_all[r]] for r in range(w)])


def global_merge(agg, engine=None):
    """engine.HashAgg -> (keys, sizes, vals|None, null_size, null_vals|None),
    globally merged and identical on every rank.  `engine` is the kernel provider
    (nvtabular_b200.engine); the gloo/CPU tests inject a stand-in to exercise the
    exchange plumbing without a GPU."""
    if engine is None:
        from . import engine
    import torch.distributed as dist
    keys, sizes, vals, null_size, null_vals = agg.export()
    w, _ = world()
    if w == 1:
        return keys, sizes, vals, null_size, null_vals
    perm, counts = engine.partition_by_owner(keys, w)
    sk = engine.gather_i64(keys, perm)
    ss = engine.gather_i64(sizes, perm)
    sv = None
    if vals is not None:
        width = agg.n_agg * 4
        sv = engine.gather_f64_rows(vals.reshape(-1, width), perm, width)
    rk, rs, rv = exchange_by_owner(sk, ss, sv, counts)
    owner = engine.HashAgg(agg.n_agg, capacity_hint=max(rk.numel(), 1))
    owner.merge(rk, rs, rv.reshape(-1) if rv is not None else None)
    ok, os_, ov, _, _ = owner.export()
    all_k = allgather_var(ok)
    all_s = allgather_var(os_)
    all_v = allgather_var(ov) if ov is not None else None
    dev = keys.device
    ns = torch.tensor([null_size], dtype=torch.int64, device=dev)
    dist.all_reduce(ns, op=dist.ReduceOp.SUM)
    nv = None
    if null_vals is not None:
        t = torch.tensor(null_vals, dtype=torch.float64, device=dev)
        sums = t[:, 0:2].contiguous()
        mn = torch.nan_to_num(t[:, 2], nan=float("inf")).contiguous()
        mx = torch.nan_to_num(t[:, 3], nan=float("-inf")).contiguous()
        dist.all_reduce(sums, op=dist.ReduceOp.SUM)
        dist.all_reduce(mn, op=dist.ReduceOp.MIN)
        dist.all_reduce(mx, op=dist.ReduceOp.MAX)
        mn[torch.isinf(mn)] = float("nan")
        mx[torch.isinf(mx)] = float("nan")
        nv = torch.cat([sums, mn[:, None], mx[:, None]], dim=1).cpu().numpy()
    return all_k, all_s, all_v, int(ns.item()), nv


def global_merge_many(aggs, engine=None, owner_pool=None):
    """Cross-GPU merge of MANY keys-only tables (one per Categorify column) with a constant
    number of collectives: the per-column partials of all columns travel in ONE all-to-all
    (keys) + ONE (sizes), each owner merges its shard of every column, and the merged shards
    come back in ONE all-gather pair.  A 26-column fit costs ~8 NCCL calls instead of ~200,
    so the exchange is bound by NVLink bytes (O(#distinct keys)), not by launch latency.
    Returns [(keys, sizes, null_size)] per table, identical on every rank."""
    if engine is None:
        from . import engine
    import os
    import time
    import torch.distributed as dist
    w, rank = world()
    trace = bool(os.environ.get("NVTB_TRACE")) and w > 1
    marks = []

    def mark(name):
        if trace:
            torch.cuda.synchronize()
            marks.append((name, time.perf_counter()))

    mark("start")
    exported = [a.export() for a in aggs]            # (keys, sizes, None, null_size, None)
    mark("export")
    if w == 1:
        return [(k, s, ns) for (k, s, _, ns, _) in exported]
    nc = len(aggs)
    dev = exported[0][0].device
    # 1. group every column's rows by owner rank
    # (no host round trip per column: counts stay on the device until all 26 are queued)
    grouped = []
    counts_dev = torch.zeros((nc, w), dtype=torch.int64, device=dev)
    for c, (k, s, _, _, _) in enumerate(exported):
        perm = engine.partition_by_owner_async(k, w, counts_dev[c])
        grouped.append((engine.gather_i64(k, perm), engine.gather_i64(s, perm)))
    counts_nc = counts_dev.cpu()
    send_k = [[None] * nc for _ in range(w)]
    send_s = [[None] * nc for _ in range(w)]
    counts = counts_nc.t().contiguous()     # [owner rank, column]
    for c, (gk, gs) in enumerate(grouped):
        off = 0
        for r in range(w):
            n_rc = int(counts[r, c])
            send_k[r][c] = gk[off: off + n_rc]
            send_s[r][c] = gs[off: off + n_rc]
            off += n_rc
    mark("partition")
    sk = torch.cat([t for r in range(w) for t in send_k[r]])
    ss = torch.cat([t for r in range(w) for t in send_s[r]])
    mark("cat")
    # 2. exchange the count matrix, then keys and sizes
    cm_send = counts.to(dev).reshape(-1)
    cm_recv = torch.empty_like(cm_send)              # cm_recv[src, c] = rows src sends me for column c
    dist.all_to_all_single(cm_recv, cm_send)
    cm_recv_h = cm_recv.view(w, nc).cpu()
    in_split = [int(x) for x in counts.sum(dim=1).tolist()]
    out_split = [int(x) for x in cm_recv_h.sum(dim=1).tolist()]
    rk = alltoallv(sk, in_split, out_split)
    rs = alltoallv(ss, in_split, out_split)
    mark("all_to_all")
    # 3. owner merge per column (exact global sizes over disjoint keys)
    src_off = [0]
    for r in range(w):
        src_off.append(src_off[-1] + out_split[r])
    owned_k, owned_s, owners = [], [], []
    for c in range(nc):
        segs_k, segs_s = [], []
        for r in range(w):
            o = src_off[r] + int(cm_recv_h[r, :c].sum())
            n = int(cm_recv_h[r, c])
            segs_k.append(rk[o: o + n])
            segs_s.append(rs[o: o + n])
        ck, cs = torch.cat(segs_k), torch.cat(segs_s)
        # owner tables are pooled by the caller: creating a table (pinned mailbox, event,
        # device counters) costs far more than merging a shard into it
        if owner_pool is not None and c < len(owner_pool) and owner_pool[c] is not None:
            owner = owner_pool[c]
            owner.reset()
        else:
            owner = engine.HashAgg(0, capacity_hint=max(ck.numel(), 1))
            if owner_pool is not None:
                while len(owner_pool) <= c:
                    owner_pool.append(None)
                owner_pool[c] = owner
        owner.merge(ck, cs)
        owners.append(owner)
    # exports in a second loop: an export needs the merged size on the host, i.e. a sync on
    # that column's merge; issued right after each merge it would drain the stream 26 times
    for owner in owners:
        ok, os_, _, _, _ = owner.export()
        owned_k.append(ok)
        owned_s.append(os_)
    mark("owner_merge")
    # 4. all-gather the merged shards of all columns at once
    n_local = torch.tensor([t.numel() for t in owned_k], dtype=torch.int64, device=dev)
    n_all = torch.empty(w * nc, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(n_all, n_local)
    n_all_h = n_all.view(w, nc).cpu()
    tot = [int(x) for x in n_all_h.sum(dim=1).tolist()]
    mx = max(max(tot), 1)
    pk = torch.zeros(mx, dtype=torch.int64, device=dev)
    ps = torch.zeros(mx, dtype=torch.int64, device=dev)
    if tot[rank]:
        pk[: tot[rank]] = torch.cat(owned_k)
        ps[: tot[rank]] = torch.cat(owned_s)
    gk = allgather_equal(pk)
    gs = allgather_equal(ps)
    ns = torch.tensor([e[3] for e in exported], dtype=torch.int64, device=dev)
    dist.all_reduce(ns, op=dist.ReduceOp.SUM)
    ns_h = ns.cpu().tolist()
    mark("allgather")
    out = []
    for c in range(nc):
        ks, szs = [], []
        for r in range(w):
            o = r * mx + int(n_all_h[r, :c].sum())
            n = int(n_all_h[r, c])
            ks.append(gk[o: o + n])
            szs.append(gs[o: o + n])
        out.append((torch.cat(ks), torch.cat(szs), int(ns_h[c])))
    mark("split")
    if trace and rank == 0:
        print("[nvtb trace] merge_many: " + ", ".join(
            f"{marks[i][0]} {1e3 * (marks[i][1] - marks[i - 1][1]):.2f} ms" for i in range(1, len(marks)))
              + f"; keys sent {sk.numel()}, owned {sum(t.numel() for t in owned_k)}", flush=True)
    return out


# =======================================================================================
# High-cardinality columns: key-RANGE exchange of sorted packed pairs
# =======================================================================================
def global_merge_sorted(aggs, engine=None, device=None):
    """Cross-GPU merge of int32 key-count columns held as SORTED accumulators (key-ordered packed
    pairs word = (key ^ 2^31) << 32 | count; csrc/sortagg.cuh).  Returns, per column,
    (ordered_pairs, null_size): the GLOBAL vocabulary in (count desc, key asc) order, identical
    on every rank, ready for engine.Vocab.build_from_pairs.

    Nothing O(U_global) is sorted twice and nothing is re-hashed:
      1. owners are key RANGES; the split points are the mean of the ranks' local quantiles, so
         the local accumulator — already key-ordered — is already grouped by owner: the send
         buffer IS the accumulator, W-1 binary searches give the split sizes
      2. ONE all-to-all of 8-byte pairs; every owner receives W key-sorted runs and merges them
         pairwise adding counts (log2 W streaming merge rounds, nvtb_pairs_merge)
      3. every owner orders ITS shard by count (stable radix on the count bits in use) and
         run-length encodes the counts: a table of (count value, #keys) — a few thousand rows
      4. the tables are all-gathered; because owners hold disjoint, increasing key ranges, the
         global position of owner r's group of count c is
             #keys with a larger count (all owners) + #keys with count c on owners < r,
         computed identically on every rank from the small tables
      5. the count-ordered shards are all-gathered (8 B per distinct key — the "encode-table
         broadcast" of SURVEY.md 8e) and copied group by group to those positions
         (nvtb_segment_copy_u64): a streaming pass, no global sort.
    Reference analogue: the split_out shuffle + per-bucket concat/groupby + sort + shared
    filesystem read of nvtabular/ops/categorify.py:1036-1049, 1054-1070, 1296-1337, 1627-1643."""
    if engine is None:
        from . import engine
    import os
    import time
    import torch.distributed as dist
    w, rank = world()
    trace = bool(os.environ.get("NVTB_TRACE")) and w > 1
    out = []
    if not aggs:
        return out
    dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
    sizes = [a.size() for a in aggs]                      # (n_unique, null_size) per column
    ns = torch.tensor([s[1] for s in sizes], dtype=torch.int64, device=dev)
    if w > 1:
        allreduce_sum_i64(ns)
    ns_h = [int(x) for x in ns.cpu().tolist()]
    for c, agg in enumerate(aggs):
        t0 = time.perf_counter()
        p = agg.export_packed(dev)
        n = p.numel()
        if w == 1:
            S = p
        else:
            # 1. splitters from the ranks' local quantiles
            q = torch.zeros(w, dtype=torch.int64, device=dev)          # [n, q_1 .. q_{w-1}]
            q[0] = n
            if n:
                idx = (torch.arange(1, w, device=dev, dtype=torch.int64) * n) // w
                q[1:] = (p[idx] >> 32) & 0xFFFFFFFF
            allq = allgather_equal(q).view(w, w)
            live = (allq[:, 0] > 0).to(torch.float64)
            nlive = live.sum().clamp(min=1.0)
            spl = torch.floor((allq[:, 1:].to(torch.float64) * live[:, None]).sum(dim=0) / nlive).to(torch.int64)
            lb = engine.pairs_lower_bounds(p, spl) if n else torch.zeros(w - 1, dtype=torch.int64, device=dev)
            edges = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), lb,
                               torch.full((1,), n, dtype=torch.int64, device=dev)])
            send_counts = edges[1:] - edges[:-1]
            all_counts = allgather_equal(send_counts).view(w, w).cpu()       # [source, owner]
            sc_h = [int(x) for x in all_counts[rank].tolist()]
            rc_h = [int(x) for x in all_counts[:, rank].tolist()]
            # 2. one all-to-all of packed pairs, then the owner's pairwise merges
            recv = alltoallv(p, sc_h, rc_h)
            del p
            runs, off = [], 0
            for r in range(w):
                runs.append(recv[off: off + rc_h[r]])
                off += rc_h[r]
            while len(runs) > 1:
                nxt = []
                for i in range(0, len(runs) - 1, 2):
                    nxt.append(engine.pairs_merge(runs[i], runs[i + 1]))
                if len(runs) & 1:
                    nxt.append(runs[-1])
                runs = nxt
            S = runs[0]
            del recv, runs
        t1 = time.perf_counter()
        # 3. owner-side order by count (desc), stable => key asc within a count
        n_s = S.numel()
        if n_s:
            cnt = S & 0xFFFFFFFF
            mx = int(cnt.max().item())
            bits = max(1, mx.bit_length())
            C = engine.radix_sort(S, 0, bits, descending=True) if bits > 1 or mx > 1 else S
            if C is not S:
                cnt = C & 0xFFFFFFFF
            vals, lens = torch.unique_consecutive(cnt, return_counts=True)
            del cnt
        else:
            C = S
            vals = torch.zeros(0, dtype=torch.int64, device=dev)
            lens = torch.zeros(0, dtype=torch.int64, device=dev)
        del S
        if w == 1:
            out.append((C, ns_h[c]))
            continue
        # 4. small tables -> destination of every (owner, count value) group
        meta = torch.tensor([vals.numel(), n_s], dtype=torch.int64, device=dev)
        allmeta_h = allgather_equal(meta).view(w, 2).cpu()
        d_all = [int(x) for x in allmeta_h[:, 0].tolist()]
        n_all = [int(x) for x in allmeta_h[:, 1].tolist()]
        d_max, n_max, n_glob = max(max(d_all), 1), max(max(n_all), 1), sum(n_all)
        tab = torch.zeros(2 * d_max, dtype=torch.int64, device=dev)
        tab[: vals.numel()] = vals
        tab[d_max: d_max + lens.numel()] = lens
        alltab = allgather_equal(tab).view(w, 2, d_max)
        g_val, g_len, g_src, pad_src = [], [], [], []
        for r in range(w):                                  # groups listed owner-major
            g_val.append(alltab[r, 0, : d_all[r]])
            ln = alltab[r, 1, : d_all[r]]
            g_len.append(ln)
            g_src.append(r * n_max + torch.cumsum(ln, 0) - ln)
        g_val, g_len, g_src = torch.cat(g_val), torch.cat(g_len), torch.cat(g_src)
        order = torch.sort(g_val, descending=True, stable=True).indices     # ties keep owner order
        dst_sorted = torch.cumsum(g_len[order], 0) - g_len[order]
        g_dst = torch.empty_like(dst_sorted)
        g_dst[order] = dst_sorted
        # padding between the owners' shards in the gathered buffer: segments that are skipped
        seg_src = [g_src]
        seg_dst = [g_dst]
        for r in range(w):
            if n_all[r] < n_max:
                seg_src.append(torch.tensor([r * n_max + n_all[r]], dtype=torch.int64, device=dev))
                seg_dst.append(torch.tensor([-1], dtype=torch.int64, device=dev))
        seg_src, seg_dst = torch.cat(seg_src), torch.cat(seg_dst)
        o2 = torch.sort(seg_src).indices
        seg_src = torch.cat([seg_src[o2], torch.tensor([w * n_max], dtype=torch.int64, device=dev)])
        seg_dst = seg_dst[o2].contiguous()
        # 5. all-gather the count-ordered shards, interleave them group by group
        padded = torch.zeros(n_max, dtype=torch.int64, device=dev)
        padded[:n_s] = C
        del C
        gathered = allgather_equal(padded)
        del padded
        ordered = torch.empty(n_glob, dtype=torch.int64, device=dev)
        if n_glob:
            engine.segment_copy(gathered, ordered, seg_src, seg_dst)
        del gathered
        out.append((ordered, ns_h[c]))
        if trace and rank == 0 and dev.type == "cuda":
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            print(f"[nvtb trace] merge_sorted col {c}: local {n} pairs, shard {n_s}, global {n_glob}; "
                  f"exchange+merge {1e3 * (t1 - t0):.2f} ms, order+gather+interleave {1e3 * (t2 - t1):.2f} ms",
                  flush=True)
    return out
