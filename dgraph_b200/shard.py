"""Multi-GPU sharding (SURVEY.md 8e): batches of independent set operations (pattern 1, below) and one huge
MergeSorted range-partitioned over lists that are sharded by list (pattern 2, at the end of the file).

The reference fans a batch of independent posting-list intersections over
goroutines (x.DivideAndRule, worker/task.go:816-987); here the same batch is
partitioned over the GPUs of one box, one process per GPU.  Units (pairs /
queries) are independent, so there is NO data-path collective; the only exchange
is the final result concatenation (an all-gatherv = all_gather of counts, then of
payloads padded to the largest shard), done with torch.distributed (NCCL on GPUs,
gloo in the CPU tests).

This module is host logic only: which units a rank owns and how results are put
back in unit order.  The compute step is passed in by the caller (libdgx on a
GPU box).
"""
from __future__ import annotations

import os
from typing import Callable, List, Sequence, Tuple

import numpy as np


def lpt_partition(costs: Sequence[int], world: int) -> List[np.ndarray]:
    """Longest-processing-time-first greedy partition of units by cost (bytes).

    Returns, per rank, the sorted unit indices it owns.  Deterministic: ties go to
    the lowest rank, units are visited in (cost desc, index asc) order.
    """
    costs = np.asarray(costs, dtype=np.int64)
    order = np.lexsort((np.arange(costs.size), -costs))
    load = np.zeros(world, dtype=np.int64)
    owner = np.empty(costs.size, dtype=np.int64)
    for u in order:
        r = int(np.argmin(load))  # first minimum -> lowest rank on ties
        owner[u] = r
        load[r] += costs[u]
    return [np.nonzero(owner == r)[0] for r in range(world)]


def contiguous_partition(costs: Sequence[int], world: int) -> List[np.ndarray]:
    """Split units 0..n-1 into `world` CONTIGUOUS blocks of roughly equal cost (cut at the cost
    prefix nearest to r/world of the total).  Imbalance is at most one unit's cost; in exchange a
    rank's results are already contiguous in unit order, so the final concatenation needs no
    scatter: rank payloads are simply laid end to end."""
    costs = np.asarray(costs, dtype=np.int64)
    n = costs.size
    pref = np.concatenate([[0], np.cumsum(costs)])
    total = int(pref[-1])
    cuts = [0]
    for r in range(1, world):
        target = total * r // world
        c = int(np.searchsorted(pref, target, side="left"))
        cuts.append(min(max(c, cuts[-1]), n))
    cuts.append(n)
    return [np.arange(cuts[r], cuts[r + 1]) for r in range(world)]


def gatherv_contiguous(dist, local_out, local_off, device=None):
    """All-gatherv for contiguous shards (contiguous_partition): returns (out, off) in unit order.
    local_off: this rank's CSR offsets (len = units + 1).  Counts travel first, then payloads padded
    to the largest shard; rank payloads are laid end to end."""
    import torch

    world = dist.get_world_size()
    dev = local_out.device if device is None else device
    meta = torch.tensor([local_off.numel() - 1, int(local_off[-1].item())], dtype=torch.int64, device=dev)
    metas = [torch.zeros(2, dtype=torch.int64, device=dev) for _ in range(world)]
    dist.all_gather(metas, meta)
    nun = [int(m[0].item()) for m in metas]
    tot = [int(m[1].item()) for m in metas]
    max_u, max_t = max(max(nun), 1), max(max(tot), 1)
    lens_local = torch.zeros(max_u, dtype=torch.int64, device=dev)
    lens_local[: local_off.numel() - 1] = local_off[1:] - local_off[:-1]
    lens_all = torch.empty(world * max_u, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(lens_all, lens_local)
    pay_local = torch.empty(max_t, dtype=torch.int64, device=dev)
    pay_local[: int(local_off[-1].item())] = local_out[: int(local_off[-1].item())]
    pay_all = torch.empty(world * max_t, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(pay_all, pay_local)
    lens_g = torch.cat([lens_all[r * max_u: r * max_u + nun[r]] for r in range(world)])
    off_g = torch.zeros(lens_g.numel() + 1, dtype=torch.int64, device=dev)
    off_g[1:] = torch.cumsum(lens_g, 0)
    out_g = torch.cat([pay_all[r * max_t: r * max_t + tot[r]] for r in range(world)])
    return out_g, off_g


def gatherv_exact(dist, parts, local_out, local_off, device=None):
    """All-gatherv for CONTIGUOUS shards (contiguous_partition) with exact sizes: returns (out, off) in unit order,
    identical on every rank.

    1. one all_gather of the per-unit result lengths (shards padded to the largest shard's unit count, which is
       static: the partition is computed from the inputs' sizes on every rank);
    2. ONE host read of those lengths (the only synchronisation): offsets and per-rank totals follow on the host;
    3. every rank's payload travels straight to its final position in `out` -- grouped point-to-point sends and
       receives of the exact sizes (ncclGroupStart/End under NCCL), no padding to the largest shard, no scatter.
    """
    import torch

    world = dist.get_world_size()
    rank = dist.get_rank()
    dev = local_out.device if device is None else device
    n_r = [len(p) for p in parts]
    max_u = max(max(n_r), 1)
    lens_local = torch.zeros(max_u, dtype=torch.int64, device=dev)
    if n_r[rank]:
        lens_local[: n_r[rank]] = local_off[1: n_r[rank] + 1] - local_off[: n_r[rank]]
    lens_all = torch.empty(world * max_u, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(lens_all, lens_local)
    lens_host = lens_all.cpu().numpy().reshape(world, max_u)          # the one host synchronisation
    tot = [int(lens_host[r, : n_r[r]].sum()) for r in range(world)]
    lens_g = np.concatenate([lens_host[r, : n_r[r]] for r in range(world)]) if sum(n_r) else np.zeros(0, np.int64)
    off_host = np.zeros(lens_g.size + 1, dtype=np.int64)
    np.cumsum(lens_g, out=off_host[1:])
    base = np.concatenate([[0], np.cumsum(tot)]).astype(np.int64)
    out_g = torch.empty(max(int(base[-1]), 1), dtype=torch.int64, device=dev)
    if dist.get_backend() == "nccl" and world > 2 and 8 * int(base[-1]) >= (64 << 20):
        # Bandwidth regime on many GPUs: NCCL's point-to-point transfers to many peers run well below the link rate,
        # its all_gather collective (ring / NVLS) runs closer to it.  The collective needs equal
        # shard sizes, so shards travel padded to the largest one (contiguous_partition balances by bytes: the padding
        # is a few percent) and are then moved to their final, compact positions at HBM speed.
        max_t = max(tot)
        send = local_out[:max_t] if local_out.numel() >= max_t else torch.cat(
            [local_out[: tot[rank]], torch.empty(max_t - tot[rank], dtype=torch.int64, device=dev)])
        buf = torch.empty(world * max_t, dtype=torch.int64, device=dev)
        dist.all_gather_into_tensor(buf, send)
        for r in range(world):
            if tot[r]:
                out_g[int(base[r]): int(base[r]) + tot[r]].copy_(buf[r * max_t: r * max_t + tot[r]])
        return out_g[: int(base[-1])], torch.from_numpy(off_host).to(dev)
    # grouped point-to-point transfers of the exact sizes (ncclGroupStart/End under NCCL), one per peer: one large
    # transfer per peer beats cutting it into pieces, and beats NCCL's uneven all_gather (one broadcast per rank).
    piece = int(os.environ.get("DGX_GATHER_PIECE", str(1 << 40)))  # values per transfer (default: one per peer)
    ops = []
    for r in range(world):
        if r == rank:
            if tot[r]:
                out_g[int(base[r]): int(base[r]) + tot[r]].copy_(local_out[: tot[r]])
            continue
        for o in range(0, tot[rank], piece):
            ops.append(dist.P2POp(dist.isend, local_out[o: min(o + piece, tot[rank])], r))
        for o in range(0, tot[r], piece):
            ops.append(dist.P2POp(dist.irecv, out_g[int(base[r]) + o: int(base[r]) + min(o + piece, tot[r])], r))
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()
    return out_g[: int(base[-1])], torch.from_numpy(off_host).to(dev)


def shard_offsets(counts: np.ndarray) -> np.ndarray:
    out = np.zeros(counts.size + 1, dtype=np.int64)
    np.cumsum(counts, out=out[1:])
    return out


def gatherv_results(dist, local_units: np.ndarray, local_out, local_off, n_units: int, device=None):
    """All-gatherv of per-unit results.

    local_units: global indices of the units this rank computed (ascending).
    local_out:   torch int64 tensor, this rank's results concatenated in local unit order.
    local_off:   torch int64 tensor (len(local_units)+1), CSR offsets into local_out.
    Returns (out, off): torch tensors holding every unit's result in GLOBAL unit order
    (identical on all ranks).
    """
    import torch

    world = dist.get_world_size()
    rank = dist.get_rank()
    dev = local_out.device if device is None else device
    # 1) per-unit lengths of every rank, padded to the largest shard (all_gather needs equal shapes)
    n_local = torch.tensor([len(local_units)], dtype=torch.int64, device=dev)
    n_all = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in range(world)]
    dist.all_gather(n_all, n_local)
    n_all = [int(t.item()) for t in n_all]
    max_units = max(max(n_all), 1)
    lens_local = torch.zeros(max_units, dtype=torch.int64, device=dev)
    ids_local = torch.full((max_units,), -1, dtype=torch.int64, device=dev)
    if len(local_units):
        lens_local[: len(local_units)] = local_off[1:] - local_off[:-1]
        ids_local[: len(local_units)] = torch.as_tensor(np.asarray(local_units), dtype=torch.int64, device=dev)
    lens_all = [torch.zeros_like(lens_local) for _ in range(world)]
    ids_all = [torch.zeros_like(ids_local) for _ in range(world)]
    dist.all_gather(lens_all, lens_local)
    dist.all_gather(ids_all, ids_local)
    # 2) payloads, padded to the largest shard
    tot_local = torch.tensor([int(local_off[-1].item()) if local_off.numel() else 0], dtype=torch.int64, device=dev)
    tot_all = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in range(world)]
    dist.all_gather(tot_all, tot_local)
    tot_all = [int(t.item()) for t in tot_all]
    max_tot = max(max(tot_all), 1)
    pay_local = torch.zeros(max_tot, dtype=torch.int64, device=dev)
    pay_local[: tot_all[rank]] = local_out[: tot_all[rank]]
    pay_all = [torch.zeros_like(pay_local) for _ in range(world)]
    dist.all_gather(pay_all, pay_local)
    # 3) scatter back into global unit order
    lens_g = torch.zeros(n_units, dtype=torch.int64, device=dev)
    for r in range(world):
        if n_all[r]:
            lens_g[ids_all[r][: n_all[r]]] = lens_all[r][: n_all[r]]
    off_g = torch.zeros(n_units + 1, dtype=torch.int64, device=dev)
    off_g[1:] = torch.cumsum(lens_g, 0)
    out_g = torch.zeros(max(int(off_g[-1].item()), 1), dtype=torch.int64, device=dev)
    for r in range(world):
        if n_all[r] == 0 or tot_all[r] == 0:
            continue
        ids = ids_all[r][: n_all[r]]
        ln = lens_all[r][: n_all[r]]
        src_off = torch.cumsum(ln, 0) - ln
        dst_off = off_g[ids]
        # element-wise destination index of every payload value of rank r
        rep = torch.repeat_interleave(torch.arange(n_all[r], device=dev), ln)
        within = torch.arange(tot_all[r], device=dev) - src_off[rep]
        out_g[dst_off[rep] + within] = pay_all[r][: tot_all[r]]
    return out_g[: int(off_g[-1].item())], off_g


def run_sharded_pairs(dist, a_lists, b_lists, compute: Callable, device=None, partition: str = "contiguous"):
    """Intersect pair i = (a_lists[i], b_lists[i]) for all i, sharded over the process group.

    compute(units, a_lists, b_lists) -> (out int64 tensor, off int64 tensor) for the units a
    rank owns (on a GPU box: one dgx_dev_filter_batch launch).  Returns results in pair order.
    partition "contiguous" (default): shards are runs of consecutive pairs balanced by bytes, results come back
    through gatherv_exact (one host sync, exact sizes).  "lpt": longest-processing-time partition (tighter balance
    when a few pairs dominate) with the general, index-scattering gatherv_results.
    """
    world = dist.get_world_size()
    rank = dist.get_rank()
    costs = [8 * (len(a) + len(b)) for a, b in zip(a_lists, b_lists)]
    if partition == "lpt":
        parts = lpt_partition(costs, world)
        mine = parts[rank]
        out, off = compute(mine, a_lists, b_lists)
        return gatherv_results(dist, mine, out, off, len(a_lists), device=device)
    parts = contiguous_partition(costs, world)
    mine = parts[rank]
    out, off = compute(mine, a_lists, b_lists)
    return gatherv_exact(dist, parts, out, off, device=device)


# ---------------------------------------------------------------------------------------------------------------
# Pattern 2 (SURVEY.md 8e): ONE huge operation over lists that start SHARDED BY LIST -- range-partition the uid space.
#
# The reference splits a posting list that outgrows one key by uid range (posting/list.go:580-646 iterator part
# selection, :2260-2271 split policy); the same idea shards one huge MergeSorted over the GPUs: G-1 splitters cut the
# uid space into G ranges, rank r merges range r of EVERY list, equal uids land on one rank (no cross-rank
# duplicates), and the results concatenate in rank order.  When a rank holds only some of the lists, each list's
# slice of range r has to travel to rank r first: one all-to-all, the single data-path collective of this package.
# ---------------------------------------------------------------------------------------------------------------

_SIGN = -(1 << 63)


def _ukey(t):
    """Order-preserving int64 key of a uint64 bit pattern held in an int64 tensor (uids above 2^63 sort last)."""
    return t ^ _SIGN


def range_splitters(dist, local_lists, oversample: int = 1024, device=None):
    """world-1 uid splitters (int64 bit patterns of uint64 values, ascending, identical on every rank).

    Every rank samples its lists at a common stride (one sample per `total / (world * oversample)` values, so a list
    weighs in proportion to its length), the samples are all-gathered, sorted, and the i/world quantiles taken.
    Two tiny collectives (totals, sample counts) + one all_gather of the samples."""
    import torch

    world = dist.get_world_size()
    dev = device if device is not None else (local_lists[0].device if local_lists else torch.device("cpu"))
    if world == 1:
        return torch.zeros(0, dtype=torch.int64, device=dev)
    tot_local = torch.tensor([sum(int(l.numel()) for l in local_lists)], dtype=torch.int64, device=dev)
    tots = torch.empty(world, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(tots, tot_local)
    total = int(tots.sum().item())
    stride = max(total // (world * oversample), 1)
    picks = [l[stride // 2:: stride] for l in local_lists if l.numel()]
    mine = _ukey(torch.cat(picks)) if picks else torch.zeros(0, dtype=torch.int64, device=dev)
    cnt = torch.tensor([mine.numel()], dtype=torch.int64, device=dev)
    cnts = torch.empty(world, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(cnts, cnt)
    cnts_h = cnts.cpu().numpy()
    cap = max(int(cnts_h.max()), 1)
    send = torch.full((cap,), (1 << 63) - 1, dtype=torch.int64, device=dev)  # pads sort last as keys
    send[: mine.numel()] = mine
    allk = torch.empty(world * cap, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(allk, send)
    keys = torch.cat([allk[r * cap: r * cap + int(cnts_h[r])] for r in range(world)])
    keys, _ = torch.sort(keys)
    if keys.numel() == 0:
        return torch.zeros(world - 1, dtype=torch.int64, device=dev)  # nothing anywhere: any splitters will do
    idx = torch.tensor([(i * keys.numel()) // world for i in range(1, world)], dtype=torch.int64, device=dev)
    return _ukey(keys[idx])


def exchange_by_range(dist, local_lists, splitters, device=None):
    """The all-to-all: rank r receives, from every rank, the slice [splitter[r-1], splitter[r]) of each of that rank's
    lists.  Returns the received runs (sorted int64 tensors, grouped by source rank, then in the source's list
    order; empty slices are dropped).  Slices are cut with lower_bound, so all copies of a uid go to ONE rank.

    Collectives: all_to_all of the slice lengths (fixed size), one host read of the cuts and one of the received
    lengths, all_to_all of the payload with the exact sizes (NCCL: ncclSend/ncclRecv inside one group)."""
    import torch

    world = dist.get_world_size()
    rank = dist.get_rank()
    dev = device if device is not None else (local_lists[0].device if local_lists else splitters.device)
    if world == 1:
        return [l for l in local_lists if l.numel()]
    nl = torch.tensor([len(local_lists)], dtype=torch.int64, device=dev)
    nls = torch.empty(world, dtype=torch.int64, device=dev)
    dist.all_gather_into_tensor(nls, nl)
    lmax = max(int(nls.max().item()), 1)
    skey = _ukey(splitters)
    # cut[l, d] .. cut[l, d + 1] = slice of local list l that belongs to rank d
    pieces = [[] for _ in range(world)]
    lens_to_h = np.zeros((world, lmax), dtype=np.int64)
    if local_lists:
        cuts = torch.stack([torch.searchsorted(_ukey(l), skey, right=False) if l.numel()
                            else torch.zeros(world - 1, dtype=torch.int64, device=dev) for l in local_lists])
        cuts_h = cuts.cpu().numpy()                                       # one host read for all the lists
        for li, l in enumerate(local_lists):
            cut_h = [0] + [int(c) for c in cuts_h[li]] + [int(l.numel())]
            for d in range(world):
                n = cut_h[d + 1] - cut_h[d]
                lens_to_h[d, li] = n
                if n:
                    pieces[d].append(l[cut_h[d]: cut_h[d + 1]])
    lens_to = torch.from_numpy(lens_to_h).to(dev)
    lens_from = torch.empty_like(lens_to)
    dist.all_to_all_single(lens_from.view(-1), lens_to.view(-1))          # row s of lens_from: rank s's slices for me
    lens_from_h = lens_from.cpu().numpy()                                    # the one host synchronisation
    in_split = [int(sum(int(p.numel()) for p in pieces[d])) for d in range(world)]
    out_split = [int(lens_from_h[s].sum()) for s in range(world)]
    send = torch.cat([p for d in range(world) for p in pieces[d]]) if sum(in_split) else torch.zeros(0, dtype=torch.int64, device=dev)
    recv = torch.empty(sum(out_split), dtype=torch.int64, device=dev)
    if dist.get_backend() == "nccl":
        dist.all_to_all_single(recv, send, output_split_sizes=out_split, input_split_sizes=in_split)
    else:  # gloo: grouped point-to-point transfers of the exact sizes
        ops, so, ro = [], 0, 0
        for r in range(world):
            if r == rank:
                recv[ro: ro + out_split[r]].copy_(send[so: so + in_split[r]])
            else:
                if in_split[r]:
                    ops.append(dist.P2POp(dist.isend, send[so: so + in_split[r]], r))
                if out_split[r]:
                    ops.append(dist.P2POp(dist.irecv, recv[ro: ro + out_split[r]], r))
            so += in_split[r]
            ro += out_split[r]
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()
    runs, o = [], 0
    for s in range(world):
        for li in range(lmax):
            n = int(lens_from_h[s, li])
            if n:
                runs.append(recv[o: o + n])
            o += n
    return runs


def run_range_merge(dist, local_lists, merge: Callable, gather: bool = True, oversample: int = 1024, device=None):
    """MergeSorted over lists sharded BY LIST across the process group (every rank passes the lists it holds).

    merge(runs) -> sorted, de-duplicated int64 tensor of the runs this rank received (on a GPU box: one
    dgx_dev_merge_sorted launch).  gather=True returns the whole result on every rank (rank-ordered all-gatherv, so
    ascending); gather=False returns this rank's uid range only (what a following range-partitioned operation wants).
    Also returns the splitters, so a second operand can be cut the same way (exchange_by_range)."""
    import torch

    world = dist.get_world_size()
    rank = dist.get_rank()
    spl = range_splitters(dist, local_lists, oversample=oversample, device=device)
    runs = exchange_by_range(dist, local_lists, spl, device=device)
    mine = merge(runs)
    if not gather or world == 1:
        return mine, spl
    parts = [np.array([r]) for r in range(world)]
    off = torch.tensor([0, int(mine.numel())], dtype=torch.int64, device=mine.device)
    out, _ = gatherv_exact(dist, parts, mine, off, device=device)
    return out, spl
