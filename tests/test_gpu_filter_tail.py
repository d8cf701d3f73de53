"""k-way IntersectSorted with a deferred sparse tail: a sample of the driving list picks how many lists the pipeline
streams (k_eff), and filter_tail_kernel searches the rest for the survivors.  Every result is checked bit-exact against
the oracle; dgx_filter_tail_queries shows whether the tail pass served a query.  Deferral happens on resident-inputs
lanes only (the sample then runs under the previous batch's pipeline) and for driving lists of at least 65536 values,
so the lane of this module is declared resident and the deferring queries are that long."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen  # noqa: E402
from test_gpu_parity import eq  # noqa: E402

pytestmark = pytest.mark.gpu
U64_TOP = (1 << 64) - 1


@pytest.fixture(scope="module")
def env():
    import torch
    from dgraph_b200 import _lib

    lib = _lib.load()
    _lib.check(lib.dgx_init(-1))
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    lane = lib.dgx_lane_create(0, C.c_void_p(stream.cuda_stream))
    assert lane
    _lib.check(lib.dgx_lane_set_resident_inputs(lane, 1))
    yield lib, lane, dev, stream
    lib.dgx_lane_destroy(lane)


def to_dev(dev, a):
    import torch
    return torch.from_numpy(np.concatenate([a, np.zeros(2, np.uint64)]).view(np.int64)).to(dev)


def submit(env, queries, cap, tensors=None, out=None):
    """One dgx_dev_filter_batch (intersection) on the lane; returns (out, off, inputs) without syncing."""
    import torch
    from dgraph_b200 import _lib

    lib, lane, dev, _ = env
    flat = tensors if tensors is not None else [to_dev(dev, l) for q in queries for l in q]
    lens = [l.size for q in queries for l in q]
    koff = np.concatenate([[0], np.cumsum([len(q) for q in queries])])
    if out is None:
        out = torch.full((cap + 8,), -1, dtype=torch.int64, device=dev)
    off = torch.zeros(len(queries) + 1, dtype=torch.int64, device=dev)
    _lib.check(lib.dgx_dev_filter_batch(lane, 0, (C.c_void_p * len(flat))(*[t.data_ptr() for t in flat]),
                                        (C.c_size_t * len(lens))(*lens),
                                        (C.c_size_t * len(koff))(*[int(x) for x in koff]), len(queries),
                                        C.c_void_p(out.data_ptr()), cap, C.c_void_p(off.data_ptr())))
    return out, off, flat


def check(out, off, queries, orc, what, want=None):
    ho, hoff = out.cpu().numpy().view(np.uint64), off.cpu().numpy().view(np.uint64)
    if want is None:
        want = [orc.intersect_sorted(q) for q in queries]
    eq(hoff, np.concatenate([[0], np.cumsum([w.size for w in want])]), f"{what}: out_off")
    for qi, w in enumerate(want):
        eq(ho[int(hoff[qi]): int(hoff[qi + 1])], w, f"{what}: query {qi} k={len(queries[qi])}")


def run(env, queries, orc, what, cap=None, want=None):
    """Submit, sync, check; returns (tail queries served, launches) of the batch."""
    from dgraph_b200 import _lib
    import torch

    lib, lane, dev, stream = env
    with torch.cuda.stream(stream):
        if cap is None:
            cap = sum(min(l.size for l in q) for q in queries)
        l0 = lib.dgx_lane_launches(lane)
        _lib.check(lib.dgx_lane_sync(lane))
        t0 = lib.dgx_filter_tail_queries(lane)
        out, off, keep = submit(env, queries, cap)
        launches = lib.dgx_lane_launches(lane) - l0
        _lib.check(lib.dgx_lane_sync(lane))
        check(out, off, queries, orc, what, want)
        return lib.dgx_filter_tail_queries(lane) - t0, launches


def sparse(rng, n, k, p=0.25, start=0):
    master = gen.zipf_gaps(rng, int(n / p), start=start)
    return [gen.thin(rng, master, p) for _ in range(k)]


def test_c2_shaped_and_dense(env, orc):
    rng = np.random.default_rng(1)
    qs = [sparse(rng, 100_000, 8) for _ in range(6)]
    tail, launches = run(env, qs, orc, "C2-shaped")
    assert tail == 6, "every C2-shaped query defers its sparse lists"
    assert launches == 5  # sample, tiles, plan, pipeline, tail
    qs = [sparse(rng, 100_000, 8, p=0.9) for _ in range(6)]
    tail, launches = run(env, qs, orc, "dense")
    assert tail == 0, "a dense query streams all of its lists"
    assert launches == 5


def test_streaming_path_kept(env, orc):
    """Lanes without resident inputs, and batches whose driving lists are too short to sample, keep the three
    launches of the streaming path (tiles, plan, pipeline) and defer nothing."""
    from dgraph_b200 import _lib

    lib, lane, dev, stream = env
    rng = np.random.default_rng(11)
    qs = [sparse(rng, 100_000, 8) for _ in range(4)]
    _lib.check(lib.dgx_lane_set_resident_inputs(lane, 0))
    try:
        tail, launches = run(env, qs, orc, "C2-shaped, lane without resident inputs")
        assert (tail, launches) == (0, 3)
    finally:
        _lib.check(lib.dgx_lane_set_resident_inputs(lane, 1))
    tail, launches = run(env, [sparse(rng, 30_000, 8) for _ in range(4)], orc, "short driving lists")
    assert (tail, launches) == (0, 3)


def test_mixed_batch(env, orc):
    rng = np.random.default_rng(2)
    qs = []
    for q in range(24):
        kind = q % 4
        if kind == 0:
            qs.append(sparse(rng, 30_000, 1))
        elif kind == 1:
            qs.append(sparse(rng, 30_000, 2))
        elif kind == 2:
            qs.append(sparse(rng, 80_000, 8))
        else:
            qs.append(sparse(rng, 80_000, 5, p=0.9))
    qs.append([np.zeros(0, np.uint64), gen.zipf_gaps(rng, 100), gen.zipf_gaps(rng, 200)])  # empty driving list
    tail, _ = run(env, qs, orc, "mixed batch")
    assert tail == 6


def late_split(rng, n, k, dense_lists):
    """A, then dense_lists supersets of A (everything survives), then lists holding ~1 % of A among other values:
    the split falls after the first of those, so more than 8 lists are streamed when dense_lists >= 8."""
    master = gen.zipf_gaps(rng, 2 * n) * np.uint64(2)
    a = gen.thin(rng, master, 0.3)
    lists = [a]
    for i in range(dense_lists):
        lists.append(np.union1d(a, gen.thin(rng, master, 0.4 + 0.01 * i)))
    odd = master + np.uint64(1)
    for i in range(k - 1 - dense_lists):
        lists.append(np.union1d(gen.thin(rng, odd, 0.95), gen.thin(rng, a, 0.01 if i == 0 else 0.5)))
    return lists


@pytest.mark.parametrize("k", [3, 9, 12, 16])
def test_wide_queries(env, orc, k):
    rng = np.random.default_rng(10 + k)
    if k == 3:
        qs = [sparse(rng, 80_000, 3, p=0.015) for _ in range(4)]
    else:
        qs = [sparse(rng, 80_000, k) for _ in range(3)]
        if k > 9:
            qs += [late_split(rng, 150_000, k, 9) for _ in range(2)]
    tail, _ = run(env, qs, orc, f"k={k}")
    assert tail == len(qs)


def test_duplicates(env, orc):
    rng = np.random.default_rng(4)
    master = gen.zipf_gaps(rng, 400_000)

    def with_copies(p):
        v = gen.thin(rng, master, p)
        return np.repeat(v, rng.integers(1, 4, v.size))

    qs = [[with_copies(0.25) for _ in range(8)] for _ in range(4)]
    # a value repeated in every list: its copies survive into the tail
    for q in qs:
        for i, l in enumerate(q):
            q[i] = np.sort(np.concatenate([l, np.full(3 + i % 3, master[1000], np.uint64)]))
    # The r-th copy of x in A survives list L iff L holds more than r copies (multiset-min), the rule of the
    # reference's two-pointer IntersectWith.  The reference's IntersectSorted chain switches to its jump / binary
    # variants once the intermediate is much shorter than the next list, and those keep fewer copies; these lists
    # shrink 4x per list, so the rule is stated through the oracle's two-pointer merge.
    want = []
    for q in qs:
        ls = sorted(q, key=len)
        w = ls[0]
        for l in ls[1:]:
            w = orc.intersect_with_lin(w, l)
        want.append(w)
    tail, _ = run(env, qs, orc, "duplicates", want=want)
    assert tail == len(qs)


def test_high_values(env, orc):
    rng = np.random.default_rng(5)
    qs = [sparse(rng, 80_000, 8, start=(1 << 32) - 150_000_000) for _ in range(3)]
    for _ in range(3):
        m = gen.zipf_gaps(rng, 400_000)
        top = np.uint64(U64_TOP) - (m[-1] - m)  # ascending, ends at 2^64 - 1
        lists = [gen.thin(rng, top, 0.25) for _ in range(8)]
        lists = [np.union1d(l, np.array([U64_TOP], np.uint64)) for l in lists]
        qs.append(lists)
    tail, _ = run(env, qs, orc, "values near 2^32 and 2^64 - 1")
    assert tail == len(qs)


def test_empty_lists(env, orc):
    rng = np.random.default_rng(6)
    qs = [sparse(rng, 80_000, 8) for _ in range(2)]
    q = sparse(rng, 80_000, 6)
    q[3] = np.zeros(0, np.uint64)  # an empty list (the shortest, so it drives the query)
    qs.append(q)
    even = gen.zipf_gaps(rng, 300_000) * np.uint64(2)
    qs.append([even[::2], even[1::2] + np.uint64(1)] + [gen.thin(rng, even, 0.6) for _ in range(4)])  # empties at once
    tail, _ = run(env, qs, orc, "empty lists")
    assert tail >= 2


def test_out_cap(env, orc):
    import torch
    from dgraph_b200 import _lib

    lib, lane, dev, stream = env
    rng = np.random.default_rng(7)
    qs = [sparse(rng, 80_000, 8) for _ in range(4)]
    total = sum(orc.intersect_sorted(q).size for q in qs)
    assert total > 0
    run(env, qs, orc, "out_cap = result", cap=total)
    with torch.cuda.stream(stream):
        out, off, keep = submit(env, qs, total - 1)
        assert lib.dgx_lane_sync(lane) == -4  # DGX_ERR_CAP
        assert (out[total - 1:].cpu() == -1).all(), "a value was written past out_cap"


def test_resident_lane(env, orc):
    """Deferring batches back to back on a resident-inputs lane (alternating workspaces), and a chain that reads the
    previous batch's output."""
    import torch
    from dgraph_b200 import _lib

    lib, lane, dev, stream = env
    rng = np.random.default_rng(8)
    batches = [[sparse(rng, int(rng.integers(70_000, 120_000)), int(rng.integers(5, 11)))
                for _ in range(int(rng.integers(1, 5)))] for _ in range(5)]
    with torch.cuda.stream(stream):
        dls = [[to_dev(dev, l) for q in b for l in q] for b in batches]
        caps = [sum(min(l.size for l in q) for q in b) for b in batches]
        outs = [torch.full((c + 8,), -1, dtype=torch.int64, device=dev) for c in caps]
        torch.cuda.synchronize()
        t0 = lib.dgx_filter_tail_queries(lane)
        for rep in range(3):
            res = [submit(env, b, c, tensors=d, out=o) for b, c, d, o in zip(batches, caps, dls, outs)]
            _lib.check(lib.dgx_lane_sync(lane))
            for i, (b, (o, off, _)) in enumerate(zip(batches, res)):
                check(o, off, b, orc, f"resident batch {i}, rep {rep}")
        assert lib.dgx_filter_tail_queries(lane) - t0 == 3 * sum(len(b) for b in batches)

        # chain: the second batch's driving list is the first one's output
        q1 = sparse(rng, 80_000, 8)
        want1 = orc.intersect_sorted(q1)
        extra = [np.union1d(want1, gen.zipf_gaps(rng, 5_000) * np.uint64(3)) for _ in range(3)]
        q2 = [want1] + extra
        want2 = orc.intersect_sorted(q2)
        d1 = [to_dev(dev, l) for l in q1]
        d2x = [to_dev(dev, l) for l in extra]
        mid = torch.full((want1.size + 8,), -7, dtype=torch.int64, device=dev)
        fin = torch.full((want1.size + 8,), -1, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        for rep in range(3):
            if rep:
                mid.fill_(-7)
            o1, off1, _ = submit(env, [q1], want1.size, tensors=d1, out=mid)
            o2, off2, _ = submit(env, [q2], want1.size, tensors=[mid] + d2x, out=fin)
            _lib.check(lib.dgx_lane_sync(lane))
            eq(fin[: int(off2[1].item())].cpu().numpy().view(np.uint64), want2, f"chained batch, rep {rep}")


def test_dyn_len_lists(env, orc):
    """Decode(pack, seek) feeds a list whose length is known on the device only.  These calls run on the pooled
    lanes of the host-pointer API, which hold no resident inputs: the lists are streamed, none deferred."""
    from dgraph_b200 import _lib, codec, pb

    lib = _lib.load()
    rng = np.random.default_rng(9)
    for seek_frac in (0.0, 0.4):
        lists = sparse(rng, 80_000, 7)
        op = orc.encode(lists[0], 256)
        pk = pb.UidPack(op.block_size, op.base, op.num_uids, op.delta_off, op.deltas)
        seek = int(lists[0][int(seek_frac * (lists[0].size - 1))])
        t0 = lib.dgx_filter_tail_queries(None)
        got = codec.DecodeIntersectSorted(pk, seek, [pb.List(l) for l in lists[1:]])
        want = orc.intersect_sorted([orc.decode(op, seek)] + lists[1:])
        eq(got.Uids, want, f"DecodeIntersectSorted, seek {seek}")
        assert lib.dgx_filter_tail_queries(None) == t0
