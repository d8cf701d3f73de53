"""@recurse on the device (dgx_recurse_filter, dgx_dev_recurse_filter and the dgx_reach_set they share): every step of
whole recursions compared with the line-by-line restatement (recurse_oracle.c), guard words past every output, the set
compared edge by edge, launches with the plan model (recurse_plan.py).  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import json
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen_recurse as gr  # noqa: E402
import recurse_oracle as ro  # noqa: E402
import recurse_plan as rp  # noqa: E402

pytestmark = pytest.mark.gpu

OK, ERR_ARG, ERR_CAP = 0, -3, -4
SENT = 0xDEADBEEFCAFEF00D
GUARD = 4
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "recurse_friend_follow.json")


@pytest.fixture(scope="module")
def lib():
    from dgraph_b200 import _lib

    L = _lib.load()
    _lib.check(L.dgx_init(-1))
    return L


def new_lane(lib):
    import torch

    stream = torch.cuda.Stream()
    ln = lib.dgx_lane_create(0, C.c_void_p(stream.cuda_stream))
    assert ln
    return ln, stream


@pytest.fixture(scope="module")
def lane(lib):
    ln, stream = new_lane(lib)
    yield ln
    lib.dgx_lane_destroy(ln)


def _b(a):
    a = np.ascontiguousarray(np.asarray(a, np.uint64))
    return a if a.size else np.zeros(1, np.uint64)


def export(s):
    f, t = s.export()
    return f.tolist(), t.tolist()


class HostEngine:
    """One algo.ReachSet per Attr, stepped through the host form."""

    def __init__(self):
        from dgraph_b200 import algo

        self.algo, self.sets = algo, {}

    def set(self, attr):
        if attr not in self.sets:
            self.sets[attr] = self.algo.ReachSet()
        return self.sets[attr]

    def step(self, attr, src, rows, dest):
        kept, d, n = self.set(attr).filter(src, rows, dest)
        return kept, d.Uids, n


class DevEngine(HostEngine):
    """The device form on one lane: inputs uploaded, outputs fenced by guard words, launches checked with the plan."""

    def __init__(self, lib, lane, slack=0):
        super().__init__()
        self.lib, self.lane, self.slack = lib, lane, slack

    def step(self, attr, src, rows, dest):
        rc, src_rc, sizes, kept, d, launches, guards = dev_step(self.lib, self.lane, self.set(attr).handle, src, rows,
                                                                dest, self.slack)
        assert rc == OK and src_rc == OK and guards
        m = sum(len(r) for r in rows)
        assert launches == rp.launches(len(rows), m + self.slack)
        return kept, d, int(sizes[0])


def dev_step(lib, lane, handle, src, rows, dest, slack=0, v_off=None, out_cap=None, dest_cap=None):
    """(rc, rc of the sync, sizes, kept rows, DestUIDs, launches, guards intact)."""
    import torch

    def up(x):
        return torch.from_numpy(_b(x).view(np.int64)).cuda()

    def sent(n):
        return torch.full((n,), SENT - (1 << 64), dtype=torch.int64, device="cuda")

    v, off = ro.csr(rows)
    if v_off is not None:
        off = np.asarray(v_off, np.uint64)
    nrows, m = len(rows), int(sum(len(r) for r in rows))
    v_cap = m + slack
    v = np.concatenate([v, np.zeros(slack + 1, np.uint64)])
    out_cap = v_cap if out_cap is None else out_cap
    dest_cap = v_cap if dest_cap is None else dest_cap
    d_src, d_v, d_off = up(src), up(v), up(off)
    d_dest = None if dest is None else up(dest)
    d_out, d_out_off, d_dout, d_sizes = sent(out_cap + GUARD), sent(nrows + 1 + GUARD), sent(dest_cap + GUARD), sent(
        2 + GUARD)
    torch.cuda.synchronize()
    l0 = lib.dgx_lane_launches(lane)
    rc = lib.dgx_dev_recurse_filter(lane, handle, d_src.data_ptr(), nrows, d_v.data_ptr(), d_off.data_ptr(), v_cap,
                                    None if d_dest is None else d_dest.data_ptr(), 0 if dest is None else len(dest),
                                    d_out.data_ptr(), d_out_off.data_ptr(), out_cap, d_dout.data_ptr(), dest_cap,
                                    d_sizes.data_ptr())
    src_rc = lib.dgx_lane_sync(lane)
    launches = lib.dgx_lane_launches(lane) - l0
    out, out_off, dout, sizes = (t.cpu().numpy().view(np.uint64) for t in (d_out, d_out_off, d_dout, d_sizes))
    guards = (np.all(out[out_cap:] == SENT) and np.all(out_off[nrows + 1:] == SENT) and
              np.all(dout[dest_cap:] == SENT) and np.all(sizes[2:] == SENT))
    if rc != OK or src_rc != OK:  # a refused step writes d_sizes = {0, 0} at most, nothing else
        guards = guards and np.all(out == SENT) and np.all(out_off == SENT) and np.all(dout == SENT)
        return rc, src_rc, sizes[:2], None, None, launches, guards
    K, D = int(sizes[0]), int(sizes[1])
    assert int(out_off[nrows]) == K and np.all(out[K:out_cap] == SENT) and np.all(dout[D:dest_cap] == SENT)
    kept = [out[int(out_off[i]):int(out_off[i + 1])].copy() for i in range(nrows)]
    return rc, src_rc, sizes[:2], kept, dout[:D].copy(), launches, guards


def checked(engine, reach, ids):
    """A step function that runs the engine and the restatement and asserts they agree."""
    def step(attr, src, rows, dest):
        want = reach.step(ids.setdefault(attr, len(ids) + 1), src, rows, dest)
        got = engine.step(attr, src, rows, dest)
        assert got[2] == want[2]
        assert np.array_equal(got[1], want[1])
        assert all(np.array_equal(a, b) for a, b in zip(got[0], want[0]))
        return want
    return step


def check_sets(engine, reach, ids):
    for attr, i in ids.items():
        f, t = reach.edges(i)
        assert engine.set(attr).size() == f.size
        assert export(engine.set(attr)) == (f.tolist(), t.tolist())


def random_recursion(rng, engine, n_max=300):
    n = int(rng.integers(2, n_max))
    preds = [f"p{i}" for i in range(int(rng.integers(1, 4)))]
    graph = gr.random_graph(rng, n, preds, mean_deg=float(rng.uniform(1, 5)), self_loops=bool(rng.random() < 0.7))
    roots = rng.choice(np.arange(1, n + 1), size=int(rng.integers(1, 6)), replace=False)
    filters = {p: rng.choice(np.arange(1, n + 1), size=int(rng.integers(0, n + 1)), replace=False)
               for p in preds if rng.random() < 0.4}
    reach, ids = ro.Reach(), {}
    steps, total, _ = gr.recurse(graph, roots, preds, int(rng.integers(1, 9)), checked(engine, reach, ids),
                                 filters=filters)
    check_sets(engine, reach, ids)
    return steps, total


@pytest.mark.parametrize("form", ["host", "device"])
def test_random_recursions(lib, lane, form):
    rng = np.random.default_rng(140 if form == "host" else 141)
    for k in range(40):
        engine = HostEngine() if form == "host" else DevEngine(lib, lane, slack=int(rng.integers(0, 3)) * (k % 2))
        random_recursion(rng, engine)


def test_friend_follow_example(lib, lane):
    with open(GOLDEN) as f:
        d = json.load(f)
    graph = {p: gr.Pred.from_edges(1003, *zip(*e)) for p, e in d["edges"].items() if e}
    c = d["cases"]["friend_follow"]
    for engine in (HostEngine(), DevEngine(lib, lane)):
        reach, ids = ro.Reach(), {}
        steps, n, _ = gr.recurse(graph, [1], c["preds"], c["depth"], checked(engine, reach, ids))
        assert n == c["edges"] and max(s.level for s in steps) == c["levels"]
        assert [s.kept for s in steps if s.level == 2][2] == 0
        check_sets(engine, reach, ids)
        assert engine.set("friend").size() == 7 and engine.set("follow").size() == 7


def _host_call(lib, s, src, rows, dest=None, v_off=None, out_cap=None, dest_cap=None, nrows=None):
    v, off = ro.csr(rows)
    if v_off is not None:
        off = np.asarray(v_off, np.uint64)
    m = int(off[-1]) if len(off) else 0
    out_cap = m if out_cap is None else out_cap
    dest_cap = m if dest_cap is None else dest_cap
    out, dout = np.full(out_cap + GUARD, SENT, np.uint64), np.full(dest_cap + GUARD, SENT, np.uint64)
    out_off = np.full(len(rows) + 1 + GUARD, SENT, np.uint64)
    n = C.c_size_t(0)
    src_a, dest_a = _b(src), None if dest is None else _b(dest)  # alive through the call
    dd = None if dest is None else dest_a.ctypes.data
    rc = lib.dgx_recurse_filter(s.handle, src_a.ctypes.data, len(rows) if nrows is None else nrows, v.ctypes.data,
                                off.ctypes.data, dd, 0 if dest is None else len(dest), out.ctypes.data,
                                out_off.ctypes.data, out_cap, dout.ctypes.data, dest_cap, C.byref(n))
    return rc, out, out_off, dout


def _seeded():
    from dgraph_b200 import algo

    s = algo.ReachSet.from_edges([1, 1, 5], [2, 9, 5])
    s.filter([1, 3], [[2, 4], [7]])
    return s


BAD_STEPS = {  # each refused on the device; the inputs are otherwise valid
    "src descending": ([3, 1], [[4], [6]], None),
    "src repeated": ([3, 3], [[4], [6]], None),
    "row descending": ([1, 3], [[4, 3], [6]], None),
    "row repeated": ([1, 3], [[4], [6, 6]], None),
    "dest descending": ([1, 3], [[4], [6]], [6, 4]),
}


@pytest.mark.parametrize("name", sorted(BAD_STEPS))
def test_refused_steps_leave_the_set_unchanged(lib, lane, name):
    src, rows, dest = BAD_STEPS[name]
    s = _seeded()
    before = export(s)
    rc, out, out_off, dout = _host_call(lib, s, src, rows, dest)
    assert rc == ERR_ARG and np.all(out == SENT) and np.all(out_off == SENT) and np.all(dout == SENT)
    assert export(s) == before
    rc, src_rc, sizes, _, _, _, guards = dev_step(lib, lane, s.handle, src, rows, dest)
    assert rc == OK and src_rc == ERR_ARG and sizes.tolist() == [0, 0] and guards
    assert export(s) == before
    # the set goes on as if the refused step had never run
    kept, d, n = s.filter([1, 3], [[2, 3], [7, 8]])
    assert n == 2 and [k.tolist() for k in kept] == [[3], [8]] and d.Uids.tolist() == [3, 8]


def test_argument_and_capacity_errors(lib, lane):
    from dgraph_b200 import algo

    s = _seeded()
    before = export(s)
    src, rows = [1, 3], [[2, 6], [7]]
    assert _host_call(lib, s, src, rows, v_off=[1, 2, 3])[0] == ERR_ARG  # offsets not from 0
    assert _host_call(lib, s, src, rows, v_off=[0, 2, 1])[0] == ERR_ARG  # decreasing
    assert _host_call(lib, s, src, rows, v_off=[0, 2, 1 << 32], out_cap=3, dest_cap=3)[0] == ERR_ARG  # 2^32 values
    assert _host_call(lib, s, src, rows, nrows=1 << 32)[0] == ERR_ARG
    assert _host_call(lib, s, src, rows, out_cap=2)[0] == ERR_CAP
    assert _host_call(lib, s, src, rows, dest_cap=2)[0] == ERR_CAP
    n = C.c_size_t(0)
    buf = np.zeros(8, np.uint64)
    off3 = np.array([0, 2, 3], np.uint64)
    assert lib.dgx_recurse_filter(s.handle, None, 2, buf.ctypes.data, off3.ctypes.data,
                                  None, 0, buf.ctypes.data, buf.ctypes.data, 3, buf.ctypes.data, 3,
                                  C.byref(n)) == ERR_ARG
    assert lib.dgx_recurse_filter(None, buf.ctypes.data, 0, None, None, None, 0, None, buf.ctypes.data, 0, None, 0,
                                  C.byref(n)) == ERR_ARG
    assert export(s) == before
    # the device form: caps, sizes and pointers at the call; bad offsets on the device
    assert dev_step(lib, lane, s.handle, src, rows, None, out_cap=2)[0] == ERR_CAP
    assert dev_step(lib, lane, s.handle, src, rows, None, dest_cap=2)[0] == ERR_CAP
    for off in ([1, 2, 3], [0, 2, 1], [0, 2, 9]):
        rc, src_rc, sizes, _, _, _, guards = dev_step(lib, lane, s.handle, src, rows, None, v_off=off)
        assert rc == OK and src_rc == ERR_ARG and sizes.tolist() == [0, 0] and guards
    assert lib.dgx_dev_recurse_filter(lane, s.handle, None, 2, None, None, 3, None, 0, None, None, 3, None, 3,
                                      None) == ERR_ARG
    assert export(s) == before
    # create: not strictly ascending, null arrays
    h = C.c_void_p()
    f, t = np.array([1, 1], np.uint64), np.array([2, 2], np.uint64)
    assert lib.dgx_reach_create(f.ctypes.data, t.ctypes.data, 2, C.byref(h)) == ERR_ARG
    assert lib.dgx_reach_create(None, None, 2, C.byref(h)) == ERR_ARG
    with pytest.raises(Exception):
        algo.ReachSet.from_edges([2, 1], [1, 1])
    # export: too small a cap
    cnt = C.c_size_t(0)
    assert lib.dgx_reach_export(s.handle, buf.ctypes.data, buf.ctypes.data, 1, C.byref(cnt)) == ERR_CAP
    assert cnt.value == len(before[0])


def test_set_bound_to_one_lane(lib, lane):
    from dgraph_b200 import algo

    other, _ = new_lane(lib)
    try:
        s = algo.ReachSet()
        rc, src_rc = dev_step(lib, lane, s.handle, [1], [[2, 3]], None)[:2]
        assert rc == OK and src_rc == OK
        # lane_sync waited for the stream, but only dgx_reach_size / export release the set
        assert dev_step(lib, other, s.handle, [2], [[3]], None)[0] == ERR_ARG
        assert _host_call(lib, s, [2], [[3]])[0] == ERR_ARG
        assert s.size() == 2
        rc, src_rc, sizes = dev_step(lib, other, s.handle, [1, 2], [[3, 4], [3]], None)[:3]
        assert rc == OK and src_rc == OK and sizes.tolist() == [2, 2]
        assert export(s) == ([1, 1, 1, 2], [2, 3, 4, 3])
    finally:
        lib.dgx_lane_destroy(other)


def test_growth_across_doublings(lib, lane):
    rng = np.random.default_rng(5)
    graph = {"a": gr.zipf_pred(rng, 20000, 4.0), "b": gr.zipf_pred(rng, 20000, 2.0)}
    for engine in (HostEngine(), DevEngine(lib, lane)):
        reach, ids = ro.Reach(), {}
        gr.recurse(graph, rng.integers(1, 20001, 50), ["a", "b"], 6, checked(engine, reach, ids))
        check_sets(engine, reach, ids)
        assert engine.set("a").size() > 4 * 1024  # the first capacity is 1024 edges


@pytest.mark.parametrize("form", ["host", "device"])
def test_handoff_mid_recursion(lib, lane, form):
    """Levels 1-3 on one set, then export -> from_edges: the rest goes on exactly as without the handoff; and the
    reverse, a set created from the restatement's map mid-way."""
    from dgraph_b200 import algo

    rng = np.random.default_rng(9)
    graph = gr.random_graph(rng, 400, ["a", "b"], mean_deg=3)
    roots = [int(np.argmax(np.diff(graph["a"].ptr)))]
    engine = HostEngine() if form == "host" else DevEngine(lib, lane)
    reach, ids = ro.Reach(), {}
    inner = checked(engine, reach, ids)
    state = {"level": 0}

    def step(attr, src, rows, dest):
        state["level"] += 1
        if state["level"] == 12:  # hand every set over: device -> host arrays -> a new device set
            for a, s in list(engine.sets.items()):
                f, t = s.export()
                s.close()
                engine.sets[a] = algo.ReachSet.from_edges(f, t)
        if state["level"] == 20:  # from the restatement's map, as a shim handing over from Go does
            for a in list(engine.sets):
                engine.sets[a].close()
                engine.sets[a] = algo.ReachSet.from_edges(*reach.edges(ids[a]))
        return inner(attr, src, rows, dest)

    gr.recurse(graph, roots, ["a", "b"], 8, step)
    assert state["level"] > 20
    check_sets(engine, reach, ids)


def test_launches_fixed_at_fixed_v_cap(lib, lane):
    """The same v_cap gives the same launch count whatever the rows, kept edges and set size are."""
    from dgraph_b200 import algo

    rng = np.random.default_rng(3)
    v_cap = 6000
    counts = set()
    for nrows, set_size in ((1, 0), (3000, 0), (2, 200000), (6000, 50000)):
        f = np.sort(rng.choice(1 << 40, set_size, replace=False)).astype(np.uint64)
        s = algo.ReachSet.from_edges(f, np.arange(set_size, dtype=np.uint64))
        src = np.sort(rng.choice(1 << 40, nrows, replace=False)).astype(np.uint64)
        lens = np.diff(np.linspace(0, v_cap, nrows + 1).astype(np.int64))
        rows = [np.sort(rng.choice(1 << 30, int(k), replace=False)).astype(np.uint64) for k in lens]
        rc, src_rc, sizes, _, _, launches, guards = dev_step(lib, lane, s.handle, src, rows, None)
        assert rc == OK and src_rc == OK and guards and int(sizes[0]) == v_cap
        assert launches == rp.launches(nrows, v_cap)
        counts.add(launches)
        s.close()
    assert len(counts) == 1
    for m in (1, 2048, 2049, 4097, 1 << 17):
        s = algo.ReachSet()
        assert dev_step(lib, lane, s.handle, [7], [np.arange(1, m + 1)], None)[5] == rp.launches(1, m)
    assert dev_step(lib, lane, s.handle, [], [], None)[5] == 0


def test_concurrent_callers(lib):
    errors = []

    def worker(k):
        try:
            random_recursion(np.random.default_rng(700 + k), HostEngine(), n_max=200)
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=worker, args=(k,)) for k in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


def test_concurrent_device_callers(lib):
    """Four threads, each with its own lane and sets, stepping whole recursions through the device form."""
    errors = []

    def worker(k):
        ln, stream = new_lane(lib)
        try:
            import torch

            with torch.cuda.stream(stream):
                for j in range(5):
                    random_recursion(np.random.default_rng(900 + 10 * k + j), DevEngine(lib, ln), n_max=200)
        except Exception as e:  # noqa: BLE001
            errors.append(e)
        finally:
            lib.dgx_lane_destroy(ln)

    ts = [threading.Thread(target=worker, args=(k,)) for k in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


def test_device_chain_from_unfiltered_rows(lib, lane):
    """rows -> filter -> DestUIDs -> the next level's packs: each sg's rows come from dgx_dev_list_uids_unfiltered_rows
    over the UidPacks of its sources (v_cap the packs' total, the offsets only on the device) and go straight into
    dgx_dev_recurse_filter; only DestUIDs' length comes back to pick the next level's packs."""
    import torch

    from dgraph_b200 import algo, codec, pb
    from oracle import pyoracle as orc

    rng = np.random.default_rng(31)
    graph = gr.random_graph(rng, 300, ["a", "b"], mean_deg=3)
    handles, keep = {}, []
    for p, g in graph.items():
        for u in range(1, 301):
            r = g.row(u)
            if r.size == 0:
                continue
            op = orc.encode(r, 64)
            pk = pb.UidPack(op.block_size, op.base, op.num_uids, op.delta_off, op.deltas).normalized()
            view = codec.view_of(pk)
            keep.append((pk, view))
            h = C.c_void_p()
            assert lib.dgx_dev_pack_upload(lane, C.byref(view), C.byref(h)) == OK
            handles[(p, u)] = h
    sets = {p: algo.ReachSet() for p in graph}
    reach, ids = ro.Reach(), {}
    filters = {"b": np.arange(1, 301, 3, dtype=np.uint64)}

    def step(attr, src, rows, dest):
        want = reach.step(ids.setdefault(attr, len(ids) + 1), src, rows, dest)
        nrows = len(src)
        tab = (C.c_void_p * nrows)(*[handles[(attr, int(u))].value if (attr, int(u)) in handles else None
                                     for u in src])
        cap = int(sum(len(r) for r in rows)) + 5  # room past the rows: v_cap > v_off[nrows]
        d_src = torch.from_numpy(_b(src).view(np.int64)).cuda()
        d_rows, d_off = (torch.zeros(n, dtype=torch.int64, device="cuda") for n in (cap + 1, nrows + 1))
        mut_off = np.zeros(nrows + 1, np.uint64)
        assert lib.dgx_dev_list_uids_unfiltered_rows(lane, tab, nrows, None, None, mut_off.ctypes.data, 0, 0,
                                                     d_rows.data_ptr(), cap, d_off.data_ptr()) == OK
        d_dest = None if dest is None else torch.from_numpy(_b(dest).view(np.int64)).cuda()
        d_out, d_dout = (torch.full((cap,), -1, dtype=torch.int64, device="cuda") for _ in range(2))
        d_oo, d_sz = torch.zeros(nrows + 1, dtype=torch.int64, device="cuda"), torch.zeros(2, dtype=torch.int64,
                                                                                             device="cuda")
        assert lib.dgx_dev_recurse_filter(lane, sets[attr].handle, d_src.data_ptr(), nrows, d_rows.data_ptr(),
                                          d_off.data_ptr(), cap, None if d_dest is None else d_dest.data_ptr(),
                                          0 if dest is None else len(dest), d_out.data_ptr(), d_oo.data_ptr(), cap,
                                          d_dout.data_ptr(), cap, d_sz.data_ptr()) == OK
        assert lib.dgx_lane_sync(lane) == OK, lib.dgx_last_error()
        k, d = (int(x) for x in d_sz.cpu().numpy())
        oo = d_oo.cpu().numpy().view(np.uint64)
        out = d_out.cpu().numpy().view(np.uint64)
        assert k == want[2] and np.array_equal(d_dout[:d].cpu().numpy().view(np.uint64), want[1])
        assert all(np.array_equal(out[int(oo[i]):int(oo[i + 1])], want[0][i]) for i in range(nrows))
        return want

    steps, total, _ = gr.recurse(graph, [int(np.argmax(np.diff(graph["a"].ptr)))], ["a", "b"], 6, step,
                                 filters=filters)
    assert total > 50 and max(s.level for s in steps) >= 3
    for p, i in ids.items():
        f, t = reach.edges(i)
        assert export(sets[p]) == (f.tolist(), t.tolist())
    for h in handles.values():
        lib.dgx_dev_pack_free(h)


def test_c14a_sized_recursion(lib, lane):
    """C14a: { friend } over the 2e6-node Zipf graph, depth 6 from 100 roots, about 1.26e7 kept edges, on the device
    form with resident per-step inputs: every step's rows, DestUIDs and kept count, and the final set, against the
    vectorised formula."""
    import torch

    from dgraph_b200 import algo

    graph = gr.c14_graph(np.random.default_rng(14))
    roots = np.random.default_rng(2).integers(1, 2_000_001, 100)
    formula = gr.KeyFormula()
    steps, total, _ = gr.plan_levels({"friend": graph["friend"]}, roots, ["friend"], 6, formula=formula)
    assert total > 10_000_000
    s = algo.ReachSet()

    def up(x):
        return torch.from_numpy(_b(x).view(np.int64)).cuda()

    for attr, src, v, v_off, out, out_off, dest_uids, kept in steps:
        m = v.size
        d_src, d_v, d_off = up(src), up(v), up(v_off)
        d_out, d_dout = (torch.empty(max(m, 1), dtype=torch.int64, device="cuda") for _ in range(2))
        d_oo, d_sz = torch.empty(src.size + 1, dtype=torch.int64, device="cuda"), torch.empty(2, dtype=torch.int64,
                                                                                                device="cuda")
        assert lib.dgx_dev_recurse_filter(lane, s.handle, d_src.data_ptr(), src.size, d_v.data_ptr(), d_off.data_ptr(),
                                          m, None, 0, d_out.data_ptr(), d_oo.data_ptr(), m, d_dout.data_ptr(), m,
                                          d_sz.data_ptr()) == OK
        assert lib.dgx_lane_sync(lane) == OK
        k, d = (int(x) for x in d_sz.cpu().numpy())
        assert k == kept and d == dest_uids.size
        assert np.array_equal(d_oo.cpu().numpy().view(np.uint64), out_off)
        assert np.array_equal(d_out[:k].cpu().numpy().view(np.uint64), out)
        assert np.array_equal(d_dout[:d].cpu().numpy().view(np.uint64), dest_uids)
    assert s.size() == total
    ef, et = s.export()
    assert np.array_equal((ef << np.uint64(32)) | et, formula.sets["friend"])
    s.close()
