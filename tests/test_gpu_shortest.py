"""shortest() without weights on the device (dgx_path_expand, dgx_dev_path_expand and the dgx_path_search they share):
every level of random searches compared with the independent formula (gen_shortest.Formula), guard words past every
output, refusals, launches with the plan model (shortest_plan.py).  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen_shortest as gs  # noqa: E402
import shortest_plan as sp  # noqa: E402

pytestmark = pytest.mark.gpu

OK, ERR_ARG, ERR_CAP = 0, -3, -4
SENT = 0xDEADBEEFCAFEF00D
GUARD = 4


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


def _up(a, slack=0):
    import torch

    a = np.asarray(a)
    a = np.concatenate([a, np.zeros(slack + 1, a.dtype)])
    return torch.from_numpy(a.view(np.int32 if a.dtype == np.uint32 else np.int64)).cuda()


def _sent(n):
    import torch

    return torch.full((n,), SENT - (1 << 64), dtype=torch.int64, device="cuda")


def dev_level(lib, lane, handle, sgs, slack=0, mutate=None, next_cap=None):
    """One level through the device form with `slack` spare room in src, v and dest.  Returns (rc, rc of the sync,
    next per sg or None, stats or None, launches, guards intact)."""
    import torch
    from dgraph_b200 import _lib, algo

    arrs = list(algo.path_level_arrays(sgs))
    R, M, D = int(arrs[1][-1]), int(arrs[3][-1]), int(arrs[5][-1])  # the room, whatever mutate does to the offsets
    if mutate:
        mutate(arrs)
    attr, src_off, src, v_off, v, dest_off, dest = arrs
    t = [_up(attr), _up(src_off), _up(src[:R], slack), _up(v_off), _up(v[:M], slack), _up(dest_off),
         _up(dest[:D], slack)]
    lv = _lib.PathLevel(len(sgs), *[x.data_ptr() for x in t])
    cap = D + slack if next_cap is None else next_cap
    d_next, d_off, d_st = _sent(cap + GUARD), _sent(len(sgs) + 1 + GUARD), _sent(3 + GUARD)
    torch.cuda.synchronize()
    l0 = lib.dgx_lane_launches(lane)
    rc = lib.dgx_dev_path_expand(lane, handle, C.byref(lv), R + slack, M + slack, D + slack, d_next.data_ptr(),
                                 d_off.data_ptr(), cap, d_st.data_ptr())
    src_rc = lib.dgx_lane_sync(lane)
    launches = lib.dgx_lane_launches(lane) - l0
    nxt, off, st = (x.cpu().numpy().view(np.uint64) for x in (d_next, d_off, d_st))
    guards = np.all(nxt[cap:] == SENT) and np.all(off[len(sgs) + 1:] == SENT) and np.all(st[3:] == SENT)
    if rc != OK or src_rc != OK:  # a refused level writes nothing
        return rc, src_rc, None, None, launches, guards and np.all(nxt == SENT) and np.all(off == SENT) and np.all(
            st == SENT)
    n = int(off[len(sgs)])
    guards = guards and np.all(nxt[n:cap] == SENT)
    return rc, src_rc, [nxt[int(off[i]):int(off[i + 1])].copy() for i in range(len(sgs))], tuple(
        int(x) for x in st[:3]), launches, guards


class Checked:
    """Runs each level through the engine and the formula and asserts they agree."""

    def __init__(self, lib, lane, form, frm, to, slack=0):
        from dgraph_b200 import algo

        self.lib, self.lane, self.form, self.slack = lib, lane, form, slack
        self.ps = algo.PathSearch(frm, to)
        self.f = gs.Formula(frm, to)

    def expand(self, sgs):
        want = self.f.expand(sgs)
        if self.form == "host":
            got = self.ps.expand(sgs)
        else:
            rc, src_rc, nxt, st, launches, guards = dev_level(self.lib, self.lane, self.ps.handle, sgs, self.slack)
            assert rc == OK and src_rc == OK and guards, self.lib.dgx_last_error()
            R, M = sum(len(s[1]) for s in sgs), sum(len(r) for s in sgs for r in s[2])
            assert launches == sp.launches(R + self.slack, M + self.slack)
            got = (nxt, st)
        assert got[1] == want[1]
        assert all(np.array_equal(a, b) for a, b in zip(got[0], want[0]))
        return want

    def check_path(self):
        u, a = self.ps.path()
        wu, wa = self.f.path()
        assert np.array_equal(u, wu) and np.array_equal(a, wa)
        return u


@pytest.mark.parametrize("form", ["host", "device"])
def test_random_searches(lib, lane, form):
    rng = np.random.default_rng(160 if form == "host" else 161)
    reached = 0
    for i in range(120):
        g, frm, to, hops = gs.random_case(rng)
        c = Checked(lib, lane, form, frm, to, slack=i % 3)
        gs.search(g, frm, to, hops, c.expand)
        reached += c.check_path().size > 0
        c.ps.close()
    assert reached > 20


def test_fixed_example(lib, lane):
    from dgraph_b200 import algo

    # 1 -> 2 over both children (the later child's attr wins), 2 -> 3 over child 1 only
    g = gs.Graph(5, [gs.pred_from_edges(5, [1], [2]), gs.pred_from_edges(5, [1, 2], [2, 3])], [(0, None), (1, None)])
    with algo.PathSearch(1, 3) as ps:
        lv = gs.search(g, 1, 3, None, ps.expand)
        assert [st for _, _, st in lv] == [(2, 1, 0), (2, 1, 2)]
        u, a = ps.path()
        assert u.tolist() == [1, 2, 3] and a.tolist() == [1, 1]


@pytest.mark.parametrize("name", ["src", "row", "dest", "expanded", "offsets"])
def test_device_refusals_leave_the_search_unchanged(lib, lane, name):
    rng = np.random.default_rng(7)
    g = gs.Graph(201, gs.random_graph(rng, 200, 2, 3.0), [(0, None), (1, None)])
    c = Checked(lib, lane, "device", 1, 150)
    levels = []

    def expand(sgs):
        if len(levels) == 1:  # refuse a broken copy of level 2 first, then run the real one
            def dup(off_i, val_i):
                def f(a):
                    off = a[off_i]
                    k = next(int(off[i]) for i in range(len(off) - 1) if off[i + 1] - off[i] >= 2)
                    a[val_i][k + 1] = a[val_i][k]
                return f

            bad_sgs, mut = sgs, None
            if name == "src":
                mut = dup(1, 2)
            elif name == "row":
                mut = dup(3, 4)
            elif name == "dest":
                mut = dup(5, 6)
            elif name == "offsets":
                def mut(a):
                    a[3][1] = 10 ** 6
            else:  # From had a kept edge at level 1, so it is expanded
                bad_sgs = [(0, np.asarray([1], np.uint64), [np.asarray([5], np.uint64)], np.asarray([5], np.uint64))]
            rc, src_rc, nxt, st, _, guards = dev_level(lib, lane, c.ps.handle, bad_sgs, mutate=mut)
            assert rc == OK and src_rc == ERR_ARG and guards
        levels.append(1)
        return c.expand(sgs)

    gs.search(g, 1, 150, 4, expand)
    c.check_path()
    c.ps.close()


def test_argument_and_capacity_errors(lib, lane):
    from dgraph_b200 import _lib, algo

    sgs = [(0, [1], [[3, 4]], [3, 4]), (1, [1], [[4, 5]], [4, 5])]
    with algo.PathSearch(1, 4) as ps:
        rc, _, _, _, _, guards = dev_level(lib, lane, ps.handle, sgs, next_cap=2)
        assert rc == ERR_CAP and guards
        arrs = algo.path_level_arrays(sgs)
        lv = _lib.PathLevel(0, *[a.ctypes.data for a in arrs])
        nxt = np.zeros(4, np.uint64)
        assert lib.dgx_path_expand(ps.handle, C.byref(lv), nxt.ctypes.data, nxt.ctypes.data, 4,
                                   C.byref(_lib.PathStats())) == ERR_ARG
        lv = _lib.PathLevel(2, *[a.ctypes.data for a in arrs])
        assert lib.dgx_path_expand(ps.handle, C.byref(lv), nxt.ctypes.data, nxt.ctypes.data, 2,
                                   C.byref(_lib.PathStats())) == ERR_CAP
        # the host form refuses a non-ascending src on the device, and the search is unchanged
        with pytest.raises(_lib.DgxError):
            ps.expand([(0, [2, 1], [[3], [4]], [3, 4])])
        with pytest.raises(_lib.DgxError):  # 2 was never discovered
            ps.expand([(0, [1, 2], [[3], [4]], [3, 4])])
        assert ps.expand(sgs)[1] == (4, 3, 1)
        u, a = ps.path()
        assert u.tolist() == [1, 4] and a.tolist() == [1]  # (1, 4) is in both sgs: the later one's attr
        n = C.c_size_t(0)
        out = np.full(4, 7, np.uint64)
        assert lib.dgx_path_result(ps.handle, out.ctypes.data, out.ctypes.data, 1, C.byref(n)) == ERR_CAP
        assert n.value == 2 and (out == 7).all()


def test_search_bound_to_one_lane(lib, lane):
    from dgraph_b200 import _lib, algo

    other, _ = new_lane(lib)
    sgs = [(0, [1], [[2, 3]], [2, 3])]
    with algo.PathSearch(1, 9) as ps:
        arrs = algo.path_level_arrays(sgs)
        t = [_up(a) for a in arrs]
        lv = _lib.PathLevel(1, *[x.data_ptr() for x in t])
        d_next, d_off, d_st = _sent(8), _sent(8), _sent(8)
        args = (C.byref(lv), 1, 2, 2, d_next.data_ptr(), d_off.data_ptr(), 2, d_st.data_ptr())
        assert lib.dgx_dev_path_expand(lane, ps.handle, *args) == OK
        assert lib.dgx_dev_path_expand(other, ps.handle, *args) == ERR_ARG  # queued on `lane`, not waited for
        assert lib.dgx_lane_sync(lane) == OK
        assert ps.path()[0].size == 0  # waits: the search is free again
        assert lib.dgx_dev_path_expand(other, ps.handle, *args) == OK
        assert lib.dgx_lane_sync(other) == ERR_ARG  # 1 already expanded
        assert ps.path()[0].size == 0
    lib.dgx_lane_destroy(other)


def test_growth_across_doublings(lib, lane):
    """A chain of 5 000 nodes in levels of 1 row: the seen and expanded sets grow past 1 024 while device-form levels
    stay queued, then the path is walked."""
    n = 5000
    g = gs.Graph(n + 1, [gs.chain(n)], [(0, None)])
    c = Checked(lib, lane, "device", 1, n)
    lv = gs.search(g, 1, n, None, c.expand)
    assert len(lv) == n - 1
    assert c.check_path().tolist() == list(range(1, n + 1))
    c.ps.close()


def test_launches_do_not_grow_with_sgs_rows_or_sets(lib, lane):
    from dgraph_b200 import algo

    def levels(width):
        """Level 1: From -> width nodes; level 2: those nodes as sources, 10 sgs, 4 values a row."""
        rng = np.random.default_rng(width)
        first = np.arange(100, 100 + width, dtype=np.uint64)
        l1 = [(0, [1], [first], first)]
        l2 = []
        for s in range(10):
            src = first[s::10]
            rows = [np.sort(rng.choice(np.arange(1000, 1000 + 10 * width, dtype=np.uint64), 4, replace=False))
                    for _ in src]
            l2.append((s % 3, src, rows, np.unique(np.concatenate(rows)) if rows else np.zeros(0, np.uint64)))
        return [l1, [sg for sg in l2 if len(sg[1])]]

    counts = []
    for width in (10, 100):  # sgs, rows, values and the sets grow tenfold
        with algo.PathSearch(1, 99999) as ps:
            for sgs in levels(width):
                R, M = sum(len(s[1]) for s in sgs), sum(len(r) for s in sgs for r in s[2])
                rc, src_rc, _, _, launches, _ = dev_level(lib, lane, ps.handle, sgs, slack=4096 - M)
                assert rc == OK and src_rc == OK, lib.dgx_last_error()
                counts.append((launches, sp.launches(R + 4096 - M, 4096)))
    assert all(a == b for a, b in counts) and len({a for a, _ in counts}) == 1


def test_concurrent_callers(lib):
    rng = np.random.default_rng(99)
    cases = [gs.random_case(rng) for _ in range(24)]
    errors = []

    def work(part):
        try:
            ln, _ = new_lane(lib) if part % 2 else (None, None)
            for g, frm, to, hops in cases[part::4]:
                c = Checked(lib, ln, "device" if ln else "host", frm, to)
                gs.search(g, frm, to, hops, c.expand)
                c.check_path()
                c.ps.close()
            if ln:
                lib.dgx_lane_destroy(ln)
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    th = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors


def test_device_chain_from_unfiltered_rows(lib, lane):
    """Each level's rows come from dgx_dev_list_uids_unfiltered_rows over the UidPacks of its sources and its dest from
    dgx_dev_merge_sorted_matrix over those rows; both go straight into dgx_dev_path_expand (one child, one sg a level)."""
    import torch

    from dgraph_b200 import _lib, algo, codec, pb
    from oracle import pyoracle as orc

    rng = np.random.default_rng(41)
    n = 400
    g = gs.Graph(n + 1, gs.random_graph(rng, n, 1, 2.0), [(0, None)])
    handles, keep = {}, []
    for u in range(1, n + 1):
        r = g.row(0, u)
        if r.size == 0:
            continue
        op = orc.encode(r, 64)
        pk = pb.UidPack(op.block_size, op.base, op.num_uids, op.delta_off, op.deltas).normalized()
        view = codec.view_of(pk)
        keep.append((pk, view))
        h = C.c_void_p()
        assert lib.dgx_dev_pack_upload(lane, C.byref(view), C.byref(h)) == OK
        handles[u] = h
    frm = int(np.argmax(np.diff(g.preds[0][0].astype(np.int64))))
    f = gs.Formula(frm, n + 7)
    ps = algo.PathSearch(frm, n + 7)
    src = np.asarray([frm], np.uint64)
    levels = 0
    while src.size and levels < 8:
        rows, dest = gs.process(g, 0, src)
        want = f.expand([(0, src, rows, dest)])
        nr = src.size
        tab = (C.c_void_p * nr)(*[handles[int(u)].value if int(u) in handles else None for u in src])
        cap = int(sum(len(r) for r in rows)) + 5
        d_rows, d_off = (torch.zeros(k, dtype=torch.int64, device="cuda") for k in (cap + 1, nr + 1))
        mut_off = np.zeros(nr + 1, np.uint64)
        assert lib.dgx_dev_list_uids_unfiltered_rows(lane, tab, nr, None, None, mut_off.ctypes.data, 0, 0,
                                                     d_rows.data_ptr(), cap, d_off.data_ptr()) == OK
        d_dest, d_dlen = torch.zeros(cap + 1, dtype=torch.int64, device="cuda"), torch.zeros(
            1, dtype=torch.int64, device="cuda")
        assert lib.dgx_dev_merge_sorted_matrix(lane, d_rows.data_ptr(), d_off.data_ptr(), nr, cap, d_dest.data_ptr(),
                                               cap, d_dlen.data_ptr()) == OK
        assert lib.dgx_lane_sync(lane) == OK
        d_doff = torch.cat([torch.zeros(1, dtype=torch.int64, device="cuda"), d_dlen])
        d_attr = torch.zeros(1, dtype=torch.int32, device="cuda")
        d_soff = torch.tensor([0, nr], dtype=torch.int64, device="cuda")
        d_src = _up(src)
        torch.cuda.synchronize()
        lv = _lib.PathLevel(1, d_attr.data_ptr(), d_soff.data_ptr(), d_src.data_ptr(), d_off.data_ptr(),
                            d_rows.data_ptr(), d_doff.data_ptr(), d_dest.data_ptr())
        d_next, d_noff, d_st = _sent(cap), _sent(2), _sent(3)
        assert lib.dgx_dev_path_expand(lane, ps.handle, C.byref(lv), nr, cap, cap, d_next.data_ptr(),
                                       d_noff.data_ptr(), cap, d_st.data_ptr()) == OK
        assert lib.dgx_lane_sync(lane) == OK, lib.dgx_last_error()
        st = tuple(int(x) for x in d_st.cpu().numpy())
        k = int(d_noff.cpu().numpy()[1])
        nxt = d_next.cpu().numpy().view(np.uint64)[:k]
        assert st == want[1] and np.array_equal(nxt, want[0][0])
        src = nxt
        levels += 1
        if st[1] == 0:
            break
    assert levels >= 3 and len(f.seen) > 50
    ps.close()
    for h in handles.values():
        lib.dgx_dev_pack_free(h)


def test_c16a_sized_search(lib, lane):
    """C16a's shape: a 2e6-node Zipf friend graph, 6 levels from one root, through both forms at once; each level's
    discovered count and next frontier equal between the forms and with a numpy BFS of the same graph."""
    import torch
    from dgraph_b200 import _lib, algo

    rng = np.random.default_rng(16)
    n = 2_000_000
    m = 10 * n
    fr = (np.minimum(rng.zipf(1.3, m), n).astype(np.uint64) * 2654435761 % n + 1).astype(np.uint64)
    to = rng.integers(1, n + 1, m).astype(np.uint64)
    off, adj = gs.pred_from_edges(n + 1, fr, to)
    frm = int(np.argmax(np.diff(off.astype(np.int64))))
    ps_h, ps_d = algo.PathSearch(frm, n + 5), algo.PathSearch(frm, n + 5)
    seen = np.zeros(n + 2, bool)
    seen[frm] = True
    src = np.asarray([frm], np.uint64)
    for level in range(6):
        lo, hi = off[src.astype(np.int64)].astype(np.int64), off[src.astype(np.int64) + 1].astype(np.int64)
        lens = hi - lo
        idx = np.repeat(lo - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens) + np.arange(lens.sum())
        v = adj[idx]
        v_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
        dest = np.unique(v)
        arrs = (np.zeros(1, np.uint32), np.asarray([0, src.size], np.uint64), src, v_off, v,
                np.asarray([0, dest.size], np.uint64), dest)
        new = dest[~seen[dest.astype(np.int64)]]
        lv = _lib.PathLevel(1, *[a.ctypes.data for a in arrs])
        nxt, noff, st = np.empty(dest.size + 1, np.uint64), np.zeros(2, np.uint64), _lib.PathStats()
        _lib.check(lib.dgx_path_expand(ps_h.handle, C.byref(lv), nxt.ctypes.data, noff.ctypes.data, dest.size,
                                       C.byref(st)))
        t = [torch.from_numpy(np.ascontiguousarray(a).view(np.int32 if a.dtype == np.uint32 else np.int64)).cuda()
             for a in arrs]
        dl = _lib.PathLevel(1, *[x.data_ptr() for x in t])
        d_next, d_noff, d_st = _sent(dest.size + 1), _sent(2), _sent(3)
        assert lib.dgx_dev_path_expand(lane, ps_d.handle, C.byref(dl), src.size, v.size, dest.size, d_next.data_ptr(),
                                       d_noff.data_ptr(), dest.size, d_st.data_ptr()) == OK
        assert lib.dgx_lane_sync(lane) == OK
        dst = tuple(int(x) for x in d_st.cpu().numpy())
        assert (st.edges, st.discovered) == (v.size, new.size) and dst == (st.edges, st.discovered, st.to_level)
        k = int(noff[1])
        assert np.array_equal(d_next.cpu().numpy().view(np.uint64)[:k], nxt[:k])
        seen[new.astype(np.int64)] = True
        src = nxt[:k].copy()
        if src.size == 0:
            break
    assert seen.sum() > 100_000
    ps_h.close()
    ps_d.close()
