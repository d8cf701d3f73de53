"""@cascade on the device (dgx_cascade and dgx_dev_cascade): random forests against the line-by-line restatement
(cascade_oracle.c) with guard words past every output, every argument and capacity error, the device-detected
refusals at dgx_lane_sync, launches against the plan model (cascade_plan.py), a device form fed by the unfiltered rows
and the matrix merge, concurrent callers and a C15a-sized call.  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import cascade_oracle as co  # noqa: E402
import cascade_plan as cp  # noqa: E402
import gen_cascade as gc  # noqa: E402

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
    ln, _ = new_lane(lib)
    yield ln
    lib.dgx_lane_destroy(ln)


def same(a, b):
    (ra, da), (rb, db) = a, b
    return (len(ra) == len(rb) and all(np.array_equal(x, y) for x, y in zip(da, db)) and
            all(len(x) == len(y) and all(np.array_equal(u, v) for u, v in zip(x, y)) for x, y in zip(ra, rb)))


def _t(a, dtype=np.uint64):
    import torch

    a = np.ascontiguousarray(np.asarray(a, dtype))
    if a.size == 0:
        a = np.zeros(1, dtype)
    return torch.from_numpy(a.view(np.int64) if dtype == np.uint64 else a).cuda()


def sent(n):
    import torch

    return torch.full((n,), SENT - (1 << 64), dtype=torch.int64, device="cuda")


def dev_call(lib, lane, nodes, slack=(), v_off=None, out_cap=None, dest_cap=None):
    """dgx_dev_cascade over per-node device arrays; node k gets slack[k] garbage values of room past its rows and
    v_off[k] (if given) replaces its offsets.  Returns (rc, rc of the sync, sizes, (rows, dests) or None, launches,
    guards intact)."""
    from dgraph_b200 import _lib
    from dgraph_b200.algo import cascade_arrays, cascade_tree

    import torch

    keep, descs = [], []
    for k, nd in enumerate(nodes):
        sl = slack[k] if k < len(slack) else 0
        lens = [r.size for r in nd.rows]
        off = np.zeros(len(lens) + 1, np.uint64)
        np.cumsum(lens, out=off[1:])
        if v_off is not None and k in v_off:
            off = np.asarray(v_off[k], np.uint64)
        vals = np.concatenate(list(nd.rows) + [np.full(sl, 7, np.uint64)]) if nd.rows or sl else np.zeros(0)
        v_cap, nrows = int(sum(lens)) + sl, len(nd.rows)
        d_v, d_off = _t(vals), _t(off)
        d_dest, d_hv = _t(nd.dest), _t(nd.has_val, np.uint8)
        keep += [d_v, d_off, d_dest, d_hv]
        descs.append(_lib.CascadeNode(d_v.data_ptr(), d_off.data_ptr(), nrows, v_cap, d_dest.data_ptr(), nd.dest.size,
                                      d_hv.data_ptr(), nd.has_val.size))
    a = cascade_arrays(nodes)
    tab = (_lib.CascadeNode * max(len(descs), 1))(*descs)
    nv = sum(d.v_cap for d in descs)
    nd_ = sum(d.ndest for d in descs)
    rows = int(a["row_off"][-1])
    out_cap = nv if out_cap is None else out_cap
    dest_cap = nd_ if dest_cap is None else dest_cap
    d_out, d_oo, d_dout, d_do, d_sz = (sent(out_cap + GUARD), sent(rows + 1 + GUARD), sent(dest_cap + GUARD),
                                       sent(len(nodes) + 1 + GUARD), sent(2 + GUARD))
    torch.cuda.synchronize()
    tree = cascade_tree(a)
    l0 = lib.dgx_lane_launches(lane)
    rc = lib.dgx_dev_cascade(lane, C.byref(tree), tab, d_out.data_ptr(), d_oo.data_ptr(), out_cap, d_dout.data_ptr(),
                             d_do.data_ptr(), dest_cap, d_sz.data_ptr())
    src = lib.dgx_lane_sync(lane)
    launches = lib.dgx_lane_launches(lane) - l0
    out, oo, dout, do, sz = (t.cpu().numpy().view(np.uint64) for t in (d_out, d_oo, d_dout, d_do, d_sz))
    guards = (np.all(out[out_cap:] == SENT) and np.all(oo[rows + 1:] == SENT) and np.all(dout[dest_cap:] == SENT) and
              np.all(do[len(nodes) + 1:] == SENT) and np.all(sz[2:] == SENT))
    if rc != OK or src != OK:  # a refused call writes d_sizes = {0, 0} at most
        guards = guards and np.all(out == SENT) and np.all(oo == SENT) and np.all(dout == SENT) and np.all(do == SENT)
        return rc, src, sz[:2], None, launches, guards
    K, D = int(sz[0]), int(sz[1])
    assert int(oo[rows]) == K and int(do[len(nodes)]) == D
    guards = guards and np.all(out[K:out_cap] == SENT) and np.all(dout[D:dest_cap] == SENT)
    from dgraph_b200.algo import cascade_split

    return rc, src, sz[:2], cascade_split(a, out, oo, dout, do), launches, guards


@pytest.mark.parametrize("form", ["host", "device"])
def test_random_forests(lib, lane, form):
    from dgraph_b200 import algo

    rng = np.random.default_rng(1501 if form == "host" else 1502)
    for _ in range(300):
        f = gc.random_forest(rng)
        want = co.cascade(f)
        if form == "host":
            rows, dests = algo.Cascade(f)
            assert same((rows, [d.Uids for d in dests]), want)
        else:
            slack = [int(x) for x in rng.integers(0, 3, len(f))]
            rc, src, _, got, launches, guards = dev_call(lib, lane, f, slack)
            assert rc == OK and src == OK, lib.dgx_last_error()
            assert guards and same(got, want)
            caps = [sum(r.size for r in nd.rows) + s for nd, s in zip(f, slack)]
            assert launches == cp.launches(gc.levels_with_work(f, caps))


def small():
    from dgraph_b200.algo import CC_CASCADE, CC_CHECKED, CC_ORDERED, CascadeNode

    d = np.array([1, 2, 3], np.uint64)
    return [CascadeNode(-1, CC_CASCADE, 1, 1, 0, d, [d]),
            CascadeNode(0, CC_CASCADE | CC_CHECKED, 0, 0, 0, np.array([5, 6], np.uint64), [[5], [], [6]], [0, 1]),
            CascadeNode(1, CC_CHECKED | CC_ORDERED, 0, 0, 0, np.array([8, 9], np.uint64), [[9, 8], []])]


def test_device_detected_refusals(lib, lane):
    from dgraph_b200 import algo
    from dgraph_b200.algo import CascadeNode

    base = small()
    assert dev_call(lib, lane, base)[0:2] == (OK, OK)
    bad_dest = list(base)
    bad_dest[1] = CascadeNode(0, base[1].flags, 0, 0, 0, np.array([6, 5], np.uint64), base[1].rows, base[1].has_val)
    bad_row = list(base)
    bad_row[1] = CascadeNode(0, base[1].flags, 0, 0, 0, base[1].dest, [[5], [], [6, 6]], base[1].has_val)
    dup_dest = list(base)
    dup_dest[0] = CascadeNode(-1, base[0].flags, 1, 1, 0, np.array([1, 1, 3], np.uint64), base[0].rows)
    for f in (bad_dest, bad_row, dup_dest):
        rc, src, sz, got, launches, guards = dev_call(lib, lane, f)
        assert rc == OK and src == ERR_ARG and guards and sz.tolist() == [0, 0]
        with pytest.raises(Exception) as e:
            algo.Cascade(f)
        assert "DGX_ERR_ARG" in str(e.value)
    # offsets only the device sees: v_off[0] != 0, decreasing, past v_cap
    for off in ([1, 1, 1, 2], [0, 1, 0, 2], [0, 1, 1, 9]):
        rc, src, sz, _, _, guards = dev_call(lib, lane, base, v_off={1: off})
        assert rc == OK and src == ERR_ARG and guards and sz.tolist() == [0, 0], off
    # the lane works again after a refusal
    assert dev_call(lib, lane, base)[0:2] == (OK, OK)


def test_argument_and_capacity_errors(lib, lane):
    from dgraph_b200 import _lib
    from dgraph_b200.algo import CascadeNode

    base = small()
    nv, nd = sum(sum(r.size for r in n.rows) for n in base), sum(n.dest.size for n in base)
    for kw, code in (({"out_cap": nv - 1}, ERR_CAP), ({"dest_cap": nd - 1}, ERR_CAP)):
        rc, src, sz, _, launches, guards = dev_call(lib, lane, base, **kw)
        assert rc == code and src == OK and guards and launches == 0 and np.all(sz == SENT)
    bad = list(base)
    bad[2] = CascadeNode(5, 0)
    rc, src, sz, _, launches, guards = dev_call(lib, lane, bad)
    assert rc == ERR_ARG and launches == 0 and guards and np.all(sz == SENT)
    tree = _lib.CascadeTree(0, None, None, None, None, None)
    assert lib.dgx_dev_cascade(lane, C.byref(tree), None, None, None, 0, None, None, 0, None) == ERR_ARG
    nodes = (_lib.CascadeNode * 1)(_lib.CascadeNode(None, None, 0, 0, None, 0, None, 0))
    par, z8, z32, z64 = (np.array([0xFFFFFFFF], np.uint32), np.zeros(1, np.uint8), np.zeros(1, np.int32),
                         np.zeros(1, np.uint64))
    t1 = _lib.CascadeTree(1, par.ctypes.data, z8.ctypes.data, z32.ctypes.data, z32.ctypes.data, z64.ctypes.data)
    d = sent(8)
    assert lib.dgx_dev_cascade(lane, C.byref(t1), nodes, d.data_ptr(), d.data_ptr(), 0, d.data_ptr(), d.data_ptr(), 0,
                               d.data_ptr()) == ERR_ARG  # a node without v_off
    # no dest value and no value: zero offsets and sizes, no launch
    empty = [CascadeNode(-1, 1, 2, 1, 0, [], [[]]), CascadeNode(0, 3, 0, 0, 0, [], [], [1])]
    rc, src, sz, got, launches, guards = dev_call(lib, lane, empty)
    assert (rc, src, launches) == (OK, OK, 0) and guards and sz.tolist() == [0, 0]
    assert [r.size for r in got[0][0]] == [0] and got[0][1] == []


def test_launches_follow_the_plan(lib, lane):
    """A chain of d levels with work: launches are 4 + 7 d whatever the rows, values and dest sizes (tenfold growth at a
    fixed depth leaves them unchanged)."""
    from dgraph_b200.algo import CC_CASCADE, CC_CHECKED, CascadeNode

    rng = np.random.default_rng(5)
    for depth in (1, 2, 4, 8):
        counts = set()
        for scale in (1, 10):
            nodes, dest = [], np.arange(1, 20 * scale + 1, dtype=np.uint64)
            nodes.append(CascadeNode(-1, CC_CASCADE, 3, 1, 0, dest, [dest]))
            for k in range(1, depth):
                rows = [np.unique(rng.integers(1, 40 * scale, int(rng.integers(0, 6)) * scale)).astype(np.uint64)
                        for _ in range(nodes[-1].dest.size)]
                d = np.unique(np.concatenate(rows)) if sum(r.size for r in rows) else np.zeros(0, np.uint64)
                nodes.append(CascadeNode(k - 1, CC_CASCADE | CC_CHECKED, 2, 1, 0, d, rows))
            rc, src, _, got, launches, guards = dev_call(lib, lane, nodes)
            assert rc == OK and src == OK and guards and same(got, co.cascade(nodes))
            assert launches == cp.launches(gc.levels_with_work(nodes))
            counts.add(launches)
        assert counts == {cp.launches(depth)}


def test_device_chain_from_unfiltered_rows(lib, lane):
    """The rows of a three-level tree come from dgx_dev_list_uids_unfiltered_rows over UidPacks (v_cap the packs' total,
    the offsets only on the device), each dest from dgx_dev_merge_sorted_matrix over those rows, and both go into
    dgx_dev_cascade where they are; the host reads a level's DestUIDs only to pick the next level's packs."""
    import torch

    from dgraph_b200 import _lib, codec, pb
    from dgraph_b200.algo import CC_CASCADE, CC_CHECKED, CascadeNode, cascade_arrays, cascade_split, cascade_tree
    from oracle import pyoracle as orc

    rng = np.random.default_rng(41)
    adj = {u: np.unique(rng.integers(1, 400, int(rng.integers(0, 12)))).astype(np.uint64) for u in range(1, 401)}
    handles, keep = {}, []
    for u, r in adj.items():
        if r.size == 0:
            continue
        op = orc.encode(r, 64)
        pk = pb.UidPack(op.block_size, op.base, op.num_uids, op.delta_off, op.deltas).normalized()
        view = codec.view_of(pk)
        keep.append((pk, view))
        h = C.c_void_p()
        assert lib.dgx_dev_pack_upload(lane, C.byref(view), C.byref(h)) == OK
        handles[u] = h

    def level(src):
        """(d_rows, d_off, cap, d_dest, dest length) of the rows of src, all on the device."""
        n = len(src)
        tab = (C.c_void_p * n)(*[handles[int(u)].value if int(u) in handles else None for u in src])
        cap = int(sum(adj[int(u)].size for u in src)) + 3
        d_rows, d_off = (torch.zeros(x, dtype=torch.int64, device="cuda") for x in (cap + 1, n + 1))
        mut_off = np.zeros(n + 1, np.uint64)
        assert lib.dgx_dev_list_uids_unfiltered_rows(lane, tab, n, None, None, mut_off.ctypes.data, 0, 0,
                                                     d_rows.data_ptr(), cap, d_off.data_ptr()) == OK
        d_dest, d_len = torch.zeros(cap, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64,
                                                                                        device="cuda")
        assert lib.dgx_dev_merge_sorted_matrix(lane, d_rows.data_ptr(), d_off.data_ptr(), n, cap, d_dest.data_ptr(),
                                               cap, d_len.data_ptr()) == OK
        return d_rows, d_off, cap, d_dest, d_len

    roots = np.arange(1, 300, 7, dtype=np.uint64)
    r1 = level(roots)
    assert lib.dgx_lane_sync(lane) == OK
    dest1 = r1[3][:int(r1[4].item())].cpu().numpy().view(np.uint64).copy()  # sizes the next level only
    r2 = level(dest1)
    assert lib.dgx_lane_sync(lane) == OK
    n2 = int(r2[4].item())
    nodes = [CascadeNode(-1, CC_CASCADE, 0, 0, 0, roots, [roots]),
             CascadeNode(0, CC_CASCADE | CC_CHECKED, 0, 0, 0, dest1, [adj[int(u)] for u in roots]),
             CascadeNode(1, CC_CASCADE | CC_CHECKED, 2, 1, 0, r2[3][:n2].cpu().numpy().view(np.uint64).copy(),
                         [adj[int(u)] for u in dest1], (rng.random(n2) < 0.3).astype(np.uint8))]
    d_root = _t(roots)
    d_root_off = _t([0, roots.size])
    hv = _t(nodes[2].has_val, np.uint8)
    descs = [_lib.CascadeNode(d_root.data_ptr(), d_root_off.data_ptr(), 1, roots.size, d_root.data_ptr(), roots.size,
                              None, 0),
             _lib.CascadeNode(r1[0].data_ptr(), r1[1].data_ptr(), roots.size, r1[2], r1[3].data_ptr(), dest1.size,
                              None, 0),
             _lib.CascadeNode(r2[0].data_ptr(), r2[1].data_ptr(), dest1.size, r2[2], r2[3].data_ptr(), n2,
                              hv.data_ptr(), n2)]
    a = cascade_arrays(nodes)
    nv, nd = 1 * roots.size + r1[2] + r2[2], roots.size + dest1.size + n2
    rows = 1 + roots.size + dest1.size
    d_out, d_oo, d_dout, d_do, d_sz = sent(nv), sent(rows + 1), sent(nd), sent(4), sent(2)
    tree = cascade_tree(a)
    assert lib.dgx_dev_cascade(lane, C.byref(tree), (_lib.CascadeNode * 3)(*descs), d_out.data_ptr(), d_oo.data_ptr(),
                               nv, d_dout.data_ptr(), d_do.data_ptr(), nd, d_sz.data_ptr()) == OK
    assert lib.dgx_lane_sync(lane) == OK, lib.dgx_last_error()
    out, oo, dout, do = (t.cpu().numpy().view(np.uint64) for t in (d_out, d_oo, d_dout, d_do))
    got = cascade_split(a, out, oo, dout, do)
    want = co.cascade(nodes)
    assert same(got, want) and sum(x.size for x in want[1]) > 0
    for h in handles.values():
        lib.dgx_dev_pack_free(h)


def test_concurrent_callers(lib):
    from dgraph_b200 import algo

    errs = []

    def host(k):
        try:
            rng = np.random.default_rng(900 + k)
            for _ in range(40):
                f = gc.random_forest(rng)
                rows, dests = algo.Cascade(f)
                assert same((rows, [d.Uids for d in dests]), co.cascade(f))
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    def dev(k):
        try:
            ln, _ = new_lane(lib)
            rng = np.random.default_rng(950 + k)
            for _ in range(40):
                f = gc.random_forest(rng)
                rc, src, _, got, _, guards = dev_call(lib, ln, f)
                assert rc == OK and src == OK and guards and same(got, co.cascade(f))
            lib.dgx_lane_destroy(ln)
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=host, args=(k,)) for k in range(3)] + [
        threading.Thread(target=dev, args=(k,)) for k in range(3)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


def test_c15a_sized_call(lib):
    """C15a: 1e6 Person roots, friend rows Zipf over 2e6 uids, through the host form, against the restatement."""
    from dgraph_b200.algo import cascade_tree

    a = gc.c15a_arrays(np.random.default_rng(15))
    want = co.cascade_flat(a)
    m, nd = int(a["v_off"][-1]), int(a["dest_off"][-1])
    out, dout = np.full(m + GUARD, SENT, np.uint64), np.full(nd + GUARD, SENT, np.uint64)
    oo, do = np.zeros(int(a["row_off"][-1]) + 1, np.uint64), np.zeros(9, np.uint64)
    p = lambda k: a[k].ctypes.data  # noqa: E731
    rc = lib.dgx_cascade(C.byref(cascade_tree(a)), p("v"), p("v_off"), p("row_off"), p("dest"), p("dest_off"),
                         p("has_val"), p("hv_off"), out.ctypes.data, oo.ctypes.data, m, dout.ctypes.data,
                         do.ctypes.data, nd)
    assert rc == OK, lib.dgx_last_error()
    K, D = int(oo[-1]), int(do[-1])
    assert np.array_equal(oo, want[1]) and np.array_equal(do, want[3])
    assert np.array_equal(out[:K], want[0][:K]) and np.array_equal(dout[:D], want[2][:D])
    assert np.all(out[K:] == SENT) and np.all(dout[D:] == SENT)
    assert m > 1.5e7 and D < nd


@pytest.mark.parametrize("form", ["host", "device"])
def test_reference_queries(lib, lane, form):
    """The reference's cascade tests over the fixture (tests/golden/cascade_person.json) at the uid level."""
    import json

    from dgraph_b200 import algo
    from test_cascade_host import GOLDEN, golden_forest, render

    with open(GOLDEN) as f:
        d = json.load(f)
    for name, case in d["cases"].items():
        nodes, specs = golden_forest(d, case)
        if form == "host":
            rows, dests = algo.Cascade(nodes)
            got = (rows, [x.Uids for x in dests])
        else:
            rc, src, _, got, _, guards = dev_call(lib, lane, nodes)
            assert rc == OK and src == OK and guards
        assert render(nodes, specs, *got) == case["want"], name
