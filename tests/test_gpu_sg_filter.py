"""@filter and first / offset on the device (dgx_sg_filter and dgx_dev_sg_filter): random trees against the
line-by-line restatement (sg_filter_oracle.c) with guard words past every output, counts-only mode, every
device-detected refusal at dgx_lane_sync, launches against the plan model (sg_filter_plan.py), a device chain from
unfiltered rows through the matrix merge and the count rows, concurrent callers and a C19a-sized call.  Runs on an H100
only (`pytest -m gpu`)."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen_sg_filter as gs  # noqa: E402
import sg_filter_golden as sgg  # noqa: E402
import sg_filter_oracle as so  # noqa: E402
import sg_filter_plan as sp  # noqa: E402

pytestmark = pytest.mark.gpu

OK, ERR_ARG, ERR_CAP = 0, -3, -4
SENT = 0xDEADBEEFCAFEF00D
CSENT = 0xA5A5A5A5
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


def _t(a, dtype=np.uint64):
    import torch

    a = np.ascontiguousarray(np.asarray(a, dtype))
    if a.size == 0:
        a = np.zeros(1, dtype)
    if dtype == np.uint64:
        return torch.from_numpy(a.view(np.int64)).cuda()
    return torch.from_numpy(a.view(np.int32)).cuda()


def sent(n, counts=False):
    import torch

    if counts:
        return torch.full((n,), CSENT - (1 << 32), dtype=torch.int32, device="cuda")
    return torch.full((n,), SENT - (1 << 64), dtype=torch.int64, device="cuda")


def same(got, want, counts_only=False):
    (gr, gc, gd), (wr, wc, wd) = got, want
    rows_ok = counts_only or (len(gr) == len(wr) and all(np.array_equal(x, y) for x, y in zip(gr, wr)))
    return rows_ok and np.array_equal(gc, wc) and np.array_equal(gd, wd)


def csr(rows):
    off = np.zeros(len(rows) + 1, np.uint64)
    np.cumsum([len(r) for r in rows], out=off[1:])
    v = np.concatenate([np.asarray(r, np.uint64) for r in rows]) if int(off[-1]) else np.zeros(0, np.uint64)
    return v, off


def host_call(lib, case, counts_only=False, dest_cap=None, out_cap=None):
    """dgx_sg_filter with guard words past every output.  Returns (rc, (rows, counts, dest) or None, guards intact)."""
    from dgraph_b200.algo import sg_filter_flat, sg_filter_leaf_arrays, sg_filter_tree

    tree, leaves, d0, rows, count, offset = case
    f = sg_filter_flat(tree)
    d0 = np.ascontiguousarray(np.asarray(d0, np.uint64))
    keep, tab = sg_filter_leaf_arrays(leaves, d0.size)
    v, v_off = csr(rows)
    v = v if v.size else np.zeros(1, np.uint64)
    nrows, m, n0 = len(rows), int(v_off[-1]), d0.size
    dest_cap = n0 if dest_cap is None else dest_cap
    out_cap = m if out_cap is None else out_cap
    dest = np.full(dest_cap + GUARD, SENT, np.uint64)
    out = np.full(out_cap + GUARD, SENT, np.uint64)
    oo = np.full(nrows + 1 + GUARD, SENT, np.uint64)
    cnt = np.full(nrows + GUARD, CSENT, np.uint32)
    n = C.c_size_t(SENT)
    t = sg_filter_tree(f)
    rc = lib.dgx_sg_filter(C.byref(t), tab, len(leaves), (d0 if n0 else np.zeros(1, np.uint64)).ctypes.data, n0,
                           v.ctypes.data, v_off.ctypes.data, nrows, count, offset, dest.ctypes.data, dest_cap,
                           C.byref(n), None if counts_only else out.ctypes.data, oo.ctypes.data, out_cap,
                           cnt.ctypes.data)
    del keep
    guards = np.all(dest[dest_cap:] == SENT) and np.all(oo[nrows + 1:] == SENT) and np.all(cnt[nrows:] == CSENT)
    guards = guards and (np.all(out == SENT) if counts_only else np.all(out[out_cap:] == SENT))
    if rc != OK:
        return rc, None, guards
    K = int(oo[nrows])
    guards = guards and np.all(dest[n.value:] == SENT) and (counts_only or np.all(out[K:] == SENT))
    res = [out[int(oo[i]):int(oo[i + 1])].copy() for i in range(nrows)]
    return rc, (res, cnt[:nrows].copy(), dest[:n.value].copy()), guards


def dev_call(lib, lane, case, slack=0, len_words=False, counts_only=False, mutate=None, null=(), dest_cap=None,
             out_cap=None):
    """dgx_dev_sg_filter with `slack` garbage slots past D0, the values and every LIST leaf; len_words passes |D0| and
    the LIST lengths as device words (with garbage above bit 32).  mutate(arrays) may break the inputs before upload;
    each argument named in `null` (d0, v, v_off, dest, dest_len, out_off, counts) is passed as NULL.
    Returns (rc, rc of the sync, dest length, (rows, counts, dest) or None, launches, guards intact)."""
    import torch

    from dgraph_b200 import _lib
    from dgraph_b200.algo import SGF_CMP, sg_filter_flat, sg_filter_tree

    tree, leaves, d0, rows, count, offset = case
    f = sg_filter_flat(tree)
    d0 = np.asarray(d0, np.uint64)
    v, v_off = csr(rows)
    a = {"d0": np.concatenate([d0, np.full(slack, 5, np.uint64)]), "v": np.concatenate([v, np.full(slack, 9, np.uint64)]),
         "v_off": v_off.copy(), "leaves": [list(lf) for lf in leaves]}
    for lf in a["leaves"]:
        if lf[0] == "list":
            lf[1] = np.concatenate([np.asarray(lf[1], np.uint64), np.full(slack, 1, np.uint64)])
    n0, nrows = d0.size, len(rows)
    hi = 0x7F << 40
    words = {"d0": n0 | hi, "lists": [len(lf[1]) | hi for lf in leaves if lf[0] == "list"]}
    if mutate:
        mutate(a, words)
    keep, descs = [], []
    li = 0
    for lf, orig in zip(a["leaves"], leaves):
        if lf[0] == "list":
            d = _t(lf[1])
            n = len(orig[1]) + (slack if len_words else 0)  # the room, or the exact length
            dl = None
            if len_words:
                dl = _t([words["lists"][li]])
                keep.append(dl)
            li += 1
            keep.append(d)
            descs.append(_lib.SgFilterLeaf(0, 0, 0, d.data_ptr(), n, dl.data_ptr() if dl is not None else None, None,
                                           None))
        else:
            d = _t(np.concatenate([np.asarray(lf[3]), np.zeros(slack, np.asarray(lf[3]).dtype)]),
                   np.uint32 if lf[0] == "count" else np.uint64)
            keep.append(d)
            descs.append(_lib.SgFilterLeaf(1, SGF_CMP[lf[1]], int(lf[2]), None, 0, None,
                                           d.data_ptr() if lf[0] == "count" else None,
                                           d.data_ptr() if lf[0] == "len" else None))
    tab = (_lib.SgFilterLeaf * max(len(descs), 1))(*descs)
    d0_cap = n0 + slack if len_words else n0
    v_cap = int(v_off[-1]) + slack
    d_d0, d_v, d_off = _t(a["d0"]), _t(a["v"]), _t(a["v_off"])
    d_len = _t([words["d0"]]) if len_words else None
    d_dest, d_dl = sent(d0_cap + GUARD), sent(1 + GUARD)
    d_out = None if counts_only else sent(v_cap + GUARD)
    d_oo, d_cnt = sent(nrows + 1 + GUARD), sent(nrows + GUARD, counts=True)
    torch.cuda.synchronize()
    t = sg_filter_tree(f)
    l0 = lib.dgx_lane_launches(lane)
    p = {k: (None if k in null else x.data_ptr()) for k, x in (("d0", d_d0), ("v", d_v), ("v_off", d_off),
                                                             ("dest", d_dest), ("dest_len", d_dl), ("out_off", d_oo),
                                                             ("counts", d_cnt))}
    rc = lib.dgx_dev_sg_filter(lane, C.byref(t), tab, len(descs), p["d0"], d0_cap,
                               d_len.data_ptr() if d_len is not None else None, p["v"], p["v_off"], nrows, v_cap, count,
                               offset, p["dest"], d0_cap if dest_cap is None else dest_cap, p["dest_len"],
                               d_out.data_ptr() if d_out is not None else None, p["out_off"],
                               v_cap if out_cap is None else out_cap, p["counts"])
    src = lib.dgx_lane_sync(lane)
    launches = lib.dgx_lane_launches(lane) - l0
    dest, dl, oo = (x.cpu().numpy().view(np.uint64) for x in (d_dest, d_dl, d_oo))
    out = d_out.cpu().numpy().view(np.uint64) if d_out is not None else None
    cnt = d_cnt.cpu().numpy().view(np.uint32)
    guards = (np.all(dest[d0_cap:] == SENT) and np.all(dl[1:] == SENT) and np.all(oo[nrows + 1:] == SENT) and
              np.all(cnt[nrows:] == CSENT) and (out is None or np.all(out[v_cap:] == SENT)))
    if rc != OK or src != OK:  # a refused call writes the dest length 0 at most
        guards = (guards and np.all(dest == SENT) and np.all(oo == SENT) and np.all(cnt == CSENT) and
                  (out is None or np.all(out == SENT)))
        return rc, src, int(dl[0]), None, launches, guards
    D, K = int(dl[0]), int(oo[nrows])
    guards = guards and np.all(dest[D:] == SENT) and (out is None or np.all(out[K:] == SENT))
    res = None if out is None else [out[int(oo[i]):int(oo[i + 1])].copy() for i in range(nrows)]
    return rc, src, D, (res, cnt[:nrows].copy(), dest[:D].copy()), launches, guards


@pytest.mark.parametrize("form", ["host", "dev", "dev_words"])
def test_random_trees(lib, lane, form):
    rng = np.random.default_rng({"host": 1900, "dev": 1901, "dev_words": 1902}[form])
    for k in range(300):
        case = gs.random_case(rng)
        want = so.sg_filter(*case)
        co = k % 5 == 4
        if form == "host":
            rc, got, guards = host_call(lib, case, counts_only=co)
            assert rc == OK and guards, (case, lib.dgx_last_error())
        else:
            rc, src, _, got, launches, guards = dev_call(lib, lane, case, slack=k % 3, len_words=form == "dev_words",
                                                         counts_only=co)
            assert rc == OK and src == OK and guards, (case, lib.dgx_last_error())
        assert same(got, want, co), case


def test_counts_only_matches_rows(lib, lane):
    rng = np.random.default_rng(1910)
    for _ in range(60):
        case = gs.random_case(rng, max_u=400)
        want = so.sg_filter(*case)
        _, got, _ = host_call(lib, case, counts_only=True)
        assert np.array_equal(got[1], want[1]) and np.array_equal(got[1], [len(r) for r in want[0]])
        _, _, _, got, _, guards = dev_call(lib, lane, case, counts_only=True)
        assert guards and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])


def _base():
    d0 = np.array([2, 4, 6, 8, 10, 12], np.uint64)
    leaves = [("list", np.array([1, 4, 6, 9, 12], np.uint64)),
              ("count", "gt", 1, np.array([0, 2, 3, 1, 5, 2], np.uint32)),
              ("len", "ge", 1, np.array([0, 1, 1, 3, 3, 4, 4], np.uint64))]
    rows = [np.array([2, 4, 6], np.uint64), np.array([], np.uint64), np.array([4, 8, 10, 12, 13], np.uint64)]
    return ("or", [("and", [0, 1]), ("not", 2)]), leaves, d0, rows, 2, 1


def test_device_detected_refusals(lib, lane):
    def swap(key, i):
        def m(a, w):
            a[key][i], a[key][i + 1] = a[key][i + 1], a[key][i]
        return m

    def leaf_swap(a, w):
        a["leaves"][0][1][1], a["leaves"][0][1][2] = a["leaves"][0][1][2], a["leaves"][0][1][1]

    def off_dec(a, w):
        a["leaves"][2][3] = np.array([0, 1, 1, 3, 2, 4, 4], np.uint64)

    def voff(vals):
        def m(a, w):
            a["v_off"] = np.array(vals, np.uint64)
        return m

    def d0_word(a, w):
        w["d0"] = 8  # the room is 6 values and 1 of slack

    def list_word(a, w):
        w["lists"][0] = 7

    cases = [swap("d0", 2), swap("v", 0), swap("v", 4), leaf_swap, off_dec, voff([1, 3, 3, 8]), voff([0, 3, 2, 8]),
             voff([0, 3, 3, 10]), d0_word, list_word]
    ok_first = dev_call(lib, lane, _base(), slack=1, len_words=True)
    assert ok_first[0] == OK and ok_first[1] == OK and ok_first[5]
    for m in cases:
        rc, src, dl, got, _, guards = dev_call(lib, lane, _base(), slack=1, len_words=True, mutate=m)
        assert rc == OK and src == ERR_ARG and dl == 0 and got is None and guards, m
        # the lane is usable again after a refusal
        rc, src, _, got, _, guards = dev_call(lib, lane, _base())
        assert rc == OK and src == OK and guards and same(got, so.sg_filter(*_base()))


def test_host_form_refusals(lib):
    base = _base()
    bad_d0 = (base[0], base[1], np.array([2, 6, 4, 8, 10, 12], np.uint64), base[3], 0, 0)
    bad_row = (base[0], base[1], base[2], [np.array([4, 2], np.uint64)], 0, 0)
    bad_leaf = (base[0], [("list", np.array([1, 1], np.uint64))] + base[1][1:], base[2], base[3], 0, 0)
    bad_off = (base[0], base[1][:2] + [("len", "ge", 1, np.array([0, 1, 1, 3, 2, 4, 4], np.uint64))], base[2],
               base[3], 0, 0)
    for case in (bad_d0, bad_row, bad_leaf, bad_off):
        rc, got, guards = host_call(lib, case)
        assert rc == ERR_ARG and got is None and guards
    rc, got, guards = host_call(lib, base)
    assert rc == OK and guards and same(got, so.sg_filter(*base))


def test_argument_and_capacity_errors(lib, lane):
    base = _base()
    assert host_call(lib, base, dest_cap=5)[0] == ERR_CAP
    assert host_call(lib, base, out_cap=7)[0] == ERR_CAP
    rc, _, guards = host_call(lib, base, out_cap=7, counts_only=True)  # counts-only mode needs no value room
    assert rc == OK and guards
    # the device form refuses the same null pointers and capacities at the call, before any launch
    for arg in ("d0", "v", "v_off", "dest", "dest_len", "out_off", "counts"):
        rc, src, _, got, launches, guards = dev_call(lib, lane, base, null=(arg,))
        assert rc == ERR_ARG and src == OK and got is None and launches == 0 and guards, arg
    empty = (base[0], base[1][:1], np.zeros(0, np.uint64), base[3], 0, 0)
    rc, src, _, got, launches, guards = dev_call(lib, lane, empty, null=("out_off",))
    assert rc == ERR_ARG and launches == 0 and guards
    for caps in ({"dest_cap": 5}, {"out_cap": 7}):
        rc, src, _, got, launches, guards = dev_call(lib, lane, base, **caps)
        assert rc == ERR_CAP and launches == 0 and guards, caps
    rc, src, _, got, launches, guards = dev_call(lib, lane, base, counts_only=True, out_cap=0)
    assert rc == OK and src == OK and guards and same(got, so.sg_filter(*base), counts_only=True)


def big_tree(scale):
    """A tree over the four leaves of gen_sg_filter.big_case: an OR of scale ANDs, each of a leaf, a NOT and a one-child
    OR, beside a chain of min(scale, 40) NOTs (the depth stays inside DGX_SGF_MAX_DEPTH).  With big_case's 7-node tree
    at scale 1, the trees grow from 7 to 77 and 647 nodes as the rows and D0 grow tenfold twice."""
    chain = 1
    for _ in range(min(scale, 40)):
        chain = ("not", chain)
    wide = ("or", [("and", [i % 4, ("not", (i + 1) % 4), ("or", [(i + 2) % 4])]) for i in range(scale)])
    return ("and", [0, ("or", [wide, chain, ("not", 3)])])


def test_launches_follow_the_plan(lib, lane):
    rng = np.random.default_rng(1930)
    seen = set()
    for scale in (1, 10, 100):
        case = gs.big_case(rng, nrows=20 * scale, nvals=400 * scale, n0=300 * scale,
                           lists=(50 * scale, 500 * scale, 200 * scale), first=3)
        for c in (case, (("and", [0, ("or", [1, 2, ("and", [1, ("not", 3)])]), ("not", ("not", 3))]),) + case[1:],
                  (big_tree(scale),) + case[1:]):
            rc, src, _, got, launches, guards = dev_call(lib, lane, c)
            assert rc == OK and src == OK and guards and same(got, so.sg_filter(*c))
            assert launches == sp.launches(c[2].size)
            seen.add(launches)
    assert seen == {sp.K["LAUNCHES"]}
    from dgraph_b200.algo import sg_filter_flat

    assert [sg_filter_flat(big_tree(k))["nnodes"] for k in (10, 100)] == [77, 647]
    empty = (0, [("list", np.array([1], np.uint64))], np.zeros(0, np.uint64), [np.array([1], np.uint64)], 0, 0)
    rc, src, dl, got, launches, guards = dev_call(lib, lane, empty)
    assert rc == OK and src == OK and dl == 0 and launches == sp.launches(0) == 0 and guards
    assert got[1].tolist() == [0]


def test_device_chain_from_unfiltered_rows(lib, lane):
    """Rows from dgx_dev_list_uids_unfiltered_rows over UidPacks, D0 from dgx_dev_merge_sorted_matrix over them (its
    length word feeds d_d0_len), a has(friend)-style COUNT leaf from dgx_dev_list_count_rows over D0's packs and a LIST
    leaf from a second matrix merge's length word: no host read between the calls (the host derives D0's keys for
    the count rows' pack table from the same edges, as Go's processTask does from the result it holds)."""
    import torch

    from dgraph_b200 import _lib, codec, pb
    from dgraph_b200.algo import sg_filter_flat, sg_filter_tree
    from oracle import pyoracle as orc

    rng = np.random.default_rng(1940)
    adj = {u: np.unique(rng.integers(1, 500, int(rng.integers(0, 10)))).astype(np.uint64) for u in range(1, 501)}
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

    def tab(src):
        return (C.c_void_p * max(len(src), 1))(*[handles[int(u)].value if int(u) in handles else None for u in src])

    src = np.arange(1, 200, 3, dtype=np.uint64)
    n = src.size
    cap = int(sum(adj[int(u)].size for u in src))
    z = np.zeros(n + 1, np.uint64)
    d_rows, d_off = (torch.zeros(x, dtype=torch.int64, device="cuda") for x in (cap + 1, n + 1))
    assert lib.dgx_dev_list_uids_unfiltered_rows(lane, tab(src), n, None, None, z.ctypes.data, 0, 0,
                                                 d_rows.data_ptr(), cap, d_off.data_ptr()) == OK
    d_d0, d_d0len = torch.zeros(cap + 1, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64,
                                                                                      device="cuda")
    assert lib.dgx_dev_merge_sorted_matrix(lane, d_rows.data_ptr(), d_off.data_ptr(), n, cap, d_d0.data_ptr(), cap,
                                           d_d0len.data_ptr()) == OK
    d0 = np.unique(np.concatenate([adj[int(u)] for u in src]))
    d_cnt = torch.zeros(cap + 1, dtype=torch.int32, device="cuda")
    zc = np.zeros(d0.size + 1, np.uint64)
    assert lib.dgx_dev_list_count_rows(lane, tab(d0), d0.size, None, None, zc.ctypes.data, 0, d_cnt.data_ptr()) == OK
    # a LIST leaf from a second merge: the rows of a few other sources
    src2 = np.arange(2, 120, 5, dtype=np.uint64)
    cap2 = int(sum(adj[int(u)].size for u in src2))
    z2 = np.zeros(src2.size + 1, np.uint64)
    d_r2, d_o2 = (torch.zeros(x, dtype=torch.int64, device="cuda") for x in (cap2 + 1, src2.size + 1))
    assert lib.dgx_dev_list_uids_unfiltered_rows(lane, tab(src2), src2.size, None, None, z2.ctypes.data, 0, 0,
                                                 d_r2.data_ptr(), cap2, d_o2.data_ptr()) == OK
    d_l, d_ll = torch.zeros(cap2 + 1, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64,
                                                                                   device="cuda")
    assert lib.dgx_dev_merge_sorted_matrix(lane, d_r2.data_ptr(), d_o2.data_ptr(), src2.size, cap2, d_l.data_ptr(),
                                           cap2, d_ll.data_ptr()) == OK
    tree = ("or", [("and", [0, 1]), ("not", 1)])
    f = sg_filter_flat(tree)
    leaves = (_lib.SgFilterLeaf * 2)(_lib.SgFilterLeaf(1, 3, 0, None, 0, None, d_cnt.data_ptr(), None),
                                     _lib.SgFilterLeaf(0, 0, 0, d_l.data_ptr(), cap2, d_ll.data_ptr(), None, None))
    d_dest, d_dl = sent(cap + GUARD), sent(1 + GUARD)
    d_out, d_oo, d_c = sent(cap + GUARD), sent(n + 1 + GUARD), sent(n + GUARD, counts=True)
    t = sg_filter_tree(f)
    assert lib.dgx_dev_sg_filter(lane, C.byref(t), leaves, 2, d_d0.data_ptr(), cap, d_d0len.data_ptr(),
                                 d_rows.data_ptr(), d_off.data_ptr(), n, cap, 3, 1, d_dest.data_ptr(), cap,
                                 d_dl.data_ptr(), d_out.data_ptr(), d_oo.data_ptr(), cap, d_c.data_ptr()) == OK
    assert lib.dgx_lane_sync(lane) == OK, lib.dgx_last_error()
    lst = np.unique(np.concatenate([adj[int(u)] for u in src2]))
    counts = np.array([adj[int(u)].size for u in d0], np.uint32)
    want = so.sg_filter(tree, [("count", "gt", 0, counts), ("list", lst)], d0, [adj[int(u)] for u in src], 3, 1)
    D = int(d_dl[0].item())
    oo = d_oo.cpu().numpy().view(np.uint64)
    out = d_out.cpu().numpy().view(np.uint64)
    got = ([out[int(oo[i]):int(oo[i + 1])] for i in range(n)], d_c.cpu().numpy().view(np.uint32)[:n],
           d_dest.cpu().numpy().view(np.uint64)[:D])
    assert same(got, want) and D > 0
    for h in handles.values():
        lib.dgx_dev_pack_free(h)


def test_concurrent_callers(lib):
    from dgraph_b200 import algo

    errs = []

    def host(k):
        try:
            rng = np.random.default_rng(1950 + k)
            for _ in range(40):
                case = gs.random_case(rng)
                rows, counts, dest = algo.SubgraphFilter(*case[:4], count=case[4], offset=case[5])
                assert same((rows, counts, dest.Uids), so.sg_filter(*case))
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    def dev(k):
        try:
            ln, _ = new_lane(lib)
            rng = np.random.default_rng(1960 + k)
            for _ in range(40):
                case = gs.random_case(rng)
                rc, src, _, got, _, guards = dev_call(lib, ln, case)
                assert rc == OK and src == OK and guards and same(got, so.sg_filter(*case))
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


def test_c19a_sized_call(lib, lane):
    """C19a: 10 000 rows of about 1e7 values, D0 of 3e6, the 7-node tree, first: 10, both forms."""
    case = gs.big_case(np.random.default_rng(19), nrows=10_000, nvals=10_000_000, n0=3_000_000)
    want = so.sg_filter(*case)
    rc, got, guards = host_call(lib, case)
    assert rc == OK and guards and same(got, want)
    rc, src, _, got, launches, guards = dev_call(lib, lane, case)
    assert rc == OK and src == OK and guards and same(got, want) and launches == sp.K["LAUNCHES"]
    assert want[2].size > 0 and sum(r.size for r in want[0]) > 0


@pytest.mark.parametrize("form", ["host", "dev", "dev_words"])
def test_reference_answers(lib, lane, form):
    """The published answers of the reference's @filter tests (tests/golden/sg_filter_common.json) through both
    forms, each also bit for bit against the restatement."""
    for label, case, counts_only, want in sgg.cases():
        if form == "host":
            rc, got, guards = host_call(lib, case, counts_only=counts_only)
            assert rc == OK and guards, label
        else:
            rc, src, _, got, _, guards = dev_call(lib, lane, case, slack=2, len_words=form == "dev_words",
                                                  counts_only=counts_only)
            assert rc == OK and src == OK and guards, label
        assert sgg.check(got, want), label
        assert same(got, so.sg_filter(*case), counts_only), label
