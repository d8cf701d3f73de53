"""dgx_math_eval / dgx_dev_math_eval on the GPU: bit-exact against the restatement of evalMathTree
(tests/math_oracle.c) in keys, words and tags, refused exactly where the restatement fails or its answer depends on map
iteration order, with guard words past every output."""
import ctypes as C
import threading

import numpy as np
import pytest

import gen_math as gm
import math_oracle as mo
import math_plan as mp

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


@pytest.fixture(scope="module")
def lane(lib):
    import torch

    stream = torch.cuda.Stream()
    ln = lib.dgx_lane_create(0, C.c_void_p(stream.cuda_stream))
    assert ln
    yield ln
    lib.dgx_lane_destroy(ln)


def _b(x, dt=np.uint64):
    x = np.ascontiguousarray(x, dt)
    return x if x.size else np.zeros(1, dt)


def _up(x, dt=np.uint64):
    import torch

    return torch.from_numpy(_b(x, dt).view(np.int64 if dt == np.uint64 else np.uint8).copy()).cuda()


def _h(t):
    a = t.cpu().numpy()
    return a.view(np.uint64) if a.dtype == np.int64 else a


def key0_mixed(maps):
    return any(m is not None and len(m[0]) > 1 and int(np.asarray(m[0])[0]) == 0 for m in maps.values())


def want(tree, maps, rng_uids):
    """The restatement's answer, or None where the device must refuse."""
    if key0_mixed(maps):
        return None
    r = mo.evaluate(tree, maps, rng_uids, seed=0)
    return None if r[0] is None or r[4] else r


def prepared(tree, maps):
    from dgraph_b200 import algo

    names = {}
    nodes = algo.math_program(tree, names)
    leaves = [None] * len(names)
    for name, j in names.items():
        leaves[j] = algo.math_leaf_arrays(maps.get(name))
    return nodes, leaves


def run_host(lib, tree, maps, rng_uids, cap):
    from dgraph_b200 import _lib

    nodes, leaves = prepared(tree, maps)
    lv = (_lib.MathLeaf * max(len(leaves), 1))()
    for j, (k, w, t, typ, nil) in enumerate(leaves):
        lv[j] = _lib.MathLeaf(k.ctypes.data, w.ctypes.data, None if t is None else t.ctypes.data, None,
                              0 if nil else k.size, typ, nil)
    r = None if rng_uids is None else _b(rng_uids)
    ok, ow = np.full(cap + GUARD, SENT, np.uint64), np.full(cap + GUARD, SENT, np.uint64)
    ot = np.full(cap + GUARD, 0xAB, np.uint8)
    info = C.c_uint64(SENT)
    prog = (_lib.MathNode * len(nodes))(*nodes)
    rc = lib.dgx_math_eval(prog, len(nodes), lv, len(leaves), None if r is None else r.ctypes.data,
                           0 if rng_uids is None else len(rng_uids), ok.ctypes.data, ow.ctypes.data, ot.ctypes.data,
                           cap, C.byref(info))
    return rc, info.value, ok, ow, ot


def run_dev(lib, lane, tree, maps, rng_uids, cap, room=3, over=0):
    """Every leaf with `room` spare entries and its count (plus `over`) in a device word."""
    import torch

    from dgraph_b200 import _lib

    nodes, leaves = prepared(tree, maps)
    keep = []
    lv = (_lib.MathLeaf * max(len(leaves), 1))()
    for j, (k, w, t, typ, nil) in enumerate(leaves):
        n = 0 if nil else k.size
        pad = lambda a, dt: np.concatenate([np.asarray(a[:n], dt), np.full(room, 5, dt)])  # noqa: E731
        dk, dw = _up(pad(k, np.uint64)), _up(pad(w, np.uint64))
        dt_ = None if t is None else _up(pad(t, np.uint8), np.uint8)
        dn = _up(np.array([n + over], np.uint64))
        keep += [dk, dw, dt_, dn]
        lv[j] = _lib.MathLeaf(dk.data_ptr(), dw.data_ptr(), None if dt_ is None else dt_.data_ptr(),
                              None if nil else dn.data_ptr(), 0 if nil else n + room, typ, nil)
    dr = None if rng_uids is None else _up(rng_uids)
    ok = torch.full((cap + GUARD,), SENT - (1 << 64), dtype=torch.int64, device="cuda")
    ow = ok.clone()
    ot = torch.full((cap + GUARD,), 0xAB, dtype=torch.uint8, device="cuda")
    di = torch.full((1,), SENT - (1 << 64), dtype=torch.int64, device="cuda")
    prog = (_lib.MathNode * len(nodes))(*nodes)
    torch.cuda.synchronize()
    l0 = lib.dgx_lane_launches(lane)
    rc = lib.dgx_dev_math_eval(lane, prog, len(nodes), lv, len(leaves), None if dr is None else dr.data_ptr(),
                               0 if rng_uids is None else len(rng_uids), ok.data_ptr(), ow.data_ptr(), ot.data_ptr(),
                               cap, di.data_ptr())
    src = lib.dgx_lane_sync(lane)
    return rc, src, int(_h(di)[0]), _h(ok), _h(ow), _h(ot), lib.dgx_lane_launches(lane) - l0


def check(w, info, ok, ow, ot, cap):
    kind, k, words, tags, _ = w
    n = k.size
    assert info & 0xFFFFFFFF == n and {0: "none", 1: "map", 2: "const"}[(info >> 32) & 0xFF] == kind
    assert (info >> 40) & 0xFF == (np.bitwise_or.reduce(1 << tags.astype(np.int64)) if n else 0)
    assert np.array_equal(ok[:n], k) and np.array_equal(ow[:n], words) and np.array_equal(ot[:n], tags)
    assert (ok[n:] == SENT).all() and (ow[n:] == SENT).all() and (ot[n:] == 0xAB).all()


def cap_of(maps, rng_uids):
    return 1 + sum(0 if m is None else len(m[0]) for m in maps.values()) + (0 if rng_uids is None else len(rng_uids))


@pytest.mark.parametrize("seed", range(4))
def test_random_programs_host_form(lib, seed):
    rng = np.random.default_rng(seed)
    refusals = 0
    for _ in range(600):
        t, maps, r = gm.case(rng, max_depth=5)
        w, cap = want(t, maps, r), cap_of(maps, r)
        rc, info, ok, ow, ot = run_host(lib, t, maps, r, cap)
        if w is None:
            refusals += 1
            assert rc == ERR_ARG and info == SENT and (ok == SENT).all(), (t, maps, r)
        else:
            assert rc == OK, (t, maps, r)
            check(w, info, ok, ow, ot, cap)
    assert refusals > 0


@pytest.mark.parametrize("seed", range(2))
def test_random_programs_device_form(lib, lane, seed):
    rng = np.random.default_rng(100 + seed)
    for _ in range(200):
        t, maps, r = gm.case(rng, max_depth=5)
        w, cap = want(t, maps, r), cap_of(maps, r)
        rc, src, info, ok, ow, ot, _ = run_dev(lib, lane, t, maps, r, cap)
        assert rc == OK
        if w is None:
            assert src == ERR_ARG and info == SENT and (ok == SENT).all(), (t, maps, r)
        else:
            assert src == OK, (t, maps, r)
            check(w, info, ok, ow, ot, cap)


def _all_pairs(vals_a, vals_b):
    """Two maps over the same keys holding every pair of the given (tag, word) values."""
    pa = [(a, b) for a in vals_a for b in vals_b]
    k = np.arange(1, len(pa) + 1, dtype=np.uint64)
    ta = np.array([p[0][0] for p in pa], np.uint8)
    wa = np.array([p[0][1] for p in pa], np.uint64)
    tb = np.array([p[1][0] for p in pa], np.uint8)
    wb = np.array([p[1][1] for p in pa], np.uint64)
    return {"a": (k, wa, ta), "b": (k, wb, tb)}


def _edge_values():
    ints = [(1, int(np.array([x], np.int64).view(np.uint64)[0])) for x in gm.I64]
    flts = [(2, int(np.array([x], np.float64).view(np.uint64)[0])) for x in gm.F64]
    return ints + flts + [(3, 0), (3, 1), (4, 0)]


@pytest.mark.parametrize("op", gm.BIN + gm.CMP)
def test_every_binary_op_on_every_value_pair(lib, lane, op):
    vals = _edge_values()
    maps = _all_pairs(vals, vals)
    t = (op, ("var", "a"), ("var", "b"))
    w, cap = want(t, maps, None), cap_of(maps, None)
    if w is None:  # a comparison meeting a bool fails on some keys: refused, by order dependence
        assert op in gm.CMP
        assert run_host(lib, t, maps, None, cap)[0] == ERR_ARG
        assert run_dev(lib, lane, t, maps, None, cap)[1] == ERR_ARG
        maps = _all_pairs(vals[:-3], vals[:-3])
        w = want(t, maps, None)
    rc, info, ok, ow, ot = run_host(lib, t, maps, None, cap)
    assert rc == OK
    check(w, info, ok, ow, ot, cap)
    rc, src, info, ok, ow, ot, _ = run_dev(lib, lane, t, maps, None, cap)
    assert rc == OK and src == OK
    check(w, info, ok, ow, ot, cap)


@pytest.mark.parametrize("op", gm.UN)
def test_every_unary_op_on_every_value(lib, lane, op):
    vals = [v for v in _edge_values() if v[0] in (1, 2)]
    # failing keys alone in one map each would be order-dependent next to good ones: one key per call
    for tag, word in vals:
        maps = {"a": (np.array([7], np.uint64), np.array([word], np.uint64), np.array([tag], np.uint8))}
        t = (op, ("var", "a"))
        w = want(t, maps, None)
        rc, info, ok, ow, ot = run_host(lib, t, maps, None, 3)
        assert rc == OK
        check(w, info, ok, ow, ot, 3)
        rc, src, info, ok, ow, ot, _ = run_dev(lib, lane, t, maps, None, 3)
        assert rc == OK and src == OK
        check(w, info, ok, ow, ot, 3)


def test_scalar_rules_and_constant_fill(lib, lane):
    z, i = np.zeros(1, np.uint64), lambda *v: np.array(v, np.int64)  # noqa: E731
    a = (np.array([3, 5, 9], np.uint64), i(1, 2, 3))
    cases = [
        (("+", ("var", "s"), ("var", "t")), {"s": (z, i(2)), "t": (z, i(5))}, None),          # {0: s+t}
        (("*", ("+", ("var", "s"), ("var", "t")), ("var", "a")), {"s": (z, i(2)), "t": (z, i(5)), "a": a}, None),
        (("-", ("var", "a"), ("var", "s")), {"s": (z, i(2)), "a": a}, None),                # {0} on the right
        (("+", ("var", "s"), ("const", 1)), {"s": (z, i(2))}, np.array([4, 8], np.uint64)),  # constant fill
        (("+", ("var", "s"), ("const", 1)), {"s": (z, i(2))}, None),                         # on uid 0
        (("+", ("var", "s"), ("const", 1)), {"s": (z, i(2))}, np.zeros(0, np.uint64)),      # an empty range
        (("*", ("var", "c"), ("const", 2.5)), {"c": (np.array([2**64 - 1], np.uint64), i(4))}, np.array([6], np.uint64)),
        (("+", ("var", "a"), ("var", "f")), {"a": a, "f": (np.array([4], np.uint64), np.array([0.5]))}, None),
        (("cond", (">", ("var", "a"), ("const", 1)), ("var", "a"), ("var", "e")),
         {"a": a, "e": (np.zeros(0, np.uint64), i())}, None),                                  # nil entries
        (("cond", ("+", ("var", "e"), ("var", "e2")), ("const", 1), ("const", 2)),
         {"e": (np.zeros(0, np.uint64), i()), "e2": (np.zeros(0, np.uint64), i())}, None),   # cond over nil: refused
        (("cond", ("+", ("var", "a"), ("var", "e")), ("const", 1), ("const", 2)),
         {"a": (np.zeros(0, np.uint64), i()), "e": (np.array([4], np.uint64), i(1))}, None),
        (("u-", ("var", "m")), {"m": (np.array([0, 4], np.uint64), i(1, 2))}, None),        # key 0 among others
        (("+", ("var", "n"), ("const", 1)), {"n": None}, None),
    ]
    for t, maps, r in cases:
        w, cap = want(t, maps, r), cap_of(maps, r)
        rc, info, ok, ow, ot = run_host(lib, t, maps, r, cap)
        rc2, src, info2, ok2, ow2, ot2, _ = run_dev(lib, lane, t, maps, r, cap)
        if w is None:
            assert rc == ERR_ARG and src == ERR_ARG, t
        else:
            assert rc == OK and rc2 == OK and src == OK, t
            check(w, info, ok, ow, ot, cap)
            check(w, info2, ok2, ow2, ot2, cap)


def test_refusals_of_order_dependent_nodes(lib, lane):
    k = np.array([1 + 30 * j for j in range(5)], np.uint64)  # one shard
    i = lambda *v: np.array(v, np.int64)  # noqa: E731
    cases = [
        (("u-", ("var", "a")), {"a": (k, i(1, -2**63, 3, 4, 5))}),
        (("<", ("var", "a"), ("var", "b")), {"a": (k, i(1, 2, 3, 4, 5)), "b": (k[:2], i(0, 0))}),
        (("cond", ("var", "c"), ("const", 1), ("const", 2)),
         {"c": (k, np.array([1, 0, 5, 0, 1], np.uint64), np.array([3, 3, 1, 3, 3], np.uint8))}),
    ]
    for t, maps in cases:
        assert want(t, maps, None) is None
        assert run_host(lib, t, maps, None, 8)[0] == ERR_ARG
        assert run_dev(lib, lane, t, maps, None, 8)[1] == ERR_ARG
    # every key failing: an empty map, whatever the order
    t, maps = ("u-", ("var", "a")), {"a": (k, i(-2**63, -2**63, -2**63, -2**63, -2**63))}
    rc, info, ok, ow, ot = run_host(lib, t, maps, None, 8)
    assert rc == OK and info == 0


def test_malformed_inputs_are_refused_on_the_device(lib, lane):
    i = lambda *v: np.array(v, np.int64)  # noqa: E731
    t = ("+", ("var", "a"), ("const", 1))
    good = {"a": (np.array([2, 5, 9], np.uint64), i(1, 2, 3))}
    cases = [
        ({"a": (np.array([2, 9, 5], np.uint64), i(1, 2, 3))}, None),                      # keys not ascending
        ({"a": (np.array([2, 5, 5], np.uint64), i(1, 2, 3))}, None),                      # a repeated key
        ({"a": (np.array([2, 5, 9], np.uint64), np.array([1, 2, 3], np.uint64),
                np.array([1, 9, 1], np.uint8))}, None),                                   # an unknown entry tag
        (good, np.array([7, 3], np.uint64)),                                              # range not ascending
    ]
    for maps, r in cases:
        rc, info, ok, ow, ot = run_host(lib, t, maps, r, 8)
        assert rc == ERR_ARG and info == SENT and (ok == SENT).all() and (ot == 0xAB).all()
        rc, src, info, ok, ow, ot, _ = run_dev(lib, lane, t, maps, r, 8)
        assert rc == OK and src == ERR_ARG and info == SENT and (ok == SENT).all() and (ot == 0xAB).all()
    # a count word past the leaf's room
    rc, src, info, ok, ow, ot, _ = run_dev(lib, lane, t, good, None, 8, room=3, over=4)
    assert rc == OK and src == ERR_ARG and info == SENT and (ok == SENT).all()
    # the same call within the room answers
    rc, src, info, ok, ow, ot, _ = run_dev(lib, lane, t, good, None, 8, room=3, over=0)
    assert rc == OK and src == OK and info & 0xFFFFFFFF == 3


def test_capacity_errors(lib, lane):
    k = np.arange(1, 11, dtype=np.uint64)
    t, maps = ("+", ("var", "a"), ("const", 1)), {"a": (k, np.arange(10, dtype=np.int64))}
    rc, info, ok, ow, ot = run_host(lib, t, maps, None, 9)
    assert rc == ERR_CAP and info & 0xFFFFFFFF == 10 and (ok == SENT).all() and (ot == 0xAB).all()
    rc, src, info, ok, ow, ot, _ = run_dev(lib, lane, t, maps, None, 9)
    assert rc == OK and src == ERR_CAP and info & 0xFFFFFFFF == 10 and (ok == SENT).all()


def test_launch_counts_do_not_depend_on_keys_or_tree(lib, lane):
    import torch

    rng = np.random.default_rng(5)

    def merge_launches(total, nrows):
        v, off = _up(np.zeros(total, np.uint64)), _up(np.zeros(nrows + 1, np.uint64))
        out, n = _up(np.zeros(total + 1, np.uint64)), _up(np.zeros(1, np.uint64))
        torch.cuda.synchronize()
        l0 = lib.dgx_lane_launches(lane)
        assert lib.dgx_dev_merge_sorted_matrix(lane, v.data_ptr(), off.data_ptr(), nrows, total, out.data_ptr(),
                                               total + 1, n.data_ptr()) == OK
        assert lib.dgx_lane_sync(lane) == OK
        return lib.dgx_lane_launches(lane) - l0

    small = ("+", ("var", "a"), ("var", "b"))
    big = ("cond", ("<", ("*", ("var", "a"), ("const", 2)), ("var", "b")), ("sqrt", ("var", "a")),
           ("max", ("-", ("var", "b"), ("var", "a")), ("floor", ("/", ("var", "a"), ("const", 3.0)))))
    launch_set = set()
    for n in (1000, 10000):
        keys = np.sort(rng.choice(np.arange(1, 4 * n, dtype=np.uint64), n, replace=False))
        maps = {x: (keys, rng.integers(0, 100, n)) for x in "ab"}  # no key fails: nothing is refused
        for t in (small, big):
            rc, src, info, *_, launches = run_dev(lib, lane, t, maps, None, 2 * n + 1)
            assert rc == OK and src == OK
            assert launches == 7 + merge_launches(2 * n, 2) == mp.launches(2 * n)
            launch_set.add(launches - merge_launches(2 * n, 2))
    assert launch_set == {7}


def test_chain_propagate_then_math_then_math(lib, lane):
    """dgx_dev_var_propagate's d_out_len is a leaf's count word, and that math() call's info word the next one's."""
    import torch

    from dgraph_b200 import _lib

    src, dest = np.array([1, 2], np.uint64), np.array([10, 11, 12], np.uint64)
    rows = [np.array([10, 11], np.uint64), np.array([11, 12], np.uint64)]
    v_off = np.array([0, 2, 4], np.uint64)
    dsrc, dv, doff, ddest = _up(src), _up(np.concatenate(rows)), _up(v_off), _up(dest)
    lv = (_lib.VarLevel * 1)(_lib.VarLevel(dsrc.data_ptr(), doff.data_ptr(), dv.data_ptr(), ddest.data_ptr(), 2, 4, 3))
    mk, mv = _up(src), _up(np.array([3, 4], np.int64).view(np.uint64))
    pk, pv, pn = _up(np.zeros(3, np.uint64)), _up(np.zeros(3, np.uint64)), _up(np.zeros(1, np.uint64))
    assert lib.dgx_dev_var_propagate(lane, 1, mk.data_ptr(), mv.data_ptr(), 2, lv, 1, pk.data_ptr(), pv.data_ptr(), 3,
                                     pn.data_ptr()) == OK
    names = {}
    from dgraph_b200 import algo

    p1 = algo.math_program(("*", ("var", "p"), ("const", 2)), names)
    l1 = (_lib.MathLeaf * 1)(_lib.MathLeaf(pk.data_ptr(), pv.data_ptr(), None, pn.data_ptr(), 3, 1, 0))
    ok1, ow1, ot1, di1 = (_up(np.zeros(4, np.uint64)), _up(np.zeros(4, np.uint64)), _up(np.zeros(4, np.uint8), np.uint8),
                          _up(np.zeros(1, np.uint64)))
    assert lib.dgx_dev_math_eval(lane, (_lib.MathNode * len(p1))(*p1), len(p1), l1, 1, None, 0, ok1.data_ptr(), ow1.data_ptr(),
                                 ot1.data_ptr(), 4, di1.data_ptr()) == OK
    p2 = algo.math_program((">", ("var", "q"), ("const", 10)), {})
    l2 = (_lib.MathLeaf * 1)(_lib.MathLeaf(ok1.data_ptr(), ow1.data_ptr(), ot1.data_ptr(), di1.data_ptr(), 4, 1, 0))
    ok2, ow2, ot2, di2 = (_up(np.zeros(4, np.uint64)), _up(np.zeros(4, np.uint64)), _up(np.zeros(4, np.uint8), np.uint8),
                          _up(np.zeros(1, np.uint64)))
    assert lib.dgx_dev_math_eval(lane, (_lib.MathNode * len(p2))(*p2), len(p2), l2, 1, None, 0, ok2.data_ptr(), ow2.data_ptr(),
                                 ot2.data_ptr(), 4, di2.data_ptr()) == OK
    assert lib.dgx_lane_sync(lane) == OK
    torch.cuda.synchronize()
    # transformTo: 10 <- 3, 11 <- 3 + 4, 12 <- 4; times 2: 6, 14, 8; > 10: false, true, false
    assert _h(di2)[0] & 0xFFFFFFFF == 3
    assert _h(ok2)[:3].tolist() == [10, 11, 12] and _h(ow2)[:3].tolist() == [0, 1, 0] and _h(ot2)[:3].tolist() == [3] * 3


def test_chain_propagate_then_math_then_level_agg(lib, lane):
    """dgx_dev_var_propagate -> dgx_dev_math_eval with no host read between them; dgx_dev_var_level_agg takes its map
    size as an exact host size, so the math info word is read once before it."""
    import torch

    from dgraph_b200 import _lib, algo

    src, dest = np.array([1, 2], np.uint64), np.array([10, 11, 12], np.uint64)
    rows = [np.array([10, 11], np.uint64), np.array([11, 12], np.uint64)]
    dsrc, dv, doff, ddest = _up(src), _up(np.concatenate(rows)), _up(np.array([0, 2, 4], np.uint64)), _up(dest)
    lv = (_lib.VarLevel * 1)(_lib.VarLevel(dsrc.data_ptr(), doff.data_ptr(), dv.data_ptr(), ddest.data_ptr(), 2, 4, 3))
    mk, mv = _up(src), _up(np.array([1.5, 4.0]).view(np.uint64))
    pk, pv, pn = _up(np.zeros(3, np.uint64)), _up(np.zeros(3, np.uint64)), _up(np.zeros(1, np.uint64))
    assert lib.dgx_dev_var_propagate(lane, 2, mk.data_ptr(), mv.data_ptr(), 2, lv, 1, pk.data_ptr(), pv.data_ptr(), 3,
                                     pn.data_ptr()) == OK
    prog = algo.math_program(("sqrt", ("*", ("var", "p"), ("const", 2))), {})
    leaf = (_lib.MathLeaf * 1)(_lib.MathLeaf(pk.data_ptr(), pv.data_ptr(), None, pn.data_ptr(), 3, 2, 0))
    ok, ow, ot, di = (_up(np.zeros(4, np.uint64)), _up(np.zeros(4, np.uint64)), _up(np.zeros(4, np.uint8), np.uint8),
                      _up(np.zeros(1, np.uint64)))
    assert lib.dgx_dev_math_eval(lane, (_lib.MathNode * len(prog))(*prog), len(prog), leaf, 1, None, 0, ok.data_ptr(),
                                 ow.data_ptr(), ot.data_ptr(), 4, di.data_ptr()) == OK
    assert lib.dgx_lane_sync(lane) == OK
    n = int(_h(di)[0]) & 0xFFFFFFFF
    assert n == 3 and (int(_h(di)[0]) >> 40) & 0xFF == 1 << 2  # float values only
    par, prow = _up(np.array([100, 200], np.uint64)), _up(np.array([10, 11, 12, 11], np.uint64))
    poff = _up(np.array([0, 3, 4], np.uint64))
    lk, lw, ln = _up(np.zeros(2, np.uint64)), _up(np.zeros(2, np.uint64)), _up(np.zeros(1, np.uint64))
    assert lib.dgx_dev_var_level_agg(lane, 2, 2, ok.data_ptr(), ow.data_ptr(), n, par.data_ptr(), 2, poff.data_ptr(),
                                     prow.data_ptr(), 4, lk.data_ptr(), lw.data_ptr(), 2, ln.data_ptr()) == OK
    assert lib.dgx_lane_sync(lane) == OK
    torch.cuda.synchronize()
    # transformTo: 10 <- 1.5, 11 <- 1.5 + 4.0, 12 <- 4.0; sqrt(2 x): sqrt 3, sqrt 11, sqrt 8; sums per parent row
    m = {10: np.sqrt(3.0), 11: np.sqrt(11.0), 12: np.sqrt(8.0)}
    assert _h(ln)[0] == 2 and _h(lk)[:2].tolist() == [100, 200]
    assert _h(lw)[:2].view(np.float64).tolist() == [m[10] + m[11] + m[12], m[11]]


def test_concurrent_callers(lib):
    rng = np.random.default_rng(9)
    cases = [gm.case(rng) for _ in range(64)]
    wants = [want(*c) for c in cases]
    errors = []

    def worker(lo):
        for j in range(lo, len(cases), 4):
            t, maps, r = cases[j]
            cap = cap_of(maps, r)
            rc, info, ok, ow, ot = run_host(lib, t, maps, r, cap)
            try:
                if wants[j] is None:
                    assert rc == ERR_ARG
                else:
                    assert rc == OK
                    check(wants[j], info, ok, ow, ot, cap)
            except AssertionError as e:  # noqa: PERF203
                errors.append((j, e))

    th = [threading.Thread(target=worker, args=(i,)) for i in range(4)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors


def test_c18_sized_call(lib):
    """math(p * 2 + a / s) over a 2e6-entry propagated map, an age map and an aggregate s."""
    rng = np.random.default_rng(18)
    n = 2_000_000
    pk = np.sort(rng.choice(np.arange(1, 4 * n, dtype=np.uint64), n, replace=False))
    ak = np.sort(rng.choice(np.arange(1, 4 * n, dtype=np.uint64), n // 2, replace=False))
    maps = {"p": (pk, rng.random(n) * 100), "a": (ak, rng.integers(1, 90, n // 2)),
            "s": (np.zeros(1, np.uint64), np.array([3.0]))}
    t = ("+", ("*", ("var", "p"), ("const", 2)), ("/", ("var", "a"), ("var", "s")))
    from dgraph_b200 import algo

    kind, k, w, tg = algo.EvalMath(t, maps)
    keys = np.union1d(pk, ak)
    assert kind == "map" and np.array_equal(k, keys) and (tg == 2).all()
    pv = np.zeros(keys.size)
    pv[np.searchsorted(keys, pk)] = maps["p"][1] * 2
    av = np.zeros(keys.size)
    av[np.searchsorted(keys, ak)] = maps["a"][1].astype(np.float64) / 3.0
    assert np.array_equal(w.view(np.float64), pv + av)


def test_reference_query_answers_through_the_library(lib, lane):
    import math_golden as mg

    from dgraph_b200 import algo

    for name, tree, maps, r, want in mg.cases():
        assert mg.values(*algo.EvalMath(tree, maps, r)) == want, name
        w = mo.evaluate(tree, maps, r)
        rc, src, info, ok, ow, ot, _ = run_dev(lib, lane, tree, maps, r, cap_of(maps, r))
        assert rc == OK and src == OK, name
        check(w, info, ok, ow, ot, cap_of(maps, r))
