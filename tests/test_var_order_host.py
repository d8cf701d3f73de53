"""Ordering by a value variable on the host (no GPU): the line-by-line restatement (var_order_oracle.c) against the
independent formula (gen_var_order.formula) over thousands of random cases, the restatement's pdqsort helpers reached
by the fixtures the GPU tests use, every argument and capacity error dgx_var_order refuses before it needs a device,
and the launch plan model."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import gen_var_order as gv
import var_order_oracle as vo
import var_order_golden as vg
import var_order_plan as vp
from dgraph_b200 import _lib
from dgraph_b200.algo import OrderByVar, var_order_leaf

GUARD = np.uint64(0xA5A5A5A5DEADBEEF)


def run(case):
    P = gv.formula(*case)
    try:
        rows, dest = vo.var_order(*case)
    except vo.NilMap:
        assert P.error == "nil"
        return "nil"
    except vo.NotSortable:
        assert P.error == "bool"
        return "bool"
    assert P.error is None
    gv.check(P, rows, dest, case[1])
    return "ok"


@pytest.mark.parametrize("seed", range(10))
def test_restatement_satisfies_formula(seed):
    rng = np.random.default_rng(1900 + seed)
    seen = set()
    for _ in range(400):
        seen.add(run(gv.random_case(rng)))
    assert "ok" in seen


@pytest.mark.parametrize("label,case,want", vg.cases(), ids=[c[0] for c in vg.cases()])
def test_reference_answers(label, case, want):
    # the published answers of the reference's tests, through the restatement and the formula
    if want == "nil":
        with pytest.raises(vo.NilMap):
            vo.var_order(*case)
        assert gv.formula(*case).error == "nil"
        return
    rows, dest = vo.var_order(*case)
    assert vg.check(rows, dest, want), label
    P = gv.formula(*case)
    assert all(r[0] == "exact" for r in P.rows)
    assert vg.check([r[1] for r in P.rows], P.dest, want), label


def test_reference_answers_catch_a_wrong_order():
    # the published ties tell Go's order apart: 23 before 31 at count 1, and 24, 25, 101 at 0, each in uid order
    for label, i in (("TestMultiCountSort", 1), ("TestQueryVarValAggMul", 2)):
        case, want = [(c, w) for lb, c, w in vg.cases() if lb == label][0]
        rows, dest = vo.var_order(*case)
        flipped = [int(x) for x in rows[0]]
        flipped[i], flipped[i + 1] = flipped[i + 1], flipped[i]
        assert vg.check(rows, dest, want) and not vg.check([flipped], dest, want), label


def test_formula_predicts_exact_rows():
    # tier 1 and the 12-entry rule: the exact permutation, ties in row order
    keys = np.arange(1, 13, dtype=np.uint64)
    m = (keys, np.array([3, 1, 3, 2, 1, 3, 2, 1, 3, 2, 1, 3], np.int64))
    for desc in (False, True):
        rows, _ = vo.var_order(m, desc, keys, [keys])
        want = sorted(keys.tolist(), key=lambda k: int(m[1][k - 1]), reverse=desc)
        assert rows[0].tolist() == want
    # -0.0 and +0.0 tie, and keep row order in a short row
    m = (np.array([1, 2, 3], np.uint64), np.array([0.0, -0.0, -1.0]))
    assert vo.var_order(m, False, [1, 2, 3], [[1, 2, 3]])[0][0].tolist() == [3, 1, 2]
    assert vo.var_order(m, True, [1, 2, 3], [[1, 2, 3]])[0][0].tolist() == [1, 2, 3]


def test_quirks():
    d = np.array([1, 2, 3, 4, 5], np.uint64)
    # a row without a mapped uid is left as the dest filter left it (not emptied, not sorted), and paged
    rows, dest = vo.var_order((np.array([9], np.uint64), np.array([1], np.int64)), True, d, [[1, 3, 5, 7]], 2, 0)
    assert rows[0].tolist() == [1, 3] and dest.tolist() == [1, 3]
    # uids without an entry are dropped from a row that has one
    rows, _ = vo.var_order((np.array([3, 5], np.uint64), np.array([2, 1], np.int64)), False, d, [[1, 3, 5]])
    assert rows[0].tolist() == [5, 3]
    # an empty map is no error; a nil map is
    assert vo.var_order((np.zeros(0, np.uint64), np.zeros(0, np.int64)), False, d, [[2, 4]])[0][0].tolist() == [2, 4]
    with pytest.raises(vo.NilMap):
        vo.var_order(None, False, d, [[2, 4]])
    # only the first mapped entry's type is checked: a later bool sorts by type id (after ints and floats)
    tagged = (np.array([1, 2, 3], np.uint64), np.array([1, 5, 0], np.uint64), np.array([3, 1, 1], np.uint8))
    with pytest.raises(vo.NotSortable):
        vo.var_order(tagged, False, d, [[1, 2, 3]])
    assert vo.var_order(tagged, False, d, [[2, 3, 1]])[0][0].tolist() == [3, 2, 1]
    # nils sort last both ways; a negative count takes the back
    nil = (np.array([1, 2, 3, 4], np.uint64), np.array([0, 7, 0, 1], np.uint64), np.array([4, 1, 4, 1], np.uint8))
    assert vo.var_order(nil, False, d, [[1, 2, 3, 4]])[0][0].tolist()[:2] == [4, 2]
    assert vo.var_order(nil, True, d, [[1, 2, 3, 4]])[0][0].tolist()[:2] == [2, 4]
    assert vo.var_order(nil, False, d, [[1, 2, 3, 4]], -2, 0)[0][0].tolist() == \
        vo.var_order(nil, False, d, [[1, 2, 3, 4]])[0][0].tolist()[2:]


def test_pdqsort_helpers_reached():
    # the long fixtures of the GPU tests reach every helper of Go's pdqsort
    rng = np.random.default_rng(0)
    n = 20000
    u = np.arange(n, dtype=np.uint64)
    cases = {"ties": (np.full(n, 1, np.uint8), rng.integers(0, 100, n).astype(np.uint64), False),
             "nil": (np.full(n, 4, np.uint8), np.zeros(n, np.uint64), True),
             "dec": (np.full(n, 1, np.uint8), np.concatenate([np.arange(n - 1, 0, -1), [1]]).astype(np.uint64), False)}
    seen = {}
    for name, (t, w, desc) in cases.items():
        vo.stats()
        ws, us = vo.go_sort(t, w, u, desc)
        seen[name] = vo.stats()
        assert sorted(us.tolist()) == u.tolist()
    assert seen["ties"]["partition_equal"] and seen["ties"]["partial_insertion_ok"] and seen["ties"]["insertion"]
    assert seen["nil"]["heap"] and seen["nil"]["break_patterns"]
    assert seen["dec"]["reverse"]


def test_go_pin_inputs():
    # the inputs tests/go_sort_pin/main.go pins against Go: tied rows past 12 entries, nils, NaN and mixed types; the
    # restatement returns a permutation of each and agrees with the formula's equivalence classes where Less is a
    # strict weak order
    pins = vo.pin_inputs()
    assert len(pins) == 40
    src = open(vo.os.path.join(vo._HERE, "go_sort_pin", "main.go")).read()
    for kind in vo.PIN_KINDS:
        assert f'case "{kind}":' in src
    for name, t, w, desc in pins:
        n = len(t)
        ws, us = vo.go_sort(t, w, np.arange(1, n + 1, dtype=np.uint64), desc)
        assert sorted(us.tolist()) == list(range(1, n + 1)), name
        vals = [(int(a), gv.value(int(a), b)) for a, b in zip(t, w)]
        if gv.weak_order(vals, desc) and n < 1000:
            got = [vals[int(x) - 1] for x in us]
            for a, b in zip(got, got[1:]):
                assert not gv.Less(b, a, desc), name


def call(m, desc, dest, rows, count=0, offset=0, out_cap=None, dest_cap=None, leaf=None, **ptr):
    """dgx_var_order with guard words; ptr replaces an argument with None (NULL).  Returns (rc, outputs untouched)."""
    keep, lf = var_order_leaf(m) if leaf is None else ([], leaf)
    d = np.ascontiguousarray(np.asarray(dest, np.uint64))
    v_off = ptr.pop("v_off_arr", None)
    if v_off is None:
        v_off = np.zeros(len(rows) + 1, np.uint64)
        np.cumsum([len(r) for r in rows], out=v_off[1:])
    v = np.concatenate([np.asarray(r, np.uint64) for r in rows] + [np.zeros(1, np.uint64)])
    nrows, M = len(rows), int(v_off[-1])
    out = np.full(max(M, 1) + 4, GUARD, np.uint64)
    oo = np.full(nrows + 5, GUARD, np.uint64)
    dout = np.full(max(d.size, 1) + 4, GUARD, np.uint64)
    n = C.c_size_t(12345)
    args = {"var": C.byref(lf), "d": d.ctypes.data if d.size else None, "v": v.ctypes.data,
            "v_off": v_off.ctypes.data, "out": out.ctypes.data, "oo": oo.ctypes.data, "dout": dout.ctypes.data,
            "len": C.byref(n)}
    args.update(ptr)
    rc = _lib.load().dgx_var_order(args["var"], int(desc), args["d"], d.size, args["v"], args["v_off"], nrows, count,
                                   offset, args["out"], args["oo"], M if out_cap is None else out_cap, args["dout"],
                                   d.size if dest_cap is None else dest_cap, args["len"])
    del keep
    untouched = np.all(out == GUARD) and np.all(oo == GUARD) and np.all(dout == GUARD) and n.value == 12345
    return rc, untouched


KEYS = np.array([2, 4, 6, 8], np.uint64)
MAP = (KEYS, np.array([3, 1, 2, 0], np.int64))
ROWS = [np.array([2, 4], np.uint64), np.array([6, 8], np.uint64)]


def test_argument_and_capacity_errors():
    ARG, CAP = _lib.DGX_ERR_ARG, _lib.DGX_ERR_CAP
    assert call(MAP, False, KEYS, ROWS, dest_cap=3) == (CAP, True)
    assert call(MAP, False, KEYS, ROWS, out_cap=3) == (CAP, True)
    for k in ("var", "len", "v_off", "oo", "dout", "d", "v", "out"):
        assert call(MAP, False, KEYS, ROWS, **{k: None}) == (ARG, True), k
    # Go's nil map ("used before definition"), a tagless map of another type, d_len in the host form, a null array
    assert call(None, False, KEYS, ROWS) == (ARG, True)
    k, w = KEYS.copy(), MAP[1].view(np.uint64).copy()
    L = _lib.MathLeaf
    assert call(None, False, KEYS, ROWS, leaf=L(k.ctypes.data, w.ctypes.data, None, None, 4, 3, 0)) == (ARG, True)
    assert call(None, False, KEYS, ROWS, leaf=L(k.ctypes.data, w.ctypes.data, None, w.ctypes.data, 4, 1, 0)) == \
        (ARG, True)
    assert call(None, False, KEYS, ROWS, leaf=L(None, w.ctypes.data, None, None, 4, 1, 0)) == (ARG, True)
    assert call(None, False, KEYS, ROWS, leaf=L(k.ctypes.data, w.ctypes.data, None, None, 1 << 32, 1, 0)) == \
        (ARG, True)
    # row offsets not starting at 0 or decreasing
    assert call(MAP, False, KEYS, ROWS, v_off_arr=np.array([1, 2, 4], np.uint64)) == (ARG, True)
    assert call(MAP, False, KEYS, ROWS, v_off_arr=np.array([0, 3, 2], np.uint64)) == (ARG, True)
    # the nil check comes before the empty shortcut
    assert call(None, False, np.zeros(0, np.uint64), []) == (ARG, True)


def test_empty_calls_need_no_device():
    for dest, rows in ((np.zeros(0, np.uint64), ROWS), (KEYS, [])):
        keep, lf = var_order_leaf(MAP)
        v = np.array([2, 4, 6, 8], np.uint64)
        v_off = np.zeros(len(rows) + 1, np.uint64)
        np.cumsum([len(r) for r in rows], out=v_off[1:])
        oo = np.full(len(rows) + 1, GUARD, np.uint64)
        n = C.c_size_t(9)
        d = np.asarray(dest, np.uint64)
        rc = _lib.load().dgx_var_order(C.byref(lf), 1, d.ctypes.data if d.size else None, d.size, v.ctypes.data,
                                       v_off.ctypes.data, len(rows), 3, 1, None if not rows else v.ctypes.data,
                                       oo.ctypes.data, int(v_off[-1]), None if not d.size else d.ctypes.data, d.size,
                                       C.byref(n))
        assert rc == _lib.DGX_OK and n.value == 0 and oo.tolist() == [0] * (len(rows) + 1)
    rows, dest = OrderByVar(MAP, True, [], ROWS, 1, 0)
    assert [r.tolist() for r in rows] == [[], []] and dest.Uids.tolist() == []


def test_launch_plan_model():
    K = vp.K
    assert (K["FIXED"], K["KEY_PASSES"], K["DIGIT_BITS"], K["MAX_INSERTION"]) == (13, 8, 8, 12)
    assert vp.launches(0, 5) == vp.launches(5, 0) == 0
    assert vp.launches(1, 1) == 37 and vp.launches(10**7, 256) == 40 and vp.launches(1, 257) == 43
    assert vp.launches(1, 65536) == 43 and vp.launches(1, 65537) == 46
    api = open(vp.os.path.join(vp.CSRC, "dgx_api.cu")).read()
    with pytest.raises(ValueError, match="restate"):
        vp.read_constants(api.replace("count_launches(l, 8);\n    return DGX_OK;\n}\n\nextern \"C\" int dgx_dev_var_order",
                                      "count_launches(l, 9);\n    return DGX_OK;\n}\n\nextern \"C\" int dgx_dev_var_order"))
    with pytest.raises(ValueError, match="restate"):
        vp.read_constants(api.replace("vo_tier_kernel<<<", "vo_tier2_kernel<<<"))
