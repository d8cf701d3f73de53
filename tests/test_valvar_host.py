"""Value variables (transformTo and evalLevelAgg, query/query.go) without a GPU: the line-by-line restatement
(valvar_oracle.c) against the independent numpy formula (gen_valvar.py), Go's chunk completion orders, the argument
errors of dgx_var_propagate / dgx_var_level_agg (refused before anything is copied, outputs untouched) and the launch
plan model (valvar_plan.py)."""
import ctypes as C
import itertools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen_valvar as gv  # noqa: E402
import valvar_oracle as vo  # noqa: E402
import valvar_plan as vp  # noqa: E402

ERR_ARG = -3
SENT = 0xDEADBEEFCAFEF00D


def _same(a, b):
    return np.array_equal(a[0], b[0]) and np.array_equal(np.asarray(a[1]).view(np.uint64),
                                                        np.asarray(b[1]).view(np.uint64))


@pytest.mark.parametrize("kind", ["int", "smallint", "dyadic"])
@pytest.mark.parametrize("part", range(4))
def test_restatement_equals_formula(kind, part):
    rng = np.random.default_rng(100 + 10 * part + ["int", "smallint", "dyadic"].index(kind))
    for _ in range(300):
        lv = gv.path(rng, int(rng.integers(1, 5)), int(rng.integers(0, 40)), hi=int(rng.integers(3, 80)),
                     avg_deg=float(rng.uniform(0.5, 5)), unordered=bool(rng.integers(2)),
                     repeats=bool(rng.integers(2)))
        k, v = gv.value_map(rng, lv[0][0], rng.random(), kind)
        assert _same(vo.propagate(k, v, [(s, r) for s, r, _ in lv]), gv.formula_propagate(k, v, lv))
        s, r, d = lv[-1]
        k2, v2 = gv.value_map(rng, d, rng.random(), kind) if d.size else gv.value_map(rng, s, 0.5, kind)
        for fn in ("min", "max", "sum", "avg"):
            assert _same(vo.level_agg(fn, k2, v2, s, r), gv.formula_level_agg(fn, k2, v2, s, r)), fn


def test_int_maps_agree_in_every_completion_order():
    rng = np.random.default_rng(7)
    for _ in range(60):
        lv = gv.path(rng, int(rng.integers(1, 4)), int(rng.integers(4, 40)), hi=30)
        k, v = gv.value_map(rng, lv[0][0], 0.7, "int")
        levels = [(s, r) for s, r, _ in lv]
        first = vo.propagate(k, v, levels)
        for order in itertools.permutations(range(4)):
            assert _same(vo.propagate(k, v, levels, order), first), order


def test_float_order_is_visible():
    """Why the device fixes Go's in-order completion: the same float map merges differently in another order."""
    keys = np.array([1, 2, 3, 4], np.uint64)
    vals = np.array([1e308, 1e308, -1e308, 1.0])
    levels = [(keys, [[9], [9], [9], [9]])]
    a = vo.propagate(keys, vals, levels, (0, 1, 2, 3))[1][0]
    b = vo.propagate(keys, vals, levels, (2, 3, 0, 1))[1][0]
    assert a != b


def test_fold_rules_at_the_edges():
    """clamp after every step of a range and at every merge, NaN to +0, later equal values winning min / max."""
    f = np.finfo(np.float64).max
    k = np.array([1, 2, 3, 4, 5, 6, 7, 8], np.uint64)
    v = np.array([f, f, -f, np.nan, 1.0, 2.0, 3.0, 4.0])
    got = vo.propagate(k, v, [(k, [[20], [20], [20], [21], [21], [22], [22], [22]])])
    # nrows 8: ranges {1,2} {3,4} {5,6} {7,8}
    assert got[0].tolist() == [20, 21, 22]
    assert got[1].tolist() == [0.0, 1.0, 9.0]  # clamp(f + f) = f, f + -f = 0; NaN -> 0, 0 + 1; 2 + 3 + 4
    _, mn = vo.level_agg("min", np.array([1, 2], np.uint64), np.array([0.0, -0.0]), [9], [[1, 2]])
    assert np.signbit(mn[0])  # 0.0 < -0.0 is false: the later -0.0 wins
    _, mx = vo.level_agg("max", np.array([1, 2], np.uint64), np.array([np.nan, 1.0]), [9], [[1, 2]])
    assert mx[0] == 0.0  # NaN < 1 is false: NaN stays, and Value() clamps it to 0
    _, av = vo.level_agg("avg", np.array([1, 2], np.uint64), np.array([(1 << 62), (1 << 62)], np.int64), [9], [[1, 2]])
    assert av[0] == float(-(1 << 62))  # the int64 sum wraps before float64(int64)


def _lib():
    from dgraph_b200 import _lib
    return _lib


def _level(src, v_off, v, dest, nrows=None):
    L = _lib()
    keep = [np.asarray(x, np.uint64) if x is not None else None for x in (src, v_off, v, dest)]
    ptr = [x.ctypes.data if x is not None else None for x in keep]
    nr = len(keep[1]) - 1 if nrows is None else nrows
    return L.VarLevel(ptr[0], ptr[1], ptr[2], ptr[3], nr, 0, 0 if keep[3] is None else keep[3].size), keep


def test_propagate_argument_errors_leave_outputs_untouched():
    L = _lib()
    lib = L.load()
    k, v = np.array([1, 2], np.uint64), np.array([5, 6], np.uint64)
    good = ([1, 2], [0, 1, 2], [7, 8], [7, 8])
    cases = {
        "unknown type": dict(typ=3),
        "no levels": dict(nl=0),
        "v_off from 1": dict(level=([1, 2], [1, 1, 2], [7, 8], [7, 8])),
        "v_off decreasing": dict(level=([1, 2], [0, 2, 1], [7, 8], [7, 8])),
        "null v": dict(level=([1, 2], [0, 1, 2], None, [7, 8])),
        "null src": dict(level=(None, [0, 1, 2], [7, 8], [7, 8])),
        "null dest": dict(level=([1, 2], [0, 1, 2], [7, 8], None), ndest=2),
        "null key": dict(key=None),
        "2^32 rows": dict(nrows=1 << 32),
        "2^32 map": dict(n=1 << 32),
    }
    for name, c in cases.items():
        lv, keep = _level(*c.get("level", good), nrows=c.get("nrows"))
        if "ndest" in c:
            lv.ndest = c["ndest"]
        arr = (L.VarLevel * 1)(lv)
        ok, ov = np.full(4, SENT, np.uint64), np.full(4, SENT, np.uint64)
        n = C.c_size_t(7)
        key = k.ctypes.data if c.get("key", 1) is not None else None
        rc = lib.dgx_var_propagate(c.get("typ", 1), key, v.ctypes.data, c.get("n", 2), arr, c.get("nl", 1),
                                   ok.ctypes.data, ov.ctypes.data, 4, C.byref(n))
        assert rc == ERR_ARG, name
        assert n.value == 7 and (ok == SENT).all() and (ov == SENT).all(), name


def test_level_agg_argument_errors_leave_outputs_untouched():
    L = _lib()
    lib = L.load()
    k, v = np.array([7, 8], np.uint64), np.array([5, 6], np.uint64)
    src, off, vals = np.array([1, 2], np.uint64), np.array([0, 1, 2], np.uint64), np.array([7, 8], np.uint64)
    P = lambda a: a.ctypes.data  # noqa: E731
    cases = {
        "unknown type": (0, 2, P(k), 2, P(src), 2, P(off), P(vals)),
        "unknown fn": (1, 4, P(k), 2, P(src), 2, P(off), P(vals)),
        "negative fn": (1, -1, P(k), 2, P(src), 2, P(off), P(vals)),
        "v_off from 1": (1, 2, P(k), 2, P(src), 2, P(np.array([1, 1, 2], np.uint64)), P(vals)),
        "v_off decreasing": (1, 2, P(k), 2, P(src), 2, P(np.array([0, 2, 1], np.uint64)), P(vals)),
        "null v_off": (1, 2, P(k), 2, P(src), 2, None, P(vals)),
        "null src": (1, 2, P(k), 2, None, 2, P(off), P(vals)),
        "null v": (1, 2, P(k), 2, P(src), 2, P(off), None),
        "null key": (1, 2, None, 2, P(src), 2, P(off), P(vals)),
        "2^32 rows": (1, 2, P(k), 2, P(src), 1 << 32, P(off), P(vals)),
        "2^32 map": (1, 2, P(k), 1 << 32, P(src), 2, P(off), P(vals)),
    }
    for name, (typ, fn, key, n, s, nr, o, vv) in cases.items():
        ok, ov = np.full(4, SENT, np.uint64), np.full(4, SENT, np.uint64)
        m = C.c_size_t(7)
        rc = lib.dgx_var_level_agg(typ, fn, key, P(v), n, s, nr, o, vv, P(ok), P(ov), 4, C.byref(m))
        assert rc == ERR_ARG, name
        assert m.value == 7 and (ok == SENT).all() and (ov == SENT).all(), name


def test_empty_inputs_need_no_device():
    from dgraph_b200 import algo

    k, v = algo.PropagateVar(np.zeros(0, np.uint64), np.zeros(0, np.int64), [([1], [[2]], [2])])
    assert k.size == 0 and v.dtype == np.int64
    k, v = algo.LevelAgg("avg", np.zeros(0, np.uint64), np.zeros(0, np.float64), [1], [[2]])
    assert k.size == 0 and v.dtype == np.float64
    k, v = algo.LevelAgg("sum", [2], np.array([3], np.int64), [1, 5], [[], []])
    assert k.size == 0


def test_launch_plan():
    assert vp.K["LEVEL"] == 9 and vp.K["AGG"] == 4 and vp.K["SORT_PER_PASS"] == 3
    assert vp.passes(0) == 1 and vp.passes(64) == 1 and vp.passes(65) == 2 and vp.passes(1 << 22) == 3
    assert vp.propagate_launches(0, [10, 10]) == 0
    assert vp.propagate_launches(3, [64, 65]) == (9 + 3) + (9 + 6)
    assert vp.level_agg_launches(1, 1, 1) == 4 and vp.level_agg_launches(1, 0, 1) == 0


def test_reference_answers_on_the_fixture():
    """The reference's nine value-variable tests on query/common_test.go's data (tests/golden/valvar_common.json):
    the restatement propagates and aggregates, the rest is computed test-side as Go does."""
    import valvar_golden as vg

    vg.check(vg.replay(lambda k, v, lv: vo.propagate(k, v, [(s, r) for s, r, _ in lv]), vo.level_agg))
