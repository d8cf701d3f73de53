"""math() on the CPU: the restatement of evalMathTree (tests/math_oracle.c) against Go's known answers, its iteration
orders against the rules dgx_math_eval refuses by, and the library's argument errors."""
import ctypes as C

import numpy as np
import pytest

import gen_math as gm
import math_oracle as mo
from dgraph_b200 import _lib, algo

I = lambda *v: np.array(v, np.int64)  # noqa: E731
F = lambda *v: np.array(v, np.float64)  # noqa: E731
U = lambda *v: np.array(v, np.uint64)  # noqa: E731


def fw(x):
    return int(np.array([x], np.float64).view(np.uint64)[0])


def iw(x):
    return int(np.array([x], np.int64).view(np.uint64)[0])


def refused(res):
    return res[0] is None or res[4]


def leaf_key0_mixed(maps):
    return any(m is not None and len(m[0]) > 1 and int(np.asarray(m[0])[0]) == 0 for m in maps.values())


@pytest.mark.parametrize("seed", range(6))
def test_accepted_cases_do_not_depend_on_iteration_order(seed):
    rng = np.random.default_rng(1000 + seed)
    accepted = refusals = 0
    for _ in range(500):
        t, maps, r = gm.case(rng)
        if leaf_key0_mixed(maps):
            continue
        base = mo.evaluate(t, maps, r, seed=0)
        outs = [mo.evaluate(t, maps, r, seed=s) for s in range(1, 9)]
        if refused(base) or any(refused(o) for o in outs):
            refusals += 1
            continue
        accepted += 1
        for o in outs:
            assert o[0] == base[0]
            for a, b in zip(o[1:4], base[1:4]):
                assert np.array_equal(a, b), (t, maps, r)
    assert accepted > 200 and refusals > 5


def same_shard_keys(n):
    return np.array([1 + 30 * i for i in range(n)], np.uint64)  # every key in shard 1


def test_refused_partial_errors_differ_across_orders():
    k = same_shard_keys(6)
    cases = [
        (("u-", ("var", "a")), {"a": (k, I(1, 2, -2**63, 4, 5, 6))}),
        (("sqrt", ("var", "a")), {"a": (k, F(1.0, -1.0, 4.0, 9.0, -2.0, 16.0))}),
        (("<", ("var", "a"), ("var", "b")), {"a": (k, I(1, 2, 3, 4, 5, 6)), "b": (k[:3], I(0, 0, 0))}),
        (("cond", ("var", "c"), ("const", 1), ("const", 2)), {"c": (k, k.view(np.int64) * 0 + 1)}),
    ]
    cases[3][1]["c"] = (k, np.array([1, 0, 1, 0, 1, 1], np.uint64), np.array([3, 3, 1, 3, 3, 3], np.uint8))
    for t, maps in cases:
        outs = {tuple(mo.evaluate(t, maps, None, seed=s)[1].tolist()) for s in range(16)}
        assert mo.evaluate(t, maps, None, seed=0)[4]
        assert len(outs) > 1, t


def test_all_keys_failing_is_deterministic_and_empty():
    k = same_shard_keys(4)
    for s in range(8):
        res = mo.evaluate(("u-", ("var", "a")), {"a": (k, I(-2**63, -2**63, -2**63, -2**63))}, None, seed=s)
        assert res[0] == "none" and not res[4]


def test_known_answers_from_the_reference():
    # TestProcessBinary / TestProcessUnary / TestProcessBinaryBoolean / TestProcessTernary (in-scope cases)
    two = U(1, 2)
    _, k, w, t, _ = mo.evaluate(("+", ("var", "a"), ("var", "b")), {"a": (two, I(2, 3)), "b": (two, I(4, 5))})
    assert k.tolist() == [1, 2] and w.view(np.int64).tolist() == [6, 8]
    _, k, w, t, _ = mo.evaluate(("*", ("var", "a"), ("var", "b")), {"a": (two, F(2.0, 3.0)), "b": (two, I(4, 5))})
    assert w.view(np.float64).tolist() == [8.0, 15.0] and t.tolist() == [2, 2]
    _, k, w, t, _ = mo.evaluate(("/", ("var", "a"), ("var", "b")), {"a": (two, I(8, 9)), "b": (two, I(4, 0))})
    assert k.tolist() == [1] and w.view(np.int64).tolist() == [2]  # division by zero drops the key
    _, k, w, t, _ = mo.evaluate(("%", ("var", "a"), ("var", "b")), {"a": (two, F(-7.5, 7.5)), "b": (two, F(2.0, -2.0))})
    assert w.view(np.float64).tolist() == [-1.5, 1.5]
    _, k, w, t, _ = mo.evaluate(("floor", ("var", "a")), {"a": (two, F(1.5, -1.5))})
    assert w.view(np.float64).tolist() == [1.0, -2.0]
    _, k, w, t, _ = mo.evaluate(("ceil", ("var", "a")), {"a": (two, I(1, -1))})
    assert w.view(np.int64).tolist() == [1, -1] and t.tolist() == [1, 1]
    _, k, w, t, _ = mo.evaluate(("sqrt", ("var", "a")), {"a": (two, I(4, 9))})
    assert w.view(np.float64).tolist() == [2.0, 3.0]
    _, k, w, t, _ = mo.evaluate(("<", ("var", "a"), ("var", "b")), {"a": (two, I(1, 5)), "b": (two, F(2.0, 5.0))})
    assert w.tolist() == [1, 0] and t.tolist() == [3, 3]
    _, k, w, t, _ = mo.evaluate(("cond", ("<", ("var", "a"), ("const", 3)), ("var", "b"), ("const", 9)),
                             {"a": (two, I(1, 5)), "b": (U(2), I(7))})
    assert t.tolist() == [4, 1] and w.tolist() == [0, 9]  # a missing branch entry is stored as nil


def test_scalar_rules():
    z = U(0)
    # s + t, both aggregates: the left becomes a constant, the right stays a map
    assert mo.evaluate(("+", ("var", "s"), ("var", "t")), {"s": (z, I(2)), "t": (z, I(3))})[:2][0] == "map"
    # s + 1: a constant, set over the range
    kind, k, w, t, _ = mo.evaluate(("+", ("var", "s"), ("const", 1)), {"s": (z, I(2))}, U(5, 6))
    assert kind == "const" and k.tolist() == [5, 6] and w.view(np.int64).tolist() == [3, 3]
    # the constant without a range lands on uid 0
    kind, k, w, t, _ = mo.evaluate(("+", ("var", "s"), ("const", 1)), {"s": (z, I(2))})
    assert kind == "const" and k.tolist() == [0]
    # {MaxUint64: n} is the constant n
    kind, k, w, t, _ = mo.evaluate(("*", ("var", "c"), ("const", 2)), {"c": (U(2**64 - 1), I(21))}, U(4))
    assert kind == "const" and w.view(np.int64).tolist() == [42]
    # int64 boundaries
    assert mo.evaluate(("*", ("const", -2**63), ("const", -1)), {})[2].view(np.int64).tolist() == [-2**63]
    assert mo.evaluate(("*", ("const", -1), ("const", -2**63)), {})[0] is None
    assert mo.evaluate(("/", ("const", -2**63), ("const", -1)), {})[2].view(np.int64).tolist() == [-2**63]
    assert mo.evaluate(("%", ("const", -2**63), ("const", -1)), {})[2].view(np.int64).tolist() == [0]
    # cond over a constant fails
    assert mo.evaluate(("cond", ("const", 1), ("const", 1), ("const", 2)), {})[0] is None
    # mixed promotion
    kind, k, w, t, _ = mo.evaluate(("+", ("var", "a"), ("var", "b")), {"a": (U(1), I(1)), "b": (U(2), F(0.5))})
    assert t.tolist() == [2, 2] and w.view(np.float64).tolist() == [1.0, 0.5]


def _noop_outputs():
    return np.full(4, 7, np.uint64), np.full(4, 7, np.uint64), np.full(4, 7, np.uint8)


@pytest.mark.parametrize("bad", ["op", "child", "leaf", "ctag", "size", "dag", "type"])
def test_argument_errors_leave_outputs_untouched(bad):
    names = {}
    nodes = algo.math_program(("+", ("var", "a"), ("const", 1)), names)
    k = U(1, 2)
    w = I(1, 2).view(np.uint64)
    leaf = (_lib.MathLeaf * 1)(_lib.MathLeaf(k.ctypes.data, w.ctypes.data, None, None, 2, 1, 0))
    nn = len(nodes)
    if bad == "op":
        nodes[2].op = 40
    elif bad == "child":
        nodes[2].child[1] = 2
    elif bad == "leaf":
        nodes[0].leaf = 3
    elif bad == "ctag":
        nodes[1].const_tag = 3
    elif bad == "size":
        nn = 65
        nodes = nodes + [nodes[0]] * 62
    elif bad == "dag":
        nodes[2].child[1] = 0
    elif bad == "type":
        leaf[0].type = 7
    prog = (_lib.MathNode * len(nodes))(*nodes)
    ok, ow, ot = _noop_outputs()
    info = C.c_uint64(99)
    rc = _lib.load().dgx_math_eval(prog, nn, leaf, 1, None, 0, ok.ctypes.data, ow.ctypes.data, ot.ctypes.data, 4,
                                   C.byref(info))
    assert rc == _lib.DGX_ERR_ARG
    assert info.value == 99 and (ok == 7).all() and (ow == 7).all() and (ot == 7).all()


@pytest.mark.parametrize("seed", range(4))
def test_formula_agrees_with_the_restatement(seed):
    """The independent formula (gen_math.formula: Go's rules over plain dicts, refusing an error or an order-dependent
    stop) against the restatement: equal wherever it answers, and where it refuses the restatement fails, stops on
    a key that another key would have passed, or meets key 0 among other keys."""
    rng = np.random.default_rng(2000 + seed)
    answered = 0
    for _ in range(1000):
        t, maps, r = gm.case(rng, max_depth=5)
        f, o = gm.formula(t, maps, r), mo.evaluate(t, maps, r, seed=seed)
        if f is None:
            assert leaf_key0_mixed(maps) or refused(o), (t, maps, r)
            continue
        answered += 1
        assert not refused(o) and f[0] == o[0], (t, maps, r)
        for a, b in zip(f[1:], o[1:4]):
            assert np.array_equal(a, b), (t, maps, r)
    assert answered > 600


def test_launch_plan_reads_the_sources():
    import math_plan as mp

    assert mp.K["FRONT"] + mp.K["BACK"] == 7
    assert mp.launches(0) == 7 and mp.launches(10) == mp.launches(2000) < mp.launches(10**7)


def test_reference_query_answers_through_the_restatement():
    import math_golden as mg

    for name, tree, maps, r, want in mg.cases():
        kind, k, w, t, _ = mo.evaluate(tree, maps, r)
        assert mg.values(kind, k, w, t) == want, name
        assert gm.formula(tree, maps, r)[0] == kind, name
