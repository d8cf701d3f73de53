"""The reference's value-variable tests (query/query0_test.go, query3_test.go) replayed on the fixture
tests/golden/valvar_common.json, with the propagation and the level aggregation supplied by the caller (the
restatement on the CPU, the library on the GPU).  Facet variables, count(pred) and the final math() are computed
here in Python float64, as Go computes them; only transformTo and evalLevelAgg come from the callee."""
from __future__ import annotations

import json
import os

import numpy as np

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "valvar_common.json")


def load():
    with open(FIXTURE) as f:
        return json.load(f)


class Level:
    """sg.SrcUIDs, sg.uidMatrix (each row uid-sorted) and sg.DestUIDs of predicate `pred` over `src`."""

    def __init__(self, fx, pred, src):
        self.src = sorted(set(int(s) for s in src))
        e = fx["edges"][pred]
        self.rows = [sorted(t for f, t, *_ in e if f == s) for s in self.src]
        self.dest = sorted({t for r in self.rows for t in r})
        self.weight = {(f, t): w[0] for f, t, *w in e if w and w[0] is not None}

    def arrays(self):
        return (np.asarray(self.src, np.uint64), [np.asarray(r, np.uint64) for r in self.rows],
                np.asarray(self.dest, np.uint64))

    def facet_var(self):
        """`@facets(L as weight)`: each destination's weights over its edges, in row order."""
        m = {}
        for s, row in zip(self.src, self.rows):
            for t in row:
                w = self.weight.get((s, t))
                if w is not None:
                    m[t] = w if t not in m else m[t] + w
        return m


def _arr(m, dtype):
    k = sorted(m)
    return np.asarray(k, np.uint64), np.asarray([m[x] for x in k], dtype)


def _math_sum(*maps):
    """math(a + b + ...) over the union of the keys, a missing value counting as 0, left to right in float64."""
    out = {}
    for k in sorted(set().union(*maps)):
        v = float(maps[0].get(k, 0))
        for m in maps[1:]:
            v = v + float(m.get(k, 0))
        out[k] = v
    return out


def replay(propagate, level_agg):
    """propagate(keys, vals, levels) -> (keys, vals); levels are (src, rows, dest).  level_agg(fn, keys, vals, src,
    rows) -> (keys, vals).  Returns {test: {var: {uid: value}}} in the fixture's `want` shape."""
    fx = load()
    prop = lambda m, dt, lvs: dict(zip(*[a.tolist() for a in propagate(*_arr(m, dt), [l.arrays() for l in lvs])]))  # noqa: E731
    agg = lambda fn, m, dt, lv: dict(zip(*[a.tolist() for a in level_agg(fn, *_arr(m, dt), *lv.arrays()[:2])]))  # noqa: E731
    got = {}
    p1 = Level(fx, "path", [1000])
    L1 = p1.facet_var()
    got["TestLevelBasedFacetVarAggSum"] = {"sumw": agg("sum", L1, np.float64, p1)}
    p2 = Level(fx, "path", p1.dest)
    L2 = p2.facet_var()
    L1_2 = prop(L1, np.float64, [p2])
    count_follow = {u: len(Level(fx, "follow", [u]).dest) for u in p2.dest}
    got["TestLevelBasedFacetVarSum"] = {"L4": _math_sum(count_follow, L2, L1_2)}
    got["TestLevelBasedFacetVarSum1"] = {"L3": _math_sum(L1_2, L2)}
    p3 = Level(fx, "path", p2.dest)
    L3 = p3.facet_var()
    got["TestLevelBasedFacetVarSum2"] = {"L4": _math_sum(prop(L1, np.float64, [p2, p3]), prop(L2, np.float64, [p3]),
                                                         L3)}
    m1 = Level(fx, "path", [1])
    a = {1: fx["age"]["1"]}
    got["TestLevelBasedSumMix1"] = {"L2": _math_sum(prop(a, np.int64, [m1]), m1.facet_var())}
    roots = fx["anyofterms_michonne_andrea_rick"]
    f = Level(fx, "friend", roots)
    x = {u: fx["age"][str(u)] for u in f.dest if str(u) in fx["age"]}
    mm = {"n": agg("min", x, np.int64, f), "s": agg("max", x, np.int64, f)}
    got["TestQueryVarValAggMinMax"] = mm
    got["TestQueryVarValAggNestedFunc"] = mm
    s = {u: len(Level(fx, "friend", [u]).dest) for u in f.dest}
    got["TestMultiLevelAgg"] = {"sum(val(s))": agg("sum", s, np.int64, f)}
    with_friends = Level(fx, "friend", [u for u in roots if Level(fx, "friend", [u]).dest])
    got["TestMultiLevelAgg1"] = {"ss": agg("sum", s, np.int64, with_friends)}
    return got


def check(got):
    """Every published value, exactly, for the uids each test prints."""
    want = load()["want"]
    for test, vars_ in want.items():
        for var, uids in vars_.items():
            for u, w in uids.items():
                g = got[test][var].get(int(u))
                assert g is not None and g == w and type(g) is type(w), (test, var, u, g, w)
