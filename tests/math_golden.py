"""The reference's query-level math() tests on tests/golden/math_common.json (query/common_test.go's ages and friend
edges): each test's program and leaf maps as valueVarAggregation hands them to evalMathTree, and its published answer.
TEST INFRASTRUCTURE ONLY: used by tests/test_math_host.py (restatement) and tests/test_gpu_math.py (library)."""
from __future__ import annotations

import json
import os

import numpy as np

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "math_common.json")


def load():
    with open(_PATH) as f:
        return json.load(f)


def _map(d, dtype=np.int64):
    ks = sorted(int(k) for k in d)
    return np.array(ks, np.uint64), np.array([d[str(k)] if str(k) in d else d[k] for k in ks], dtype)


def cases(g=None):
    """(name, tree, maps, range_uids, want {uid: value}) for each test of the fixture."""
    g = g or load()
    roots = g["anyofterms_michonne_andrea_rick"]
    age = {int(k): v for k, v in g["age"].items()}
    friends = {}
    for s, d in g["friend"]:
        friends.setdefault(s, []).append(d)
    root_ages = {str(u): age[u] for u in roots if u in age}  # ageVar as age over the root block
    double = ("*", ("var", "ageVar"), ("const", 2))
    out = []
    for name in ("TestMathVarAlias", "TestMathVarAlias2", "TestMathVar3"):
        out.append((name, double, {"ageVar": _map(root_ages)}, np.array(roots, np.uint64), g["want"][name]["a"]))
    # x2 as sum(val(x)) and c as count(friend) per row of the var block over uid(me); an empty me for Ceil1
    me = [1]
    x2 = {str(u): sum(age[f] for f in friends.get(u, []) if f in age) for u in me}
    c = {str(u): len(friends.get(u, [])) for u in me}
    ceil2 = ("ceil", ("/", ("*", ("const", 1.0), ("var", "x2")), ("var", "c")))
    out.append(("TestMathCeil1", ("ceil", ("/", ("var", "x2"), ("var", "c"))),
                {"x2": _map({}), "c": _map({})}, np.zeros(0, np.uint64), g["want"]["TestMathCeil1"]["ceilAge"]))
    out.append(("TestMathCeil2", ceil2, {"x2": _map(x2), "c": _map(c)}, np.array(me, np.uint64),
                g["want"]["TestMathCeil2"]["ceilAge"]))
    out.append(("TestMathAlias", ("+", ("var", "p"), ("const", 1)), {"p": _map(c)}, np.array(me, np.uint64),
                g["want"]["TestMathAlias"]["score"]))
    out.append(("TestQueryConstMathVal", ("*", ("/", ("const", 24), ("const", 8)), ("const", 3)), {},
                np.array(roots, np.uint64), g["want"]["TestQueryConstMathVal"]["a"]))
    return out


def values(kind, keys, words, tags):
    """The result as {uid: int or float}, what the query's JSON prints."""
    if kind == "none":
        return {}
    out = {}
    for k, w, t in zip(keys.tolist(), words.tolist(), tags.tolist()):
        x = np.array([w], np.uint64)
        out[str(k)] = int(x.view(np.int64)[0]) if t == 1 else float(x.view(np.float64)[0])
    return out
