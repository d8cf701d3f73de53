"""The reference's @filter tests on tests/golden/sg_filter_common.json (query/common_test.go's names, friend and school
edges): each test's filtered node as ProcessGraph hands it to the filter block -- D0, the uid matrix, the resolved
leaves and the tree -- and its published answer.  TEST INFRASTRUCTURE ONLY: used by tests/test_sg_filter_host.py
(restatement and formula) and tests/test_gpu_sg_filter.py (library, both forms).

Leaf resolution, as the shim does it: a literal uid(...) is a LIST of its sorted arguments; anyofterms(name, ...) is
a LIST, the fixture's term row; uid_in(pred, x) is a COUNT over row lengths, the rows of pred over D0 intersected with
{x} (handleUidPostings' Intersect = uidsPresent), compared gt 0; has(pred) and le(count(pred), n) are COUNTs over
pl.Length, pred's edge count per D0 value, compared gt 0 and le n.  A root with a function has one row, its DestUIDs.
"""
from __future__ import annotations

import json
import os

import numpy as np

_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sg_filter_common.json")
U64 = np.uint64


def load():
    with open(_PATH) as f:
        return json.load(f)


def cases(g=None):
    """(label, (tree, leaves, d0, rows, count, offset), counts_only, want) for each published answer."""
    g = g or load()
    adj = {p: {} for p in g["edges"]}
    for p, es in g["edges"].items():
        for s, d in es:
            adj[p].setdefault(s, []).append(d)
    T = {q: np.array(r, U64) for q, r in g["anyofterms"].items()}

    def arr(u):
        return np.array(sorted(u), U64)

    def rows_of(p, src):
        return [arr(adj[p].get(int(u), [])) for u in src]

    def merged(rows):
        return arr(set().union(*[set(int(x) for x in r) for r in rows]))

    def has_count(cmp, n, p, d0):  # pl.Length per D0 value
        return ("count", cmp, n, np.array([len(adj[p].get(int(u), [])) for u in d0], np.uint32))

    def uid_in(p, d0, present):  # row lengths of pred's rows intersected with uidsPresent
        lens = [len(set(adj[p].get(int(u), [])) & set(present)) for u in d0]
        return ("len", "gt", 0, np.concatenate([[0], np.cumsum(lens)]).astype(U64))

    def root(d0):
        d0 = arr(d0)
        return d0, [d0]

    def child(p, src):
        rows = rows_of(p, src)
        return merged(rows), rows

    w = g["want"]
    out = []

    def add(label, tree, leaves, node, count=0, offset=0, counts_only=False, want=None):
        out.append((label, (tree, leaves, node[0], node[1], count, offset), counts_only,
                    w[label.split("/")[0]] if want is None else want))

    people = [23, 1, 24, 25, 31]
    add("TestUidFunctionInFilter", 0, [("list", arr([1, 24]))], root(people))
    add("TestUidFunctionInFilter2", 0, [("list", arr([23, 1]))], child("friend", arr(people)))
    add("TestUidFunctionInFilter4", ("not", 0), [("list", arr([1, 31]))], root(T["Michonne Andrea"]))
    d0 = arr([1, 23, 24])
    add("TestUidInFunction", 0, [uid_in("friend", d0, [23])], root(d0))
    add("TestUidInFunction1", 0, [uid_in("school", d0, [5000])], root(d0))
    fr = child("friend", d0)
    add("TestUidInFunction2", 0, [uid_in("school", fr[0], [5000])], fr)
    mrd = T["Michonne Rick Daryl"]
    add("TestCountAtRootWithAlias4", 0, [has_count("le", 2, "friend", mrd)], root(mrd))
    add("TestHasFuncAtRootFilter", 0, [has_count("gt", 0, "friend", mrd)], root(mrd))
    f1 = child("friend", arr([1]))
    add("TestToFastJSONFilterOrFirst", ("or", [0, 1, 2]),
        [("list", T["Andrea"]), ("list", T["Glenn SomethingElse"]), ("list", T["Daryl"])], f1, count=2)
    add("TestToFastJSONFilterOrOffset", ("or", [0, 1, 2]),
        [("list", T["Andrea"]), ("list", T["Glenn Rhee"]), ("list", T["Daryl Dixon"])], f1, offset=1)
    oc = w["TestToFastJSONFilterOrCount"]
    add("TestToFastJSONFilterOrCount/count(friend)", ("or", [0, 1]), [("list", T["Andrea"]), ("list", T["Andrea Rhee"])],
        f1, counts_only=True, want={"counts": oc["counts"]})
    add("TestToFastJSONFilterOrCount/friend", 0, [("list", T["Andrea"])], f1, want={"rows": oc["rows"]})
    return out


def check(got, want, g=None):
    """got = (rows or None, counts, dest) against the published answer: names in result order, names per row,
    the node's count(uid), or the count(pred @filter) values."""
    g = g or load()
    names = {int(k): v for k, v in g["names"].items()}
    rows, counts, dest = got
    ok = True
    if "names" in want:
        ok &= [names.get(int(u)) for u in dest] == want["names"]
    if "rows" in want:
        ok &= [[names.get(int(u)) for u in r] for r in rows] == want["rows"]
    if "count" in want:
        ok &= len(dest) == want["count"]
    if "counts" in want:
        ok &= [int(c) for c in counts] == want["counts"]
    return bool(ok)
