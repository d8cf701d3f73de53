"""Random @filter cases and an independent formula for them (no Go restatement): D0[i] is in D1 iff the tree holds at
D0[i] (a LIST leaf by membership, a COUNT leaf by comparing its count, AND / OR / NOT as Python's all / any / not);
rows keep their values in D1, then slice by the page rule; the new dest is D1 without paging and the union of the
kept rows with it.  sg_filter_oracle.c restates Go's code; tests check that the two agree.

A case is (tree, leaves, d0, rows, count, offset) in the shapes algo.SubgraphFilter takes.
"""
from __future__ import annotations

import operator

import numpy as np

CMPS = {"le": operator.le, "ge": operator.ge, "lt": operator.lt, "gt": operator.gt, "eq": operator.eq}
# first / offset pairs at every PageRange edge, for rows of a few values
PAGES = [(0, 0), (1, 0), (2, 0), (3, 1), (0, 1), (0, 2), (0, 7), (10, 0), (1, 5), (-1, 0), (-2, 0), (-3, 4),
         (-7, 0), (0, -1), (2, -3), (-2**31, 0), (2**31 - 1, 0), (0, 2**31 - 1), (5, 2**31 - 1), (-1, -5)]


def count_of(lf, i):
    if lf[0] == "count":
        return int(lf[3][i])
    return int(lf[3][i + 1]) - int(lf[3][i])


def holds(t, leaves, sets, i, x):
    if isinstance(t, (int, np.integer)):
        lf = leaves[t]
        if lf[0] == "list":
            return x in sets[t]
        return CMPS[lf[1]](count_of(lf, i), int(lf[2]))
    if t[0] == "not":
        return not holds(t[1], leaves, sets, i, x)
    vals = (holds(c, leaves, sets, i, x) for c in t[1])
    return all(vals) if t[0] == "and" else any(vals)


def page(r, count, offset):
    if count < 0:
        return r[max(len(r) + count, 0):]
    r = r[max(offset, 0):]
    return r[:count] if count > 0 else r


def formula(tree, leaves, d0, rows, count=0, offset=0):
    """(rows, counts, dest) by the per-D0 rule, over Python ints and sets."""
    sets = [set(int(u) for u in lf[1]) if lf[0] == "list" else None for lf in leaves]
    d1 = [int(x) for i, x in enumerate(d0) if holds(tree, leaves, sets, i, int(x))]
    s1 = set(d1)
    out = [[int(y) for y in r if int(y) in s1] for r in rows]
    if count != 0 or offset != 0:
        out = [page(r, count, offset) for r in out]
        dest = sorted(set().union(*[set(r) for r in out])) if out else []
    else:
        dest = d1
    return out, [len(r) for r in out], dest


def _sorted_subset(rng, universe, p):
    return np.sort(universe[rng.random(universe.size) < p]).astype(np.uint64)


def random_tree(rng, nleaves, depth=0):
    if depth >= 4 or rng.random() < 0.3 + 0.15 * depth:
        return int(rng.integers(nleaves))
    r = rng.random()
    if r < 0.25:
        return ("not", random_tree(rng, nleaves, depth + 1))
    return ("and" if r < 0.6 else "or", [random_tree(rng, nleaves, depth + 1) for _ in range(rng.integers(1, 4))])


def random_leaves(rng, universe, n0, k):
    leaves = []
    for _ in range(k):
        r = rng.random()
        if r < 0.55:  # literal or function leaves, reaching outside D0, sometimes empty
            leaves.append(("list", _sorted_subset(rng, universe, rng.choice([0.0, 0.1, 0.5, 0.9]))))
        elif r < 0.8:
            leaves.append(("count", str(rng.choice(list(CMPS))), int(rng.integers(-1, 4)),
                           rng.integers(0, 4, size=n0).astype(np.uint32)))
        else:
            off = np.concatenate([[rng.integers(0, 50)], rng.integers(0, 3, size=n0)]).cumsum().astype(np.uint64)
            leaves.append(("len", str(rng.choice(list(CMPS))), int(rng.integers(-1, 3)), off))
    return leaves


def random_case(rng, max_u=60):
    """A small case: D0 (sometimes empty), rows partly outside D0, 1-5 leaves, a tree of depth up to 4 with nested
    NOT, and a first / offset pair from PAGES or a random one."""
    universe = np.arange(1, int(rng.integers(1, max_u)) + 1, dtype=np.uint64)
    d0 = _sorted_subset(rng, universe, rng.choice([0.0, 0.3, 0.7, 1.0]))
    rows = []
    for _ in range(int(rng.integers(0, 7))):
        if rng.random() < 0.6 and d0.size:
            rows.append(np.sort(rng.choice(d0, size=int(rng.integers(0, d0.size + 1)), replace=False)))
        else:
            rows.append(_sorted_subset(rng, universe, rng.random()))
    k = int(rng.integers(1, 6))
    leaves = random_leaves(rng, universe, d0.size, k)
    tree = random_tree(rng, k)
    count, offset = PAGES[int(rng.integers(len(PAGES)))] if rng.random() < 0.7 else \
        (int(rng.integers(-4, 5)), int(rng.integers(-2, 5)))
    return tree, leaves, d0, rows, count, offset


def big_case(rng, nrows, nvals, n0, lists=(100_000, 1_000_000, 500_000), first=10, universe=None):
    """A C19a-shaped case: nrows rows of about nvals values in all over a universe of about 4 n0, D0 of n0 values,
    and the tree AND(COUNT > 1, OR(LIST a, LIST b), NOT(LIST c)) with first: `first`."""
    U = universe or 4 * n0
    d0 = np.unique(rng.integers(1, U, size=n0 + n0 // 6, dtype=np.uint64))  # about n0 distinct values
    per = max(1, nvals // max(nrows, 1))
    lens = rng.integers(0, 2 * per + 1, size=nrows)
    off = np.zeros(nrows + 1, np.uint64)
    np.cumsum(lens, out=off[1:])
    vals = rng.integers(1, U, size=int(off[-1]), dtype=np.uint64)
    rows = []
    for i in range(nrows):
        r = np.unique(vals[int(off[i]):int(off[i + 1])])
        rows.append(r)
    la, lb, lc = (np.unique(rng.integers(1, U, size=n, dtype=np.uint64)) for n in lists)
    cnt = rng.integers(0, 4, size=d0.size).astype(np.uint32)
    leaves = [("count", "gt", 1, cnt), ("list", la), ("list", lb), ("list", lc)]
    tree = ("and", [0, ("or", [1, 2]), ("not", 3)])
    return tree, leaves, d0, rows, first, 0
