"""An independent formula for the compare functions, written from Go's rules with Python / numpy primitives, and a
seeded case generator weighted to their corners.  TEST INFRASTRUCTURE ONLY: it cross-checks compare_oracle.c, the
line-by-line restatement, and gives the GPU tests their inputs.

The rules (types/compare.go, types/sort.go): ge is not Less(v, a), le not Less(a, v), gt Less(a, v), lt Less(v, a), eq
Equal(v, a), between ge(v, a) and le(v, b); Less of a bool is an error, which makes every op but eq false.  Floats
follow IEEE (every comparison with NaN false, -0 == +0), datetimes the instant (seconds, then nanoseconds), strings
Python's bytes order (unsigned bytewise, a proper prefix less).
"""
from __future__ import annotations

import numpy as np

from dgraph_b200 import algo

INT, FLOAT, BOOL, TIME, STR = algo.VAL_INT64, algo.VAL_FLOAT64, algo.VAL_BOOL, algo.VAL_DATETIME, algo.VAL_STRING
TYPES = (INT, FLOAT, BOOL, TIME, STR)
OPS = ("le", "ge", "lt", "gt", "eq", "between")


def _vec(typ, vals):
    """Values as numpy keys: float64 for floats, int64 for ints and bools, (sec, nsec) pairs, bytes objects."""
    if typ == FLOAT:
        return np.asarray(vals, np.float64)
    if typ in (INT, BOOL):
        return np.asarray([int(v) for v in vals], np.int64)
    if typ == TIME:
        return [(int(s), int(n)) for s, n in vals]
    return [v.encode() if isinstance(v, str) else bytes(v) for v in vals]


def _less(typ, x, a):
    """Less(x, a) elementwise against one argument; None where Go errors."""
    if typ == BOOL:
        return None
    if typ in (INT, FLOAT):
        return x < a
    return np.asarray([xi < a for xi in x], bool)


def op_mask(typ, op, vals, args) -> np.ndarray:
    """CompareVals / CompareBetween of every value against the arguments (eq: any of them)."""
    x = _vec(typ, vals)
    n = len(vals)
    A = _vec(typ, args)
    if op == "eq":
        m = np.zeros(n, bool)
        for a in A:
            if typ in (INT, FLOAT):
                m |= x == a
            elif typ == BOOL:
                m |= (x != 0) == (a != 0)
            else:
                m |= np.asarray([xi == a for xi in x], bool)
        return m
    if typ == BOOL:
        return np.zeros(n, bool)

    def lt(p, q):  # Less(p, q) with p or q the vector
        if typ in (INT, FLOAT):
            return p < q
        if isinstance(p, list):
            return np.asarray([pi < q for pi in p], bool)
        return np.asarray([p < qi for qi in q], bool)

    if op == "ge":
        return ~lt(x, A[0])
    if op == "le":
        return ~lt(A[0], x)
    if op == "gt":
        return lt(A[0], x)
    if op == "lt":
        return lt(x, A[0])
    return ~lt(x, A[0]) & ~lt(A[1], x)  # between


def compare_uids(typ, uids, values, bad, op, args, cands):
    """(dest, row lengths) or None (a candidate owns a bad value)."""
    pos = {int(u): i for i, u in enumerate(uids)}
    rl = np.zeros(len(cands), np.uint32)
    for i, c in enumerate(cands):
        k = pos.get(int(c))
        if k is None or not values[k]:
            continue
        if bad is not None and any(bad[k]):
            return None
        rl[i] = int(op_mask(typ, op, values[k], args).sum())
    return np.asarray(cands, np.uint64)[rl > 0], rl


def compare_rows(typ, uids, values, bad, op, args, rows, row_arg):
    pos = {int(u): i for i, u in enumerate(uids)}
    out = []
    for r, row in enumerate(rows):
        k = int(row_arg[r])
        if k == algo.CMP_NO_ARG:
            out.append(np.asarray(row, np.uint64))
            continue
        a = args[k:k + 2] if op == "between" else args[k:k + 1]
        kept = []
        for u in row:
            i = pos.get(int(u))
            if i is None:
                continue
            good = [v for j, v in enumerate(values[i]) if bad is None or not bad[i][j]]
            if good and op_mask(typ, op, good, a).any():
                kept.append(int(u))
        out.append(np.asarray(kept, np.uint64))
    return out


# ---- seeded cases ----------------------------------------------------------------------------------------------
_FLOATS = [0.0, -0.0, float("nan"), float("inf"), -float("inf"), 1.5, -1.5, 1e308, -1e-308, 5e-324, 2.0 ** 53]
_INTS = [0, 1, -1, 2 ** 63 - 1, -2 ** 63, 2 ** 62, -(2 ** 62), 42]
_TIMES = [(0, 0), (0, 1), (-1, 999999999), (-14516064000, 0), (1262304000, 0), (1262304000, 500), (-1, 0),
          (253402300799, 999999999)]
_STRS = [b"", b"a", b"ab", b"abc", b"\x00", b"a\x00", b"\xff", b"\x80a", b"\xc3\xa9", b"abcdefghijklmnop",
         b"abcdefghijklmnopq", b"Alice", b"alice"]


def rand_value(rng, typ):
    if typ == FLOAT:
        return _FLOATS[rng.integers(len(_FLOATS))] if rng.random() < 0.6 else float(rng.normal() * 10)
    if typ == INT:
        return _INTS[rng.integers(len(_INTS))] if rng.random() < 0.5 else int(rng.integers(-50, 50))
    if typ == BOOL:
        return bool(rng.integers(2))
    if typ == TIME:
        if rng.random() < 0.5:
            return _TIMES[rng.integers(len(_TIMES))]
        return (int(rng.integers(-15000000000, 2000000000)), int(rng.integers(0, 3)) * 333333333)
    if rng.random() < 0.5:
        return _STRS[rng.integers(len(_STRS))]
    n = int(rng.integers(0, 40))
    return bytes(rng.choice([0, 97, 98, 255], n).astype(np.uint8))


def rand_case(rng, typ=None, op=None, nuids=None):
    """(typ, uids, values, bad, op, args, cands): a column, a UidList and a call."""
    typ = TYPES[rng.integers(len(TYPES))] if typ is None else typ
    op = OPS[rng.integers(len(OPS))] if op is None else op
    n = int(rng.integers(0, 12)) if nuids is None else nuids
    uids = np.unique(rng.integers(1, 4 * n + 8, n).astype(np.uint64))
    values = [[rand_value(rng, typ) for _ in range(int(rng.integers(0, 4)))] for _ in uids]
    bad = None
    if rng.random() < 0.15:
        bad = [[bool(rng.random() < 0.1) for _ in vs] for vs in values]
    nargs = 2 if op == "between" else (int(rng.integers(1, 5)) if op == "eq" else 1)
    args = [rand_value(rng, typ) for _ in range(nargs)]
    if nargs and rng.random() < 0.3:  # an argument equal to a stored value
        stored = [v for vs in values for v in vs]
        if stored:
            args[0] = stored[rng.integers(len(stored))]
    cands = np.unique(np.concatenate([uids[rng.random(uids.size) < 0.7],
                                      rng.integers(1, 4 * n + 8, 3).astype(np.uint64)])).astype(np.uint64)
    return typ, uids, values, bad, op, args, cands


def column(typ, uids, values, bad):
    return algo.ValColumn(typ, uids, values, bad)
