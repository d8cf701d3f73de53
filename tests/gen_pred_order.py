"""An independent formula for ordering a uid matrix by a predicate's values without its index, and random cases.

Go's pdqsort is not stable, so the formula names Go's answer only for rows where any correct sort gives it: W (the
row's dest uids with a value) of at most 12 entries with no NaN (pdqsort runs insertionSort, stable under a strict
weak order), or W whose sort keys are all distinct (the order is unique).  Those rows are W ordered by np.lexsort --
ranks of the values, then the row position, so ties keep row order -- then N (the dest uids without a value, or with
a bad one) in row order, then x.PageRange(count, offset, |U|).  For every other row `check` holds the answer to what
any correct one must be: before paging, W's uids as a multiset in value order (up to ties) and N as it is.
"""
from __future__ import annotations

import struct

import numpy as np

from dgraph_b200 import algo

T_INT, T_FLOAT, T_TIME, T_STR = algo.VAL_INT64, algo.VAL_FLOAT64, algo.VAL_DATETIME, algo.VAL_STRING
TYPES = (T_INT, T_FLOAT, T_TIME, T_STR)
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1


def page_range(count, offset, n):
    """x.PageRange (x/x.go)."""
    if n == 0 or (count == 0 and offset == 0):
        return 0, n
    if count < 0:
        c = max(count, -n)
        return ((n + c) % n + n) % n, n
    s = max(offset, 0)
    if s > n:
        return n, n
    return s, n if count == 0 else min(s + count, n)


class ListPredicate(ValueError):
    pass


def _values(col):
    """uid -> (values, bad flags) of a ValColumn, values as Python objects: int, float, (sec, nsec) or bytes."""
    out = {}
    bad = col.bad
    for i, u in enumerate(col.uid.tolist()):
        lo, hi = int(col.val_off[i]), int(col.val_off[i + 1])
        vs = []
        for j in range(lo, hi):
            if col.type == T_STR:
                b0, b1 = int(col.str.byte_off[j]), int(col.str.byte_off[j + 1])
                vs.append(bytes(col.str.bytes[b0:b1]))
            elif col.type == T_INT:
                vs.append(int(np.asarray(col.word[j]).view(np.int64)))
            elif col.type == T_FLOAT:
                vs.append(float(np.asarray(col.word[j]).view(np.float64)))
            else:
                vs.append((int(np.asarray(col.word[j]).view(np.int64)), int(col.nsec[j])))
        out[u] = (vs, [bool(bad[j]) for j in range(lo, hi)] if bad is not None else [False] * (hi - lo))
    return out


def _split(col, dest, rows):
    """Per row (U, W uids, W values, N)."""
    vals = _values(col)
    ds = set(np.asarray(dest, np.uint64).tolist())
    res = []
    for r in rows:
        U = [x for x in np.asarray(r, np.uint64).tolist() if x in ds]
        wu, wv, N = [], [], []
        for x in U:
            vs, bs = vals.get(x, ([], []))
            if len(vs) > 1:
                raise ListPredicate(x)
            if len(vs) == 0 or bs[0]:
                N.append(x)
            else:
                wu.append(x)
                wv.append(vs[0])
        res.append((U, wu, wv, N))
    return res


def _ranks(typ, wv):
    """Dense ranks of the values under Go's order (equal values share a rank); NaN gets its own rank -1."""
    if typ == T_FLOAT:
        keys = [v + 0.0 for v in wv]  # -0.0 folds onto +0.0
        fin = sorted({k for k in keys if k == k})
        idx = {k: i for i, k in enumerate(fin)}
        return np.asarray([idx[k] if k == k else -1 for k in keys], np.int64)
    uniq = sorted(set(wv))
    idx = {k: i for i, k in enumerate(uniq)}
    return np.asarray([idx[k] for k in wv], np.int64)


def row_exact(typ, wv):
    """Whether any correct sort gives Go's order of this W."""
    rk = _ranks(typ, wv)
    if (rk < 0).any():
        return False
    return len(wv) <= 12 or np.unique(rk).size == len(wv)


def formula(col, desc, dest, rows, count=0, offset=0):
    """(rows, dest): each row exactly where row_exact holds, None elsewhere; dest when every row is exact, else None.
    Raises ListPredicate for a row uid with several values and ValueError for a negative count."""
    if count < 0:
        raise ValueError("negative count")
    out, exact = [], True
    for U, wu, wv, N in _split(col, dest, rows):
        if not row_exact(col.type, wv):
            out.append(None)
            exact = False
            continue
        rk = _ranks(col.type, wv)
        order = np.lexsort((np.arange(len(wv)), -rk if desc else rk)) if wv else np.zeros(0, np.int64)
        full = [wu[i] for i in order] + N
        s, e = page_range(count, offset, len(U))
        out.append(np.asarray(full[s:e], np.uint64))
    if not exact:
        return out, None
    held = set(x for r in out for x in r.tolist())
    return out, np.asarray([d for d in np.asarray(dest, np.uint64).tolist() if d in held], np.uint64)


def _sorted_ok(typ, vals, desc):
    """Whether vals are in Go's order up to ties (no NaN)."""
    rk = _ranks(typ, vals)
    if (rk < 0).any():
        return True  # an inconsistent comparator: no order to hold it to
    d = np.diff(rk)
    return bool((d <= 0).all() if desc else (d >= 0).all())


def check(case, got_rows, got_dest, full=None):
    """Asserts that (got_rows, got_dest) can be Go's answer: exact rows equal, and for the others, when unpaged (or
    given the unpaged answer `full`), W's uids in value order and N after them."""
    col, desc, dest, rows, count, offset = case
    want, wdest = formula(*case)
    split = _split(col, dest, rows)
    vals = _values(col)
    for i, (w, g) in enumerate(zip(want, got_rows)):
        g = np.asarray(g, np.uint64)
        if w is not None:
            assert np.array_equal(g, w), (i, g.tolist(), w.tolist())
            continue
        U, wu, wv, N = split[i]
        f = g if (count == 0 and offset == 0) else (None if full is None else np.asarray(full[i], np.uint64))
        if f is None:
            s, e = page_range(count, offset, len(U))
            assert g.size == e - s, i
            continue
        fl = f.tolist()
        assert sorted(fl[:len(wu)]) == sorted(wu) and fl[len(wu):] == N, i
        assert _sorted_ok(col.type, [vals[x][0][0] for x in fl[:len(wu)]], desc), i
    held = set(x for r in got_rows for x in np.asarray(r, np.uint64).tolist())
    d = np.asarray([x for x in np.asarray(dest, np.uint64).tolist() if x in held], np.uint64)
    assert np.array_equal(np.asarray(got_dest, np.uint64), d)
    if wdest is not None:
        assert np.array_equal(d, wdest)


# ---- random cases -------------------------------------------------------------------------------------------------

def _rand_value(rng, typ, pool):
    if pool is not None and rng.random() < 0.6:
        return pool[int(rng.integers(len(pool)))]
    if typ == T_INT:
        k = rng.random()
        if k < 0.1:
            return int(rng.choice([I64_MIN, I64_MAX, I64_MIN + 1, I64_MAX - 1, 0, -1]))
        return int(rng.integers(-50, 50)) if k < 0.6 else int(rng.integers(I64_MIN, I64_MAX, dtype=np.int64))
    if typ == T_FLOAT:
        k = rng.random()
        if k < 0.15:
            return float(rng.choice([0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, 5e-324, -1.5]))
        return float(rng.integers(-20, 20)) / 2 if k < 0.6 else float(rng.normal() * 1e6)
    if typ == T_TIME:
        sec = int(rng.choice([-86400 * 365 * 70, -1, 0, 1, 1_600_000_000])) + int(rng.integers(-5, 5))
        ns = int(rng.choice([0, 1, 999_999_999, 500_000_000])) if rng.random() < 0.5 else int(rng.integers(0, 10**9))
        return (sec, ns)
    k = rng.random()
    base = [b"", b"a", b"ab", b"ab\0", b"ab\0\0", b"abcdefgh", b"abcdefghX", b"abcdefghY", b"abcdefgh\0",
            b"\xff\xfe", b"\x80", b"abcdefg", b"zzzzzzzzzzzzzzzzzz1", b"zzzzzzzzzzzzzzzzzz2"]
    if k < 0.5:
        return base[int(rng.integers(len(base)))]
    n = int(rng.integers(0, 24))
    alpha = np.frombuffer(b"ab\0\xff", np.uint8) if rng.random() < 0.5 else np.arange(256, dtype=np.uint8)
    return bytes(rng.choice(alpha, n).tolist())


def random_case(rng, typ=None, nrows=None, maxrow=40):
    """(col, desc, dest, rows, count, offset) with ties, nulls, bad values and uids outside dest or the column."""
    typ = typ if typ is not None else TYPES[int(rng.integers(len(TYPES)))]
    nu = int(rng.integers(1, 120))
    universe = np.unique(rng.integers(1, 400, nu).astype(np.uint64))
    in_col = universe[rng.random(universe.size) < rng.choice([0.3, 0.8, 1.0])]
    pool = None
    if rng.random() < 0.6:
        pool = [_rand_value(rng, typ, None) for _ in range(int(rng.integers(1, 5)))]
    values = [[_rand_value(rng, typ, pool)] for _ in in_col]
    pbad = rng.choice([0.0, 0.0, 0.1, 0.5])
    bad = [[bool(rng.random() < pbad)] for _ in in_col] if pbad else None
    col = algo.ValColumn(typ, in_col, values, bad)
    dest = universe[rng.random(universe.size) < rng.choice([0.7, 1.0])]
    nrows = nrows if nrows is not None else int(rng.integers(1, 8))
    rows = []
    for _ in range(nrows):
        k = int(rng.integers(0, min(maxrow, universe.size) + 1))
        rows.append(np.sort(rng.choice(universe, k, replace=False)).astype(np.uint64))
    desc = bool(rng.random() < 0.5)
    k = rng.random()
    count, offset = (0, 0) if k < 0.4 else (int(rng.integers(0, 15)), int(rng.integers(-3, 20)))
    return col, desc, dest, rows, count, offset


def f64_bits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]
