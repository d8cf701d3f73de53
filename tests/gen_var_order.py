"""An independent formula for ordering a uid matrix by a value variable, and random cases for it.

Python's `sorted` is stable and Go's pdqsort is not, so the formula cannot name Go's permutation of tied values.  It
predicts what any correct answer must hold, and the exact rows where only one answer is correct:
- a row whose W (its dest-filtered uids with a map entry, in row order) is empty is its dest-filtered uids, paged;
- a row whose first W entry is a bool is Go's "isn't sortable" error;
- a tier-1 row (one numeric tag, no NaN, and at most 12 entries or no tie) is W stably sorted, paged: exact;
- every other row holds W's uids as a multiset (before paging), and where byValue.Less is a strict weak order (no NaN,
  and no two entries each Less than the other) its sequence of values is the sorted one, position by position up
  to equivalence, so each page holds the values it must;
- the new dest is the dest values some output row holds: exact without paging, and over the rows as given otherwise.
"""
from __future__ import annotations

import functools
import math
import struct

import numpy as np

T_INT, T_FLOAT, T_BOOL, T_NIL = 1, 2, 3, 4
GO_TID = {T_INT: 2, T_FLOAT: 3, T_BOOL: 4, T_NIL: 0}


def f64(w):
    return struct.unpack("<d", struct.pack("<Q", int(w)))[0]


def i64(w):
    return struct.unpack("<q", struct.pack("<Q", int(w)))[0]


def value(tag, w):
    """The Python value of a tagged word: int, float, bool or None."""
    return {T_INT: i64, T_FLOAT: f64, T_BOOL: lambda x: bool(x), T_NIL: lambda x: None}[tag](w)


def less_go(a, b):
    """types.less with mismatchedLess over (tag, value) pairs: int/float meet as floats, other mismatches by Go's type
    id, a bool pair is never less."""
    (ta, va), (tb, vb) = a, b
    if ta != tb:
        if ta in (T_INT, T_FLOAT) and tb in (T_INT, T_FLOAT):
            return float(va) < float(vb)
        return GO_TID[ta] < GO_TID[tb]
    if ta in (T_INT, T_FLOAT):
        return va < vb
    return False


def equal_go(a, b):
    return a[0] == b[0] and a[0] != T_NIL and a[1] == b[1]  # Python: -0.0 == 0.0, NaN != NaN


def Less(a, b, desc):
    """byValue.Less."""
    if a[0] == T_NIL and b[0] == T_NIL:
        return desc
    if a[0] == T_NIL:
        return False
    if b[0] == T_NIL:
        return True
    if equal_go(a, b):
        return False
    return (not less_go(a, b)) if desc else less_go(a, b)


def page(xs, count, offset):
    """x.PageRange applied to a list."""
    n = len(xs)
    if n == 0 or (count == 0 and offset == 0):
        return list(xs)
    if count < 0:
        c = max(count, -n)
        return list(xs[((n + c) % n + n) % n:])
    s = max(offset, 0)
    if s > n:
        return []
    return list(xs[s:] if count == 0 else xs[s:s + count])


def is_nan(v):
    return v[0] == T_FLOAT and isinstance(v[1], float) and math.isnan(v[1])


def tier1(vals):
    """One numeric tag, no NaN, and at most 12 entries or no two equal values."""
    tags = {t for t, _ in vals}
    if len(tags) != 1 or not tags <= {T_INT, T_FLOAT} or any(is_nan(v) for v in vals):
        return False
    return len(vals) <= 12 or len({v for _, v in vals}) == len(vals)


def weak_order(vals, desc):
    """Whether byValue.Less is a strict weak order on the row: no NaN, and no two entries each Less than the other
    (for desc: two nils, two unequal bools, or an int and a float of one numeric value)."""
    if any(is_nan(v) for v in vals):
        return False
    distinct = {}
    for v in vals:
        distinct[(v[0], v[1], math.copysign(1.0, v[1]) if v[0] == T_FLOAT else 0)] = v
    cnt = {}
    for v in vals:
        cnt[v] = cnt.get(v, 0) + 1
    ds = list(distinct.values())
    for i, a in enumerate(ds):
        for b in ds[i:]:
            if a is b and cnt.get(a, 0) < 2 and a[0] != T_NIL:
                continue
            if a is b and a[0] == T_NIL and sum(t == T_NIL for t, _ in vals) < 2:
                continue
            if Less(a, b, desc) and Less(b, a, desc):
                return False
    return True


class Prediction:
    def __init__(self):
        self.error = None
        self.rows = []  # per row: ("exact", uids) or ("multiset", W uids, expected values or None, vals by uid)
        self.dest = None  # exact new dest, or None (then it is the dest values the returned rows hold)
        self.dest_set = None
        self.count = self.offset = 0


def map_dict(m):
    """uid -> (tag, value) of a map in the forms algo.OrderByVar takes; None for a nil map."""
    if m is None:
        return None
    if len(m) == 3:
        return {int(k): (int(t), value(int(t), w)) for k, w, t in zip(m[0], m[1], m[2])}
    vals = np.asarray(m[1])
    t = T_INT if vals.dtype == np.int64 else T_FLOAT
    return {int(k): (t, (int(v) if t == T_INT else float(v))) for k, v in zip(m[0], vals)}


def formula(m, desc, dest, rows, count=0, offset=0):
    P = Prediction()
    P.count, P.offset = count, offset
    mp = map_dict(m)
    if mp is None:
        P.error = "nil"
        return P
    ds = {int(x) for x in dest}
    P.dest_set = ds
    paged = count != 0 or offset != 0
    exact_dest = True
    for r in rows:
        U = [int(x) for x in r if int(x) in ds]
        W = [x for x in U if x in mp]
        if not W:
            P.rows.append(("exact", page(U, count, offset)))
            continue
        vals = [mp[x] for x in W]
        if vals[0][0] == T_BOOL:
            P.error = "bool"
            return P
        if tier1(vals):
            P.rows.append(("exact", page(sorted(W, key=lambda x: mp[x][1], reverse=bool(desc)), count, offset)))
            continue
        want = None
        if weak_order(vals, desc):
            key = functools.cmp_to_key(lambda a, b: -1 if Less(a, b, desc) else (1 if Less(b, a, desc) else 0))
            want = sorted(vals, key=key)
        P.rows.append(("multiset", W, want, {x: mp[x] for x in W}))
        if paged:
            exact_dest = False
    if exact_dest:
        hit = set()
        for kind, *rest in P.rows:
            hit.update(rest[0])
        P.dest = sorted(hit)
    return P


def check(P, got_rows, got_dest, desc):
    """Whether (rows, dest) an implementation returned satisfies the prediction: raises AssertionError otherwise."""
    assert len(got_rows) == len(P.rows)
    for i, (pred, got) in enumerate(zip(P.rows, got_rows)):
        got = [int(x) for x in got]
        if pred[0] == "exact":
            assert got == pred[1], (i, got, pred[1])
            continue
        _, W, want, byuid = pred
        assert len(set(got)) == len(got) and set(got) <= set(W), (i, "uids")
        n = len(W)
        if P.count == 0 and P.offset == 0:
            assert sorted(got) == sorted(W), (i, "multiset")
        exp = page(list(range(n)), P.count, P.offset)
        assert len(got) == len(exp), (i, "page length")
        if want is not None:
            for pos, x in zip(exp, got):  # position pos of the sorted row holds a value equivalent to want[pos]
                a, b = byuid[x], want[pos]
                if a[0] == b[0] == T_NIL:  # the one nil a weak order admits for desc is Less than itself
                    continue
                assert not Less(a, b, desc) and not Less(b, a, desc), (i, pos, a, b)
    dest = [int(x) for x in got_dest]
    if P.dest is not None:
        assert dest == P.dest, ("dest", dest, P.dest)
    else:
        hit = sorted({int(x) for r in got_rows for x in r} & P.dest_set)
        assert dest == hit, ("dest", dest, hit)


# ---- random cases ---------------------------------------------------------------------------------------------------

def _word(tag, v):
    if tag == T_INT:
        return int(np.array([v], np.int64).view(np.uint64)[0])
    if tag == T_FLOAT:
        return int(np.array([v], np.float64).view(np.uint64)[0])
    if tag == T_BOOL:
        return int(bool(v))
    return 0


FLOATS = [0.0, -0.0, 1.5, -1.5, 2.0, float("nan"), 1e300, -1e300, 3.0, 0.25]


def random_map(rng, keys, kind):
    """A map over `keys` in one of the forms: "int", "float" (typed) or "math" (tagged, nil / bool / NaN / -0.0)."""
    k = np.array(sorted(keys), np.uint64)
    nv = int(rng.integers(1, 6))  # few distinct values: heavy ties
    if kind == "int":
        return k, rng.integers(-nv, nv + 1, k.size).astype(np.int64)
    if kind == "float":
        pool = [FLOATS[i] for i in rng.choice(len(FLOATS), size=nv)]
        if rng.random() < 0.5:
            pool = [p for p in pool if not math.isnan(p)] or [0.0]
        return k, np.array([pool[i] for i in rng.integers(0, len(pool), k.size)], np.float64)
    tags = rng.choice([T_INT, T_FLOAT, T_BOOL, T_NIL], size=k.size, p=rng.dirichlet(np.ones(4)))
    words = []
    for t in tags:
        if t == T_INT:
            words.append(_word(t, int(rng.integers(-nv, nv + 1))))
        elif t == T_FLOAT:
            words.append(_word(t, FLOATS[int(rng.integers(0, len(FLOATS)))]))
        elif t == T_BOOL:
            words.append(int(rng.integers(0, 2)))
        else:
            words.append(0)
    return k, np.array(words, np.uint64), tags.astype(np.uint8)


def random_case(rng, max_rows=6, max_len=80, universe=160):
    """(map, desc, dest, rows, count, offset) with heavy ties, nils, bools, NaN, -0.0, negative counts and offsets past
    the end."""
    U = np.arange(1, universe + 1, dtype=np.uint64)
    dest = np.sort(rng.choice(U, size=int(rng.integers(0, universe)), replace=False))
    mk = rng.choice(U, size=int(rng.integers(0, universe)), replace=False)
    kind = rng.choice(["int", "float", "math"])
    m = random_map(rng, mk.tolist(), kind)
    if kind == "math" and rng.random() < 0.7:  # a bool first in W is an error: keep most cases sortable
        k, w, t = m
        t = np.where(t == T_BOOL, T_NIL, t).astype(np.uint8) if rng.random() < 0.5 else t
        m = (k, np.where(t == T_NIL, 0, w).astype(np.uint64), t)
    rows = []
    for _ in range(int(rng.integers(0, max_rows + 1))):
        n = int(rng.integers(0, max_len + 1))
        rows.append(np.sort(rng.choice(U, size=min(n, universe), replace=False)))
    count = int(rng.choice([0, 0, 1, 3, 10, 100, -1, -4, -1000]))
    offset = int(rng.choice([0, 0, 1, 5, 50, 1000, -3]))
    return m, bool(rng.random() < 0.5), dest, rows, count, offset
