"""Random math() programs and value maps for the dgx_math_eval tests: trees over every in-scope op, constants and up
to four variables, maps of int64, float64, bool and nil entries drawn from a small uid universe (so keys share shards)
with the int64 and float64 edge values, {0: v} aggregates, {MaxUint64: v} counts, empty and nil maps."""
from __future__ import annotations

import numpy as np

BIN = ["+", "-", "*", "/", "%", "min", "max"]
UN = ["u-", "sqrt", "floor", "ceil"]
CMP = ["<", ">", "<=", ">=", "==", "!="]
I64 = [0, 1, -1, 2, -2, 3, 7, -7, 2**62, -(2**62), 2**63 - 1, -(2**63), 2**31, 10**9]
F64 = [0.0, -0.0, 0.5, -0.5, 1.5, -2.25, 3.0, 1e308, -1e308, float("inf"), float("-inf"), float("nan"), 5e-324,
       -5e-324, 2.0**53, 0.1, 7.0]
INT, FLT, BOOL, NIL = 1, 2, 3, 4


def _word(rng, tag):
    if tag == INT:
        return int(np.array([I64[rng.integers(len(I64))] if rng.random() < 0.5 else int(rng.integers(-9, 10))],
                            np.int64).view(np.uint64)[0])
    if tag == FLT:
        v = F64[rng.integers(len(F64))] if rng.random() < 0.5 else float(rng.integers(-9, 10)) / 2
        return int(np.array([v], np.float64).view(np.uint64)[0])
    if tag == BOOL:
        return int(rng.integers(2))
    return 0


def value_map(rng, universe=64, size=None, tags=(INT, FLT)):
    """A tagged map (keys, words, tags) over uids 1 .. universe."""
    if size is None:
        size = int(rng.integers(0, 12))
    keys = np.sort(rng.choice(np.arange(1, universe + 1, dtype=np.uint64), size=min(size, universe), replace=False))
    tg = np.array([tags[rng.integers(len(tags))] for _ in keys], np.uint8)
    w = np.array([_word(rng, t) for t in tg], np.uint64)
    return keys, w, tg


def leaf_map(rng):
    r = rng.random()
    if r < 0.06:
        return None
    if r < 0.12:
        return np.zeros(0, np.uint64), np.zeros(0, np.uint64), np.zeros(0, np.uint8)
    if r < 0.27:  # an aggregate
        t = [INT, FLT, BOOL, NIL][rng.integers(4)] if rng.random() < 0.2 else [INT, FLT][rng.integers(2)]
        return np.zeros(1, np.uint64), np.array([_word(rng, t)], np.uint64), np.array([t], np.uint8)
    if r < 0.33:  # count(uid)
        return np.array([2**64 - 1], np.uint64), np.array([int(rng.integers(0, 50))], np.uint64), np.array([INT], np.uint8)
    tags = (INT, FLT) if rng.random() < 0.8 else (INT, FLT, BOOL, NIL)
    return value_map(rng, tags=tags)


def tree(rng, depth, nvars):
    if depth == 0 or rng.random() < 0.25:
        if rng.random() < 0.3:
            if rng.random() < 0.5:
                return ("const", int(rng.integers(-5, 6)))
            return ("const", float(F64[rng.integers(len(F64))]) if rng.random() < 0.3 else float(rng.integers(-8, 9)) / 4)
        return ("var", f"v{rng.integers(nvars)}")
    r = rng.random()
    if r < 0.45:
        return (BIN[rng.integers(len(BIN))], tree(rng, depth - 1, nvars), tree(rng, depth - 1, nvars))
    if r < 0.6:
        return (UN[rng.integers(len(UN))], tree(rng, depth - 1, nvars))
    if r < 0.85:
        return (CMP[rng.integers(len(CMP))], tree(rng, depth - 1, nvars), tree(rng, depth - 1, nvars))
    return ("cond", tree(rng, depth - 1, nvars), tree(rng, depth - 1, nvars), tree(rng, depth - 1, nvars))


def case(rng, max_depth=4):
    """(tree, maps, range_uids or None)."""
    nv = int(rng.integers(1, 5))
    t = tree(rng, int(rng.integers(1, max_depth + 1)), nv)
    while nodes(t) > 64:  # DGX_MATH_MAX_NODES
        t = tree(rng, int(rng.integers(1, max_depth + 1)), nv)
    maps = {f"v{i}": leaf_map(rng) for i in range(nv)}
    rr = rng.random()
    rng_uids = None if rr < 0.3 else np.sort(rng.choice(np.arange(1, 100, dtype=np.uint64), int(rng.integers(0, 6)),
                                                        replace=False))
    return t, maps, rng_uids


def nodes(t):
    return 1 + sum(nodes(c) for c in t[1:]) if t[0] not in ("var", "const") else 1


# ---- an independent formula: Go's rules over plain dicts, refusing where the answer is an error or order-dependent ----

MAXU64 = 2**64 - 1
_F = lambda w: np.array([w], np.uint64).view(np.float64)[0]  # noqa: E731
_W = lambda x: int(np.array([x], np.float64).view(np.uint64)[0])  # noqa: E731
_I = lambda w: w - 2**64 if w >= 2**63 else w  # noqa: E731


class Refused(Exception):
    pass


def _clamp(x):
    if np.isnan(x):
        return 0.0
    if np.isinf(x):
        return np.finfo(np.float64).max * (1 if x > 0 else -1)
    return x


def _num(v):
    """A missing or nil value is int64 0."""
    return (INT, 0) if v is None or v[0] == NIL else v


def _bin(op, a, b):
    (ta, wa), (tb, wb) = _num(a), _num(b)
    if BOOL in (ta, tb):
        return None
    if ta != tb:
        x = float(_I(wa)) if ta == INT else _F(wa)
        y = float(_I(wb)) if tb == INT else _F(wb)
        ta = FLT
    elif ta == INT:
        x, y = _I(wa), _I(wb)
        if op in ("min", "max"):
            return (INT, wa if (x < y) == (op == "min") else wb)
        if op == "+":
            r = x + y
        elif op == "-":
            r = x - y
        elif op == "*":
            r = x * y
        elif op in ("/", "%"):
            if y == 0:
                return None
            q = abs(x) // abs(y) * (1 if (x < 0) == (y < 0) else -1)  # truncated division
            r = q if op == "/" else x - q * y
            if op == "/" and r == 2**63:
                r = -(2**63)  # MinInt64 / -1 wraps
        if not -(2**63) <= r < 2**63:
            return None
        return (INT, r % 2**64)
    else:
        x, y = _F(wa), _F(wb)
    with np.errstate(all="ignore"):
        if op == "min":
            return (FLT, _W(_clamp(x if x < y else y)))
        if op == "max":
            return (FLT, _W(_clamp(y if x < y else x)))
        if op in ("/", "%") and y == 0:
            return None
        r = {"+": np.add, "-": np.subtract, "*": np.multiply, "/": np.divide, "%": np.fmod}[op](np.float64(x),
                                                                                              np.float64(y))
    return (FLT, _W(_clamp(r)))


def _un(op, a):
    t, w = _num(a)
    if t == BOOL:
        return None
    if t == INT:
        x = _I(w)
        if op == "u-":
            return None if x == -(2**63) else (INT, (-x) % 2**64)
        if op == "sqrt":
            return None if x < 0 else (FLT, _W(_clamp(np.sqrt(np.float64(x)))))
        return (INT, w)
    x = _F(w)
    with np.errstate(all="ignore"):
        if op == "sqrt" and x < 0:
            return None
        r = {"u-": np.negative, "sqrt": np.sqrt, "floor": np.floor, "ceil": np.ceil}[op](np.float64(x))
    return (FLT, _W(_clamp(r)))


def _cmp(op, a, b):
    (ta, wa), (tb, wb) = a, (b if b is not None else (NIL, 0))
    if ta == NIL and tb == NIL:
        lt = gt = eq = False
    elif ta in (INT, FLT) and tb in (INT, FLT):
        if ta == tb == INT:
            x, y = _I(wa), _I(wb)
        else:
            x = float(_I(wa)) if ta == INT else _F(wa)
            y = float(_I(wb)) if tb == INT else _F(wb)
        lt, gt, eq = x < y, y < x, x == y
    else:
        return None
    v = {"<": lt, ">": gt, "<=": lt or eq, ">=": gt or eq, "==": eq, "!=": not eq}[op]
    return (BOOL, int(v))


def _over(keys, f):
    """An Iterate over keys: every key kept, or none when every key fails; some failing is order-dependent."""
    out = {k: f(k) for k in keys}
    bad = sum(v is None for v in out.values())
    if bad and bad < len(out):
        raise Refused("some keys fail")
    return {} if bad else out


def _node(t, maps):
    """("const", v) | ("nil",) | ("map", {key: (tag, word)})."""
    op = t[0]
    if op == "const":
        v = t[1]
        return ("const", (FLT, _W(v)) if isinstance(v, float) else (INT, v % 2**64))
    if op == "var":
        m = maps.get(t[1])
        if m is None:
            return ("nil",)
        k, w, tg = (list(map(int, m[0])), list(map(int, m[1])), list(map(int, m[2]))) if len(m) == 3 else \
            (list(map(int, m[0])), list(map(int, np.ascontiguousarray(m[1]).view(np.uint64))),
             [FLT if np.asarray(m[1]).dtype == np.float64 else INT] * len(m[0]))
        d = dict(zip(k, zip(tg, w)))
        if len(d) == 1 and MAXU64 in d:
            return ("nil",) if d[MAXU64][0] == NIL else ("const", d[MAXU64])
        if len(d) > 1 and 0 in d:
            raise Refused("key 0 among other keys")
        return ("map", d)
    kids = [_node(c, maps) for c in t[1:]]
    if op in BIN:
        L, R = kids
        cl = L[1] if L[0] == "const" else None
        cr = R[1] if R[0] == "const" else None
        ml = L[1] if L[0] == "map" else {}
        mr = R[1] if R[0] == "map" else {}
        if len(ml) == 1 and 0 in ml:
            cl, ml = (ml[0] if ml[0][0] != NIL else None), {}
        elif len(mr) == 1 and 0 in mr:
            cr, mr = (mr[0] if mr[0][0] != NIL else None), {}
        if ml or mr:
            out = {}
            for k in set(ml) | set(mr):
                r = _bin(op, cl if cl else ml.get(k), cr if cr else mr.get(k))
                if r is not None:
                    out[k] = r
            return ("map", out)
        if cl and cr:
            r = _bin(op, cl, cr)
            if r is None:
                raise Refused("an error evalMathTree returns")
            return ("const", r)
        return ("nil",)
    if op in UN:
        (C,) = kids
        if C[0] == "const":
            r = _un(op, C[1])
            if r is None:
                raise Refused("an error evalMathTree returns")
            return ("const", r)
        m = C[1] if C[0] == "map" else {}
        return ("map", _over(m, lambda k: _un(op, m[k])))
    if op in CMP:
        L, R = kids
        m = L[1] if L[0] == "map" else {}
        rv = (lambda k: R[1]) if R[0] == "const" else (lambda k: R[1].get(k)) if R[0] == "map" else (lambda k: None)
        return ("map", _over(m, lambda k: _cmp(op, m[k], rv(k))))
    A, B, Cc = kids
    if A[0] != "map":
        raise Refused("cond over a constant or a nil map")

    def pick(k):
        v = A[1][k]
        if v[0] != BOOL:
            return None
        X = B if v[1] else Cc
        if X[0] == "const":
            return X[1]
        return X[1].get(k, (NIL, 0)) if X[0] == "map" else (NIL, 0)

    return ("map", _over(A[1], pick))


def formula(t, maps, range_uids=None):
    """(kind, keys, words, tags) as dgx_math_eval returns them, or None where it refuses."""
    try:
        r = _node(t, maps)
    except Refused:
        return None
    if r[0] == "map" and r[1]:
        d = r[1]
        if any(v[0] == INT for v in d.values()) and any(v[0] == FLT for v in d.values()):
            d = {k: ((FLT, _W(float(_I(v[1])))) if v[0] == INT else v) for k, v in d.items()}
        ks = sorted(d)
        return ("map", np.array(ks, np.uint64), np.array([d[k][1] for k in ks], np.uint64),
                np.array([d[k][0] for k in ks], np.uint8))
    if r[0] == "const":
        ks = [0] if range_uids is None else [int(x) for x in range_uids]
        return ("const", np.array(ks, np.uint64), np.array([r[1][1]] * len(ks), np.uint64),
                np.array([r[1][0]] * len(ks), np.uint8))
    e = np.zeros(0, np.uint64)
    return ("none", e, e.copy(), np.zeros(0, np.uint8))
