"""Value-variable inputs and an independent numpy formula for transformTo / evalLevelAgg (query/query.go).

The formula is exact where every summation order gives the same bits: int64 maps (wrapping sums on uint64) and float64
maps whose values are small dyadic rationals (every partial sum is exactly representable).  It shares no code with
the line-by-line restatement (valvar_oracle.c).
"""
from __future__ import annotations

import numpy as np

U64 = np.uint64


def sorted_uids(rng, n, hi):
    """n distinct uids in [1, hi], ascending."""
    return np.sort(rng.choice(np.arange(1, hi + 1, dtype=U64), size=min(n, hi), replace=False)).astype(U64)


def level(rng, src, nv_hi, universe, avg_deg=3.0, unordered=True, repeats=True):
    """One level over `src` (ascending): rows of Poisson(avg_deg) values drawn from `universe`, shuffled (ordered
    children keep their order) and with repeats when asked.  Returns (src, rows, dest)."""
    rows = []
    for _ in range(len(src)):
        d = int(rng.poisson(avg_deg)) if repeats else min(int(rng.poisson(avg_deg)), len(universe))
        r = rng.choice(universe, size=d, replace=repeats).astype(U64) if d else np.zeros(0, U64)
        if not unordered:
            r = np.unique(r)
        rows.append(r)
    dest = np.unique(np.concatenate(rows)) if rows and sum(r.size for r in rows) else np.zeros(0, U64)
    return np.asarray(src, U64), rows, dest.astype(U64)


def path(rng, nlevels, nroots, hi=400, avg_deg=3.0, unordered=True, repeats=True):
    """A path of nlevels levels: level 0's src are nroots uids, each later level's src is the previous dest."""
    src = sorted_uids(rng, nroots, hi)
    levels = []
    for _ in range(nlevels):
        universe = np.arange(1, hi + 1, dtype=U64)
        lv = level(rng, src, hi, universe, avg_deg, unordered, repeats)
        levels.append(lv)
        src = lv[2]
    return levels


def value_map(rng, keys_from, frac, kind):
    """A map over a fraction of keys_from: kind 'int' (wide int64 that wrap), 'dyadic' (k / 8, exact sums) or
    'wild' (float64 with +-0, +-Inf, NaN, huge and tiny values)."""
    keys = np.sort(rng.choice(keys_from, size=max(1, int(len(keys_from) * frac)), replace=False)).astype(U64) \
        if len(keys_from) else np.zeros(0, U64)
    n = keys.size
    if kind == "int":
        vals = rng.integers(-(1 << 63), (1 << 63) - 1, size=n, dtype=np.int64, endpoint=True)
    elif kind == "smallint":
        vals = rng.integers(-50, 50, size=n).astype(np.int64)
    elif kind == "dyadic":
        vals = rng.integers(-64, 64, size=n).astype(np.float64) / 8.0
    else:
        pool = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1.7e308, -1.7e308, 1e308, 5e-324, 1.0, -2.5, 0.1, 3.0],
                        np.float64)
        vals = np.where(rng.random(n) < 0.5, rng.choice(pool, size=n), rng.normal(0, 1e3, size=n))
    return keys, vals


def formula_propagate(keys, vals, levels):
    """transformTo for maps whose sums do not depend on order: per level, every contributing row adds the source's
    value to each of its values (np.add.at; int64 through uint64 so that it wraps)."""
    keys = np.asarray(keys, U64)
    isf = np.asarray(vals).dtype == np.float64
    cur = dict(zip(keys.tolist(), np.asarray(vals).tolist()))
    for src, rows, dest in levels:
        dest = np.asarray(dest, U64)
        acc = np.zeros(dest.size, np.float64 if isf else U64)
        hit = np.zeros(dest.size, bool)
        for s, r in zip(np.asarray(src, U64).tolist(), rows):
            if s not in cur or len(r) == 0:
                continue
            idx = np.searchsorted(dest, np.asarray(r, U64))
            add = np.float64(cur[s]) if isf else np.int64(cur[s]).view(U64)
            np.add.at(acc, idx, add)
            hit[idx] = True
        if isf:
            acc = np.clip(acc, -np.finfo(np.float64).max, np.finfo(np.float64).max)
        cur = dict(zip(dest[hit].tolist(), (acc[hit] if isf else acc[hit].view(np.int64)).tolist()))
    k = np.asarray(sorted(cur), U64)
    return k, np.asarray([cur[x] for x in k.tolist()], np.float64 if isf else np.int64)


def formula_level_agg(fn, keys, vals, src, rows):
    """evalLevelAgg per row for order-free inputs: numpy min / max / sum / mean over the present values."""
    keys = np.asarray(keys, U64)
    vals = np.asarray(vals)
    isf = vals.dtype == np.float64
    ok, ov = [], []
    for s, r in zip(np.asarray(src, U64).tolist(), rows):
        r = np.asarray(r, U64)
        j = np.searchsorted(keys, r)
        j = np.minimum(j, max(keys.size - 1, 0))
        present = keys.size > 0
        pres = (keys[j] == r) if present else np.zeros(r.size, bool)
        x = vals[j[pres]] if present else vals[:0]
        if x.size == 0:
            continue
        if fn == "min":
            y = x.min()
        elif fn == "max":
            y = x.max()
        elif fn == "sum":
            y = x.sum() if isf else x.view(U64).sum(dtype=U64).view(np.int64)
        else:
            y = (x.sum() if isf else float(np.int64(x.view(U64).sum(dtype=U64).view(np.int64)))) / x.size
        ok.append(s)
        ov.append(y)
    dt = np.float64 if fn == "avg" or isf else np.int64
    return np.asarray(ok, U64), np.asarray(ov, dt)
