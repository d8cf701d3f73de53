"""An independent numpy formula for @groupby over one uid attribute, and the random cases the tests draw.

For parent row ul: the rows whose source is in ul (np.isin), expanded to (value, source) edges, sorted by (value,
source) with np.lexsort, cut into runs of equal values, and the runs ordered by (size, value).  Laid out as
dgx_groupby_uid lays out its result: (keys, counts, grp_off, mem_off, members)."""
from __future__ import annotations

import numpy as np

U64_MAX = (1 << 64) - 1


def groupby_uid(parents, src, rows):
    src = np.asarray(src, np.uint64)
    lens = np.array([len(r) for r in rows], np.int64)
    v = np.concatenate([np.asarray(r, np.uint64) for r in rows]) if lens.sum() else np.zeros(0, np.uint64)
    row_of = np.repeat(np.arange(len(rows)), lens)
    keys, counts, members, grp_off, mem_off = [], [], [], [0], [0]
    for ul in parents:
        sel = np.isin(src, np.asarray(ul, np.uint64))[row_of]
        d, s = v[sel], src[row_of[sel]]
        o = np.lexsort((s, d))
        d, s = d[o], s[o]
        starts = np.flatnonzero(np.r_[True, d[1:] != d[:-1]]) if d.size else np.zeros(0, np.int64)
        sizes = np.diff(np.r_[starts, d.size])
        gk = d[starts]
        for g in np.lexsort((gk, sizes)):
            keys.append(int(gk[g]))
            counts.append(int(sizes[g]))
            members.extend(s[starts[g]:starts[g] + sizes[g]].tolist())
            mem_off.append(len(members))
        grp_off.append(len(keys))
    return (np.array(keys, np.uint64), np.array(counts, np.uint64), np.array(grp_off, np.uint64),
            np.array(mem_off, np.uint64), np.array(members, np.uint64))


def _uids(rng, n, lo, hi):
    """n distinct sorted uids in [lo, hi]."""
    n = min(n, hi - lo + 1)
    if hi - lo < 4 * n + 16:
        return np.sort(rng.choice(np.arange(lo, hi + 1, dtype=np.uint64), n, replace=False))
    return np.unique(rng.integers(lo, hi, n, dtype=np.uint64, endpoint=True))


def case(rng, kind: str = "mixed", nrows=None, npar=None, nd=None):
    """(parents, src, rows, dest) of one random call.  kind: "small" uids near 0, "high" near 2^64 - 1, "mixed" both,
    "hub" a destination in every row."""
    nrows = int(rng.integers(0, 40)) if nrows is None else nrows
    npar = int(rng.integers(0, 6)) if npar is None else npar
    nd = int(rng.integers(1, 30)) if nd is None else nd
    if kind == "high":
        lo, hi = U64_MAX - 4000, U64_MAX
    elif kind == "small":
        lo, hi = 0, 4000
    else:
        lo, hi = 0, U64_MAX
    if kind == "mixed":
        pool = np.unique(np.r_[_uids(rng, 3 * nrows + nd + 8, 0, 500), _uids(rng, 3 * nrows + nd + 8, U64_MAX - 500, U64_MAX),
                                np.array([0, U64_MAX], np.uint64)])
    else:
        pool = _uids(rng, 3 * nrows + nd + 8, lo, hi)
    src = np.sort(rng.choice(pool, min(nrows, pool.size), replace=False))
    nrows = src.size
    dest = np.sort(rng.choice(pool, min(nd, pool.size), replace=False))
    rows = []
    for _ in range(nrows):
        k = int(rng.integers(0, dest.size + 1)) if rng.random() < 0.8 else 0
        r = set(rng.choice(dest, k, replace=False).tolist())
        if kind == "hub":
            r.add(int(dest[0]))
        rows.append(np.array(sorted(r), np.uint64))
    parents = []
    for _ in range(npar):
        a = rng.random()
        if a < 0.15:
            parents.append(np.zeros(0, np.uint64))
        elif a < 0.3:
            parents.append(src.copy())
        else:
            extra = np.array([99999], np.uint64) if rng.random() < 0.5 else np.zeros(0, np.uint64)
            pick = rng.choice(pool, int(rng.integers(0, pool.size + 1)), replace=False)
            parents.append(np.unique(np.r_[pick, extra]).astype(np.uint64))
    return parents, src, rows, dest


def dest_of(rows):
    return np.unique(np.concatenate([np.asarray(r, np.uint64) for r in rows])) if any(len(r) for r in rows) \
        else np.zeros(0, np.uint64)


def c13_rows(rng, nrows=10 ** 6, ndest=10 ** 6, per_row=32):
    """1e6 source rows, destinations drawn Zipf-popular over ndest uids (per_row draws a row, repeats dropped: about 2e7
    values in all), as flat CSR: (src, v, v_off, dest)."""
    src = np.arange(1, nrows + 1, dtype=np.uint64) * 2
    dest_uids = np.arange(1, ndest + 1, dtype=np.uint64) * 3 + 1
    lens = rng.poisson(per_row, nrows).astype(np.int64)
    row = np.repeat(np.arange(nrows, dtype=np.int64), lens)
    d = np.minimum(rng.zipf(1.3, row.size), ndest) - 1
    d = (d * 2654435761) % ndest  # popular destinations spread over the uid range
    key = row * ndest + d
    key = np.unique(key)
    row, d = key // ndest, key % ndest
    v = dest_uids[d]
    v_off = np.zeros(nrows + 1, np.uint64)
    np.cumsum(np.bincount(row, minlength=nrows), out=v_off[1:])
    return src, v, v_off, np.unique(v)
