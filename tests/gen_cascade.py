"""Forests for @cascade (query/query.go populateVarMap) and an independent formula for the result.

- random_forest(): 1-8 levels, 1-6 children a node, 1-3 roots: Zipf rows, empty rows, rows and has_val shorter than the
  parent's dest, counts_len set, every flag combination (SKIP only on leaves), ordered (shuffled) rows, uids near 2^64,
  and first / offset negative, zero, past the row length and at the int32 limits.
- formula(): the result written from the semantics rather than the Go control flow: nodes bottom-up in reverse
  pre-order, dest pruned with vectorised masks, rows filtered with np.isin and cut with a closed form of PageRange.  It
  shares no code with the line-by-line restatement (cascade_oracle.c).
"""
from __future__ import annotations

import numpy as np

from dgraph_b200.algo import CC_CASCADE, CC_CHECKED, CC_FILTERED, CC_ORDERED, CC_SKIP, CascadeNode

FIRSTS = [0, 0, 0, 1, 2, 3, -1, -2, -5, 7, 100, -100, 2**31 - 1, -2**31]
OFFSETS = [0, 0, 0, 1, 2, -1, 3, 5, 100, 2**31 - 1, -2**31]


def page_range(count, offset, n):
    """x.PageRange in closed form."""
    if n == 0:
        return 0, 0
    if count < 0:
        return max(n + count, 0), n
    s = min(max(offset, 0), n)
    return s, n if count == 0 else min(s + count, n)


def _page_vec(count, offset, n):
    """page_range over an array of row lengths."""
    if count < 0:
        s, e = np.maximum(n + count, 0), n
    else:
        s = np.minimum(max(offset, 0), n)
        e = n if count == 0 else np.minimum(s + count, n)
    return np.where(n == 0, 0, s), np.where(n == 0, 0, e)


def _filter_rows(rows, keep_set, page=None):
    """Every row filtered by membership in keep_set (order kept), then cut by page = (first, offset)."""
    if not rows:
        return []
    lens = np.array([r.size for r in rows], np.int64)
    vals = np.concatenate(rows) if lens.sum() else np.zeros(0, np.uint64)
    rid = np.repeat(np.arange(lens.size), lens)
    m = np.isin(vals, keep_set)
    if page is not None:
        before = np.cumsum(m) - m                      # kept values before each value
        start = np.zeros(lens.size, np.int64)
        start[1:] = np.cumsum(lens)[:-1]
        row_before = np.where(lens > 0, before[np.minimum(start, max(vals.size - 1, 0))], 0) if vals.size else start
        rank = before - row_before[rid]
        s, e = _page_vec(page[0], page[1], np.bincount(rid[m], minlength=lens.size))
        m &= (rank >= s[rid]) & (rank < e[rid])
    kept = vals[m]
    return [a.copy() for a in np.split(kept, np.cumsum(np.bincount(rid[m], minlength=lens.size))[:-1])]


def formula(nodes):
    """([rows of each node], [dest of each node]) after @cascade."""
    n = len(nodes)
    kids = [[] for _ in range(n)]
    for k, nd in enumerate(nodes):
        if nd.parent >= 0:
            kids[nd.parent].append(k)
    rows, dests = [None] * n, [None] * n
    for k in reversed(range(n)):  # children come after their parent in pre-order
        nd = nodes[k]
        cascade, skip = bool(nd.flags & CC_CASCADE), bool(nd.flags & CC_SKIP)
        dest = nd.dest
        if cascade and not skip:
            i = np.arange(dest.size)
            keep = np.ones(dest.size, bool)
            for c in kids[k]:
                if not nodes[c].flags & CC_CHECKED:
                    continue
                lens = np.zeros(dest.size, np.int64)
                w = min(dest.size, len(rows[c]))
                lens[:w] = [r.size for r in rows[c][:w]]
                hv = np.zeros(dest.size, np.uint8)
                w = min(dest.size, nodes[c].has_val.size)
                hv[:w] = nodes[c].has_val[:w]
                keep &= ~((lens == 0) & (hv == 0) & (i >= nodes[c].counts_len))
            dests[k] = dest[keep]
        else:
            dests[k] = dest.copy()
        if cascade and (nd.parent >= 0 or nd.first != 0 or nd.offset != 0):
            rows[k] = _filter_rows(nd.rows, dests[k], (nd.first, nd.offset))
        elif nd.flags & CC_FILTERED and not skip:
            rows[k] = _filter_rows(nd.rows, dest)
        else:
            rows[k] = [r.copy() for r in nd.rows]
    return rows, dests


def _row(rng, pool, zipf_a=1.6, cap=30):
    if rng.random() < 0.25 or pool.size == 0:
        return np.zeros(0, np.uint64)
    k = int(min(rng.zipf(zipf_a), cap))
    return np.unique(pool[rng.integers(0, pool.size, k)])


def random_forest(rng, max_levels=8, max_children=6, max_nodes=40):
    """A random forest of algo.CascadeNode in pre-order."""
    levels = int(rng.integers(1, max_levels + 1))
    base = np.uint64(0) if rng.random() < 0.8 else np.uint64(2**64 - 1024)
    universe = int(rng.integers(4, 120))
    pool = base + np.arange(1, universe + 1, dtype=np.uint64)
    nodes = []

    def make(parent, level):
        root = parent < 0
        f = 0
        for bit, p in ((CC_CASCADE, 0.6), (CC_CHECKED, 0.6), (CC_FILTERED, 0.3), (CC_ORDERED, 0.25)):
            if rng.random() < p:
                f |= bit
        leaf = level + 1 >= levels or len(nodes) >= max_nodes or rng.random() < 0.15
        if leaf and rng.random() < 0.1:
            f |= CC_SKIP
        if root:
            dest = np.sort(rng.choice(pool, size=int(rng.integers(0, min(universe, 24) + 1)), replace=False))
            rows = [dest.copy()] if rng.random() < 0.9 else [_row(rng, pool) for _ in range(int(rng.integers(0, 3)))]
            p = 1
        else:
            p = nodes[parent].dest.size
            nrows = p if rng.random() < 0.75 else int(rng.integers(0, p + 1))
            value_only = rng.random() < 0.1
            rows = [] if value_only else [_row(rng, pool) for _ in range(nrows)]
            union = np.unique(np.concatenate(rows)) if rows and sum(r.size for r in rows) else np.zeros(0, np.uint64)
            if f & CC_FILTERED:
                union = union[rng.random(union.size) < 0.7]
            if rng.random() < 0.15:  # dest values no row holds
                union = np.union1d(union, rng.choice(pool, size=min(3, universe), replace=False))
            dest = union.astype(np.uint64)
        if f & CC_ORDERED:
            rows = [rng.permutation(r) for r in rows]
        hv_len = p if rng.random() < 0.5 else int(rng.integers(0, p + 2))
        dense = 0.8 if not rows else 0.15
        has_val = (rng.random(hv_len) < dense).astype(np.uint8)
        counts_len = 0 if rng.random() < 0.8 else int(rng.integers(0, p + 2))
        first = int(rng.choice(FIRSTS)) if rng.random() < 0.6 else 0
        offset = int(rng.choice(OFFSETS)) if rng.random() < 0.5 else 0
        k = len(nodes)
        nodes.append(CascadeNode(parent, f, first, offset, counts_len, dest.astype(np.uint64), rows, has_val))
        if not leaf and not f & CC_SKIP:
            for _ in range(int(rng.integers(1, max_children + 1))):
                if len(nodes) >= max_nodes:
                    break
                make(k, level + 1)

    for _ in range(int(rng.integers(1, 4))):
        make(-1, 0)
    return nodes


def levels_with_work(nodes, v_caps=None):
    """D of the launch formula: levels holding a dest value or a value slot (v_caps[k] overrides a node's value count,
    as the device form's room does)."""
    depth, work = [], {}
    for k, nd in enumerate(nodes):
        d = 0 if nd.parent < 0 else depth[nd.parent] + 1
        depth.append(d)
        vals = sum(r.size for r in nd.rows) if v_caps is None else v_caps[k]
        work[d] = work.get(d, False) or nd.dest.size > 0 or vals > 0
    return sum(work.values())


def zipf_rows(rng, nrows, universe, mean_deg, a=1.3):
    """nrows strictly ascending rows over 1..universe with Zipf-popular values and Poisson degrees: (values, offsets)."""
    deg = rng.poisson(mean_deg, nrows).astype(np.int64)
    rid = np.repeat(np.arange(nrows, dtype=np.int64), deg)
    val = np.minimum(rng.zipf(a, rid.size), universe).astype(np.uint64)
    val = (val * np.uint64(2654435761)) % np.uint64(universe) + np.uint64(1)  # popular uids spread over the range
    o = np.lexsort((val, rid))
    rid, val = rid[o], val[o]
    keep = np.ones(val.size, bool)
    keep[1:] = (rid[1:] != rid[:-1]) | (val[1:] != val[:-1])
    rid, val = rid[keep], val[keep]
    off = np.zeros(nrows + 1, np.uint64)
    np.cumsum(np.bincount(rid, minlength=nrows), out=off[1:])
    return val, off


def c15a_arrays(rng, roots=1_000_000, universe=2_000_000, values=20_000_000):
    """C15a in the flat form of algo.cascade_arrays: TestCascadeWithPaginationDeep scaled up.  `me(func: type(Person))
    @cascade { name gender friend { name friend(first: 2, offset: 1) { name alive } } }` with every child consulted
    (@cascade with no fields is __all__ and reaches every level); friend rows Zipf over `universe` uids, about `values`
    values a level, has_val densities 0.8 (name) and 0.5 (gender, alive)."""
    C = CC_CASCADE | CC_CHECKED
    par = [-1, 0, 0, 0, 3, 3, 5, 5]
    flags = [CC_CASCADE, C, C, C, C, C, C, C]
    first = [0, 0, 0, 0, 0, 2, 0, 0]
    offset = [0, 0, 0, 0, 0, 1, 0, 0]
    persons = np.sort(rng.choice(universe, roots, replace=False)).astype(np.uint64) + np.uint64(1)
    v1, o1 = zipf_rows(rng, persons.size, universe, values / persons.size)
    d3 = np.unique(v1)
    v2, o2 = zipf_rows(rng, d3.size, universe, values / d3.size)
    d5 = np.unique(v2)
    dens = lambda n, p: (rng.random(n) < p).astype(np.uint8)  # noqa: E731
    node_rows = [[persons], [], [], (v1, o1), [], (v2, o2), [], []]
    dests = [persons, np.zeros(0, np.uint64), np.zeros(0, np.uint64), d3, np.zeros(0, np.uint64), d5,
             np.zeros(0, np.uint64), np.zeros(0, np.uint64)]
    hvs = [np.zeros(0, np.uint8), dens(persons.size, 0.8), dens(persons.size, 0.5), np.zeros(0, np.uint8),
           dens(d3.size, 0.8), np.zeros(0, np.uint8), dens(d5.size, 0.8), dens(d5.size, 0.5)]
    vs, voffs, nrows = [], [np.zeros(1, np.uint64)], []
    base = np.uint64(0)
    for r in node_rows:
        if isinstance(r, tuple):
            v, o = r
        else:
            v = np.concatenate(r) if r else np.zeros(0, np.uint64)
            o = np.zeros(len(r) + 1, np.uint64)
            np.cumsum([x.size for x in r], out=o[1:])
        vs.append(v)
        voffs.append(o[1:] + base)
        base += np.uint64(v.size)
        nrows.append(o.size - 1)

    def off(sizes):
        o = np.zeros(len(sizes) + 1, np.uint64)
        np.cumsum(sizes, out=o[1:])
        return o

    return {"nnodes": 8, "parent": np.array([0xFFFFFFFF if p < 0 else p for p in par], np.uint32),
            "flags": np.array(flags, np.uint8), "first": np.array(first, np.int32),
            "offset": np.array(offset, np.int32), "counts_len": np.zeros(8, np.uint64),
            "v": np.ascontiguousarray(np.concatenate(vs)), "v_off": np.concatenate(voffs), "row_off": off(nrows),
            "dest": np.ascontiguousarray(np.concatenate(dests)), "dest_off": off([d.size for d in dests]),
            "has_val": np.ascontiguousarray(np.concatenate(hvs)), "hv_off": off([h.size for h in hvs])}
