"""Graphs and recursions for @recurse (query/recurse.go expandRecurse), and an independent formula for one sg's step.

- Graph: a uid predicate per name as CSR adjacency over uids 1..n (strictly ascending rows), from random small graphs
  with hubs, cycles, self-loops and empty rows up to Zipf out-degree graphs of millions of nodes.
- Formula: one sg's step written directly from the semantics, vectorised with numpy: the taken edges of an Attr are a
  sorted structured (from, to) array, and the step's edges are matched against it with searchsorted.  It shares no code
  with the line-by-line restatement (recurse_oracle.c).
- recurse(): the exec / expandChildren / depth / edge-limit loop of expandRecurse (:51-164) over any step function.
"""
from __future__ import annotations

import numpy as np

EDGE = np.dtype([("f", "<u8"), ("t", "<u8")])


class Pred:
    """A uid predicate: uid u's values are idx[ptr[u]:ptr[u + 1]] (u < ptr.size - 1; larger uids have none)."""

    def __init__(self, ptr, idx):
        self.ptr, self.idx = np.asarray(ptr, np.int64), np.asarray(idx, np.uint64)

    @classmethod
    def from_edges(cls, n, frm, to):
        f, t = np.asarray(frm, np.uint64), np.asarray(to, np.uint64)
        o = np.lexsort((t, f))
        f, t = f[o], t[o]
        keep = np.ones(f.size, bool)
        keep[1:] = (f[1:] != f[:-1]) | (t[1:] != t[:-1])
        f, t = f[keep], t[keep]
        ptr = np.zeros(n + 2, np.int64)
        np.add.at(ptr, f.astype(np.int64) + 1, 1)
        return cls(np.cumsum(ptr), t.copy())

    def csr(self, src):
        """sg.uidMatrix for SrcUIDs = src as (values, offsets), vectorised."""
        s = np.minimum(np.asarray(src, np.int64), self.ptr.size - 2)
        lo = np.where(np.asarray(src, np.int64) <= self.ptr.size - 2, self.ptr[s], 0)
        hi = np.where(np.asarray(src, np.int64) <= self.ptr.size - 2, self.ptr[s + 1], 0)
        lens = hi - lo
        off = np.zeros(lens.size + 1, np.uint64)
        np.cumsum(lens, out=off[1:])
        idx = np.repeat(lo - off[:-1].astype(np.int64), lens) + np.arange(int(off[-1]), dtype=np.int64)
        return self.idx[idx], off

    def row(self, u):
        u = int(u)
        if u + 1 >= self.ptr.size:
            return np.zeros(0, np.uint64)
        return self.idx[self.ptr[u]:self.ptr[u + 1]]

    def matrix(self, src):
        """sg.uidMatrix for SrcUIDs = src: one row per source (ProcessGraph with no order)."""
        return [self.row(u) for u in np.asarray(src, np.uint64)]


def random_graph(rng, n, preds, mean_deg=3.0, hub_frac=0.1, self_loops=True):
    """Small random multi-predicate graph over uids 1..n: a few hubs with many values, many nodes with none."""
    g = {}
    for name in preds:
        frm, to = [], []
        hubs = rng.choice(np.arange(1, n + 1), size=max(1, int(n * hub_frac)), replace=False)
        for u in range(1, n + 1):
            if rng.random() < 0.3:
                continue  # an empty row
            d = rng.poisson(mean_deg * (4 if u in hubs else 1))
            tv = np.where(rng.random(d) < 0.4, rng.choice(hubs, size=d), rng.integers(1, n + 1, size=d))
            if not self_loops:
                tv = tv[tv != u]
            frm += [u] * tv.size
            to += tv.tolist()
        g[name] = Pred.from_edges(n, frm, to)
    return g


def zipf_pred(rng, n, mean_deg, a=2.0, hub_pop=1.1):
    """Zipf out-degrees scaled to about mean_deg per node; half the targets Zipf-popular among the highest-degree nodes
    (hubs), half uniform."""
    deg = np.minimum(rng.zipf(a, n), 100_000).astype(np.float64)
    deg = np.maximum(1, np.round(deg * mean_deg / deg.mean())).astype(np.int64)
    m = int(deg.sum())
    frm = np.repeat(np.arange(1, n + 1, dtype=np.uint64), deg)
    by_deg = np.argsort(-deg, kind="stable").astype(np.uint64) + np.uint64(1)  # the popular targets are the hubs
    pop = by_deg[np.minimum(rng.zipf(hub_pop, m), n) - 1]
    uni = rng.integers(1, n + 1, size=m).astype(np.uint64)
    to = np.where(rng.random(m) < 0.5, pop, uni)
    return Pred.from_edges(n, frm, to)


class Formula:
    """The step of one sg, from the semantics: keep (from, to) iff to passes dest and (attr, from, to) was never kept."""

    def __init__(self):
        self.sets = {}

    def edges(self, attr):
        e = self.sets.get(attr, np.zeros(0, EDGE))
        return e["f"].copy(), e["t"].copy()

    def load(self, attr, frm, to):
        self.sets[attr] = np.rec.fromarrays([np.asarray(frm, np.uint64), np.asarray(to, np.uint64)], dtype=EDGE)

    def step(self, attr, src, rows, dest=None):
        lens = np.array([len(r) for r in rows], np.int64)
        to = np.concatenate([np.asarray(r, np.uint64) for r in rows]) if lens.sum() else np.zeros(0, np.uint64)
        frm = np.repeat(np.asarray(src, np.uint64), lens)
        ok = np.ones(to.size, bool) if dest is None else np.isin(to, np.asarray(dest, np.uint64))
        e = np.rec.fromarrays([frm, to], dtype=EDGE)
        have = self.sets.get(attr, np.zeros(0, EDGE))
        pos = np.searchsorted(have, e)
        seen = (pos < have.size) & (have[np.minimum(pos, max(have.size - 1, 0))] == e) if have.size else np.zeros(
            e.size, bool)
        keep = ok & ~seen
        kept_e = np.asarray(e[keep], EDGE)
        if kept_e.size:
            self.sets[attr] = np.sort(np.concatenate([np.asarray(have, EDGE), kept_e]))
        row_of = np.repeat(np.arange(len(rows)), lens)
        kept = [to[keep & (row_of == i)] for i in range(len(rows))]
        return kept, np.unique(to[keep]), int(keep.sum())


class Step:
    """One recorded sg step: level, position in exec, attr, the step of the sg it was expanded from (None at level 1),
    inputs and what the step gave."""
    __slots__ = ("level", "pos", "attr", "parent", "src", "rows", "dest", "kept_rows", "dest_uids", "kept")

    def __init__(self, **kw):
        for k, v in kw.items():
            setattr(self, k, v)


def merge_sorted(rows):
    return np.unique(np.concatenate([np.asarray(r, np.uint64) for r in rows])) if rows else np.zeros(0, np.uint64)


def recurse(graph, roots, preds, depth, step, filters=None, limit=None, allow_loop=False):
    """expandRecurse (:51-164) from the root uids over the predicates `preds` (names into graph, in block order),
    calling step(attr, src, rows, dest) -> (rows, DestUIDs, kept) for every sg with loop: false.  filters maps a
    predicate to the uids its filter lets through (the sg's DestUIDs after filtering are the merged rows ∩ that set).
    Returns (steps, numEdges, error) with error True when the edge limit stopped the query."""
    filters = filters or {}
    roots = np.unique(np.asarray(roots, np.uint64))
    exec_ = [(p, roots, None) for p in preds]  # expandChildren(start): one sg per predicate, SrcUIDs = start.DestUIDs
    steps, num_edges = [], 0
    level = 0
    while True:
        if level >= depth:
            return steps, num_edges, False
        level += 1
        out = []
        for pos, (attr, src, parent) in enumerate(exec_):
            rows = graph[attr].matrix(src) if attr in graph else [np.zeros(0, np.uint64) for _ in src]
            if len(rows) == 0:
                continue
            dest = None
            if attr in filters:
                dest = np.intersect1d(merge_sorted(rows), np.asarray(filters[attr], np.uint64))
            if allow_loop:
                if dest is not None:
                    rows = [np.intersect1d(r, dest) for r in rows]
                num_edges += len(src) * sum(len(r) for r in rows)
                kept_rows, dest_uids, kept = rows, merge_sorted(rows), None
            else:
                kept_rows, dest_uids, kept = step(attr, src, rows, dest)
                num_edges += kept
            steps.append(Step(level=level, pos=pos, attr=attr, parent=parent, src=np.asarray(src, np.uint64),
                              rows=rows, dest=dest, kept_rows=kept_rows, dest_uids=np.asarray(dest_uids, np.uint64),
                              kept=kept))
            if len(dest_uids):
                out += [(p, np.asarray(dest_uids, np.uint64), len(steps) - 1) for p in preds]
        if limit is not None and num_edges > limit:
            return steps, num_edges, True
        if not out:
            return steps, num_edges, False
        exec_ = out


class KeyFormula:
    """The formula on CSR rows with uids below 2^32, each edge one u64 key from << 32 | to: fast enough for
    recursions of 1e7 edges."""

    def __init__(self):
        self.sets = {}

    def edges(self, attr):
        k = self.sets.get(attr, np.zeros(0, np.uint64))
        return k >> np.uint64(32), k & np.uint64(0xFFFFFFFF)

    def step_csr(self, attr, src, v, v_off, dest=None):
        lens = np.diff(v_off.astype(np.int64))
        key = (np.repeat(np.asarray(src, np.uint64), lens) << np.uint64(32)) | v
        keep = np.ones(v.size, bool) if dest is None else np.isin(v, dest)
        have = self.sets.get(attr, np.zeros(0, np.uint64))
        if have.size:
            pos = np.minimum(np.searchsorted(have, key), have.size - 1)
            keep &= have[pos] != key
        if keep.any():
            self.sets[attr] = np.union1d(have, key[keep])
        ck = np.zeros(v.size + 1, np.uint64)
        np.cumsum(keep, out=ck[1:])
        out_off = ck[v_off.astype(np.int64)]
        return v[keep], out_off, np.unique(v[keep]), int(keep.sum())


def plan_levels(graph, roots, preds, depth, limit=None, formula=None):
    """expandRecurse over CSR matrices with KeyFormula: every sg's inputs and outputs, in exec order, for a bench or a
    large test to replay.  Each step is (attr, src, v, v_off, out, out_off, dest_uids, kept).  Returns (steps,
    numEdges, error)."""
    f = KeyFormula() if formula is None else formula
    roots = np.unique(np.asarray(roots, np.uint64))
    exec_ = [(p, roots) for p in preds]
    steps, total, level = [], 0, 0
    while level < depth:
        level += 1
        out = []
        for attr, src in exec_:
            v, v_off = graph[attr].csr(src)
            o, o_off, d, k = f.step_csr(attr, src, v, v_off)
            total += k
            steps.append((attr, src, v, v_off, o, o_off, d, k))
            if d.size:
                out += [(p, d) for p in preds]
        if limit is not None and total > limit:
            return steps, total, True
        if not out:
            break
        exec_ = out
    return steps, total, False


def c14_graph(rng, n=2_000_000):
    """The C14 graph: friend with Zipf out-degrees of mean 8, follow with mean 2, over uids 1..n."""
    return {"friend": zipf_pred(rng, n, 8.0), "follow": zipf_pred(rng, n, 2.0)}
