"""Graphs, Go's exec structure and an independent numpy formula for shortest() without weights (query/shortest.go
expandOut + shortestPath at unit cost, DESIGN section 5).  TEST INFRASTRUCTURE ONLY.

- Graph: uid predicates as CSR adjacency over uids 1 .. nnodes - 1, and the query's children: (predicate, filter), the
  filter being the allowed uids of an anyofterms-style filter or None.
- search: Go's exec structure.  Level 1 has one sg per child over SrcUIDs = {From}; after each level every sg
  with a non-empty DestUIDs spawns one sg per child over its next SrcUIDs, so level k has up to nchild^k sgs.  search
  runs levels through an `expand(sgs)` callable (PathSearch.expand, or Formula.expand) and stops as the library's
  caller does: at maxHops, when To was reached, when a level discovered nothing, or when no sg had a DestUIDs.
- Formula: the level rules restated with numpy set operations, independent of the restatement's heap and maps and of
  the device: kept = row values in the sg's dest; discovered = kept values not yet seen; parent = the smallest source
  with a kept edge into the node; attr = attr of the largest sg index holding (parent, node); next = dest - expanded.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np


@dataclass
class Graph:
    nnodes: int                                   # uids are 1 .. nnodes - 1
    preds: list = field(default_factory=list)     # (off, adj): adj[off[u] .. off[u+1]) ascending
    children: list = field(default_factory=list)  # (predicate index, allowed uids ascending or None)

    def row(self, p: int, u: int) -> np.ndarray:
        off, adj = self.preds[p]
        if u >= self.nnodes:
            return np.zeros(0, np.uint64)
        return adj[int(off[u]):int(off[u + 1])]


def pred_from_edges(nnodes: int, frm, to):
    """CSR adjacency of the edges (frm[k], to[k]); duplicates collapse."""
    f, t = np.asarray(frm, np.uint64), np.asarray(to, np.uint64)
    if f.size:
        e = np.unique(np.stack([f, t], 1), axis=0)
        f, t = e[:, 0], e[:, 1]
    off = np.zeros(nnodes + 1, np.uint64)
    np.add.at(off, f.astype(np.int64) + 1, 1)
    return np.cumsum(off).astype(np.uint64), np.ascontiguousarray(t, np.uint64)


def random_graph(rng, n, npred, mean_deg, zipf=False, self_loops=True):
    preds = []
    for _ in range(npred):
        m = int(rng.poisson(mean_deg * n))
        if zipf:
            f = np.minimum(rng.zipf(1.6, m), n).astype(np.uint64)
            f = (f * 2654435761 % n + 1).astype(np.uint64)  # hubs spread over the uid range
        else:
            f = rng.integers(1, n + 1, m).astype(np.uint64)
        t = rng.integers(1, n + 1, m).astype(np.uint64)
        if not self_loops:
            keep = f != t
            f, t = f[keep], t[keep]
        preds.append(pred_from_edges(n + 1, f, t))
    return preds


def chain(n, cycle=False):
    f = np.arange(1, n, dtype=np.uint64)
    t = f + 1
    if cycle:
        f, t = np.append(f, n), np.append(t, 1)
    return pred_from_edges(n + 1, f, t)


def random_case(rng):
    """A random search: (graph, from, to, max_hops) over random, Zipf, chain or cycle predicates, one to three
    children (a predicate may appear twice), some children filtered, To sometimes unreachable or outside the graph."""
    kind = rng.integers(0, 6)
    n = int(rng.integers(2, 60))
    if kind == 0:
        preds = [chain(n, cycle=bool(rng.random() < 0.5))]
    else:
        preds = random_graph(rng, n, int(rng.integers(1, 4)), float(rng.uniform(0.3, 3.5)), zipf=kind == 1,
                             self_loops=bool(rng.random() < 0.6))
    children = []
    for _ in range(int(rng.integers(1, 4))):
        p = int(rng.integers(0, len(preds)))
        allow = None
        if rng.random() < 0.3:
            allow = np.sort(rng.choice(np.arange(1, n + 1, dtype=np.uint64), int(rng.integers(0, n + 1)),
                                       replace=False)).astype(np.uint64)
        children.append((p, allow))
    g = Graph(n + 1, preds, children)
    frm = int(rng.integers(1, n + 1))
    to = int(rng.integers(1, n + 3))  # n + 1, n + 2: never reachable
    if to == frm:
        to = frm % (n + 2) + 1
    hops = None if rng.random() < 0.6 else int(rng.integers(1, 8))
    if len(children) > 1:  # Go's exec list grows as nchild^level: keep a level below ~2 000 sgs
        cap = int(np.log(2000) / np.log(len(children)))
        hops = cap if hops is None else min(hops, cap)
    return g, frm, to, hops


def process(graph: Graph, child: int, src) -> tuple:
    """ProcessGraph + updateUidMatrix for one child sg: (rows, dest)."""
    p, allow = graph.children[child]
    rows = [graph.row(p, int(u)) for u in np.asarray(src, np.uint64)]
    dest = np.unique(np.concatenate(rows)) if rows else np.zeros(0, np.uint64)
    dest = dest.astype(np.uint64)
    if allow is not None:
        dest = dest[np.isin(dest, allow)]
    return [r[np.isin(r, dest)] for r in rows], dest


def search(graph: Graph, frm: int, to: int, max_hops, expand):
    """Runs levels of Go's exec structure through expand(sgs) -> (next per sg, (edges, discovered, to_level)).  Returns
    the list of (sgs, next, stats) per level."""
    hops = (1 << 31) - 1 if max_hops is None else max_hops
    exec_ = [(c, np.asarray([frm], np.uint64)) for c in range(len(graph.children))]
    out = []
    while len(out) < hops and exec_:
        sgs = []
        for c, src in exec_:
            rows, dest = process(graph, c, src)
            sgs.append((c, src, rows, dest))
        nxt, st = expand(sgs)
        out.append((sgs, nxt, st))
        if st[2] or st[1] == 0:
            break
        exec_ = [(c, nxt[i]) for i, sg in enumerate(sgs) if sg[3].size for c in range(len(graph.children))]
    return out


class Formula:
    """The level rules over numpy sets (no heap, no map): the independent statement of what dgx_path_expand returns."""

    def __init__(self, frm: int, to: int):
        self.to = to
        self.seen = {frm: (0, 0, 0)}  # uid -> (parent, attr, level)
        self.expanded = np.zeros(0, np.uint64)
        self.level = 0
        self.to_level = 0

    def expand(self, sgs):
        us, vs, ss = [], [], []
        edges = 0
        for s, (_, src, rows, dest) in enumerate(sgs):
            d = np.asarray(dest, np.uint64)
            for u, r in zip(np.asarray(src, np.uint64), rows):
                r = np.asarray(r, np.uint64)
                k = r[np.isin(r, d)]
                edges += k.size
                us.append(np.full(k.size, u, np.uint64))
                vs.append(k)
                ss.append(np.full(k.size, s, np.int64))
        u = np.concatenate(us) if us else np.zeros(0, np.uint64)
        v = np.concatenate(vs) if vs else np.zeros(0, np.uint64)
        s = np.concatenate(ss) if ss else np.zeros(0, np.int64)
        srcs = np.unique(u)
        if any(self.seen.get(int(x), (0, 0, -1))[2] != self.level for x in srcs):
            raise ValueError("a source with a kept edge was not discovered at the previous level")
        seen = np.fromiter(self.seen.keys(), np.uint64, len(self.seen))
        new = ~np.isin(v, seen)
        nodes, inv = np.unique(v[new], return_inverse=True)
        par = np.full(nodes.size, np.iinfo(np.uint64).max, np.uint64)
        np.minimum.at(par, inv, u[new])
        best = np.full(nodes.size, -1, np.int64)
        on = u[new] == par[inv]
        np.maximum.at(best, inv[on], s[new][on])
        self.level += 1
        for x, p, b in zip(nodes.tolist(), par.tolist(), best.tolist()):
            self.seen[x] = (p, int(sgs[b][0]), self.level)
        self.expanded = np.union1d(self.expanded, srcs).astype(np.uint64)
        if not self.to_level and self.to in self.seen:
            self.to_level = self.level
        nxt = [np.asarray(d, np.uint64)[~np.isin(np.asarray(d, np.uint64), self.expanded)] for _, _, _, d in sgs]
        return nxt, (edges, int(nodes.size), self.to_level)

    def path(self):
        if not self.to_level:
            return np.zeros(0, np.uint64), np.zeros(0, np.uint32)
        uids, attrs, cur = [], [], self.to
        for _ in range(self.to_level):
            p, a, _ = self.seen[cur]
            uids.append(cur)
            attrs.append(a)
            cur = p
        uids.append(cur)
        return np.asarray(uids[::-1], np.uint64), np.asarray(attrs[::-1], np.uint32)


def fixture_case(d: dict, name: str):
    """One case of tests/golden/shortest_path_follow.json as (graph, from, to, child predicate names).  A child's
    `not_anyofterms` filter keeps the uids whose name has no such term (nodes without a name pass), applied to that
    child's dest and so to its rows, as ProcessGraph does."""
    c = d["cases"][name]
    n = 1 + max(max(max(e) for e in es) if es else 0 for es in d["edges"].values())
    preds, children, names = [], [], []
    for ch in c["children"]:
        es = d["edges"][ch["pred"]]
        preds.append(pred_from_edges(n + 1, [e[0] for e in es], [e[1] for e in es]))
        allow = None
        if ch.get("not_anyofterms"):
            term = ch["not_anyofterms"].lower()
            allow = np.asarray([u for u in range(1, n + 1)
                                if term not in d["names"].get(str(u), "").lower().split()], np.uint64)
        children.append((len(preds) - 1, allow))
        names.append(ch["pred"])
    return Graph(n + 1, preds, children), c["from"], c["to"], names


def level_arrays(graph: Graph, exec_):
    """One level of exec sgs [(child, src)] as the CSR arrays of dgx_path_level, built with numpy gathers (ProcessGraph
    + updateUidMatrix per sg, vectorised): (attr u32, src_off, src, v_off, v, dest_off, dest)."""
    attr, srcs, vs, lens_all, dests = [], [], [], [], []
    for c, src in exec_:
        p, allow = graph.children[c]
        off, adj = graph.preds[p]
        s = np.asarray(src, np.uint64)
        si = np.minimum(s, graph.nnodes - 1).astype(np.int64)
        lo, hi = off[si].astype(np.int64), off[si + 1].astype(np.int64)
        lens = np.where(s < graph.nnodes, hi - lo, 0)
        idx = np.repeat(lo - np.concatenate([[0], np.cumsum(lens)[:-1]]), lens) + np.arange(int(lens.sum()))
        v = adj[idx]
        dest = np.unique(v).astype(np.uint64)
        if allow is not None:
            dest = dest[np.isin(dest, allow)]
        keep = np.isin(v, dest)
        rid = np.repeat(np.arange(s.size), lens)
        attr.append(c)
        srcs.append(s)
        vs.append(v[keep])
        lens_all.append(np.bincount(rid[keep], minlength=s.size))
        dests.append(dest)
    cat = lambda xs: np.concatenate(xs).astype(np.uint64) if xs else np.zeros(0, np.uint64)  # noqa: E731
    offs = lambda n: np.concatenate([[0], np.cumsum(n)]).astype(np.uint64)  # noqa: E731
    return (np.asarray(attr, np.uint32), offs([a.size for a in srcs]), cat(srcs), offs(cat(lens_all)), cat(vs),
            offs([d.size for d in dests]), cat(dests))


class VecFormula:
    """Formula's level rules over dense per-uid arrays, for searches with millions of nodes (tools/bench_ops.py C16)."""

    def __init__(self, nnodes: int, frm: int, to: int):
        self.level_of = np.full(nnodes + 1, -1, np.int64)
        self.parent = np.zeros(nnodes + 1, np.uint64)
        self.attr = np.zeros(nnodes + 1, np.int64)
        self.expanded = np.zeros(nnodes + 1, bool)
        self.level_of[frm] = 0
        self.frm, self.to, self.level, self.to_level = frm, to, 0, 0

    def expand(self, arrays):
        attr, src_off, src, v_off, v, dest_off, dest = arrays
        nsg = attr.size
        row_sg = np.repeat(np.arange(nsg), np.diff(src_off.astype(np.int64)))
        val_row = np.repeat(np.arange(src.size), np.diff(v_off.astype(np.int64)))
        s = row_sg[val_row]
        u = src[val_row]
        dsg = np.repeat(np.arange(nsg), np.diff(dest_off.astype(np.int64)))
        # kept: (sg, value) pairs present in the sg's dest
        key = s.astype(np.uint64) << np.uint64(40) | v
        dkey = dsg.astype(np.uint64) << np.uint64(40) | dest
        kept = np.isin(key, dkey)
        u, v, s = u[kept], v[kept], s[kept]
        srcs = np.unique(u).astype(np.int64)
        if (self.level_of[srcs] != self.level).any():
            raise ValueError("a source with a kept edge was not discovered at the previous level")
        new = self.level_of[v.astype(np.int64)] < 0
        vn, un, sn = v[new].astype(np.int64), u[new], s[new]
        nodes = np.unique(vn)
        par = np.full(self.parent.size, np.iinfo(np.uint64).max, np.uint64)
        np.minimum.at(par, vn, un)
        best = np.full(self.parent.size, -1, np.int64)
        on = un == par[vn]
        np.maximum.at(best, vn[on], sn[on])
        self.level += 1
        self.level_of[nodes] = self.level
        self.parent[nodes] = par[nodes]
        self.attr[nodes] = attr[best[nodes]].astype(np.int64)
        self.expanded[srcs] = True
        if not self.to_level and self.to < self.level_of.size and self.level_of[self.to] >= 0:
            self.to_level = self.level
        keep = ~self.expanded[np.minimum(dest, self.expanded.size - 1).astype(np.int64)]
        nxt = dest[keep]
        noff = np.concatenate([[0], np.cumsum(np.bincount(dsg[keep], minlength=nsg))]).astype(np.uint64)
        return nxt, noff, (int(kept.sum()), int(nodes.size), self.to_level)

    def path(self):
        if not self.to_level:
            return np.zeros(0, np.uint64), np.zeros(0, np.uint32)
        uids, attrs, cur = [self.to], [], self.to
        for _ in range(self.to_level):
            attrs.append(int(self.attr[cur]))
            cur = int(self.parent[cur])
            uids.append(cur)
        return np.asarray(uids[::-1], np.uint64), np.asarray(attrs[::-1], np.uint32)


def plan(graph: Graph, frm: int, to: int, max_hops):
    """The levels of one search with Go's exec structure, each level's arrays and the VecFormula's answer:
    [(arrays, next, next_off, stats)], and the formula (for its path)."""
    f = VecFormula(graph.nnodes, frm, to)
    hops = (1 << 31) - 1 if max_hops is None else max_hops
    exec_ = [(c, np.asarray([frm], np.uint64)) for c in range(len(graph.children))]
    out = []
    while len(out) < hops and exec_:
        arrs = level_arrays(graph, exec_)
        nxt, noff, st = f.expand(arrs)
        out.append((arrs, nxt, noff, st))
        if st[2] or st[1] == 0:
            break
        dn = np.diff(arrs[5].astype(np.int64))
        exec_ = [(c, nxt[int(noff[i]):int(noff[i + 1])]) for i in range(arrs[0].size) if dn[i]
                 for c in range(len(graph.children))]
    return out, f
