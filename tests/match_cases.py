"""Shared pieces of the match() tests (tests/test_match_host.py, tests/test_gpu_match.py): raw dgx_match calls with
guard words, the golden fixture as columns and trigram leaves, the launch plan, and the argument errors the library
refuses before anything is copied."""
from __future__ import annotations

import ctypes as C
import json
import os

import numpy as np

import gen_trigram as gt
import trigram_plan as tp

SENTINEL = 0xA5A5A5A5A5A5A5A5
OK, ERR_ARG, ERR_CAP = 0, -3, -4
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "match_common.json")
FZ_LAUNCHES = 5  # fz_lookup, scan_u64, fz_test, fz_long, compact


def column(uids, values):
    from dgraph_b200 import algo

    return algo.StrColumn(uids, values)


def values_of(uids, values) -> dict:
    return {int(u): list(vs) for u, vs in zip(uids, values)}


def trigram_leaves(index: dict, query: bytes, kinds=("list",)):
    """uidsForMatch's leaves: one raw leaf (gen_trigram form) per distinct byte trigram of the query, its row the uids
    whose values hold it; kinds cycles over "list" and "pack"."""
    toks = list(dict.fromkeys(query[i:i + 3] for i in range(len(query) - 2)))
    out = []
    for k, t in enumerate(toks):
        row = np.array(sorted(index.get(t, ())), np.uint64)
        if kinds[k % len(kinds)] == "list":
            out.append(("list", row))
        else:
            out.append(("pack", row if row.size else None, None, 0))
    return out


def trigram_index(uids, values) -> dict:
    idx = {}
    for u, vs in zip(uids, values):
        for v in vs:
            for i in range(len(v) - 2):
                idx.setdefault(v[i:i + 3], set()).add(int(u))
    return idx


def launches(leaves, nuids: int) -> int:
    """Launches of one call: 0 without a candidate slot; the one-OR trigram plan's then 5, or 5 for a UidList."""
    if nuids:
        return FZ_LAUNCHES
    bounds = [gt.leaf_bound(lf) for lf in leaves]
    p = tp.plan([(gt.QOR, list(range(len(leaves))), [])], bounds)
    if p.root_bound == 0:
        return 0
    npacks = sum(1 for lf in leaves if lf[0] == "pack")
    return tp.launches(p, npacks) + FZ_LAUNCHES


def golden():
    with open(GOLDEN) as f:
        g = json.load(f)
    cols = {}
    for pred, tr in g["triples"].items():
        uids = [u for u, _ in tr]
        vals = [[bytes.fromhex(h)] for _, h in tr]
        cols[pred] = (uids, vals)
    return g, cols


class Raw:
    """One dgx_match call's arguments in the ABI's form: pack leaves first, then the lists.  The column is given as
    arrays so that malformed columns can be built."""

    def __init__(self, col, query, max, uids=(), leaves=(), list_off=None, mut_off=None, nvals=None, nbytes=None):
        from dgraph_b200 import algo

        self.col = col
        self.cs = col.struct()
        if nvals is not None:
            self.cs.nvals = nvals
        if nbytes is not None:
            self.cs.nbytes = nbytes
        self.q = query.encode() if isinstance(query, str) else bytes(query)
        self.qa = np.frombuffer(self.q + b"\0", np.uint8)
        self.max = max
        self.uids = np.ascontiguousarray(np.asarray(uids, np.uint64))
        pids = [j for j, lf in enumerate(leaves) if lf[0] == "pack"]
        lids = [j for j, lf in enumerate(leaves) if lf[0] == "list"]
        al = gt.to_algo(leaves)
        self.packs = [al[j][0] for j in pids]
        self.muts = [al[j][1] for j in pids]
        self.npacks = len(pids)
        self.mu, self.mf, self.mut_off = algo._mut_csr(self.muts)
        if mut_off is not None:
            self.mut_off = np.asarray(mut_off, np.uint64)
        arrs = [np.asarray(al[j], np.uint64) for j in lids]
        self.list_off = np.zeros(len(arrs) + 1, np.uint64)
        np.cumsum([a.size for a in arrs], out=self.list_off[1:])
        self.lists = np.concatenate(arrs) if int(self.list_off[-1]) else np.zeros(1, np.uint64)
        if list_off is not None:
            self.list_off = np.asarray(list_off, np.uint64)
        self.nlists = self.list_off.size - 1
        self.refs, self._keep = algo._refs_of(self.packs)
        self.bound = self.uids.size if self.uids.size else (
            sum(gt.leaf_bound(leaves[j]) for j in pids) + sum(gt.leaf_bound(leaves[j]) for j in lids))

    def host(self, after: int, out_cap: int):
        from dgraph_b200 import _lib

        out = np.full(max(out_cap, 1) + 4, SENTINEL, np.uint64)
        n = C.c_size_t(SENTINEL)
        u = self.uids if self.uids.size else np.zeros(1, np.uint64)
        rc = _lib.load().dgx_match(self.refs, self.npacks, self.mu.ctypes.data, self.mf.ctypes.data,
                                   self.mut_off.ctypes.data, self.lists.ctypes.data, self.list_off.ctypes.data,
                                   self.nlists, after, u.ctypes.data, self.uids.size, C.byref(self.cs),
                                   self.qa.ctypes.data, len(self.q), self.max, out.ctypes.data, out_cap, C.byref(n))
        return rc, out, n.value


def error_cases():
    """(name, Raw keyword arguments, expected rc, found on the device) of every refused argument."""
    c = column([3, 5, 9], [[b"abc"], [b"abd", b""], [b"\xff"]])
    bad_off = column([3, 5], [[b"ab"], [b"cd"]])
    bad_off.val_off = np.array([0, 2, 1], np.uint64)
    off0 = column([3], [[b"ab"]])
    off0.val_off = np.array([1, 1], np.uint64)
    boff = column([3], [[b"ab", b"c"]])
    boff.byte_off = np.array([0, 2, 1], np.uint64)
    desc = column([5, 3], [[b"ab"], [b"cd"]])
    return [
        ("max -1", dict(col=c, query="abc", max=-1, uids=[3]), ERR_ARG, False),
        ("max 2^31", dict(col=c, query="abc", max=1 << 31, uids=[3]), ERR_ARG, False),
        ("query 4097 runes", dict(col=c, query="a" * 4097, max=1, uids=[3]), ERR_ARG, False),
        ("query 4097 bad bytes", dict(col=c, query=b"\xff" * 4097, max=1, uids=[3]), ERR_ARG, False),
        ("nvals != val_off[n]", dict(col=c, query="abc", max=1, uids=[3], nvals=3), ERR_ARG, False),
        ("nbytes != byte_off[nvals]", dict(col=c, query="abc", max=1, uids=[3], nbytes=6), ERR_ARG, False),
        ("val_off decreasing", dict(col=bad_off, query="abc", max=1, uids=[3]), ERR_ARG, False),
        ("val_off[0] != 0", dict(col=off0, query="abc", max=1, uids=[3]), ERR_ARG, False),
        ("byte_off decreasing", dict(col=boff, query="abc", max=1, uids=[3]), ERR_ARG, False),
        ("list_off decreasing", dict(col=c, query="abc", max=1, list_off=[0, 2, 1]), ERR_ARG, False),
        ("mut_off decreasing", dict(col=c, query="abc", max=1, leaves=[("pack", None, (np.array([3], np.uint64),
                                    np.array([0], np.uint8)), 0)] * 2, mut_off=[0, 1, 0]), ERR_ARG, False),
        ("leaf bounds of 2^32", dict(col=c, query="abc", max=1, leaves=[("pack", None, (np.array([3], np.uint64),
                                     np.array([0], np.uint8)), 0)], list_off=[0, (1 << 32) - 1]), ERR_ARG, False),
        ("DGX_MUT_VALUE", dict(col=c, query="abc", max=1, leaves=[("pack", None, (np.array([3], np.uint64),
                               np.array([2], np.uint8)), 0)]), ERR_ARG, True),
        ("candidates not ascending", dict(col=c, query="abc", max=1, uids=[5, 3]), ERR_ARG, True),
        ("candidates repeated", dict(col=c, query="abc", max=1, uids=[3, 3]), ERR_ARG, True),
        ("list leaf not ascending", dict(col=c, query="abc", max=1, leaves=[("list", np.array([5, 3], np.uint64))]),
         ERR_ARG, True),
        ("column uids not ascending", dict(col=desc, query="abc", max=1, uids=[3]), ERR_ARG, True),
    ]
