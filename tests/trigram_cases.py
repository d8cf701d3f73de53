"""Raw dgx_trigram_query calls and the argument errors the library refuses before anything is copied, shared by the CPU
test of the checks (tests/test_trigram_host.py) and the GPU test (tests/test_gpu_trigram_query.py)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from gen_trigram import QAND, QOR

SENTINEL = 0xA5A5A5A5A5A5A5A5
OK, ERR_ARG, ERR_CAP = 0, -3, -4


class Raw:
    """One call's arguments in the ABI's form: pack leaves first (pb.UidPack or None, with their layers), then the
    lists.  list_off / mut_off override the offsets computed from the lists and layers (malformed offsets)."""

    def __init__(self, tree, packs=(), muts=None, lists=(), list_off=None, mut_off=None, keys=None):
        from dgraph_b200 import algo

        self.tree = tree
        self.qt, self.qa = algo.query_tree(tree)
        self.npacks = len(packs)
        self.packs = list(packs)
        self.muts = list(muts) if muts is not None else [None] * len(packs)
        self.mu, self.mf, self.mut_off = algo._mut_csr(self.muts)
        if mut_off is not None:
            self.mut_off = np.asarray(mut_off, np.uint64)
        arrs = [np.asarray(a, np.uint64) for a in lists]
        self.list_off = np.zeros(len(arrs) + 1, np.uint64)
        np.cumsum([a.size for a in arrs], out=self.list_off[1:])
        self.lists = np.concatenate(arrs) if int(self.list_off[-1]) else np.zeros(1, np.uint64)
        if list_off is not None:
            self.list_off = np.asarray(list_off, np.uint64)
        self.nlists = self.list_off.size - 1
        self.refs, self._keep = algo._refs_of(self.packs, keys)

    def host(self, after: int, out_cap: int, out=None):
        from dgraph_b200 import _lib

        out = np.full(max(out_cap, 1) + 4, SENTINEL, np.uint64) if out is None else out
        n = C.c_size_t(SENTINEL)
        rc = _lib.load().dgx_trigram_query(C.byref(self.qt), self.refs, self.npacks, self.mu.ctypes.data,
                                           self.mf.ctypes.data, self.mut_off.ctypes.data, self.lists.ctypes.data,
                                           self.list_off.ctypes.data, self.nlists, after, out.ctypes.data, out_cap,
                                           C.byref(n))
        return rc, out, n.value


def _chain(depth: int):
    return [(QAND if i % 2 else QOR, [0], [i + 1] if i + 1 < depth else []) for i in range(depth)]


def error_cases():
    """(name, Raw arguments, expected rc) of every argument the library refuses before anything is copied."""
    one = np.array([5, 9], np.uint64)
    mu = (np.array([3], np.uint64), np.array([0], np.uint8))
    return [
        ("no node", dict(tree=[], lists=[one]), ERR_ARG),
        ("op 1", dict(tree=[(1, [0], [])], lists=[one]), ERR_ARG),
        ("op 4", dict(tree=[(QOR, [0], [1]), (4, [0], [])], lists=[one]), ERR_ARG),
        ("empty AND", dict(tree=[(QOR, [0], [1]), (QAND, [], [])], lists=[one]), ERR_ARG),
        ("no parent", dict(tree=[(QOR, [0], []), (QOR, [0], [])], lists=[one]), ERR_ARG),
        ("sub before parent", dict(tree=[(QOR, [0], [0])], lists=[one]), ERR_ARG),
        ("sub past nnodes", dict(tree=[(QOR, [0], [2]), (QOR, [0], [])], lists=[one]), ERR_ARG),
        ("two parents", dict(tree=[(QOR, [0], [1, 2]), (QOR, [0], [2]), (QOR, [0], [])], lists=[one]), ERR_ARG),
        ("leaf out of range", dict(tree=[(QOR, [1], [])], lists=[one]), ERR_ARG),
        ("depth 33", dict(tree=_chain(33), lists=[one]), ERR_ARG),
        ("2^16 nodes", dict(tree=[(QOR, [0], list(range(1, 1 << 16)))] + [(QOR, [0], [])] * ((1 << 16) - 1),
                            lists=[one]), ERR_ARG),
        ("2^16 leaves", dict(tree=[(QOR, [0], [])], lists=[one] * (1 << 16)), ERR_ARG),
        ("2^20 leaf references", dict(tree=[(QOR, [0] * (1 << 20), [])], lists=[one]), ERR_ARG),
        ("bounds of 2^32", dict(tree=[(QOR, [0, 1], [])], packs=[None], muts=[mu], list_off=[0, (1 << 32) - 1]),
         ERR_ARG),
        ("list_off decreasing", dict(tree=[(QOR, [0, 1], [])], list_off=[0, 2, 1]), ERR_ARG),
        ("list_off[0] != 0", dict(tree=[(QOR, [0], [])], list_off=[1, 2]), ERR_ARG),
        ("mut_off decreasing", dict(tree=[(QOR, [0, 1], [])], packs=[None, None], muts=[mu, mu], mut_off=[0, 1, 0]),
         ERR_ARG),
        ("DGX_MUT_VALUE", dict(tree=[(QOR, [0], [])], packs=[None], muts=[(np.array([3], np.uint64),
                                                                          np.array([2], np.uint8))]), ERR_ARG),
    ]
