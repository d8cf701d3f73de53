"""ctypes binding of shortest_oracle.c: shortest() without weights (query/shortest.go expandOut + shortestPath)
restated line by line.  TEST INFRASTRUCTURE ONLY: the checker of dgx_path_search in tests/ and the CPU leg of
tools/bench_ops.py C16.

The library is compiled on first use into the temporary directory (the tree itself may be read-only), under a name
keyed by the source's contents.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile
from dataclasses import dataclass

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "shortest_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    with open(_SRC, "rb") as fh:
        h = hashlib.sha256(fh.read()).hexdigest()[:16]
    so = os.path.join(tempfile.gettempdir(), f"dgx_shortest_oracle_{os.getuid()}_{h}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-std=c11", "-shared", "-o", tmp, _SRC])
        os.replace(tmp, so)  # atomic: concurrent test processes never load a half-written file
    L = C.CDLL(so)
    vp, sz, u64, i64 = C.c_void_p, C.c_size_t, C.c_uint64, C.c_int64
    L.orc_shortest.restype = i64
    L.orc_shortest.argtypes = [C.c_int, vp, vp, u64, C.c_int, vp, vp, vp, u64, u64, i64, u64, vp, vp, sz,
                               vp, vp, vp, vp, C.POINTER(sz), vp, vp, vp, C.POINTER(sz), vp, C.POINTER(sz)]
    _lib = L
    return L


@dataclass
class Result:
    levels: int            # levels expandOut ran
    level_edges: list      # numEdges added by each level
    level_sgs: list        # exec sgs of each level
    dist: dict             # uid -> (hop, parent, attr)
    adj: dict              # (from, to) -> attr (adjacencyMap, last writer)
    path: np.ndarray       # Go's path From .. To, empty when not reached


def run(graph, frm: int, to: int, max_hops: int, seed: int) -> Result:
    """graph: gen_shortest.Graph.  seed: the neighbour order standing in for Go's map iteration (nonzero)."""
    L = lib()
    offs = [np.ascontiguousarray(o, np.uint64) for o, _ in graph.preds]
    adjs = [np.ascontiguousarray(a if a.size else np.zeros(1, np.uint64), np.uint64) for _, a in graph.preds]
    po = (C.c_void_p * len(offs))(*[o.ctypes.data for o in offs])
    pa = (C.c_void_p * len(adjs))(*[a.ctypes.data for a in adjs])
    nch = len(graph.children)
    cp = np.asarray([p for p, _ in graph.children] or [0], np.int32)
    allows = [None if f is None else np.ascontiguousarray(f if f.size else np.zeros(1, np.uint64), np.uint64)
              for _, f in graph.children]
    pl = (C.c_void_p * max(nch, 1))(*[None if f is None else f.ctypes.data for f in allows])
    nl = np.asarray([0 if f is None else g.size for (_, g), f in zip(graph.children, allows)] or [0], np.uint64)
    n = graph.nnodes
    ne = max(sum(int(a.size) for _, a in graph.preds), 1)
    cap_levels = n + 2
    le, ls = np.zeros(cap_levels, np.uint64), np.zeros(cap_levels, np.uint64)
    du, dh, dp, da = np.zeros(n, np.uint64), np.zeros(n, np.int64), np.zeros(n, np.uint64), np.zeros(n, np.int64)
    af, at, aa = np.zeros(ne, np.uint64), np.zeros(ne, np.uint64), np.zeros(ne, np.int64)
    path = np.zeros(n, np.uint64)
    nd, na, npath = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    hops = (1 << 31) - 1 if max_hops is None else int(max_hops)
    levels = L.orc_shortest(len(offs), po, pa, n, nch, cp.ctypes.data, pl, nl.ctypes.data, frm, to, hops, seed,
                            le.ctypes.data, ls.ctypes.data, cap_levels, du.ctypes.data, dh.ctypes.data,
                            dp.ctypes.data, da.ctypes.data, C.byref(nd), af.ctypes.data, at.ctypes.data,
                            aa.ctypes.data, C.byref(na), path.ctypes.data, C.byref(npath))
    if levels < 0:
        raise MemoryError("shortest oracle: allocation failed")
    dist = {int(u): (int(h), int(p), int(a)) for u, h, p, a in zip(du[:nd.value], dh[:nd.value], dp[:nd.value],
                                                                   da[:nd.value])}
    adj = {(int(f), int(t)): int(a) for f, t, a in zip(af[:na.value], at[:na.value], aa[:na.value])}
    return Result(int(levels), le[:levels].tolist(), ls[:levels].tolist(), dist, adj, path[:npath.value].copy())
