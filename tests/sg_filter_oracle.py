"""ctypes binding of sg_filter_oracle.c: a subgraph's @filter tree and first / offset (query/query.go filterCopy,
ProcessGraph's filter block, applyPagination, updateUidMatrix, x.PageRange, the DoCount block and worker/compare.go
evalCompare) restated line by line.  TEST INFRASTRUCTURE ONLY: the checker of dgx_sg_filter in tests/ and the CPU leg
of tools/bench_ops.py C19.

The library is compiled on first use into the temporary directory (the tree itself may be read-only), under a name
keyed by the sources' contents.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from dgraph_b200.algo import sg_filter_flat

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "sg_filter_oracle.c"), os.path.join(os.path.dirname(_HERE), "oracle", "oracle.c")]
_DEPS = [os.path.join(os.path.dirname(_HERE), "oracle", "oracle.h")]
KIND = {"list": 0, "count": 1, "len": 1}
CMP = {"le": 0, "ge": 1, "lt": 2, "gt": 3, "eq": 4}

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    h = hashlib.sha256()
    for f in _SRCS + _DEPS:
        with open(f, "rb") as fh:
            h.update(fh.read())
    so = os.path.join(tempfile.gettempdir(), f"dgx_sg_filter_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-o", tmp] + _SRCS)
        os.replace(tmp, so)  # atomic: concurrent test processes never load a half-written file
    L = C.CDLL(so)
    vp = C.c_void_p
    L.orc_sg_filter.argtypes = [C.c_size_t] + [vp] * 11 + [C.c_size_t, vp, vp, C.c_size_t, C.c_int32, C.c_int32] + \
        [vp] * 5
    L.orc_sg_filter.restype = C.c_int
    _lib = L
    return L


def counts_of(lf, n0):
    """c_i of a COUNT leaf for the first n0 values of D0, as int64."""
    a = np.asarray(lf[3])
    if lf[0] == "count":
        return a[:n0].astype(np.int64)
    return (a[1:n0 + 1].astype(np.uint64) - a[:n0].astype(np.uint64)).astype(np.int64)


def _csr(arrs, dt):
    off = np.zeros(len(arrs) + 1, np.uint64)
    np.cumsum([a.size for a in arrs], out=off[1:])
    flat = np.concatenate([a.astype(dt) for a in arrs]) if int(off[-1]) else np.zeros(1, dt)
    return np.ascontiguousarray(flat), off


def sg_filter(tree, leaves, d0, rows, count=0, offset=0):
    """(rows, counts, dest) of the restatement: the filtered and paged rows, their lengths and the new DestUIDs."""
    f = sg_filter_flat(tree)
    d0 = np.ascontiguousarray(np.asarray(d0, np.uint64))
    n0 = d0.size
    lists = [np.asarray(lf[1], np.uint64) if lf[0] == "list" else np.zeros(0, np.uint64) for lf in leaves]
    cv = [counts_of(lf, n0) if lf[0] != "list" else np.zeros(0, np.int64) for lf in leaves]
    la, lo = _csr(lists, np.uint64)
    ca, co = _csr(cv, np.int64)
    kind = np.array([KIND[lf[0]] for lf in leaves] or [0], np.int32)
    cmp = np.array([CMP.get(lf[1], 0) if lf[0] != "list" else 0 for lf in leaves] or [0], np.int32)
    thr = np.array([int(lf[2]) if lf[0] != "list" else 0 for lf in leaves] or [0], np.int64)
    v, v_off = _csr([np.asarray(r, np.uint64) for r in rows], np.uint64)
    nrows = len(rows)
    m = int(v_off[-1])
    dest = np.empty(max(n0, 1), np.uint64)
    out = np.empty(max(m, 1), np.uint64)
    out_off = np.zeros(nrows + 1, np.uint64)
    counts = np.zeros(max(nrows, 1), np.uint32)
    n = C.c_size_t(0)
    d0p = d0 if n0 else np.zeros(1, np.uint64)
    rc = lib().orc_sg_filter(f["nnodes"], f["op"].ctypes.data, f["parent"].ctypes.data, f["leaf"].ctypes.data,
                             kind.ctypes.data, cmp.ctypes.data, thr.ctypes.data, la.ctypes.data, lo.ctypes.data,
                             ca.ctypes.data, co.ctypes.data, d0p.ctypes.data, n0, v.ctypes.data, v_off.ctypes.data,
                             nrows, count, offset, dest.ctypes.data, C.addressof(n), out.ctypes.data,
                             out_off.ctypes.data, counts.ctypes.data)
    if rc != 0:
        raise MemoryError("sg_filter oracle: allocation failed")
    res = [out[int(out_off[i]):int(out_off[i + 1])].copy() for i in range(nrows)]
    return res, counts[:nrows].copy(), dest[:n.value].copy()
