"""ctypes binding of valvar_oracle.c: transformTo and evalLevelAgg (query/query.go) restated line by line.  TEST
INFRASTRUCTURE ONLY: the checker of dgx_var_propagate / dgx_var_level_agg in tests/ and the CPU leg of
tools/bench_ops.py C17.

The library is compiled on first use into the temporary directory (the tree itself may be read-only), under a name
keyed by the source's contents.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "valvar_oracle.c")
_lib = None
INT64, FLOAT64 = 1, 2
AGG = {"min": 0, "max": 1, "sum": 2, "avg": 3}
IN_ORDER = (0, 1, 2, 3)


def lib():
    global _lib
    if _lib is not None:
        return _lib
    with open(_SRC, "rb") as fh:
        h = hashlib.sha256(fh.read()).hexdigest()[:16]
    so = os.path.join(tempfile.gettempdir(), f"dgx_valvar_oracle_{os.getuid()}_{h}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        # -ffp-contract=off: every add is one IEEE add, as in Go
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-ffp-contract=off", "-fPIC", "-std=c11", "-shared",
                               "-o", tmp, _SRC, "-lm"])
        os.replace(tmp, so)  # atomic: concurrent test processes never load a half-written file
    L = C.CDLL(so)
    vp, sz, i64, ci = C.c_void_p, C.c_size_t, C.c_int64, C.c_int
    L.orc_propagate.restype = i64
    L.orc_propagate.argtypes = [ci, vp, vp, sz, sz, vp, vp, vp, vp, vp, vp, vp]
    L.orc_level_agg.restype = i64
    L.orc_level_agg.argtypes = [ci, ci, vp, vp, sz, vp, sz, vp, vp, vp, vp]
    _lib = L
    return L


def _words(vals):
    v = np.ascontiguousarray(vals)
    typ = FLOAT64 if v.dtype == np.float64 else INT64
    if v.dtype not in (np.float64, np.int64):
        raise TypeError(v.dtype)
    return typ, v.view(np.uint64)


def _a(x):
    x = np.ascontiguousarray(x, np.uint64)
    return x if x.size else np.zeros(1, np.uint64)


def _csr(rows):
    off = np.zeros(len(rows) + 1, np.uint64)
    np.cumsum([len(r) for r in rows], out=off[1:])
    flat = np.concatenate([np.asarray(r, np.uint64) for r in rows]) if int(off[-1]) else np.zeros(1, np.uint64)
    return flat, off


def propagate(keys, vals, levels, order=IN_ORDER):
    """levels: [(src, rows)] (dest is not read by transformTo).  Returns (keys, values) ascending by key."""
    return propagate_csr(keys, vals, [(src, *_csr(rows)) for src, rows in levels], order)


def propagate_csr(keys, vals, levels, order=IN_ORDER):
    """propagate() over levels given as flat (src, v, v_off) arrays."""
    typ, w = _words(vals)
    k = _a(keys)
    keep = []
    srcs, nrows, offs, vs = [], [], [], []
    for src, v, o in levels:
        s, v, o = _a(src), _a(v), np.ascontiguousarray(o, np.uint64)
        keep += [s, v, o]
        srcs.append(s.ctypes.data)
        offs.append(o.ctypes.data)
        vs.append(v.ctypes.data)
        nrows.append(o.size - 1)
    nl = len(levels)
    P = C.c_void_p * nl
    nr = np.asarray(nrows, np.uint64)
    cap = max(int(keep[-1][-1]), 1)
    ok, ov = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    ordr = np.asarray(order, np.int32)
    m = lib().orc_propagate(typ, k.ctypes.data, _a(w).ctypes.data, int(np.size(keys)), nl, P(*srcs), nr.ctypes.data, P(*offs), P(*vs), ordr.ctypes.data, ok.ctypes.data,
                            ov.ctypes.data)
    if m < 0:
        raise MemoryError("valvar oracle: allocation failed")
    return ok[:m].copy(), ov[:m].view(np.float64 if typ == FLOAT64 else np.int64).copy()


def level_agg(fn, keys, vals, src, rows):
    """Returns (keys, values): float64 for avg, the map's dtype otherwise."""
    return level_agg_csr(fn, keys, vals, src, *_csr(rows))


def level_agg_csr(fn, keys, vals, src, v, o):
    """level_agg() over the rows as flat (v, v_off) arrays."""
    typ, w = _words(vals)
    v, o = _a(v), np.ascontiguousarray(o, np.uint64)
    n = o.size - 1
    ok, ov = np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1), np.uint64)
    m = lib().orc_level_agg(typ, AGG[fn], _a(keys).ctypes.data, _a(w).ctypes.data, int(np.size(keys)),
                            _a(src).ctypes.data, n, o.ctypes.data, v.ctypes.data, ok.ctypes.data, ov.ctypes.data)
    if m < 0:
        raise MemoryError("valvar oracle: allocation failed")
    out = FLOAT64 if fn == "avg" or typ == FLOAT64 else INT64
    return ok[:m].copy(), ov[:m].view(np.float64 if out == FLOAT64 else np.int64).copy()
