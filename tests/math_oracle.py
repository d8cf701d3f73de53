"""ctypes binding of math_oracle.c: math() (query/math.go evalMathTree and valueVarAggregation's math branch) restated
line by line, with Go's map iteration order drawn from a seed.  TEST INFRASTRUCTURE ONLY: the checker of
dgx_math_eval in tests/.

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

from dgraph_b200 import algo

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "math_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    with open(_SRC, "rb") as fh:
        h = hashlib.sha256(fh.read()).hexdigest()[:16]
    so = os.path.join(tempfile.gettempdir(), f"dgx_math_oracle_{os.getuid()}_{h}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        # -ffp-contract=off: every operation is one IEEE operation, as in Go
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-ffp-contract=off", "-fPIC", "-std=c11", "-shared",
                               "-o", tmp, _SRC, "-lm"])
        os.replace(tmp, so)
    L = C.CDLL(so)
    vp, sz = C.c_void_p, C.c_size_t
    L.orc_math.restype = C.c_int64
    L.orc_math.argtypes = [vp, vp, vp, vp, vp, sz, vp, vp, vp, vp, vp, vp, sz, C.c_int, C.c_uint64, vp, vp, vp, vp, vp]
    _lib = L
    return L


def evaluate(tree, maps, range_uids=None, seed=0):
    """(kind, keys, words, tags, partial) as algo.EvalMath returns them, kind None where evalMathTree errs; partial:
    an Iterate stopped by an error that another key would not have raised (the answer depends on map order)."""
    names = {}
    nodes = algo.math_program(tree, names)
    nn = len(nodes)
    if nn > 64:
        raise ValueError("the restatement holds at most 64 nodes")
    op = np.array([n.op for n in nodes], np.uint8)
    ctag = np.array([n.const_tag for n in nodes], np.uint8)
    child = np.array([[n.child[c] for c in range(3)] for n in nodes], np.uint16).ravel()
    leaf = np.array([n.leaf for n in nodes], np.uint32)
    cword = np.array([n.const_word for n in nodes], np.uint64)
    nl = max(len(names), 1)
    keep, K, W, T = [], (C.c_void_p * nl)(), (C.c_void_p * nl)(), (C.c_void_p * nl)()
    lens, nil = np.zeros(nl, np.uint64), np.zeros(nl, np.uint8)
    total = 1
    for name, j in names.items():
        k, w, t, typ, isnil = algo.math_leaf_arrays(maps.get(name))
        if t is None:
            t = np.full(k.size, typ, np.uint8)
        keep += [k, w, t]
        K[j], W[j], T[j] = k.ctypes.data, w.ctypes.data, t.ctypes.data
        lens[j] = 0 if isnil else k.size
        nil[j] = isnil
        total += int(lens[j])
    r = np.zeros(1, np.uint64) if range_uids is None else np.ascontiguousarray(range_uids, np.uint64)
    nr = 0 if range_uids is None else r.size
    cap = max(total, nr, 1)
    ok, ow, ot = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64), np.zeros(cap, np.uint8)
    n, part = C.c_uint64(0), C.c_int(0)
    p = lambda a: a.ctypes.data if a.size else np.zeros(1, np.uint64).ctypes.data  # noqa: E731
    kind = lib().orc_math(p(op), p(ctag), p(child), p(leaf), p(cword), nn, K, W, T, lens.ctypes.data, nil.ctypes.data,
                          r.ctypes.data if r.size else None, nr, int(range_uids is not None), seed, ok.ctypes.data,
                          ow.ctypes.data, ot.ctypes.data, C.byref(n), C.byref(part))
    if kind < 0:
        return None, None, None, None, bool(part.value)
    m = n.value
    return algo.MATH_KIND[kind], ok[:m].copy(), ow[:m].copy(), ot[:m].copy(), bool(part.value)
