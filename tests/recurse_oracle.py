"""ctypes binding of recurse_oracle.c: one sg of one level of @recurse (query/recurse.go expandRecurse :96-135) restated
line by line against a keyed reachMap.  TEST INFRASTRUCTURE ONLY: the checker of dgx_recurse_filter in tests/ and the
CPU leg of tools/bench_ops.py C14.

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

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "recurse_oracle.c"), os.path.join(os.path.dirname(_HERE), "oracle", "oracle.c")]
_DEPS = [os.path.join(os.path.dirname(_HERE), "oracle", "oracle.h")]

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    h = hashlib.sha256()
    for f in _SRCS + _DEPS:
        with open(f, "rb") as fh:
            h.update(fh.read())
    so = os.path.join(tempfile.gettempdir(), f"dgx_recurse_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-o", tmp] + _SRCS)
        os.replace(tmp, so)  # atomic: concurrent test processes never load a half-written file
    L = C.CDLL(so)
    vp, sz, u64 = C.c_void_p, C.c_size_t, C.c_uint64
    L.orc_reach_new.restype = vp
    L.orc_reach_new.argtypes = []
    L.orc_reach_free.argtypes = [vp]
    L.orc_reach_free.restype = None
    L.orc_reach_insert.argtypes = [vp, u64, u64, u64]
    L.orc_reach_insert.restype = C.c_int
    L.orc_reach_size.argtypes = [vp]
    L.orc_reach_size.restype = sz
    L.orc_reach_export.argtypes = [vp, u64, vp, vp]
    L.orc_reach_export.restype = sz
    L.orc_recurse_sg.argtypes = [vp, u64, vp, sz, vp, vp, C.c_int, vp, sz, C.c_int, vp, vp, vp, C.POINTER(sz)]
    L.orc_recurse_sg.restype = u64
    _lib = L
    return L


def csr(rows):
    """Rows as (flat uint64 values, uint64 offsets); the flat array has at least one element."""
    arrs = [np.asarray(r, np.uint64) for r in rows]
    off = np.zeros(len(arrs) + 1, np.uint64)
    np.cumsum([a.size for a in arrs], out=off[1:])
    flat = np.concatenate(arrs) if int(off[-1]) else np.zeros(1, np.uint64)
    return np.ascontiguousarray(flat), off


def _arr(a):
    a = np.ascontiguousarray(np.asarray(a, np.uint64))
    return a if a.size else np.zeros(1, np.uint64)


class Reach:
    """reachMap of one expandRecurse: the keys of every Attr (an integer per distinct Attr string)."""

    def __init__(self):
        self._h = lib().orc_reach_new()
        if not self._h:
            raise MemoryError("recurse oracle: allocation failed")

    def insert(self, attr: int, frm, to):
        for f, t in zip(np.asarray(frm, np.uint64).tolist(), np.asarray(to, np.uint64).tolist()):
            if lib().orc_reach_insert(self._h, attr, f, t) < 0:
                raise MemoryError("recurse oracle: allocation failed")

    def edges(self, attr: int):
        """(from, to) of one Attr's keys, ascending."""
        n = lib().orc_reach_size(self._h)
        f, t = np.empty(max(n, 1), np.uint64), np.empty(max(n, 1), np.uint64)
        k = lib().orc_reach_export(self._h, attr, f.ctypes.data, t.ctypes.data)
        o = np.lexsort((t[:k], f[:k]))
        return f[:k][o].copy(), t[:k][o].copy()

    def step(self, attr: int, src, rows, dest=None, allow_loop=False):
        """One sg (:102-134): (rows after the step, DestUIDs, numEdges added)."""
        v, v_off = csr(rows)
        m = int(v_off[-1])
        out, out_off = np.empty(max(m, 1), np.uint64), np.zeros(len(rows) + 1, np.uint64)
        dout, dlen = np.empty(max(m, 1), np.uint64), C.c_size_t(0)
        s, d = _arr(src), _arr([] if dest is None else dest)
        n = lib().orc_recurse_sg(self._h, attr, s.ctypes.data, len(rows), v.ctypes.data, v_off.ctypes.data,
                                 dest is not None, d.ctypes.data, 0 if dest is None else len(dest), bool(allow_loop),
                                 out.ctypes.data, out_off.ctypes.data, dout.ctypes.data, C.byref(dlen))
        if n == (1 << 64) - 1:
            raise MemoryError("recurse oracle: allocation failed")
        kept = [out[int(out_off[i]):int(out_off[i + 1])].copy() for i in range(len(rows))]
        return kept, dout[:dlen.value].copy(), int(n)

    def close(self):
        if self._h:
            lib().orc_reach_free(self._h)
            self._h = None

    def __del__(self):
        self.close()
