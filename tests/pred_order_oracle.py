"""ctypes binding of pred_order_oracle.c: ordering a uid matrix by a predicate without its index (query/query.go
applyOrderAndPagination's predicate branch, worker/sort.go sortWithoutIndex, sortByValue, paginate, types.Sort and
Go's pdqsort) restated line by line.  TEST INFRASTRUCTURE ONLY: the checker of dgx_pred_order in tests/.

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

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "pred_order_oracle.c")

_lib = None


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("insertion", "heap", "partition", "partition_equal", "partial_insertion",
                                          "partial_insertion_ok", "break_patterns", "reverse")]


class NotSortable(ValueError):
    """Go's "Value of type: bool isn't sortable"."""


class NegativeCount(ValueError):
    """processSort's "We do not yet support negative or infinite count with sorting"."""


class ListPredicate(ValueError):
    """processSort's "Sorting not supported on attr ... of type: [scalar]"."""


def lib():
    global _lib
    if _lib is not None:
        return _lib
    with open(_SRC, "rb") as fh:
        h = hashlib.sha256(fh.read()).hexdigest()[:16]
    so = os.path.join(tempfile.gettempdir(), f"dgx_pred_order_oracle_{os.getuid()}_{h}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-std=gnu11", "-shared", "-o", tmp, _SRC])
        os.replace(tmp, so)  # atomic: concurrent test processes never load a half-written file
    L = C.CDLL(so)
    vp, sz = C.c_void_p, C.c_size_t
    L.orc_pred_order.argtypes = [C.c_int, vp, vp, sz, vp, vp, vp, vp, vp, C.c_int, vp, sz, vp, vp, sz, C.c_int32,
                                 C.c_int32, vp, vp, vp, C.POINTER(sz)]
    L.orc_pred_order.restype = C.c_int
    L.orc_pred_order_stats.argtypes = [C.POINTER(Stats), C.c_int]
    L.orc_pred_order_stats.restype = None
    _lib = L
    return L


def _nz(a, dt):
    a = np.ascontiguousarray(a, dt)
    return a if a.size else np.zeros(1, dt)


def pred_order(col, desc, dest, rows, count=0, offset=0):
    """(rows, dest) of the restatement for an algo.ValColumn.  Raises NotSortable, NegativeCount or ListPredicate where
    Go returns an error."""
    dest = np.ascontiguousarray(np.asarray(dest, np.uint64))
    rows = [np.asarray(r, np.uint64) for r in rows]
    nrows = len(rows)
    v_off = np.zeros(nrows + 1, np.uint64)
    np.cumsum([r.size for r in rows], out=v_off[1:])
    M = int(v_off[-1])
    v = _nz(np.concatenate(rows) if M else np.zeros(0, np.uint64), np.uint64)
    out = np.empty(max(M, 1), np.uint64)
    out_off = np.zeros(nrows + 1, np.uint64)
    dout = np.empty(max(dest.size, 1), np.uint64)
    dn = C.c_size_t(0)
    uid, voff = _nz(col.uid, np.uint64), np.ascontiguousarray(col.val_off, np.uint64)
    if col.str is not None:
        boff, byts = np.ascontiguousarray(col.str.byte_off, np.uint64), _nz(col.str.bytes, np.uint8)
        word = nsec = None
    else:
        boff = byts = None
        word = _nz(col.word, np.uint64)
        nsec = None if col.nsec is None else _nz(col.nsec, np.uint32)
    bad = None if col.bad is None else _nz(col.bad, np.uint8)
    ad = lambda a: None if a is None else a.ctypes.data  # noqa: E731
    dd = _nz(dest, np.uint64)
    rc = lib().orc_pred_order(col.type, uid.ctypes.data, voff.ctypes.data, col.uid.size, ad(word), ad(nsec),
                              ad(boff), ad(byts), ad(bad), int(bool(desc)), dd.ctypes.data, dest.size, v.ctypes.data,
                              v_off.ctypes.data, nrows, count, offset, out.ctypes.data, out_off.ctypes.data,
                              dout.ctypes.data, C.byref(dn))
    if rc == 1:
        raise NotSortable("isn't sortable")
    if rc == 2:
        raise NegativeCount("negative count")
    if rc == 3:
        raise ListPredicate("list predicate")
    if rc != 0:
        raise MemoryError("pred_order oracle: allocation failed")
    return [out[int(out_off[i]):int(out_off[i + 1])].copy() for i in range(nrows)], dout[:dn.value].copy()


def stats(reset=True) -> dict:
    """Which pdqsort helpers ran since the last reset (per thread)."""
    s = Stats()
    lib().orc_pred_order_stats(C.byref(s), int(reset))
    return {n: getattr(s, n) for n, _ in Stats._fields_}
