"""ctypes binding of compare_oracle.c: types.CompareVals / Less / Equal and the two Go loops that call them
(handleValuePostings' compareAttrFn branch and handleCompareFunction's filterRow) restated line by line.  TEST
INFRASTRUCTURE ONLY: the checker of dgx_compare_uids / dgx_compare_rows and their device forms.

A column is a dgraph_b200.algo.ValColumn and arguments a dgraph_b200.algo.ValArgs.  The library is compiled on first
use into the temporary directory (the tree itself may be read-only), under a name keyed by the source's contents.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "compare_oracle.c")
_lib = None


class _Col(C.Structure):
    _fields_ = [("type", C.c_int), ("uid", C.c_void_p), ("val_off", C.c_void_p), ("word", C.c_void_p),
                ("nsec", C.c_void_p), ("bad", C.c_void_p), ("byte_off", C.c_void_p), ("bytes", C.c_void_p),
                ("n", C.c_size_t)]


class _Args(C.Structure):
    _fields_ = [("word", C.c_void_p), ("nsec", C.c_void_p), ("bytes", C.c_void_p), ("byte_off", C.c_void_p),
                ("n", C.c_size_t)]


def lib():
    global _lib
    if _lib is not None:
        return _lib
    with open(_SRC, "rb") as fh:
        h = hashlib.sha256(fh.read()).hexdigest()[:16]
    so = os.path.join(tempfile.gettempdir(), f"dgx_compare_oracle_{os.getuid()}_{h}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-std=c11", "-shared", "-o", tmp, _SRC])
        os.replace(tmp, so)  # atomic: concurrent test processes never load a half-written file
    L = C.CDLL(so)
    L.orc_compare_uids.argtypes = [C.c_int, C.POINTER(_Args), C.POINTER(_Col), C.c_void_p, C.c_size_t, C.c_void_p,
                                   C.c_void_p]
    L.orc_compare_uids.restype = C.c_long
    L.orc_compare_rows.argtypes = [C.c_int, C.POINTER(_Args), C.POINTER(_Col), C.c_void_p, C.c_void_p, C.c_size_t,
                                   C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_compare_rows.restype = C.c_size_t
    _lib = L
    return L


def _a(x):
    return None if x is None else x.ctypes.data


def _structs(col, args):
    from dgraph_b200 import algo

    a = args if isinstance(args, algo.ValArgs) else algo.ValArgs(col.type, args)
    s = col.str
    cs = _Col(col.type, _a(col.uid), _a(col.val_off), _a(col.word), _a(col.nsec), _a(col.bad),
              _a(s.byte_off) if s is not None else None, _a(s.bytes) if s is not None else None, col.uid.size)
    return cs, _Args(_a(a.word), _a(a.nsec), _a(a.bytes), _a(a.off), a.n), a


def compare_uids(col, op, args, uids):
    """(dest, row lengths) of the value path, or None where Go returns the conversion error."""
    from dgraph_b200 import algo

    u = np.ascontiguousarray(np.asarray(uids, np.uint64))
    cs, ast, keep = _structs(col, args)
    dest = np.empty(max(u.size, 1), np.uint64)
    rl = np.zeros(max(u.size, 1), np.uint32)
    n = lib().orc_compare_uids(algo.CMP_OPS[op] if isinstance(op, str) else op, C.byref(ast), C.byref(cs),
                               u.ctypes.data, u.size, dest.ctypes.data, rl.ctypes.data)
    if n < 0:
        return None
    return dest[:n].copy(), rl[: u.size].copy()


def compare_rows(col, op, args, rows, row_arg):
    """The index rows after filterRow on every row row_arg selects."""
    from dgraph_b200 import algo

    off = np.zeros(len(rows) + 1, np.uint64)
    np.cumsum([len(r) for r in rows], out=off[1:])
    v = np.ascontiguousarray(np.concatenate([np.asarray(r, np.uint64) for r in rows]) if int(off[-1])
                             else np.zeros(1, np.uint64))
    ra = np.ascontiguousarray(np.asarray(row_arg, np.uint32)) if len(rows) else np.zeros(1, np.uint32)
    cs, ast, keep = _structs(col, args)
    out = np.empty(max(int(off[-1]), 1), np.uint64)
    oo = np.zeros(len(rows) + 1, np.uint64)
    lib().orc_compare_rows(algo.CMP_OPS[op] if isinstance(op, str) else op, C.byref(ast), C.byref(cs), v.ctypes.data,
                           off.ctypes.data, len(rows), ra.ctypes.data, out.ctypes.data, oo.ctypes.data)
    return [out[int(oo[i]):int(oo[i + 1])].copy() for i in range(len(rows))]
