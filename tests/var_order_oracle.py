"""ctypes binding of var_order_oracle.c: ordering a uid matrix by a value variable (query/query.go
applyOrderAndPagination's value-variable branch, sortAndPaginateUsingVar, updateDestUids, types.Sort and Go's pdqsort)
restated line by line.  TEST INFRASTRUCTURE ONLY: the checker of dgx_var_order in tests/ and the CPU leg of
tools/bench_ops.py C20.

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
_SRC = os.path.join(_HERE, "var_order_oracle.c")
T_INT, T_FLOAT, T_BOOL, T_NIL = 1, 2, 3, 4  # DGX_VAL_*

_lib = None


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("insertion", "heap", "partition", "partition_equal", "partial_insertion",
                                          "partial_insertion_ok", "break_patterns", "reverse")]


class NilMap(ValueError):
    """Go's "Variable: [x] used before definition." (a nil UidToVal)."""


class NotSortable(ValueError):
    """Go's "Value of type: bool isn't sortable" (a row's first entry is a bool)."""


def lib():
    global _lib
    if _lib is not None:
        return _lib
    with open(_SRC, "rb") as fh:
        h = hashlib.sha256(fh.read()).hexdigest()[:16]
    so = os.path.join(tempfile.gettempdir(), f"dgx_var_order_oracle_{os.getuid()}_{h}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-std=gnu11", "-shared", "-o", tmp, _SRC])
        os.replace(tmp, so)  # atomic: concurrent test processes never load a half-written file
    L = C.CDLL(so)
    vp, sz = C.c_void_p, C.c_size_t
    L.orc_var_order.argtypes = [vp, vp, vp, sz, C.c_int, C.c_int, vp, sz, vp, vp, sz, C.c_int32, C.c_int32, vp, vp,
                                vp, C.POINTER(sz)]
    L.orc_var_order.restype = C.c_int
    L.orc_var_order_sort.argtypes = [vp, vp, vp, sz, C.c_int]
    L.orc_var_order_sort.restype = C.c_int
    L.orc_var_order_stats.argtypes = [C.POINTER(Stats), C.c_int]
    L.orc_var_order_stats.restype = None
    _lib = L
    return L


def map_arrays(m):
    """(keys u64, words u64, tags u8, nil) of a map: None (Go's nil map), (keys, int64 or float64 values) or (keys,
    u64 words, u8 tags) as algo.EvalMath returns them."""
    if m is None:
        return np.zeros(0, np.uint64), np.zeros(0, np.uint64), np.zeros(0, np.uint8), 1
    if len(m) == 3:
        return (np.ascontiguousarray(m[0], np.uint64), np.ascontiguousarray(m[1], np.uint64),
                np.ascontiguousarray(m[2], np.uint8), 0)
    vals = np.asarray(m[1])
    if vals.dtype not in (np.int64, np.float64):
        raise TypeError(f"a value map holds int64 or float64 values, not {vals.dtype}")
    t = T_INT if vals.dtype == np.int64 else T_FLOAT
    return (np.ascontiguousarray(m[0], np.uint64), np.ascontiguousarray(vals).view(np.uint64).copy(),
            np.full(vals.size, t, np.uint8), 0)


def _nz(a, dt):
    a = np.ascontiguousarray(a, dt)
    return a if a.size else np.zeros(1, dt)


def var_order(m, desc, dest, rows, count=0, offset=0):
    """(rows, dest) of the restatement.  Raises NilMap or NotSortable where Go returns an error."""
    k, w, t, nil = map_arrays(m)
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
    kk, ww, tt, dd = _nz(k, np.uint64), _nz(w, np.uint64), _nz(t, np.uint8), _nz(dest, np.uint64)
    rc = lib().orc_var_order(kk.ctypes.data, ww.ctypes.data, tt.ctypes.data, k.size, nil, int(bool(desc)),
                             dd.ctypes.data, dest.size, v.ctypes.data, v_off.ctypes.data, nrows, count, offset,
                             out.ctypes.data, out_off.ctypes.data, dout.ctypes.data, C.byref(dn))
    if rc == 1:
        raise NilMap("used before definition")
    if rc == 2:
        raise NotSortable("isn't sortable")
    if rc != 0:
        raise MemoryError("var_order oracle: allocation failed")
    return [out[int(out_off[i]):int(out_off[i + 1])].copy() for i in range(nrows)], dout[:dn.value].copy()


def go_sort(tags, words, uids, desc):
    """sort.Sort(byValue) of one W in place: (words, uids) after the sort.  Raises NotSortable for a bool first."""
    t = _nz(tags, np.uint8)
    w = _nz(words, np.uint64).copy()
    u = _nz(uids, np.uint64).copy()
    n = len(tags)
    rc = lib().orc_var_order_sort(t.ctypes.data, w.ctypes.data, u.ctypes.data, n, int(bool(desc)))
    if rc == 2:
        raise NotSortable("isn't sortable")
    return w[:n], u[:n]


def stats(reset=True) -> dict:
    """Which pdqsort helpers ran since the last reset (per thread)."""
    s = Stats()
    lib().orc_var_order_stats(C.byref(s), int(reset))
    return {n: getattr(s, n) for n, _ in Stats._fields_}


PIN_KINDS, PIN_SIZES = ("mod13", "nil", "nanmix", "mixed"), (13, 50, 100, 1000, 5000)


def pin_inputs():
    """[(name, tags, words, desc)]: the fixed tied inputs tests/go_sort_pin/main.go sorts with Go's sort.Sort."""
    out = []
    for kind in PIN_KINDS:
        for n in PIN_SIZES:
            i = np.arange(n)
            if kind == "mod13":
                t, w = np.full(n, T_INT), ((i * 7919) % 13).astype(np.int64).view(np.uint64)
            elif kind == "nil":
                t, w = np.full(n, T_NIL), np.zeros(n, np.uint64)
            elif kind == "nanmix":
                f = np.where(i % 5 == 0, np.nan, ((i * 31) % 17).astype(np.float64))
                t, w = np.full(n, T_FLOAT), f.view(np.uint64)
            else:
                f = (i % 7).astype(np.float64).view(np.uint64)
                k = (i % 7).astype(np.int64).view(np.uint64)
                t = np.where(i % 3 == 0, T_FLOAT, np.where(i % 3 == 1, T_INT, T_NIL))
                w = np.where(i % 3 == 0, f, np.where(i % 3 == 1, k, 0)).astype(np.uint64)
            for desc in (False, True):
                out.append((f"{kind} {n} {'true' if desc else 'false'}", t.astype(np.uint8), w, desc))
    return out


def print_pins():
    """The restatement's lines in the format of tests/go_sort_pin/main.go."""
    for name, t, w, desc in pin_inputs():
        _, u = go_sort(t, w, np.arange(1, len(t) + 1, dtype=np.uint64), desc)
        print(f"{name}: {' '.join(str(int(x)) for x in u)}")
