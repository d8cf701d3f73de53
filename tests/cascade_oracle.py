"""ctypes binding of cascade_oracle.c: @cascade over a forest (query/query.go populateVarMap :1445-1527, updateUidMatrix
:1425-1439, x.PageRange and ProcessQuery's root pagination :3004-3011) restated line by line.  TEST INFRASTRUCTURE ONLY:
the checker of dgx_cascade in tests/ and the CPU leg of tools/bench_ops.py C15.

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

from dgraph_b200.algo import cascade_arrays, cascade_split

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "cascade_oracle.c"), os.path.join(os.path.dirname(_HERE), "oracle", "oracle.c")]
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
    so = os.path.join(tempfile.gettempdir(), f"dgx_cascade_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-o", tmp] + _SRCS)
        os.replace(tmp, so)  # atomic: concurrent test processes never load a half-written file
    L = C.CDLL(so)
    vp = C.c_void_p
    L.orc_cascade.argtypes = [C.c_size_t] + [vp] * 16
    L.orc_cascade.restype = C.c_int
    _lib = L
    return L


def cascade_flat(a):
    """The restatement over the flat arrays of algo.cascade_arrays: (out, out_off, dest_out, dest_out_off)."""
    m, nd = int(a["v_off"][-1]), int(a["dest_off"][-1])
    out, dest_out = np.empty(max(m, 1), np.uint64), np.empty(max(nd, 1), np.uint64)
    out_off = np.zeros(int(a["row_off"][-1]) + 1, np.uint64)
    dest_off = np.zeros(a["nnodes"] + 1, np.uint64)
    args = [a[k].ctypes.data for k in ("parent", "flags", "first", "offset", "counts_len", "v", "v_off", "row_off",
                                       "dest", "dest_off", "has_val", "hv_off")]
    if lib().orc_cascade(a["nnodes"], *args, out.ctypes.data, out_off.ctypes.data, dest_out.ctypes.data,
                         dest_off.ctypes.data) != 0:
        raise MemoryError("cascade oracle: allocation failed")
    return out, out_off, dest_out, dest_off


def cascade(nodes):
    """([rows of each node], [dest of each node]) after @cascade, for a list of algo.CascadeNode."""
    a = cascade_arrays(nodes)
    return cascade_split(a, *cascade_flat(a))
