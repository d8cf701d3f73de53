"""ctypes binding of list_uids_unfiltered_oracle.c: posting.List.Uids with opts.Intersect == nil and the count of
List.Postings for one unsplit list, restated line by line on top of the CPU oracle (oracle/oracle.c) and the iterator
of list_uids_oracle.c.  TEST INFRASTRUCTURE ONLY: the checker of dgx_list_uids_unfiltered_rows and dgx_list_count_rows
in tests/ and smoke(), and the CPU legs of tools/bench_ops.py C10.

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
_SRCS = [os.path.join(_HERE, "list_uids_unfiltered_oracle.c"), os.path.join(os.path.dirname(_HERE), "oracle", "oracle.c")]
_DEPS = [os.path.join(_HERE, "list_uids_oracle.c"), os.path.join(os.path.dirname(_HERE), "oracle", "oracle.h")]

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    h = hashlib.sha256()
    for f in _SRCS + _DEPS:
        with open(f, "rb") as fh:
            h.update(fh.read())
    so = os.path.join(tempfile.gettempdir(), f"dgx_list_uids_unfiltered_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-o", tmp] + _SRCS)
        os.replace(tmp, so)  # atomic: concurrent test processes never load a half-written file
    L = C.CDLL(so)
    L.orc_list_uids_unfiltered.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_int32,
                                           C.c_void_p]
    L.orc_list_uids_unfiltered.restype = C.c_size_t
    L.orc_list_count.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64]
    L.orc_list_count.restype = C.c_size_t
    _lib = L
    return L


def _layer(p, mut_uids, mut_flags):
    mu = np.ascontiguousarray(np.asarray(mut_uids, dtype=np.uint64))
    mf = np.ascontiguousarray(np.asarray(mut_flags, dtype=np.uint8))
    assert mu.size == mf.size
    h = p.handle() if p is not None else None
    return (C.cast(h, C.c_void_p) if h else None), mu, mf


def list_uids_unfiltered(p, mut_uids, mut_flags, after_uid: int, first: int = 0) -> np.ndarray:
    """List.Uids of one unsplit list with Intersect == nil (posting/list.go:1758-1874): iterate with the REF filter
    above after_uid, then the cut of opts.First (an int32: 0 is MaxInt32).  p: an oracle.pyoracle.Pack, or None for a
    delete-all marker (or an empty immutable layer); the mutable layer resolved to one (uid, flags) entry per uid."""
    hp, mu, mf = _layer(p, mut_uids, mut_flags)
    out = np.empty((int(p.num_uids.sum(dtype=np.uint64)) if p is not None else 0) + mu.size + 1, dtype=np.uint64)
    n = lib().orc_list_uids_unfiltered(hp, mu.ctypes.data, mf.ctypes.data, mu.size, after_uid, first, out.ctypes.data)
    return out[:n].copy()


def list_count(p, mut_uids, mut_flags, after_uid: int) -> int:
    """countForUidPostings with a nil facets tree: the REF postings List.Postings yields above after_uid."""
    hp, mu, mf = _layer(p, mut_uids, mut_flags)
    return int(lib().orc_list_count(hp, mu.ctypes.data, mf.ctypes.data, mu.size, after_uid))
