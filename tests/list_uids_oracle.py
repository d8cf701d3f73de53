"""ctypes binding of list_uids_oracle.c: posting.List.Uids of one unsplit list restated line by line on top of the CPU
oracle (oracle/oracle.c).  TEST INFRASTRUCTURE ONLY: the checker of dgx_list_uids_rows in tests/ and smoke(), and the
CPU legs of tools/bench_ops.py C9.

The library is compiled on first use from list_uids_oracle.c and oracle/oracle.c into the temporary directory (the
tree itself may be read-only), under a name keyed by the sources' contents.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "list_uids_oracle.c"), os.path.join(os.path.dirname(_HERE), "oracle", "oracle.c")]
_HDR = os.path.join(os.path.dirname(_HERE), "oracle", "oracle.h")

COMPRESSED, PROBE, ITERATE = 0, 1, 2
MUT_DEL, MUT_VALUE = 1, 2

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    h = hashlib.sha256()
    for f in _SRCS + [_HDR]:
        with open(f, "rb") as fh:
            h.update(fh.read())
    so = os.path.join(tempfile.gettempdir(), f"dgx_list_uids_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-o", tmp] + _SRCS)
        os.replace(tmp, so)  # atomic: concurrent test processes never load a half-written file
    L = C.CDLL(so)
    L.orc_list_uids.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p,
                                C.c_size_t, C.c_void_p]
    L.orc_list_uids.restype = C.c_size_t
    _lib = L
    return L


def list_uids(p, mode: int, mut_uids, mut_flags, after_uid: int, v) -> np.ndarray:
    """List.Uids of one unsplit list (posting/list.go:1758-1874) with Intersect = v, branch `mode`, the mutable layer
    resolved to one (uid, flags) entry per uid.  p: an oracle.pyoracle.Pack, or None for a delete-all marker (or an
    empty immutable layer)."""
    v = np.ascontiguousarray(np.asarray(v, dtype=np.uint64))
    mu = np.ascontiguousarray(np.asarray(mut_uids, dtype=np.uint64))
    mf = np.ascontiguousarray(np.asarray(mut_flags, dtype=np.uint8))
    assert mu.size == mf.size
    out = np.empty(max(v.size, 1), dtype=np.uint64)
    h = p.handle() if p is not None else None
    hp = C.cast(h, C.c_void_p) if h else None
    n = lib().orc_list_uids(hp, mode, mu.ctypes.data, mf.ctypes.data, mu.size, after_uid, v.ctypes.data, v.size,
                            out.ctypes.data)
    return out[:n].copy()
