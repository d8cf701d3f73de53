"""ctypes binding of groupby_oracle.c: @groupby over one uid attribute (query/groupby.go formResult, formGroups,
groupLess, fillGroupedVars) restated line by line.  TEST INFRASTRUCTURE ONLY: the checker of dgx_groupby_uid in tests/
and the CPU leg of tools/bench_ops.py C13.

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
_SRC = os.path.join(_HERE, "groupby_oracle.c")

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    with open(_SRC, "rb") as fh:
        h = hashlib.sha256(fh.read()).hexdigest()[:16]
    so = os.path.join(tempfile.gettempdir(), f"dgx_groupby_oracle_{os.getuid()}_{h}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-shared", "-o", tmp, _SRC])
        os.replace(tmp, so)  # atomic: concurrent test processes never load a half-written file
    L = C.CDLL(so)
    L.orc_groupby_uid.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orc_groupby_uid.restype = C.c_size_t
    _lib = L
    return L


def csr(rows):
    """Rows as (flat uint64 values, uint64 offsets); the flat array has at least one element."""
    arrs = [np.asarray(r, np.uint64) for r in rows]
    off = np.zeros(len(arrs) + 1, np.uint64)
    np.cumsum([a.size for a in arrs], out=off[1:])
    flat = np.concatenate(arrs) if int(off[-1]) else np.zeros(1, np.uint64)
    return np.ascontiguousarray(flat), off


class Call:
    """The arguments of one call, prepared once (the bench times the call itself)."""

    def __init__(self, parents, src, rows):
        self.src = np.ascontiguousarray(np.asarray(src, np.uint64)) if len(src) else np.zeros(1, np.uint64)
        self.nrows = len(rows)
        self.v, self.v_off = csr(rows)
        self.par, self.par_off = csr(parents)
        self.npar = len(parents)
        # room: every (parent, source) pair a parent reaches is one row's values
        lens = np.diff(self.v_off.astype(np.int64))
        s = np.asarray(src, np.uint64)
        self.cap = max(sum(int(lens[np.isin(s, np.asarray(pr, np.uint64))].sum()) for pr in parents), 1)

    def run(self):
        """(keys, count(uid), grp_off, mem_off, members) of every parent's ordered groups."""
        keys, agg = np.empty(self.cap, np.uint64), np.empty(self.cap, np.uint64)
        mem, mem_off = np.empty(self.cap, np.uint64), np.empty(self.cap + 1, np.uint64)
        grp_off = np.empty(self.npar + 1, np.uint64)
        n = lib().orc_groupby_uid(self.src.ctypes.data, self.nrows, self.v.ctypes.data, self.v_off.ctypes.data,
                                  self.par.ctypes.data, self.par_off.ctypes.data, self.npar, keys.ctypes.data,
                                  agg.ctypes.data, grp_off.ctypes.data, mem_off.ctypes.data, mem.ctypes.data)
        if n == (1 << 64) - 1:
            raise MemoryError("groupby oracle: allocation failed")
        if self.npar == 0:
            grp_off[0] = 0
        return keys[:n].copy(), agg[:n].copy(), grp_off, mem_off[:n + 1].copy(), mem[:int(mem_off[n])].copy()


def groupby_uid(parents, src, rows):
    """formResult for every parent row of sg.uidMatrix: (keys, counts, grp_off, mem_off, members), as dgx_groupby_uid
    lays them out."""
    return Call(parents, src, rows).run()


def grouped_vars(src, rows) -> dict:
    """fillGroupedVars for `f as count(uid)`: key -> the last (only) aggregate, over every child row."""
    keys, agg, _, _, _ = groupby_uid([src], src, rows)
    return {int(k): int(a) for k, a in zip(keys, agg)}
