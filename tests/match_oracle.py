"""ctypes binding of match_oracle.c: handleMatchFunction with uidsForMatch, matchFuzzy and levenshteinDistance
(worker/task.go:1526-1620, worker/match.go:24-100) restated line by line.  TEST INFRASTRUCTURE ONLY: the checker of
dgx_match / dgx_dev_match in tests/ and smoke(), and the CPU legs of tools/bench_ops.py C21.

A column is a dgraph_b200.algo.StrColumn.  Trigram leaves are given as trigram_oracle.py takes them: a pack leaf is
(pack, mut) or (pack, mut, approx_len) with an oracle.pyoracle.Pack or None, a list leaf an ascending array.

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
_SRCS = [os.path.join(_HERE, "match_oracle.c"), os.path.join(os.path.dirname(_HERE), "oracle", "oracle.c")]
_DEPS = [os.path.join(_HERE, f) for f in ("list_uids_unfiltered_oracle.c", "list_uids_oracle.c")] + [
    os.path.join(os.path.dirname(_HERE), "oracle", "oracle.h")]

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    h = hashlib.sha256()
    for f in _SRCS + _DEPS:
        with open(f, "rb") as fh:
            h.update(fh.read())
    so = os.path.join(tempfile.gettempdir(), f"dgx_match_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-o", tmp] + _SRCS)
        os.replace(tmp, so)  # atomic: concurrent test processes never load a half-written file
    L = C.CDLL(so)
    L.orc_match.argtypes = [C.c_void_p] * 4 + [C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64, C.c_void_p,
                                               C.c_size_t] + [C.c_void_p] * 4 + [C.c_size_t, C.c_void_p, C.c_size_t,
                                                                                 C.c_int64, C.c_void_p]
    L.orc_match.restype = C.c_size_t
    L.orc_levenshtein.argtypes = [C.c_char_p, C.c_size_t, C.c_char_p, C.c_size_t]
    L.orc_levenshtein.restype = C.c_int64
    _lib = L
    return L


def _b(x) -> bytes:
    return x.encode() if isinstance(x, str) else bytes(x)


def levenshtein(s, t) -> int:
    """levenshteinDistance(s, t)."""
    s, t = _b(s), _b(t)
    return int(lib().orc_levenshtein(s, len(s), t, len(t)))


def _csr(arrs, dtype):
    off = np.zeros(len(arrs) + 1, np.uint64)
    np.cumsum([len(a) for a in arrs], out=off[1:])
    flat = np.concatenate([np.asarray(a, dtype) for a in arrs]) if int(off[-1]) else np.zeros(1, dtype)
    return np.ascontiguousarray(flat), off


class Call:
    """The arguments of one call, prepared once (the bench times the call itself)."""

    def __init__(self, col, query, threshold: int, uids=None, leaves=()):
        self.col = col
        self.q = _b(query)
        self.max = threshold
        self.uids = np.ascontiguousarray(np.zeros(0, np.uint64) if uids is None else np.asarray(uids, np.uint64))
        pack_ids = [j for j, lf in enumerate(leaves) if isinstance(lf, tuple)]
        list_ids = [j for j, lf in enumerate(leaves) if not isinstance(lf, tuple)]
        self.packs = [leaves[j][0] for j in pack_ids]
        self.handles = (C.c_void_p * max(len(pack_ids), 1))(
            *[C.cast(p.handle(), C.c_void_p) if p is not None else None for p in self.packs])
        muts = [leaves[j][1] for j in pack_ids]
        self.mu, self.mut_off = _csr([np.zeros(0, np.uint64) if m is None else m[0] for m in muts], np.uint64)
        self.mf, _ = _csr([np.zeros(0, np.uint8) if m is None else m[1] for m in muts], np.uint8)
        self.lists, self.list_off = _csr([np.asarray(leaves[j], np.uint64) for j in list_ids], np.uint64)
        self.npacks, self.nlists = len(pack_ids), len(list_ids)
        bounds = [(int(p.num_uids.sum(dtype=np.uint64)) if p is not None else 0) for p in self.packs]
        self.cap = max(self.uids.size if self.uids.size else
                        sum(bounds) + int(self.mut_off[-1]) + int(self.list_off[-1]), 1)

    def run(self, after: int = 0, out: np.ndarray | None = None) -> np.ndarray:
        out = np.empty(self.cap, np.uint64) if out is None else out
        c = self.col
        u = self.uids if self.uids.size else np.zeros(1, np.uint64)
        qb = np.frombuffer(self.q + b"\0", np.uint8)
        n = lib().orc_match(C.cast(self.handles, C.c_void_p), self.mu.ctypes.data, self.mf.ctypes.data,
                            self.mut_off.ctypes.data, self.npacks, self.lists.ctypes.data, self.list_off.ctypes.data,
                            self.nlists, after, u.ctypes.data, self.uids.size, c.uid.ctypes.data,
                            c.val_off.ctypes.data, c.byte_off.ctypes.data, c.bytes.ctypes.data, c.uid.size,
                            qb.ctypes.data, len(self.q), self.max, out.ctypes.data)
        return out[:n].copy()



def match(col, query, threshold: int, uids=None, leaves=(), after: int = 0) -> np.ndarray:
    """handleMatchFunction's one result row: the candidates (uids when non-empty, else uidsForMatch over the leaves
    from after) whose values pass matchFuzzy(query, val, threshold)."""
    return Call(col, query, threshold, uids, leaves).run(after)
