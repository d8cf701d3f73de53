"""ctypes binding of trigram_oracle.c: uidsForRegex (worker/trigram.go:24-102) restated line by line on top of the
List.Uids restatements.  TEST INFRASTRUCTURE ONLY: the checker of dgx_trigram_query in tests/ and the CPU legs of
tools/bench_ops.py C12.

Leaves are given as the product's algo.UidsForRegex takes them, with oracle packs: a pack leaf is (pack, mut) or
(pack, mut, approx_len) -- pack an oracle.pyoracle.Pack or None, mut None or (uids, flags) -- and a list leaf is an
ascending array.  approx_len picks the branch of each filtered read (probe when len(Intersect) < approx_len); it
defaults to ExactLen + |mut|, the reference's ApproxLen up to the pack's BlockSize rounding.

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
_SRCS = [os.path.join(_HERE, "trigram_oracle.c"), os.path.join(os.path.dirname(_HERE), "oracle", "oracle.c")]
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
    so = os.path.join(tempfile.gettempdir(), f"dgx_trigram_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-o", tmp] + _SRCS)
        os.replace(tmp, so)  # atomic: concurrent test processes never load a half-written file
    L = C.CDLL(so)
    L.orc_uids_for_regex.argtypes = [C.c_void_p] * 10 + [C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_uint64,
                                                          C.c_void_p]
    L.orc_uids_for_regex.restype = C.c_size_t
    _lib = L
    return L


def _csr(arrs, dtype):
    off = np.zeros(len(arrs) + 1, np.uint64 if dtype == np.uint64 else np.uint32)
    np.cumsum([len(a) for a in arrs], out=off[1:])
    flat = np.concatenate([np.asarray(a, dtype) for a in arrs]) if int(off[-1]) else np.zeros(1, dtype)
    return np.ascontiguousarray(flat), off


class Query:
    """The arguments of one call, prepared once (the bench times the call itself)."""

    def __init__(self, tree, leaves):
        pack_ids = [j for j, lf in enumerate(leaves) if isinstance(lf, tuple)]
        list_ids = [j for j, lf in enumerate(leaves) if not isinstance(lf, tuple)]
        order = {j: k for k, j in enumerate(pack_ids + list_ids)}  # the ABI's numbering: pack leaves first
        self.op = np.array([t[0] for t in tree] or [0], np.uint8)
        self.leaf_idx, self.leaf_off = _csr([[order[j] for j in t[1]] for t in tree], np.uint32)
        self.sub_idx, self.sub_off = _csr([list(t[2]) for t in tree], np.uint32)
        self.packs = [leaves[j][0] for j in pack_ids]
        self.handles = (C.c_void_p * max(len(pack_ids), 1))(
            *[C.cast(p.handle(), C.c_void_p) if p is not None else None for p in self.packs])
        muts = [leaves[j][1] for j in pack_ids]
        self.mu, self.mut_off = _csr([np.zeros(0, np.uint64) if m is None else m[0] for m in muts], np.uint64)
        self.mf, _ = _csr([np.zeros(0, np.uint8) if m is None else m[1] for m in muts], np.uint8)
        nmut = np.diff(self.mut_off.astype(np.int64))
        self.approx = np.array([leaves[j][2] if len(leaves[j]) > 2 else
                                (int(p.num_uids.sum(dtype=np.uint64)) if p is not None else 0) + int(nmut[k])
                                for k, (j, p) in enumerate(zip(pack_ids, self.packs))] or [0], np.uint64)
        self.lists, self.list_off = _csr([np.asarray(leaves[j], np.uint64) for j in list_ids], np.uint64)
        self.npacks, self.nlists = len(pack_ids), len(list_ids)
        bounds = [(int(p.num_uids.sum(dtype=np.uint64)) if p is not None else 0) + int(nmut[k])
                  for k, p in enumerate(self.packs)] + list(np.diff(self.list_off.astype(np.int64)))
        self.cap = max(sum(bounds), 1)  # the root's result lies in the union of all leaves

    def run(self, after: int, out: np.ndarray | None = None) -> np.ndarray:
        out = np.empty(self.cap, np.uint64) if out is None else out
        n = lib().orc_uids_for_regex(
            self.op.ctypes.data, self.leaf_off.ctypes.data, self.leaf_idx.ctypes.data, self.sub_off.ctypes.data,
            self.sub_idx.ctypes.data, C.cast(self.handles, C.c_void_p), self.mu.ctypes.data, self.mf.ctypes.data,
            self.mut_off.ctypes.data, self.approx.ctypes.data, self.npacks, self.lists.ctypes.data,
            self.list_off.ctypes.data, self.nlists, after, out.ctypes.data)
        if n == (1 << 64) - 1:
            raise ValueError("errRegexTooWide: a node that is neither QAnd nor QOr")
        return out[:n].copy()


def uids_for_regex(tree, leaves, after: int) -> np.ndarray:
    """uidsForRegex(attr, arg, query, &pb.List{}) with arg.q.First = MaxInt32 and arg.q.AfterUid = after."""
    return Query(tree, leaves).run(after)
