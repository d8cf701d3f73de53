"""ctypes binding of backup_codec_oracle.c: codec.DecodeToBuffer / codec.EncodeFromBuffer and encoding/binary's
PutUvarint / Uvarint, restated on top of the CPU oracle (oracle/oracle.c).  TEST INFRASTRUCTURE ONLY: the checker of
dgx_decode_to_buffer_rows and dgx_encode_from_buffer_rows in tests/ and smoke(), and the CPU legs of
tools/bench_ops.py C11.

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
_ROOT = os.path.dirname(_HERE)
_SRCS = [os.path.join(_HERE, "backup_codec_oracle.c"), os.path.join(_ROOT, "oracle", "oracle.c")]
_DEPS = [os.path.join(_ROOT, "oracle", "oracle.h")]

OVERFLOW, TRUNCATED = -1, -2  # orc_encode_from_buffer: where the reference panics / loops forever

_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    h = hashlib.sha256()
    for f in _SRCS + _DEPS:
        with open(f, "rb") as fh:
            h.update(fh.read())
    so = os.path.join(tempfile.gettempdir(), f"dgx_backup_codec_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        tmp = f"{so}.{os.getpid()}.tmp"
        cc = os.environ.get("CC", "gcc")
        subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-pthread", "-shared", "-o", tmp] + _SRCS)
        os.replace(tmp, so)  # atomic: concurrent test processes never load a half-written file
    L = C.CDLL(so)
    L.orc_put_uvarint.argtypes = [C.c_void_p, C.c_uint64]
    L.orc_put_uvarint.restype = C.c_size_t
    L.orc_uvarint.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_long)]
    L.orc_uvarint.restype = C.c_uint64
    L.orc_decode_to_buffer.argtypes = [C.c_void_p, C.c_void_p]
    L.orc_decode_to_buffer.restype = C.c_size_t
    L.orc_encode_from_buffer.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_void_p)]
    L.orc_encode_from_buffer.restype = C.c_int
    _lib = L
    return L


def put_uvarint(x: int) -> bytes:
    out = np.zeros(16, np.uint8)
    n = lib().orc_put_uvarint(out.ctypes.data, x)
    return out[:n].tobytes()


def uvarint(buf: bytes):
    """binary.Uvarint(buf) -> (value, n)."""
    a = np.frombuffer(bytes(buf) + b"\0", np.uint8)
    n = C.c_long(0)
    v = lib().orc_uvarint(a.ctypes.data, len(buf), C.byref(n))
    return int(v), n.value


def decode_to_buffer(p) -> bytes:
    """codec.DecodeToBuffer(pack).  p: an oracle.pyoracle.Pack (nil or not)."""
    h = p.handle() if p is not None else None
    n = int(p.num_uids.sum(dtype=np.uint64)) if p is not None else 0
    out = np.zeros(10 * n + 1, np.uint8)
    k = lib().orc_decode_to_buffer(C.cast(h, C.c_void_p) if h else None, out.ctypes.data)
    return out[:k].tobytes()


def encode_from_buffer(buf: bytes, block_size: int):
    """codec.EncodeFromBuffer(buf, blockSize) -> (rc, oracle.pyoracle.Pack): rc 0, or OVERFLOW / TRUNCATED where the
    reference panics / never returns."""
    from oracle import pyoracle as orc

    a = np.frombuffer(bytes(buf) + b"\0", np.uint8)
    h = C.c_void_p(0)
    rc = lib().orc_encode_from_buffer(a.ctypes.data, len(buf), block_size, C.byref(h))
    return rc, orc.Pack(C.cast(h, C.POINTER(orc._Pack)) if h.value else None)
