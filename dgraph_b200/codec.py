"""Host-side mirror of dgraph's `codec` package decode path over libdgx.

codec.Decode (codec/codec.go:444-452) and the ApproxLen / ExactLen helpers.
Decode is one C-ABI call (dgx_decode); the lengths are metadata sums over the
pack header, as in the reference.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

import numpy as np

from . import _lib
from .pb import List, UidPack


def view_of(pack: UidPack) -> _lib.PackView:
    """dgx_pack_view over the pack's arrays (keeps no references: caller keeps `pack` alive)."""
    v = _lib.PackView()
    v.block_size = int(pack.block_size)
    v.nblocks = pack.nblocks
    v.base = pack.base.ctypes.data
    v.num_uids = pack.num_uids.ctypes.data
    v.delta_off = pack.delta_off.ctypes.data
    v.deltas = pack.deltas.ctypes.data if pack.deltas.size else None
    return v


def ApproxLen(pack: Optional[UidPack]) -> int:
    """codec.ApproxLen (codec/codec.go:418-423)."""
    return 0 if pack is None else pack.nblocks * int(pack.block_size)


def ExactLen(pack: Optional[UidPack]) -> int:
    """codec.ExactLen (codec/codec.go:427-440)."""
    return 0 if pack is None or pack.nblocks == 0 else int(pack.num_uids.sum(dtype=np.uint64))


def Decode(pack: Optional[UidPack], seek: int) -> np.ndarray:
    """codec.Decode(pack, seek): uids from Seek(seek, SeekStart) onward; nil pack -> empty."""
    if pack is None or pack.nblocks == 0:
        return np.zeros(0, dtype=np.uint64)
    lib = _lib.load()
    pack = pack.normalized()
    cap = ExactLen(pack)
    out = np.empty(max(cap, 1), dtype=np.uint64)
    n = C.c_size_t(0)
    v = view_of(pack)
    _lib.check(lib.dgx_decode(C.byref(v), seek, out.ctypes.data_as(C.c_void_p), cap, C.byref(n)))
    return out[: n.value]


def DecodeIntersectSorted(pack: Optional[UidPack], seek: int, lists: Sequence[List]) -> List:
    """codec.Decode(pack, seek) then algo.IntersectSorted([decoded] + lists), fused on the device."""
    lib = _lib.load()
    arrs = [np.zeros(0, np.uint64) if l.Uids is None else l.Uids for l in lists]
    k = len(arrs)
    ptrs = (C.c_void_p * max(k, 1))(*[a.ctypes.data if a.size else None for a in arrs])
    lens = (C.c_size_t * max(k, 1))(*[a.size for a in arrs])
    cap = min([a.size for a in arrs] + [ExactLen(pack)])
    out = np.empty(max(cap, 1), dtype=np.uint64)
    n = C.c_size_t(0)
    if pack is None or pack.nblocks == 0:
        vp = None
    else:
        pack = pack.normalized()
        v = view_of(pack)
        vp = C.byref(v)
    _lib.check(lib.dgx_decode_intersect_sorted(vp, seek, ptrs, lens, k, out.ctypes.data_as(C.c_void_p), cap, C.byref(n)))
    return List(out[: n.value])


SeekStart, SeekCurrent = 0, 1  # codec.SeekStart / codec.SeekCurrent (codec/codec.go:29-36)
_SK_SEEK, _SK_SEEK_TO_BLOCK, _SK_LINEAR_SEEK, _SK_NEXT, _SK_UNPACK = range(5)


class Decoder:
    """codec.Decoder (codec/codec.go:139-384) over libdgx: every positioned call is ONE C-ABI call
    (dgx_pack_seek) evaluated on the device; this object only carries what the Go struct carries
    between calls -- the pack, blockIdx and the current uid slice."""

    def __init__(self, pack: Optional[UidPack]):
        self.Pack = None if pack is None else pack.normalized()
        self.blockIdx = 0
        self.uids = np.zeros(0, dtype=np.uint64)

    def _call(self, kind: int, uid: int = 0, whence: int = 0) -> np.ndarray:
        if self.Pack is None or self.Pack.nblocks == 0:
            self.uids = np.zeros(0, dtype=np.uint64)
            return self.uids
        lib = _lib.load()
        cap = max(int(self.Pack.num_uids.max()), 1)
        out = np.empty(cap, dtype=np.uint64)
        n, blk = C.c_size_t(0), C.c_size_t(0)
        v = view_of(self.Pack)
        _lib.check(lib.dgx_pack_seek(C.byref(v), kind, uid, whence, self.blockIdx,
                                     out.ctypes.data_as(C.c_void_p), cap, C.byref(n), C.byref(blk)))
        self.blockIdx = blk.value
        self.uids = out[: n.value]
        return self.uids

    def UnpackBlock(self) -> np.ndarray:
        return self._call(_SK_UNPACK)

    def Seek(self, uid: int, whence: int) -> np.ndarray:
        return self._call(_SK_SEEK, uid, whence)

    def SeekToBlock(self, uid: int, whence: int) -> np.ndarray:
        return self._call(_SK_SEEK_TO_BLOCK, uid, whence)

    def LinearSeek(self, seek: int) -> np.ndarray:
        return self._call(_SK_LINEAR_SEEK, seek)

    def Next(self) -> np.ndarray:
        return self._call(_SK_NEXT)

    def Uids(self) -> np.ndarray:
        return self.uids

    def BlockIdx(self) -> int:
        return self.blockIdx

    def Valid(self) -> bool:
        return self.Pack is not None and self.blockIdx < self.Pack.nblocks

    def PeekNextBase(self) -> int:
        b = self.blockIdx + 1
        if self.Pack is not None and b < self.Pack.nblocks:
            return int(self.Pack.base[b])
        return 0xFFFFFFFFFFFFFFFF

    def ApproxLen(self) -> int:
        return 0 if self.Pack is None else int(self.Pack.block_size) * (self.Pack.nblocks - self.blockIdx)


def _pack_out_arrays(n_uids: int, block_size: int):
    lib = _lib.load()
    nb_cap, db_cap = C.c_size_t(0), C.c_size_t(0)
    lib.dgx_encode_bound(n_uids, block_size, C.byref(nb_cap), C.byref(db_cap))
    return nb_cap.value, db_cap.value


def _call_pack_out(fn, n_uids: int, block_size: int) -> Optional[UidPack]:
    """Run `fn(base, num, doff, deltas, &nblocks, &delta_bytes, &view)`, growing the arrays once on DGX_ERR_CAP (the
    sizes it returns suffice, so a second DGX_ERR_CAP is an error)."""
    nb_cap, db_cap = _pack_out_arrays(n_uids, block_size)
    for _ in range(2):
        base = np.empty(max(nb_cap, 1), np.uint64)
        num = np.empty(max(nb_cap, 1), np.uint32)
        doff = np.zeros(max(nb_cap, 1) + 1, np.uint64)
        deltas = np.empty(max(db_cap, 1), np.uint8)
        nb, db = C.c_size_t(nb_cap), C.c_size_t(db_cap)
        view = _lib.PackView()
        rc = fn(base.ctypes.data_as(C.c_void_p), num.ctypes.data_as(C.c_void_p), doff.ctypes.data_as(C.c_void_p),
                deltas.ctypes.data_as(C.c_void_p), C.byref(nb), C.byref(db), C.byref(view))
        if rc == -4 and (nb.value > nb_cap or db.value > db_cap):   # DGX_ERR_CAP: exact sizes came back
            nb_cap, db_cap = max(nb_cap, nb.value), max(db_cap, db.value)
            continue
        _lib.check(rc)
        if nb.value == 0:
            return None   # the nil pack
        return UidPack(block_size, base[: nb.value].copy(), num[: nb.value].copy(), doff[: nb.value + 1].copy(),
                       deltas[: db.value].copy())
    raise _lib.DgxError(-4, "pack output did not fit after resizing")


def Encode(uids, blockSize: int) -> Optional[UidPack]:
    """codec.Encode(uids, blockSize) (codec/codec.go:393-399) on the device; no uids -> nil pack (None)."""
    lib = _lib.load()
    u = np.ascontiguousarray(np.asarray(uids, dtype=np.uint64))
    if u.size == 0:
        return None
    return _call_pack_out(lambda b, n, d, dl, pnb, pdb, pv: lib.dgx_encode(
        u.ctypes.data_as(C.c_void_p), u.size, blockSize, b, n, d, dl, pnb, pdb, pv), u.size, blockSize)
