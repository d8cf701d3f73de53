"""Fixtures shared by the backup codec tests: hand-built packs (the oracle's pack struct over numpy arrays) and the
uid lists whose packs reach every edge of DecodeToBuffer / EncodeFromBuffer."""
from __future__ import annotations

import ctypes as C
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(__file__))
import gen  # noqa: E402

M64 = (1 << 64) - 1


class HandPack:
    """An oracle pack over caller-owned arrays (oracle.pyoracle.Pack would free them): base, NumUids, delta_off and the
    delta bytes of any block table, including ones codec.Encode never writes."""

    def __init__(self, block_size, base, num_uids, delta_off, deltas):
        from oracle import pyoracle as orc

        self.block_size = int(block_size)
        self.base = np.ascontiguousarray(base, np.uint64)
        self.num_uids = np.ascontiguousarray(num_uids, np.uint32)
        self.delta_off = np.ascontiguousarray(delta_off, np.uint64)
        self.deltas = np.zeros(int(self.delta_off[-1]) + 32, np.uint8)
        self.deltas[: int(self.delta_off[-1])] = np.asarray(deltas, np.uint8)
        self.nblocks = self.base.size
        s = orc._Pack()
        s.block_size, s.nblocks = self.block_size, self.nblocks
        s.base = self.base.ctypes.data_as(C.POINTER(C.c_uint64))
        s.num_uids = self.num_uids.ctypes.data_as(C.POINTER(C.c_uint32))
        s.delta_off = self.delta_off.ctypes.data_as(C.POINTER(C.c_uint64))
        s.deltas = self.deltas.ctypes.data_as(C.POINTER(C.c_uint8))
        self._s = s

    def handle(self):
        return C.pointer(self._s)

    def uid_pack(self):
        from dgraph_b200 import pb

        return pb.UidPack(self.block_size, self.base, self.num_uids, self.delta_off,
                          self.deltas[: int(self.delta_off[-1])])


def pack_of(uids, block_size):
    """HandPack of codec.Encode(uids, block_size) (tests/gen.py's numpy encoder); None for no uids."""
    p = gen.encode_pack_np(np.asarray(uids, np.uint64), block_size)
    return None if p is None else HandPack(*p)


def group(vals):
    """One go-groupvarint group of four u32 values."""
    lens = [1 if v < 1 << 8 else 2 if v < 1 << 16 else 3 if v < 1 << 24 else 4 for v in vals]
    tag = lens[0] - 1 | (lens[1] - 1) << 2 | (lens[2] - 1) << 4 | (lens[3] - 1) << 6
    out = [tag]
    for v, l in zip(vals, lens):
        out += [(v >> (8 * t)) & 0xFF for t in range(l)]
    return out


def wrap_pack():
    """Two blocks: the first one's running sum wraps past 2^64 (base 2^64 - 3, delta 5 -> uid 2), the second one starts
    below the first one's last uid: both boundary and internal deltas wrap."""
    return HandPack(256, [M64 - 2, 1 << 40], [2, 3], [0, 5, 12], group([5, 0, 0, 0]) + group([7, 1 << 20, 0, 0]))


def zero_block_pack():
    """A block with NumUids 0 between two full ones: the reference's loop stops there, and so does the device."""
    return HandPack(256, [10, 500, 900], [2, 0, 2], [0, 5, 5, 10], group([3, 0, 0, 0]) + group([4, 0, 0, 0]))


def edge_lists(rng):
    """(name, uids) lists whose packs cover the edges: 2^32 crossings, a first uid of 0, uids near 2^64, single uids,
    non-ascending input."""
    hi = np.uint64(1 << 32)
    return [
        ("zipf", gen.zipf_gaps(rng, 3000)),
        ("first_zero", np.concatenate([np.zeros(1, np.uint64), gen.zipf_gaps(rng, 700)])),
        ("crossings", np.sort(rng.integers(0, 8, 600).astype(np.uint64) * hi + rng.integers(0, 1 << 20, 600).astype(np.uint64))),
        ("near_max", np.uint64(M64) - np.sort(rng.integers(0, 1 << 36, 500).astype(np.uint64))[::-1]),
        ("one", np.array([123456789], np.uint64)),
        ("max_only", np.array([M64], np.uint64)),
        ("descending", np.sort(rng.integers(0, 1 << 62, 300).astype(np.uint64))[::-1].copy()),
    ]


def pack_images(packs):
    """Flat images (dgx_pack_image_view layout) of `packs` (oracle packs, None = nil), back to back in one 16-byte
    aligned buffer: (img, img_off, nblocks, delta_bytes), what dgx_encode_from_buffer_rows returns for them."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    n = len(packs)
    nb = np.array([0 if p is None else p.nblocks for p in packs], np.uint64)
    db = np.array([0 if p is None else int(p.delta_off[-1]) for p in packs], np.uint64)
    size = np.array([lib.dgx_pack_image_size(int(a), int(b)) if a else 0 for a, b in zip(nb, db)], np.uint64)
    off = np.zeros(n + 1, np.uint64)
    np.cumsum(size, out=off[1:])
    raw = np.zeros(int(off[-1]) + 32, np.uint8)
    img = raw[(-raw.ctypes.data) % 16:][: int(off[-1]) + 16]
    for i, p in enumerate(packs):
        if p is None or not nb[i]:
            continue
        k, o = int(nb[i]), int(off[i])
        meta = lib.dgx_pack_image_size(k, 0)
        img[o: o + 8 * k] = p.base.view(np.uint8)
        img[o + 8 * k: o + 16 * k + 8] = p.delta_off.view(np.uint8)
        img[o + 16 * k + 8: o + 20 * k + 8] = p.num_uids.view(np.uint8)
        img[o + meta: o + meta + int(db[i])] = p.deltas
    return img, off, nb, db
