"""Blocks whose running sum passes 2^32, through every kernel that reads a pack, bit-exact against the oracle.

The Encoder starts a new block whenever the upper 32 bits change, so its packs never need more than a 32-bit sum
inside a block; the reference still sums `last + uint64(delta)` (codec.go:191-196), and a hand-built pack can rely on
it.  One block of 9 uids is expanded in shared memory by the warp; one of 300 uids (more than 256) is walked by one
thread from global memory.  Runs on an H100 only (`pytest -m gpu`)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
from pack_geometry import ArrayPack  # noqa: E402
from test_gpu_parity import L, eq  # noqa: E402

pytestmark = pytest.mark.gpu

BASE = 5
STEP = 0xFFFFFFFF  # every delta at its largest: uid i is BASE + i * (2^32 - 1)


@pytest.fixture(scope="module")
def dgx():
    import dgraph_b200
    from dgraph_b200 import _lib

    lib = _lib.load()
    _lib.check(lib.dgx_init(-1))
    return dgraph_b200


def one_block(dgx, n):
    """(device pack, oracle pack, uids) of one block of n uids, every group tag 0xFF and every delta 0xFFFFFFFF."""
    base = np.array([BASE], np.uint64)
    num = np.array([n], np.uint32)
    deltas = np.full(17 * ((n + 2) // 4), 0xFF, np.uint8)
    delta_off = np.array([0, deltas.size], np.uint64)
    u = np.uint64(BASE) + np.arange(n, dtype=np.uint64) * np.uint64(STEP)
    assert int(u[-1]) > 2**32
    return dgx.pb.UidPack(n, base, num, delta_off, deltas), ArrayPack(n, base, num, delta_off, deltas), u


def probe_lists(u):
    """Ascending lists against the block: every other uid with near misses between them (short: the list searches
    the block), every uid with eight near misses after each (long: the block searches the list), and one uid."""
    near = u[1::2] + np.uint64(1)
    dense = (u[:, None] + np.arange(9, dtype=np.uint64)).ravel()
    return [np.unique(np.concatenate([u[::2], near])), dense, u[u.size // 2: u.size // 2 + 1]]


@pytest.mark.parametrize("n", [9, 300], ids=["smem", "serial"])
def test_running_sum_past_2_32(dgx, orc, n):
    p, op, u = one_block(dgx, n)
    mid = int(u[n // 2])
    eq(orc.decode(op, 0), u, "oracle")

    # codec.Decode, from the start and from seeks inside the block
    for seek in (0, mid, mid + 1):
        eq(dgx.codec.Decode(p, seek), orc.decode(op, seek), f"Decode seek {seek}")

    # every dgx_pack_seek kind, each from a fresh decoder
    for uid in (0, BASE, mid, mid + 1, int(u[-1]), int(u[-1]) + 1):
        for whence in (0, 1):
            for name, ref in (("Seek", "seek"), ("SeekToBlock", "seek_to_block")):
                dec, rd = dgx.codec.Decoder(p), orc.Decoder(op)
                eq(getattr(dec, name)(uid, whence), getattr(rd, ref)(uid, whence), f"{name}({uid}, {whence})")
                assert dec.BlockIdx() == rd.block_idx, (name, uid, whence)
        dec, rd = dgx.codec.Decoder(p), orc.Decoder(op)
        eq(dec.LinearSeek(uid), rd.linear_seek(uid), f"LinearSeek({uid})")
        assert dec.BlockIdx() == rd.block_idx, ("LinearSeek", uid)
    dec, rd = dgx.codec.Decoder(p), orc.Decoder(op)
    eq(dec.UnpackBlock(), rd.unpack_block(), "UnpackBlock")
    eq(dec.Next(), rd.next(), "Next")
    assert dec.BlockIdx() == rd.block_idx

    lists = probe_lists(u)
    # IntersectCompressedWith, afterUID before and inside the block
    for li, v in enumerate(lists):
        for after in (0, mid, mid + 1):
            o = dgx.pb.List(None)
            dgx.algo.IntersectCompressedWith(p, after, L(dgx, v), o)
            eq(o.Uids, orc.intersect_compressed_with(op, after, v), f"IntersectCompressedWith list {li} after {after}")

    # the rows form: the pack in several rows of one call, next to an empty row
    for li, v in enumerate(lists):
        for after in (0, mid):
            out, off = dgx.algo.IntersectCompressedWithRows([p, None, p], after, v)
            want = orc.intersect_compressed_with(op, after, v)
            for r, w in enumerate((want, np.zeros(0, np.uint64), want)):
                eq(out[int(off[r]): int(off[r + 1])], w, f"rows list {li} after {after} row {r}")

    # the matrix form: short rows (one lane each), long rows (the whole warp) and an empty row
    rows = lists + [u[:3] + np.uint64(1), u[-3:], np.zeros(0, np.uint64)]
    out, off = dgx.algo.IntersectCompressedWithMatrix(p, rows)
    for r, v in enumerate(rows):
        want = orc.intersect_compressed_with(op, 0, v) if v.size else np.zeros(0, np.uint64)
        eq(out[int(off[r]): int(off[r + 1])], want, f"matrix row {r}")
