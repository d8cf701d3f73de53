"""codec.DecodeToBuffer / codec.EncodeFromBuffer without a GPU: the oracle's uvarint rules and the numpy writer and
reader pinned against each other, the restore-after-backup round trip on the oracle, and every argument
dgx_decode_to_buffer_rows / dgx_encode_from_buffer_rows refuse before a device is needed."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import backup_codec_cases as cases  # noqa: E402
import backup_codec_oracle as bco  # noqa: E402
from gen_uvarint import put_uvarints_np, read_uvarints_np  # noqa: E402

ERR_ARG = -3
M64 = (1 << 64) - 1

KNOWN = [
    (0, "00"), (1, "01"), (127, "7f"), (128, "8001"), (300, "ac02"), (16384, "808001"),
    (1 << 63, "80" * 9 + "01"), (M64, "ff" * 9 + "01"),
]


@pytest.mark.parametrize("value,hexbytes", KNOWN)
def test_uvarint_known_answers(value, hexbytes):
    want = bytes.fromhex(hexbytes)
    assert bco.put_uvarint(value) == want
    assert put_uvarints_np([value]).tobytes() == want
    assert bco.uvarint(want) == (value, len(want))
    assert read_uvarints_np(want).tolist() == [value]


def test_uvarint_non_minimal_read():
    assert bco.uvarint(bytes.fromhex("8000")) == (0, 2)
    assert read_uvarints_np(bytes.fromhex("8000")).tolist() == [0]
    assert bco.uvarint(bytes.fromhex("ff" * 9 + "00")) == ((1 << 63) - 1, 10)


@pytest.mark.parametrize("stream", ["80" * 9 + "02", "80" * 10 + "00", "ff" * 11 + "01"])
def test_uvarint_overflow(stream):
    b = bytes.fromhex(stream)
    v, n = bco.uvarint(b)
    assert n < 0
    assert read_uvarints_np(b) is None
    assert bco.encode_from_buffer(b, 256)[0] == bco.OVERFLOW


@pytest.mark.parametrize("stream", ["80", "0580", "ff" * 9, "01" + "80" * 10])
def test_uvarint_truncated(stream):
    b = bytes.fromhex(stream)
    assert read_uvarints_np(b) is None
    rc, _ = bco.encode_from_buffer(b, 256)
    assert rc in (bco.OVERFLOW, bco.TRUNCATED)


def test_uvarint_truncated_tail_is_n_zero():
    assert bco.uvarint(bytes.fromhex("ff" * 9))[1] == 0
    assert bco.encode_from_buffer(bytes.fromhex("05ff"), 256)[0] == bco.TRUNCATED


@pytest.mark.parametrize("seed", range(6))
def test_oracle_against_numpy_writer_and_reader(seed):
    rng = np.random.default_rng(seed)
    bits = rng.integers(0, 65, 4000)
    vals = np.array([int(rng.integers(0, 1 << 63)) >> (63 - b) if b < 64 else int(rng.integers(0, 1 << 63)) | (1 << 63)
                     for b in bits], dtype=np.uint64)
    stream = put_uvarints_np(vals)
    assert stream.tobytes() == b"".join(bco.put_uvarint(int(v)) for v in vals)
    assert np.array_equal(read_uvarints_np(stream), vals)
    buf, got = stream.tobytes(), []
    while buf:
        v, n = bco.uvarint(buf)
        assert n > 0
        got.append(v)
        buf = buf[n:]
    assert got == vals.tolist()


def _roundtrip(hp, bs):
    """EncodeFromBuffer(DecodeToBuffer(P), bs) == Encode(Decode(P, 0), bs), array by array."""
    from oracle import pyoracle as orc

    stream = bco.decode_to_buffer(hp)
    uids = orc.decode(hp, 0)
    prev = np.concatenate([np.zeros(1, np.uint64), uids[:-1]])
    assert stream == put_uvarints_np(uids - prev).tobytes()  # wrapping u64 deltas
    rc, got = bco.encode_from_buffer(stream, bs)
    want = orc.encode(uids, bs)
    assert rc == 0
    assert got.is_nil == want.is_nil
    for f in ("base", "num_uids", "delta_off", "deltas"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f


@pytest.mark.parametrize("bs", [1, 5, 256, 5000])
def test_roundtrip_on_the_oracle(bs):
    rng = np.random.default_rng(bs)
    for name, uids in cases.edge_lists(rng):
        _roundtrip(cases.pack_of(uids, bs), bs)
    _roundtrip(cases.wrap_pack(), bs)


def test_first_uid_zero_and_nil():
    hp = cases.pack_of(np.array([0, 1, 2], np.uint64), 256)
    assert bco.decode_to_buffer(hp) == bytes([0, 1, 1])
    assert bco.decode_to_buffer(None) == b""
    rc, p = bco.encode_from_buffer(b"", 256)
    assert rc == 0 and p.is_nil


def test_zero_block_stops_the_oracle():
    assert bco.decode_to_buffer(cases.zero_block_pack()) == bytes([10, 3])


def test_wrap_pack_stream():
    """Uids 2^64-3, 2, 2^40, 2^40+7, 2^40+7+2^20: the second and third deltas wrap to 10-byte values' neighbours."""
    want = [M64 - 2, 5, (1 << 40) - 2, 7, 1 << 20]
    assert read_uvarints_np(bco.decode_to_buffer(cases.wrap_pack())).tolist() == want


# ---- the C ABI's host checks: nothing here needs a device --------------------------------------------------------
def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def test_zero_rows_need_no_device():
    from dgraph_b200 import _lib, codec

    lib = _lib.load()
    off = np.full(1, 7, np.uint64)
    assert lib.dgx_decode_to_buffer_rows(None, 0, None, _p(off), 0) == 0 and off.tolist() == [0]
    off[:] = 7
    assert lib.dgx_encode_from_buffer_rows(None, None, 0, 256, None, 0, _p(off), None, None) == 0 and off.tolist() == [0]
    out, o = codec.DecodeToBufferRows([])
    assert out.size == 0 and o.tolist() == [0]
    assert codec.EncodeFromBufferRows([], 256) == []


def test_all_empty_rows_need_no_device():
    from dgraph_b200 import _lib

    lib = _lib.load()
    buf_off = np.zeros(4, np.uint64)
    img_off, nb, db = np.full(4, 9, np.uint64), np.full(3, 9, np.uint64), np.full(3, 9, np.uint64)
    assert lib.dgx_encode_from_buffer_rows(None, _p(buf_off), 3, 256, None, 0, _p(img_off), _p(nb), _p(db)) == 0
    assert img_off.tolist() == [0] * 4 and nb.tolist() == [0] * 3 and db.tolist() == [0] * 3


def _enc(buf, buf_off, img=None, null=()):
    from dgraph_b200 import _lib

    n = len(buf_off) - 1
    buf, buf_off = np.frombuffer(bytes(buf) + b"\0", np.uint8), np.asarray(buf_off, np.uint64)
    arrs = {"buf": buf, "buf_off": buf_off, "img_off": np.zeros(n + 1, np.uint64), "nblocks": np.zeros(n, np.uint64),
            "delta_bytes": np.zeros(n, np.uint64)}
    a = {k: (None if k in null else _p(v)) for k, v in arrs.items()}
    return _lib.load().dgx_encode_from_buffer_rows(a["buf"], a["buf_off"], n, 256, img, 0 if img is None else 64,
                                                   a["img_off"], a["nblocks"], a["delta_bytes"])


@pytest.mark.parametrize("buf_off", [[1, 2], [0, 2, 1], [0, 1 << 32]])
def test_encode_bad_offsets(buf_off):
    assert _enc(b"\x01\x01", buf_off) == ERR_ARG


@pytest.mark.parametrize("null", ["buf", "buf_off", "img_off", "nblocks", "delta_bytes"])
def test_encode_null_arrays(null):
    assert _enc(b"\x01\x01", [0, 2], null=(null,)) == ERR_ARG


def test_encode_unaligned_image():
    raw = np.zeros(96, np.uint8)
    addr = raw.ctypes.data + ((-raw.ctypes.data) % 16) + 8
    assert _enc(b"\x01\x01", [0, 2], img=C.c_void_p(addr)) == ERR_ARG


def test_decode_null_arrays():
    from dgraph_b200 import _lib, algo

    lib = _lib.load()
    refs, keep = algo._refs_of([cases.pack_of([1, 2, 3], 256).uid_pack()])
    assert lib.dgx_decode_to_buffer_rows(refs, 1, None, None, 0) == ERR_ARG
    off = np.zeros(2, np.uint64)
    assert lib.dgx_decode_to_buffer_rows(None, 1, None, _p(off), 0) == ERR_ARG


def test_decode_malformed_pack():
    from dgraph_b200 import _lib, algo

    bad = cases.HandPack(256, [5], [9], [0, 4], [0, 0, 0, 0]).uid_pack()  # 9 uids need two 5-byte groups
    refs, keep = algo._refs_of([bad])
    off = np.zeros(2, np.uint64)
    assert _lib.load().dgx_decode_to_buffer_rows(refs, 1, None, _p(off), 0) == ERR_ARG


def test_decode_exact_len_total():
    from dgraph_b200 import _lib, algo, pb

    # block tables claiming 2^31 uids each (never read: the total is refused first)
    big = pb.UidPack(256, np.array([1], np.uint64), np.array([1 << 31], np.uint32), np.array([0, 5], np.uint64),
                     np.zeros(5, np.uint8))
    refs, keep = algo._refs_of([big, big])
    off = np.zeros(3, np.uint64)
    assert _lib.load().dgx_decode_to_buffer_rows(refs, 2, None, _p(off), 0) == ERR_ARG
