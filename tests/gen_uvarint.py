"""Unsigned varint (LEB128) streams in numpy: the writer and reader of BackupPostingList.uid_bytes (encoding/binary
PutUvarint / Uvarint), independent of oracle/ (tests/test_backup_codec_host.py checks both against the oracle byte for
byte), as tests/gen.py's encode_pack_np is for group-varint packs."""
from __future__ import annotations

import numpy as np


def put_uvarints_np(values) -> np.ndarray:
    """PutUvarint of every value, back to back: little-endian groups of 7 bits, high bit set on every byte but the
    last; max(1, ceil(bits / 7)) bytes per value."""
    v = np.ascontiguousarray(np.asarray(values, dtype=np.uint64))
    if v.size == 0:
        return np.zeros(0, np.uint8)
    nbits = np.zeros(v.size, np.int64)
    for k in range(64):
        nbits[(v >> np.uint64(k)) != 0] = k + 1
    lens = np.maximum(1, (nbits + 6) // 7)
    off = np.concatenate([[0], np.cumsum(lens)])
    out = np.zeros(int(off[-1]), np.uint8)
    for t in range(10):
        m = lens > t
        byte = ((v[m] >> np.uint64(7 * t)) & np.uint64(0x7F)).astype(np.uint8)
        more = (lens[m] > t + 1).astype(np.uint8) << 7
        out[off[:-1][m] + t] = byte | more
    return out


def read_uvarints_np(buf):
    """Uvarint over the whole stream: the values, or None where binary.Uvarint would report an error (a value of more
    than 10 bytes, a 10th byte > 1, or a stream that ends inside a value).  Non-minimal encodings are accepted."""
    b = np.frombuffer(bytes(buf), np.uint8) if not isinstance(buf, np.ndarray) else buf.astype(np.uint8)
    if b.size == 0:
        return np.zeros(0, np.uint64)
    if b[-1] >= 0x80:
        return None
    ends = np.nonzero(b < 0x80)[0]
    starts = np.concatenate([[0], ends[:-1] + 1])
    lens = ends - starts + 1
    if (lens > 10).any() or ((lens == 10) & (b[ends] > 1)).any():
        return None
    vals = np.zeros(ends.size, np.uint64)
    for t in range(10):
        m = lens > t
        vals[m] |= (b[starts[m] + t].astype(np.uint64) & np.uint64(0x7F)) << np.uint64(7 * t)
    return vals
