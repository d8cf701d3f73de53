"""Host model of the backup codec on the device (backup_codec_kernel.cuh, and tb_plan, tb_launch, bf_plan, bf_launch and
the four entry points in dgx_api.cu), and fixtures aimed at its tile, value, row, segment and block boundaries.

Bytes -> packs (dgx_encode_from_buffer_rows / dgx_dev_encode_from_buffer_rows), nine launches:
  - bf_values_kernel: one CTA per EN_TILE bytes, EN_VT bytes a thread; a byte < 0x80 ends a value, whose start is found
    by scanning back over at most 10 continuation bytes (across thread and tile edges); the value's row is the last
    row whose offset is <= its start (empty rows share offsets); the thread whose value starts a row writes that row's
    base prefix; two look-backs per tile: the value count, and the wrapping u64 value sum (lookback_wide);
  - bf_segments_kernel: uid = call-wide prefix - row base; a segment starts at the first value, a row change or an
    upper-word change, the thread's previous value loaded across tile edges; the grid is sized for the bytes, so
    tiles past the value count return;
  - bf_segcount_kernel, scan_u64_kernel, bf_sizes_kernel, scan_u64_kernel: blocks of BlockSize values per segment,
    their group bytes and offsets;
  - bf_rows_kernel, scan_u64_kernel: per row its blocks, delta bytes and image bytes, and the truncated-row check;
  - bf_write_kernel: the images, or on a malformed stream the offset and size arrays zeroed.
Packs -> bytes (dgx_decode_to_buffer_rows / dgx_dev_decode_to_buffer_rows), four launches: tb_blocks_kernel (a thread
per block: its last uid and internal varint bytes; NumUids 0 marks the row's stop with atomicMin), tb_sizes_kernel
(the boundary varint, nothing from the stop on), scan_u64_kernel, tb_write_kernel.  The host forms run the write pass
again once they know the exact size.

The model restates all of it in integer arithmetic; the packs' bytes come from gen.encode_pack_np and the images from
backup_codec_cases.pack_images, and the model's plan must agree with both.  What the kernels decide is named as
*events*; fixtures name the events they must reach, and the model refuses a name that is not registered in EVENTS.
The constants and the statements the model restates are read from the CUDA sources as text, so a rewrite fails here
loudly instead of leaving the fixtures aimed at stale edges.

Not reachable by any fixture: lookback_wide's multi-round path (none of the 32 tiles before a tile has published its
inclusive prefix) depends on scheduling; fixtures of 33 and more tiles make it possible but cannot force it.  Value
counts of 2^32 and more (seg_start and vrow are u32) need about 52 bytes of HBM per input byte; only the host's
check_offsets limit on the byte count covers them.

tests/test_backup_codec_geometry.py checks the fixtures on the CPU; tests/test_gpu_backup_codec_edges.py runs them
through the kernels.
"""
from __future__ import annotations

import os
import re
import sys
from collections import namedtuple
from types import SimpleNamespace

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import encode_geometry as eg  # noqa: E402
import gen  # noqa: E402
import gen_uvarint as guv  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")
U64 = (1 << 64) - 1
M32 = 0xFFFFFFFF
OK, ERR_ARG, ERR_CAP = 0, -3, -4


def _src(fn):
    with open(os.path.join(CSRC, fn)) as f:
        return f.read()


def _one(pat, text, what):
    m = re.search(pat, text)
    if not m:
        raise ValueError(f"{what} changed: restate it in the backup codec model (tests/backup_codec_geometry.py)")
    return m


def read_constants() -> dict:
    bc, enc, com, api = (_src(f) for f in ("backup_codec_kernel.cuh", "encode_kernel.cuh", "common.cuh", "dgx_api.cu"))
    m = _one(r"constexpr int EN_NT = (\d+), EN_VT = (\d+), EN_TILE = EN_NT \* EN_VT;", enc, "EN_NT / EN_VT / EN_TILE")
    K = {"EN_NT": int(m.group(1)), "EN_VT": int(m.group(2))}
    widths = {int(_one(p, t, "the tb_* grid width").group(1)) for p, t in (
        (r"__launch_bounds__\((\d+)\) tb_blocks_kernel", bc), (r"__launch_bounds__\((\d+)\) tb_sizes_kernel", bc),
        (r"__launch_bounds__\((\d+)\) tb_write_kernel", bc), (r"tb_blocks_kernel<<<g_blk, (\d+), 0", api),
        (r"tb_sizes_kernel<<<g_blk, (\d+), 0", api), (r"\(P\.nblk \+ \d+\) / (\d+)\);", api),
        (r"tb_write_kernel<<<\(unsigned\)\(\(nthreads \+ \d+\) / (\d+)\)", api))}
    if len(widths) != 1:
        raise ValueError(f"the tb_* grid width changed: {sorted(widths)}: restate it in the backup codec model")
    K["TB_NT"] = widths.pop()
    m = _one(r"while \(c < (\d+) && k > c && P\.buf\[k - 1 - c\] >= 0x80\) \+\+c;", bc, "the backward scan")
    K["SCAN"] = int(m.group(1))
    if K["SCAN"] != 10:
        raise ValueError(f"the backward scan reads {K['SCAN']} continuation bytes, binary.Uvarint 9 and an 11th: "
                         "restate it in the backup codec model")
    m = _one(r"if \(c >= (\d+) \|\| \(c == (\d+) && P\.buf\[k\] > (\d+)\)\) bad = true;", bc, "the overflow rule")
    K["OVF"] = tuple(int(g) for g in m.groups())
    if K["OVF"] != (10, 9, 1):
        raise ValueError(f"the overflow rule is {K['OVF']}, binary.Uvarint's (10, 9, 1): restate it in the backup codec "
                         "model")
    _one(r"if \(P\.row_off\[row\] == start\[i\]\) P\.rowbase\[row\] = run - x\[i\];", bc, "the rowbase condition")
    _one(r"const u64 row = last_le\(P\.row_off, P\.nrows \+ 1, start\[i\]\);", bc, "the value's row")
    _one(r"if \(j == 0 \|\| row != prow \|\| \(u >> 32\) != \(prev >> 32\)\) \{ flags \|= 1u << i; \+\+cnt; \}", bc,
         "bf_segments_kernel's segment-start condition")
    _one(r"if \(e0 > 0 && e0 <= m\) \{ prow = P\.vrow\[e0 - 1\]; prev = uid\(e0 - 1\); \}", bc,
         "bf_segments_kernel's previous-value load")
    _one(r"if \(\(u64\)tile \* EN_TILE >= m && tile != 0\) return;", bc, "bf_segments_kernel's early return")
    _one(r"P\.seg_cnt\[s\] = \(\(u64\)P\.seg_start\[s \+ 1\] - P\.seg_start\[s\] \+ P\.bsz - 1\) / P\.bsz;", bc,
         "bf_segcount_kernel's ceiling")
    _one(r"if \(o1 > o0 && P\.buf\[o1 - 1\] >= 0x80\) atomicExch\(P\.bad, 1\);", bc, "bf_rows_kernel's truncated-row check")
    _one(r"if \(b >= P\.stop\[P\.jobs\[j\]\.row\]\) \{ P\.bytes\[g\] = 0; return; \}", bc, "tb_sizes_kernel's stop skip")
    _one(r"const u64 prev = b \? P\.last\[g - 1\] : 0;", bc, "tb_sizes_kernel's previous block `b ? P.last[g - 1] : 0`")
    _one(r"if \(num == 0\) atomicMin\(P\.stop \+ P\.jobs\[j\]\.row, b\);", bc, "tb_blocks_kernel's stop atomicMin")
    _one(r"if \(pm && lane > __ffs\(pm\) - 1\) v = 0;", bc, "lookback_wide's cut at the nearest prefix")
    _one(r"for \(u64 z = nb \* 20 \+ 8; z < meta; \+\+z\) im\[z\] = 0;\s*"
         r"for \(u64 z = meta \+ db; z < meta \+ \(\(db \+ 15\) & ~15ull\); \+\+z\) im\[z\] = 0;", bc,
         "bf_write_kernel's zero fill of the image padding")
    _one(r"return \(nb \* 8 \+ \(nb \+ 1\) \* 8 \+ nb \* 4 \+ 15\) & ~15ull;", com, "pack_image_meta_bytes")
    _one(r"P\.bsz = block_size \? block_size : 1;", api, "bf_plan's BlockSize `P.bsz = block_size ? block_size : 1`")
    K["TB_LAUNCHES"] = int(_one(r"launches = (\d+);\s*\}\s*const uint64_t nthreads", api, "tb_launch's launches").group(1))
    K["BF_LAUNCHES"] = int(_one(r"launches = (\d+);\s*\}\s*bf_write_kernel", api, "bf_launch's launches").group(1))
    _one(r"if \(!out \|\| total == 0\) return ps\.synced\(DGX_OK\);[^}]*?tb_launch\(l, R, true\)", api,
         "dgx_decode_to_buffer_rows's write pass")
    _one(r"if \(!img \|\| total == 0\) return DGX_OK;[^}]*?bf_launch\(l, R, true\)", api,
         "dgx_encode_from_buffer_rows's write pass")
    return K


K = read_constants()
EN_VT = K["EN_VT"]
EN_TILE = K["EN_NT"] * EN_VT
TB_LAUNCHES, BF_LAUNCHES = K["TB_LAUNCHES"], K["BF_LAUNCHES"]
SCAN = K["SCAN"]
OVF_C, OVF_C9, OVF_LAST = K["OVF"]


def meta_bytes(nb):
    """pack_image_meta_bytes."""
    return (nb * 8 + (nb + 1) * 8 + nb * 4 + 15) & ~15


def uvarint_len(x):
    return max(1, -(-int(x).bit_length() // 7))


# ---- events -----------------------------------------------------------------------------------------------------------

EVENTS = {
    "val: a 10-byte value ending in 0x01", "val: a 10-byte value ending in 0x00, non-minimal", "val: non-minimal 80 00",
    "val: n = 2048k - 1 bytes", "val: n = 2048k bytes", "val: n = 2048k + 1 bytes",
    "val: 33 or more tiles of look-back", "val: a tile's value sum wraps u64",
    "val: the call-wide prefix wraps before a later row's first value",
    "bad: overflow, a 10th byte > 1 across a tile edge", "bad: overflow, 11 or more bytes across a tile edge",
    "bad: a row ends inside a value, an empty row follows", "bad: the last row ends inside a value",
    "row: starts on a tile's first byte", "row: starts inside a thread's range", "row: leading empty rows",
    "row: trailing empty rows", "row: an interior run of empty rows",
    "row: its first value's terminator lies in the tile after its start",
    "seg: upper-word change at a value tile's first value", "seg: upper-word change at a thread's first value",
    "seg: row change at a value tile's first value", "seg: row change with the same upper word",
    "seg: m = 2048k - 1", "seg: m = 2048k", "seg: m = 2048k + 1", "seg: tiles past m return early",
    "seg: more than 2048 segments",
    "blk: segment of bsz * k values", "blk: segment of bsz * k + 1 values", "blk: segment of bsz * k - 1 values",
    "blk: num 129", "blk: num 130", "blk: num 257", "blk: num 258", "blk: more than 2048 blocks",
    "bsz 0", "bsz 1", "bsz 2^31 - 1", "bsz 2^32 - 1",
    "img: 2048 rows, one tile", "img: 2049 rows, two tiles", "img: delta padding of 0 bytes",
    "img: delta padding of 15 bytes",
    "restore: every row empty, no launch", "restore: OK", "restore: CAP", "restore: ARG with an image",
    "restore: ARG without an image", "restore: sizes only",
    "bk: internal delta wraps", "bk: boundary delta wraps", "bk: first uid 0", "bk: NumUids 0 as block 0",
    "bk: NumUids 0 as the last block", "bk: NumUids 0 twice in one row", "bk: blocks with data after the stop",
    "bk: nblk = 256k - 1", "bk: nblk = 256k + 1", "bk: nblk = 2048k - 1", "bk: nblk = 2048k + 1",
    "bk: more than 32 byte-scan tiles", "bk: a nil pack between packs", "bk: an empty pack between packs",
    "bk: the same pack in several rows", "bk: a row's first block after another pack's last",
    "backup: total 0 bytes, the write skipped", "backup: OK", "backup: CAP", "backup: sizes only",
    "cap: out_cap exact", "cap: out_cap one short", "cap: img_cap exact", "cap: img_cap one short",
} | {f"val: length {L} ending at thread offset {o}" for L in range(1, 11) for o in range(EN_VT)} \
  | {f"val: terminator at a tile's first byte, {c} bytes back in the previous tile" for c in range(1, 10)} \
  | {f"img: metadata padding of {p} bytes" for p in (0, 4, 8, 12)} \
  | {f"bk: boundary varint of {L} bytes, its {w} value" for L in range(1, 11) for w in ("smallest", "largest")} \
  | {f"bk: internal delta of {L} bytes" for L in range(1, 6)}


def _add(ev, name):
    if name not in EVENTS:
        raise KeyError(f"event {name!r} is not registered in backup_codec_geometry.EVENTS")
    ev.add(name)


def row_verdict(b) -> str | None:
    """What orc_encode_from_buffer answers for one row alone: None (valid), "overflow" (the reference panics: a value
    of more than 10 bytes or a 10th byte > 1) or "truncated" (it never returns: the row ends inside a value)."""
    b = np.frombuffer(bytes(b), np.uint8)
    if b.size == 0:
        return None
    ends = np.nonzero(b < 0x80)[0]
    lens = ends - np.concatenate([[-1], ends[:-1]])
    if ((lens > 10) | ((lens == 10) & (b[ends] > 1))).any():
        return "overflow"
    tail = b.size - (int(ends[-1]) + 1 if ends.size else 0)
    return None if tail == 0 else "overflow" if tail > 10 else "truncated"


# ---- bytes -> packs ---------------------------------------------------------------------------------------------------

Restore = namedtuple("Restore", "rc sync launches img_off nblocks delta_bytes written")


class RestorePlan:
    """One dgx_encode_from_buffer_rows / dgx_dev_encode_from_buffer_rows call over `rows` (bytes each) at BlockSize
    `block_size`: the nine kernels' plan, and what each entry point answers at a given img_cap."""

    def __init__(self, rows, block_size, ev=None):
        ev = set() if ev is None else ev
        self.events = ev
        self.rows = [bytes(r) for r in rows]
        self.nrows = nr = len(self.rows)
        self.block_size = block_size
        self.bsz = B = block_size if block_size else 1
        lens = [len(r) for r in self.rows]
        self.row_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64) if nr else np.zeros(1, np.int64)
        self.buf = b = np.frombuffer(b"".join(self.rows), np.uint8)
        self.n = n = int(b.size)
        self.verdicts = [row_verdict(r) for r in self.rows]
        self._row_events(ev, lens)
        if n == 0:
            _add(ev, "restore: every row empty, no launch")
            self.bad, self.m = False, 0
            self._empty_result()
            return
        self.tiles = -(-n // EN_TILE)
        r = n % EN_TILE
        if n >= EN_TILE - 1 and r in (EN_TILE - 1, 0, 1):
            _add(ev, {EN_TILE - 1: "val: n = 2048k - 1 bytes", 0: "val: n = 2048k bytes", 1: "val: n = 2048k + 1 bytes"}[r])
        if self.tiles - 1 >= 33:
            _add(ev, "val: 33 or more tiles of look-back")

        # bf_values_kernel: terminators, their scan back, their values
        cont = b >= 0x80
        idx = np.arange(n)
        run = idx - np.maximum.accumulate(np.where(~cont, idx, -1))      # continuation bytes ending at every byte
        k = np.nonzero(~cont)[0]
        c = np.where(k > 0, np.minimum(run[np.maximum(k - 1, 0)], SCAN), 0)
        self.k, self.c = k, c
        self.start = s = k - c
        self.length = c + 1
        self.tile, self.thread, self.offset = k // EN_TILE, (k % EN_TILE) // EN_VT, k % EN_VT
        self.overflow = (c >= OVF_C) | ((c == OVF_C9) & (b[k] > OVF_LAST))
        v = np.zeros(k.size, np.uint64)
        for t in range(10):
            m_t = t <= c
            v[m_t] |= (b[s[m_t] + t].astype(np.uint64) & np.uint64(0x7F)) << np.uint64(7 * t)
        self.x = v
        self.vrow = np.searchsorted(self.row_off, s, side="right") - 1    # last_le over row_off
        self.sets_rowbase = self.row_off[self.vrow] == s
        self.truncated_rows = [i for i in range(nr) if lens[i] and self.rows[i][-1] >= 0x80]
        self.bad = bool(self.overflow.any()) or bool(self.truncated_rows)
        self._value_events(ev, b, k, c, s, v)
        assert self.bad == any(self.verdicts), "the kernels' verdict differs from the reference's"

        # the two look-backs of every tile
        m = self.m = int(k.size)
        self.tile_count = np.bincount(self.tile, minlength=self.tiles).astype(np.int64)
        self.count_prefix = np.cumsum(self.tile_count)
        self.tile_sum = [0] * self.tiles
        for t, val in zip(self.tile.tolist(), v.tolist()):
            self.tile_sum[t] += val
        if any(s_ > U64 for s_ in self.tile_sum):
            _add(ev, "val: a tile's value sum wraps u64")
        self.tile_sum = [s_ & U64 for s_ in self.tile_sum]
        acc, self.sum_prefix = 0, []
        for s_ in self.tile_sum:
            acc = (acc + s_) & U64
            self.sum_prefix.append(acc)
        self.tiles_behind = np.arange(self.tiles)
        if self.bad:
            self._empty_result()
            return

        # uids: the call-wide prefix minus the row's base
        self.pre = np.cumsum(v, dtype=np.uint64)
        rowbase = {}
        for i in np.nonzero(self.sets_rowbase)[0].tolist():
            rowbase[int(self.vrow[i])] = int(self.pre[i]) - int(v[i]) & U64
        true_pre = np.concatenate([[0], np.cumsum([int(q) for q in v.tolist()], dtype=object)])
        for i in np.nonzero(self.sets_rowbase)[0].tolist():
            if self.vrow[i] > 0 and true_pre[i] > U64:
                _add(ev, "val: the call-wide prefix wraps before a later row's first value")
        self.rowbase = rowbase
        rb = np.array([rowbase[int(r_)] for r_ in self.vrow.tolist()], np.uint64)
        self.uids = self.pre - rb

        # bf_segments_kernel
        hi = self.uids >> np.uint64(32)
        j = np.arange(m)
        flag = np.ones(m, bool)
        flag[1:] = (self.vrow[1:] != self.vrow[:-1]) | (hi[1:] != hi[:-1])
        self.seg_start = np.nonzero(flag)[0]
        self.seg_tile, self.seg_thread = self.seg_start // EN_TILE, (self.seg_start % EN_TILE) // EN_VT
        self.nseg = int(self.seg_start.size)
        self.seg_tiles_live = max(1, -(-m // EN_TILE))
        self._segment_events(ev, j, hi, flag)

        # bf_segcount_kernel, the segment scan, bf_sizes_kernel, the byte scan
        seg_len = np.diff(np.append(self.seg_start, m))
        self.seg_cnt = -(-seg_len // B)
        self.seg_blk = np.concatenate([[0], np.cumsum(self.seg_cnt)]).astype(np.int64)
        self.nblk = nb = int(self.seg_blk[-1])
        bseg = np.repeat(np.arange(self.nseg), self.seg_cnt)
        self.blk_start = (self.seg_start[bseg] + (np.arange(nb) - self.seg_blk[bseg]) * B).astype(np.int64)
        self.blk_num = np.minimum(np.append(self.seg_start, m)[bseg + 1] - self.blk_start, B).astype(np.int64)
        self.brow = self.vrow[self.blk_start]
        self.blk_bytes = np.array([self._group_bytes(int(a), int(q)) for a, q in zip(self.blk_start, self.blk_num)],
                                  np.int64)
        self._block_events(ev, seg_len, B, block_size)

        # bf_rows_kernel and the image scan
        self.nblocks = np.bincount(self.brow, minlength=nr).astype(np.int64)
        self.delta_bytes = np.bincount(self.brow, weights=self.blk_bytes, minlength=nr).astype(np.int64)
        self.img_bytes = np.array([meta_bytes(int(q)) + (int(d) + 15 & ~15) if q else 0
                                   for q, d in zip(self.nblocks, self.delta_bytes)], np.int64)
        self.img_off = np.concatenate([[0], np.cumsum(self.img_bytes)]).astype(np.uint64)
        for q, d in zip(self.nblocks.tolist(), self.delta_bytes.tolist()):
            if q:
                _add(ev, f"img: metadata padding of {meta_bytes(q) - (20 * q + 8)} bytes")
                if d % 16 == 0:
                    _add(ev, "img: delta padding of 0 bytes")
                if d % 16 == 1:
                    _add(ev, "img: delta padding of 15 bytes")
        if nr == EN_TILE:
            _add(ev, "img: 2048 rows, one tile")
        if nr == EN_TILE + 1:
            _add(ev, "img: 2049 rows, two tiles")
        self.total = int(self.img_off[-1])

    def _empty_result(self):
        nr = self.nrows
        self.uids = np.zeros(0, np.uint64)
        self.vrow = np.zeros(0, np.int64)
        self.img_off = np.zeros(nr + 1, np.uint64)
        self.nblocks = np.zeros(nr, np.int64)
        self.delta_bytes = np.zeros(nr, np.int64)
        self.total = 0

    def _group_bytes(self, a, q):
        """enc_block_bytes: a tag and gv_len of four u32 deltas per group, the last group zero-padded."""
        ng = (q + 2) // 4 if q > 1 else 1
        d = np.zeros(4 * ng, np.uint64)
        d[: q - 1] = (self.uids[a + 1: a + q] - self.uids[a: a + q - 1]) & np.uint64(M32)
        return ng + int(eg.gv_len(d).sum())

    def _row_events(self, ev, lens):
        empty = [L == 0 for L in lens]
        nr = len(lens)
        if nr >= 2 and empty[0] and empty[1] and not all(empty):
            _add(ev, "row: leading empty rows")
        if nr >= 2 and empty[-1] and empty[-2] and not all(empty):
            _add(ev, "row: trailing empty rows")
        first = next((i for i, e in enumerate(empty) if not e), nr)
        last = max((i for i, e in enumerate(empty) if not e), default=-1)
        for i in range(first + 1, last - 1):
            if empty[i] and empty[i + 1]:
                _add(ev, "row: an interior run of empty rows")
        for i in range(1, nr):
            o = int(self.row_off[i])
            if lens[i]:
                if o % EN_TILE == 0:
                    _add(ev, "row: starts on a tile's first byte")
                if o % EN_VT:
                    _add(ev, "row: starts inside a thread's range")
        for i, vd in enumerate(self.verdicts):
            if vd == "truncated" and i + 1 < nr and lens[i + 1] == 0:
                _add(ev, "bad: a row ends inside a value, an empty row follows")
        nonempty = [i for i in range(nr) if lens[i]]
        if nonempty and self.rows[nonempty[-1]][-1] >= 0x80:
            _add(ev, "bad: the last row ends inside a value")

    def _value_events(self, ev, b, k, c, s, v):
        ok = ~self.overflow
        for L, o in set(zip((c[ok] + 1).tolist(), self.offset[ok].tolist())):
            _add(ev, f"val: length {L} ending at thread offset {o}")
        edge = (k % EN_TILE == 0) & (c >= 1) & ok
        for cc in set(c[edge].tolist()):
            _add(ev, f"val: terminator at a tile's first byte, {cc} bytes back in the previous tile")
        if ((c == 9) & (b[k] == 1)).any():
            _add(ev, "val: a 10-byte value ending in 0x01")
        if ((c == 9) & (b[k] == 0)).any():
            _add(ev, "val: a 10-byte value ending in 0x00, non-minimal")
        if ((c == 1) & (b[k] == 0) & (b[s] == 0x80)).any():
            _add(ev, "val: non-minimal 80 00")
        cross = s // EN_TILE != k // EN_TILE
        if (self.overflow & cross & (c == OVF_C9) & (b[k] > OVF_LAST)).any():
            _add(ev, "bad: overflow, a 10th byte > 1 across a tile edge")
        if (self.overflow & cross & (c >= OVF_C)).any():
            _add(ev, "bad: overflow, 11 or more bytes across a tile edge")
        first = self.sets_rowbase & (self.tile != s // EN_TILE)
        if first.any():
            _add(ev, "row: its first value's terminator lies in the tile after its start")

    def _segment_events(self, ev, j, hi, flag):
        m = j.size
        same_row = np.zeros(m, bool)
        same_row[1:] = self.vrow[1:] == self.vrow[:-1]
        hi_chg = np.zeros(m, bool)
        hi_chg[1:] = hi[1:] != hi[:-1]
        row_chg = np.zeros(m, bool)
        row_chg[1:] = ~same_row[1:]
        if (same_row & hi_chg & (j % EN_TILE == 0)).any():
            _add(ev, "seg: upper-word change at a value tile's first value")
        if (same_row & hi_chg & (j % EN_VT == 0) & (j % EN_TILE != 0)).any():
            _add(ev, "seg: upper-word change at a thread's first value")
        if (row_chg & (j % EN_TILE == 0)).any():
            _add(ev, "seg: row change at a value tile's first value")
        if (row_chg & ~hi_chg).any():
            _add(ev, "seg: row change with the same upper word")
        if m >= EN_TILE - 1 and m % EN_TILE in (EN_TILE - 1, 0, 1):
            _add(ev, {EN_TILE - 1: "seg: m = 2048k - 1", 0: "seg: m = 2048k", 1: "seg: m = 2048k + 1"}[m % EN_TILE])
        if self.tiles > self.seg_tiles_live:
            _add(ev, "seg: tiles past m return early")
        if self.nseg > EN_TILE:
            _add(ev, "seg: more than 2048 segments")

    def _block_events(self, ev, seg_len, B, bsz):
        for v_, name in ((0, "bsz 0"), (1, "bsz 1"), ((1 << 31) - 1, "bsz 2^31 - 1"), ((1 << 32) - 1, "bsz 2^32 - 1")):
            if bsz == v_:
                _add(ev, name)
        if B > 2:
            big = seg_len >= B
            if (big & (seg_len % B == 0)).any():
                _add(ev, "blk: segment of bsz * k values")
            if (big & (seg_len % B == 1)).any():
                _add(ev, "blk: segment of bsz * k + 1 values")
            if ((seg_len >= B - 1) & (seg_len % B == B - 1)).any():
                _add(ev, "blk: segment of bsz * k - 1 values")
        for q in (129, 130, 257, 258):
            if (self.blk_num == q).any():
                _add(ev, f"blk: num {q}")
        if self.nblk > EN_TILE:
            _add(ev, "blk: more than 2048 blocks")

    # ---- results ----

    def row_uids(self, r):
        return self.uids[self.vrow == r]

    def decoded_stream(self, r):
        """DecodeToBuffer of row r's restored pack.  A block keeps its deltas as u32 added to its base, so a uid below
        the one before it inside a block comes back as that uid plus a multiple of 2^32: the stream comes back
        unchanged (up to non-minimal varints) exactly when the row's uids never decrease inside a block."""
        out = []
        for a, q in zip(self.blk_start[self.brow == r].tolist(), self.blk_num[self.brow == r].tolist()):
            d = (self.uids[a + 1: a + q] - self.uids[a: a + q - 1]) & np.uint64(M32)
            out.append(self.uids[a] + np.concatenate([np.zeros(1, np.uint64), np.cumsum(d, dtype=np.uint64)]))
        u = np.concatenate(out) if out else np.zeros(0, np.uint64)
        return guv.put_uvarints_np(np.diff(np.concatenate([np.zeros(1, np.uint64), u]))).tobytes()

    def packs(self):
        """Every row's pack (None: nil) from gen.encode_pack_np, checked against the plan's blocks and group bytes."""
        out = []
        for r in range(self.nrows):
            pk = gen.encode_pack_np(self.row_uids(r), self.block_size) if not self.bad and self.n else None
            if pk is None:
                assert self.nblocks[r] == 0
                out.append(None)
                continue
            _, base, num, doff, deltas = pk
            sel = self.brow == r
            assert np.array_equal(base, self.uids[self.blk_start[sel]]), f"row {r}: bases"
            assert np.array_equal(num.astype(np.int64), self.blk_num[sel]), f"row {r}: NumUids"
            assert np.array_equal(np.diff(doff.astype(np.int64)), self.blk_bytes[sel]), f"row {r}: group bytes"
            out.append(SimpleNamespace(block_size=self.block_size, nblocks=base.size, base=base, num_uids=num,
                                       delta_off=doff, deltas=deltas))
        return out

    def image(self):
        """(img, img_off, nblocks, delta_bytes) of backup_codec_cases.pack_images over the rows' packs."""
        import backup_codec_cases as cases

        img, off, nb, db = cases.pack_images(self.packs())
        assert np.array_equal(off, self.img_off) and np.array_equal(nb, self.nblocks.astype(np.uint64))
        assert np.array_equal(db, self.delta_bytes.astype(np.uint64))
        return img, off, nb, db

    def host(self, img_cap, ev=None):
        """dgx_encode_from_buffer_rows with an image of img_cap bytes (None: no image)."""
        ev = self.events if ev is None else ev
        if self.n == 0:
            return Restore(OK, None, 0, self.img_off, self.nblocks, self.delta_bytes, False)
        if self.bad:
            _add(ev, "restore: ARG without an image" if img_cap is None else "restore: ARG with an image")
            return Restore(ERR_ARG, None, BF_LAUNCHES, self.img_off, self.nblocks, self.delta_bytes, False)
        if img_cap is None:
            _add(ev, "restore: sizes only")
            return Restore(OK, None, BF_LAUNCHES, self.img_off, self.nblocks, self.delta_bytes, False)
        if self.total > img_cap:
            _add(ev, "restore: CAP")
            return Restore(ERR_CAP, None, BF_LAUNCHES, self.img_off, self.nblocks, self.delta_bytes, False)
        _add(ev, "restore: OK")
        return Restore(OK, None, BF_LAUNCHES + 1, self.img_off, self.nblocks, self.delta_bytes, True)

    def dev(self, img_cap, ev=None):
        """dgx_dev_encode_from_buffer_rows: the call answers DGX_OK, dgx_lane_sync what the kernels found."""
        ev = self.events if ev is None else ev
        if self.n == 0:
            return Restore(OK, OK, 0, self.img_off, self.nblocks, self.delta_bytes, False)
        h = self.host(img_cap, ev)
        return Restore(OK, h.rc, BF_LAUNCHES, h.img_off, h.nblocks, h.delta_bytes, h.written)

    def cap_of(self, choice, ev=None):
        """img_cap named by `choice`: "none", "exact", "short" or "big"."""
        ev = self.events if ev is None else ev
        if choice == "exact":
            _add(ev, "cap: img_cap exact")
        if choice == "short":
            _add(ev, "cap: img_cap one short")
        return {"none": None, "exact": self.total, "short": self.total - 1, "big": self.total + 4096}[choice]


# ---- packs -> bytes ---------------------------------------------------------------------------------------------------

class BPack:
    """A pack as a list of blocks (base, NumUids, the u32 internal deltas), including tables codec.Encode never
    writes (blocks with NumUids 0, blocks whose bases do not ascend, sums that wrap)."""

    def __init__(self, block_size, blocks):
        self.block_size = block_size
        self.blocks = [(int(b) & U64, int(q), [int(d) & M32 for d in ds]) for b, q, ds in blocks]
        for _, q, ds in self.blocks:
            assert len(ds) == max(q - 1, 0)

    @classmethod
    def of_uids(cls, u, bsz):
        p = gen.encode_pack_np(np.asarray(u, np.uint64), bsz)
        _, base, num, _, _ = p
        u = np.asarray(u, np.uint64)
        st = np.concatenate([[0], np.cumsum(num.astype(np.int64))])
        return cls(bsz, [(int(base[i]), int(num[i]), ((u[st[i] + 1: st[i + 1]] - u[st[i]: st[i + 1] - 1])
                                                      & np.uint64(M32)).tolist()) for i in range(base.size)])

    def block_uids(self, i):
        b, q, ds = self.blocks[i]
        out, x = [], b
        for t in range(q):
            if t:
                x = (x + ds[t - 1]) & U64
            out.append(x)
        return out

    def hand(self):
        """The pack as backup_codec_cases.HandPack: group-varint groups, one all-zero group for a 1-uid block, none for
        NumUids 0."""
        import backup_codec_cases as cases

        doff, data = [0], []
        for _, q, ds in self.blocks:
            if q:
                d = ds + [0] * ((-len(ds)) % 4 or (4 if not ds else 0))
                for g in range(0, len(d), 4):
                    data += cases.group(d[g: g + 4])
            doff.append(len(data))
        return cases.HandPack(self.block_size, [b for b, _, _ in self.blocks], [q for _, q, _ in self.blocks], doff,
                              data)


Backup = namedtuple("Backup", "rc sync launches out_off written")


class BackupPlan:
    """One dgx_decode_to_buffer_rows / dgx_dev_decode_to_buffer_rows call over `packs` (BPack or None each)."""

    def __init__(self, packs, ev=None):
        ev = set() if ev is None else ev
        self.events = ev
        self.packs = packs
        self.nrows = nr = len(packs)
        self.jobs, nblk = [], 0
        self.row_blk = []
        for r, p in enumerate(packs):
            self.row_blk.append(nblk)
            if p is None or not p.blocks:
                continue
            self.jobs.append((r, nblk, len(p.blocks)))
            nblk += len(p.blocks)
        self.row_blk.append(nblk)
        self.nblk = nblk
        self.stop = [next((i for i, (_, q, _) in enumerate(p.blocks) if q == 0), None) if p is not None else None
                     for p in packs]
        inner, bnd, last = [], [], []
        self.streams = []
        for r, p in enumerate(packs):
            if p is None or not p.blocks:
                self.streams.append(b"")
                continue
            prev = 0
            uids = []
            for i, (b, q, ds) in enumerate(p.blocks):
                u = p.block_uids(i)
                lst = u[-1] if q else b
                stopped = self.stop[r] is not None and i >= self.stop[r]
                inner.append(0 if stopped else sum(uvarint_len(d) for d in ds))
                bnd.append(0 if stopped else uvarint_len((b - prev) & U64))
                if not stopped:
                    self._boundary_events(ev, r, i, b, prev, ds)
                    uids += u
                prev = lst
                last.append(lst)
            vals = np.diff(np.array([0] + uids, dtype=object)) if uids else []
            self.streams.append(guv.put_uvarints_np(np.array([int(v) & U64 for v in vals], np.uint64)).tobytes())
        self.inner = np.array(inner, np.int64)
        self.boundary = np.array(bnd, np.int64)
        self.bytes = self.inner + self.boundary
        self.boff = np.concatenate([[0], np.cumsum(self.bytes)]).astype(np.int64)
        self.byte_tile = np.arange(nblk) // EN_TILE
        self.out_off = self.boff[self.row_blk].astype(np.uint64)
        self.total = int(self.out_off[-1]) if nr else 0
        assert [len(s) for s in self.streams] == np.diff(self.out_off.astype(np.int64)).tolist()
        self._events(ev)

    def _boundary_events(self, ev, r, i, b, prev, ds):
        d = (b - prev) & U64
        L = uvarint_len(d)
        if d == (min(1 << 7 * L, 1 << 64) - 1):
            _add(ev, f"bk: boundary varint of {L} bytes, its largest value")
        if d == (0 if L == 1 else 1 << 7 * (L - 1)):
            _add(ev, f"bk: boundary varint of {L} bytes, its smallest value")
        if i and b < prev:
            _add(ev, "bk: boundary delta wraps")
        if i == 0 and b == 0:
            _add(ev, "bk: first uid 0")
        for x in ds:
            _add(ev, f"bk: internal delta of {uvarint_len(x)} bytes")
        if (b + sum(ds)) > U64:
            _add(ev, "bk: internal delta wraps")
        if i == 0 and r and any(j[1] > 0 for j in self.jobs if j[0] < r):
            _add(ev, "bk: a row's first block after another pack's last")

    def _events(self, ev):
        nb = self.nblk
        for k, below, above in ((256, "bk: nblk = 256k - 1", "bk: nblk = 256k + 1"),
                                (EN_TILE, "bk: nblk = 2048k - 1", "bk: nblk = 2048k + 1")):
            if nb >= k - 1 and nb % k == k - 1:
                _add(ev, below)
            if nb > k and nb % k == 1:
                _add(ev, above)
        if -(-nb // EN_TILE) > 32:
            _add(ev, "bk: more than 32 byte-scan tiles")
        for r, p in enumerate(self.packs):
            if p is None or not p.blocks:
                continue
            zs = [i for i, (_, q, _) in enumerate(p.blocks) if q == 0]
            if 0 in zs:
                _add(ev, "bk: NumUids 0 as block 0")
            if len(p.blocks) - 1 in zs:
                _add(ev, "bk: NumUids 0 as the last block")
            if len(zs) >= 2:
                _add(ev, "bk: NumUids 0 twice in one row")
            if zs and any(q for _, q, _ in p.blocks[zs[0] + 1:]):
                _add(ev, "bk: blocks with data after the stop")
        live = [r for r, p in enumerate(self.packs) if p is not None and p.blocks]
        for a, z in zip(live, live[1:]):
            if any(self.packs[i] is None for i in range(a + 1, z)):
                _add(ev, "bk: a nil pack between packs")
        for r in live[1:-1]:
            if not self.streams[r]:
                _add(ev, "bk: an empty pack between packs")
        ids = [id(self.packs[r]) for r in live]
        if len(set(ids)) < len(ids):
            _add(ev, "bk: the same pack in several rows")

    def host(self, out_cap, ev=None):
        """dgx_decode_to_buffer_rows with an output of out_cap bytes (None: no output, sizes only)."""
        ev = self.events if ev is None else ev
        if self.nrows == 0:
            return Backup(OK, None, 0, self.out_off, False)
        if out_cap is None:
            _add(ev, "backup: sizes only")
            return Backup(OK, None, TB_LAUNCHES, self.out_off, False)
        if self.total == 0:
            _add(ev, "backup: total 0 bytes, the write skipped")
            return Backup(OK, None, TB_LAUNCHES, self.out_off, False)
        if self.total > out_cap:
            _add(ev, "backup: CAP")
            return Backup(ERR_CAP, None, TB_LAUNCHES, self.out_off, False)
        _add(ev, "backup: OK")
        return Backup(OK, None, TB_LAUNCHES + 1, self.out_off, True)

    def dev(self, out_cap, ev=None):
        """dgx_dev_decode_to_buffer_rows: four launches; dgx_lane_sync reports CAP."""
        ev = self.events if ev is None else ev
        if self.nrows == 0:
            return Backup(OK, OK, 0, self.out_off, False)
        cap = 0 if out_cap is None else out_cap
        sync = ERR_CAP if out_cap is not None and self.nblk and self.total > cap else OK
        return Backup(OK, sync, TB_LAUNCHES, self.out_off, out_cap is not None and sync == OK and self.total > 0)

    def cap_of(self, choice, ev=None):
        ev = self.events if ev is None else ev
        if choice == "exact":
            _add(ev, "cap: out_cap exact")
        if choice == "short":
            _add(ev, "cap: out_cap one short")
        return {"none": None, "exact": self.total, "short": self.total - 1}[choice]


# ---- fixtures ---------------------------------------------------------------------------------------------------------

RestoreFixture = namedtuple("RestoreFixture", "name rows bsz caps events")
BackupFixture = namedtuple("BackupFixture", "name packs caps events")


def simulate_restore(rows, block_size, caps=("exact",)):
    """The plan of one restore call, and every entry point's answer at each img_cap choice: (plan, {choice: (host,
    dev)}).  The events reached are plan.events."""
    p = RestorePlan(rows, block_size)
    out = {}
    for ch in caps:
        cap = p.cap_of(ch)
        out[ch] = (p.host(cap), p.dev(cap))
    return p, out


def simulate_backup(packs, caps=("exact",)):
    p = BackupPlan(packs)
    out = {}
    for ch in caps:
        cap = p.cap_of(ch)
        out[ch] = (p.host(cap), p.dev(cap))
    return p, out


class Stream:
    """Rows of uvarint bytes built value by value, tracking the byte position and the value count of the call."""

    def __init__(self):
        self.rows = [bytearray()]
        self.pos = 0
        self.nval = 0

    def row(self, empties=0):
        self.rows += [bytearray() for _ in range(empties)] + [bytearray()]
        return self

    def raw(self, bs, values=1):
        self.rows[-1] += bytes(bs)
        self.pos += len(bs)
        self.nval += values
        return self

    def value(self, L, last=0x05, cont=0x81):
        """A value of L bytes: L - 1 continuation bytes and the terminator `last`."""
        return self.raw([cont] * (L - 1) + [last])

    def pad_to(self, p):
        """1-byte values (uid + 1) up to byte position p."""
        assert p >= self.pos, (p, self.pos)
        return self.raw([1] * (p - self.pos), p - self.pos)

    def pad_values(self, m):
        """1-byte values up to value count m."""
        assert m >= self.nval
        return self.raw([1] * (m - self.nval), m - self.nval)

    def deltas(self, d):
        d = np.asarray(d, np.uint64)
        return self.raw(guv.put_uvarints_np(d).tobytes(), d.size)

    def out(self):
        return [bytes(r) for r in self.rows]


def stream_of(u):
    u = np.asarray(u, np.uint64)
    return guv.put_uvarints_np(np.diff(np.concatenate([np.zeros(1, np.uint64), u]))).tobytes()


def lengths_stream():
    """Every value length 1-10 ending at every offset of a thread's range; a terminator at the first byte of tiles 1-9
    whose value starts 1-9 bytes back; the 10-byte values ending in 0x01 and 0x00 and a non-minimal 80 00 on tile
    edges as well."""
    s = Stream()
    for L in range(1, 11):
        for o in range(EN_VT):
            e = s.pos + L - 1
            e += (o - e) % EN_VT
            s.pad_to(e - L + 1).value(L, 0x01 if L == 10 else 0x05)
    for c in range(1, 10):
        t = -(-s.pos // EN_TILE) + (1 if s.pos % EN_TILE == 0 else 0)
        s.pad_to(t * EN_TILE - c).value(c + 1, 0x01 if c == 9 else 0x07, cont=0xC3)
    t = -(-s.pos // EN_TILE) + 1
    s.pad_to(t * EN_TILE - 9).raw([0x80] * 9 + [0x00])
    s.pad_to((t + 1) * EN_TILE - 1).raw([0x80, 0x00])
    s.pad_to((t + 2) * EN_TILE - 9).raw([0xFF] * 9 + [0x01])
    return s.pad_to(s.pos + 5).out()


def row_edges_stream():
    """Leading, interior and trailing runs of empty rows; rows that start on a tile's first byte and inside a thread's
    range; a row whose first value (3 bytes) starts 2 bytes before a tile edge; every row change in one upper word."""
    s = Stream().row(1).row()
    s.pad_to(EN_TILE).row().deltas([3, 300, 70000] * 20).pad_to(EN_TILE + 203).row()
    s.deltas([5] * 100).pad_to(3 * EN_TILE - 2).row(2).value(3).pad_to(3 * EN_TILE + 40).row()
    s.deltas(np.arange(1, 400) * 37).row(1)
    return s.out()


def value_tiles_stream(m):
    """One-byte values with upper-word changes (a 5-byte value of 2^32) at value 296 (a thread's first) and value 2048
    (a tile's first), a row change at value 4096 (a tile's first) into the same upper word, m values in all."""
    s = Stream()
    s.pad_values(37 * EN_VT).deltas([1 << 32]).pad_values(EN_TILE).deltas([1 << 32])
    s.pad_values(2 * EN_TILE).row().deltas([(2 << 32) + 9]).pad_values(3 * EN_TILE - 5)
    s.deltas([1 << 32]).pad_values(m)
    return s.out()


def wide_values_stream():
    """10-byte values near 2^63: every tile's sum and the call-wide prefix wrap, the row bases with them; bytes
    outnumber values tenfold, so value tiles past m return early."""
    s = Stream()
    for r in range(3):
        if r:
            s.row()
        s.deltas([(1 << 63) + 12345 * (i + 1) + r for i in range(700)])
    return s.out()


def random_rows(rng, nrows, size, wide=False):
    out = []
    for _ in range(nrows):
        n = int(rng.integers(0, size))
        d = rng.integers(0, 1 << int(rng.integers(1, 40)), n, dtype=np.uint64)
        if wide and n:
            d[rng.integers(0, n, max(1, n // 50))] += np.uint64(1 << 32)
        out.append(guv.put_uvarints_np(d).tobytes())
    return out


def exact_bytes_stream(rng, n):
    rows = random_rows(rng, 5, n // 40, wide=True)
    s = Stream()
    s.rows = [bytearray(r) for r in rows]
    s.pos = sum(len(r) for r in rows)
    assert s.pos <= n - 2
    return s.pad_to(n).out()


def segments_stream(lengths, step=3):
    """Segments of the given lengths, each in its own upper word."""
    return [stream_of(eg.runs(lengths, step))]


def bad_stream(kind):
    """A malformed call: the bad bytes in the second of three rows (or the last)."""
    good = stream_of(np.arange(1, 300) * 1000)
    s = Stream().raw(good, 0)
    if kind == "tenth byte 2":
        s.row().pad_to(EN_TILE - 9).raw([0x80] * 9 + [0x02]).row().raw(good, 0)
    elif kind == "eleven":
        s.row().pad_to(2 * EN_TILE - 11).raw([0xFF] * 11 + [0x01]).row().raw(good, 0)
    elif kind == "row ends inside":
        s.row().raw([3, 4, 0x85]).row(1).raw([3, 4]).raw(good, 0)
    elif kind == "last row ends inside":
        s.row().raw([3, 4, 0xFF, 0xFF])
    return s.out()


def many_rows(rng, nrows):
    """nrows short rows of 1 to 4 blocks (BlockSize 2), empty ones among them."""
    out = []
    for i in range(nrows):
        k = int(rng.integers(0, 9)) if i % 7 else 0
        out.append(guv.put_uvarints_np(rng.integers(0, 1 << 30, k, dtype=np.uint64)).tobytes())
    return out


def all_restore_fixtures():
    rng = np.random.default_rng(5200)
    F = []

    def add(name, rows, bsz, events, caps=("exact", "short", "none")):
        F.append(RestoreFixture(name, [bytes(r) for r in rows], bsz, caps, set(events)))

    add("value lengths at thread offsets and tile edges", lengths_stream(), 256,
        {f"val: length {L} ending at thread offset {o}" for L in range(1, 11) for o in range(EN_VT)}
        | {f"val: terminator at a tile's first byte, {c} bytes back in the previous tile" for c in range(1, 10)}
        | {"val: a 10-byte value ending in 0x01", "val: a 10-byte value ending in 0x00, non-minimal",
           "val: non-minimal 80 00", "cap: img_cap exact", "cap: img_cap one short", "restore: OK", "restore: CAP",
           "restore: sizes only"})
    add("row edges and empty rows", row_edges_stream(), 3, {
        "row: leading empty rows", "row: trailing empty rows", "row: an interior run of empty rows",
        "row: starts on a tile's first byte", "row: starts inside a thread's range",
        "row: its first value's terminator lies in the tile after its start", "seg: row change with the same upper word"})
    for m, ev in ((3 * EN_TILE - 1, "seg: m = 2048k - 1"), (3 * EN_TILE, "seg: m = 2048k"),
                  (3 * EN_TILE + 1, "seg: m = 2048k + 1")):
        add(f"value tiles, m = {m}", value_tiles_stream(m), 100, {
            ev, "seg: upper-word change at a value tile's first value", "seg: upper-word change at a thread's first value",
            "seg: row change at a value tile's first value", "seg: row change with the same upper word"})
    add("10-byte values, wrapping sums", wide_values_stream(), 64, {
        "val: a tile's value sum wraps u64", "val: the call-wide prefix wraps before a later row's first value",
        "seg: tiles past m return early", "val: length 10 ending at thread offset 3"})
    add("33 or more tiles of look-back", random_rows(rng, 9, 9000, wide=True), 256, {"val: 33 or more tiles of look-back"})
    for k, r in ((2, -1), (2, 0), (3, 1)):
        n = EN_TILE * k + r
        add(f"n = {n} bytes", exact_bytes_stream(rng, n), 10,
            {{-1: "val: n = 2048k - 1 bytes", 0: "val: n = 2048k bytes", 1: "val: n = 2048k + 1 bytes"}[r]})
    lone = segments_stream([1] * 2100, step=1)
    add("2100 one-value segments, bs 1", lone, 1, {"seg: more than 2048 segments", "blk: more than 2048 blocks",
                                                    "bsz 1"})
    add("2100 one-value segments, bs 0", lone, 0, {"seg: more than 2048 segments", "bsz 0"})
    add("segments of bsz k - 1, k, k + 1", segments_stream([30, 31, 29, 10, 11, 9, 1]), 10, {
        "blk: segment of bsz * k values", "blk: segment of bsz * k + 1 values", "blk: segment of bsz * k - 1 values"})
    add("num 129 to 258", segments_stream([129, 130, 257, 258, 3]), 1000, {
        "blk: num 129", "blk: num 130", "blk: num 257", "blk: num 258"})
    wide = random_rows(rng, 4, 3000, wide=True)
    add("bs 2^31 - 1", wide, (1 << 31) - 1, {"bsz 2^31 - 1"})
    add("bs 2^32 - 1", wide, (1 << 32) - 1, {"bsz 2^32 - 1"})
    add("2048 rows", many_rows(rng, EN_TILE), 2, {
        "img: 2048 rows, one tile", "img: delta padding of 0 bytes", "img: delta padding of 15 bytes"}
        | {f"img: metadata padding of {p} bytes" for p in (0, 4, 8, 12)})
    add("2049 rows", many_rows(rng, EN_TILE + 1), 2, {"img: 2049 rows, two tiles"})
    bad_caps = ("none", "big")
    add("malformed: a 10th byte of 0x02 across a tile edge", bad_stream("tenth byte 2"), 256, {
        "bad: overflow, a 10th byte > 1 across a tile edge", "restore: ARG with an image",
        "restore: ARG without an image"}, bad_caps)
    add("malformed: 11 continuation bytes across a tile edge", bad_stream("eleven"), 256, {
        "bad: overflow, 11 or more bytes across a tile edge"}, bad_caps)
    add("malformed: a row ends inside a value, an empty row follows", bad_stream("row ends inside"), 256, {
        "bad: a row ends inside a value, an empty row follows"}, bad_caps)
    add("malformed: the last row ends inside a value", bad_stream("last row ends inside"), 256, {
        "bad: the last row ends inside a value"}, bad_caps)
    add("every row empty", [b""] * 3, 256, {"restore: every row empty, no launch"}, ("none", "big"))
    return F


def boundary_pack():
    """Blocks whose boundary deltas take each varint length 1-10 at its smallest and largest value, internal deltas of
    every length 1-5, a first uid of 0 and boundaries that wrap."""
    blocks, last = [], 0
    targets = [0, 1 << 64 - 1]
    for L in range(1, 11):
        targets += [min(1 << 7 * L, 1 << 64) - 1, 0 if L == 1 else 1 << 7 * (L - 1)]
    inner = [1, 1 << 7, 1 << 14, 1 << 21, 1 << 28, M32]
    for i, d in enumerate(targets):
        base = (last + d) & U64
        ds = [inner[(i + t) % len(inner)] for t in range(i % 6 + 1)]
        blocks.append((base, len(ds) + 1, ds))
        last = (base + sum(ds)) & U64
    blocks.append((U64 - 2, 2, [5]))
    return BPack(256, blocks)


def stop_packs():
    """NumUids 0 as block 0, as the last block, and twice in one row 600 blocks apart, with data after each."""
    one = [(10 * i + 5, 2, [3]) for i in range(900)]
    first = BPack(256, [(77, 0, [])] + one[:40])
    lastz = BPack(256, one[:30] + [(999, 0, [])])
    twice = BPack(256, one[:100] + [(1, 0, [])] + one[100:700] + [(2, 0, [])] + one[700:])
    return [first, lastz, twice]


def interleaved_packs(rng):
    """Nil and empty packs between packs; a row's first base far below the previous pack's last uid; one pack in three
    rows."""
    big = BPack.of_uids(np.cumsum(rng.integers(1, 1 << 20, 3000, dtype=np.uint64)) + np.uint64(1 << 40), 256)
    small = BPack.of_uids(np.arange(5, 2000, 7, dtype=np.uint64), 64)
    empty = BPack(256, [(123, 0, []), (456, 3, [1, 2])])
    return [None, big, None, empty, small, None, big, empty, big, small, None]


def ones_pack(nblk, base=1):
    """nblk blocks of one uid each."""
    return BPack(1, [(base + 3 * i, 1, []) for i in range(nblk)])


def all_backup_fixtures():
    rng = np.random.default_rng(5201)
    F = []

    def add(name, packs, events, caps=("exact", "short", "none")):
        F.append(BackupFixture(name, packs, caps, set(events)))

    add("boundary varints of every length", [boundary_pack(), None, boundary_pack()],
        {f"bk: boundary varint of {L} bytes, its {w} value" for L in range(1, 11) for w in ("smallest", "largest")}
        | {f"bk: internal delta of {L} bytes" for L in range(1, 6)}
        | {"bk: first uid 0", "bk: boundary delta wraps", "bk: internal delta wraps", "cap: out_cap exact",
           "cap: out_cap one short", "backup: OK", "backup: CAP", "backup: sizes only"})
    add("NumUids 0 blocks", stop_packs(), {"bk: NumUids 0 as block 0", "bk: NumUids 0 as the last block",
                                           "bk: NumUids 0 twice in one row", "bk: blocks with data after the stop"})
    add("interleaved nil and empty packs", interleaved_packs(rng), {
        "bk: a nil pack between packs", "bk: an empty pack between packs", "bk: the same pack in several rows",
        "bk: a row's first block after another pack's last"})
    for nb, ev in ((255, "bk: nblk = 256k - 1"), (257, "bk: nblk = 256k + 1"), (2047, "bk: nblk = 2048k - 1"),
                   (4097, "bk: nblk = 2048k + 1")):
        add(f"nblk = {nb}", [ones_pack(nb - 100), None, ones_pack(100, 7)], {ev})
    p = ones_pack(8200)
    add("37 byte-scan tiles, one pack in nine rows", [p] * 9, {"bk: more than 32 byte-scan tiles",
                                                              "bk: the same pack in several rows"})
    add("total 0 bytes", [None, BPack(256, [(5, 0, []), (6, 2, [1])]), None], {
        "backup: total 0 bytes, the write skipped"}, ("exact", "none"))
    add("zipf packs", [BPack.of_uids(gen.zipf_gaps(rng, int(rng.integers(1, 4000))), int(bs))
                       for bs in (1, 5, 256, 1000, 256, 64)], set())
    return F
