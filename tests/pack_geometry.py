"""Host model of the UidPack readers' block walk (decode_kernel.cuh, compressed_kernel.cuh,
list_uids_unfiltered_kernel.cuh and the launches of dgx_api.cu), and fixtures aimed at its window, batch and warp
boundaries.

Every reader that takes a pack walks it with the same plan: a warp owns D_BPW blocks and takes them in batches of up
to 32; one window per batch holds at most D_WB delta bytes from a 16-byte-aligned win0; the batch takes the leading run
of blocks that fit; a block of more than 256 uids (or a run of 0) goes to a lane-serial slow path; the walk resumes
behind what it took.  The model restates, from a pack's real arrays (base, num, delta_off, deltas):
  - decode_seek_kernel and decode_warp_run: the seek, each batch's win0, fits, run, window bytes, the slow path, every
    expanded block's groups and expand_block rounds, the trimmed head and the parity of each block's first output word;
    decode_batch_kernel's job table and job_of;
  - icw_range_by_v / icw_range_by_block (which must agree), icw_probe_blocks' touched mask, f, run and want, the side
    that searches, and for the rows form each block's slot and the ballot rounds of 32 probes; compact_kernel's tiles;
  - icw_mx_locate_kernel's units and icw_mx_probe_kernel's lanes of units: window rounds, leaders, short (lane-serial)
    and long (whole-warp) units, the serial group of a block of more than 256 uids;
  - luu_locate, luu_rows_kernel (skip, sblk, |S_i|, len, count) and luu_write_blocks: the start clamped to sblk, each
    lane's js, je and lower, the live prefix and the run, the blocks never loaded, and each insert's position.
The walks are exact set arithmetic over the decoded blocks, so the model also yields each call's result, which the
tests compare with the oracle.  What the kernels decide is named as *events*; fixtures name the events they must
reach, and the model refuses a name that is not registered in EVENTS.

The constants are read from the CUDA sources; the slow-path test, the probe-direction test and the two range-side
choices are matched as text, so a rewrite fails here loudly instead of leaving the fixtures aimed at stale edges.

tests/test_pack_geometry.py checks the fixtures on the CPU; tests/test_gpu_pack_edges.py runs them through the
kernels.
"""
from __future__ import annotations

import ctypes as C
import os
import re
from bisect import bisect_left, bisect_right
from collections import namedtuple

import numpy as np

from oracle import pyoracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")
U64 = (1 << 64) - 1
MAX_FIRST = 0x7FFFFFFF


def _src(fn):
    with open(os.path.join(CSRC, fn)) as f:
        return f.read()


def _const(text, fn, name):
    m = re.search(r"\bconstexpr\s+\w+\s+" + name + r"\s*=\s*(\d+)u?\s*;", text)
    if not m:
        raise KeyError(f"constexpr {name} not found in {fn}: the pack model needs it")
    return int(m.group(1))


def read_constants() -> dict:
    dec, icw, luu, api = _src("decode_kernel.cuh"), _src("compressed_kernel.cuh"), \
        _src("list_uids_unfiltered_kernel.cuh"), _src("dgx_api.cu")
    K = {n: _const(dec, "decode_kernel.cuh", n) for n in ("D_BPW", "D_WB", "D_WARPS", "D_MAXG", "D_STAGE")}
    K["MX_SERIAL"] = _const(icw, "compressed_kernel.cuh", "MX_SERIAL")
    m = re.search(r"constexpr int CP_NT = (\d+), CP_VT = (\d+), CP_TILE = CP_NT \* CP_VT;", icw)
    if not m:
        raise KeyError("CP_NT / CP_VT / CP_TILE not found in compressed_kernel.cuh")
    K["CP_NT"], K["CP_VT"] = int(m.group(1)), int(m.group(2))
    slow = [re.findall(p, t) for p, t in (
        (r"\(num > (\d+)u && lane < nb\)", dec),                              # decode_warp_run
        (r"\(num > (\d+)u && lane >= f && lane < f \+ \(run \? run : 1\)\)", icw),  # icw_probe_blocks
        (r"num <= (\d+)u && \(dnext - win0 <= \(u64\)D_WB\)", icw),          # icw_mx_probe_kernel
        (r"\(num > (\d+)u && lane < run\)", luu))]                            # luu_write_blocks
    if any(len(s) != 1 for s in slow) or len({s[0] for s in slow}) != 1:
        raise ValueError("the slow-path test `num > 256u` of a pack reader changed: restate it in the pack model "
                         "(tests/pack_geometry.py)")
    K["SLOW_NUM"] = int(slow[0][0])
    m = re.search(r"if \(hi - lo <= (\d+)u \* n\) \{", icw)
    if not m:
        raise ValueError("icw_probe_slice's probe-direction test `hi - lo <= 4u * n` changed: restate it in the model")
    K["PROBE_RATIO"] = int(m.group(1))
    if not re.search(r"if \(m < nb\) icw_ranges_by_v_kernel", api):
        raise ValueError("icw_impl's range-side choice `m < nb` changed: restate it in the pack model")
    if not re.search(r"J\.by_v = pnb > m;", api):
        raise ValueError("icw_rows_impl's range-side choice `pnb > m` changed: restate it in the pack model")
    return K


K = read_constants()
D_BPW, D_WB, SLOW_NUM, MX_SERIAL = K["D_BPW"], K["D_WB"], K["SLOW_NUM"], K["MX_SERIAL"]
CP_TILE = K["CP_NT"] * K["CP_VT"]

# ---- events -----------------------------------------------------------------------------------------------------------

_SHARED = (
    "win0 aligned", "win0 misaligned by 15", "window of exactly D_WB bytes", "next block one byte past the window",
    "zero-byte window", "all 32 lanes fit", "run cut at lane 1", "run cut at lane 31", "partial last batch",
    "slow path, block alone past the window", "slow block at lane 0", "slow block at lane 31",
    "slow block at the first lane of a warp's second batch", "fast batch after a slow one in the same warp",
    "two slow blocks in one run", "expand 0 groups", "expand 32 groups", "expand 33 groups", "expand 64 groups",
    "delta 0xFFFFFFFF", "running sum past 2^32")
_READERS = ("dec", "icw", "mx", "luu")
EVENTS = {f"{r}: {e}" for r in _READERS for e in _SHARED} - {
    # the matrix cuts its run before a block of more than 256 uids, so such a block always leads its own group
    "mx: slow block at lane 31", "mx: two slow blocks in one run",
    "mx: slow block at the first lane of a warp's second batch",
    # a matrix warp is 32 positions, not batches of a 64-block run: there is no partial batch of blocks
    "mx: partial last batch",
} | {
    "dec: seek 0", "dec: seek on a block's base", "dec: seek on a block's last uid", "dec: seek between two blocks",
    "dec: seek below the first base", "dec: seek above the last uid", "dec: trimmed head, first word odd",
    "dec: trimmed head, first word even", "dec: later block written from an odd word",
    "batch: empty pack left out of the table", "batch: warp starts a later job", "batch: second warp of a job",
    "batch: 65th block alone in its warp",
    "icw: ranges by v", "icw: ranges by block", "icw: m = nb - 1", "icw: m = nb", "icw: m = nb + 1",
    "icw: after splits a block's v elements (by v)", "icw: after equal to a base", "icw: after one below a base",
    "icw: after past the last uid", "icw: v holds a block's base", "icw: v holds a base - 1",
    "icw: v holds a block's last uid", "icw: v below the first base", "icw: v above the last uid",
    "icw: batch touches nothing", "icw: all lanes from f > 0 fit", "icw: touched block at lane 31 only",
    "icw: run cut by an untouched block, touched blocks past it", "icw: slice of 4n searches the block",
    "icw: slice of 4n + 1 is searched by the block", "icw: window stops at the last touched block",
    "compact: m a multiple of the tile", "compact: m one past a tile", "compact: several tiles",
    "rows: slot equals hi - lo", "rows: slot equals NumUids", "rows: matches at lanes 31 and 0 of consecutive rounds",
    "rows: packs on both sides of the range choice", "rows: gather grid set by the row count",
    "rows: empty and NULL rows",
    "mx: unit of MX_SERIAL elements", "mx: unit of MX_SERIAL + 1 elements", "mx: block with 31 units",
    "mx: block with 32 units", "mx: block with 33 units", "mx: block with 65 units",
    "mx: a block's units span two warps", "mx: row starts in the previous row's last block",
    "mx: window round cut by the byte budget", "mx: slow group at f > 0",
    "luu: after below the first base", "luu: after on a block's last uid", "luu: after on a base",
    "luu: after on the pack's last uid", "luu: seek block on a warp boundary", "luu: warp starts at the seek block",
    "luu: cut on a block's first position", "luu: cut one past a block's first position",
    "luu: cut on the last value of lane 31's block", "luu: cut on an insert", "luu: cut on a pack uid",
    "luu: cut right after a drop", "luu: blocks past the cut never loaded", "luu: cut inside a slow-path walk",
    "luu: entry on the next block's base", "luu: entry below the first base", "luu: entry above the last uid",
    "luu: drop of a block's last uid, next base one more", "luu: row of length 0 next to full rows",
    "luu: insert past the cut",
}


def _add(ev, name):
    if name not in EVENTS:
        raise KeyError(f"event {name!r} is not registered in pack_geometry.EVENTS")
    ev.add(name)


# ---- packs ------------------------------------------------------------------------------------------------------------

def gv_bytes_used(t):
    return 5 + (t & 3) + ((t >> 2) & 3) + ((t >> 4) & 3) + (t >> 6)


def gv_groups(num):
    return (num + 2) // 4 if num > 1 else 0


class Pack:
    """A pack from its arrays, each block decoded the way gv_walk_block reads it (bytes past the end read as 0)."""

    def __init__(self, base, num, delta_off, deltas, block_size=256):
        self.block_size = int(block_size)
        self.base = [int(x) for x in base]
        self.num = [int(x) for x in num]
        self.doff = [int(x) for x in delta_off]
        self.deltas = np.ascontiguousarray(np.asarray(deltas, np.uint8))
        self.nb = len(self.base)
        self.uoff = [0]
        for n in self.num:
            self.uoff.append(self.uoff[-1] + n)
        raw = self.deltas.tobytes() + bytes(64)
        self.blocks, self.maxdelta = [], []
        for b in range(self.nb):
            out, md, p, last = [self.base[b]], 0, self.doff[b], self.base[b]
            while len(out) < self.num[b]:
                tag, d = raw[p], p + 1
                for j in range(4):
                    if len(out) >= self.num[b]:
                        break
                    ln = ((tag >> (2 * j)) & 3) + 1
                    v = int.from_bytes(raw[d:d + ln], "little")
                    d += ln
                    md = max(md, v)
                    last = (last + v) & U64
                    out.append(last)
                p += gv_bytes_used(tag)
            self.blocks.append(out[: self.num[b]])
            self.maxdelta.append(md)
        self.flat = [u for blk in self.blocks for u in blk]

    def arrays(self):
        return (self.block_size, np.asarray(self.base, np.uint64), np.asarray(self.num, np.uint32),
                np.asarray(self.doff, np.uint64), self.deltas)

    def block_of(self, x):  # pack_block_of: last b with base[b] <= x, or -1
        return bisect_right(self.base, x) - 1


def check_table(pk):
    """walk_block_table's acceptance test (dgx_api.cu): every block holds at least 5 bytes per group."""
    for b in range(pk.nb):
        need = 5 * ((pk.num[b] + 2) // 4) if pk.num[b] > 1 else 0
        assert pk.doff[b + 1] >= pk.doff[b] and pk.doff[b + 1] - pk.doff[b] >= need, b


def _block_offsets(n, nbytes=None, width=1, start=1):
    """Low 32 bits of a block of n uids whose deltas take nbytes bytes as the Encoder writes them (or are all `width`
    bytes wide): the widths are chosen so that the byte count lands where a fixture needs it."""
    if n == 1:
        return [start]
    g = (n - 1 + 3) // 4
    pad = 4 * g - (n - 1)
    if nbytes is None:
        lens = [width] * (n - 1)
    else:
        extra = nbytes - g - pad - (n - 1)
        assert 0 <= extra <= 3 * (n - 1), (n, nbytes)
        lens = []
        for _ in range(n - 1):
            a = min(3, extra)
            extra -= a
            lens.append(1 + a)
    out = [start]
    for i, ln in enumerate(lens):
        out.append(out[-1] + (1 << (8 * (ln - 1))) + i % 7)
    assert out[-1] < 1 << 32
    return out


def seg_pack(specs, seg0=1):
    """A pack from the numpy Encoder (gen.encode_pack_np) whose block k lies alone in 32-bit segment seg0 + k:
    specs[k] = (n, nbytes) or (n, None, width), or a list of low-32 offsets."""
    import gen

    uids = []
    for k, s in enumerate(specs):
        offs = s if isinstance(s, list) else _block_offsets(s[0], s[1], *(s[2:] or (1,)))
        uids.extend(((seg0 + k) << 32) | o for o in offs)
    bs = max(256, max(len(s) if isinstance(s, list) else s[0] for s in specs))
    enc = gen.encode_pack_np(np.array(uids, np.uint64), bs)
    pk = Pack(enc[1], enc[2], enc[3], enc[4], bs)
    assert pk.nb == len(specs)
    return pk


def run_pack(nblocks, per=9, start=1 << 33, step=3):
    """A pack of nblocks blocks of `per` uids `step` apart, BlockSize `per` (10 bytes a block at per = 9)."""
    import gen

    u = start + np.cumsum(np.full(nblocks * per, step, np.uint64))
    enc = gen.encode_pack_np(u, per)
    return Pack(enc[1], enc[2], enc[3], enc[4], per)


def hand_pack(blocks, block_size=256):
    """A pack written by hand: blocks = [(base, deltas bytes, num)], every block's bytes back to back."""
    base = [b for b, _, _ in blocks]
    num = [n for _, _, n in blocks]
    raw = b"".join(d for _, d, _ in blocks)
    doff = [0]
    for _, d, _ in blocks:
        doff.append(doff[-1] + len(d))
    pk = Pack(base, num, doff, np.frombuffer(raw, np.uint8).copy() if raw else np.zeros(0, np.uint8), block_size)
    check_table(pk)
    return pk


def gv_encode(deltas):
    """go-groupvarint groups of 4 of a list of u32 deltas, the last group zero-padded."""
    out = bytearray()
    d = list(deltas) + [0] * (-len(deltas) % 4)
    for g in range(0, len(d), 4):
        lens = [1 + (x >= 1 << 8) + (x >= 1 << 16) + (x >= 1 << 24) for x in d[g:g + 4]]
        out.append(sum((ln - 1) << (2 * j) for j, ln in enumerate(lens)))
        for x, ln in zip(d[g:g + 4], lens):
            out += x.to_bytes(ln, "little")
    return bytes(out)


def concat_packs(packs):
    """Packs in disjoint uid ranges as one list of uids: what a union of them decodes to."""
    return np.array(sorted(u for p in packs if p is not None for u in p.flat), np.uint64)


# ---- the shared plan ----------------------------------------------------------------------------------------------------

def _lead(fits):
    n = 0
    while n < len(fits) and fits[n]:
        n += 1
    return n


def _run_events(ev, R, f, run, nlanes):
    if f == 0 and run == 32:
        _add(ev, f"{R}: all 32 lanes fit")
    cut = f + run
    if run and cut < nlanes and cut in (1, 31):
        _add(ev, f"{R}: run cut at lane {cut}")


def _window_events(ev, R, pk, first, win0, wend, nxt):
    r = pk.doff[first] & 15
    if r == 0:
        _add(ev, f"{R}: win0 aligned")
    elif r == 15:
        _add(ev, f"{R}: win0 misaligned by 15")
    if wend - win0 == D_WB:
        _add(ev, f"{R}: window of exactly D_WB bytes")
    if wend == win0:
        _add(ev, f"{R}: zero-byte window")
    if nxt is not None and nxt - win0 == D_WB + 1:
        _add(ev, f"{R}: next block one byte past the window")
    assert 0 <= wend - win0 <= D_WB


def _expand_events(ev, R, pk, b):
    g = gv_groups(pk.num[b])
    if g in (0, 32, 33, 64):
        _add(ev, f"{R}: expand {g} groups")
    if pk.maxdelta[b] == 0xFFFFFFFF:
        _add(ev, f"{R}: delta 0xFFFFFFFF")
    if pk.blocks[b][-1] - pk.base[b] >= 1 << 32:
        _add(ev, f"{R}: running sum past 2^32")
    return (g + 31) // 32  # expand_block rounds


def _slow_events(ev, R, pk, b, lanes, forced, nbatch):
    if forced:
        _add(ev, f"{R}: slow path, block alone past the window")
    big = [i for i in lanes if pk.num[b + i] > SLOW_NUM]
    for i in big:
        if i == 0:
            _add(ev, f"{R}: slow block at lane 0")
            if nbatch == 1:
                _add(ev, f"{R}: slow block at the first lane of a warp's second batch")
        if i == 31:
            _add(ev, f"{R}: slow block at lane 31")
    if len(big) >= 2:
        _add(ev, f"{R}: two slow blocks in one run")


Batch = namedtuple("Batch", "b f run win0 wend slow")

# ---- decode -------------------------------------------------------------------------------------------------------------

Decoded = namedtuple("Decoded", "events result launches first_block skip out_len batches")


def decode_seek(pk, seek, ev):
    first = trim = 0
    if pk.nb and seek:
        idx = bisect_left(pk.base, seek)
        if idx == 0:
            _add(ev, "dec: seek below the first base")
        elif idx < pk.nb and pk.base[idx] == seek:
            _add(ev, "dec: seek on a block's base")
            first = idx
        else:
            b = idx - 1
            below = sum(u < seek for u in pk.blocks[b])
            if below < pk.num[b]:
                first, trim = b, below
                if below == pk.num[b] - 1 and pk.blocks[b][-1] == seek:
                    _add(ev, "dec: seek on a block's last uid")
            else:
                first = idx
                if idx == pk.nb:
                    _add(ev, "dec: seek above the last uid")
                else:
                    _add(ev, "dec: seek between two blocks")
    elif pk.nb:
        _add(ev, "dec: seek 0")
    skip = (pk.uoff[first] if first < pk.nb else pk.uoff[pk.nb]) + trim
    return first, skip, pk.uoff[pk.nb] - skip


def _decode_warp(ev, pk, first, skip, gw, out, out_word, batches):
    b = first + gw * D_BPW
    bend = min(b + D_BPW, pk.nb)
    nbatch, prev_slow = 0, False
    while b < bend:
        nl = min(32, bend - b)
        if nl < 32:
            _add(ev, "dec: partial last batch")
        win0 = pk.doff[b] & ~15
        fits = [pk.doff[b + i + 1] - win0 <= D_WB for i in range(nl)]
        n = _lead(fits)
        forced = n == 0
        n = max(n, 1)
        wend = pk.doff[b + n]
        _run_events(ev, "dec", 0, n if not forced else 0, nl)
        if wend - win0 > D_WB or any(pk.num[b + i] > SLOW_NUM for i in range(n)):
            _slow_events(ev, "dec", pk, b, range(n), forced, nbatch)
            for i in range(n):
                for e, y in enumerate(pk.blocks[b + i]):
                    if pk.uoff[b + i] + e >= skip:
                        out[pk.uoff[b + i] + e - skip] = y
            batches.append(Batch(b, 0, n, win0, wend, True))
            prev_slow = True
            b += n
            nbatch += 1
            continue
        if prev_slow:
            _add(ev, "dec: fast batch after a slow one in the same warp")
        _window_events(ev, "dec", pk, b, win0, wend, pk.doff[b + n + 1] if n < nl else None)
        for i in range(n):
            bi = b + i
            _expand_events(ev, "dec", pk, bi)
            e0 = max(skip - pk.uoff[bi], 0)
            if e0 < pk.num[bi]:
                word = out_word + pk.uoff[bi] + e0 - skip
                if e0 > 0:
                    _add(ev, f"dec: trimmed head, first word {'odd' if word & 1 else 'even'}")
                elif word & 1:
                    _add(ev, "dec: later block written from an odd word")
                for e in range(e0, pk.num[bi]):
                    out[pk.uoff[bi] + e - skip] = pk.blocks[bi][e]
        batches.append(Batch(b, 0, n, win0, wend, False))
        b += n
        nbatch += 1


def decode_plan(pk, seek=0, out_word=0) -> Decoded:
    """dgx_decode / dgx_dev_decode of pk from `seek`, the output starting at a word of parity out_word."""
    ev = set()
    first, skip, out_len = decode_seek(pk, seek, ev)
    out = [None] * out_len
    batches = []
    for gw in range(-(-pk.nb // D_BPW)):
        _decode_warp(ev, pk, first, skip, gw, out, out_word, batches)
    assert None not in out
    return Decoded(ev, np.array(out, np.uint64), 1 + (1 if pk.nb else 0), first, skip, out_len, batches)


def job_of(starts, x):
    """job_of: the last job whose start is <= x, by the kernel's search."""
    lo, hi = 0, len(starts)
    while hi - lo > 1:
        mid = (lo + hi) >> 1
        if starts[mid] <= x:
            lo = mid
        else:
            hi = mid
    return lo


BatchDecoded = namedtuple("BatchDecoded", "events results launches warp_base jobs")


def decode_batch_plan(packs) -> BatchDecoded:
    """decode_batch_kernel over packs (None: a NULL pack), each decoded in full into its own list."""
    ev = set()
    jobs, wb, warps = [], [], 0
    for i, p in enumerate(packs):
        if p is None or p.nb == 0:
            _add(ev, "batch: empty pack left out of the table")
            continue
        jobs.append(i)
        wb.append(warps)
        warps += -(-p.nb // D_BPW)
        if p.nb % D_BPW == 1 and p.nb > D_BPW:
            _add(ev, "batch: 65th block alone in its warp")
    outs = {i: [None] * len(packs[i].flat) for i in jobs}
    for gw in range(warps):
        j = job_of(wb, gw)
        assert wb[j] <= gw and (j + 1 == len(wb) or gw < wb[j + 1])
        if gw == wb[j] and j > 0:
            _add(ev, "batch: warp starts a later job")
        if gw > wb[j]:
            _add(ev, "batch: second warp of a job")
        _decode_warp(ev, packs[jobs[j]], 0, 0, gw - wb[j], outs[jobs[j]], 0, [])
    res = [np.array(outs[i], np.uint64) if i in outs else np.zeros(0, np.uint64) for i in range(len(packs))]
    return BatchDecoded(ev, res, 1 if jobs else 0, wb, jobs)


# ---- IntersectCompressedWith ------------------------------------------------------------------------------------------

def icw_ranges_by_v(pk, v, after):
    m = len(v)
    vlo, vhi = [0] * pk.nb, [0] * pk.nb
    for j in range(m):
        x = v[j]
        if x < after:
            continue
        b = pk.block_of(x)
        if b < 0:
            continue
        bp = bn = -2
        if j > 0 and v[j - 1] >= after:
            bp = pk.block_of(v[j - 1])
        if j + 1 < m:
            bn = pk.block_of(v[j + 1])
        if bp != b:
            vlo[b] = j
        if bn != b:
            vhi[b] = j + 1
    return vlo, vhi


def icw_ranges_by_block(pk, v, after):
    m = len(v)
    vlo, vhi = [0] * pk.nb, [0] * pk.nb
    for b in range(pk.nb):
        lo = bisect_left(v, max(pk.base[b], after))
        hi = bisect_left(v, pk.base[b + 1]) if b + 1 < pk.nb else m
        if hi > lo:
            vlo[b], vhi[b] = lo, hi
    return vlo, vhi


def _icw_input_events(ev, pk, v, after):
    m, nb = len(v), pk.nb
    if m - nb in (-1, 0, 1):
        _add(ev, f"icw: m = nb{'' if m == nb else (' + 1' if m > nb else ' - 1')}")
    vs = set(v)
    last = pk.flat[-1]
    for b in range(nb):
        if pk.base[b] in vs:
            _add(ev, "icw: v holds a block's base")
        if pk.base[b] - 1 in vs and b > 0:
            _add(ev, "icw: v holds a base - 1")
        if pk.blocks[b][-1] in vs:
            _add(ev, "icw: v holds a block's last uid")
        if after == pk.base[b] and b > 0:
            _add(ev, "icw: after equal to a base")
        if after == pk.base[b] - 1 and b > 0:
            _add(ev, "icw: after one below a base")
    if after > last:
        _add(ev, "icw: after past the last uid")
    if v and v[0] < pk.base[0]:
        _add(ev, "icw: v below the first base")
    if v and v[-1] > last:
        _add(ev, "icw: v above the last uid")
    if m < nb:
        for j in range(1, m):
            if v[j - 1] < after <= v[j] and pk.block_of(v[j - 1]) == pk.block_of(v[j]) >= 0:
                _add(ev, "icw: after splits a block's v elements (by v)")


def _probe_rounds(ev, hits):
    """The ballot rounds of 32 probes: hits is the ordered list of probe outcomes of one slice."""
    rounds = [hits[i:i + 32] for i in range(0, len(hits), 32)]
    for a, c in zip(rounds, rounds[1:]):
        if len(a) == 32 and a[31] and c[0]:
            _add(ev, "rows: matches at lanes 31 and 0 of consecutive rounds")


def _icw_warp(ev, pk, vlo, vhi, v, b, match, batches):
    """icw_probe_blocks over blocks [b, b + D_BPW): match(block, j) for every v[j] found in the pack."""
    bend = min(b + D_BPW, pk.nb)
    nbatch, prev_slow = 0, False
    while b < bend:
        nl = min(32, bend - b)
        if nl < 32:
            _add(ev, "icw: partial last batch")
        touched = [i for i in range(nl) if vhi[b + i] > vlo[b + i]]
        if not touched:
            _add(ev, "icw: batch touches nothing")
            b += 32
            continue
        f = touched[0]
        win0 = pk.doff[b + f] & ~15
        run = _lead([pk.doff[b + i + 1] - win0 <= D_WB for i in range(f, nl)])
        _run_events(ev, "icw", f, run, nl)
        if f > 0 and f + run == 32:
            _add(ev, "icw: all lanes from f > 0 fit")
        r = run if run else 1
        if run == 0 or any(pk.num[b + i] > SLOW_NUM for i in range(f, f + r)):
            _slow_events(ev, "icw", pk, b, range(f, f + r), run == 0, nbatch)
            for i in touched:
                if i < f + r:
                    blk = set(pk.blocks[b + i])
                    for j in range(vlo[b + i], vhi[b + i]):
                        if v[j] in blk:
                            match(b + i, j)
            batches.append(Batch(b, f, r, win0, None, True))
            prev_slow = True
            b += f + r
            nbatch += 1
            continue
        if prev_slow:
            _add(ev, "icw: fast batch after a slow one in the same warp")
        want = [i for i in touched if i < f + run]
        last_t = want[-1]
        wend = pk.doff[b + last_t + 1]
        if want == [31]:
            _add(ev, "icw: touched block at lane 31 only")
        if last_t + 1 < f + run:
            _add(ev, "icw: window stops at the last touched block")
        if f + run < nl and any(i > f + run for i in touched) and f + run not in touched:
            _add(ev, "icw: run cut by an untouched block, touched blocks past it")
        _window_events(ev, "icw", pk, b + f, win0, wend,
                       pk.doff[b + last_t + 2] if last_t + 1 == f + run and f + run < nl else None)
        for i in want:
            bi = b + i
            _expand_events(ev, "icw", pk, bi)
            lo, hi, n = vlo[bi], vhi[bi], pk.num[bi]
            blk = pk.blocks[bi]
            if hi - lo <= K["PROBE_RATIO"] * n:
                if hi - lo == K["PROBE_RATIO"] * n:
                    _add(ev, "icw: slice of 4n searches the block")
                hits = [v[j] in set(blk) for j in range(lo, hi)]
            else:
                if hi - lo == K["PROBE_RATIO"] * n + 1:
                    _add(ev, "icw: slice of 4n + 1 is searched by the block")
                sl = set(v[lo:hi])
                hits = [y in sl for y in blk]
            _probe_rounds(ev, hits)
            for j in range(lo, hi):
                if v[j] in set(blk):
                    match(bi, j)
        batches.append(Batch(b, f, run, win0, wend, False))
        b += f + run
        nbatch += 1


Icw = namedtuple("Icw", "events result launches by_v batches writers")


def icw_plan(pk, after, v) -> Icw:
    """dgx_intersect_compressed: v ∩ pack[>= after], with the compaction's tiles."""
    ev = set()
    v = [int(x) for x in v]
    m = len(v)
    if pk is None or pk.nb == 0 or m == 0:
        return Icw(ev, np.zeros(0, np.uint64), 0, None, [], 0)
    by_v = m < pk.nb
    if by_v:
        _add(ev, "icw: ranges by v")
    else:
        _add(ev, "icw: ranges by block")
    _icw_input_events(ev, pk, v, after)
    vlo, vhi = (icw_ranges_by_v if by_v else icw_ranges_by_block)(pk, v, after)
    keep = [False] * m
    batches = []

    def match(_b, j):
        keep[j] = True

    for w in range(-(-pk.nb // D_BPW)):
        _icw_warp(ev, pk, vlo, vhi, v, w * D_BPW, match, batches)
    tiles = -(-m // CP_TILE)
    writers = sum(1 for t in range(tiles) if t * CP_TILE + CP_TILE >= m)
    if m % CP_TILE == 0:
        _add(ev, "compact: m a multiple of the tile")
    if m % CP_TILE == 1 and m > 1:
        _add(ev, "compact: m one past a tile")
    if tiles > 1:
        _add(ev, "compact: several tiles")
    return Icw(ev, np.array([x for x, k in zip(v, keep) if k], np.uint64), 3, by_v, batches, writers)


IcwRows = namedtuple("IcwRows", "events results launches grid_rows")


def icw_rows_plan(packs, after, v) -> IcwRows:
    """dgx_intersect_compressed_rows: every pack against the same v from the same after, one flat block space."""
    ev = set()
    v = [int(x) for x in v]
    m = len(v)
    jobs = [p for p in packs if p is not None and p.nb]
    if len(jobs) < len(packs):
        _add(ev, "rows: empty and NULL rows")
    nb = sum(p.nb for p in jobs)
    if nb == 0 or m == 0:
        return IcwRows(ev, [np.zeros(0, np.uint64) for _ in packs], 0, False)
    sides = {p.nb > m for p in jobs}
    if len(sides) == 2:
        _add(ev, "rows: packs on both sides of the range choice")
    grid_rows = len(packs) + 1 > 32 * nb
    if grid_rows:
        _add(ev, "rows: gather grid set by the row count")
    res = []
    for p in packs:
        if p is None or p.nb == 0:
            res.append(np.zeros(0, np.uint64))
            continue
        _icw_input_events(ev, p, v, after)
        vlo, vhi = (icw_ranges_by_v if p.nb > m else icw_ranges_by_block)(p, v, after)
        for b in range(p.nb):
            n = vhi[b] - vlo[b] if vhi[b] > vlo[b] else 0
            if n and n < p.num[b]:
                _add(ev, "rows: slot equals hi - lo")
            if n and p.num[b] < n:
                _add(ev, "rows: slot equals NumUids")
        got = {}

        def match(b, j, got=got):
            got.setdefault(b, []).append(v[j])

        for w in range(-(-p.nb // D_BPW)):
            _icw_warp(ev, p, vlo, vhi, v, w * D_BPW, match, [])
        res.append(np.array([x for b in sorted(got) for x in sorted(got[b])], np.uint64))
    return IcwRows(ev, res, 6, grid_rows)


# ---- the matrix -------------------------------------------------------------------------------------------------------

Matrix = namedtuple("Matrix", "events results launches units")


def matrix_plan(pk, rows) -> Matrix:
    """dgx_intersect_compressed_matrix: IntersectCompressedWith(pack, 0, row) for every row."""
    ev = set()
    rows = [[int(x) for x in r] for r in rows]
    v = [x for r in rows for x in r]
    m = len(v)
    if pk is None or pk.nb == 0 or m == 0:
        return Matrix(ev, [np.zeros(0, np.uint64) for _ in rows], 0, 0)
    units = []  # (block, lo, hi) of every unit, in the order icw_mx_locate_kernel finds them
    s = 0
    prev_last_blk = None
    for r in rows:
        e = s + len(r)
        for k in range(s, e):
            b = pk.block_of(v[k])
            if b >= 0 and (k == s or v[k - 1] < pk.base[b]):
                end = k + bisect_left(v[k:e], pk.base[b + 1]) if b + 1 < pk.nb else e
                units.append((b, k, end))
                if k == s and prev_last_blk == b:
                    _add(ev, "mx: row starts in the previous row's last block")
        if e > s:
            prev_last_blk = pk.block_of(v[e - 1])
        s = e
    units.sort(key=lambda u: u[0])  # block order; the order of one block's units is the atomics' and does not matter
    per = {}
    for b, lo, hi in units:
        per[b] = per.get(b, 0) + 1
        if hi - lo == MX_SERIAL:
            _add(ev, "mx: unit of MX_SERIAL elements")
        if hi - lo == MX_SERIAL + 1:
            _add(ev, "mx: unit of MX_SERIAL + 1 elements")
    pos = 0
    for b in sorted(per):
        if per[b] in (31, 32, 33, 65):
            _add(ev, f"mx: block with {per[b]} units")
        if pos // 32 != (pos + per[b] - 1) // 32:
            _add(ev, "mx: a block's units span two warps")
        pos += per[b]
    keep = [False] * m
    for p0 in range(0, len(units), 32):
        lanes = units[p0:p0 + 32]
        nin = len(lanes)
        f, prev_slow = 0, False
        while f < nin:
            win0 = pk.doff[lanes[f][0]] & ~15
            ok = [pk.num[u[0]] <= SLOW_NUM and pk.doff[u[0] + 1] - win0 <= D_WB for u in lanes[f:]]
            run = _lead(ok)
            if run == 0:
                bf = lanes[f][0]
                grp = [i for i in range(f, nin) if lanes[i][0] == bf]
                if pk.num[bf] > SLOW_NUM and f == 0:
                    _add(ev, "mx: slow block at lane 0")
                if pk.num[bf] <= SLOW_NUM:
                    _add(ev, "mx: slow path, block alone past the window")
                if f > 0:
                    _add(ev, "mx: slow group at f > 0")
                blk = set(pk.blocks[bf])
                for i in grp:
                    for j in range(lanes[i][1], lanes[i][2]):
                        keep[j] |= v[j] in blk
                f += len(grp)
                prev_slow = True
                continue
            if prev_slow:
                _add(ev, "mx: fast batch after a slow one in the same warp")
            rend = f + run
            if rend < nin and pk.num[lanes[rend][0]] <= SLOW_NUM:
                _add(ev, "mx: window round cut by the byte budget")
            _run_events(ev, "mx", f, run, nin if nin < 32 else 32)
            wend = pk.doff[lanes[rend - 1][0] + 1]
            _window_events(ev, "mx", pk, lanes[f][0], win0, wend,
                           pk.doff[lanes[rend][0] + 1] if rend < nin else None)
            seen = set()
            for i in range(f, rend):
                b, lo, hi = lanes[i]
                if b not in seen:
                    seen.add(b)
                    _expand_events(ev, "mx", pk, b)
                blk = set(pk.blocks[b])
                for j in range(lo, hi):
                    keep[j] |= v[j] in blk
            f = rend
    res, s = [], 0
    for r in rows:
        res.append(np.array([v[j] for j in range(s, s + len(r)) if keep[j]], np.uint64))
        s += len(r)
    return Matrix(ev, res, 6, len(units))


# ---- unfiltered List.Uids ---------------------------------------------------------------------------------------------

def luu_locate(pk, x):
    """luu_locate: (block, pack uids <= x, x is a pack uid)."""
    b = pk.block_of(x)
    if b < 0:
        return b, 0, False
    le = 0
    hit = False
    for y in pk.blocks[b]:
        if y > x:
            break
        le += 1
        if y == x:
            hit = True
            break
    return b, pk.uoff[b] + le, hit


Luu = namedtuple("Luu", "events results counts launches count_launches lens sblk")


def first_of(first):
    return MAX_FIRST if first == 0 else (1 if first < 0 else first)


def luu_plan(rows, after, first=0) -> Luu:
    """dgx_list_uids_unfiltered_rows / dgx_list_count_rows: rows = [(pack or None, mut uids, mut flags)]."""
    ev = set()
    most = first_of(first)
    res, counts, lens, sblks = [], [], [], []
    nonempty = []
    for pk, mu, mf in rows:
        mu, mf = [int(x) for x in mu], [int(x) for x in mf]
        cls, rank = [], []
        for x, fl in zip(mu, mf):
            c, rk = (0, 0), 0
            if x > after:
                hit = False
                if pk is not None and pk.nb:
                    b, le, hit = luu_locate(pk, x)
                    rk = le - (1 if hit else 0)
                    if b < 0:
                        _add(ev, "luu: entry below the first base")
                    elif hit and x == pk.base[b] and b > 0:
                        _add(ev, "luu: entry on the next block's base")
                    if x > pk.flat[-1]:
                        _add(ev, "luu: entry above the last uid")
                    if hit and fl and b + 1 < pk.nb and x == pk.blocks[b][-1] and pk.base[b + 1] == x + 1:
                        _add(ev, "luu: drop of a block's last uid, next base one more")
                if hit and fl:
                    c = (1, 0)
                if not hit and not fl:
                    c = (0, 1)
            cls.append(c)
            rank.append(rk)
        ex = [(0, 0)]
        for c in cls:
            ex.append((ex[-1][0] + c[0], ex[-1][1] + c[1]))
        skip = sb = 0
        total = 0
        if pk is not None and pk.nb:
            b, le, _ = luu_locate(pk, after)
            skip = le
            total = pk.uoff[pk.nb]
            if b < 0:
                _add(ev, "luu: after below the first base")
            else:
                sb = b if le - pk.uoff[b] < pk.num[b] else b + 1
                if after == pk.base[b] and b > 0:
                    _add(ev, "luu: after on a base")
                if after == pk.blocks[b][-1]:
                    if b + 1 == pk.nb:
                        _add(ev, "luu: after on the pack's last uid")
                    else:
                        _add(ev, "luu: after on a block's last uid")
                if sb % D_BPW == 0 and 0 < sb < pk.nb:
                    _add(ev, "luu: seek block on a warp boundary")
        n = total - skip - ex[-1][0] + ex[-1][1]
        ln = min(n, most)
        counts.append(n)
        lens.append(ln)
        sblks.append(sb)
        nonempty.append(ln > 0)
        out = [None] * ln

        def pos_of(y, q, js, je):
            j = js + bisect_left(mu[js:je], y)
            if j < je and mu[j] == y and cls[j][0]:
                return None
            return q - skip - ex[j][0] + ex[j][1]

        if pk is not None and pk.nb:
            for w in range(-(-pk.nb // D_BPW)):
                _luu_warp(ev, pk, w * D_BPW, skip, sb, ln, mu, ex, pos_of, out)
        for k, (x, c) in enumerate(zip(mu, cls)):
            if c[1]:
                p = rank[k] - skip - ex[k][0] + ex[k][1]
                if p < ln:
                    out[p] = x
                else:
                    _add(ev, "luu: insert past the cut")
        assert None not in out
        res.append(np.array(out, np.uint64))
        if 0 < ln < n:
            last = out[-1]
            if last in mu and cls[mu.index(last)][1]:
                _add(ev, "luu: cut on an insert")
            else:
                _add(ev, "luu: cut on a pack uid")
                q = pk.flat.index(last)
                if q > 0 and pk.flat[q - 1] in mu and cls[mu.index(pk.flat[q - 1])][0]:
                    _add(ev, "luu: cut right after a drop")
    if not all(nonempty) and any(nonempty):
        _add(ev, "luu: row of length 0 next to full rows")
    return Luu(ev, res, counts, 5, 3, lens, sblks)


def _luu_warp(ev, pk, b, skip, sb, ln, mu, ex, pos_of, out):
    bend = min(b + D_BPW, pk.nb)
    if b < sb:
        b = sb
        if b < bend and ln:
            _add(ev, "luu: warp starts at the seek block")
    if b >= bend or ln == 0:
        return
    nbatch, prev_slow = 0, False
    while b < bend:
        nl = min(32, bend - b)
        if nl < 32:
            _add(ev, "luu: partial last batch")
        lane = []
        for i in range(nl):
            bi = b + i
            js = bisect_left(mu, pk.base[bi])
            je = bisect_left(mu, pk.base[bi + 1]) if bi + 1 < pk.nb else len(mu)
            lower = pk.uoff[bi] - skip - ex[js][0] + ex[js][1] if bi > sb else 0
            lane.append((js, je, lower))
        live = [i for i in range(nl) if lane[i][2] < ln]
        if not live:
            _add(ev, "luu: blocks past the cut never loaded")
            if lane[0][2] == ln:
                _add(ev, "luu: cut on a block's first position")
            return
        last = live[-1]
        assert live == list(range(last + 1))
        if last + 1 < nl:
            _add(ev, "luu: blocks past the cut never loaded")
            if lane[last + 1][2] == ln:
                _add(ev, "luu: cut on a block's first position")
        if lane[last][2] == ln - 1 and last > 0:
            _add(ev, "luu: cut one past a block's first position")
        win0 = pk.doff[b] & ~15
        run = _lead([i <= last and pk.doff[b + i + 1] - win0 <= D_WB for i in range(nl)])
        _run_events(ev, "luu", 0, run, last + 1)
        n = run if run else 1
        slow = run == 0 or any(pk.num[b + i] > SLOW_NUM for i in range(run))
        if slow:
            _slow_events(ev, "luu", pk, b, range(n), run == 0, nbatch)
            prev_slow = True
        else:
            if prev_slow:
                _add(ev, "luu: fast batch after a slow one in the same warp")
            _window_events(ev, "luu", pk, b, win0, pk.doff[b + run],
                           pk.doff[b + run + 1] if run <= last else None)
        for i in range(n):
            bi = b + i
            js, je, _ = lane[i]
            if not slow:
                _expand_events(ev, "luu", pk, bi)
            for e, y in enumerate(pk.blocks[bi]):
                q = pk.uoff[bi] + e
                if q < skip:
                    continue
                p = pos_of(y, q, js, je)
                if p is not None and p < ln:
                    out[p] = y
                    if p == ln - 1 and e == pk.num[bi] - 1 and i == 31:
                        _add(ev, "luu: cut on the last value of lane 31's block")
                if p is not None and p >= ln and slow:
                    _add(ev, "luu: cut inside a slow-path walk")
                    break
        b += n
        nbatch += 1


# ---- the oracle side ----------------------------------------------------------------------------------------------------

class ArrayPack(pyoracle.Pack):
    """An oracle pack over arrays held here: the oracle's encoder cannot make a hand-built pack (deltas past 2^32,
    trailing bytes, blocks without delta bytes)."""

    def __init__(self, block_size, base, num, delta_off, deltas):
        self.arrays = (base, num, delta_off, deltas)
        self.s = pyoracle._Pack(block_size, base.size, base.ctypes.data_as(C.POINTER(C.c_uint64)),
                                num.ctypes.data_as(C.POINTER(C.c_uint32)),
                                delta_off.ctypes.data_as(C.POINTER(C.c_uint64)),
                                deltas.ctypes.data_as(C.POINTER(C.c_uint8)))
        super().__init__(C.pointer(self.s))

    def __del__(self):
        pass  # the arrays are numpy's


def oracle_pack(pk):
    """The model's pack as an oracle pack over the same arrays; None for a NULL pack."""
    if pk is None:
        return None
    bs, base, num, doff, deltas = pk.arrays()
    return ArrayPack(bs, base, num, doff, deltas if deltas.size else np.zeros(1, np.uint8))


# ---- fixtures -----------------------------------------------------------------------------------------------------------

Fixture = namedtuple("Fixture", "name kind args events")


def simulate(f):
    """The model's run of a fixture: decode (pack, seek, out_word), batch (packs), icw (pack, after, v), rows (packs,
    after, v), mx (pack, rows), luu (rows, after, first)."""
    return {"decode": decode_plan, "batch": decode_batch_plan, "icw": icw_plan, "rows": icw_rows_plan,
            "mx": matrix_plan, "luu": luu_plan}[f.kind](*f.args)


# Blocks of 256 uids laid out so that windows end exactly on D_WB and one byte past it, from win0 misaligned by 0
# (block 0, block 4) and by 15 (block 9, block 14).  A block of 256 uids with 4-byte deltas takes 1085 bytes.
WIN_SIZES = [1085, 1085, 1085, 841, 1085, 1085, 1085, 842, 1070, 1085, 1085, 1085, 826, 1071, 1085, 1085, 1085, 827,
             1085, 1085]


def window_pack():
    return seg_pack([(256, s) for s in WIN_SIZES])


def groups_pack():
    """Blocks of 1, 126, 129, 130, 255 and 256 uids (0, 32, 32, 33, 64 and 64 groups) at every delta width, and one
    block of two uids 0xFFFFFFFF apart."""
    return seg_pack([(1, None), (126, None, 2), (129, None, 3), (130, None, 4), (255, None, 1), (256, None, 2),
                     [0, 0xFFFFFFFF], (256, None, 3)])


def slow_pack():
    """129 blocks of 9 uids with blocks of 257 and 258 uids (the slow path) at lane 31 of warp 0's first batch, at
    lanes 0 and 1 of warp 1's first batch and at lane 0 of its second batch."""
    sp = [(9, None)] * 129
    for b, n in ((31, 257), (64, 258), (65, 257), (96, 257)):
        sp[b] = (n, None)
    return seg_pack(sp)


def cut31_pack():
    """28 blocks of 10 bytes and then blocks of 1085: the run of batch 0 is cut at lane 31; 72 blocks in all."""
    return seg_pack([(9, None)] * 28 + [(256, 1085)] * 4 + [(9, None)] * 40)


def hand_built():
    """Blocks the Encoder never writes: 40 blocks of one uid without delta bytes (a window of 0 bytes), one of 9 uids
    whose deltas are all 0xFFFFFFFF (a running sum past 2^32), one of 200 uids padded to 4200 bytes (alone past the
    window), one of 100 uids, one of 50 uids padded to 4050 bytes (cuts the run at lane 1) and seven blocks of 9."""
    blocks = [((k + 1) << 40, b"", 1) for k in range(40)]
    blocks.append((41 << 40, gv_encode([0xFFFFFFFF] * 8), 9))
    blocks.append((42 << 40, gv_encode([3] * 199).ljust(4200, b"\0"), 200))
    blocks.append((43 << 40, gv_encode([5] * 99), 100))
    blocks.append((44 << 40, gv_encode([7] * 49).ljust(4050, b"\0"), 50))
    blocks += [((45 + k) << 40, gv_encode([2] * 8), 9) for k in range(7)]
    return hand_pack(blocks)


def unit_pack(nblocks=8, per=256, step=16):
    """nblocks blocks of `per` uids `step` apart (BlockSize per): room for v elements between the uids."""
    import gen

    u = (1 << 34) + np.arange(nblocks * per, dtype=np.uint64) * np.uint64(step)
    enc = gen.encode_pack_np(u, per)
    return Pack(enc[1], enc[2], enc[3], enc[4], per)


def _misses(pk, b, k):
    """k values inside block b's range that are not pack uids (the uids are at least 2 apart)."""
    return [u + 1 for u in pk.blocks[b][:k]]


def _decode_fixtures():
    W, H, G, S, R = window_pack(), hand_built(), groups_pack(), slow_pack(), cut31_pack()
    last3 = W.blocks[3][-1]
    fx = [
        Fixture("decode window pack", "decode", (W, 0, 0), {
            "dec: seek 0", "dec: window of exactly D_WB bytes", "dec: next block one byte past the window",
            "dec: win0 aligned", "dec: expand 64 groups"}),
        Fixture("decode from block 9 (win0 + 15, exactly D_WB)", "decode", (W, W.base[9], 0), {
            "dec: seek on a block's base", "dec: win0 misaligned by 15", "dec: window of exactly D_WB bytes"}),
        Fixture("decode from block 14 (win0 + 15, one byte past)", "decode", (W, W.base[14], 0), {
            "dec: win0 misaligned by 15", "dec: next block one byte past the window"}),
        Fixture("decode from a block's last uid, even word", "decode", (W, last3, 0), {
            "dec: seek on a block's last uid", "dec: trimmed head, first word even",
            "dec: later block written from an odd word"}),
        Fixture("decode from a block's last uid, odd word", "decode", (W, last3, 1), {
            "dec: seek on a block's last uid", "dec: trimmed head, first word odd"}),
        Fixture("decode from inside a block, odd word", "decode", (W, W.blocks[5][2], 1), {
            "dec: trimmed head, first word odd", "dec: later block written from an odd word"}),
        Fixture("decode between two blocks", "decode", (W, last3 + 1, 0), {"dec: seek between two blocks"}),
        Fixture("decode below the first base", "decode", (W, 1, 0), {"dec: seek below the first base"}),
        Fixture("decode above the last uid", "decode", (W, W.flat[-1] + 1, 0), {"dec: seek above the last uid"}),
        Fixture("decode hand-built blocks", "decode", (H, 0, 0), {
            "dec: zero-byte window", "dec: all 32 lanes fit", "dec: slow path, block alone past the window",
            "dec: run cut at lane 1", "dec: running sum past 2^32", "dec: delta 0xFFFFFFFF", "dec: expand 0 groups",
            "dec: partial last batch", "dec: fast batch after a slow one in the same warp"}),
        Fixture("decode group counts and delta widths", "decode", (G, 0, 0), {
            "dec: expand 0 groups", "dec: expand 32 groups", "dec: expand 33 groups", "dec: expand 64 groups",
            "dec: delta 0xFFFFFFFF"}),
        Fixture("decode slow blocks", "decode", (S, 0, 0), {
            "dec: slow block at lane 0", "dec: slow block at lane 31",
            "dec: slow block at the first lane of a warp's second batch",
            "dec: fast batch after a slow one in the same warp", "dec: two slow blocks in one run"}),
        Fixture("decode run cut at lane 31", "decode", (R, 0, 0), {"dec: run cut at lane 31"}),
    ]
    packs = [run_pack(1, start=1 << 36), None, run_pack(63, start=2 << 36), run_pack(64, start=3 << 36),
             Pack([], [], [0], np.zeros(0, np.uint8)), run_pack(65, start=4 << 36), run_pack(129, start=5 << 36)]
    fx.append(Fixture("job table of 1, 63, 64, 65 and 129 blocks", "batch", (packs,), {
        "batch: empty pack left out of the table", "batch: warp starts a later job", "batch: second warp of a job",
        "batch: 65th block alone in its warp"}))
    fx.append(Fixture("job table of window, hand-built and slow packs", "batch", ([W, H, S, G],), {
        "batch: warp starts a later job", "dec: zero-byte window", "dec: slow block at lane 31"}))
    return fx


def _icw_fixtures():
    W, H, G, S = window_pack(), hand_built(), groups_pack(), slow_pack()
    U = unit_pack()
    T = run_pack(100)
    fx = []
    # blocks 9..12 (win0 + 15, exactly D_WB) and 14..17 (win0 + 15, one byte past), after splitting block 9's elements
    core = [W.blocks[9][1], W.blocks[9][3], W.blocks[9][5], W.blocks[10][0], W.blocks[11][-1], W.blocks[12][7] + 1,
            W.base[14], W.blocks[14][-1], W.blocks[15][9], W.blocks[16][-1], W.blocks[17][2]]
    extra = [1, W.flat[-1] + 5, W.base[2] - 1, W.base[2], W.blocks[5][4], W.blocks[6][-1], W.blocks[7][3] + 1,
             W.blocks[18][1], W.blocks[19][0], W.blocks[19][8], W.blocks[19][9]]
    for m, name in ((19, "m = nb - 1"), (20, "m = nb"), (21, "m = nb + 1")):
        v = sorted(core + extra[: m - len(core)])
        side = {"icw: ranges by v", "icw: after splits a block's v elements (by v)"} if m < 20 else {"icw: ranges by block"}
        fx.append(Fixture(f"icw window edges, {name}", "icw", (W, W.blocks[9][2], v), side | {
            f"icw: {name}", "icw: win0 misaligned by 15", "icw: window of exactly D_WB bytes",
            "icw: next block one byte past the window"}))
    every3 = sorted(set(W.flat[::3]) | {u + 1 for u in W.flat[1::7]} | {W.base[b] - 1 for b in range(1, 20)}
                    | {1, W.flat[-1] + 9})
    fx += [
        Fixture("icw after on a base", "icw", (W, W.base[6], every3), {
            "icw: after equal to a base", "icw: v holds a block's base", "icw: v holds a base - 1",
            "icw: v holds a block's last uid", "icw: v below the first base", "icw: v above the last uid",
            "icw: ranges by block", "icw: expand 64 groups"}),
        Fixture("icw after one below a base", "icw", (W, W.base[6] - 1, every3), {"icw: after one below a base"}),
        Fixture("icw after past the last uid", "icw", (W, W.flat[-1] + 1, every3), {"icw: after past the last uid"}),
        Fixture("icw touched blocks around an untouched one too large", "icw",
                (W, 0, [W.blocks[0][4], W.blocks[1][7], W.blocks[5][1]]), {
                    "icw: run cut by an untouched block, touched blocks past it",
                    "icw: window stops at the last touched block", "icw: ranges by v"}),
        Fixture("icw lane 31 only, then an untouched batch", "icw", (T, 0, [T.blocks[31][3], T.blocks[70][0]]), {
            "icw: touched block at lane 31 only", "icw: all lanes from f > 0 fit", "icw: batch touches nothing"}),
        Fixture("icw slices of 4n and 4n + 1", "icw", (U, 0, _slices(U)), {
            "icw: slice of 4n searches the block", "icw: slice of 4n + 1 is searched by the block"}),
        Fixture("icw hand-built blocks", "icw", (H, 0, sorted(set(H.flat[::2]) | {H.flat[-1] + 1})), {
            "icw: zero-byte window", "icw: slow path, block alone past the window", "icw: run cut at lane 1",
            "icw: running sum past 2^32", "icw: delta 0xFFFFFFFF", "icw: expand 0 groups",
            "icw: fast batch after a slow one in the same warp", "icw: all 32 lanes fit", "icw: partial last batch"}),
        Fixture("icw group counts", "icw", (G, 0, sorted(G.flat[::2])), {
            "icw: expand 0 groups", "icw: expand 32 groups", "icw: expand 33 groups", "icw: expand 64 groups",
            "icw: delta 0xFFFFFFFF"}),
        Fixture("icw slow blocks", "icw", (S, 0, sorted(S.flat[::2])), {
            "icw: slow block at lane 0", "icw: slow block at lane 31",
            "icw: slow block at the first lane of a warp's second batch",
            "icw: fast batch after a slow one in the same warp", "icw: two slow blocks in one run"}),
        Fixture("icw run cut at lane 31", "icw", (cut31_pack(), 0, sorted(cut31_pack().flat[::2])),
                {"icw: run cut at lane 31"}),
    ]
    pool = sorted(set(W.flat) | {u + 1 for u in W.flat})
    for m, ev in ((2047, set()), (2048, {"compact: m a multiple of the tile"}), (2049, {"compact: m one past a tile"}),
                  (4096, {"compact: m a multiple of the tile", "compact: several tiles"})):
        fx.append(Fixture(f"icw compaction, m = {m}", "icw", (W, 0, pool[:m]), ev))
    # the rows form
    m30 = sorted(set(W.flat[::200]) | set(T.flat[::40]))[:30]
    fx += [
        Fixture("rows on both sides of the range choice", "rows", ([W, None, T, G, Pack([], [], [0], np.zeros(0, np.uint8)), S],
                                                                   W.blocks[9][2], m30), {
            "rows: packs on both sides of the range choice", "rows: empty and NULL rows"}),
        Fixture("rows slots and ballot rounds", "rows", ([U, U], 0, _slices(U) + _rounds(U)), {
            "rows: slot equals NumUids", "rows: slot equals hi - lo",
            "rows: matches at lanes 31 and 0 of consecutive rounds"}),
        Fixture("rows window edges", "rows", ([W, T, W], W.blocks[9][2], sorted(core + extra)), {
            "icw: win0 misaligned by 15", "icw: window of exactly D_WB bytes",
            "icw: next block one byte past the window"}),
        Fixture("rows more rows than 32 blocks each", "rows", ([G] + [None] * 300, 0, sorted(G.flat[::3])), {
            "rows: gather grid set by the row count"}),
        Fixture("rows hand-built and slow packs", "rows", ([H, S, H], 0, sorted(set(H.flat[::2]) | set(S.flat[::3]))), {
            "icw: zero-byte window", "icw: slow block at lane 31", "icw: slow path, block alone past the window"}),
    ]
    return fx


def _slices(U):
    """Block 1's range holds 4n values (n = 256: the slice searches the block), block 3's 4n + 1 (the block searches
    the slice); block 5 holds fewer than n."""
    n = U.num[1]
    s1 = [U.base[1] + k for k in range(0, 4 * n)]
    s3 = [U.base[3] + k for k in range(0, 4 * n + 1)]
    s5 = [U.base[5] + 16 * k for k in range(0, 40)]
    return sorted(s1 + s3 + s5)


def _rounds(U):
    """Block 6's slice of 64 values, matches at probes 31 and 32 (lanes 31 and 0 of consecutive ballot rounds)."""
    b = U.base[6]
    return [b + 16 * k if k in (0, 31, 32, 63) else b + 16 * k + 3 for k in range(64)]


def _mx_fixtures():
    W, H, S = window_pack(), hand_built(), slow_pack()
    U = unit_pack(8, 256, 16)
    fx = []
    rows = [W.blocks[0][:8], [W.blocks[1][k] + 1 if k % 2 else W.blocks[1][k] for k in range(9)],
            [W.blocks[b][3] for b in range(1, 6)], [W.blocks[b][5] for b in range(9, 13)],
            [W.blocks[b][7] for b in range(14, 18)]]
    fx.append(Fixture("matrix units of 8 and 9, window rounds", "mx", (W, rows), {
        "mx: unit of MX_SERIAL elements", "mx: unit of MX_SERIAL + 1 elements", "mx: window round cut by the byte budget",
        "mx: win0 misaligned by 15", "mx: window of exactly D_WB bytes", "mx: next block one byte past the window",
        "mx: row starts in the previous row's last block", "mx: win0 aligned", "mx: expand 64 groups"}))
    rows = []
    for r in range(65):
        row = [U.blocks[0][r]]
        if r < 33:
            row.append(U.blocks[1][r] + 1)
        if r < 32:
            row.append(U.blocks[2][r])
        if r < 31:
            row.append(U.blocks[3][r] + (r % 2))
        rows.append(row)
    fx.append(Fixture("matrix blocks of 65, 33, 32 and 31 units", "mx", (U, rows), {
        "mx: block with 65 units", "mx: block with 33 units", "mx: block with 32 units", "mx: block with 31 units",
        "mx: a block's units span two warps", "mx: all 32 lanes fit"}))
    fx.append(Fixture("matrix slow blocks", "mx", (S, [[S.blocks[b][1] for b in range(0, 32)] + [S.blocks[64][2]],
                                                        [S.blocks[b][0] for b in range(65, 100)]]), {
        "mx: slow group at f > 0", "mx: slow block at lane 0", "mx: fast batch after a slow one in the same warp"}))
    fx.append(Fixture("matrix hand-built blocks", "mx", (H, [H.flat[::2], H.flat[1::3]]), {
        "mx: zero-byte window", "mx: slow path, block alone past the window", "mx: running sum past 2^32",
        "mx: delta 0xFFFFFFFF", "mx: expand 0 groups"}))
    fx.append(Fixture("matrix run cut at lane 1", "mx", (H, [[H.blocks[42][3], H.blocks[43][7]], [H.blocks[44][1]]]),
                      {"mx: run cut at lane 1"}))
    G = groups_pack()
    fx.append(Fixture("matrix group counts", "mx", (G, [G.flat[::2], G.flat[1::5]]), {
        "mx: expand 0 groups", "mx: expand 32 groups", "mx: expand 33 groups", "mx: expand 64 groups"}))
    R = cut31_pack()
    fx.append(Fixture("matrix run cut at lane 31", "mx", (R, [[R.blocks[b][0] for b in range(R.nb)]]),
                      {"mx: run cut at lane 31"}))
    return fx


def _luu_fixtures():
    W, H, G, S, R = window_pack(), hand_built(), groups_pack(), slow_pack(), cut31_pack()
    T = run_pack(100)
    C1 = run_pack(100, step=1)  # next base one more than the block's last uid
    none = (np.zeros(0, np.uint64), np.zeros(0, np.uint8))
    fx = []

    def row(pk, mu=(), mf=()):
        return (pk, np.array(mu, np.uint64), np.array(mf, np.uint8))

    fx += [
        Fixture("luu from block 9 (win0 + 15, exactly D_WB)", "luu", ([row(W)], W.base[9] - 1, 0), {
            "luu: win0 misaligned by 15", "luu: window of exactly D_WB bytes", "luu: warp starts at the seek block"}),
        Fixture("luu from block 14 (win0 + 15, one byte past)", "luu", ([row(W)], W.base[14] - 1, 0), {
            "luu: win0 misaligned by 15", "luu: next block one byte past the window"}),
        Fixture("luu after on a block's last uid", "luu", ([row(W), row(W)], W.blocks[3][-1], 0), {
            "luu: after on a block's last uid", "luu: win0 aligned", "luu: next block one byte past the window"}),
        Fixture("luu after on a base, below the first base", "luu", ([row(W), row(run_pack(100, start=1 << 40))],
                                                                      W.base[6], 0), {
            "luu: after on a base", "luu: after below the first base", "luu: all 32 lanes fit"}),
        Fixture("luu after on the pack's last uid, next to full rows", "luu",
                ([row(W, [W.flat[-1] + 3], [0]), row(T), row(None), row(W)], W.flat[-1], 0), {
                    "luu: after on the pack's last uid", "luu: row of length 0 next to full rows"}),
        Fixture("luu seek block on a warp boundary", "luu", ([row(S)], S.blocks[63][-1], 0), {
            "luu: seek block on a warp boundary", "luu: slow block at lane 0"}),
        Fixture("luu cut on a block's first position", "luu", ([row(T)], 0, 9 * 40), {
            "luu: cut on a block's first position", "luu: blocks past the cut never loaded", "luu: cut on a pack uid"}),
        Fixture("luu cut one past a block's first position", "luu", ([row(T)], 0, 9 * 40 + 1), {
            "luu: cut one past a block's first position"}),
        Fixture("luu cut on the last value of lane 31's block", "luu", ([row(T)], 0, 9 * 32), {
            "luu: cut on the last value of lane 31's block", "luu: cut on a block's first position"}),
        Fixture("luu entries at the block edges", "luu", ([row(C1, [5, C1.blocks[3][-1], C1.base[4], C1.base[7],
                                                                    C1.blocks[9][4] + 0, C1.flat[-1] + 7],
                                                              [0, 1, 1, 0, 1, 0])], 0, 0), {
            "luu: entry below the first base", "luu: entry on the next block's base", "luu: entry above the last uid",
            "luu: drop of a block's last uid, next base one more"}),
        Fixture("luu cut on an insert", "luu", ([row(T, [T.blocks[5][2] + 1], [0])], 0, 9 * 5 + 3 + 1), {
            "luu: cut on an insert"}),
        Fixture("luu cut right after a drop", "luu", ([row(T, [T.blocks[5][2]], [1])], 0, 9 * 5 + 3), {
            "luu: cut right after a drop", "luu: cut on a pack uid"}),
        Fixture("luu insert past the cut", "luu", ([row(T, [T.blocks[50][2] + 1], [0])], 0, 9 * 20), {
            "luu: insert past the cut"}),
        Fixture("luu slow path with the cut inside", "luu", ([row(S)], 0, 9 * 31 + 100), {
            "luu: cut inside a slow-path walk", "luu: slow block at lane 31"}),
        Fixture("luu slow blocks", "luu", ([row(S)], 0, 0), {
            "luu: slow block at lane 0", "luu: slow block at lane 31",
            "luu: slow block at the first lane of a warp's second batch",
            "luu: fast batch after a slow one in the same warp", "luu: two slow blocks in one run",
            "luu: partial last batch"}),
        Fixture("luu hand-built blocks", "luu", ([row(H, [H.base[3], H.blocks[40][4] + 1], [1, 0])], 0, 0), {
            "luu: zero-byte window", "luu: slow path, block alone past the window", "luu: run cut at lane 1",
            "luu: running sum past 2^32", "luu: delta 0xFFFFFFFF", "luu: expand 0 groups"}),
        Fixture("luu group counts", "luu", ([row(G)], 0, 0), {
            "luu: expand 0 groups", "luu: expand 32 groups", "luu: expand 33 groups", "luu: expand 64 groups"}),
        Fixture("luu run cut at lane 31", "luu", ([row(R)], 0, 0), {"luu: run cut at lane 31"}),
    ]
    del none
    return fx


def all_fixtures():
    return _decode_fixtures() + _icw_fixtures() + _mx_fixtures() + _luu_fixtures()
