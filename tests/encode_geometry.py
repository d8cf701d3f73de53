"""Host model of codec.Encode on the device (encode_kernel.cuh, and dgx_encode_bound, encode_impl, encode_to_host and
packed_op_host in dgx_api.cu), and fixtures aimed at its segment, block and capacity boundaries.

A call encodes n ascending uids in five launches:
  - enc_segments_kernel: one CTA per EN_TILE uids (the grid sized for the n argument, which for a packed op is only an
    upper bound on the count read from the device); each thread looks at EN_VT uids, loads the uid before its first
    one, and flags the indices where the upper 32 bits change; the tile that reaches n closes the list with n;
  - enc_segscan_kernel: one CTA turns segment lengths into first blocks, SEGSCAN segments a round, with a carry; when
    the segments do not fit seg_cap = min(n, nblocks_cap) + SEG_SPARE entries it reports a block count that suffices;
  - enc_sizes_kernel and enc_write_kernel: a warp per block, lane g on group g, 32 groups a round with a carry;
  - scan_u64_kernel: EN_TILE block byte lengths a tile.
encode_to_host then answers DGX_OK, or DGX_ERR_CAP with sizes for the next call.  The model restates all of it in
integer arithmetic from the uids, BlockSize and capacities; the pack itself comes from gen.encode_pack_np, and the
model's block plan and group widths must agree with it.  What the kernels decide is named as *events*; fixtures name
the events they must reach, and the model refuses a name that is not registered in EVENTS.

The constants, the gv_len thresholds, seg_cap, the bound's spare blocks and group size, the overflow report and the
packed caps are read from the CUDA sources as text, so a rewrite fails here loudly instead of leaving the fixtures
aimed at stale edges.

tests/test_encode_geometry.py checks the fixtures on the CPU; tests/test_gpu_encode_edges.py runs them through the
kernels.
"""
from __future__ import annotations

import os
import re
from collections import namedtuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")
U64 = (1 << 64) - 1
OK, ERR_CAP = 0, -4


def _src(fn):
    with open(os.path.join(CSRC, fn)) as f:
        return f.read()


def _one(pat, text, what):
    m = re.search(pat, text)
    if not m:
        raise ValueError(f"{what} changed: restate it in the encode model (tests/encode_geometry.py)")
    return m


def read_constants() -> dict:
    enc, api = _src("encode_kernel.cuh"), _src("dgx_api.cu")
    m = _one(r"constexpr int EN_NT = (\d+), EN_VT = (\d+), EN_TILE = EN_NT \* EN_VT;", enc, "EN_NT / EN_VT / EN_TILE")
    K = {"EN_NT": int(m.group(1)), "EN_VT": int(m.group(2))}
    widths = {int(_one(p, t, "the segscan CTA width").group(1)) for p, t in (
        (r"__launch_bounds__\((\d+)\) enc_segscan_kernel", enc),
        (r"start < nseg; start \+= (\d+)\)", enc),
        (r"block_exclusive_scan<(\d+)>\(\(u32\)nblk", enc),
        (r"enc_segscan_kernel<<<1, (\d+),", api))}
    if len(widths) != 1:
        raise ValueError(f"the segscan CTA width changed: {sorted(widths)}: restate it in the encode model")
    K["SEGSCAN"] = widths.pop()
    m = _one(r"return v < \(1u << (\d+)\) \? 1u : \(v < \(1u << (\d+)\) \? 2u : \(v < \(1u << (\d+)\) \? 3u : 4u\)\);",
             enc, "gv_len's thresholds `v < (1u << 8)`")
    K["GV"] = tuple(1 << int(g) for g in m.groups())
    _one(r"if \(e0 > 0 && e0 <= n\) \{ prev_hi = \(u32\)\(P\.u\[e0 - 1\] >> 32\); have_prev = true; \}", enc,
         "enc_segments_kernel's have_prev load")
    _one(r"unsigned char\* p = dst \+ carry \+ inc - bytes;", enc, "enc_write_kernel's group offset")
    _one(r"nb = n / P\.bsz \+ nseg;\s*P\.counts\[1\] = nb < n \? nb : n;", enc, "enc_segscan_kernel's overflow report")
    K["SEG_SPARE"] = int(_one(r"const size_t seg_cap = std::min<size_t>\(n, nblocks_cap\) \+ (\d+);", api,
                              "encode_impl's seg_cap").group(1))
    K["SPARE"] = int(_one(r"const size_t nb = n \? \(n \+ B - 1\) / B \+ (\d+) : 0;", api,
                          "dgx_encode_bound's spare blocks").group(1))
    g = {int(_one(p, api, "the 17-byte group bound").group(1)) for p in (
        r"\*delta_cap = (\d+) \* \(n / 4 \+ nb \+ 1\);",
        r"nb > E\.nblocks_cap \? (\d+) \* \(E\.n / 4 \+ nb \+ 1\) : l->h_word\[2\];",
        r"db_cap = std::max\(db_cap, (\d+) \* \(cap / 4 \+ nb_cap \+ 1\)\);")}
    if len(g) != 1:
        raise ValueError("the 17-byte group bound differs between its uses: restate it in the encode model")
    K["GROUP_MAX"] = g.pop()
    _one(r"nb_cap = std::max\(nb_cap, std::min\(\*nblocks, cap\)\);", api, "packed_op_host's block capacity")
    K["LAUNCHES"] = int(_one(r"enc_write_kernel<<<[^;]*;\s*CK\(cudaGetLastError\(\)\);\s*l->launches \+= (\d+);", api,
                             "encode_impl's launch count").group(1))
    return K


K = read_constants()
EN_VT, SEGSCAN, SEG_SPARE, SPARE, GROUP_MAX = K["EN_VT"], K["SEGSCAN"], K["SEG_SPARE"], K["SPARE"], K["GROUP_MAX"]
EN_TILE = K["EN_NT"] * EN_VT
LAUNCHES = K["LAUNCHES"]

# ---- events -----------------------------------------------------------------------------------------------------------

WIDTHS = (0, 0xFF, 0x100, 0xFFFF, 0x10000, 0xFFFFFF, 0x1000000, 0xFFFFFFFF)
EVENTS = {
    "seg: upper-word change at a tile's first index", "seg: upper-word change at a thread's first index",
    "seg: upper-word change at the last uid", "seg: n = 2048k - 1", "seg: n = 2048k", "seg: n = 2048k + 1",
    "seg: one tile", "seg: 16 or more tiles of look-back", "seg: tiles past the device count return",
    "seg: empty list closed by tile 0", "seg: starts past seg_cap dropped",
    "scan: nseg = 1024, one full round", "scan: nseg = 1025, a second round", "scan: nseg = 2049, three rounds",
    "scan: nseg + 1 = seg_cap", "scan: nseg + 1 = seg_cap + 1, overflow",
    "scan: overflow reports floor(n / bsz) + nseg", "scan: overflow report clamped to n",
    "scan: overflow where nseg is the block count", "scan: overflow where blocks exceed nseg",
    "scan: blocks over nblocks_cap", "scan: blocks = bound", "scan: blocks = bound + 1",
    "blk: segment of bsz * k uids", "blk: segment of bsz * k + 1 uids", "blk: segment of bsz * k - 1 uids",
    "blk: 1-uid block, one all-zero group", "blk: num 129, 32 groups", "blk: num 130, 33 groups",
    "blk: num 257, 64 groups", "blk: num 258, 65 groups", "blk: num mod 4 = 0", "blk: num mod 4 = 1",
    "blk: num mod 4 = 2", "blk: num mod 4 = 3", "write: one g0 round", "write: two g0 rounds, carry",
    "write: three g0 rounds", "blk: zero delta across a block edge", "blk: zero delta across a tile edge",
    "uid 0", "uid 2^64 - 1", "bsz 0 acts as 1", "bsz does not divide 2048", "bsz 2^31 - 1", "bsz 2^32 - 1",
    "bytes scan: 2048 blocks, one tile", "bytes scan: 2049 blocks, two tiles", "bytes scan: skipped",
    "host: OK", "host: CAP on blocks", "host: CAP on delta bytes only", "host: deltas sized from the block count",
    "calls: first call OK", "calls: OK after one retry",
    "caps: zero", "caps: blocks one short", "caps: delta bytes one short", "caps: exact",
    "packed: empty result, nil pack", "packed: 2048 uids in a capacity of several tiles",
    "packed: result segments overflow the bound",
} | {f"delta {w:#x} at j = {j}" for w in WIDTHS for j in range(4)}


def _add(ev, name):
    if name not in EVENTS:
        raise KeyError(f"event {name!r} is not registered in encode_geometry.EVENTS")
    ev.add(name)


# ---- the plan of one call ---------------------------------------------------------------------------------------------

def bound(n, bsz):
    """dgx_encode_bound: (nblocks_cap, delta_cap)."""
    B = bsz if bsz else 1
    nb = (n + B - 1) // B + SPARE if n else 0
    return nb, GROUP_MAX * (n // 4 + nb + 1)


def gv_len(d):
    """gv_len over an array of u32 deltas."""
    g1, g2, g3 = K["GV"]
    return 1 + (d >= g1).astype(np.int64) + (d >= g2) + (d >= g3)


def pack_of(u, bsz):
    import gen

    return gen.encode_pack_np(u, bsz)


Call = namedtuple("Call", "rc nblocks delta_bytes caps launches")


class Plan:
    """One call: the five kernels' plan over uids `u` with the kernel's n = len(u), the n argument `n_arg` (>= len(u);
    the workspace and the first grid are sized for it), BlockSize `bsz`, the workspace capacities `nb_cap` / `db_cap`
    and the caller's `cap_nb` / `cap_db` (the same for dgx_encode)."""

    def __init__(self, u, bsz, nb_cap, db_cap, n_arg=None, cap_nb=None, cap_db=None, ev=None):
        ev = set() if ev is None else ev
        u = np.ascontiguousarray(np.asarray(u, np.uint64))
        n = int(u.size)
        n_arg = n if n_arg is None else n_arg
        cap_nb = nb_cap if cap_nb is None else cap_nb
        cap_db = db_cap if cap_db is None else cap_db
        B = max(bsz, 1) & 0xFFFFFFFF
        self.n, self.bsz, self.nb_cap, self.db_cap = n, B, nb_cap, db_cap

        # enc_segments_kernel
        self.tiles_a = max(1, -(-n_arg // EN_TILE))
        live = max(1, -(-n // EN_TILE))
        self.closing_tile = live - 1
        if self.tiles_a > live:
            _add(ev, "seg: tiles past the device count return")
        if n == 0:
            _add(ev, "seg: empty list closed by tile 0")
        if self.tiles_a == 1:
            _add(ev, "seg: one tile")
        if live >= 16:
            _add(ev, "seg: 16 or more tiles of look-back")
        if n >= EN_TILE - 1:
            r = n % EN_TILE
            if r == EN_TILE - 1:
                _add(ev, "seg: n = 2048k - 1")
            elif r == 0:
                _add(ev, "seg: n = 2048k")
            elif r == 1:
                _add(ev, "seg: n = 2048k + 1")
        hi = u >> np.uint64(32)
        chg = np.ones(n, bool)
        chg[1:] = hi[1:] != hi[:-1]
        starts = np.nonzero(chg)[0]
        self.nseg = nseg = int(starts.size)
        inner = starts[starts > 0]
        if (inner % EN_TILE == 0).any():
            _add(ev, "seg: upper-word change at a tile's first index")
        if ((inner % EN_VT == 0) & (inner % EN_TILE != 0)).any():
            _add(ev, "seg: upper-word change at a thread's first index")
        if n > 1 and chg[-1]:
            _add(ev, "seg: upper-word change at the last uid")
        self.seg_cap = min(n_arg, nb_cap) + SEG_SPARE
        if nseg + 1 > self.seg_cap:
            _add(ev, "seg: starts past seg_cap dropped")
        seg_len = np.diff(np.append(starts, n))

        # enc_segscan_kernel
        self.blocks_per_seg = -(-seg_len // B)
        exact_nb = int(self.blocks_per_seg.sum())
        self.exact_nblocks = exact_nb
        self.overflow = nseg + 1 > self.seg_cap
        if nseg + 1 == self.seg_cap:
            _add(ev, "scan: nseg + 1 = seg_cap")
        if nseg == self.seg_cap:
            _add(ev, "scan: nseg + 1 = seg_cap + 1, overflow")
        if self.overflow:
            self.rounds = 0
            rep = n // B + nseg
            _add(ev, "scan: overflow reports floor(n / bsz) + nseg" if rep < n else "scan: overflow report clamped to n")
            _add(ev, "scan: overflow where nseg is the block count" if exact_nb == nseg
                 else "scan: overflow where blocks exceed nseg")
            counts1 = min(rep, n)
            assert counts1 >= exact_nb and counts1 > nb_cap, "the overflow report must suffice and exceed the capacity"
        else:
            self.rounds = -(-nseg // SEGSCAN)
            self.carries = [int(self.blocks_per_seg[:r * SEGSCAN].sum()) for r in range(self.rounds + 1)]
            if nseg == SEGSCAN:
                _add(ev, "scan: nseg = 1024, one full round")
            elif nseg == SEGSCAN + 1:
                _add(ev, "scan: nseg = 1025, a second round")
            elif nseg == 2 * SEGSCAN + 1:
                _add(ev, "scan: nseg = 2049, three rounds")
            counts1 = exact_nb
            if counts1 > nb_cap:
                _add(ev, "scan: blocks over nblocks_cap")
        bnb = bound(n, bsz)[0]
        if n and exact_nb == bnb:
            _add(ev, "scan: blocks = bound")
        if n and exact_nb == bnb + 1:
            _add(ev, "scan: blocks = bound + 1")

        # blocks (enc_sizes_kernel), groups (enc_write_kernel), block bytes (scan_u64_kernel)
        blk_seg = np.repeat(np.arange(nseg), self.blocks_per_seg)
        first = np.concatenate([[0], np.cumsum(self.blocks_per_seg)[:-1]]).astype(np.int64) if nseg else np.zeros(0, np.int64)
        k_in = np.arange(exact_nb) - first[blk_seg] if exact_nb else np.zeros(0, np.int64)
        self.blk_start = (starts[blk_seg] + k_in * B).astype(np.int64)
        seg_end = np.append(starts, n)[blk_seg + 1] if exact_nb else np.zeros(0, np.int64)
        self.num = np.minimum(seg_end - self.blk_start, B).astype(np.int64)
        self.ngroups = np.where(self.num > 1, (self.num + 2) // 4, 1)
        self._block_events(ev, u, seg_len, B, bsz)
        self.group_bytes = self._groups(ev, u)
        self.blk_bytes = np.add.reduceat(self.group_bytes, np.concatenate([[0], np.cumsum(self.ngroups)[:-1]])) \
            if exact_nb else np.zeros(0, np.int64)
        self.delta_off = np.concatenate([[0], np.cumsum(self.blk_bytes)]).astype(np.int64)
        ran = counts1 <= nb_cap
        if ran:
            self.tiles_b_live = max(1, -(-counts1 // EN_TILE))
            if counts1 == EN_TILE:
                _add(ev, "bytes scan: 2048 blocks, one tile")
            if counts1 == EN_TILE + 1:
                _add(ev, "bytes scan: 2049 blocks, two tiles")
            counts2 = int(self.delta_off[-1])
        else:
            _add(ev, "bytes scan: skipped")
            counts2 = 0
        self.counts = (nseg, counts1, counts2)
        self.written = ran and counts2 <= db_cap

        # encode_to_host
        nb = counts1
        db = GROUP_MAX * (n_arg // 4 + nb + 1) if nb > nb_cap else counts2
        if nb > nb_cap:
            _add(ev, "host: deltas sized from the block count")
            assert db >= int(self.delta_off[-1]), "the delta bytes returned with the block count must suffice"
        if nb > cap_nb or nb > nb_cap:
            rc = ERR_CAP
            _add(ev, "host: CAP on blocks")
        elif db > cap_db or db > db_cap:
            rc = ERR_CAP
            _add(ev, "host: CAP on delta bytes only")
        else:
            rc = OK
            _add(ev, "host: OK")
        self.rc, self.nb_out, self.db_out = rc, nb, db
        self.events = ev

    def _block_events(self, ev, u, seg_len, B, bsz):
        if bsz == 0:
            _add(ev, "bsz 0 acts as 1")
        if bsz == (1 << 31) - 1:
            _add(ev, "bsz 2^31 - 1")
        if bsz == (1 << 32) - 1:
            _add(ev, "bsz 2^32 - 1")
        if B > 1 and EN_TILE % B:
            _add(ev, "bsz does not divide 2048")
        if B > 1 and (seg_len >= B).any():
            r = seg_len % B
            big = seg_len >= B
            if (big & (r == 0)).any():
                _add(ev, "blk: segment of bsz * k uids")
            if (big & (r == 1)).any():
                _add(ev, "blk: segment of bsz * k + 1 uids")
            if ((seg_len >= B - 1) & (r == B - 1)).any() and B > 2:
                _add(ev, "blk: segment of bsz * k - 1 uids")
        num = self.num
        if (num == 1).any():
            _add(ev, "blk: 1-uid block, one all-zero group")
        for k, g in ((129, 32), (130, 33), (257, 64), (258, 65)):
            if (num == k).any():
                _add(ev, f"blk: num {k}, {g} groups")
        for r in range(4):
            if ((num > 1) & (num % 4 == r)).any():
                _add(ev, f"blk: num mod 4 = {r}")
        rounds = -(-self.ngroups // 32)
        for k, name in ((1, "write: one g0 round"), (2, "write: two g0 rounds, carry"), (3, "write: three g0 rounds")):
            if (rounds == k).any():
                _add(ev, name)
        n = u.size
        if n:
            if int(u[0]) == 0:
                _add(ev, "uid 0")
            if int(u[-1]) == U64:
                _add(ev, "uid 2^64 - 1")
            dup = np.zeros(n, bool)
            dup[1:] = u[1:] == u[:-1]
            bstart = np.zeros(n, bool)
            bstart[self.blk_start] = True
            if (dup & bstart).any():
                _add(ev, "blk: zero delta across a block edge")
            idx = np.arange(n)
            if (dup & ~bstart & (idx % EN_TILE == 0)).any():
                _add(ev, "blk: zero delta across a tile edge")

    def _groups(self, ev, u):
        """Byte length of every group, blocks in order: a tag and gv_len of each of the four deltas."""
        ng = int(self.ngroups.sum())
        D = np.zeros((ng, 4), np.uint64)
        real = np.zeros((ng, 4), bool)
        if ng:
            goff = np.concatenate([[0], np.cumsum(self.ngroups)[:-1]])
            blk = np.repeat(np.arange(self.num.size), self.num - 1)          # the delta positions of every block
            pos = np.arange(blk.size) - np.repeat(np.cumsum(self.num - 1) - (self.num - 1), self.num - 1) + 1
            i = self.blk_start[blk] + pos
            g, j = goff[blk] + (pos - 1) // 4, (pos - 1) % 4
            D[g, j] = (u[i] - u[i - 1]) & np.uint64(0xFFFFFFFF)
            real[g, j] = True
            assert ((u[i] >> np.uint64(32)) == (u[i - 1] >> np.uint64(32))).all(), "a block spans two upper words"
        for w in WIDTHS:
            for j in range(4):
                if (real[:, j] & (D[:, j] == w)).any():
                    _add(ev, f"delta {w:#x} at j = {j}")
        return (1 + gv_len(D).sum(axis=1)).astype(np.int64)

    def check_pack(self, pk):
        """The plan's blocks and bytes against the pack's arrays (gen.encode_pack_np's tuple)."""
        _, base, num, doff, deltas = pk
        assert self.exact_nblocks == base.size
        assert np.array_equal(self.num, num.astype(np.int64))
        assert np.array_equal(self.delta_off, doff.astype(np.int64))
        tags = deltas[doff[:-1].astype(np.int64)] if base.size else np.zeros(0, np.uint8)
        go = np.concatenate([[0], np.cumsum(self.ngroups)[:-1]]).astype(np.int64)
        assert np.array_equal(self.group_bytes[go], 5 + (tags & 3) + ((tags >> 2) & 3) + ((tags >> 4) & 3) + (tags >> 6))


def calls(u, bsz, caps, ev=None):
    """dgx_encode from the caller's capacities `caps` (nblocks, delta bytes), called again with the sizes it returns
    until DGX_OK; each Call's caps, outcome and launches.  Raises if a second retry would be needed."""
    ev = set() if ev is None else ev
    out = []
    n = len(u)
    while True:
        if n == 0:
            out.append(Call(OK, 0, 0, caps, 0))
            break
        p = Plan(u, bsz, caps[0], caps[1], ev=ev)
        out.append(Call(p.rc, p.nb_out, p.db_out, caps, LAUNCHES))
        if p.rc == OK:
            break
        if len(out) == 2:
            raise AssertionError(f"a second DGX_ERR_CAP after the sizes the first call returned: {out}")
        caps = (p.nb_out, p.db_out)
    _add(ev, "calls: first call OK" if len(out) == 1 else "calls: OK after one retry")
    return out


def resolve_caps(u, bsz, choice, ev=None):
    """The caller's capacities named by `choice`: "bound", "zero", "nb-1", "db-1" or "exact"."""
    ev = set() if ev is None else ev
    if choice == "bound":
        return bound(len(u), bsz)
    pk = pack_of(u, bsz)
    nb, db = pk[1].size, pk[4].size
    _add(ev, {"zero": "caps: zero", "nb-1": "caps: blocks one short", "db-1": "caps: delta bytes one short",
              "exact": "caps: exact"}[choice])
    return {"zero": (0, 0), "nb-1": (nb - 1, db), "db-1": (nb, db - 1), "exact": (nb, db)}[choice]


# ---- packed ops -------------------------------------------------------------------------------------------------------

PACKED_OPS = ("intersect", "difference", "merge", "intersect_sorted")


def packed_result(op, lists):
    """(result uids, the n argument packed_op_host encodes with) of one packed op over the operands' uids."""
    ls = [np.unique(np.asarray(l, np.uint64)) for l in lists]
    if op == "intersect":
        return np.intersect1d(ls[0], ls[1]), min(ls[0].size, ls[1].size)
    if op == "difference":
        return np.setdiff1d(ls[0], ls[1]), ls[0].size
    if op == "merge":
        return np.unique(np.concatenate(ls)), sum(l.size for l in ls)
    r = ls[0]
    for l in ls[1:]:
        r = np.intersect1d(r, l)
    return r, min(l.size for l in ls)


def packed_calls(op, lists, bsz, ev=None):
    """The packed op through the Python wrapper: the first call with dgx_encode_bound(n argument), then one retry with
    the returned sizes; packed_op_host's own workspace caps from each."""
    ev = set() if ev is None else ev
    ops = list(lists) if op in ("merge", "intersect_sorted") else list(lists[:2])
    res, cap = packed_result(op, ops)
    cnb, cdb = bound(cap, bsz)
    out = []
    while True:
        bnb, bdb = bound(cap, bsz)
        nb_cap = max(bnb, min(cnb, cap))
        db_cap = max(bdb, GROUP_MAX * (cap // 4 + nb_cap + 1))
        p = Plan(res, bsz, nb_cap, db_cap, n_arg=cap, cap_nb=cnb, cap_db=cdb, ev=ev)
        if p.overflow:
            _add(ev, "packed: result segments overflow the bound")
        out.append(Call(p.rc, p.nb_out, p.db_out, (cnb, cdb), None))
        if p.rc == OK:
            break
        if len(out) == 2:
            raise AssertionError(f"{op}: a second DGX_ERR_CAP after the sizes the first call returned: {out}")
        cnb, cdb = p.nb_out, p.db_out
    _add(ev, "calls: first call OK" if len(out) == 1 else "calls: OK after one retry")
    if res.size == 0:
        _add(ev, "packed: empty result, nil pack")
    if res.size == EN_TILE and cap >= 3 * EN_TILE:
        _add(ev, "packed: 2048 uids in a capacity of several tiles")
    return res, out


# ---- fixtures ---------------------------------------------------------------------------------------------------------

Fixture = namedtuple("Fixture", "name uids bsz caps events")
PackedFixture = namedtuple("PackedFixture", "name lists bsz events")


def simulate(f):
    """Every capacity choice of a fixture: {choice: [Call, ...]}, and the events reached."""
    ev = set()
    seqs = {c: calls(f.uids, f.bsz, resolve_caps(f.uids, f.bsz, c, ev), ev) for c in f.caps}
    if len(f.uids):
        Plan(f.uids, f.bsz, *bound(len(f.uids), f.bsz), ev=ev)
    return seqs, ev


def simulate_packed(f):
    ev = set()
    return {op: packed_calls(op, f.lists, f.bsz, ev) for op in PACKED_OPS}, ev


def words(his, los):
    """uids (hi << 32) | lo."""
    return (np.asarray(his, np.uint64) << np.uint64(32)) | np.asarray(los, np.uint64)


def runs(lengths, step=3, hi0=1):
    """Segments of the given lengths, each in its own upper word, uids `step` apart inside a segment."""
    his = np.repeat(np.arange(hi0, hi0 + len(lengths)), lengths)
    los = np.concatenate([np.arange(L) * step + 7 for L in lengths]) if len(lengths) else np.zeros(0)
    return words(his, los)


def changes_at(n, at, step=3):
    """n uids `step` apart whose upper word steps at every index in `at`."""
    hi = np.zeros(n, np.int64)
    for a in at:
        hi[a:] += 1
    return words(hi + 5, np.arange(n) * step + 11)


def tile_edges_list():
    """Upper-word changes at a tile's first index (2048), at a thread's first index (296) and at the last uid, and
    duplicates inside a block across the tile edge at 4096 and across the block edge at 4098 (BlockSize 5)."""
    n = 3 * EN_TILE + 1
    u = changes_at(n, [37 * EN_VT, EN_TILE, n - 1])
    u[4096] = u[4095]
    u[4098] = u[4097]
    return u


def tiles_list(n, rng, nchg=3):
    u = np.cumsum(rng.integers(1, 300, n, dtype=np.uint64)) + np.uint64(1 << 33)
    for a in sorted(rng.choice(np.arange(1, n), nchg, replace=False)):
        u[a:] += np.uint64(1 << 32)
    return u


def three_call_list():
    """800 uids alone in their upper word, then 200 in one upper word: with BlockSize 2 the bound gives 564 blocks, the
    segments overflow it, and the exact count (900) exceeds the segment count (801)."""
    return np.concatenate([words(np.arange(1, 801), np.full(800, 9)), words(np.full(200, 900), np.arange(200) * 2)])


def seg_cap_list(extra):
    """75 + extra single-uid segments, then one segment of 2560 - extra uids: n = 2635, BlockSize 256, the bound 75
    blocks, seg_cap 77; extra 0 fills seg_cap exactly (nseg + 1 = 77), extra 1 overflows it by one."""
    return runs([1] * (75 + extra) + [2560 - extra])


def spare_list(singles):
    """One segment of 3 * 256 + 1 uids and `singles` one-uid segments, BlockSize 256: 64 singles make the block count
    the bound's, 65 one more."""
    return runs([3 * 256 + 1] + [1] * singles)


def deltas_list():
    """BlockSize 5 blocks, each in its own upper word, one of WIDTHS at one position of its group (the others 1, or 0
    beside 0xFFFFFFFF so that the block stays in its upper word)."""
    out, hi = [], 100
    for w in WIDTHS:
        for j in range(4):
            d = [0 if w == 0xFFFFFFFF else 1] * 4
            d[j] = w
            lo = np.concatenate([[0], np.cumsum(d)])
            out.append(words(np.full(5, hi), lo))
            hi += 1
    # the widths below 2^32 - 1 in turn inside one block of 141 uids as well: each lands at every position
    d = np.tile(np.array([w for w in WIDTHS if w != 0xFFFFFFFF], np.uint64), 20)
    out.append(words(np.full(d.size + 1, hi), np.concatenate([[0], np.cumsum(d)])))
    return np.concatenate(out)


def extremes_list():
    return np.array([0, 0, 0, 5, 1 << 32, (1 << 32) + 1, U64 - 3, U64 - 1, U64, U64], np.uint64)


def random_list(rng, n):
    u = np.cumsum(rng.integers(0, 5000, n, dtype=np.uint64)) + np.uint64(rng.integers(0, 1 << 40))
    for a in rng.choice(np.arange(1, n), 4, replace=False):
        u[a:] += np.uint64(int(rng.integers(1, 3)) << 32)
    return u


def all_fixtures():
    rng = np.random.default_rng(4100)
    F = []

    def add(name, u, bsz, events, caps=("bound",)):
        F.append(Fixture(name, np.ascontiguousarray(np.asarray(u, np.uint64)), bsz, caps, set(events)))

    te = tile_edges_list()
    add("tile edges, bs 5", te, 5, {
        "seg: upper-word change at a tile's first index", "seg: upper-word change at a thread's first index",
        "seg: upper-word change at the last uid", "seg: n = 2048k + 1", "blk: zero delta across a block edge",
        "blk: zero delta across a tile edge", "bsz does not divide 2048", "calls: first call OK", "host: OK"})
    add("tile edges, capacities", te, 10, {"caps: zero", "caps: blocks one short", "caps: delta bytes one short",
                                           "caps: exact", "host: CAP on blocks", "host: CAP on delta bytes only",
                                           "calls: OK after one retry", "host: deltas sized from the block count"},
        caps=("zero", "nb-1", "db-1", "exact"))
    for k, r in ((1, -1), (2, 0), (2, 1), (3, -1), (1, 0)):
        n = EN_TILE * k + r
        ev = {{-1: "seg: n = 2048k - 1", 0: "seg: n = 2048k", 1: "seg: n = 2048k + 1"}[r]}
        for bsz in (10, 1000, 256):
            add(f"n = {n}, bs {bsz}", tiles_list(n, rng, 2), bsz, ev)
    add("many tiles, bs 1000", tiles_list(40 * EN_TILE + 3, rng, 5), 1000, {"seg: 16 or more tiles of look-back"})
    add("nseg 1024, bs 2", runs([4] * 1024), 2, {"scan: nseg = 1024, one full round",
                                                 "bytes scan: 2048 blocks, one tile"})
    add("nseg 1025, bs 3", runs([3] * 1024 + [1]), 3, {"scan: nseg = 1025, a second round"})
    add("nseg 2049, bs 1", runs([1] * 2049), 1, {"scan: nseg = 2049, three rounds",
                                                                       "bytes scan: 2049 blocks, two tiles"})
    add("nseg + 1 = seg_cap", seg_cap_list(0), 256, {"scan: nseg + 1 = seg_cap", "scan: blocks over nblocks_cap",
                                                     "bytes scan: skipped", "calls: OK after one retry"})
    add("nseg = seg_cap", seg_cap_list(1), 256, {
        "scan: nseg + 1 = seg_cap + 1, overflow", "seg: starts past seg_cap dropped",
        "scan: overflow reports floor(n / bsz) + nseg", "scan: overflow where blocks exceed nseg"})
    add("three calls before the fix", three_call_list(), 2, {
        "scan: overflow report clamped to n", "scan: overflow where blocks exceed nseg", "calls: OK after one retry"})
    add("every uid its own segment", np.sort(rng.choice(np.arange(1, 1 << 20, dtype=np.uint64), 5000,
                                                        replace=False)) << np.uint64(32), 256,
        {"scan: overflow where nseg is the block count", "scan: overflow report clamped to n"})
    add("segments of bsz k - 1, k, k + 1", runs([30, 31, 29, 10, 11, 9, 1]), 10, {
        "blk: segment of bsz * k uids", "blk: segment of bsz * k + 1 uids", "blk: segment of bsz * k - 1 uids",
        "blk: 1-uid block, one all-zero group"})
    add("num 129 to 260", runs([129, 130, 131, 132, 257, 258, 259, 260]), 1000, {
        "blk: num 129, 32 groups", "blk: num 130, 33 groups", "blk: num 257, 64 groups", "blk: num 258, 65 groups",
        "blk: num mod 4 = 0", "blk: num mod 4 = 1", "blk: num mod 4 = 2", "blk: num mod 4 = 3",
        "write: one g0 round", "write: two g0 rounds, carry", "write: three g0 rounds"})
    add("65 segments: blocks = bound", spare_list(64), 256, {"scan: blocks = bound", "calls: first call OK"})
    add("66 segments: blocks = bound + 1", spare_list(65), 256, {"scan: blocks = bound + 1",
                                                                 "scan: blocks over nblocks_cap",
                                                                 "calls: OK after one retry"})
    add("delta widths, bs 5", deltas_list(), 5, {f"delta {w:#x} at j = {j}" for w in WIDTHS for j in range(4)})
    add("uid 0 and 2^64 - 1, bs 2", extremes_list(), 2, {"uid 0", "uid 2^64 - 1", "blk: zero delta across a block edge"})
    add("uid 0 and 2^64 - 1, bs 0", extremes_list(), 0, {"uid 0", "uid 2^64 - 1", "bsz 0 acts as 1"})
    base = random_list(rng, 5000)
    for bsz, ev in ((0, {"bsz 0 acts as 1"}), (1, set()), (256, set()), ((1 << 31) - 1, {"bsz 2^31 - 1"}),
                    ((1 << 32) - 1, {"bsz 2^32 - 1"})):
        add(f"random 5000, bs {bsz}", base, bsz, ev)
    return F


def all_packed_fixtures():
    rng = np.random.default_rng(4101)
    x = np.sort(rng.choice(np.arange(1, 1 << 24, dtype=np.uint64), EN_TILE, replace=False))
    a = np.arange(1, 3000, 2, dtype=np.uint64)
    return [
        PackedFixture("disjoint operands", [a, a + np.uint64(1)], 5, {"packed: empty result, nil pack"}),
        PackedFixture("four copies of 2048 uids", [x, x, x, x], 10,
                      {"packed: 2048 uids in a capacity of several tiles", "packed: empty result, nil pack"}),
        PackedFixture("segments overflow the bound", [three_call_list(), three_call_list()], 2,
                      {"packed: result segments overflow the bound", "scan: overflow where blocks exceed nseg",
                       "calls: OK after one retry"}),
    ]
