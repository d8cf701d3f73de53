"""Host model of the value-column tests -- match() (match_kernel.cuh), the regexp() value test (regex_kernel.cuh) and
the compare functions (compare_kernel.cuh) -- as dgx_api.cu's fz_run, rx_run, cmp_uids_run and cmp_rows_run launch
them, with fixtures aimed at every grid, tile, chunk and alignment boundary.

The three ops share one front end and one string reader, so one model restates them:
  - the front end: fz_lookup_kernel's thread space max(ccap, n + 1, nvals + 1) (the index path's ccap is 0), each
    refusal with the thread and CTA that detects it, the count word's low 32 bits and nc, the value counts and `vlo`,
    the pair-offset scan by EN_TILE tiles, each pair's owner by the kernels' lower_bound over pair_off[0 .. nc], and
    compact_kernel by CP_TILE tiles;
  - the string reader: rx_span / rx_load, recording the column bytes every load reads.  A load reads a whole aligned
    16-byte segment only when the segment lies inside [bytes, bytes + nbytes); otherwise it reads the segment's bytes
    inside the column one at a time.  Results cannot show a whole-segment read past the column (every byte outside the
    value is masked), so the model keeps the read set and tests/test_value_column_geometry.py holds it inside the
    column over every alignment;
  - match(): the tier from W alone, the long-tier queue and the warp and pass of the fixed 2 * SMs grid that takes
    each queued pair, the warp's rune count round by round (32-byte ballots of fz_starts), the shortcuts, and of the
    blocked-Myers wavefront the lane holding the score ((W - 1) & 31) and whether the horizontal carry wraps from lane
    31 to lane 0 (W > 32).  Distances come from match_oracle.levenshtein;
  - regexp(): the shared-memory decision and layout (the table, the class map at round16(2 nt), term at +256) as a
    byte image the kernel's reads are taken from, the warp-tier queue, the thread tier's walk with its stop at an
    absorbing state, and rx_long_kernel's chunks (g0, nseg, per, each lane's [s0, s1), the state vectors, their
    convergence, the all-absorbed break and lane 0's composition) over the library's own tables
    (algo.RegexProg(...).tables());
  - compare: cmp_pairs_kernel's fixed grid with a bad value refusing from any stride, cmp_finish_kernel's counts for
    t < nc only, eq's argument set as cmp_args builds it, the device's binary search, cmp_bytes over segments with the
    argument's bytes read only below its length, and the index path (cmp_rows_kernel's slot space and row owner,
    CMP_NO_ARG, bad values skipped, cmp_place_kernel's pos[min(v_off[t], v_cap)]).
Answers are held to the existing restatements (match_oracle.c, regex_oracle.py, compare_oracle.c); the model adds the
geometry, not a fourth semantics.

What the kernels decide is named as *events*; fixtures name the events they must reach and the model refuses a name
not registered in EVENTS.  Fixed-grid events take the SM count, and fixtures(sms) builds the stride fixtures for it.
Named *mutants* (MUTANTS) are one-line slips the model can apply; a fixture names the mutants it kills.  Slips that
are invisible by design are not mutants, and tests assert the invisibility instead:
  - the warp tier at `len >= 4096` rather than `len > 4096`: both tiers compute the same answer;
  - the class map placed at 2 nt rather than round16(2 nt) by writer and reader alike: the reads follow the writes.
    The visible slip, a reader that does not round, is a mutant;
  - cmp_place_kernel's `min(v_off[t], v_cap)`: a call that reaches it unrefused has v_off ascending up to
    v_off[nrows] <= v_cap, so the min never decides; it guards the reads of a refused call's offsets only, and the
    model checks every index it forms is at most v_cap;
  - `smem <= 48 * 1024` in rx_run: with 2 nt <= RX_SMEM_TABLE and nstates <= 4096 it always holds.
A warp tier at `nstates <= 65` writes state 64's row past its warp's maps[] rows; the model raises on that write
rather than restating the shared-memory overlap.

Edges no fixture reaches, with reasons:
  - 32-bit counts (candidates, uids, values, bytes at 2^32): both forms refuse them at the call;
  - which warp or thread pulls which queued item, and the order of the long-tier queue: the scheduler and the
    queue's atomics choose them.  The model takes the queue in pair order, and the stride fixtures give neighbouring
    items different answers, so a warp that took the wrong item, or only its first, changes the output whatever the
    order;
  - the trigram branch's candidates: its plan and launches are the trigram query's, which its own edge tests cover;
  - the blocked-Myers wavefront step by step: the fixtures aim at the score's owner lane and the lane 31 -> lane 0
    carry, and the distance itself is match_oracle's.

The constants and the statements the model restates are read from the CUDA sources as text, so a rewrite fails here
loudly ("restate it in the value-column model") instead of leaving the fixtures aimed at stale edges.
tests/test_value_column_geometry.py checks the fixtures on the CPU; tests/test_gpu_value_column_edges.py runs them
through the kernels.
"""
from __future__ import annotations

import bisect
import functools
import math
import os
import re
import struct
from collections import namedtuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")
H100_SMS = 132
U64 = (1 << 64) - 1


def _src(fn):
    with open(os.path.join(CSRC, fn)) as f:
        return f.read()


def _one(pat, text, what):
    m = re.search(pat, text)
    if not m:
        raise ValueError(f"{what} changed: restate it in the value-column model (tests/value_column_geometry.py)")
    return m


def _fn(name, text):
    """The body of the function or kernel `name` (a definition starting a line, through its closing brace)."""
    head = r"(?ms)^(?:static |__global__ |__device__ |extern \"C\" |template <[^\n]*>\n__global__ )[^\n]*\b"
    return _one(head + name + r"\(.*?\n\}\n", text, name).group(0)


MK, RK, CK, CPK, ENK, API = ("match_kernel.cuh", "regex_kernel.cuh", "compare_kernel.cuh", "compressed_kernel.cuh",
                             "encode_kernel.cuh", "dgx_api.cu")
OWNER = r"const u64 c = lower_bound_g\(\w+\.pair_off, nc \+ 1, p \+ 1\) - 1;"
# (file, function or None for the whole file, statement as a regex, what it restates)
STATEMENTS = [
    (MK, None, r"constexpr int FZ_LONG_NT = 256;", "FZ_LONG_NT"),
    (RK, None, r"constexpr int RX_NT = 256;", "RX_NT"),
    (RK, None, r"constexpr int RX_WARP_STATES = 64;", "RX_WARP_STATES"),
    (RK, None, r"constexpr u64 RX_LONG_BYTES = 4096;", "RX_LONG_BYTES"),
    (RK, None, r"constexpr u32 RX_SMEM_TABLE = 32768;", "RX_SMEM_TABLE"),
    (RK, None, r"constexpr u32 RX_ABSORB = 2, RX_ACCEPT = 4;", "the term bits"),
    (RK, None, r"constexpr u32 RX_START = 2;", "RX_START"),
    (CK, None, r"constexpr u32 CMP_NT = 256;", "CMP_NT"),
    (CK, None, r"constexpr u32 CMP_NO_ARG = 0xFFFFFFFFu;", "CMP_NO_ARG"),
    (CPK, None, r"constexpr int CP_NT = 256, CP_VT = 8, CP_TILE = CP_NT \* CP_VT;", "CP_TILE"),
    (ENK, None, r"constexpr int EN_NT = 256, EN_VT = 8, EN_TILE = EN_NT \* EN_VT;", "EN_TILE"),
    # grids and launches
    (API, "fz_run", r"fz_lookup_kernel<<<gb_grid\(std::max<uint64_t>\(\{ccap, col\.n \+ 1, col\.nvals \+ 1\}\)\), 256",
     "match()'s lookup grid"),
    (API, "fz_run", r"fz_long_kernel<<<\(unsigned\)\(2 \* g_num_sms\), FZ_LONG_NT, 0, l->stream>>>\(P\);",
     "the long tier's grid"),
    (API, "fz_run", r"count_launches\(l, 5\);", "match()'s launches"),
    (API, "rx_run", r"fz_lookup_kernel<<<gb_grid\(std::max<uint64_t>\(\{ccap, col\.n \+ 1, col\.nvals \+ 1\}\)\), 256",
     "regexp()'s lookup grid"),
    (API, "rx_run", r"const unsigned tgrid = \(unsigned\)std::min<uint64_t>\(gb_grid\(col\.nvals\), 8ull \* g_num_sms\);",
     "rx_test_kernel's grid"),
    (API, "rx_run", r"rx_long_kernel<<<\(unsigned\)\(2 \* g_num_sms\), RX_NT, 0, l->stream>>>\(P\);",
     "the warp tier's grid"),
    (API, "rx_run", r"P\.warp = R\.nstates <= \(uint32_t\)RX_WARP_STATES;", "the warp tier's state bound"),
    (API, "rx_run", r"const size_t smem = \(\(size_t\)R\.nstates \* R\.nclasses \* 2 \+ 15\) / 16 \* 16 \+ 256 \+ "
     r"R\.nstates;", "the shared-memory size"),
    (API, "rx_run", r"if \(R\.trans\.size\(\) \* 2 <= RX_SMEM_TABLE && smem <= 48 \* 1024\)\s*"
     r"rx_test_kernel<true>", "the SMEM condition"),
    (API, "rx_run", r"count_launches\(l, 5\);", "regexp()'s launches"),
    (API, "cmp_uids_run", r"const unsigned tgrid = \(unsigned\)std::min<uint64_t>\(gb_grid\(S\.nvals\), "
     r"8ull \* g_num_sms\);", "cmp_pairs_kernel's grid"),
    (API, "cmp_uids_run", r"fz_lookup_kernel<<<gb_grid\(std::max<uint64_t>\(\{ccap, S\.n \+ 1, S\.nvals \+ 1\}\)\), 256",
     "the value path's lookup grid"),
    (API, "cmp_uids_run", r"count_launches\(l, 5\);", "the value path's launches"),
    (API, "cmp_rows_run", r"fz_lookup_kernel<<<gb_grid\(std::max<uint64_t>\(S\.n \+ 1, S\.nvals \+ 1\)\), 256",
     "the index path's lookup grid"),
    (API, "cmp_rows_run", r"const uint64_t nt = std::max<uint64_t>\(v_cap, nrows \+ 1\);", "the index path's slots"),
    (API, "cmp_rows_run", r"count_launches\(l, 4\);", "the index path's launches"),
    (API, "cmp_uids_run", r"cmp_args\(op, col->type, args, op == DGX_SGF_CMP_EQ, &A\)|count_launches", "eq's set"),
    # the front end
    (MK, "fz_lookup_kernel", r"const u64 raw = P\.cand_len \? \*P\.cand_len & 0xFFFFFFFFull : P\.ccap;\s*"
     r"const u64 nc = raw <= P\.ccap \? raw : 0;", "the count word"),
    (MK, "fz_lookup_kernel", r"if \(t < nc\) \{\s*const u64 x = P\.cand\[t\];\s*"
     r"if \(t > 0 && P\.cand\[t - 1\] >= x\) fz_refuse\(P\);", "the candidate order check"),
    (MK, "fz_lookup_kernel", r"if \(P\.byte_off && t < P\.nvals && P\.byte_off\[t\] > P\.byte_off\[t \+ 1\]\) "
     r"fz_refuse\(P\);", "the byte offset check"),
    (MK, "fz_test_kernel", OWNER, "the owner search (match)"),
    (RK, "rx_test_kernel", OWNER, "the owner search (regexp)"),
    (CK, "cmp_pairs_kernel", OWNER, "the owner search (compare)"),
    # match()
    (MK, "fz_test_kernel", r"if \(P\.W > 1\) \{", "the long tier's test"),
    (MK, "fz_starts", r"for \(u32 k = 1; k <= 3 && k <= i; \+\+k\) \{\s*if \(\(s\[i - k\] & 0xC0\) == 0x80\) continue;"
     r"\s*u32 r;\s*return fz_decode\(s, len, i - k, &r\) <= k;", "fz_starts"),
    (MK, "fz_long_kernel", r"for \(u64 q = \(u64\)blockIdx\.x \* \(FZ_LONG_NT / 32\) \+ \(threadIdx\.x >> 5\); q < nq; "
     r"q \+= nwarps\)", "the long tier's queue loop"),
    (MK, "fz_long_kernel", r"for \(u64 b = 0; b < len; b \+= 32\) \{", "the rune count's rounds"),
    (MK, "fz_long_kernel", r"const u32 owner = \(W - 1\) & 31;", "the score's owner"),
    # regexp()
    (RK, "rx_span", r"return RxSpan\{\(const uint4\*\)base, off \+ b0, off \+ b0 \+ len, off, off \+ nbytes\};",
     "rx_span"),
    (RK, "rx_load", r"if \(g \* 16 >= sp\.clo && g \* 16 \+ 16 <= sp\.chi\) return __ldg\(sp\.seg \+ g\);",
     "rx_load's whole-segment test"),
    (RK, "rx_load", r"if \(g \* 16 \+ k >= sp\.clo && g \* 16 \+ k < sp\.chi\)", "rx_load's byte test"),
    (RK, "rx_test_kernel", r"unsigned char\* c = rx_smem \+ \(\(nt \* 2 \+ 15\) & ~15u\);", "the class map's offset"),
    (RK, "rx_test_kernel", r"c\[256 \+ i\] = P\.term\[i\];", "term's offset"),
    (RK, "rx_test_kernel", r"tab = RxTab\{c, t, c \+ 256, P\.nclasses\};", "the shared table's reads"),
    (RK, "rx_test_kernel", r"if \(P\.warp && len > RX_LONG_BYTES\) \{", "the warp tier's queue test"),
    (RK, "rx_test_kernel", r"for \(u64 q = sp\.lo & ~15ull; q < sp\.hi && !\(tab\.term\[s\] & RX_ABSORB\); q \+= 16\)",
     "the thread tier's walk"),
    (RK, "rx_long_kernel", r"const u64 g0 = sp\.lo / 16, nseg = \(sp\.hi \+ 15\) / 16 - g0, per = \(nseg \+ 31\) / 32;"
     r"\s*const u64 s0 = g0 \+ \(u64\)lane \* per, s1 = min\(s0 \+ per, g0 \+ nseg\);", "the warp's chunks"),
    (RK, "rx_long_kernel", r"if \(single\) \{\s*if \(tab\.term\[v\] & RX_ABSORB\) break;", "the single walk's stop"),
    (RK, "rx_long_kernel", r"if \(conv && live != 0xFFFFu\) \{ single = true; v = live; \}\s*else if \(conv\) break;",
     "the convergence"),
    (RK, "rx_long_kernel", r"u32 st = v;\s*for \(int l = 1; l < 32 && !\(tab\.term\[st\] & RX_ABSORB\); \+\+l\) "
     r"st = maps\[wid\]\[st\]\[l\];", "lane 0's composition"),
    # compare
    (CK, "cmp_bytes", r"if \(q \+ k < sp\.lo \|\| q \+ k >= sp\.hi \|\| i >= alen\) continue;", "cmp_bytes' bounds"),
    (CK, "cmp_test", r"if \(cmp_order\(P, x, mid\) > 0\) lo = mid \+ 1; else hi = mid;", "eq's search"),
    (CK, "cmp_pairs_kernel", r"if \(cmp_bad\(P, j\)\) \{ fz_refuse\(F\); return; \}", "the value path's refusal"),
    (CK, "cmp_finish_kernel", r"if \(P\.counts && t < F\.words\[FZ_W_N\]\) P\.counts\[t\] = P\.hits\[t\];",
     "the count guard"),
    (CK, "cmp_rows_kernel", r"const u64 r = lower_bound_g\(P\.v_off, P\.nrows \+ 1, t \+ 1\) - 1;", "the row owner"),
    (CK, "cmp_rows_kernel", r"if \(k == CMP_NO_ARG\) \{\s*keep = 1;", "CMP_NO_ARG"),
    (CK, "cmp_rows_kernel", r"if \(cmp_bad\(P, j\)\) continue;", "the index path's bad values"),
    (CK, "cmp_place_kernel", r"if \(t <= P\.nrows\) P\.out_off\[t\] = bad \? 0 : P\.pos\[min\(P\.v_off\[t\], P\.v_cap\)\];",
     "cmp_place_kernel's min"),
]


def check_sources(texts=None):
    """Every pinned statement in the sources (texts: {file: text} to check instead of the files)."""
    cache = {}
    for fn, func, pat, what in STATEMENTS:
        if fn not in cache:
            cache[fn] = texts[fn] if texts is not None and fn in texts else _src(fn)
        body = _fn(func, cache[fn]) if func else cache[fn]
        _one(pat, body, what)


check_sources()
FZ_LONG_NT, RX_NT, RX_WARP_STATES, RX_LONG_BYTES, RX_SMEM_TABLE = 256, 256, 64, 4096, 32768
ABSORB, ACCEPT, START = 2, 4, 2
CMP_NT, CP_TILE, EN_TILE = 256, 256 * 8, 256 * 8
NO_ARG = 0xFFFFFFFF
LAUNCHES = {"match": 5, "regex": 5, "cmp": 5, "rows": 4}
T_INT, T_FLOAT, T_BOOL, T_TIME, T_STR = 1, 2, 3, 5, 6
OPS = {"le": 0, "ge": 1, "lt": 2, "gt": 3, "eq": 4, "between": 5}


def long_warps(sms):
    return 2 * sms * (FZ_LONG_NT // 32)


def pair_stride(sms, nvals):
    return min(-(-nvals // 256), 8 * sms) * 256


# ---------------------------------------------------------------------------------------------------------------
# events and mutants
ALIGN_KINDS = ("rx_thread_first", "rx_thread_last", "rx_warp_first", "rx_warp_last", "cmp_first", "cmp_last", "fz")
EVENTS = set("""
fe.count_below_ccap fe.junk_past_count fe.count_high_bits fe.refuse_count_word fe.col_refuse_past_ccap
fe.refuse_last_cta fe.byte_refuse_last_value fe.cand_refuse_last_thread fe.zero_before_counted
fe.counted_at_scan_tile_end fe.counted_at_scan_tile_start fe.kept_at_compact_tile_end fe.kept_at_compact_tile_start
fz.short fz.long fz.empty_value fz.sc_pass fz.sc_fail fz.dp fz.rune_straddles_round fz.lookback3_across_round
fz.invalid_at_round_start fz.owner_second_word fz.owner_first_word fz.carry_wraps fz.W64
fz.q_nw_minus_1 fz.q_nw fz.q_nw_plus_1 fz.q_three_passes
rx.smem rx.gmem rx.nt_16383 rx.nt_16384 rx.nt_16385 rx.thread_absorb_stop rx.len_4096_thread rx.len_4097_warp
rx.ns64_warp rx.ns65_thread rx.long_empty_lane rx.long_accept_through_empty_lanes rx.long_lo_15 rx.long_all_absorbed rx.long_converged
rx.long_decided_in_lane31 rx.long_carry_matters rx.long_line_start_at_edge rx.long_lane0_absorbs
rx.np_eq_stride rx.np_stride_plus_1 rx.q_nw_minus_1 rx.q_nw rx.q_nw_plus_1 rx.q_three_passes
cmp.np_eq_stride cmp.np_stride_plus_1 cmp.bad_only_in_later_stride cmp.counts_past_count cmp.eq_set_folded
cmp.eq_hit_first cmp.eq_hit_last cmp.eq_miss_between cmp.str_prefix cmp.eq_nan_only
idx.vcap_beyond_m idx.nrows_past_vcap idx.row_edge_on_cta_edge idx.no_arg_next_to_filtered idx.only_last_of_many
idx.bad_skipped idx.refused
""".split()) | {f"align.{k}.{o}" for k in ALIGN_KINDS for o in range(16)}

MUTANTS = {
    "owner lower_bound(p)": "each pair's owner found with lower_bound(pair_off, p) - 1",
    "candidate order over ccap": "the candidate order checked for t < ccap instead of t < nc",
    "count word unmasked": "the count word used whole, not its low 32 bits",
    "long warp first pair only": "a long-tier warp takes only its first queued pair",
    "rune count as bytes": "the long tier's rune count taken as the value's bytes",
    "fz_starts two bytes": "fz_starts looks back two bytes, not three",
    "score lane (W-1)>>5": "the long tier reads the score from lane (W - 1) >> 5",
    "empty chunks dead": "rx_long_kernel composes the lanes with empty chunks as the dead state",
    "compose from RX_START": "lane 0's composition starts at RX_START instead of lane 0's state",
    "term at c + nstates": "rx_test_kernel<true> reads term at c + nstates",
    "class map unrounded": "rx_test_kernel<true> reads the class map at 2 nt instead of round16(2 nt)",
    "first segment whole": "rx_load reads the column's first segment whole whatever clo is",
    "warp tier at 65 states": "the warp tier takes DFAs of up to 65 states",
    "pairs one stride": "the fixed-grid pair loops take only their first stride",
    "eq first above": "eq's search finds the first argument above the value",
    "counts over ccap": "cmp_finish_kernel writes counts for every slot below ccap",
    "NO_ARG filtered": "a CMP_NO_ARG row is filtered against argument 0",
    "first value only": "cmp_rows_kernel tests only a uid's first value",
}


class Events:
    def __init__(self):
        self.s = set()

    def __call__(self, name, cond=True):
        if name not in EVENTS:
            raise KeyError(f"unregistered event {name}")
        if cond:
            self.s.add(name)


class Fault(Exception):
    """A mutant that makes the kernel read or write outside what the model can restate."""


# ---------------------------------------------------------------------------------------------------------------
# the string reader: rx_span / rx_load
@functools.lru_cache(maxsize=None)
def rx_load(clo, chi, g, whole_first=False):
    """(first, end, whole) of the column bytes load g reads, in segment coordinates: rx_load's two paths."""
    if (g * 16 >= clo or whole_first) and g * 16 + 16 <= chi:
        return g * 16, g * 16 + 16, True
    return max(g * 16, clo), min(g * 16 + 16, chi), False


class Reader:
    """One column's bytes seen from its aligned base: clo = the column's offset inside its first segment."""

    def __init__(self, data: bytes, clo: int, mut=None):
        self.data, self.clo, self.chi = data, clo, clo + len(data)
        self.whole_first = mut == "first segment whole"
        self.oob = False
        self.byte_first = self.byte_last = False

    def span(self, b0, ln):
        return self.clo + b0, self.clo + b0 + ln

    def load(self, g):
        a, b, whole = rx_load(self.clo, self.chi, g, self.whole_first)
        if a < self.clo or b > self.chi:
            self.oob = True
        if not whole and g * 16 < self.clo:
            self.byte_first = True
        if not whole and g * 16 + 16 > self.chi:
            self.byte_last = True
        return a, b

    def byte(self, x):
        return self.data[x - self.clo]


def segs_read(clo, nbytes, lo, hi, kind, alen=None):
    """The loads of one consumer over value [lo, hi) (segment coordinates): the thread tier's walk, the warp tier's
    chunks, or cmp_bytes against an argument of alen bytes equal to the value's prefix."""
    if kind == "thread":
        return range(lo // 16, -(-hi // 16))
    if kind == "warp":
        g0, nseg = lo // 16, -(-hi // 16) - lo // 16
        per = -(-nseg // 32)
        out = []
        for lane in range(32):
            s0 = g0 + lane * per
            if s0 >= g0 + nseg:
                break  # the rest of the lanes have empty chunks
            out.extend(range(s0, min(s0 + per, g0 + nseg)))
        return out
    out, i, q = [], 0, lo & ~15
    while q < hi and i < alen:
        out.append(q // 16)
        i += min(alen - i, min(q + 16, hi) - max(q, lo))
        q += 16
    return out


# ---------------------------------------------------------------------------------------------------------------
# fixtures
Fixture = namedtuple("Fixture", "name case events kills")


def str_arrays(values):
    """(val_off, byte_off, data) of a list of lists of bytes."""
    val_off = np.zeros(len(values) + 1, np.int64)
    np.cumsum([len(vs) for vs in values], out=val_off[1:])
    flat = [v for vs in values for v in vs]
    byte_off = np.zeros(len(flat) + 1, np.int64)
    np.cumsum([len(v) for v in flat], out=byte_off[1:])
    return val_off, byte_off, b"".join(flat)


def f64(w):
    return struct.unpack("<d", struct.pack("<Q", w & U64))[0]


def s64(w):
    w &= U64
    return w - (1 << 64) if w >> 63 else w


def words_of(typ, vals):
    if typ == T_INT:
        return [v & U64 for v in vals], [0] * len(vals)
    if typ == T_FLOAT:
        return [struct.unpack("<Q", struct.pack("<d", float(v)))[0] for v in vals], [0] * len(vals)
    if typ == T_BOOL:
        return [1 if v else 0 for v in vals], [0] * len(vals)
    return [v[0] & U64 for v in vals], [v[1] for v in vals]


class Column:
    """A fixture's column as the device reads it: uids, val_off, and string bytes or typed words, with the broken
    arrays a lane-form fixture hands over."""

    def __init__(self, case):
        typ = case.get("typ", T_STR)
        self.typ = typ
        self.uid = np.asarray(case["uids"], np.uint64)
        vals = case["values"]
        self.n = self.uid.size
        if typ == T_STR:
            self.val_off, self.byte_off, self.data = str_arrays(vals)
            self.nvals = self.byte_off.size - 1
        else:
            self.val_off = np.zeros(len(vals) + 1, np.int64)
            np.cumsum([len(vs) for vs in vals], out=self.val_off[1:])
            self.word, self.nsec = words_of(typ, [v for vs in vals for v in vs])
            self.byte_off, self.data = None, b""
            self.nvals = len(self.word)
        bad = case.get("bad")
        self.bad = None if bad is None else [bool(b) for bs in bad for b in bs]
        for k, v in case.get("broken", {}).items():
            setattr(self, k, np.asarray(v, np.int64 if k != "uid" else np.uint64))


# ---------------------------------------------------------------------------------------------------------------
# the front end
def front(ev, col, cands, word, ccap, mut):
    """fz_lookup_kernel, the pair scan and the owner search: (nc, vlo, pair_off, owner of each pair) or None when the
    call is refused."""
    n, nvals = col.n, col.nvals
    T = max(ccap, n + 1, nvals + 1)
    grid = -(-T // 256)
    raw = ccap if word is None else (word if mut == "count word unmasked" else word & 0xFFFFFFFF)
    ev("fe.count_high_bits", word is not None and word >> 32 != 0)
    nc = raw if raw <= ccap else 0
    refuse = []
    if raw > ccap:
        ev("fe.refuse_count_word")
        refuse.append(0)
    vo, bo = col.val_off, col.byte_off
    if vo[0] != 0 or vo[n] != nvals or (bo is not None and (bo[0] != 0 or bo[nvals] != len(col.data))):
        refuse.append(0)
    u = col.uid
    bad_t = set(np.nonzero(u[1:] <= u[:-1])[0] + 1) | set(np.nonzero(vo[:-1] > vo[1:])[0])
    if bo is not None:
        bt = np.nonzero(bo[:-1] > bo[1:])[0]
        ev("fe.byte_refuse_last_value", nvals - 1 in set(bt) and T == nvals + 1)
        bad_t |= set(bt)
    for t in bad_t:
        ev("fe.col_refuse_past_ccap", ccap > 0 and t >= ccap)
    c = np.asarray(cands, np.uint64)
    lim = ccap if mut == "candidate order over ccap" else nc
    ct = set(np.nonzero(c[1:lim] <= c[:lim - 1])[0] + 1) if lim > 1 else set()
    ev("fe.cand_refuse_last_thread", T - 1 in ct)
    refuse += sorted(bad_t | ct)
    if refuse:
        ev("fe.refuse_last_cta", grid > 1 and any(t // 256 == grid - 1 for t in refuse))
        return None
    ev("fe.count_below_ccap", word is not None and nc < ccap)
    ev("fe.junk_past_count", nc < ccap and nc > 0 and bool(np.any(c[nc:ccap] <= c[nc - 1:ccap - 1])))
    k = np.searchsorted(u, c[:nc])
    hit = (k < n) & (u[np.minimum(k, max(n - 1, 0))] == c[:nc]) if n else np.zeros(nc, bool)
    kk = np.minimum(k, max(n - 1, 0))
    cnt = np.where(hit, vo[kk + 1] - vo[kk], 0) if n else np.zeros(nc, np.int64)
    vlo = np.where(hit, vo[kk], 0) if n else np.zeros(nc, np.int64)
    for e in (EN_TILE - 1, 2 * EN_TILE - 1):
        for i, name in ((e, "fe.counted_at_scan_tile_end"), (e + 1, "fe.counted_at_scan_tile_start")):
            if 0 < i < nc - 1 and cnt[i] and not cnt[i - 1] and not cnt[i + 1]:
                ev(name)
    ev("fe.zero_before_counted", nc > 1 and bool(np.any((cnt[:-1] == 0) & (cnt[1:] > 0))))
    pair_off = np.zeros(nc + 1, np.int64)
    np.cumsum(cnt, out=pair_off[1:])
    npairs = int(pair_off[-1])
    p = np.arange(npairs, dtype=np.int64)
    owner = np.searchsorted(pair_off, p if mut == "owner lower_bound(p)" else p + 1, "left") - 1
    if np.any(owner < 0) or np.any(owner >= nc):
        raise Fault("owner outside the candidates")
    j = vlo[owner] + (p - pair_off[owner])
    if np.any(j >= nvals):
        raise Fault("value outside the column")
    return nc, owner, j


def compact(ev, cands, keep, ccap):
    out = [int(cands[c]) for c in np.nonzero(keep)[0]]
    for e in (CP_TILE - 1, 2 * CP_TILE - 1):
        for i, name in ((e, "fe.kept_at_compact_tile_end"), (e + 1, "fe.kept_at_compact_tile_start")):
            if 0 < i < ccap - 1 and keep[i] and not keep[i - 1] and not keep[i + 1]:
                ev(name)
    return out


# ---------------------------------------------------------------------------------------------------------------
# match()
def decode(b, i, ln):
    """fz_decode: (rune, width)."""
    b0 = b[i]
    if b0 < 0x80:
        return b0, 1
    if b0 < 0xC2 or b0 > 0xF4:
        return 0xFFFD, 1
    need = 1 if b0 < 0xE0 else 2 if b0 < 0xF0 else 3
    if i + need >= ln:
        return 0xFFFD, 1
    lo, hi = {0xE0: (0xA0, 0xBF), 0xED: (0x80, 0x9F), 0xF0: (0x90, 0xBF), 0xF4: (0x80, 0x8F)}.get(b0, (0x80, 0xBF))
    if not lo <= b[i + 1] <= hi or any(not 0x80 <= b[i + k] <= 0xBF for k in range(2, need + 1)):
        return 0xFFFD, 1
    return 0, need + 1


def runes(b):
    n, i = 0, 0
    while i < len(b):
        i += decode(b, i, len(b))[1]
        n += 1
    return n


def starts(s, i, back=3):
    """fz_starts: (is a rune start, the look-back distance that decided)."""
    if (s[i] & 0xC0) != 0x80:
        return True, 0
    for k in range(1, min(back, i) + 1):
        if (s[i - k] & 0xC0) == 0x80:
            continue
        return decode(s, i - k, len(s))[1] <= k, k
    return True, 0


def round_runes(ev, s, mut):
    if mut == "rune count as bytes":
        return len(s)
    n = 0
    for b in range(0, len(s), 32):
        for i in range(b, min(b + 32, len(s))):
            st, k = starts(s, i, 2 if mut == "fz_starts two bytes" else 3)
            if i % 32 < k:
                ev("fz.rune_straddles_round", not st)
                ev("fz.lookback3_across_round", not st and k == 3)
            if i == b and b > 0 and st and (s[i] & 0xC0) == 0x80:
                ev("fz.invalid_at_round_start")
            n += st
    return n


def shortcut(n, m, mx):
    if abs(n - m) > mx:
        return 0
    return 1 if mx >= max(n, m) else -1


def run_match(ev, f, col, reader, cands, word, ccap, sms, mut):
    import match_oracle as mo

    q, mx = f["query"], f["max"]
    q = q.encode() if isinstance(q, str) else q
    m = runes(q)
    W = max(1, -(-m // 64))
    ev("fz.short" if W == 1 else "fz.long")
    ev(f"align.fz.{reader.clo}")
    fr = front(ev, col, cands, word, ccap, mut)
    if fr is None:
        return ("refused",)
    nc, owner, jj = fr
    keep = np.zeros(ccap, bool)
    queue = []
    for c, j in zip(owner.tolist(), jj.tolist()):
        b0, b1 = int(col.byte_off[j]), int(col.byte_off[j + 1])
        if b1 == b0:
            ev("fz.empty_value")
            continue
        if W > 1:
            queue.append((c, b0, b1))
            continue
        v = col.data[b0:b1]
        sc = shortcut(runes(v), m, mx)
        ev(("fz.sc_fail", "fz.sc_pass", "fz.dp")[sc if sc >= 0 else 2])
        if sc == 1 or (sc < 0 and mo.levenshtein(v, q) <= mx):
            keep[c] = True
    NW = long_warps(sms)
    nq = len(queue)
    ev("fz.q_nw_minus_1", nq == NW - 1)
    ev("fz.q_nw", nq == NW)
    ev("fz.q_nw_plus_1", nq == NW + 1)
    ev("fz.q_three_passes", nq > 2 * NW)
    owner_lane = (W - 1) & 31
    if W > 1:
        ev("fz.owner_first_word", 2 < W <= 32)
        ev("fz.owner_second_word", 32 < W < 64)
        ev("fz.carry_wraps", W > 32)
        ev("fz.W64", W == 64)
    memo = {}
    for qi, (c, b0, b1) in enumerate(queue):
        if mut == "long warp first pair only" and qi >= NW:
            continue
        v = col.data[b0:b1]
        key = v
        if key not in memo:
            n = round_runes(ev, v, mut)
            sc = shortcut(n, m, mx)
            ev(("fz.sc_fail", "fz.sc_pass", "fz.dp")[sc if sc >= 0 else 2])
            if sc >= 0:
                memo[key] = sc == 1
            else:
                true_n = runes(v)
                if n > true_n:
                    raise Fault("the wavefront decodes past the value")
                score = mo.levenshtein(_prefix_runes(v, n), q)
                lane = ((W - 1) >> 5) if mut == "score lane (W-1)>>5" else owner_lane
                if lane != owner_lane:
                    score = m
                memo[key] = score <= mx
        if memo[key]:
            keep[c] = True
    return ("ok", compact(ev, cands, keep, ccap), None)


def _prefix_runes(v, n):
    i = 0
    for _ in range(n):
        i += decode(v, i, len(v))[1]
    return v[:i]


# ---------------------------------------------------------------------------------------------------------------
# regexp()
@functools.lru_cache(maxsize=None)
def dfa(pattern, fold=False):
    """(cls, trans, term, nstates, nclasses) from the library's compiler."""
    from dgraph_b200 import algo

    cls, trans, term = algo.RegexProg(pattern, fold).tables()
    return cls, trans, term, trans.shape[0], trans.shape[1]


def smem_plan(ns, nc):
    nt = ns * nc
    smem = (nt * 2 + 15) // 16 * 16 + 256 + ns
    return nt * 2 <= RX_SMEM_TABLE and smem <= 48 * 1024, (nt * 2 <= RX_SMEM_TABLE), smem


def smem_tables(cls, trans, term, ns, nc, mut):
    """The tables rx_test_kernel<true> reads, taken from the shared-memory image it writes."""
    nt = ns * nc
    size = (nt * 2 + 15) // 16 * 16 + 256 + ns
    img = bytearray(size)
    img[:2 * nt] = trans.astype("<u2").tobytes()
    c = (nt * 2 + 15) & ~15
    img[c:c + 256] = cls.tobytes()
    img[c + 256:c + 256 + ns] = term.tobytes()
    rc = 2 * nt if mut == "class map unrounded" else c
    rt = rc + ns if mut == "term at c + nstates" else rc + 256
    if rt + ns > size or rc + 256 > size:
        raise Fault("a shared read past the table")
    rcls = np.frombuffer(bytes(img[rc:rc + 256]), np.uint8)
    rterm = np.frombuffer(bytes(img[rt:rt + ns]), np.uint8)
    rtrans = np.frombuffer(bytes(img[:2 * nt]), "<u2").reshape(ns, nc)
    if int(rtrans.max(initial=0)) >= ns:
        raise Fault("a transition past the states")
    return rcls, rtrans, rterm


class Dfa:
    def __init__(self, cls, trans, term):
        self.nxt = trans[:, cls].astype(np.int64)  # state x byte
        self.term = term
        self.ns = trans.shape[0]

    def seg(self, rd, g, lo, hi, s):
        a, b = rd.load(g)
        for x in range(max(a, lo), min(b, hi)):
            s = int(self.nxt[s, rd.byte(x)])
        return s

    def absorbs(self, s):
        return bool(self.term[s] & ABSORB)


def rx_thread(ev, D, rd, lo, hi):
    s, q = START, lo & ~15
    while q < hi and not D.absorbs(s):
        s = D.seg(rd, q // 16, lo, hi, s)
        q += 16
    ev("rx.thread_absorb_stop", q < hi)
    return bool(D.term[s] & ACCEPT)


def rx_warp(ev, D, rd, lo, hi, mut):
    g0 = lo // 16
    nseg = -(-hi // 16) - g0
    per = -(-nseg // 32)
    S = D.ns
    ev("rx.long_lo_15", lo % 16 == 15)
    maps, v0 = [], START
    for lane in range(32):
        s0 = g0 + lane * per
        s1 = min(s0 + per, g0 + nseg)
        empty = s0 >= s1
        ev("rx.long_empty_lane", empty)
        single, v, mp = lane == 0, START, list(range(S))
        for g in range(s0, s1):
            if single:
                if D.absorbs(v):
                    ev("rx.long_lane0_absorbs", lane == 0)
                    break
                v = D.seg(rd, g, lo, hi, v)
                continue
            a, b = rd.load(g)
            bs = [rd.byte(x) for x in range(max(a, lo), min(b, hi))]
            for k in range(S):
                x = mp[k]
                for by in bs:
                    x = int(D.nxt[x, by])
                mp[k] = x
            live = {x for x in mp if not D.absorbs(x)}
            if len(live) == 1:
                ev("rx.long_converged")
                single, v = True, live.pop()
            elif not live:
                ev("rx.long_all_absorbed")
                break
        if single and lane:
            mp = [x if D.absorbs(x) else v for x in mp]
        if empty and mut == "empty chunks dead":
            mp = [0] * S
        if lane == 0:
            v0 = v
        maps.append(mp)
    st = START if mut == "compose from RX_START" else v0
    for lane in range(1, 32):
        if D.absorbs(st):
            break
        ev("rx.long_decided_in_lane31", lane == 31 and not D.term[st] & ACCEPT and D.term[maps[31][st]] & ACCEPT)
        ch = g0 + lane * per
        ev("rx.long_accept_through_empty_lanes", ch >= g0 + nseg and bool(D.term[st] & ACCEPT))
        if ch < g0 + nseg:
            ev("rx.long_carry_matters", st not in (START, 3) and bool(D.term[maps[lane][st]] & ACCEPT)
               and not D.term[maps[lane][START]] & ACCEPT)  # a match across the chunk edge
            ev("rx.long_line_start_at_edge", st == 3 and lo <= ch * 16 - 1 < hi and rd.byte(ch * 16 - 1) == 10)
        st = maps[lane][st]
    return bool(D.term[st] & ACCEPT)


def plain_walk(D, rd, lo, hi):
    s = START
    for x in range(lo, hi):
        if D.absorbs(s):
            break
        s = int(D.nxt[s, rd.byte(x)])
    return bool(D.term[s] & ACCEPT)


def run_regex(ev, f, col, reader, cands, word, ccap, sms, mut):
    cls, trans, term, ns, nc = dfa(f["pattern"], f.get("fold", False))
    use_smem, _, _ = smem_plan(ns, nc)
    nt = ns * nc
    ev("rx.smem" if use_smem else "rx.gmem")
    ev("rx.nt_16384", nt == 16384)
    ev("rx.nt_16385", nt == 16385)
    ev("rx.nt_16383", use_smem and nt == 16383)  # odd: the class map's offset is rounded up past the table
    Dt = Dfa(*smem_tables(cls, trans, term, ns, nc, mut)) if use_smem else Dfa(cls, trans, term)
    Dw = Dfa(cls, trans, term)
    warp = ns <= (RX_WARP_STATES + 1 if mut == "warp tier at 65 states" else RX_WARP_STATES)
    if warp and ns > RX_WARP_STATES:
        raise Fault("a state row past the warp's maps")
    fr = front(ev, col, cands, word, ccap, mut)
    if fr is None:
        return ("refused",)
    ncand, owner, jj = fr
    np_ = owner.size
    S = pair_stride(sms, col.nvals)
    ev("rx.np_eq_stride", np_ == S and S == 8 * sms * 256)
    ev("rx.np_stride_plus_1", np_ == S + 1 and S == 8 * sms * 256)
    keep = np.zeros(ccap, bool)
    queue = []
    memo = {}
    first_seg_end, last_seg_start = 16, (reader.chi - 1) // 16 * 16
    for p, (c, j) in enumerate(zip(owner.tolist(), jj.tolist())):
        if mut == "pairs one stride" and p >= S:
            continue
        b0, b1 = int(col.byte_off[j]), int(col.byte_off[j + 1])
        if b1 == b0:
            continue
        lo, hi = reader.span(b0, b1 - b0)
        if warp and b1 - b0 > RX_LONG_BYTES:
            ev("rx.len_4097_warp", b1 - b0 == RX_LONG_BYTES + 1)
            ev("rx.ns64_warp", ns == RX_WARP_STATES)
            queue.append((c, lo, hi))
            continue
        ev("rx.len_4096_thread", b1 - b0 == RX_LONG_BYTES)
        ev("rx.ns65_thread", ns == RX_WARP_STATES + 1 and b1 - b0 > RX_LONG_BYTES)
        edge = lo < first_seg_end or hi > last_seg_start
        if edge:
            rd0 = (reader.byte_first, reader.byte_last)
            reader.byte_first = reader.byte_last = False
            hit = rx_thread(ev, Dt, reader, lo, hi)
            ev(f"align.rx_thread_first.{reader.clo}", reader.byte_first or (reader.clo == 0 and lo < 16))
            ev(f"align.rx_thread_last.{reader.chi % 16}", reader.byte_last or (reader.chi % 16 == 0 and
                                                                              hi > last_seg_start))
            reader.byte_first, reader.byte_last = rd0[0] or reader.byte_first, rd0[1] or reader.byte_last
        else:
            key = (col.data[b0:b1], lo % 16)
            if key not in memo:
                memo[key] = rx_thread(ev, Dt, reader, lo, hi) if np_ < 5000 else plain_walk(Dt, reader, lo, hi)
            hit = memo[key]
        if hit:
            keep[c] = True
    NW = 2 * sms * (RX_NT // 32)
    nq = len(queue)
    ev("rx.q_nw_minus_1", nq == NW - 1)
    ev("rx.q_nw", nq == NW)
    ev("rx.q_nw_plus_1", nq == NW + 1)
    ev("rx.q_three_passes", nq > 2 * NW)
    wmemo = {}
    for qi, (c, lo, hi) in enumerate(queue):
        if mut == "long warp first pair only" and qi >= NW:
            continue
        edge = lo < 16 or hi > last_seg_start
        key = (col.data[lo - reader.clo:hi - reader.clo], lo % 16)
        if edge or key not in wmemo:
            bf, bl = reader.byte_first, reader.byte_last
            reader.byte_first = reader.byte_last = False
            r = rx_warp(ev, Dw, reader, lo, hi, mut)
            if edge:
                ev(f"align.rx_warp_first.{reader.clo}", reader.byte_first or (reader.clo == 0 and lo < 16))
                ev(f"align.rx_warp_last.{reader.chi % 16}", reader.byte_last or (reader.chi % 16 == 0 and
                                                                                hi > last_seg_start))
            reader.byte_first, reader.byte_last = bf or reader.byte_first, bl or reader.byte_last
            if not edge:
                wmemo[key] = r
        else:
            r = wmemo[key]
        if r:
            keep[c] = True
    return ("ok", compact(ev, cands, keep, ccap), None)


# ---------------------------------------------------------------------------------------------------------------
# compare
def eq_set(typ, args):
    """cmp_args' eq set: sorted, deduplicated under Equal, NaN dropped, -0 folded to +0, bools to 0 / 1."""
    if typ == T_STR:
        return [(0, 0, a) for a in sorted(set(args))]
    w, ns = words_of(typ, args)
    items = list(zip(w, ns))
    if typ == T_FLOAT:
        items = [(0 if f64(x) == 0 else x, n) for x, n in items if not math.isnan(f64(x))]
        key = lambda t: f64(t[0])  # noqa: E731
    elif typ == T_BOOL:
        items = [(1 if x else 0, n) for x, n in items]
        key = lambda t: t[0]  # noqa: E731
    else:
        key = lambda t: (s64(t[0]), t[1])  # noqa: E731
    out = []
    for t in sorted(items, key=key):
        if not out or key(out[-1]) != key(t):
            out.append(t)
    return [(x, n, b"") for x, n in out]


def raw_args(typ, args):
    if typ == T_STR:
        return [(0, 0, a) for a in args]
    w, ns = words_of(typ, args)
    return [(x, n, b"") for x, n in zip(w, ns)]


class Cmp:
    def __init__(self, ev, typ, op, args, rd, mut):
        self.ev, self.typ, self.op, self.A, self.rd, self.mut = ev, typ, op, args, rd, mut
        self.arg_oob = False

    def isnan(self, w):
        return self.typ == T_FLOAT and math.isnan(f64(w))

    def cmp_bytes(self, lo, hi, a):
        rd, i, q = self.rd, 0, lo & ~15
        while q < hi and i < len(a):
            s, e = rd.load(q // 16)
            for x in range(q, q + 16):
                if x < lo or x >= hi or i >= len(a):
                    continue
                b = rd.byte(x)
                if b != a[i]:
                    return -1 if b < a[i] else 1
                i += 1
            q += 16
        ln = hi - lo
        self.ev("cmp.str_prefix", min(ln, len(a)) > 0 and ln != len(a) and i == min(ln, len(a)))
        return -1 if ln < len(a) else (1 if ln > len(a) else 0)

    def order(self, x, k):
        a = self.A[k]
        if self.typ == T_STR:
            return self.cmp_bytes(x[0], x[1], a[2])
        if self.typ == T_FLOAT:
            va, vb = f64(a[0]), f64(x[0])
        else:
            va, vb = s64(a[0]), s64(x[0])
        if vb != va:
            return -1 if vb < va else 1
        if self.typ == T_TIME:
            return -1 if x[1] < a[1] else (1 if x[1] > a[1] else 0)
        return 0

    def ge(self, x, k):
        if self.typ == T_BOOL:
            return False
        if self.isnan(x[0]) or self.isnan(self.A[k][0]):
            return True
        return self.order(x, k) >= 0

    def le(self, x, k):
        if self.typ == T_BOOL:
            return False
        if self.isnan(x[0]) or self.isnan(self.A[k][0]):
            return True
        return self.order(x, k) <= 0

    def test(self, x, k, ne):
        op = self.op
        if op == "ge":
            return self.ge(x, k)
        if op == "le":
            return self.le(x, k)
        if op == "between":
            return self.ge(x, k) and self.le(x, k + 1)
        if op in ("gt", "lt"):
            if self.typ == T_BOOL or self.isnan(x[0]) or self.isnan(self.A[k][0]):
                return False
            c = self.order(x, k)
            return c > 0 if op == "gt" else c < 0
        if self.typ == T_BOOL:
            return any((self.A[i][0] != 0) == (x[0] != 0) for i in range(k, k + ne))
        if self.isnan(x[0]):
            return False
        lo, hi = k, k + ne
        while lo < hi:
            mid = (lo + hi) >> 1
            o = self.order(x, mid)
            if (o >= 0 if self.mut == "eq first above" else o > 0):
                lo = mid + 1
            else:
                hi = mid
        hit = lo < k + ne and not self.isnan(self.A[lo][0]) and self.order(x, lo) == 0
        if hit and ne > 1 and self.typ != T_STR:
            self.ev("cmp.eq_hit_first", lo == k)
            self.ev("cmp.eq_hit_last", lo == k + ne - 1)
        self.ev("cmp.eq_miss_between", not hit and k < lo < k + ne and self.typ != T_STR)
        return hit


def value_of(col, rd, j):
    if col.typ == T_STR:
        return rd.span(int(col.byte_off[j]), int(col.byte_off[j + 1] - col.byte_off[j]))
    return col.word[j], col.nsec[j]


def is_bad(col, j):
    return (col.bad is not None and col.bad[j]) or (col.typ == T_TIME and col.nsec[j] >= 1000000000)


def run_cmp(ev, f, col, reader, cands, word, ccap, sms, mut, op, args):
    typ = col.typ
    A = eq_set(typ, args) if op == "eq" else raw_args(typ, args)
    if op == "eq" and typ != T_STR:
        ev("cmp.eq_set_folded", len(A) < len(args))
        ev("cmp.eq_nan_only", len(A) == 0)
    ne = len(A) if op == "eq" else 1
    fr = front(ev, col, cands, word, ccap, mut)
    if fr is None:
        return ("refused",)
    nc, owner, jj = fr
    S = pair_stride(sms, col.nvals)
    C = Cmp(ev, typ, op, A, reader, mut)
    hits = np.zeros(ccap, np.int64)
    bad_p = []
    edge_hi = (reader.chi - 1) // 16 * 16
    for p, (c, j) in enumerate(zip(owner.tolist(), jj.tolist())):
        if mut == "pairs one stride" and p >= S:
            continue
        if is_bad(col, j):
            bad_p.append(p)
            continue
        if ne == 0:
            continue
        x = value_of(col, reader, j)
        if typ == T_STR and (x[0] < 16 or x[1] > edge_hi):
            bf, bl = reader.byte_first, reader.byte_last
            reader.byte_first = reader.byte_last = False
            t = C.test(x, 0, ne)
            ev(f"align.cmp_first.{reader.clo}", reader.byte_first or (reader.clo == 0 and x[0] < 16))
            ev(f"align.cmp_last.{reader.chi % 16}", reader.byte_last or (reader.chi % 16 == 0 and x[1] > edge_hi))
            reader.byte_first, reader.byte_last = bf or reader.byte_first, bl or reader.byte_last
        else:
            t = C.test(x, 0, ne)
        if t:
            hits[c] += 1
    if bad_p:
        ev("cmp.bad_only_in_later_stride", min(bad_p) >= S)
        return ("refused",)
    ev("cmp.np_eq_stride", owner.size == S and S == 8 * sms * 256)
    ev("cmp.np_stride_plus_1", owner.size == S + 1 and S == 8 * sms * 256)
    keep = hits > 0
    counts = [None] * ccap
    lim = ccap if mut == "counts over ccap" else nc
    for t in range(lim):
        counts[t] = int(hits[t])
    ev("cmp.counts_past_count", nc < ccap)
    return ("ok", compact(ev, cands, keep, ccap), tuple(counts))


def run_rows(ev, f, col, reader, v, v_off, v_cap, row_arg, sms, mut, op, args):
    typ = col.typ
    A = raw_args(typ, args)
    nrows = len(v_off) - 1
    fr = front(ev, col, [], None, 0, mut)
    m = int(v_off[nrows])
    if fr is None or v_off[0] != 0 or m > v_cap or any(v_off[t] > v_off[t + 1] for t in range(nrows)):
        ev("idx.refused")
        return ("refused", nrows)
    ev("idx.vcap_beyond_m", v_cap > m)
    ev("idx.nrows_past_vcap", nrows + 1 > v_cap)
    for r in range(1, nrows):
        e = int(v_off[r])
        if 0 < e < m and e % 256 == 0 and v_off[r - 1] < e < v_off[r + 1]:
            ev("idx.row_edge_on_cta_edge")
    for r in range(nrows - 1):
        a, b = row_arg[r], row_arg[r + 1]
        if v_off[r] < v_off[r + 1] and v_off[r + 1] < v_off[r + 2] and (a == NO_ARG) != (b == NO_ARG):
            ev("idx.no_arg_next_to_filtered")
    C = Cmp(ev, typ, op, A, reader, mut)
    flag = [0] * v_cap
    vo = col.val_off
    for t in range(m):
        r = bisect.bisect_left(v_off, t + 1) - 1
        k = row_arg[r]
        if k == NO_ARG and mut != "NO_ARG filtered":
            flag[t] = 1
            continue
        k = 0 if k == NO_ARG else k
        x = int(v[t])
        i = int(np.searchsorted(col.uid, np.uint64(x)))
        if i < col.n and int(col.uid[i]) == x:
            js = list(range(int(vo[i]), int(vo[i + 1])))
            if mut == "first value only":
                js = js[:1]
            res = []
            for j in js:
                if is_bad(col, j):
                    res.append(None)
                    continue
                res.append(C.test(value_of(col, reader, j), k, 1))
                if res[-1]:
                    break
            if res and res[-1]:
                ev("idx.only_last_of_many", len(res) >= 3 and len(js) == len(res) and not any(res[:-1]))
                ev("idx.bad_skipped", None in res)
                flag[t] = 1
    pos = [0] * (v_cap + 1)
    for t in range(v_cap):
        pos[t + 1] = pos[t] + flag[t]
    out_off = []
    for t in range(nrows + 1):
        if int(v_off[t]) > v_cap:
            raise Fault("out_off's index past v_cap")
        out_off.append(pos[min(int(v_off[t]), v_cap)])
    out = [int(v[t]) for t in range(v_cap) if flag[t]]
    return ("ok", tuple(out_off), tuple(out))


# ---------------------------------------------------------------------------------------------------------------
# one call
FORMS = ("host", "lane")


def lane_only(case):
    return case.get("word") is not None or "broken" in case or case.get("v_cap") is not None


def forms(case):
    return ("lane",) if lane_only(case) else FORMS


def run(f, form, sms=H100_SMS, mut=None):
    """(result per call, events, read-set violation) of fixture f through one form."""
    case = f.case
    ev = Events()
    col = Column(case)
    shift = case.get("shift", 0) if form == "lane" else 0
    reader = Reader(col.data, shift, mut)
    kind = case["kind"]
    res = []
    try:
        if kind == "rows":
            v = np.concatenate([np.asarray(r, np.uint64) for r in case["rows"]] + [np.zeros(0, np.uint64)])
            v_off = np.zeros(len(case["rows"]) + 1, np.int64)
            np.cumsum([len(r) for r in case["rows"]], out=v_off[1:])
            v_cap = case.get("v_cap") if form == "lane" and case.get("v_cap") is not None else int(v_off[-1])
            v = np.concatenate([v, np.full(max(v_cap - v.size, 0), 7, np.uint64)])
            for op, args in case["calls"]:
                res.append(run_rows(ev, f, col, reader, v, v_off.tolist(), v_cap, case["row_arg"], sms, mut, op,
                                    args))
        else:
            cands = np.asarray(case["cands"], np.uint64)
            word = case.get("word") if form == "lane" else None
            ccap = cands.size
            if kind == "match":
                res.append(run_match(ev, case, col, reader, cands, word, ccap, sms, mut))
            elif kind == "regex":
                res.append(run_regex(ev, case, col, reader, cands, word, ccap, sms, mut))
            else:
                for op, args in case["calls"]:
                    res.append(run_cmp(ev, case, col, reader, cands, word, ccap, sms, mut, op, args))
    except Fault as e:
        return ("fault", str(e)), ev.s, True
    return tuple(res), ev.s, reader.oob


# ---------------------------------------------------------------------------------------------------------------
# fixtures
AL = b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ"


def literal(A, L):
    return bytes(AL[i % A] for i in range(L)).decode()


# patterns whose DFA has nstates x nclasses table entries just under, exactly at and just over RX_SMEM_TABLE / 2:
# a literal over A distinct letters has A + 2 classes and L + 4 states (tests/test_value_column_geometry.py checks)
TABLE_PATTERNS = {16383: literal(41, 377), 16384: literal(30, 508), 16385: literal(27, 561)}


def _fill(rng, n, alphabet=b"xyz "):
    return rng.choice(np.frombuffer(alphabet, np.uint8), n).tobytes()


def _uids(n, step=3):
    return list(range(5, 5 + step * n, step))


def _fx(name, events, kills=(), **case):
    return Fixture(name, case, frozenset(events), frozenset(kills))


def front_fixtures():
    out = []
    col = dict(uids=[3, 5, 9, 12], values=[[b"xab"], [b"ab"], [b"zz"], [b"ab\nab"]])
    out.append(_fx("fe_count_below_ccap_junk", {"fe.count_below_ccap", "fe.junk_past_count"},
                   {"candidate order over ccap"}, kind="regex", pattern="ab", cands=[3, 5, 9, 4, 2, 1], word=3,
                   **col))
    out.append(_fx("fe_count_high_bits", {"fe.count_high_bits"}, {"count word unmasked"}, kind="regex",
                   pattern="ab", cands=[3, 5, 9, 12], word=2 | (0xABC << 32), **col))
    out.append(_fx("fe_count_over_ccap", {"fe.refuse_count_word"}, kind="regex", pattern="ab", cands=[3, 5, 9],
                   word=4, **col))
    # column refusals the candidates do not cover: a uid order break on a thread past ccap, in the lookup's last CTA
    uids = list(range(1, 601))
    uids[520] = uids[519]
    out.append(_fx("fe_col_refuse_past_ccap", {"fe.col_refuse_past_ccap", "fe.refuse_last_cta"}, kind="match",
                   query="ab", max=1, cands=[2, 3], uids=uids, values=[[b"ab"]] * 600,
                   broken={"uid": uids}))
    # the last value's byte offsets descend: detected by thread nvals - 1, the lookup's last checking thread
    vals = [[b"ab"]] * 299
    vo, bo, _ = str_arrays(vals)
    bo = bo.copy()
    bo[-2] = bo[-1] + 1
    out.append(_fx("fe_byte_refuse_last_value", {"fe.byte_refuse_last_value"}, kind="regex", pattern="ab",
                   cands=list(range(1, 300)), uids=list(range(1, 300)), values=vals, broken={"byte_off": bo}))
    # a candidate descent on thread ccap - 1 = the lookup's last thread
    c = list(range(1, 514))
    c[-1] = 0
    out.append(_fx("fe_cand_refuse_last_thread", {"fe.cand_refuse_last_thread", "fe.refuse_last_cta"}, kind="regex",
                   pattern="ab", cands=c, uids=[1, 2], values=[[b"ab"], [b"a"]]))
    # zero-count runs around counted candidates at the scan and compaction tile edges
    n = 2 * EN_TILE + 9
    cands = list(range(1, 2 * n, 2))
    counted = [EN_TILE - 1, EN_TILE, 2 * EN_TILE - 1, 2 * EN_TILE, 7]
    ucol = sorted(cands[i] for i in counted if i not in (EN_TILE, 2 * EN_TILE - 1))
    out.append(_fx("fe_zero_runs_tile_edges", {"fe.counted_at_scan_tile_end", "fe.kept_at_compact_tile_end",
                                               "fe.counted_at_scan_tile_start", "fe.kept_at_compact_tile_start",
                                               "fe.zero_before_counted"}, {"owner lower_bound(p)"}, kind="regex",
                   pattern="ab", cands=cands, uids=ucol, values=[[b"zab", b"q"]] * len(ucol)))
    # compare: counts past the count word stay untouched, and kept candidates at the tile edges
    out.append(_fx("cmp_counts_past_count", {"cmp.counts_past_count"}, {"counts over ccap"}, kind="cmp", typ=T_INT,
                   calls=[("ge", [10])], cands=[1, 3, 5, 7, 9, 11], word=4, uids=[3, 5, 9, 11],
                   values=[[20, 5, 30], [], [1], [40]]))
    return out


def match_fixtures(sms):
    out = []
    out.append(_fx("fz_short_tier", {"fz.short", "fz.sc_pass", "fz.sc_fail", "fz.dp", "fz.empty_value"},
                   kind="match", query="ab", max=2, cands=[1, 2, 3, 4, 5],
                   uids=[1, 2, 3, 4], values=[[b"sitting"], [b""], [b"abc"], [b"abcdefghijklmn", b"x"]]))
    q = "a" * 65
    emoji = "\U0001F600".encode()
    v1 = b"a" * 29 + emoji + b"a" * 37          # 67 runes; the emoji's bytes 29 .. 32 straddle the round edge
    v2 = b"a" * 32 + b"\x80" + b"a" * 30        # a lone continuation byte at the round start: a rune of its own
    out.append(_fx("fz_rune_count_rounds", {"fz.long", "fz.rune_straddles_round", "fz.lookback3_across_round",
                                            "fz.invalid_at_round_start"},
                   {"rune count as bytes", "fz_starts two bytes"}, kind="match", query=q, max=2, cands=[1, 2],
                   uids=[1, 2], values=[[v1], [v2]]))
    rng = np.random.default_rng(31)
    for W, nm, evs in ((17, "fz_owner_w17", {"fz.owner_first_word"}), (33, "fz_owner_w33",
                                                                     {"fz.owner_second_word", "fz.carry_wraps"}),
                       (64, "fz_owner_w64", {"fz.W64"})):
        m = 64 * (W - 1) + 7 if W < 64 else 4096
        qq = _fill(rng, m, b"abcdefgh")
        v = qq[:m // 2] + qq[m // 2 + 1:]       # one deletion: distance 1
        vfar = _fill(rng, m, b"abcdefgh")
        out.append(_fx(nm, evs | {"fz.dp"}, {"score lane (W-1)>>5"}, kind="match", query=qq, max=1,
                       cands=[1, 2], uids=[1, 2], values=[[v], [vfar]]))
    NW = long_warps(sms)
    for nq, ev in ((NW - 1, "fz.q_nw_minus_1"), (NW, "fz.q_nw"), (NW + 1, "fz.q_nw_plus_1"),
                   (2 * NW + 1, "fz.q_three_passes")):
        # neighbouring queued pairs alternate: a pass (10 runes) and a fail (200 runes), both by the shortcuts
        vals = [[b"b" * (10 if i % 2 == 0 else 200)] for i in range(nq)]
        out.append(_fx(f"fz_long_queue_{nq}", {ev}, {"long warp first pair only"} if nq > NW else (), kind="match",
                       query=q, max=70, cands=list(range(1, nq + 1)), uids=list(range(1, nq + 1)), values=vals))
    return out


def regex_fixtures(sms):
    out = []
    rng = np.random.default_rng(41)
    out.append(_fx("rx_thread_absorb_stop", {"rx.thread_absorb_stop", "rx.smem"}, kind="regex", pattern="ab",
                   cands=[1, 2], uids=[1, 2], values=[[b"ab" + b"x" * 300], [b"x" * 300]]))
    for nt, evs in ((16383, {"rx.nt_16383", "rx.smem"}), (16384, {"rx.nt_16384", "rx.smem"}),
                    (16385, {"rx.nt_16385", "rx.gmem"})):
        p = TABLE_PATTERNS[nt]
        hay = [p.encode(), p[:-1].encode() + b"!", b"zz" + p.encode() + b"zz"]
        out.append(_fx(f"rx_table_{nt}", evs, {"class map unrounded", "term at c + nstates"} if nt == 16383 else (),
                       kind="regex", pattern=p, cands=[1, 2, 3], uids=[1, 2, 3], values=[[h] for h in hay]))
    # the warp tier's bounds: 64 / 65 states, 4096 / 4097 bytes
    for ns in (64, 65):
        c = dfa("ab" * 5)[3] - 10
        pat = "ab" * ((ns - c) // 2) + "a" * ((ns - c) % 2)
        vals = []
        for ln in (4096, 4097, 4097):
            b = bytearray(b"b" * ln)
            if len(vals) != 2:
                b[ln - len(pat):] = pat.encode()
            vals.append([bytes(b)])
        evs = {"rx.len_4096_thread"} | ({"rx.ns64_warp", "rx.len_4097_warp"} if ns == 64 else {"rx.ns65_thread"})
        out.append(_fx(f"rx_warp_bound_{ns}", evs, {"warp tier at 65 states"} if ns == 65 else (), kind="regex",
                       pattern=pat, cands=[1, 2, 3], uids=[1, 2, 3], values=vals))
    # rx_long_kernel's chunks
    L = 4097  # a value from byte 15 of its segment over 257 segments: per 9, lanes 29 .. 31 empty
    v_end = bytearray(_fill(rng, L))
    v_end[-6:] = b"needle"
    out.append(_fx("rx_chunks_empty_lanes", {"rx.long_accept_through_empty_lanes", "rx.long_lo_15"},
                   {"empty chunks dead"},
                   kind="regex", pattern="needle$", cands=[1, 2], uids=[1, 2],
                   values=[[b"x" * 15, bytes(v_end)], [bytes(v_end[:-1]) + b"x"]]))
    L = 288 * 16                           # 288 segments, per 9: lane 31's chunk is the last nine
    v31 = bytearray(_fill(rng, L))
    v31[-20:-14] = b"needle"
    out.append(_fx("rx_chunks_lane31", {"rx.long_decided_in_lane31"}, kind="regex", pattern="needle", cands=[1],
                   uids=[1], values=[[bytes(v31)]]))
    L, e = 288 * 16, 9 * 16                # per 9: lane 1's chunk starts at byte 144
    ve = bytearray(_fill(rng, L))
    ve[e - 3:e + 3] = b"needle"
    vn = bytearray(_fill(rng, L))
    vn[e - 1] = 10
    vn[e:e + 6] = b"needle"
    vx = bytearray(_fill(rng, L))
    vx[e:e + 6] = b"needle"
    out.append(_fx("rx_chunks_needle_across_edge", {"rx.long_carry_matters", "rx.long_converged"},
                   {"compose from RX_START"}, kind="regex", pattern="needle", cands=[1], uids=[1],
                   values=[[bytes(ve)]]))
    out.append(_fx("rx_chunks_newline_at_edge", {"rx.long_line_start_at_edge"}, kind="regex", pattern="^needle",
                   cands=[1, 2], uids=[1, 2], values=[[bytes(vn)], [bytes(vx)]]))
    out.append(_fx("rx_chunks_all_absorbed", {"rx.long_all_absorbed", "rx.long_lane0_absorbs"}, kind="regex",
                   pattern="a", cands=[1, 2], uids=[1, 2], values=[[b"a" * 5000], [b"x" * 5000]]))
    # strides of the fixed grids
    NW = 2 * sms * (RX_NT // 32)
    for nq, ev in ((NW - 1, "rx.q_nw_minus_1"), (NW, "rx.q_nw"), (NW + 1, "rx.q_nw_plus_1"),
                   (2 * NW + 1, "rx.q_three_passes")):
        base = b"a" * 4097
        hit = b"a" * 2000 + b"needle" + b"a" * 2105
        vals = [[hit if i % 2 == 0 else base] for i in range(nq)]
        out.append(_fx(f"rx_warp_queue_{nq}", {ev}, {"long warp first pair only"} if nq > NW else (), kind="regex",
                       pattern="needle", cands=list(range(1, nq + 1)), uids=list(range(1, nq + 1)), values=vals))
    S = 8 * sms * 256
    for np_, ev in ((S, "rx.np_eq_stride"), (S + 1, "rx.np_stride_plus_1")):
        vals = [[b"xab" if i % 2 == 0 else b"xba"] for i in range(S + 1)]
        u = list(range(1, S + 2))
        out.append(_fx(f"rx_pair_stride_{np_}", {ev}, {"pairs one stride"} if np_ > S else (), kind="regex",
                       pattern="ab", cands=u[:np_], uids=u, values=vals))
    return out


def compare_fixtures(sms):
    out = []
    nan, nz = float("nan"), -0.0
    out.append(_fx("cmp_eq_float_set", {"cmp.eq_set_folded", "cmp.eq_hit_first", "cmp.eq_hit_last",
                                        "cmp.eq_miss_between"}, {"eq first above"}, kind="cmp", typ=T_FLOAT,
                   calls=[("eq", [2.5, nan, nz, 0.0, 2.5, 9.0, -1.0])], cands=[1, 2, 3, 4, 5, 6],
                   uids=[1, 2, 3, 4, 5, 6], values=[[-1.0], [0.0], [nz], [nan], [9.0], [1.0]]))
    out.append(_fx("cmp_eq_nan_only", {"cmp.eq_nan_only"}, kind="cmp", typ=T_FLOAT, calls=[("eq", [nan, nan])],
                   cands=[1, 2], uids=[1, 2], values=[[nan], [1.0]]))
    S = 8 * sms * 256
    for np_, bad, ev in ((S, False, "cmp.np_eq_stride"), (S + 1, False, "cmp.np_stride_plus_1"),
                         (S + 1, True, "cmp.bad_only_in_later_stride")):
        u = list(range(1, S + 2))
        vals = [[100 if i % 2 == 0 else 0] for i in range(S + 1)]
        bads = [[False]] * S + [[bad]]
        out.append(_fx(f"cmp_pair_stride_{np_}{'_bad' if bad else ''}", {ev}, {"pairs one stride"} if np_ > S else (),
                       kind="cmp", typ=T_INT, calls=[("ge", [50])], cands=u[:np_], uids=u, values=vals, bad=bads))
    return out


def rows_fixtures():
    out = []
    uids = list(range(1, 700))
    vals = [[i % 7, i % 5, i % 3] for i in range(len(uids))]
    vals[10] = [1, 2, 40]                  # only the last of three passes ge 30
    bad = [[False] * 3 for _ in uids]
    bad[11] = [False, True, False]
    vals[11] = [1, 99, 50]                 # a bad value skipped, a later one passes
    col = dict(kind="rows", typ=T_INT, uids=uids, values=vals, bad=bad)
    rows = [list(range(1, 257)), [11, 12, 13], list(range(300, 300 + 253)), [5, 11, 12]]
    out.append(_fx("idx_row_edges", {"idx.row_edge_on_cta_edge", "idx.no_arg_next_to_filtered",
                                     "idx.only_last_of_many", "idx.bad_skipped"},
                   {"NO_ARG filtered", "first value only"}, calls=[("ge", [30])],
                   rows=rows, row_arg=[NO_ARG, 0, NO_ARG, 0], **col))
    out.append(_fx("idx_vcap_beyond", {"idx.vcap_beyond_m"}, calls=[("lt", [3])], rows=[[1, 2, 3], [4, 9]],
                   row_arg=[0, 0], v_cap=300, **col))
    out.append(_fx("idx_refused_vcap_below_m", {"idx.refused"}, calls=[("lt", [3])], rows=[[1, 2], [4, 9]],
                   row_arg=[0, NO_ARG], v_cap=3, **col))
    rows = [[] for _ in range(300)]
    rows[0], rows[299] = [1, 2], [3]
    out.append(_fx("idx_nrows_past_vcap", {"idx.nrows_past_vcap"}, calls=[("eq", [1, 2])],
                   rows=rows, row_arg=[0] + [NO_ARG] * 298 + [1], **col))
    return out


def align_fixtures():
    """A lane-form column whose bytes start at offset k of a segment, for every k in 1 .. 15; the column's bytes
    are a multiple of 16, so its end is at offset k too."""
    out = []
    rng = np.random.default_rng(51)
    for k in range(1, 16):
        short = b"needle"
        longv = bytearray(_fill(rng, 4101 + 4 * k))
        longv[100:106] = b"needle"
        mid = _fill(rng, 16 * 3)
        pad = (-(len(short) + len(longv) + len(mid))) % 16
        for nm, vals, evs in (("a", [short, mid + b"x" * pad, bytes(longv)], ("rx_thread_first", "rx_warp_last")),
                              ("b", [bytes(longv), mid + b"x" * pad, short], ("rx_warp_first", "rx_thread_last"))):
            out.append(_fx(f"align_rx_{nm}_{k}", {f"align.{e}.{k}" for e in evs}, {"first segment whole"},
                           kind="regex", pattern="needle",
                           shift=k, cands=[1, 2, 3], uids=[1, 2, 3], values=[[v] for v in vals]))
        sv = [b"ab", b"abd", b"ab\xff", b"zz" * 9, b"", b"abc" + b"q" * 20]
        sv.append(b"m" * ((-(sum(len(v) for v in sv) + 3)) % 16 + 16))
        sv.append(b"abc")                   # the column's last bytes
        calls = [("eq", [b"abc", b"ab", b"zz" * 9]), ("le", [b"abd"]), ("lt", [b"ab"]), ("ge", [b"ab\xff"]),
                 ("gt", [b"zz"]), ("between", [b"ab", b"abd"])]
        u = list(range(1, len(sv) + 1))
        out.append(_fx(f"align_cmp_{k}", {f"align.cmp_first.{k}", f"align.cmp_last.{k}"}, {"first segment whole"},
                       kind="cmp", typ=T_STR,
                       shift=k, calls=calls, cands=u, uids=u, values=[[v] for v in sv]))
        out.append(_fx(f"align_fz_{k}", {f"align.fz.{k}"}, kind="match", query="needle", max=2, shift=k,
                       cands=[1, 2], uids=[1, 2], values=[[b"neddle"], [b"x" * k + b"needl"]]))
    return out


def fixtures(sms=H100_SMS):
    return (front_fixtures() + match_fixtures(sms) + regex_fixtures(sms) + compare_fixtures(sms) + rows_fixtures()
            + align_fixtures())
