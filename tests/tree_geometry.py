"""Host model of the two tree evaluators: regexp()'s trigram query (trigram_kernel.cuh tg_leaves_kernel /
tg_gather_kernel / tg_eval_kernel, compressed_kernel.cuh compact_kernel, dgx_api.cu trigram_impl) and math()'s program
(math_kernel.cuh mt_check_kernel ... mt_write_kernel, dgx_api.cu mt_run), with fixtures aimed at every chunk, CTA and
tile boundary of both.

regexp().  The plan (bounds, driving leaves, the all-OR skip, the one-driver case in which the gather is the result and
the launches) is trigram_plan.py's.  On top of it the model restates: tg_leaves_kernel's leaf table in strides of TG_NT
threads with the pack / list split at npacks, its DGX_MUT_VALUE scan over the nmut flags in strides of TG_NT, and the
scan of the driving rows' lengths in chunks of TG_NT with the carry of each chunk's total; tg_gather_kernel's row of a
position, lower_bound(drive_off, t + 1) - 1 (empty rows share an offset with the next one), its cut at min(dcap,
drive_off[nd]) and the 256-thread CTA of each position; the candidates as the union of the gathered rows;
tg_eval_kernel's stackless pre-order walk step by step (opening a node, an OR without children, a leaf's hit or miss,
the close loop and how many levels one leaf closes, the threads past ncand that write keep = 0); compact_kernel's tiles
of CP_TILE slots over dcap.

math().  The thread space of mt_check_kernel and mt_gather_kernel over the leaves' rooms (cap_off): the leaf that owns
each thread when rooms of 0 sit between others, count words below the room, the range's checks from cap_total on;
mt_plan_kernel's leaf kinds and its split into scalar and vector nodes, the scalar nodes' values taken from
gen_math's formula; mt_eval_kernel's thread per key of U, each node's present and failed keys counted per warp and per
CTA and summed, the root's tag set per CTA and combined; mt_finish_kernel's refusals from the global counts, the COND
over nil rule and the int-to-float promotion; the root scan's EN_TILE tiles over ulen; mt_write_kernel's grid of
max(cap, nrange or 1) threads for a constant over a range.  Per-key values use gen_math's rules.

What the kernels decide is named as *events* (EVENTS); fixtures name the events they must reach and the model refuses
a name that is not registered.  Named *mutants* (MUTANTS) are plausible one-line slips; a fixture names the mutants it
kills, and tests/test_tree_geometry.py checks that the mutated model's output differs from the oracle's on it.  No
mutated kernel is built: a broken drive_off or cap_off could send the gather or the merge out of bounds.

Edges the kernels have that no fixture reaches at test scale:
  - leaf bound totals of 2^32 or more, which the host refuses (and so the u32 sums of tg_leaves_kernel's scan);
  - 2^20 leaf references, or trees of 2^16 - 1 nodes over 2^16 - 1 leaves (the host's limits; the fixtures stop at
    3 073 driving leaves);
  - the look-back order of the multi-CTA scans (compact_kernel, the root scan): the scheduler chooses which CTA
    publishes first; the fixtures of two and three tiles make a multi-CTA scan possible but cannot choose its order;
  - u32 wrap of mt_eval_kernel's per-node counts (2^32 keys);
  - count words whose high 32 bits are set (the device form reads the low 32 bits of an info word).

The constants and the statements the model restates are read from the CUDA sources as text, so a rewrite fails here
loudly instead of leaving the fixtures aimed at stale edges.  tests/test_tree_geometry.py checks the fixtures on the
CPU; tests/test_gpu_tree_edges.py runs them through the kernels.
"""
from __future__ import annotations

import itertools
import os
import re
from collections import namedtuple

import numpy as np

import gen_math as gm
import gen_trigram as gt
import math_plan as mp
import trigram_plan as tp
from merge_geometry import tree_launches

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")
OK, ERR_ARG, ERR_CAP = 0, -3, -4
U64 = (1 << 64) - 1
POISON = 0xBAD0BAD0BAD0BAD0    # what a mutant reads where the kernel would read outside its row
QAND, QOR = gt.QAND, gt.QOR
MUT_DEL, MUT_VALUE = 1, 2


def _src(fn):
    path = os.path.join(ROOT, "include", fn) if fn.endswith(".h") else os.path.join(CSRC, fn)
    with open(path) as f:
        return f.read()


def _one(pat, text, what):
    m = re.search(pat, text)
    if not m:
        raise ValueError(f"{what} changed: restate it in the tree model (tests/tree_geometry.py)")
    return m


def _fn(name, text):
    """The body of the function or kernel `name` (a definition starting a line, through its closing brace)."""
    head = r"(?ms)^(?:static |__global__ |__device__ |extern \"C\" )[^\n]*\b"
    return _one(head + name + r"\(.*?\n\}\n", text, name).group(0)


# (file, function or None for the whole file, statement as a regex, what it restates)
STATEMENTS = [
    ("trigram_kernel.cuh", "tg_leaves_kernel", r"for \(u64 k = tid; k < P\.nmut; k \+= TG_NT\)\s*"
     r"if \(P\.flags\[k\] & LU_VALUE\) bad = 1;", "the layers' flag strides"),
    ("trigram_kernel.cuh", "tg_leaves_kernel", r"for \(u32 i = tid; i < P\.nleaves; i \+= TG_NT\) \{",
     "the leaf table's strides"),
    ("trigram_kernel.cuh", "tg_leaves_kernel", r"if \(i < P\.npacks\) \{", "the pack / list split"),
    ("trigram_kernel.cuh", "tg_leaves_kernel", r"if \(bad\) L\.n = 0;", "a value flag empties every leaf"),
    ("trigram_kernel.cuh", "tg_leaves_kernel", r"for \(u32 b = 0; b < P\.ndrive; b \+= TG_NT\) \{",
     "the chunks of the driving rows"),
    ("trigram_kernel.cuh", "tg_leaves_kernel", r"if \(i < P\.ndrive\) P\.drive_off\[i\] = carry \+ ex;\s*"
     r"carry \+= total;", "the chunk carry"),
    ("trigram_kernel.cuh", "tg_leaves_kernel", r"P\.drive_off\[P\.ndrive\] = carry;\s*"
     r"if \(P\.len_word\) \*P\.len_word = carry;", "the driving rows' total"),
    ("trigram_kernel.cuh", "tg_gather_kernel", r"if \(t >= P\.dcap \|\| t >= P\.drive_off\[P\.ndrive\]\) return;",
     "the gather's cut"),
    ("trigram_kernel.cuh", "tg_gather_kernel", r"const u64 d = lower_bound_g\(P\.drive_off, \(u64\)P\.ndrive \+ 1, "
     r"t \+ 1\) - 1;", "the row of a position"),
    ("trigram_kernel.cuh", "tg_gather_kernel", r"P\.gathered\[t\] = L\.p\[t - P\.drive_off\[d\]\];",
     "the gathered value"),
    ("trigram_kernel.cuh", "tg_eval_kernel", r"if \(t >= \*P\.ncand\) \{\s*P\.keep\[t\] = 0;",
     "the threads past ncand"),
    ("trigram_kernel.cuh", "tg_eval_kernel", r"u32 cur = 0, pc = 1;", "the walk's start"),
    ("trigram_kernel.cuh", "tg_eval_kernel", r"if \(end != pc \+ 1\) \{[^\n]*\s*cur = pc\+\+;\s*continue;",
     "opening a node"),
    ("trigram_kernel.cuh", "tg_eval_kernel", r"r = false;[^\n]*\s*pc = end;", "an OR without children"),
    ("trigram_kernel.cuh", "tg_eval_kernel", r"r = tg_member\(P\.leaf\[e\.w0\], x\);\s*\+\+pc;", "a leaf's test"),
    ("trigram_kernel.cuh", "tg_eval_kernel", r"if \(is_and == r && pc != end\) break;", "the close loop's stop"),
    ("trigram_kernel.cuh", "tg_eval_kernel", r"pc = end;\s*if \(f\.w1 == kTgNoParent\) \{\s*P\.keep\[t\] = r;"
     r"\s*return;\s*\}\s*cur = f\.w1;", "closing a node"),
    ("compressed_kernel.cuh", "compact_kernel", r"const u64 e0 = t0 \+ \(u64\)tid \* CP_VT;", "a tile's slots"),
    ("compressed_kernel.cuh", "compact_kernel", r"if \(e0 \+ i < P\.m && P\.keep\[e0 \+ i\]\)", "the kept slots"),
    ("dgx_api.cu", None, r"P->prog\[at\]\.w0 = kTgNode \| \(t->op\[i\] == DGX_QAND \? kTgAnd : 0u\) \| "
     r"\(uint32_t\)P->prog\.size\(\);", "a node's program entry"),
    ("dgx_api.cu", "trigram_impl", r"const bool gather_is_result = T\.all_or && !merge;", "the gather as the result"),
    ("dgx_api.cu", "trigram_impl", r"const unsigned g_val = \(unsigned\)\(\(dcap \+ 255\) / 256\);",
     "the gather's grid"),
    ("dgx_api.cu", "trigram_impl", r"tg_gather_kernel<<<g_val, 256, 0, l->stream>>>\(P\);", "the gather's CTAs"),
    ("dgx_api.cu", "trigram_impl", r"const uint64_t tiles = \(dcap \+ CP_TILE - 1\) / CP_TILE;",
     "the compaction's tiles"),
    ("dgx_api.cu", "trigram_impl", r"P\.ncand = P\.drive_off \+ nd;", "ncand without a merge"),
    ("math_kernel.cuh", "mt_check_kernel", r"while \(P\.cap_off\[j \+ 1\] <= t\) \+\+j;", "a check thread's leaf"),
    ("math_kernel.cuh", "mt_check_kernel", r"if \(i < n && i < L\.n\) \{", "the count word below the room"),
    ("math_kernel.cuh", "mt_check_kernel", r"\} else if \(P\.range && t - P\.cap_total < P\.nrange\) \{",
     "the range's check threads"),
    ("math_kernel.cuh", "mt_check_kernel", r"if \(i > 0 && P\.range\[i - 1\] >= P\.range\[i\]\) bad = true;",
     "the range's order"),
    ("math_kernel.cuh", "mt_plan_kernel", r"\} else if \(n == 1 && \(L\.key\[0\] == ~0ull \|\| L\.key\[0\] == 0\)\) \{",
     "the one-entry leaves"),
    ("math_kernel.cuh", "mt_plan_kernel", r"lk\[j\] = L\.key\[0\] == 0 \? MK_MAP0 : lt\[j\] == MT_NIL \? MK_NIL : "
     r"MK_CONST;", "the one-entry leaves' kinds"),
    ("math_kernel.cuh", "mt_gather_kernel", r"while \(P\.cap_off\[j \+ 1\] <= t\) \+\+j;", "a gather thread's leaf"),
    ("math_kernel.cuh", "mt_gather_kernel", r"if \(i < P\.row_off\[j \+ 1\] - a\) P\.cat\[a \+ i\] = "
     r"P\.leaf\[j\]\.key\[i\];", "the gathered keys"),
    ("math_kernel.cuh", "mt_eval_kernel", r"const bool on = t < \*P\.ulen;", "the keys of U"),
    ("math_kernel.cuh", "mt_eval_kernel", r"const u32 pc = __popc\(__ballot_sync\(0xffffffffu, rt != MT_ABS\)\);",
     "a warp's present count"),
    ("math_kernel.cuh", "mt_eval_kernel", r"const u32 ec = __popc\(__ballot_sync\(0xffffffffu, fail\)\);",
     "a warp's failed count"),
    ("math_kernel.cuh", "mt_eval_kernel", r"if \(s_cnt\[i\]\) atomicAdd\(P\.cnt \+ i, s_cnt\[i\]\);\s*"
     r"if \(s_err\[i\]\) atomicAdd\(P\.nerr \+ i, s_err\[i\]\);", "a CTA's counts"),
    ("math_kernel.cuh", "mt_eval_kernel", r"if \(r != MT_ABS\) atomicOr\(&s_tags, 1u << r\);", "a CTA's root tags"),
    ("math_kernel.cuh", "mt_eval_kernel", r"atomicOr\(\(unsigned long long\*\)\(P\.words \+ MT_W_TAGS\), "
     r"\(unsigned long long\)s_tags\);", "the root tags combined"),
    ("math_kernel.cuh", "mt_finish_kernel", r"const u32 keys = P\.cnt\[N\.child\[0\]\], e = P\.nerr\[i\];",
     "a node's keys and failures"),
    ("math_kernel.cuh", "mt_finish_kernel", r"bool refuse = e > 0 && e < keys;", "the order-dependence refusal"),
    ("math_kernel.cuh", "mt_finish_kernel", r"all_empty = all_empty && P\.cnt\[N\.nilc\[c\]\] == 0;",
     "the COND over nil rule"),
    ("math_kernel.cuh", "mt_finish_kernel", r"if \(\(tags & \(1u << MT_INT\)\) && \(tags & \(1u << MT_FLT\)\)\) \{",
     "the promotion"),
    ("math_kernel.cuh", "mt_write_kernel", r"if \(t < \(P\.range \? P\.nrange : 1\)\) \{", "the constant's entries"),
    ("math_kernel.cuh", "mt_write_kernel", r"\} else if \(kind == 1 && t < \*P\.ulen && P\.flag\[t\]\) \{",
     "the root's entries"),
    ("dgx_api.cu", "gb_grid", r"return \(unsigned\)std::max<uint64_t>\(1, \(n \+ 255\) / 256\);", "gb_grid"),
    ("dgx_api.cu", "mt_run", r"mt_check_kernel<<<gb_grid\(cap \+ \(d_range \? nrange : 0\)\), 256, 0, l->stream>>>",
     "the check's grid"),
    ("dgx_api.cu", "mt_run", r"mt_eval_kernel<<<gb_grid\(cap\), 256, 0, l->stream>>>", "the eval's grid"),
    ("dgx_api.cu", "mt_run", r"scan_u64_kernel<<<\(unsigned\)tiles, EN_NT, 0, l->stream>>>\(P\.flag, P\.pos, ulen, c1,",
     "the root scan"),
    ("dgx_api.cu", "mt_run", r"mt_write_kernel<<<gb_grid\(std::max<uint64_t>\(cap, d_range \? nrange : 1\)\), 256, 0, "
     r"l->stream>>>", "the write's grid"),
    ("dgx_api.cu", "mt_run", r"h_cap_off\[j \+ 1\] = h_cap_off\[j\] \+ L\.n;", "the rooms' offsets"),
]


def read_constants() -> dict:
    text = {f: _src(f) for f in ("dgx_api.cu", "trigram_kernel.cuh", "math_kernel.cuh", "compressed_kernel.cuh",
                                 "encode_kernel.cuh", "dgx.h")}
    tk, mk, ck, enc, h = (text[f] for f in ("trigram_kernel.cuh", "math_kernel.cuh", "compressed_kernel.cuh",
                                            "encode_kernel.cuh", "dgx.h"))
    K = {"TG_NT": int(_one(r"constexpr int TG_NT = (\d+);", tk, "TG_NT").group(1))}
    m = _one(r"constexpr int CP_NT = (\d+), CP_VT = (\d+), CP_TILE = CP_NT \* CP_VT;", ck, "CP_TILE")
    K["CP_NT"], K["CP_VT"] = int(m.group(1)), int(m.group(2))
    m = _one(r"constexpr int EN_NT = (\d+), EN_VT = (\d+), EN_TILE = EN_NT \* EN_VT;", enc, "EN_TILE")
    K["EN_TILE"] = int(m.group(1)) * int(m.group(2))
    K["MAX_NODES"] = int(_one(r"#define DGX_MATH_MAX_NODES (\d+)", h, "DGX_MATH_MAX_NODES").group(1))
    K["MAX_LEAVES"] = int(_one(r"#define DGX_MATH_MAX_LEAVES (\d+)", h, "DGX_MATH_MAX_LEAVES").group(1))
    m = _one(r"constexpr int MT_MAX_NODES = (\d+), MT_MAX_LEAVES = (\d+);", mk, "MT_MAX_NODES")
    if (int(m.group(1)), int(m.group(2))) != (K["MAX_NODES"], K["MAX_LEAVES"]):
        raise ValueError("the kernel's program limits changed: they are not dgx.h's, restate it in the tree model")
    grids = {}
    for fn, kern in (("trigram_kernel.cuh", "tg_gather_kernel"), ("trigram_kernel.cuh", "tg_eval_kernel"),
                     ("math_kernel.cuh", "mt_check_kernel"), ("math_kernel.cuh", "mt_gather_kernel"),
                     ("math_kernel.cuh", "mt_eval_kernel"), ("math_kernel.cuh", "mt_write_kernel")):
        grids[kern] = int(_one(r"__global__ void __launch_bounds__\((\d+)\) " + kern, text[fn],
                               f"{kern}'s CTA").group(1))
    if set(grids.values()) != {256}:
        raise ValueError("a 256-thread grid changed: restate it in the tree model (tests/tree_geometry.py)")
    K["GRID_NT"] = 256
    K.update({"TG_MAX_NODES": tp.K["MAX_NODES"], "TG_MAX_LEAVES": tp.K["MAX_LEAVES"], "TG_MAX_REFS": tp.K["MAX_REFS"],
              "TG_MAX_DEPTH": tp.K["MAX_DEPTH"]})
    for fn, func, pat, what in STATEMENTS:
        _one(pat, _fn(func, text[fn]) if func else text[fn], what)
    return K


K = read_constants()
TG_NT, CP_TILE, EN_TILE, NT = K["TG_NT"], K["CP_NT"] * K["CP_VT"], K["EN_TILE"], K["GRID_NT"]

MUTANTS = {
    # regexp()
    "chunk carry dropped": "tg_leaves_kernel writes drive_off[i] = ex: every chunk of TG_NT rows restarts at 0",
    "gather takes the first equal offset": "tg_gather_kernel's row is the first of the rows sharing its offset "
                                           "(an empty row in front of it)",
    "empty OR is true": "tg_eval_kernel reads an OR without children as a hit",
    "one level closed per leaf": "tg_eval_kernel's close loop closes one node, then reads the next entry",
    "keep past ncand": "tg_eval_kernel evaluates the slots past ncand (stale candidates) instead of writing keep = 0",
    # math()
    "tags of CTA 0 only": "mt_eval_kernel's root tag set taken from CTA 0 alone (the promotion misses later CTAs)",
    "refusal per CTA": "mt_finish_kernel's refusals decided from one CTA's counts instead of the global ones",
    "keys of the node": "mt_finish_kernel's keys read as the node's own present count, not its first child's",
    "room-0 leaf owns threads": "a thread's leaf is the first of the leaves that share its room's offset",
    "range fill over cap": "mt_write_kernel's grid over cap threads: a constant over a wider range loses entries",
    "root over cap": "the root's flags, scan and write run over cap slots instead of ulen (stale keys written)",
}

# ---- events -----------------------------------------------------------------------------------------------------------

NDRIVE = (1023, 1024, 1025, 2048, 2049, 3073)
NCAND = (2047, 2048, 2049, 4096, 4097)
CAP_EDGES = ("256k - 1", "256k", "256k + 1")
ULEN = (31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 4097)
NRANGE = (0, 1, 255, 256, 257, 2049)
EVENTS = {
    "tg leaves: a second stride of the leaf table", "tg leaves: only leaves at index TG_NT or above referenced",
    "tg mut: a value flag only at index TG_NT", "tg mut: a value flag only at the last of nmut > TG_NT",
    "tg mut: nmut > TG_NT without a value flag",
    "tg drive: a carry into a chunk", "tg drive: a chunk whose rows are all empty",
    "tg drive: the only non-empty driving row is TG_NT", "tg drive: an AND driven through an OR of more than TG_NT leaves",
    "tg gather: empty driving rows first", "tg gather: empty driving rows last",
    "tg gather: a run of empty driving rows", "tg gather: a row boundary on a CTA edge",
    "tg gather: dcap above drive_off[nd] by a CTA or more", "tg gather: positions in 3 or more CTAs",
    "tg after: a cut at a leaf's first uid", "tg after: a cut at a leaf's last uid",
    "tg path: the gather is the result", "tg path: eval without a merge", "tg path: merge then eval",
    "tg path: all-OR merge, out_cap the root bound", "tg path: out_cap one short of the root bound",
    "tg eval: opening a node", "tg eval: an OR without children", "tg eval: a leaf hit", "tg eval: a leaf miss",
    "tg eval: the close loop goes on to a next child", "tg eval: the walk closes at the root",
    "tg eval: one leaf closes 2 levels", "tg eval: one leaf closes 3 to 31 levels", "tg eval: one leaf closes 32 levels",
    "tg eval: threads past ncand", "tg eval: an AND decided by a miss", "tg eval: an OR decided by a hit",
    "tg truth: leaf i holds u + 1 iff bit i of u is set",
    "tg compact: kept at a tile's first and last slot only", "tg compact: every candidate kept",
    "tg compact: no candidate kept", "tg compact: dcap of 2 or more tiles",
    "mt space: a room of 0 first", "mt space: a room of 0 last", "mt space: rooms of 0 between leaves",
    "mt space: a count word below the room", "mt space: range checks from cap_total on",
    "mt plan: a general map holding 2^64 - 1", "mt plan: a {MaxUint64: v} constant", "mt plan: a {0: v} aggregate",
    "mt plan: a scalar subtree inside a vector node", "mt plan: 64 nodes", "mt plan: 16 general leaves",
    "mt plan: a nil leaf", "mt plan: an empty leaf",
    "mt eval: U in 3 or more CTAs", "mt eval: a node's failures in 3 CTAs", "mt eval: a failure in lane 0 of the last CTA",
    "mt eval: a failure in lane 31 of the last CTA", "mt eval: half or more of a node's keys fail",
    "mt eval: a unary node fails", "mt eval: a compare node fails", "mt eval: a cond node fails",
    "mt finish: refused, some keys fail", "mt finish: not refused, every key fails in 3 CTAs",
    "mt finish: COND over a binary node whose only key is in the last CTA", "mt finish: refused, COND over nil",
    "mt finish: promotion from the last CTA only", "mt finish: promotion from CTA 0 only",
    "mt finish: floats below the root, no promotion", "mt finish: ERR_CAP",
    "mt scan: root keys absent on both sides of a 32, 256 and 2048 edge", "mt scan: 3 tiles over ulen",
    "mt check: a range descending only at its last pair, on a CTA's first thread",
    "mt write: a constant over a range past one CTA", "mt write: a constant over an empty range",
} | {f"tg drive: ndrive = {n}" for n in NDRIVE} \
  | {f"tg leaves: npacks = {n} of more than TG_NT leaves" for n in (1023, 1024, 1025)} \
  | {f"tg compact: ncand = {n}" for n in NCAND} \
  | {f"mt eval: ulen = {n}" for n in ULEN} \
  | {f"mt write: nrange = {n}" for n in NRANGE} \
  | {f"mt space: cap_total = {d}" for d in CAP_EDGES}


def _add(ev, name):
    if name not in EVENTS:
        raise KeyError(f"event {name!r} is not registered in tree_geometry.EVENTS")
    ev.add(name)


def _lower_bound(a, n, x):
    """lower_bound_g restated: the first index in [0, n) whose value is not below x (binary search, as the device
    does it even when a mutant leaves a unsorted)."""
    lo, hi = 0, n
    while lo < hi:
        mid = (lo + hi) // 2
        if a[mid] < x:
            lo = mid + 1
        else:
            hi = mid
    return lo


def _grid(n):
    """gb_grid(n) CTAs of 256 threads, as threads."""
    return max(1, -(-n // NT)) * NT


# ---- regexp() ---------------------------------------------------------------------------------------------------------

TgCall = namedtuple("TgCall", "form out_cap")     # form "host" / "dev"; out_cap: "spare", "exact" or "short"
TgCase = namedtuple("TgCase", "tree leaves after")
TgFix = namedtuple("TgFix", "name cases calls events kills")
TgOut = namedtuple("TgOut", "rc sync n out launches")   # out: the values written (None: nothing written)


def tg_children(tree, lb, bound, i):
    """dgx_api.cu TgBuild::children: leaves then subs, an AND's sorted (stably) by bound."""
    op, ls, subs = tree[i]
    ch = [(lb[j], ("leaf", j)) for j in ls] + [(bound[s], ("node", s)) for s in subs]
    return sorted(ch, key=lambda c: c[0]) if op == QAND else ch


def tg_program(tree, lb, bound):
    """TgBuild::emit: the pre-order program of (w0, w1) as (kind, is_and, end, parent) / (leaf, j)."""
    prog = []

    def emit(i, parent):
        at = len(prog)
        prog.append(None)
        for _, (kind, j) in tg_children(tree, lb, bound, i):
            if kind == "node":
                emit(j, at)
            else:
                prog.append(("leaf", j))
        prog[at] = ("node", tree[i][0] == QAND, len(prog), parent)

    emit(0, None)
    return prog


def _member(row, x):
    """tg_member: a binary search in the leaf's row (a set lookup: the rows are ascending and distinct)."""
    return x in row


def tg_walk(prog, rows, x, mut, ev):
    """tg_eval_kernel's walk for one candidate: keep."""
    cur, pc, r = 0, 1, False
    for _ in range(4 * len(prog) + 4):
        if pc >= len(prog):          # only a mutant runs off the program
            return r
        e = prog[pc]
        if e[0] == "node":
            _add(ev, "tg eval: opening a node")
            if e[2] != pc + 1:
                cur, pc = pc, pc + 1
                continue
            _add(ev, "tg eval: an OR without children")
            r = "empty OR is true" in mut
            pc = e[2]
        else:
            r = _member(rows[e[1]], x)
            _add(ev, "tg eval: a leaf hit" if r else "tg eval: a leaf miss")
            pc += 1
        closed = 0
        while True:
            f = prog[cur]
            is_and, end, parent = f[1], f[2], f[3]
            if is_and == r and pc != end:
                _add(ev, "tg eval: the close loop goes on to a next child")
                break
            if pc != end:
                _add(ev, "tg eval: an AND decided by a miss" if is_and else "tg eval: an OR decided by a hit")
            pc = end
            closed += 1
            if parent is None:
                _add(ev, "tg eval: the walk closes at the root")
                _closed(ev, closed)
                return r
            cur = parent
            if "one level closed per leaf" in mut:
                break
        _closed(ev, closed)
    if mut:
        return True                  # a mutant's walk that never closes the root: a garbage keep
    raise AssertionError("the walk does not end")


def _closed(ev, k):
    if k == 2:
        _add(ev, "tg eval: one leaf closes 2 levels")
    elif 3 <= k <= 31:
        _add(ev, "tg eval: one leaf closes 3 to 31 levels")
    elif k == 32:
        _add(ev, "tg eval: one leaf closes 32 levels")


def tg_cap(p, call):
    """The call's out_cap: the root's bound with 5 spare slots, exactly the bound, or one short of it."""
    if p.rc != OK:
        return 0
    return p.root_bound + {"spare": 5, "exact": 0, "short": -1}[call.out_cap]


def tg_npacks(leaves):
    n = sum(1 for lf in leaves if lf[0] == "pack")
    assert all(lf[0] == "pack" for lf in leaves[:n]), "pack leaves come first (the ABI's numbering)"
    return n


def tg_run(case: TgCase, call: TgCall, mut=frozenset(), ev=None) -> TgOut:
    """One dgx_trigram_query (host form) or dgx_dev_trigram_query call: rc, the lane's sync code (dev form), the
    length, the values written to out and the launches."""
    ev = set() if ev is None else ev
    tree, leaves, after = case
    npacks, nleaves = tg_npacks(leaves), len(leaves)
    lb = [gt.leaf_bound(lf) for lf in leaves]
    p0 = tp.plan(tree, lb)
    cap = tg_cap(p0, call)
    if p0.rc != OK:
        return TgOut(p0.rc, None, None, None, 0)
    flags = np.concatenate([lf[2][1] for lf in leaves[:npacks] if lf[2] is not None] or [np.zeros(0, np.uint8)])
    value = np.flatnonzero(flags & MUT_VALUE)
    if flags.size > TG_NT:
        if value.size == 0:
            _add(ev, "tg mut: nmut > TG_NT without a value flag")
        elif value.tolist() == [TG_NT]:
            _add(ev, "tg mut: a value flag only at index TG_NT")
        elif value.tolist() == [flags.size - 1]:
            _add(ev, "tg mut: a value flag only at the last of nmut > TG_NT")
    if call.form == "host" and value.size:
        return TgOut(ERR_ARG, None, None, None, 0)
    p = tp.plan(tree, lb, cap)
    if p.rc != OK:
        _add(ev, "tg path: out_cap one short of the root bound")
        return TgOut(p.rc, None, None, None, 0)
    if p.root_bound == 0:
        return TgOut(OK, OK if call.form == "dev" else None, 0, np.zeros(0, np.uint64), 0)
    bad = call.form == "dev" and value.size > 0
    # tg_leaves_kernel: the leaf table, TG_NT leaves per stride, packs below npacks
    rows = []
    for i in range(nleaves):
        if i >= TG_NT:
            _add(ev, "tg leaves: a second stride of the leaf table")
        r = gt.leaf_set(leaves[i], after) if i < npacks else np.asarray(leaves[i][1], np.uint64)
        rows.append(np.zeros(0, np.uint64) if bad else np.asarray(r, np.uint64))
    if nleaves > TG_NT and npacks in (1023, 1024, 1025):
        _add(ev, f"tg leaves: npacks = {npacks} of more than TG_NT leaves")
    refs = {j for t in tree for j in t[1]}
    if refs and min(refs) >= TG_NT:
        _add(ev, "tg leaves: only leaves at index TG_NT or above referenced")
    for lf in leaves[:npacks]:
        if lf[1] is not None and len(lf[1]) and after:
            if after == int(lf[1][0]):
                _add(ev, "tg after: a cut at a leaf's first uid")
            if after == int(lf[1][-1]):
                _add(ev, "tg after: a cut at a leaf's last uid")
    drive, nd, dcap = p.drive, len(p.drive), p.dcap
    if tree[0][0] == QAND and nd > TG_NT:
        _add(ev, "tg drive: an AND driven through an OR of more than TG_NT leaves")
    if npacks == 0 and 1 <= nleaves <= 5 and all(
            np.array_equal(rows[i], np.flatnonzero((np.arange(2 ** nleaves) >> i) & 1) + 1) for i in range(nleaves)):
        _add(ev, "tg truth: leaf i holds u + 1 iff bit i of u is set")
    if nd in NDRIVE:
        _add(ev, f"tg drive: ndrive = {nd}")
    # the driving rows' offsets: a block scan per TG_NT rows, each chunk's total carried into the next
    lens = [rows[d].size for d in drive]
    off, carry = [], 0
    for b in range(0, nd, TG_NT):
        chunk = lens[b:b + TG_NT]
        ex = np.concatenate([[0], np.cumsum(chunk)[:-1]]).astype(np.int64)
        if b and carry:
            _add(ev, "tg drive: a carry into a chunk")
        if b and not any(chunk):
            _add(ev, "tg drive: a chunk whose rows are all empty")
        off += [int(e) + (0 if "chunk carry dropped" in mut else carry) for e in ex]
        carry += int(sum(chunk))
    off.append(carry)
    nonempty = [k for k in range(nd) if lens[k]]
    if nonempty == [TG_NT]:
        _add(ev, "tg drive: the only non-empty driving row is TG_NT")
    if nd >= 2 and lens[0] == 0:
        _add(ev, "tg gather: empty driving rows first")
    if nd >= 2 and lens[-1] == 0:
        _add(ev, "tg gather: empty driving rows last")
    later = np.flip(np.cumsum(np.flip(np.asarray(lens + [0], np.int64)))) if nd else np.zeros(1, np.int64)
    if any(lens[k] == 0 and lens[k + 1] == 0 and lens[k - 1] and later[k + 2] for k in range(1, nd - 1)):
        _add(ev, "tg gather: a run of empty driving rows")
    if any(o % NT == 0 and 0 < o < carry for o in off[1:nd]):
        _add(ev, "tg gather: a row boundary on a CTA edge")
    if dcap >= carry + NT:
        _add(ev, "tg gather: dcap above drive_off[nd] by a CTA or more")
    # tg_gather_kernel: thread t < min(dcap, drive_off[nd]) copies position t of its row
    m = min(dcap, off[nd])
    if m > 2 * NT:
        _add(ev, "tg gather: positions in 3 or more CTAs")
    gathered = np.zeros(m, np.uint64)
    for t in range(m):
        d = _lower_bound(off, nd + 1, t + 1) - 1
        if "gather takes the first equal offset" in mut:
            d = off.index(off[d])
        row, k = rows[drive[d]], t - off[d]
        gathered[t] = row[k] if 0 <= k < row.size else POISON
    merge = nd >= 2
    launches = (tp.K["ROWS"] if npacks else 0) + 2
    if merge:
        launches += tp.K["MERGE"] + tree_launches(-(-dcap // tp.K["XM_T"]))
        cand = np.unique(gathered)   # merge_matrix_impl: the union of the sorted rows
    else:
        cand = gathered
    if p.all_or:
        if not merge:
            _add(ev, "tg path: the gather is the result")
        elif call.out_cap == "exact":
            _add(ev, "tg path: all-OR merge, out_cap the root bound")
        out = cand
    else:
        _add(ev, "tg path: merge then eval" if merge else "tg path: eval without a merge")
        prog = tg_program(tree, lb, p.bound)
        sets = [set(r.tolist()) for r in rows]
        ncand = cand.size
        keep = np.zeros(dcap, bool)
        for t in range(dcap):
            if t >= ncand:
                _add(ev, "tg eval: threads past ncand")
                keep[t] = "keep past ncand" in mut
                continue
            keep[t] = tg_walk(prog, sets, int(cand[t]), mut, ev)
        slots = np.concatenate([cand, np.full(dcap - ncand, POISON, np.uint64)])
        # compact_kernel: tiles of CP_TILE slots over dcap, the kept ones in order
        tiles = -(-dcap // CP_TILE)
        if tiles >= 2:
            _add(ev, "tg compact: dcap of 2 or more tiles")
        kk = keep[:ncand]
        if ncand in NCAND:
            _add(ev, f"tg compact: ncand = {ncand}")
        if ncand > 2:
            edges = {i for k in range(tiles) for i in (k * CP_TILE, k * CP_TILE + CP_TILE - 1) if i < ncand}
            if kk.all():
                _add(ev, "tg compact: every candidate kept")
            elif not kk.any():
                _add(ev, "tg compact: no candidate kept")
            elif set(np.flatnonzero(kk).tolist()) == edges:
                _add(ev, "tg compact: kept at a tile's first and last slot only")
        out = slots[keep]
        launches += 2
    return TgOut(OK, (ERR_ARG if bad else OK) if call.form == "dev" else None, int(out.size), out, launches)


def tg_oracle(case: TgCase):
    """trigram_oracle's answer; the caller checks it against gen_trigram.want."""
    import trigram_oracle as tgo

    return tgo.uids_for_regex(case.tree, gt.to_oracle(case.leaves), case.after)


def tg_expected(case: TgCase, call: TgCall):
    """(rc, sync, values) a call must give: the plan's refusals, a value flag's, then the oracle's answer."""
    tree, leaves, after = case
    lb = [gt.leaf_bound(lf) for lf in leaves]
    p = tp.plan(tree, lb, tg_cap(tp.plan(tree, lb), call))
    flags = [lf[2][1] for lf in leaves if lf[0] == "pack" and lf[2] is not None]
    value = any((np.asarray(f) & MUT_VALUE).any() for f in flags)
    if p.rc == ERR_ARG or (value and call.form == "host"):
        return ERR_ARG, None, None
    if p.rc == ERR_CAP:
        return ERR_CAP, None, None
    if value:
        return OK, ERR_ARG, np.zeros(0, np.uint64)
    return OK, OK if call.form == "dev" else None, gt.want(tree, leaves, after)


# ---- regexp() fixtures ------------------------------------------------------------------------------------------------

TG_DEFAULT = (TgCall("host", "spare"), TgCall("dev", "spare"))
TG_EXACT = (TgCall("host", "exact"), TgCall("dev", "exact"), TgCall("host", "short"), TgCall("dev", "short"))


def _lst(u):
    return ("list", np.asarray(u, np.uint64))


def _pk(u, mut=None):
    u = None if u is None or not len(u) else np.asarray(u, np.uint64)
    return ("pack", u, mut, 0)


def _tg(name, cases, events, kills=(), calls=TG_DEFAULT):
    return TgFix(name, tuple(TgCase(*c) for c in cases), calls, set(events), set(kills))


def _or_rows(n, width=3, empty=()):
    """n list leaves, leaf i holding (i % width) + 1 uids of its own range (empty rows where named)."""
    return [_lst([] if i in empty else [10 * i + 1 + k for k in range(i % width + 1)]) for i in range(n)]


def _filter_of(leaves, keep_every=2, extra=0):
    """A list holding every keep_every-th value of the leaves' union, with `extra` values of its own past them."""
    u = np.unique(np.concatenate([lf[1] for lf in leaves if lf[1] is not None and len(lf[1])]))
    hi = int(u[-1]) if u.size else 0
    return _lst(np.concatenate([u[::keep_every], np.arange(hi + 1, hi + 1 + extra, dtype=np.uint64)]))


def tg_fixtures():
    fx = []
    for n in NDRIVE:
        rows = _or_rows(n)
        cases = [([(QOR, list(range(n)), [])], rows, 0)]
        evs = {f"tg drive: ndrive = {n}", "tg drive: a carry into a chunk"} if n > TG_NT else {f"tg drive: ndrive = {n}"}
        kills = {"chunk carry dropped"} if n > TG_NT else set()
        if n == 1025:
            only = [_lst([]) for _ in range(1025)]
            only[TG_NT] = _lst([5, 6, 7])
            cases.append(([(QOR, list(range(1025)), [])], only, 0))
            rows2 = _or_rows(n, width=2)
            cases.append(([(QAND, [1025], [1]), (QOR, list(range(1025)), [])], rows2 + [_filter_of(rows2, 3, 4 * n)], 0))
            evs |= {"tg drive: the only non-empty driving row is TG_NT", "tg drive: an AND driven through an OR of more than TG_NT leaves"}
        if n == 2048:
            emp = _or_rows(n, empty=set(range(TG_NT, 2048)))
            cases.append(([(QOR, list(range(n)), [])], emp, 0))
            evs.add("tg drive: a chunk whose rows are all empty")
        fx.append(_tg(f"ndrive {n}", cases, evs, kills))
    # the leaf table past TG_NT leaves, the pack / list split at 1023, 1024 and 1025
    for npk in (1023, 1024, 1025):
        nl = 1100
        leaves = []
        for i in range(nl):
            u = [7 * i + 1, 7 * i + 3]
            if i >= npk:
                leaves.append(_lst(u))
            elif i % 50 == 0:
                leaves.append(_pk(u + [7 * i + 5], (np.array([7 * i + 5], np.uint64), np.array([MUT_DEL], np.uint8))))
            else:
                leaves.append(_pk(None, (np.array(u, np.uint64), np.zeros(2, np.uint8))))
        hi = list(range(TG_NT, nl))
        cases = [([(QOR, list(range(nl)), [])], leaves, 0),
                 ([(QOR, hi[:40], [1]), (QAND, [hi[0]], [2]), (QOR, hi[::7], [])], leaves, 0)]
        fx.append(_tg(f"npacks {npk}", cases, {f"tg leaves: npacks = {npk} of more than TG_NT leaves",
                                               "tg leaves: only leaves at index TG_NT or above referenced"}))
    # nmut past TG_NT: a value flag only at index TG_NT, only at the last entry; none
    nm = TG_NT + 6
    mu = np.arange(1, nm + 1, dtype=np.uint64) * 3
    cases = []
    for at in (TG_NT, nm - 1, None):
        fl = np.zeros(nm, np.uint8)
        fl[1::5] = MUT_DEL
        if at is not None:
            fl[at] = MUT_VALUE
        cases.append(([(QOR, [0, 1], [])], [_pk(mu[::2], (mu, fl)), _lst([2, 4, 8])], 0))
    fx.append(_tg("nmut past TG_NT", cases, {"tg mut: a value flag only at index TG_NT",
                                             "tg mut: a value flag only at the last of nmut > TG_NT",
                                             "tg mut: nmut > TG_NT without a value flag"}))
    # the gather: empty rows first, last and in runs; a row boundary on a CTA edge
    lens = [0, 0, 100, 156, 0, 0, 0, 300, 1, 0, 255, 0, 0]
    rows, base = [], 1
    for ln in lens:
        rows.append(_lst(np.arange(base, base + ln, dtype=np.uint64) * 2))
        base += ln + 3
    n = len(rows)
    cases = [([(QOR, list(range(n)), [])], rows, 0),
             ([(QAND, [n], [1]), (QOR, list(range(n)), [])], rows + [_filter_of(rows, 2, extra=900)], 0)]
    fx.append(_tg("gather rows", cases, {"tg gather: empty driving rows first", "tg gather: empty driving rows last",
                                         "tg gather: a run of empty driving rows",
                                         "tg gather: a row boundary on a CTA edge"},
                  {"gather takes the first equal offset"}))
    # dcap well above the rows: DEL layers and after cuts at a leaf's first and last uid
    a = np.arange(1, 701, dtype=np.uint64) * 5
    dl = a[100:600]
    pa = _pk(a, (dl, np.full(dl.size, MUT_DEL, np.uint8)))
    b = np.arange(1, 301, dtype=np.uint64) * 7
    pb = _pk(b, (b[:200], np.full(200, MUT_DEL, np.uint8)))
    big = np.arange(1, 4000, dtype=np.uint64)
    tree = [(QAND, [2], [1]), (QOR, [0, 1], [])]
    cases = [(tree, [pa, pb, _lst(big)], 0), (tree, [pa, pb, _lst(big[big > a[0]])], int(a[0])),
             (tree, [pa, pb, _lst(big[big > b[-1]])], int(b[-1]))]
    fx.append(_tg("dcap past the rows", cases, {"tg gather: dcap above drive_off[nd] by a CTA or more",
                                                "tg after: a cut at a leaf's first uid",
                                                "tg after: a cut at a leaf's last uid", "tg eval: threads past ncand"},
                  {"keep past ncand"}))
    # the three paths
    u = np.arange(1, 3000, dtype=np.uint64)
    small, mid = _lst(u[::7]), _lst(u[::3])
    cases = [([(QAND, [0, 1], [])], [small, mid], 0),
             ([(QOR, [], [1]), (QOR, [0], [])], [mid, small], 0),
             ([(QOR, [0, 1], [])], [small, mid], 0)]
    fx.append(_tg("paths", cases, {"tg path: eval without a merge", "tg path: the gather is the result",
                                   "tg path: all-OR merge, out_cap the root bound",
                                   "tg path: out_cap one short of the root bound"}, calls=TG_EXACT))
    fx.append(_tg_truth())
    fx.append(_tg_depth32())
    # compaction: ncand at the tile edges, kept at the edges only, all, none
    for n in NCAND:
        h = (n + 1) // 2
        rows = [_lst(np.arange(1, h + 1, dtype=np.uint64) * 2), _lst(np.arange(1, n - h + 1, dtype=np.uint64) * 2 + 1)]
        cand = np.arange(2, n + 2, dtype=np.uint64)
        pad = np.arange(10 * n, 10 * n + n + 8, dtype=np.uint64)
        edges = cand[[i for k in range(3) for i in (k * CP_TILE, k * CP_TILE + CP_TILE - 1) if i < n]]
        cases = [([(QAND, [2], [1]), (QOR, [0, 1], [])], rows + [_lst(np.union1d(sel, pad))], 0)
                 for sel in (edges, cand, np.zeros(0, np.uint64))]
        fx.append(_tg(f"compact ncand {n}", cases, {f"tg compact: ncand = {n}",
                                                    "tg compact: kept at a tile's first and last slot only",
                                                    "tg compact: every candidate kept",
                                                    "tg compact: no candidate kept"}))
    return fx


def _shapes(n):
    """Every rooted ordered tree of n nodes as parent lists in pre-order."""
    if n == 1:
        return [[None]]
    out = []
    for s in _shapes(n - 1):
        # attach node n-1 to any node on the rightmost path (keeps pre-order numbering)
        path, j = [], n - 2
        while j is not None:
            path.append(j)
            j = s[j]
        out += [s + [p] for p in path]
    return out


def _tg_truth():
    """k <= 5 leaves over 2^k uids, uid u + 1 in leaf i iff bit i of u: every tree shape of up to 4 nodes under every
    AND / OR labelling, leaves drawn from a seeded generator (empty ORs and shared leaves included)."""
    rng = np.random.default_rng(4242)
    cases = []
    for nn in range(1, 5):
        for par in _shapes(nn):
            for ops in itertools.product((QAND, QOR), repeat=nn):
                for rep in range(2):
                    k = int(rng.integers(1, 6))
                    u = np.arange(2 ** k, dtype=np.uint64)
                    leaves = [_lst(u[(u >> np.uint64(i)) & np.uint64(1) == 1] + np.uint64(1)) for i in range(k)]
                    tree = []
                    for i in range(nn):
                        subs = [j for j in range(nn) if par[j] == i]
                        ls = [int(x) for x in rng.integers(0, k, int(rng.integers(0, 3)))]
                        if ops[i] == QAND and not ls and not subs:
                            ls = [int(rng.integers(0, k))]
                        if rep == 1 and ops[i] == QOR and not subs:
                            ls = []                                  # an empty OR
                        tree.append((ops[i], ls, subs))
                    cases.append((tree, leaves, 0))
    return _tg("truth table", cases, {"tg truth: leaf i holds u + 1 iff bit i of u is set", "tg eval: an OR without children",
                                      "tg eval: one leaf closes 2 levels", "tg eval: one leaf closes 3 to 31 levels"},
               {"empty OR is true", "one level closed per leaf"})


def _tg_depth32():
    """Chains of 32 nodes, AND first and OR first: node i holds leaf i and sub i + 1, the last node leaves 31 and 32.
    The AND levels' leaves and leaf 32 hold 1 .. 200, the OR levels' 10 values of their own, so every AND's leaf sorts
    before its sub and a value of 1 .. 200 hits every AND leaf, misses every OR leaf and reaches leaf 32, which closes
    all 32 levels at once."""
    cases = []
    every = np.arange(1, 201, dtype=np.uint64)
    for first in (QAND, QOR):
        ops = [first if i % 2 == 0 else (QOR if first == QAND else QAND) for i in range(32)]
        leaves = [_lst(every) if i == 32 or ops[i] == QAND else _lst(np.arange(10, dtype=np.uint64) + 1000 + 10 * i)
                  for i in range(33)]
        tree = [(ops[i], [i], [i + 1]) if i < 31 else (ops[i], [31, 32], []) for i in range(32)]
        cases.append((tree, leaves, 0))
    # AND first, each AND level's leaf missing one value, and a last root leaf (sorted after the chain, its bound
    # larger) holding every value: a value that fails inside the chain must not reach it
    ops = [QAND if i % 2 == 0 else QOR for i in range(32)]
    leaves = [_lst(np.delete(every, i)) if i < 32 and ops[i] == QAND else
              _lst(np.arange(10, dtype=np.uint64) + 1000 + 10 * i) for i in range(32)]
    leaves += [_lst(every), _lst(np.arange(1, 400, dtype=np.uint64))]
    tree = [(ops[i], [i], [i + 1]) if i < 31 else (ops[i], [31, 32], []) for i in range(32)]
    tree[0] = (QAND, [0, 33], [1])
    cases.append((tree, leaves, 0))
    return _tg("depth 32", cases, {"tg eval: one leaf closes 32 levels"}, {"one level closed per leaf"})


# ---- math() -----------------------------------------------------------------------------------------------------------

MtCall = namedtuple("MtCall", "form out_cap room")   # out_cap None: enough room; room: spare entries per leaf (dev)
MtCase = namedtuple("MtCase", "tree maps range")
MtFix = namedtuple("MtFix", "name cases calls events kills")
MtOut = namedtuple("MtOut", "rc sync info keys words tags launches")
INT, FLT, BOOL, NIL = gm.INT, gm.FLT, gm.BOOL, gm.NIL
ABS = 0
MK_CONST, MK_NIL, MK_EMPTY, MK_MAP0, MK_VEC = range(5)
UN_OPS, CMP_OPS, BIN_OPS = set(gm.UN), set(gm.CMP), set(gm.BIN)


def mt_nodes(tree):
    """The post-order program of algo.math_program: (op, children, tree) per node; variables keep their names."""
    nodes = []

    def walk(t):
        kids = [walk(c) for c in t[1:]] if t[0] not in ("var", "const") else []
        nodes.append((t[0], kids, t))
        return len(nodes) - 1

    walk(tree)
    return nodes


def mt_leaf(m):
    """(keys, words, tags) lists and nil of one map, as algo.math_leaf_arrays gives them to the library."""
    if m is None:
        return [], [], [], True
    if len(m) == 3:
        return [int(x) for x in m[0]], [int(x) for x in np.asarray(m[1], np.uint64)], [int(x) for x in m[2]], False
    v = np.ascontiguousarray(m[1])
    t = FLT if v.dtype == np.float64 else INT
    return [int(x) for x in m[0]], [int(x) for x in v.view(np.uint64)], [t] * len(m[0]), False


def mt_room(case: MtCase, call: MtCall):
    """Every leaf's (name, entries, room) in leaf order; the dev form's spare room sits past the count."""
    names = []
    for op, _, t in mt_nodes(case.tree):
        if op == "var" and t[1] not in names:
            names.append(t[1])
    out = []
    for nm in names:
        k, _, _, nil = mt_leaf(case.maps.get(nm))
        n = 0 if nil else len(k)
        extra = 0 if nil or call.form == "host" else (call.room.get(nm, 0) if isinstance(call.room, dict)
                                                      else call.room or 0)
        out.append((nm, n, n + extra))
    return out


def _scalar(t, maps):
    """A scalar node's kind and value from gen_math's formula: (kind, (tag, word)); None where it is refused."""
    try:
        r = gm._node(t, maps)
    except gm.Refused:
        return None
    if r[0] == "const":
        return MK_CONST, r[1]
    if r[0] == "nil":
        return MK_NIL, (ABS, 0)
    if not r[1]:
        return MK_EMPTY, (ABS, 0)
    assert list(r[1]) == [0], "a scalar node's keys lie within {0}"
    return MK_MAP0, r[1][0]


def _val(tw):
    return None if tw is None or tw[0] == ABS else tw


def mt_run(case: MtCase, call: MtCall, mut=frozenset(), ev=None) -> MtOut:
    """One dgx_math_eval (host form) or dgx_dev_math_eval call: rc, sync code (dev form), the info word (None when
    untouched), the entries written and the launches."""
    ev = set() if ev is None else ev
    tree, maps, rng_u = case
    nodes = mt_nodes(tree)
    rooms = mt_room(case, call)
    cap = sum(r[2] for r in rooms)
    launches = mp.K["FRONT"] + (mp.K["MERGE"] + tree_launches(-(-cap // mp.K["XM_T"])) if cap else 0) + mp.K["BACK"]
    dev = call.form == "dev"

    def refused():
        return MtOut(OK if dev else ERR_ARG, ERR_ARG if dev else None, None, None, None, None, launches if dev else 0)

    # the check / gather thread space over the rooms
    off = np.concatenate([[0], np.cumsum([r[2] for r in rooms])]).astype(np.int64).tolist()
    rs = [r[2] for r in rooms]
    if rs and rs[0] == 0 and any(rs):
        _add(ev, "mt space: a room of 0 first")
    if rs and rs[-1] == 0 and any(rs):
        _add(ev, "mt space: a room of 0 last")
    if any(rs[j] == 0 and any(rs[:j]) and any(rs[j + 1:]) for j in range(len(rs))):
        _add(ev, "mt space: rooms of 0 between leaves")
    if any(r[1] < r[2] for r in rooms):
        _add(ev, "mt space: a count word below the room")
    if cap > 1 and cap % NT in (NT - 1, 0, 1):
        _add(ev, f"mt space: cap_total = {CAP_EDGES[(cap % NT + 1) % NT]}")
    leaf = {}
    seen = {nm: set() for nm, _, _ in rooms}
    for t in range(cap):
        j = _lower_bound(off, len(off), t + 1) - 1          # the last leaf whose room starts at or before t
        if "room-0 leaf owns threads" in mut:
            j = off.index(off[j])
        nm, n, room = rooms[j]
        i = t - off[j]
        if i < n and i < room:
            seen[nm].add(i)
    bad = False
    for nm, n, _ in rooms:
        k, w, tg, nil = mt_leaf(maps.get(nm))
        keep = sorted(seen[nm])
        leaf[nm] = (k, w, tg, nil, keep)
        if any(k[i - 1] >= k[i] for i in keep if i > 0) or any(not INT <= tg[i] <= NIL for i in keep):
            bad = True
    if rng_u is not None:
        r = [int(x) for x in rng_u]
        if len(r) and cap:
            _add(ev, "mt space: range checks from cap_total on")
        for i in range(1, len(r)):
            if r[i - 1] >= r[i]:
                bad = True
                if i == len(r) - 1 and (cap + i) % NT == 0:
                    _add(ev, "mt check: a range descending only at its last pair, on a CTA's first thread")
    # mt_plan_kernel: the leaf kinds, then the scalar nodes (gen_math's values) and the vector nodes' sources
    kinds, rooms_n = {}, {nm: n for nm, n, _ in rooms}
    for nm, n, _ in rooms:
        k, w, tg, nil, _ = leaf[nm]
        if nil:
            kinds[nm] = MK_NIL
            _add(ev, "mt plan: a nil leaf")
        elif n == 0:
            kinds[nm] = MK_EMPTY
            _add(ev, "mt plan: an empty leaf")
        elif n == 1 and k[0] in (0, U64):
            kinds[nm] = MK_MAP0 if k[0] == 0 else MK_NIL if tg[0] == NIL else MK_CONST
            _add(ev, "mt plan: a {0: v} aggregate" if k[0] == 0 else "mt plan: a {MaxUint64: v} constant")
        elif k[0] == 0:
            bad = True
            kinds[nm] = MK_EMPTY
        else:
            kinds[nm] = MK_VEC
            if U64 in k:
                _add(ev, "mt plan: a general map holding 2^64 - 1")
    if bad:
        return refused()
    if len(nodes) == K["MAX_NODES"]:
        _add(ev, "mt plan: 64 nodes")
    if sum(1 for v in kinds.values() if v == MK_VEC) == K["MAX_LEAVES"]:
        _add(ev, "mt plan: 16 general leaves")
    kind, val = [], []
    for i, (op, kids, t) in enumerate(nodes):
        if op == "var":
            vec = kinds[t[1]] == MK_VEC
        elif op == "const":
            vec = False
        elif op in BIN_OPS:
            vec = kind[kids[0]] == MK_VEC or kind[kids[1]] == MK_VEC
        else:
            vec = kind[kids[0]] == MK_VEC
        if vec:
            kind.append(MK_VEC)
            val.append(None)
            if op != "var" and any(kind[c] != MK_VEC and nodes[c][0] != "const" for c in kids):
                _add(ev, "mt plan: a scalar subtree inside a vector node")
            continue
        s = _scalar(t, maps)
        if s is None:
            return refused()
        kind.append(s[0])
        val.append(s[1])
    # the key union: the general leaves' gathered keys
    U = sorted({leaf[nm][0][i] for nm in leaf if kinds[nm] == MK_VEC for i in leaf[nm][4]})
    ulen = len(U)
    if ulen in ULEN:
        _add(ev, f"mt eval: ulen = {ulen}")
    if ulen > 2 * NT:
        _add(ev, "mt eval: U in 3 or more CTAs")
    index = {nm: {leaf[nm][0][i]: i for i in range(rooms_n[nm])} for nm in leaf}
    nct = max(1, -(-ulen // NT))
    nn = len(nodes)
    cnt = np.zeros((nn, nct), np.int64)
    err = np.zeros((nn, nct), np.int64)
    errs_at = [[] for _ in range(nn)]
    res = [[None] * ulen for _ in range(nn)]

    def src(c, ti):
        """A vector node's child c at key index ti: its per-key value, a broadcast constant, or missing."""
        if kind[c] == MK_VEC:
            return res[c][ti]
        return None

    for i, (op, kids, t) in enumerate(nodes):
        if kind[i] != MK_VEC:
            continue
        for ti, u in enumerate(U):
            r, fail = None, False
            if op == "var":
                j = index[t[1]].get(u)      # lower_bound over the leaf's counted keys, found or not
                if j is not None:
                    k, w, tg, _, _ = leaf[t[1]]
                    r = (tg[j], w[j])
            elif op in BIN_OPS:
                A, B = kids
                lconv = kind[A] == MK_MAP0
                rconv = not lconv and kind[B] == MK_MAP0
                ca = src(A, ti) if kind[A] == MK_VEC else (val[A] if kind[A] == MK_CONST or
                                                          (lconv and val[A][0] != NIL) else None)
                cb = src(B, ti) if kind[B] == MK_VEC else (val[B] if kind[B] == MK_CONST or
                                                          (rconv and val[B][0] != NIL) else None)
                present = (kind[A] == MK_VEC and _val(ca)) or (kind[B] == MK_VEC and _val(cb))
                if present:
                    r = gm._bin(op, _val(ca), _val(cb))
            else:
                a = src(kids[0], ti)
                if a is not None:
                    if op in UN_OPS:
                        r = gm._un(op, a)
                    elif op in CMP_OPS:
                        B = kids[1]
                        b = src(B, ti) if kind[B] == MK_VEC else val[B] if kind[B] == MK_CONST else None
                        r = gm._cmp(op, a, b)
                    else:  # cond
                        if a[0] != BOOL:
                            r = None
                        else:
                            X = kids[1] if a[1] else kids[2]
                            x = src(X, ti) if kind[X] == MK_VEC else val[X] if kind[X] == MK_CONST else None
                            r = x if x is not None else (NIL, 0)
                    fail = r is None
            res[i][ti] = r
            c = ti // NT
            if r is not None:
                cnt[i, c] += 1
            if fail:
                err[i, c] += 1
                errs_at[i].append(ti)
        if err[i].sum():
            _add(ev, {**{o: "mt eval: a unary node fails" for o in UN_OPS},
                      **{o: "mt eval: a compare node fails" for o in CMP_OPS}}.get(op, "mt eval: a cond node fails"))
            if (err[i] > 0).sum() >= 3:
                _add(ev, "mt eval: a node's failures in 3 CTAs")
            if nct >= 3 and errs_at[i] == [(nct - 1) * NT]:
                _add(ev, "mt eval: a failure in lane 0 of the last CTA")
            if nct >= 3 and errs_at[i] == [(nct - 1) * NT + 31]:
                _add(ev, "mt eval: a failure in lane 31 of the last CTA")
            if 2 * err[i].sum() >= cnt[kids[0]].sum() > err[i].sum() and nct >= 3:
                _add(ev, "mt eval: half or more of a node's keys fail")
    # mt_finish_kernel: the refusals from the summed counts
    for i, (op, kids, t) in enumerate(nodes):
        if kind[i] != MK_VEC or op == "var" or op in BIN_OPS:
            continue
        keys_of = cnt[i] if "keys of the node" in mut else cnt[kids[0]]
        if "refusal per CTA" in mut:
            refuse = any(0 < err[i, c] < keys_of[c] for c in range(nct))
        else:
            e, keys = int(err[i].sum()), int(keys_of.sum())
            refuse = 0 < e < keys
            if refuse:
                _add(ev, "mt finish: refused, some keys fail")
            elif e and e == keys and (err[i] > 0).sum() >= 3:
                _add(ev, "mt finish: not refused, every key fails in 3 CTAs")
        A = kids[0]
        if op == "cond" and nodes[A][0] in BIN_OPS:
            nilc = [c for c in nodes[A][1] if kind[c] == MK_VEC]
            if "refusal per CTA" in mut:
                empty = any(all(cnt[c, x] == 0 for c in nilc) for x in range(nct))
            else:
                empty = all(cnt[c].sum() == 0 for c in nilc)
                if empty:
                    _add(ev, "mt finish: refused, COND over nil")
                elif all(cnt[c].sum() == 1 and cnt[c, nct - 1] == 1 for c in nilc) and nct >= 3:
                    _add(ev, "mt finish: COND over a binary node whose only key is in the last CTA")
            refuse = refuse or empty
        if refuse:
            return refused()
    root = nn - 1
    words_out = {}
    if kind[root] == MK_CONST:
        kd, ln = 2, (len(rng_u) if rng_u is not None else 1)
        tags = 1 << val[root][0]
    elif kind[root] == MK_MAP0:
        kd, ln, tags = 1, 1, 1 << val[root][0]
    elif kind[root] == MK_VEC and cnt[root].sum():
        kd, ln = 1, int(cnt[root].sum())
        per = [0] * nct
        for ti, r in enumerate(res[root]):
            if r is not None:
                per[ti // NT] |= 1 << r[0]
        tags = per[0] if "tags of CTA 0 only" in mut else int(np.bitwise_or.reduce(per))
        all_tags = int(np.bitwise_or.reduce(per))
        if all_tags & (1 << INT) and all_tags & (1 << FLT):
            fl = [c for c in range(nct) if per[c] & (1 << FLT)]
            if fl == [nct - 1] and nct >= 3:
                _add(ev, "mt finish: promotion from the last CTA only")
            if fl == [0] and nct >= 3:
                _add(ev, "mt finish: promotion from CTA 0 only")
        elif any(r is not None and r[0] == FLT for i in range(nn - 1) if kind[i] == MK_VEC for r in res[i]):
            _add(ev, "mt finish: floats below the root, no promotion")
        if (tags & (1 << INT)) and (tags & (1 << FLT)):
            tags &= ~(1 << INT)
            words_out["promote"] = True
    else:
        kd, ln, tags = 0, 0, 0
    if ln == 0:
        tags = 0
    info = ln | kd << 32 | tags << 40
    out_cap = call.out_cap if call.out_cap is not None else max(cap + 1, len(rng_u) if rng_u is not None else 1)
    if ln > out_cap:
        _add(ev, "mt finish: ERR_CAP")
        return MtOut(OK if dev else ERR_CAP, ERR_CAP if dev else None, info, None, None, None, launches if dev else 0)
    # the root scan's tiles over ulen, and mt_write_kernel
    if kind[root] == MK_VEC and ulen:
        if -(-ulen // EN_TILE) >= 3:
            _add(ev, "mt scan: 3 tiles over ulen")
        absent = [res[root][ti] is None for ti in range(ulen)]
        if all(any(absent[e - 1] and absent[e] for e in range(m, ulen, m)) for m in (32, 256, 2048)):
            _add(ev, "mt scan: root keys absent on both sides of a 32, 256 and 2048 edge")
    keys, wds, tgs = [], [], []
    if kd == 2:
        nr = len(rng_u) if rng_u is not None else 1
        if rng_u is not None:
            if nr in NRANGE:
                _add(ev, f"mt write: nrange = {nr}")
            if nr == 0:
                _add(ev, "mt write: a constant over an empty range")
            if nr > NT:
                _add(ev, "mt write: a constant over a range past one CTA")
        threads = _grid(cap if "range fill over cap" in mut else max(cap, nr if rng_u is not None else 1))
        for t in range(min(nr, threads)):
            keys.append(int(rng_u[t]) if rng_u is not None else 0)
            wds.append(val[root][1])
            tgs.append(val[root][0])
    elif kd == 1 and kind[root] == MK_MAP0:
        keys, wds, tgs = [0], [val[root][1]], [val[root][0]]
    elif kd == 1:
        for ti, r in enumerate(res[root]):
            if r is None:
                continue
            g, w = r
            if g == INT and words_out.get("promote"):
                g, w = FLT, gm._W(float(gm._I(w)))
            keys.append(U[ti])
            wds.append(w)
            tgs.append(g)
    if "root over cap" in mut and kind[root] == MK_VEC and cap > ulen and dev:
        keys += [POISON] * (cap - ulen)
        wds += [POISON] * (cap - ulen)
        tgs += [ABS] * (cap - ulen)
    return MtOut(OK, OK if dev else None, info, np.array(keys, np.uint64), np.array(wds, np.uint64),
                 np.array(tgs, np.uint8), launches)


def mt_malformed(case: MtCase):
    """Input the library refuses that evalMathTree never sees: key 0 among other keys, a range not ascending."""
    tree, maps, r = case
    return any(m is not None and len(m[0]) > 1 and int(np.asarray(m[0])[0]) == 0 for m in maps.values()) or (
        r is not None and any(int(r[i - 1]) >= int(r[i]) for i in range(1, len(r))))


def mt_expected(case: MtCase):
    """The oracle's (kind, keys, words, tags), or None where the library refuses: math_oracle (with its partial
    answer flag) and key 0 among other keys; gen_math.formula must agree."""
    import math_oracle as mo

    if mt_malformed(case):
        return None
    tree, maps, r = case
    w = mo.evaluate(tree, maps, r, seed=0)
    return None if w[0] is None or w[4] else w[:4]


# ---- math() fixtures --------------------------------------------------------------------------------------------------

MT_DEFAULT = (MtCall("host", None, 0), MtCall("dev", None, 3))


def _mt(name, cases, events, kills=(), calls=MT_DEFAULT):
    return MtFix(name, tuple(MtCase(*c) for c in cases), calls, set(events), set(kills))


def _ints(keys, vals):
    return (np.asarray(keys, np.uint64), np.asarray(vals, np.int64))


def _tagged(keys, words, tags):
    return (np.asarray(keys, np.uint64), np.asarray(words, np.uint64), np.asarray(tags, np.uint8))


def _fw(x):
    return gm._W(float(x))


MIN64 = -(2 ** 63)


def mt_fixtures():
    fx = []
    # U lengths at the warp, CTA and tile edges, root keys absent on both sides of every edge
    for n in ULEN:
        keys = np.arange(1, n + 1, dtype=np.uint64) * 3
        edge = {j for m in (32, 256, 2048) for e in range(m, n, m) for j in (e - 1, e)}
        ka = keys[[j for j in range(n) if j not in edge]]
        maps = {"a": _ints(ka, np.arange(ka.size) % 7), "b": _ints(keys, np.arange(n) % 5)}
        evs = {f"mt eval: ulen = {n}"}
        if n > 2048:
            evs.add("mt scan: root keys absent on both sides of a 32, 256 and 2048 edge")
        if n == 4097:
            evs.add("mt scan: 3 tiles over ulen")
        fx.append(_mt(f"ulen {n}", [(("<", ("var", "a"), ("var", "b")), maps, None)], evs, {"root over cap"}))
    # promotion: the only float root entry last (in the last CTA), first; floats only below the root
    n = 600
    keys = np.arange(1, n + 1, dtype=np.uint64)
    last = _tagged(keys, list(range(n - 1)) + [_fw(2.5)], [INT] * (n - 1) + [FLT])
    first = _tagged(keys, [_fw(0.5)] + list(range(1, n)), [FLT] + [INT] * (n - 1))
    z = _ints(keys[::2], np.ones(n // 2))
    cases = [(("+", ("var", "a"), ("var", "z")), {"a": last, "z": z}, None),
             (("+", ("var", "a"), ("var", "z")), {"a": first, "z": z}, None),
             ((">", ("+", ("var", "a"), ("var", "z")), ("const", 3)), {"a": last, "z": z}, None)]
    fx.append(_mt("promotion", cases, {"mt finish: promotion from the last CTA only",
                                       "mt finish: promotion from CTA 0 only",
                                       "mt finish: floats below the root, no promotion"}, {"tags of CTA 0 only"}))
    # refusal counts: a unary, a compare and a cond node failing on one key in lane 0 or 31 of the last CTA
    cases = []
    for lane in (0, 31):
        m = 2 * NT + lane + 1                         # U: three CTAs, the last holding lanes 0 .. lane
        keys = np.arange(1, m + 1, dtype=np.uint64) * 2
        fk = 2 * NT + lane                             # the failing key's index in U
        ka = np.concatenate([keys[:2 * NT], keys[fk:fk + 1]])   # child 0's keys: none else in the last CTA
        zz = _ints(keys, np.arange(m) % 3)
        vals = np.arange(ka.size, dtype=np.int64) % 9
        vals[-1] = MIN64
        cases.append((("max", ("u-", ("var", "a")), ("var", "z")), {"a": _ints(ka, vals), "z": zz}, None))
        w = (np.arange(ka.size) % 4).astype(np.uint64)
        tg = np.full(ka.size, INT, np.uint8)
        tg[-1] = BOOL
        cases.append((("max", ("<", ("var", "a"), ("var", "z")), ("var", "z")), {"a": _tagged(ka, w, tg), "z": zz},
                      None))
        cw = (np.arange(ka.size) % 2).astype(np.uint64)
        ct = np.full(ka.size, BOOL, np.uint8)
        ct[-1] = INT
        cases.append((("max", ("cond", ("var", "c"), ("const", 1), ("const", 2)), ("var", "z")),
                      {"c": _tagged(ka, cw, ct), "z": zz}, None))
    fx.append(_mt("one failing key in the last CTA", cases,
                  {"mt eval: a failure in lane 0 of the last CTA", "mt eval: a failure in lane 31 of the last CTA",
                   "mt eval: a unary node fails", "mt eval: a compare node fails", "mt eval: a cond node fails",
                   "mt finish: refused, some keys fail"}, {"refusal per CTA"}))
    # every key failing across 3 CTAs: not refused, an empty result
    m = 3 * NT - 7
    keys = np.arange(1, m + 1, dtype=np.uint64) * 5
    cases = [(("u-", ("var", "a")), {"a": _ints(keys, np.full(m, MIN64))}, None),
             (("<", ("var", "a"), ("const", 1)), {"a": _tagged(keys, np.ones(m), np.full(m, BOOL))}, None),
             (("cond", ("var", "c"), ("const", 1), ("const", 2)), {"c": _ints(keys, np.arange(m))}, None)]
    fx.append(_mt("every key failing", cases, {"mt finish: not refused, every key fails in 3 CTAs",
                                               "mt eval: a node's failures in 3 CTAs"}))
    # half the keys failing: refused from the first child's count
    vals = np.arange(m, dtype=np.int64)
    vals[::2] = MIN64
    vals2 = vals.copy()
    vals2[-2:] = MIN64
    fx.append(_mt("half the keys failing", [(("u-", ("var", "a")), {"a": _ints(keys, vals)}, None),
                                            (("floor", ("u-", ("var", "a"))), {"a": _ints(keys[:-1], vals2[:-1])},
                                             None)],
                  {"mt eval: half or more of a node's keys fail"}, {"keys of the node"}))
    # the COND over nil rule
    m = 2 * NT + 40
    keys = np.arange(1, m + 1, dtype=np.uint64) * 4
    zz = _ints(keys[:-1], np.arange(m - 1) % 6)
    one = _ints(keys[-1:], [7])
    cases = [(("cond", (">", ("+", ("var", "a"), ("const", 1)), ("const", 3)), ("var", "z"), ("const", 2)),
              {"a": one, "z": zz}, None),
             (("cond", ("+", ("var", "a"), ("const", 1)), ("var", "z"), ("const", 2)), {"a": one, "z": zz}, None),
             (("cond", ("+", ("u-", ("var", "m")), ("const", 1)), ("var", "z"), ("const", 2)),
              {"m": _ints(keys[:60:3], np.full(20, MIN64)), "z": zz}, None)]
    fx.append(_mt("cond over nil", cases, {"mt finish: COND over a binary node whose only key is in the last CTA",
                                           "mt finish: refused, COND over nil"}, {"refusal per CTA"}))
    # leaf thread spaces: 16 leaves with rooms of 0 first, between and last
    maps, names = {}, []
    for j in range(16):
        nm = f"l{j}"
        names.append(nm)
        maps[nm] = _ints([], []) if j in (0, 3, 4, 9, 15) else _ints(np.arange(1, 40, dtype=np.uint64) * 16 + j,
                                                                      np.full(39, j))
    t = ("var", names[0])
    for nm in names[1:]:
        t = ("+", t, ("var", nm))
    calls = (MtCall("host", None, 0), MtCall("dev", None, 0),
             MtCall("dev", None, {nm: (2 if j % 2 else 0) for j, nm in enumerate(names)}))
    # an empty int64 map is an empty leaf, not the aggregate {0: 0}: e - 1 is nil, so a + (e - 1) is a
    empty = (("+", ("var", "l1"), ("-", ("var", "l0"), ("const", 1))), {"l0": maps["l0"], "l1": maps["l1"]}, None)
    fx.append(_mt("rooms of 0", [(t, maps, None), empty], {"mt space: a room of 0 first", "mt space: a room of 0 last",
                                                    "mt space: rooms of 0 between leaves"},
                  {"room-0 leaf owns threads"}, calls))
    # rooms summing to 256k - 1, 256k, 256k + 1
    cases = []
    for tot in (2 * NT - 1, 2 * NT, 2 * NT + 1):
        ka = np.arange(1, 101, dtype=np.uint64) * 3
        kb = np.arange(1, tot - 100 + 1, dtype=np.uint64) * 2
        cases.append((("-", ("var", "a"), ("var", "b")), {"a": _ints(ka, ka.astype(np.int64)),
                                                           "b": _ints(kb, np.ones(kb.size))}, None))
    fx.append(_mt("rooms at a CTA edge", cases, {f"mt space: cap_total = {d}" for d in CAP_EDGES},
                  calls=(MtCall("host", None, 0), MtCall("dev", None, 0))))
    # 2^64 - 1 in a general map, next to the {MaxUint64: v} constant
    g = _ints([5, 9, 1 << 40, U64], [1, 2, 3, 4])
    c = _ints([U64], [3])
    fx.append(_mt("MaxUint64 keys", [(("*", ("var", "g"), ("var", "c")), {"g": g, "c": c}, None),
                                     (("-", ("var", "c"), ("var", "g")), {"g": g, "c": c}, np.array([4, 8], np.uint64)),
                                     (("+", ("var", "g"), ("var", "n")), {"g": g, "n": None}, None)],
                  {"mt plan: a general map holding 2^64 - 1", "mt plan: a {MaxUint64: v} constant",
                   "mt plan: a nil leaf"}))
    # a constant over ranges, no general leaf
    s = _ints([0], [2])
    cases = [(("+", ("var", "s"), ("const", 1)), {"s": s}, np.arange(1, nr + 1, dtype=np.uint64) * 7) for nr in NRANGE]
    fx.append(_mt("constant over ranges", cases, {f"mt write: nrange = {nr}" for nr in NRANGE} |
                  {"mt write: a constant over an empty range", "mt write: a constant over a range past one CTA",
                   "mt space: range checks from cap_total on"}, {"range fill over cap"}))
    # a range that descends only at its last pair, at a CTA edge; out_cap one short
    r = np.arange(1, NT + 1, dtype=np.uint64) * 3
    r[-1] = r[-2]
    fx.append(_mt("range descending at a CTA edge", [(("+", ("var", "s"), ("const", 1)), {"s": s}, r)],
                  {"mt check: a range descending only at its last pair, on a CTA's first thread"},
                  calls=(MtCall("host", None, 0), MtCall("dev", None, 0))))
    r = np.arange(1, 300, dtype=np.uint64)
    fx.append(_mt("out_cap one short", [(("+", ("var", "s"), ("const", 1)), {"s": s}, r)], {"mt finish: ERR_CAP"},
                  calls=(MtCall("host", r.size - 1, 0), MtCall("dev", r.size - 1, 0), MtCall("host", r.size, 0))))
    # program limits: a 64-node post-order chain; 16 general leaves; scalar {0: v} subtrees inside vector nodes
    keys = np.arange(1, 300, dtype=np.uint64) * 11
    t = ("var", "a")
    for i in range(63):
        t = (["u-", "floor", "ceil"][i % 3], t)
    chain = (t, {"a": _ints(keys, np.arange(keys.size) - 100)}, None)
    maps = {f"g{j}": _ints(np.arange(1, 60, dtype=np.uint64) * (j + 2), np.full(59, j + 1)) for j in range(16)}
    t = ("var", "g0")
    for j in range(1, 16):
        t = (["+", "max", "-", "min"][j % 4], t, ("var", f"g{j}"))
    sixteen = (t, maps, None)
    t = ("var", "a")
    smaps = {"a": _ints(keys, np.arange(keys.size)), **{f"s{j}": _ints([0], [j + 1]) for j in range(4)}}
    for j in range(15):
        t = ("+", t, ("*", ("var", f"s{j % 4}"), ("const", 2 if j % 2 else 1.5)))
    t = ("u-", ("u-", ("u-", t)))
    mixed = (t, smaps, None)
    assert gm.nodes(chain[0]) == gm.nodes(mixed[0]) == 64
    fx.append(_mt("program limits", [chain, sixteen, mixed], {"mt plan: 64 nodes", "mt plan: 16 general leaves",
                                                              "mt plan: a scalar subtree inside a vector node"}))
    return fx


def all_fixtures():
    return tg_fixtures() + mt_fixtures()


def outcomes(f, mut=frozenset()):
    """(per case and call: the model's outcome), the events the fixture reaches."""
    ev: set = set()
    run = tg_run if isinstance(f, TgFix) else mt_run
    return [[run(c, call, mut, ev) for call in f.calls] for c in f.cases], ev
