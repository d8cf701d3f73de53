"""Host model of @cascade's level kernels (cascade_kernel.cuh, dgx_api.cu cc_plan / cc_run) and of @filter's tree
evaluator driving them (sg_filter_kernel.cuh, dgx_api.cu sf_run), with fixtures aimed at every node, level, CTA and
tile boundary of both.

@cascade.  The launch count is cascade_plan.py's.  On top of it the model restates cc_plan's level order (deepest
level first, node order inside a level), the slot bases vb / ob / db / hb and the levels with work; for each kernel's
thread space, the node that owns each thread (cc_node_of: the last node whose base is <= t, so a node of zero slots
owns none), with its CTA and scan tile; cc_gather_kernel's offset check; per level, cc_keep_kernel's order check inside
a node and its prune loop over the checked children's *final* rows, has_val and counts_len; the three scans of
scan_u64_kernel as EN_TILE tiles, each carrying the total of the tiles before it; cc_filter_kernel's new dest, its
row search lower_bound(VO, nrows + 1, p + 1) - 1 (empty rows share an offset with the next row), the slack of a value
room, the order check of unordered rows and the KEEP / OLD / NEW test; cc_page_range and cc_page_kernel's rank
fx[t] - fx[row start] for each row's survivor count; cc_compact_kernel; cc_count_kernel with the node-order count scan
over 2 NN; cc_place_kernel.  Every device-side refusal is recorded with the kernel thread's CTA and tile.

@filter.  The launch count is sg_filter_plan.py's.  The model restates sf_run's one NEW node (ndest = d0_cap until
sf_check_kernel writes |D0|, ordered rows, counts-only compacting the offsets alone) and the scans' size words (|D0|,
v_off[nrows], |D1|); sf_check_kernel's thread space max(d0_cap, slots, nrows + 1, v_cap), the leaf that owns each check
slot (zero-slot COUNT-over-counts leaves share sb with the next leaf) and every check; sf_eval_kernel's stackless
pre-order walk step by step (which levels one leaf closes, where an AND or OR stops); cascade's filter, page and compact
kernels over the one node; sf_mark_kernel and sf_out_kernel for paged and unpaged D2.

What the kernels decide is named as *events* (EVENTS); fixtures name the events they must reach and the model refuses
a name that is not registered.  Named *mutants* (MUTANTS) are plausible one-line slips; a fixture names the mutants it
kills, and tests/test_cascade_geometry.py checks that the mutated model's output differs from the oracle's on it.  No
mutated kernel is built: a slot owned by the wrong node or a walk past its program reads outside the arrays.

Edges the kernels have that no fixture reaches at test scale:
  - totals of 2^32 rows, values, dest values or leaf slots, which the host refuses (and so the u32 row index rw and
    the u32 counts of sf_out_kernel);
  - the look-back order of the multi-CTA scans: the scheduler chooses which tile publishes first; the fixtures of two
    to 64 tiles make a multi-CTA scan happen but cannot choose its order;
  - forests of 2^16 - 1 nodes that also hold values in most nodes (the fixture of 65 535 nodes is mostly empty);
  - length words whose high 32 bits are set (the device form reads the low 32 bits; the fixtures set some high bits
    but cannot make the low word wrap).

The constants and the statements the model restates are read from the CUDA sources as text, so a rewrite fails here
loudly instead of leaving the fixtures aimed at stale edges.  tests/test_cascade_geometry.py checks the fixtures on the
CPU; tests/test_gpu_cascade_edges.py runs them through the kernels.
"""
from __future__ import annotations

import itertools
import os
import re
from collections import namedtuple

import numpy as np

import cascade_plan as cp
import sg_filter_plan as sp
from dgraph_b200.algo import CC_CASCADE, CC_CHECKED, CC_FILTERED, CC_ORDERED, CC_SKIP, CascadeNode, sg_filter_flat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")
OK, ERR_ARG, ERR_CAP = 0, -3, -4
POISON = 0xBAD0BAD0BAD0BAD0     # what a mutant reads where the kernel would read outside an array
BIG = 1 << 62                   # an index read outside an array (a mutant's)


def _src(fn):
    path = os.path.join(ROOT, "include", fn) if fn.endswith(".h") else os.path.join(CSRC, fn)
    with open(path) as f:
        return f.read()


def _one(pat, text, what):
    m = re.search(pat, text)
    if not m:
        raise ValueError(f"{what} changed: restate it in the cascade model (tests/cascade_geometry.py)")
    return m


def _fn(name, text):
    """The body of the function or kernel `name` (a definition starting a line, through its closing brace)."""
    head = r"(?ms)^(?:static |__global__ |__device__ |extern \"C\" )[^\n]*\b"
    return _one(head + name + r"\(.*?\n\}\n", text, name).group(0)


CK, SK, API = "cascade_kernel.cuh", "sg_filter_kernel.cuh", "dgx_api.cu"
# (file, function or None for the whole file, statement as a regex, what it restates)
STATEMENTS = [
    (CK, "cc_node_of", r"if \(N\[mid\]\.\*F <= t\) lo = mid; else hi = mid;", "the last node of equal bases"),
    (CK, "cc_gather_kernel", r"bool bad = r == 0 \? x != n\.v_base : x < n\.v_off\[r - 1\];\s*"
     r"if \(r == n\.nrows && x - n\.v_base > n\.vcap\) bad = true;", "the offset check"),
    (CK, "cc_gather_kernel", r"P\.VO\[t\] = P\.OO\[t\] = n\.vb \+ \(x - n\.v_base\);", "the gathered offsets"),
    (CK, "cc_keep_kernel", r"if \(i > 0 && P\.D\[p - 1\] >= P\.D\[p\]\) cc_refuse\(P\);", "the dest order check"),
    (CK, "cc_keep_kernel", r"for \(u32 k = n\.ck_b; k < n\.ck_e && keep; \+\+k\) \{\s*const CcNode& c = N\[P\.ck\[k\]\];"
     r"\s*const bool no_row = i >= c\.nrows \|\| P\.OO\[c\.ob \+ i \+ 1\] == P\.OO\[c\.ob \+ i\];\s*"
     r"const bool no_val = i >= c\.nhv \|\| P\.H\[c\.hb \+ i\] == 0;\s*"
     r"if \(no_row && no_val && i >= c\.counts_len\) keep = 0;", "the prune loop"),
    (CK, "cc_filter_kernel", r"P\.ND\[n\.db \+ P\.kx\[t\] - P\.kx\[n\.db - L\.da\]\] = P\.D\[p\];", "the new dest's place"),
    (CK, "cc_filter_kernel", r"P\.NDE\[L\.a \+ t\] = P\.kx\[n\.db \+ n\.ndest - L\.da\] - P\.kx\[n\.db - L\.da\];",
     "the new dest's length"),
    (CK, "cc_filter_kernel", r"if \(p < P\.VO\[n\.ob \+ n\.nrows\]\) \{", "the slack of a value room"),
    (CK, "cc_filter_kernel", r"const u64 r = lower_bound_g\(P\.VO \+ n\.ob, n\.nrows \+ 1, p \+ 1\) - 1;",
     "the row search"),
    (CK, "cc_filter_kernel", r"if \(!n\.ordered && P\.VO\[n\.ob \+ r\] != p && P\.V\[p - 1\] >= x\) cc_refuse\(P\);",
     "the row order check"),
    (CK, "cc_filter_kernel", r"if \(n\.mode != CC_ROWS_KEEP\) \{\s*const u64 j = lower_bound_g\(P\.D \+ n\.db, n\.ndest, "
     r"x\);\s*f = j < n\.ndest && P\.D\[n\.db \+ j\] == x && \(n\.mode == CC_ROWS_OLD \|\| P\.keep\[n\.db - L\.da \+ j\]\);",
     "the mode test"),
    (CK, "cc_page_range", r"s = 0;\s*e = n;\s*if \(n == 0 \|\| \(count == 0 && offset == 0\)\) return;\s*"
     r"if \(count < 0\) \{\s*if \(-count > n\) count = -n;\s*s = \(\(\(n \+ count\) % n\) \+ n\) % n;\s*return;\s*\}\s*"
     r"s = offset < 0 \? 0 : offset;\s*if \(s > n\) \{ s = n; return; \}\s*if \(count == 0\) return;\s*"
     r"if \(s \+ count < n\) e = s \+ count;", "PageRange"),
    (CK, "cc_page_kernel", r"if \(n\.mode != CC_ROWS_NEW\) return;", "the page cut of NEW nodes only"),
    (CK, "cc_page_kernel", r"const u64 rs = P\.VO\[n\.ob \+ r\] - L\.va, re = P\.VO\[n\.ob \+ r \+ 1\] - L\.va;\s*"
     r"long long s, e;\s*cc_page_range\(n\.first, n\.offset, \(long long\)\(P\.fx\[re\] - P\.fx\[rs\]\), s, e\);\s*"
     r"const long long rank = \(long long\)\(P\.fx\[t\] - P\.fx\[rs\]\);\s*if \(rank < s \|\| rank >= e\) P\.fv\[t\] = 0;",
     "the rank in its row"),
    (CK, "cc_compact_kernel", r"P\.OV\[n\.vb \+ P\.fy\[t\] - P\.fy\[n\.vb - L\.va\]\] = P\.V\[p\];", "the kept values"),
    (CK, "cc_compact_kernel", r"P\.OO\[q\] = n\.vb \+ P\.fy\[P\.VO\[q\] - L\.va\] - P\.fy\[n\.vb - L\.va\];",
     "the offset write"),
    (CK, "cc_count_kernel", r"P\.cnt\[n\.id\] = P\.OO\[n\.ob \+ n\.nrows\] - n\.vb;\s*"
     r"P\.cnt\[P\.nnodes \+ n\.id\] = P\.NDE\[t\];", "the node-order counts"),
    (CK, "cc_place_kernel", r"if \(\*P\.bad\) \{\s*if \(t == 0\) P\.sizes\[0\] = P\.sizes\[1\] = 0;\s*return;",
     "a refused call's sizes"),
    (CK, "cc_place_kernel", r"const u64 NN = P\.nnodes, dbase = P\.cx\[NN\];", "dbase"),
    (CK, "cc_place_kernel", r"if \(t < P\.OO\[n\.ob \+ n\.nrows\]\) P\.out\[P\.cx\[n\.id\] \+ t - n\.vb\] = P\.OV\[t\];",
     "the placed values"),
    (CK, "cc_place_kernel", r"if \(r < n\.nrows\) P\.out_off\[n\.out_row \+ r\] = P\.cx\[n\.id\] \+ P\.OO\[t\] - n\.vb;",
     "the placed offsets"),
    (CK, "cc_place_kernel", r"if \(t - n\.db < P\.NDE\[k\]\) P\.dest_out\[P\.cx\[NN \+ n\.id\] - dbase \+ t - n\.db\] = "
     r"P\.ND\[t\];", "the placed dest"),
    (API, "cc_plan", r"for \(int64_t d = maxd; d >= 0 && n; --d\) \{", "the level order"),
    (API, "cc_plan", r"const bool paged = cascade && \(!root \|\| t->first\[k\] != 0 \|\| t->offset\[k\] != 0\);\s*"
     r"c\.mode = paged \? CC_ROWS_NEW : \(f & DGX_CASCADE_FILTERED\) && !skip \? CC_ROWS_OLD : CC_ROWS_KEEP;\s*"
     r"c\.prune = cascade && !skip;", "a node's mode"),
    (API, "cc_plan", r"if \(L\.nv == 0 && L\.nd == 0\) continue;", "a level without work"),
    (API, "cc_run", r"h_words\[2 \* D\] = 2 \* NN;", "the count scan's size"),
    (API, "cc_run", r"scan\(P\.cnt, P\.cx, d_words \+ 2 \* D, 2 \* NN\);", "the node-order count scan"),
    (API, "cc_run", r"scan\(P\.keep, P\.kx, L\.n_dest, L\.nd\);\s*cc_filter_kernel<<<gb_grid\(std::max<uint64_t>\(\{"
     r"L\.nd, L\.nv, L\.b - L\.a\}\)\), 256, 0, l->stream>>>\(P, L\);\s*scan\(P\.fv, P\.fx, L\.n_val, L\.nv\);", "a level"),
    (API, "sf_run", r"s\.sb = slots;", "a leaf's first check slot"),
    (API, "sf_run", r"slots \+= L\.n \+ 1;", "a LIST leaf's check slots"),
    (API, "sf_run", r"if \(L\.off\) slots \+= d0_cap;", "a COUNT leaf's check slots"),
    (API, "sf_run", r"c\.ndest = d0_cap;[^\n]*\s*c\.mode = CC_ROWS_NEW;\s*c\.ordered = 1;", "the one NEW node"),
    (API, "sf_run", r"S\.paged = count != 0 \|\| offset != 0;", "paging"),
    (API, "sf_run", r"if \(S\.counts_only\) Lc\.nv = 0;", "counts-only"),
    (API, "sf_run", r"sf_check_kernel<<<gb_grid\(std::max<uint64_t>\(\{d0_cap, slots, nrows \+ 1, v_cap\}\)\), 256, 0, "
     r"l->stream>>>\(S\);", "the check's grid"),
    (API, "sf_run", r"scan\(P\.keep, P\.kx, L\.n_dest, d0_cap\);", "the D1 scan"),
    (API, "sf_run", r"scan\(P\.fv, P\.fx, L\.n_val, v_cap\);", "the value scan"),
    (API, "sf_run", r"scan\(P\.fv, P\.fy, L\.n_val, v_cap\);", "the paged scan"),
    (API, "sf_run", r"scan\(S\.mark, mx, P\.NDE, d0_cap\);", "the mark scan"),
    (API, "sf_check_args", r"for \(size_t k = n; k-- > 0;\) end\[k\] = kids\[k\]\.empty\(\) \? pos\[k\] \+ 1 : "
     r"end\[kids\[k\]\.back\(\)\];", "a subtree's end"),
    (SK, "sf_word_len", r"const u64 n = \*w & 0xffffffffull;\s*over = n > room;\s*return over \? 0 : n;", "a length word"),
    (SK, "sf_check_kernel", r"P\.node->ndest = n0;\s*P\.words\[0\] = n0;\s*P\.words\[1\] = P\.v_off\[P\.nrows\];",
     "the size words"),
    (SK, "sf_check_kernel", r"if \(t > 0 && t < n0 && P\.d0\[t - 1\] >= P\.d0\[t\]\) sf_refuse\(P\);", "D0's order"),
    (SK, "sf_check_kernel", r"if \(P\.leaf\[mid\]\.sb <= t\) lo = mid; else hi = mid;", "the leaf search"),
    (SK, "sf_check_kernel", r"if \(lover && j == 0\) sf_refuse\(P\);\s*"
     r"if \(j > 0 && j < n && L\.p\[j - 1\] >= L\.p\[j\]\) sf_refuse\(P\);", "a LIST leaf's checks"),
    (SK, "sf_check_kernel", r"\} else if \(j < n0 && L\.off\[j \+ 1\] < L\.off\[j\]\) \{", "a COUNT leaf's check"),
    (SK, "sf_check_kernel", r"if \(t == 0 \? x != 0 : x < P\.v_off\[t - 1\]\) sf_refuse\(P\);\s*"
     r"if \(t == P\.nrows && x > P\.v_cap\) sf_refuse\(P\);", "the offset checks"),
    (SK, "sf_check_kernel", r"const u64 nv = min\(P\.v_off\[P\.nrows\], P\.v_cap\);", "the checked values"),
    (SK, "sf_check_kernel", r"const u64 r = lower_bound_g\(P\.v_off, P\.nrows \+ 1, t \+ 1\) - 1;\s*"
     r"if \(P\.v_off\[r\] != t\) sf_refuse\(P\);", "a row start may descend"),
    (SK, "sf_leaf_holds", r"const long long c = L\.cnt \? \(long long\)L\.cnt\[i\] : \(long long\)\(L\.off\[i \+ 1\] - "
     r"L\.off\[i\]\);", "a COUNT leaf's count"),
    (SK, "sf_eval_kernel", r"if \(\*P\.bad \|\| t >= P\.node->ndest\) \{\s*P\.keep\[t\] = 0;", "the slots past |D0|"),
    (SK, "sf_eval_kernel", r"u32 cur = kSfNoParent, pc = 0;", "the walk's start"),
    (SK, "sf_eval_kernel", r"if \(e\.w0 & kSfNode\) \{[^\n]*\s*cur = pc\+\+;\s*continue;", "opening a node"),
    (SK, "sf_eval_kernel", r"r = sf_leaf_holds\(P\.leaf\[e\.w0\], t, x\);\s*\+\+pc;", "a leaf's test"),
    (SK, "sf_eval_kernel", r"if \(cur == kSfNoParent\) \{\s*P\.keep\[t\] = r;\s*return;", "the walk's end"),
    (SK, "sf_eval_kernel", r"const u32 op = \(f\.w0 >> 28\) & 7u, end = f\.w0 & kSfEndMask;\s*"
     r"if \(op == SF_NOT\) r = !r;\s*else if \(\(op == SF_AND\) == r && pc != end\) break;[^\n]*\s*pc = end;\s*"
     r"cur = f\.w1;", "closing a node"),
    (SK, "sf_mark_kernel", r"if \(!P\.paged\) \{\s*if \(t < n1\) P\.mark\[t\] = 1;\s*return;\s*\}\s*"
     r"if \(t < P\.v_cap && P\.fv\[t\]\) P\.mark\[lower_bound_g\(P\.d1, n1, P\.v\[t\]\)\] = 1;", "the marks"),
    (SK, "sf_out_kernel", r"if \(\*P\.bad\) \{\s*if \(t == 0\) \*P\.dest_len = 0;\s*return;", "a refused call's length"),
    (SK, "sf_out_kernel", r"if \(t < n1 && P\.mark\[t\]\) P\.dest_out\[P\.mx\[t\]\] = P\.d1\[t\];\s*"
     r"if \(t == 0\) \*P\.dest_len = P\.mx\[n1\];\s*if \(t < P\.nrows\) P\.counts\[t\] = \(u32\)\(P\.oo\[t \+ 1\] - "
     r"P\.oo\[t\]\);", "D2 and the counts"),
]


def read_constants() -> dict:
    text = {f: _src(f) for f in (API, CK, SK, "encode_kernel.cuh", "dgx.h")}
    m = _one(r"constexpr int EN_NT = (\d+), EN_VT = (\d+), EN_TILE = EN_NT \* EN_VT;", text["encode_kernel.cuh"],
             "EN_TILE")
    K = {"EN_NT": int(m.group(1)), "EN_VT": int(m.group(2))}
    K["EN_TILE"] = K["EN_NT"] * K["EN_VT"]
    K["CC_MAX_NODES"] = 1 << int(_one(r"constexpr size_t kCcMaxNodes = size_t\(1\) << (\d+);", text[API],
                                      "kCcMaxNodes").group(1))
    K["CC_MAX_DEPTH"] = int(_one(r"constexpr uint32_t kCcMaxDepth = (\d+);", text[API], "kCcMaxDepth").group(1))
    for k in ("MAX_NODES", "MAX_LEAVES", "MAX_DEPTH"):
        K["SGF_" + k] = int(_one(r"#define DGX_SGF_%s (\d+)" % k, text["dgx.h"], "DGX_SGF_" + k).group(1))
    grids = {}
    for fn, kern in ((CK, "cc_gather_kernel"), (CK, "cc_keep_kernel"), (CK, "cc_filter_kernel"),
                     (CK, "cc_page_kernel"), (CK, "cc_compact_kernel"), (CK, "cc_count_kernel"),
                     (CK, "cc_place_kernel"), (SK, "sf_check_kernel"), (SK, "sf_eval_kernel"),
                     (SK, "sf_mark_kernel"), (SK, "sf_out_kernel")):
        grids[kern] = int(_one(r"__global__ void __launch_bounds__\((\d+)\) " + kern, text[fn],
                               f"{kern}'s CTA").group(1))
    if set(grids.values()) != {256}:
        raise ValueError("a 256-thread grid changed: restate it in the cascade model (tests/cascade_geometry.py)")
    _one(r"return \(unsigned\)std::max<uint64_t>\(1, \(n \+ 255\) / 256\);", _fn("gb_grid", text[API]), "gb_grid")
    K["GRID_NT"] = 256
    for fn, func, pat, what in STATEMENTS:
        _one(pat, _fn(func, text[fn]) if func else text[fn], what)
    return K


K = read_constants()
EN_TILE, NT = K["EN_TILE"], K["GRID_NT"]
NODE, END_MASK, NO_PARENT = 1 << 31, (1 << 28) - 1, 0xFFFFFFFF
SF_AND, SF_OR, SF_NOT = 1, 2, 3
KEEP, OLD, NEW = 0, 1, 2

MUTANTS = {
    # @cascade
    "node_of takes the first of equal bases": "cc_node_of returns the first node of a run of equal slot bases, so a "
                                              "node of zero slots owns the next node's slots",
    "dest rank not relative to its node": "cc_filter_kernel places a kept dest at db + kx[t] (the level's rank), "
                                          "without - kx[db - da]",
    "row rank relative to the level": "cc_page_kernel's rank is fx[t], not fx[t] - fx[row start]",
    "page on the pre-filter length": "cc_page_range gets the row's length, not its survivor count",
    "prune reads the gathered rows": "cc_keep_kernel reads a checked child's gathered offsets (VO), not its final ones",
    "dest order across node edges": "cc_keep_kernel checks D[p - 1] < D[p] for every thread but the first (t > 0), "
                                    "not inside a node (i > 0)",
    "negative count clamp dropped": "cc_page_range without if (-count > n) count = -n",
    "row search at p": "cc_filter_kernel's row is lower_bound(VO, p) - 1, so a value after empty rows is misread",
    "scans without tile carry": "scan_u64_kernel's tiles each start from 0, not from the tiles before them",
    "count scan over NN": "cc_run scans the node-order counts over NN entries, not 2 NN",
    # @filter
    "leaf search takes the first of an equal sb": "sf_check_kernel's leaf is the first of the leaves sharing a first "
                                                  "slot, so a zero-slot COUNT leaf owns the next leaf's slots",
    "eval without pc != end": "sf_eval_kernel's stop test without pc != end: an AND after a hit (or OR after a miss) "
                              "at its last child reads past its subtree",
    "NOT decoded as OR": "sf_eval_kernel decodes the op with the wrong mask, so a NOT closes as a one-child OR",
    "|D0| read as d0_cap": "sf_check_kernel ignores the length word of D0: the slack past |D0| is checked, evaluated "
                           "and kept",
    "sf_mark marks all of D1 when paged": "sf_mark_kernel marks every D1 position whether or not paging is on",
}

WHERE = ("in a CTA's last thread", "at a second tile's first slot")
REFUSALS = ("dest order", "row order", "offset start", "offset decrease", "offset past room")
EVENTS = {
    "cc plan: a level without work between levels with work", "cc plan: the root level without work",
    "cc plan: a node at depth kCcMaxDepth - 1", "cc plan: 2 to 63 levels with work",
    "cc plan: a forest of 2^16 - 1 nodes",
    "cc space: a zero-slot node first in a level's value slots", "cc space: a zero-slot node between value slots",
    "cc space: a zero-slot node last in a level's value slots",
    "cc space: a zero-slot node first in a level's dest slots", "cc space: a zero-slot node between dest slots",
    "cc space: a zero-slot node last in a level's dest slots",
    "cc space: a zero-slot node first in a level's has_val slots", "cc space: a zero-slot node between has_val slots",
    "cc space: a zero-slot node last in a level's has_val slots",
    "cc space: a node's first value slot on a CTA edge", "cc space: a node's first value slot on a tile edge",
    "cc space: a node's first dest slot on a CTA edge", "cc space: a node's first dest slot on a tile edge",
    "cc space: a row boundary on a CTA edge", "cc space: a row of 256 values",
    "cc space: empty rows sharing an offset on a CTA edge", "cc space: a level's values in 3 or more tiles",
    "cc space: a device value room with slack across a tile edge",
    "cc keep: a dest pruned", "cc keep: a checked child with nrows == i", "cc keep: a checked child with nhv == i",
    "cc keep: kept by counts_len == i + 1", "cc keep: pruned at i == counts_len",
    "cc keep: a child row emptied by the child's own filter", "cc keep: a child row emptied by the child's page cut",
    "cc keep: a CASCADE node without a checked child", "cc keep: a dest that descends across a node edge",
    "cc keep: a later node's kept dest compacted across a tile edge",
    "cc filter: KEEP, OLD and NEW nodes in one level", "cc filter: a value dropped by OLD",
    "cc filter: a value dropped by NEW", "cc filter: an ORDERED row that descends",
    "cc filter: a row that descends from the row before", "cc filter: a row after empty rows starts on a CTA edge",
    "cc filter: the slack of a value room",
    "cc page: PageRange without first or offset",
    "cc page: a negative first past the row, clamped", "cc page: a negative first inside the row",
    "cc page: a negative offset", "cc page: an offset past the row", "cc page: an offset only",
    "cc page: first cuts inside the row", "cc page: first reaches past the row",
    "cc page: kept values on both sides of a tile edge", "cc page: the page cut on both sides of a tile edge",
    "cc page: a row's survivors fewer than its values",
    "cc scan: keep flags over 2 tiles with a carry", "cc scan: value flags over 2 tiles with a carry",
    "cc scan: node-order counts in 1 tile", "cc scan: node-order counts over 2 tiles",
    "cc scan: node-order counts over 64 tiles",
    "cc refuse: at the root level", "cc refuse: at a level 32 or more deep",
    "sf space: |D0| of 255", "sf space: |D0| of 256", "sf space: |D0| of 257", "sf space: |D0| of 2047",
    "sf space: |D0| of 2048", "sf space: |D0| of 2049", "sf space: |D0| of 4097",
    "sf space: a length word below d0_cap by a tile", "sf space: v_off[nrows] below v_cap across a tile edge",
    "sf space: nrows above d0_cap", "sf space: no rows", "sf space: a LIST leaf of room 0",
    "sf space: a zero-slot leaf first", "sf space: a zero-slot leaf between others", "sf space: a zero-slot leaf last",
    "sf space: a leaf boundary on a CTA edge", "sf space: check slots past d0_cap, v_cap and nrows",
    "sf space: a descent in a LIST's slack, accepted",
    "sf space: a count of 2^32 or more",
    "sf refuse: a LIST descends at its first checked slot", "sf refuse: a LIST descends at its last checked slot",
    "sf refuse: a length word over its room", "sf refuse: D0's length word over d0_cap", "sf refuse: D0 descends",
    "sf refuse: a COUNT leaf's offsets decrease", "sf refuse: row offsets", "sf refuse: a row descends",
    "sf eval: opening a node", "sf eval: a leaf hit", "sf eval: a leaf miss", "sf eval: the walk ends at a leaf root",
    "sf eval: the close loop goes on to a next child", "sf eval: one leaf closes 64 levels",
    "sf eval: one leaf closes 2 to 63 levels", "sf eval: an odd chain of NOTs closed by one leaf",
    "sf eval: an even chain of NOTs closed by one leaf", "sf eval: an AND of one child", "sf eval: an OR of one child",
    "sf eval: an AND stopped by a miss before its last child", "sf eval: an OR stopped by a hit before its last child",
    "sf eval: an AND decided by a miss at its last child", "sf eval: an OR decided by a hit at its last child",
    "sf eval: a program of the node limit", "sf eval: a leaf table of the leaf limit, one entry never evaluated",
    "sf eval: slack D0 values that hold, not evaluated",
    "sf truth: leaf i holds u + 1 iff bit i of u is set",
    "sf d1: empty", "sf d1: 2048 values", "sf d1: 2049 values",
    "sf d2: paged, a D1 value no kept row holds", "sf d2: unpaged", "sf out: counts-only",
} | {f"cc refuse: {k} {w}" for k in REFUSALS for w in WHERE}


def _add(ev, name):
    if name not in EVENTS:
        raise KeyError(f"event {name!r} is not registered in cascade_geometry.EVENTS")
    if ev is not None:
        ev.add(name)


def _cmod(a, b):
    """C's % on signed integers (truncating)."""
    q = abs(a) // abs(b)
    return a - b * (q if (a >= 0) == (b > 0) else -q)


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


def _scan(x, n, ev, what, mut):
    """scan_u64_kernel over x[0:n]: the exclusive scan into out[0..n], out[n] the total.  Each EN_TILE tile starts from
    the total of the tiles before it (its look-back)."""
    out = np.zeros(n + 1, np.int64)
    np.cumsum(np.asarray(x[:n], np.int64), out=out[1:])
    tiles = max(1, -(-n // EN_TILE))
    if tiles > 1 and out[EN_TILE] > 0 and what:
        _add(ev, what)
    if "scans without tile carry" in mut:
        for k in range(tiles - 1, 0, -1):
            lo = k * EN_TILE
            hi = n + 1 if k == tiles - 1 else lo + EN_TILE
            out[lo:hi] -= out[lo]
    return out


def _page_range(count, offset, n, mut=frozenset()):
    """cc_page_range: x.PageRange(count, offset, n) -> [s, e)."""
    s, e = 0, n
    if n == 0 or (count == 0 and offset == 0):
        return s, e
    if count < 0:
        if -count > n and "negative count clamp dropped" not in mut:
            count = -n
        return _cmod(_cmod(n + count, n) + n, n), e
    s = 0 if offset < 0 else offset
    if s > n:
        return n, e
    if count == 0:
        return s, e
    return s, (s + count if s + count < n else e)


def _page_events(ev, count, offset, n, m):
    """The PageRange branch a row of n survivors (m values) takes."""
    if n < m:
        _add(ev, "cc page: a row's survivors fewer than its values")
    if count == 0 and offset == 0:   # n > 0: a row without survivors has no thread in cc_page_kernel
        _add(ev, "cc page: PageRange without first or offset")
    elif count < 0:
        _add(ev, "cc page: a negative first past the row, clamped" if -count > n else
             "cc page: a negative first inside the row")
    else:
        if offset < 0:
            _add(ev, "cc page: a negative offset")
        if offset > n:
            _add(ev, "cc page: an offset past the row")
        elif count == 0:
            _add(ev, "cc page: an offset only")
        elif max(offset, 0) + count < n:
            _add(ev, "cc page: first cuts inside the row")
        else:
            _add(ev, "cc page: first reaches past the row")


# ---- the level kernels, shared by @cascade and @filter ----------------------------------------------------------------

class _State:
    """The device arrays of one call: node fields (level order) and the flat slot arrays."""


def _node_of(base, a, b, t, mut):
    """cc_node_of over [a, b): the last node whose base is <= t, for an array of slots t."""
    q = np.searchsorted(base[a:b], t, "right") - 1 + a
    if "node_of takes the first of equal bases" in mut:
        q = np.searchsorted(base[a:b], base[q], "left") + a
    return q


def _refuse(S, ev, kind, t, level):
    """Record a refusal by thread t of a kernel (level: its depth, None for the gather)."""
    S.bad = True
    if ev is None:
        return
    for tt in np.atleast_1d(t):
        if tt % NT == NT - 1:
            _add(ev, f"cc refuse: {kind} in a CTA's last thread")
        if tt == EN_TILE:
            _add(ev, f"cc refuse: {kind} at a second tile's first slot")
    if level == 0:
        _add(ev, "cc refuse: at the root level")
    elif level is not None and level >= 32:
        _add(ev, "cc refuse: at a level 32 or more deep")


def _keep_kernel(S, L, ev, mut):
    """cc_keep_kernel: dest order inside a node, and the keep flag from the checked children's final rows."""
    nd = L["nd"]
    t = np.arange(nd)
    p = L["da"] + t
    o = _node_of(S.db, L["a"], L["b"], p, mut)
    i = p - S.db[o]
    inside = (t > 0) if "dest order across node edges" in mut else (i > 0)
    D = S.D
    desc = np.zeros(nd, bool)
    desc[1:] = D[p[1:] - 1] >= D[p[1:]]
    if ev is not None and np.any(desc & ~(i > 0)):
        _add(ev, "cc keep: a dest that descends across a node edge")
    bad = inside & desc
    if bad.any():
        _refuse(S, ev, "dest order", t[bad], L["depth"])
    keep = np.ones(nd, np.int64)
    OO = S.VO if "prune reads the gathered rows" in mut else S.OO
    runs = np.flatnonzero(np.r_[True, o[1:] != o[:-1]]) if nd else np.zeros(0, int)
    for lo, hi in zip(runs, list(runs[1:]) + [nd]):
        q = o[lo]
        if not S.prune[q]:
            continue
        if ev is not None and S.ck_b[q] == S.ck_e[q]:
            _add(ev, "cc keep: a CASCADE node without a checked child")
        ii = i[lo:hi]
        k = np.ones(hi - lo, bool)
        for c in S.ck[S.ck_b[q]:S.ck_e[q]]:
            has = ii < S.nrows[c]
            jj = np.where(has, ii, 0)
            no_row = ~has | (OO[S.ob[c] + jj + 1] == OO[S.ob[c] + jj])
            hv = ii < S.nhv[c]
            no_val = ~hv | (S.H[np.minimum(S.hb[c] + np.where(hv, ii, 0), max(S.H.size - 1, 0))] == 0) \
                if S.H.size else np.ones(ii.size, bool)
            gone = no_row & no_val & (ii >= S.counts_len[c])
            if ev is not None:
                for r in np.unique(ii[has & (S.OO[S.ob[c] + jj + 1] == S.OO[S.ob[c] + jj]) &
                                      (S.VO[S.ob[c] + jj + 1] != S.VO[S.ob[c] + jj])]):
                    vals = S.V[S.VO[S.ob[c] + r]:S.VO[S.ob[c] + r + 1]]
                    dest = S.ND[S.db[c]:S.db[c] + S.NDE[c]] if S.mode[c] == NEW else S.D[S.db[c]:S.db[c] + S.ndest[c]]
                    _add(ev, "cc keep: a child row emptied by the child's page cut" if np.isin(vals, dest).any()
                         else "cc keep: a child row emptied by the child's own filter")
                if np.any(k & (ii == S.nrows[c]) & ~no_val | k & (ii == S.nrows[c]) & gone):
                    _add(ev, "cc keep: a checked child with nrows == i")
                if np.any(k & (ii == S.nhv[c])):
                    _add(ev, "cc keep: a checked child with nhv == i")
                if np.any(k & no_row & no_val & (ii + 1 == S.counts_len[c])):
                    _add(ev, "cc keep: kept by counts_len == i + 1")
                if np.any(k & gone & (ii == S.counts_len[c])):
                    _add(ev, "cc keep: pruned at i == counts_len")
            k &= ~gone
        keep[lo:hi] = k
    if ev is not None and not keep.all():
        _add(ev, "cc keep: a dest pruned")
    return keep


def _filter_kernel(S, L, keep, kx, ev, mut):
    """cc_filter_kernel: the new dest, its length, each value's row, the order check and the mode test."""
    a, b, da, va, nd, nv = L["a"], L["b"], L["da"], L["va"], L["nd"], L["nv"]
    t = np.flatnonzero(keep[:nd])
    p = da + t
    o = _node_of(S.db, a, b, p, mut)
    idx = S.db[o] + kx[t] - (0 if "dest rank not relative to its node" in mut else kx[S.db[o] - da])
    for j, x in zip(idx, S.D[p]):
        if 0 <= j < S.ND.size:
            S.ND[j] = x
    if ev is not None:
        for q in np.unique(o[t >= EN_TILE]):
            if np.any((t < EN_TILE) & (o == q)) and kx[S.db[q] - da] > 0:
                _add(ev, "cc keep: a later node's kept dest compacted across a tile edge")
    for q in range(a, b):
        S.NDE[q] = kx[S.db[q] + S.ndest[q] - da] - kx[S.db[q] - da]
    fv = np.zeros(nv, np.int64)
    rw = np.zeros(nv, np.int64)
    t = np.arange(nv)
    p = va + t
    o = _node_of(S.vb, a, b, p, mut)
    end = S.VO[S.ob[o] + S.nrows[o]]
    used = p < end
    if ev is not None and np.any(~used & (S.vcap[o] > 0)):
        _add(ev, "cc filter: the slack of a value room")
    key = p + (0 if "row search at p" in mut else 1)
    for q in np.unique(o[used]):
        sel = np.flatnonzero(used & (o == q))
        offs = S.VO[S.ob[q]:S.ob[q] + S.nrows[q] + 1]
        if np.all(np.diff(offs) >= 0):
            r = np.searchsorted(offs, key[sel], "left") - 1
        else:
            r = np.array([_lower_bound(offs, offs.size, k) - 1 for k in key[sel]])
        x = S.V[p[sel]]
        start = np.where(r >= 0, offs[np.maximum(r, 0)], BIG)
        prev = S.V[np.maximum(p[sel] - 1, 0)]
        desc = (start != p[sel]) & (prev >= x)
        if ev is not None and np.any((start == p[sel]) & ((p[sel] - va) % NT == 0) &
                                     (offs[np.maximum(r - 1, 0)] == p[sel]) & (r > 0)):
            _add(ev, "cc filter: a row after empty rows starts on a CTA edge")
        if ev is not None and np.any((start == p[sel]) & (prev >= x) & (p[sel] > S.vb[q])):
            _add(ev, "cc filter: a row that descends from the row before")
        if desc.any():
            if S.ordered[q]:
                if ev is not None:
                    _add(ev, "cc filter: an ORDERED row that descends")
            else:
                _refuse(S, ev, "row order", t[sel][desc], L["depth"])
        if S.mode[q] == KEEP:
            f = np.ones(sel.size, bool)
        else:
            dest = S.D[S.db[q]:S.db[q] + S.ndest[q]]
            j = np.searchsorted(dest, x, "left")
            jj = np.minimum(j, max(dest.size - 1, 0))
            f = (j < dest.size) & (dest[jj] == x) if dest.size else np.zeros(sel.size, bool)
            if S.mode[q] == NEW:
                f &= keep[np.minimum(S.db[q] - da + jj, max(nd - 1, 0))].astype(bool) if nd else False
            if ev is not None and not f.all():
                _add(ev, "cc filter: a value dropped by OLD" if S.mode[q] == OLD else "cc filter: a value dropped by NEW")
        f &= r >= 0      # a mutant's row before the node: read outside its offsets
        fv[sel] = f
        rw[sel] = r
    return fv, rw


def _page_kernel(S, L, fv, rw, fx, ev, mut):
    """cc_page_kernel: a NEW node's surviving value stays iff its rank in its row is inside the row's page."""
    a, b, va, nv = L["a"], L["b"], L["va"], L["nv"]
    t = np.flatnonzero(fv[:nv])
    o = _node_of(S.vb, a, b, va + t, mut)
    new = S.mode[o] == NEW
    t, o = t[new], o[new]
    out = fv.copy()
    rows = {}
    for tt, q in zip(t, o):
        r = rw[tt]
        rs, re = S.VO[S.ob[q] + r] - va, S.VO[S.ob[q] + r + 1] - va
        n = (re - rs) if "page on the pre-filter length" in mut else fx[re] - fx[rs]
        s, e = _page_range(int(S.first[q]), int(S.offset[q]), int(n), mut)
        rank = fx[tt] - (0 if "row rank relative to the level" in mut else fx[rs])
        keep = s <= rank < e
        if not keep:
            out[tt] = 0
        if ev is not None:
            rows.setdefault((q, r), []).append((tt, keep))
            if (q, r) not in getattr(S, "paged_rows", set()):
                S.paged_rows = getattr(S, "paged_rows", set()) | {(q, r)}
                _page_events(ev, int(S.first[q]), int(S.offset[q]), int(fx[re] - fx[rs]), int(re - rs))
    if ev is not None:
        for (q, r), vals in rows.items():
            edges = {tt // EN_TILE for tt, _ in vals}
            if len(edges) < 2:
                continue
            kept = [tt for tt, k in vals if k]
            if kept and len({tt // EN_TILE for tt in kept}) > 1:
                _add(ev, "cc page: kept values on both sides of a tile edge")
                dropped = [tt for tt, k in vals if not k]
                if dropped and min(dropped) < min(kept) and max(dropped) > max(kept):
                    _add(ev, "cc page: the page cut on both sides of a tile edge")
    return out


def _compact_kernel(S, L, fv, fy, mut, values=True):
    """cc_compact_kernel: the kept values to the front of their node's slots, and the new row offsets."""
    a, b, va, nv, oa, no = L["a"], L["b"], L["va"], L["nv"], L["oa"], L["no"]
    if values:
        t = np.flatnonzero(fv[:nv])
        o = _node_of(S.vb, a, b, va + t, mut)
        idx = S.vb[o] + fy[t] - fy[S.vb[o] - va]
        S.OV[idx] = S.V[va + t]
    q = oa + np.arange(no)
    o = _node_of(S.ob, a, b, q, mut)
    S.OO[q] = S.vb[o] + fy[S.VO[q] - va] - fy[S.vb[o] - va]


# ---- @cascade ---------------------------------------------------------------------------------------------------------

CcCase = namedtuple("CcCase", "nodes slack v_off forms")   # slack: {k: values of node k's room past its rows} (device
#                                                            form); v_off: {k: node k's offsets} (device form)
CcOut = namedtuple("CcOut", "rc sync sizes out out_off dest_out dest_off launches")


def cc_case(nodes, slack=None, v_off=None, forms=("host", "dev")):
    return CcCase(nodes, slack or {}, v_off or {}, forms if not v_off else ("dev",))


def cc_inputs(case: CcCase, form: str):
    """Per node in node order: (v with its room, v_off, nrows, v_cap, dest, has_val) as the call gets them."""
    src = []
    for k, nd in enumerate(case.nodes):
        lens = [r.size for r in nd.rows]
        off = np.zeros(len(lens) + 1, np.uint64)
        if any(lens):
            np.cumsum(lens, out=off[1:])
        v = np.concatenate(list(nd.rows)).astype(np.uint64) if any(lens) else np.zeros(0, np.uint64)
        if form == "dev":
            v = np.concatenate([v, np.asarray(case.slack.get(k, ()), np.uint64)])
            if k in case.v_off:
                off = np.asarray(case.v_off[k], np.uint64)
        src.append((v, off, len(lens), v.size, nd.dest, nd.has_val))
    return src


def cc_plan(nodes, src, ev):
    """cc_plan: the level order, the slot bases and the levels (with a flag for work)."""
    n = len(nodes)
    depth = []
    for nd in nodes:
        depth.append(0 if nd.parent < 0 else depth[nd.parent] + 1)
    order = sorted(range(n), key=lambda k: (-depth[k], k))
    pos = np.empty(n, np.int64)
    pos[order] = np.arange(n)
    S = _State()
    S.id = np.array(order, np.int64)
    S.depth = np.array([depth[k] for k in order], np.int64)
    cnt = lambda j: np.array([src[k][j] for k in order], np.int64)  # noqa: E731
    S.vcap, S.nrows = cnt(3), cnt(2)
    S.ndest = np.array([src[k][4].size for k in order], np.int64)
    S.nhv = np.array([src[k][5].size for k in order], np.int64)
    for f, c in (("vb", S.vcap), ("ob", S.nrows + 1), ("db", S.ndest), ("hb", S.nhv)):
        base = np.zeros(n + 1, np.int64)
        np.cumsum(c, out=base[1:])
        setattr(S, f, base[:n])
        setattr(S, f.replace("b", "tot"), int(base[n]))
    out_row = np.zeros(n + 1, np.int64)
    np.cumsum([src[k][2] for k in range(n)], out=out_row[1:])
    S.out_row = out_row[S.id]
    S.rows = int(out_row[n])
    checked = [[] for _ in range(n)]
    for k, nd in enumerate(nodes):
        if nd.parent >= 0 and nd.flags & CC_CHECKED:
            checked[nd.parent].append(int(pos[k]))
    S.mode, S.prune, S.ordered = (np.zeros(n, np.int64) for _ in range(3))
    S.first, S.offset, S.counts_len, S.ck_b, S.ck_e = (np.zeros(n, np.int64) for _ in range(5))
    ck = []
    for q, k in enumerate(order):
        nd = nodes[k]
        root, cascade, skip = nd.parent < 0, bool(nd.flags & CC_CASCADE), bool(nd.flags & CC_SKIP)
        paged = cascade and (not root or nd.first != 0 or nd.offset != 0)
        S.mode[q] = NEW if paged else OLD if nd.flags & CC_FILTERED and not skip else KEEP
        S.prune[q] = cascade and not skip
        S.ordered[q] = bool(nd.flags & CC_ORDERED)
        S.first[q], S.offset[q] = (nd.first, nd.offset) if paged else (0, 0)
        S.counts_len[q] = nd.counts_len
        S.ck_b[q] = len(ck)
        if S.prune[q]:
            ck += checked[k]
        S.ck_e[q] = len(ck)
    S.ck = np.array(ck, np.int64)
    levels = []
    maxd = max(depth) if n else -1
    bounds = np.searchsorted(-S.depth, np.arange(-maxd, 1), "left").tolist() + [n]
    for i, d in enumerate(range(maxd, -1, -1)):
        a, b = bounds[i], bounds[i + 1]
        L = {"a": a, "b": b, "depth": d, "va": int(S.vb[a]), "nv": int(S.vb[b - 1] + S.vcap[b - 1] - S.vb[a]),
             "da": int(S.db[a]), "nd": int(S.db[b - 1] + S.ndest[b - 1] - S.db[a]), "oa": int(S.ob[a]),
             "no": int(S.ob[b - 1] + S.nrows[b - 1] + 1 - S.ob[a])}
        L["work"] = L["nv"] > 0 or L["nd"] > 0
        levels.append(L)
        if ev is None:
            continue
        for field, cnts, name in ((S.vb, S.vcap, "value"), (S.db, S.ndest, "dest"), (S.hb, S.nhv, "has_val")):
            c = cnts[a:b]
            nz = np.flatnonzero(c)
            if nz.size:
                z = np.flatnonzero(c == 0)
                if np.any(z < nz[0]):
                    _add(ev, f"cc space: a zero-slot node first in a level's {name} slots")
                if np.any((z > nz[0]) & (z < nz[-1])):
                    _add(ev, f"cc space: a zero-slot node between {name} slots")
                if np.any(z > nz[-1]):
                    _add(ev, f"cc space: a zero-slot node last in a level's {name} slots")
        for field, cnts, base, name in ((S.vb, S.vcap, L["va"], "value"), (S.db, S.ndest, L["da"], "dest")):
            rel = field[a:b][cnts[a:b] > 0] - base
            if np.any((rel > 0) & (rel % NT == 0)):
                _add(ev, f"cc space: a node's first {name} slot on a CTA edge")
            if np.any((rel > 0) & (rel % EN_TILE == 0)):
                _add(ev, f"cc space: a node's first {name} slot on a tile edge")
        if L["nv"] > 2 * EN_TILE:
            _add(ev, "cc space: a level's values in 3 or more tiles")
    if ev is not None and n:
        work = [L["work"] for L in levels]
        for i, L in enumerate(levels):
            if not L["work"] and any(work[:i]) and any(work[i + 1:]):
                _add(ev, "cc plan: a level without work between levels with work")
        if not levels[-1]["work"] and any(work):
            _add(ev, "cc plan: the root level without work")
        if maxd == K["CC_MAX_DEPTH"] - 1:
            _add(ev, "cc plan: a node at depth kCcMaxDepth - 1")
        if 2 <= sum(work) <= 63:
            _add(ev, "cc plan: 2 to 63 levels with work")
        if n == K["CC_MAX_NODES"] - 1:
            _add(ev, "cc plan: a forest of 2^16 - 1 nodes")
    return S, levels


def cc_run(case: CcCase, form: str, mut=frozenset(), ev=None) -> CcOut:
    """One call of dgx_cascade ("host") or dgx_dev_cascade ("dev") through the model."""
    nodes = case.nodes
    n = len(nodes)
    src = cc_inputs(case, form)
    nrows = sum(s[2] for s in src)
    empty = CcOut(OK, OK if form == "dev" else None, np.zeros(2, np.int64), np.zeros(0, np.uint64),
                  np.zeros(nrows + 1, np.int64), np.zeros(0, np.uint64), np.zeros(n + 1, np.int64), 0)
    refused = CcOut(OK, ERR_ARG, np.zeros(2, np.int64), None, None, None, None, None) if form == "dev" else \
        CcOut(ERR_ARG, None, None, None, None, None, None, None)
    if n == 0 or (form == "host" and sum(s[3] for s in src) == 0 and sum(s[4].size for s in src) == 0):
        return empty
    S, levels = cc_plan(nodes, src, ev)
    work = [L for L in levels if L["work"]]
    if not work:
        return empty
    launches = cp.launches(len(work))
    refused = refused._replace(launches=launches)
    S.bad = False
    oq = [src[k] for k in S.id]
    # cc_gather_kernel
    S.V = np.concatenate([s[0] for s in oq] + [np.zeros(0, np.uint64)]).astype(np.uint64)
    if "node_of takes the first of equal bases" in mut and S.vtot:
        t = np.arange(S.vtot)
        o = _node_of(S.vb, 0, n, t, mut)
        j = t - S.vb[o]
        V = np.full(S.vtot, POISON, np.uint64)
        ok = j < S.vcap[o]
        V[ok] = S.V[(S.vb[o] + j)[ok]]
        S.V = V
    off = np.concatenate([s[1] for s in oq]).astype(np.int64)   # thread t: offset slot t of node qi[t]
    qi = np.repeat(np.arange(n), S.nrows + 1)
    r = np.arange(S.otot) - S.ob[qi]
    start = np.where(r == 0, off != 0, False)
    decrease = (r > 0) & (off < np.r_[0, off[:-1]])
    past = (r == S.nrows[qi]) & (off > S.vcap[qi])
    for kind, bad in (("offset start", start), ("offset decrease", decrease), ("offset past room", past)):
        if bad.any():
            _refuse(S, ev, kind, np.flatnonzero(bad), None)
    if S.bad:
        return refused
    VO = S.vb[qi] + off
    S.VO, S.OO = VO, VO.copy()
    S.D = np.concatenate([s[4] for s in oq] + [np.zeros(0, np.uint64)]).astype(np.uint64)
    S.H = np.concatenate([s[5] for s in oq] + [np.zeros(0, np.uint8)]).astype(np.uint8)
    if "node_of takes the first of equal bases" in mut:
        for arr, base, cnts in (("D", S.db, S.ndest), ("H", S.hb, S.nhv)):
            A = getattr(S, arr)
            t = np.arange(A.size)
            o = _node_of(base, 0, n, t, mut)
            j = t - base[o]
            B = np.full(A.size, POISON if arr == "D" else 0x5A, A.dtype)
            ok = j < cnts[o]
            B[ok] = A[(base[o] + j)[ok]]
            setattr(S, arr, B)
    if ev is not None:
        for q, s in enumerate(oq):
            if s[3] > s[1][-1] and (S.vb[q] + int(s[1][-1])) // EN_TILE != (S.vb[q] + s[3] - 1) // EN_TILE:
                _add(ev, "cc space: a device value room with slack across a tile edge")
    S.NDE = S.ndest.copy()
    S.ND = np.full(S.dtot, POISON, np.uint64)
    S.OV = np.full(S.vtot, POISON, np.uint64)
    for L in work:
        if ev is not None:
            modes = set(S.mode[L["a"]:L["b"]].tolist())
            if modes == {KEEP, OLD, NEW}:
                _add(ev, "cc filter: KEEP, OLD and NEW nodes in one level")
            offs = S.VO[L["oa"]:L["oa"] + L["no"]] - L["va"]
            inner = offs[(offs > 0) & (offs < L["nv"])]
            if np.any(inner % NT == 0):
                _add(ev, "cc space: a row boundary on a CTA edge")
                u, c = np.unique(inner[inner % NT == 0], return_counts=True)
                if np.any(c > 1):
                    _add(ev, "cc space: empty rows sharing an offset on a CTA edge")
            if np.any(np.diff(offs) == NT):
                _add(ev, "cc space: a row of 256 values")
        keep = _keep_kernel(S, L, ev, mut)
        if S.bad:
            return refused
        kx = _scan(keep, L["nd"], ev, "cc scan: keep flags over 2 tiles with a carry", mut)
        fv, rw = _filter_kernel(S, L, keep, kx, ev, mut)
        if S.bad:
            return refused
        fx = _scan(fv, L["nv"], ev, "cc scan: value flags over 2 tiles with a carry", mut)
        fv = _page_kernel(S, L, fv, rw, fx, ev, mut)
        fy = _scan(fv, L["nv"], ev, None, mut)
        _compact_kernel(S, L, fv, fy, mut)
    # cc_count_kernel, the node-order count scan, cc_place_kernel
    NN = n
    cnt = np.zeros(2 * NN, np.int64)
    cnt[S.id] = S.OO[S.ob + S.nrows] - S.vb
    cnt[NN + S.id] = S.NDE
    if ev is not None:
        tiles = -(-2 * NN // EN_TILE)
        _add(ev, {1: "cc scan: node-order counts in 1 tile", 2: "cc scan: node-order counts over 2 tiles"}.get(
            tiles, "cc scan: node-order counts over 64 tiles" if tiles == 64 else "cc scan: node-order counts in 1 tile"))
    if "count scan over NN" in mut:
        cx = np.full(2 * NN + 1, BIG, np.int64)
        cx[:NN + 1] = _scan(cnt, NN, None, None, mut)
    else:
        cx = _scan(cnt, 2 * NN, None, None, mut)
    dbase = int(cx[NN])
    out = np.full(S.vtot, POISON, np.uint64)
    out_off = np.zeros(S.rows + 1, np.int64)
    dest_out = np.full(S.dtot, POISON, np.uint64)
    t = np.arange(S.vtot)
    o = _node_of(S.vb, 0, n, t, mut)
    sel = t < S.OO[S.ob[o] + S.nrows[o]]
    idx = cx[S.id[o[sel]]] + t[sel] - S.vb[o[sel]]
    ok = (idx >= 0) & (idx < out.size)
    out[idx[ok]] = S.OV[t[sel][ok]]
    row = r < S.nrows[qi]
    out_off[(S.out_row[qi] + r)[row]] = (cx[S.id[qi]] + S.OO - S.vb[qi])[row]
    t = np.arange(S.dtot)
    o = _node_of(S.db, 0, n, t, mut)
    sel = t - S.db[o] < S.NDE[o]
    idx = cx[NN + S.id[o[sel]]] - dbase + t[sel] - S.db[o[sel]]
    ok = (idx >= 0) & (idx < dest_out.size)
    dest_out[idx[ok]] = S.ND[t[sel][ok]]
    dest_off = np.append(cx[NN:2 * NN] - dbase, cx[2 * NN] - dbase)
    out_off[S.rows] = dbase
    sizes = np.array([dbase, cx[2 * NN] - dbase], np.int64)
    return CcOut(OK, OK if form == "dev" else None, sizes, out, out_off, dest_out, dest_off, launches)


def cc_malformed(case: CcCase, form: str) -> bool:
    """The inputs break dgx.h's rules: a dest or an unordered row that does not strictly ascend, or (device form)
    offsets that do not start at 0, decrease or end past the room."""
    for k, (v, off, nrows, cap, dest, _) in enumerate(cc_inputs(case, form)):
        if np.any(dest[1:] <= dest[:-1]):
            return True
        o = off.astype(np.int64)
        if o[0] != 0 or np.any(np.diff(o) < 0) or o[-1] > cap:
            return True
        if not case.nodes[k].flags & CC_ORDERED:
            for r in range(nrows):
                row = v[o[r]:o[r + 1]]
                if np.any(row[1:] <= row[:-1]):
                    return True
    return False


def cc_expected(case: CcCase, form: str):
    """The restatement's (cascade_oracle.c) answer in the model's terms: None for a refused call, else (sizes, out,
    out_off, dest_out, dest_off)."""
    import cascade_oracle as co
    from dgraph_b200.algo import cascade_arrays

    if cc_malformed(case, form):
        return None
    a = cascade_arrays(case.nodes)
    out, out_off, dest_out, dest_off = co.cascade_flat(a)
    K_, D_ = int(out_off[-1]), int(dest_off[-1])
    return np.array([K_, D_], np.int64), out[:K_], out_off.astype(np.int64), dest_out[:D_], dest_off.astype(np.int64)


def cc_agrees(o: CcOut, w, form) -> bool:
    if w is None:
        return (o.rc, o.sync) == ((OK, ERR_ARG) if form == "dev" else (ERR_ARG, None)) and \
            (form != "dev" or list(o.sizes) == [0, 0])
    sizes, out, out_off, dest_out, dest_off = w
    if (o.rc, o.sync) != ((OK, OK) if form == "dev" else (OK, None)):
        return False
    return (np.array_equal(o.sizes, sizes) and np.array_equal(o.out_off, out_off) and
            np.array_equal(o.dest_off, dest_off) and np.array_equal(o.out[:sizes[0]], out) and
            np.array_equal(o.dest_out[:sizes[1]], dest_out))


# ---- @filter ----------------------------------------------------------------------------------------------------------

SfCall = namedtuple("SfCall", "form counts_only")   # form "host", "dev" (no length words) or "dev_words"
SfCase = namedtuple("SfCase", "tree leaves d0 rows count offset d0_slack v_slack list_slack d0_word list_words v_off")
SfOut = namedtuple("SfOut", "rc sync dest_len dest out out_off counts launches")
HI = 0x7F << 40     # garbage above a length word's low 32 bits


def sf_case(tree, leaves, d0, rows, count=0, offset=0, d0_slack=(), v_slack=(), list_slack=(), d0_word=None,
            list_words=None, v_off=None):
    return SfCase(tree, leaves, np.asarray(d0, np.uint64), [np.asarray(r, np.uint64) for r in rows], count, offset,
                  np.asarray(d0_slack, np.uint64), np.asarray(v_slack, np.uint64), np.asarray(list_slack, np.uint64),
                  d0_word, list_words, v_off)


def sf_inputs(case: SfCase, call: SfCall) -> dict:
    """The arrays and sizes of the call: D0 with its slack and d0_cap, its length word, the leaves (LIST: uids with
    room and length word; COUNT: counts or offsets over d0_cap), the values with v_cap and the offsets."""
    words = call.form == "dev_words"
    n0 = case.d0.size
    d0 = np.concatenate([case.d0, case.d0_slack]) if words else case.d0.copy()
    d0_cap = d0.size
    lens = [r.size for r in case.rows]
    v_off = np.zeros(len(lens) + 1, np.uint64)
    np.cumsum(lens, out=v_off[1:])
    v = np.concatenate(case.rows).astype(np.uint64) if sum(lens) else np.zeros(0, np.uint64)
    if call.form != "host":
        v = np.concatenate([v, case.v_slack])
        if case.v_off is not None:
            v_off = np.asarray(case.v_off, np.uint64)
    leaves, li = [], 0
    for lf in case.leaves:
        if lf[0] == "list":
            u = np.asarray(lf[1], np.uint64)
            d = {"kind": "list", "p": u, "room": u.size, "word": None}
            if words:
                d["p"] = np.concatenate([u, case.list_slack])
                d["room"] = d["p"].size
                d["word"] = (case.list_words[li] if case.list_words is not None else u.size) | HI
            li += 1
        else:
            a = np.asarray(lf[3], np.uint32 if lf[0] == "count" else np.uint64)
            pad = d0_cap - n0
            if pad:
                a = np.concatenate([a, np.full(pad, 0 if lf[0] == "count" else a[-1], a.dtype)])
            d = {"kind": lf[0], "cmp": lf[1], "thr": int(lf[2]), "a": a}
        leaves.append(d)
    word = ((case.d0_word if case.d0_word is not None else n0) | HI) if words else None
    return {"d0": d0, "d0_cap": d0_cap, "d0_word": word, "leaves": leaves, "v": v, "v_off": v_off,
            "nrows": len(lens), "v_cap": v.size}


def sf_program(tree):
    """sf_check_args's pre-order program: (w0, w1) per entry."""
    f = sg_filter_flat(tree)
    n, op, parent, leaf = f["nnodes"], f["op"], f["parent"], f["leaf"]
    kids = [[] for _ in range(n)]
    for k in range(1, n):
        kids[int(parent[k])].append(k)
    end = [0] * n
    for k in range(n - 1, -1, -1):   # sg_filter_flat numbers in pre-order: pos[k] = k
        end[k] = k + 1 if not kids[k] else end[kids[k][-1]]
    prog = []
    for k in range(n):
        pe = NO_PARENT if k == 0 else int(parent[k])
        prog.append((int(leaf[k]), pe) if op[k] == 0 else (NODE | int(op[k]) << 28 | end[k], pe))
    return prog


def _walk(prog, verdict, mut, ev):
    """sf_eval_kernel's walk for one D0 value whose leaves hold as `verdict` says: (keep, levels each leaf closed)."""
    cur, pc, r = NO_PARENT, 0, False
    closes = []
    while True:
        if pc >= len(prog):
            return None, closes   # a mutant's walk past the program: the kernel reads what lies beyond it
        w0, w1 = prog[pc]
        if w0 & NODE:
            _add(ev, "sf eval: opening a node")
            cur = pc
            pc += 1
            continue
        r = bool(verdict[w0])
        _add(ev, "sf eval: a leaf hit" if r else "sf eval: a leaf miss")
        pc += 1
        closed, nots = [], 0
        while True:
            if cur == NO_PARENT:
                closes.append((closed, True))
                return int(r), closes
            f0, f1 = prog[cur]
            op, end = (f0 >> 28) & 7, f0 & END_MASK
            if op == SF_NOT and "NOT decoded as OR" in mut:
                op = SF_OR
            if op == SF_NOT:
                r = not r
            elif (op == SF_AND) == r and (pc != end or "eval without pc != end" in mut):
                break
            closed.append((op, pc == end, r, end - cur))
            pc = end
            cur = f1
        closes.append((closed, False))


def _walk_events(prog, closes, ev):
    for closed, at_root in closes:
        if at_root and not closed:
            _add(ev, "sf eval: the walk ends at a leaf root")
        if not at_root:
            _add(ev, "sf eval: the close loop goes on to a next child")
        lv = len(closed)
        if lv == 64:
            _add(ev, "sf eval: one leaf closes 64 levels")
        elif lv >= 2:
            _add(ev, "sf eval: one leaf closes 2 to 63 levels")
        run = 0
        for op, _, _, _ in closed + [(None, 0, 0, 0)]:
            if op == SF_NOT:
                run += 1
                continue
            if run >= 2:
                _add(ev, "sf eval: an odd chain of NOTs closed by one leaf" if run % 2 else
                     "sf eval: an even chain of NOTs closed by one leaf")
            run = 0
        for op, last, r, size in closed:
            if op == SF_AND and size == 2:
                _add(ev, "sf eval: an AND of one child")
            if op == SF_OR and size == 2:
                _add(ev, "sf eval: an OR of one child")
            if op == SF_AND and not r:
                _add(ev, "sf eval: an AND decided by a miss at its last child" if last else
                     "sf eval: an AND stopped by a miss before its last child")
            if op == SF_OR and r:
                _add(ev, "sf eval: an OR decided by a hit at its last child" if last else
                     "sf eval: an OR stopped by a hit before its last child")


def _holds(lf, i, x, n0):
    """sf_leaf_holds over the first n0 D0 values at once."""
    if lf["kind"] == "list":
        n = lf["n"]
        return np.isin(x, lf["p"][:n])
    a = lf["a"]
    c = [int(v) for v in a[:n0]] if lf["kind"] == "count" else \
        [int(a[j + 1]) - int(a[j]) for j in range(n0)]
    thr = lf["thr"]
    op = {"le": lambda u: u <= thr, "ge": lambda u: u >= thr, "lt": lambda u: u < thr, "gt": lambda u: u > thr,
          "eq": lambda u: u == thr}[lf["cmp"]]
    return np.array([op(u) for u in c], bool)


def sf_run(case: SfCase, call: SfCall, mut=frozenset(), ev=None) -> SfOut:
    """One call of dgx_sg_filter ("host") or dgx_dev_sg_filter ("dev", "dev_words") through the model."""
    ev = set() if ev is None else ev
    I = sf_inputs(case, call)
    host = call.form == "host"
    d0, d0_cap, nrows, v_cap = I["d0"], I["d0_cap"], I["nrows"], I["v_cap"]
    v, v_off = I["v"], I["v_off"].astype(np.int64)
    if call.counts_only:
        _add(ev, "sf out: counts-only")
    if d0_cap == 0:
        return SfOut(OK, None if host else OK, 0, np.zeros(0, np.uint64), None if call.counts_only else
                     np.zeros(0, np.uint64), np.zeros(nrows + 1, np.int64), np.zeros(nrows, np.int64), 0)
    prog = sf_program(case.tree)
    # the leaf table and its check slots
    slots, sb = 0, []
    for lf in I["leaves"]:
        sb.append(slots)
        if lf["kind"] == "list":
            slots += lf["room"] + 1
        elif lf["kind"] == "len":
            slots += d0_cap
    nl = len(I["leaves"])
    sizes = [(lf["room"] + 1 if lf["kind"] == "list" else d0_cap if lf["kind"] == "len" else 0) for lf in I["leaves"]]
    z = [j for j, s in enumerate(sizes) if s == 0]
    nz = [j for j, s in enumerate(sizes) if s]
    if z and nz:
        if z[0] < nz[0]:
            _add(ev, "sf space: a zero-slot leaf first")
        if any(nz[0] < j < nz[-1] for j in z):
            _add(ev, "sf space: a zero-slot leaf between others")
        if z[-1] > nz[-1]:
            _add(ev, "sf space: a zero-slot leaf last")
    if any(lf["kind"] == "list" and lf["room"] == 0 for lf in I["leaves"]):
        _add(ev, "sf space: a LIST leaf of room 0")
    if any(s > 0 and s % NT == 0 for s, c in zip(sb, sizes) if c):
        _add(ev, "sf space: a leaf boundary on a CTA edge")
    T = max(d0_cap, slots, nrows + 1, v_cap)
    if slots > max(d0_cap, v_cap, nrows + 1):
        _add(ev, "sf space: check slots past d0_cap, v_cap and nrows")
    if nrows > d0_cap:
        _add(ev, "sf space: nrows above d0_cap")
    if nrows == 0:
        _add(ev, "sf space: no rows")
    # sf_check_kernel
    bad = False
    word = I["d0_word"]
    if "|D0| read as d0_cap" in mut:
        word = None
    n0 = d0_cap if word is None else word & 0xFFFFFFFF
    if n0 > d0_cap:
        _add(ev, "sf refuse: D0's length word over d0_cap")
        bad, n0 = True, 0
    for e in (255, 256, 257, 2047, 2048, 2049, 4097):
        if n0 == e:
            _add(ev, f"sf space: |D0| of {e}")
    if word is not None and d0_cap - n0 >= EN_TILE:
        _add(ev, "sf space: a length word below d0_cap by a tile")
    if n0 > 1 and np.any(d0[1:n0] <= d0[:n0 - 1]):
        _add(ev, "sf refuse: D0 descends")
        bad = True
    sbs = np.array(sb, np.int64)
    for lf in I["leaves"]:
        if lf["kind"] == "list":
            lf["n"] = lf["room"] if lf["word"] is None else lf["word"] & 0xFFFFFFFF
    for t in range(slots):
        lo = int(np.searchsorted(sbs, t, "right")) - 1
        if "leaf search takes the first of an equal sb" in mut:
            lo = int(np.searchsorted(sbs, sbs[lo], "left"))
        lf, j = I["leaves"][lo], t - sb[lo]
        if lf["kind"] == "list":
            n = lf["n"]
            if n > lf["room"]:
                if j == 0:
                    _add(ev, "sf refuse: a length word over its room")
                    bad = True
                n = 0
            if 0 < j < n and lf["p"][j - 1] >= lf["p"][j]:
                bad = True
                if j == 1:
                    _add(ev, "sf refuse: a LIST descends at its first checked slot")
                if j == n - 1:
                    _add(ev, "sf refuse: a LIST descends at its last checked slot")
            if n <= j < lf["room"] and lf["p"][j] <= lf["p"][j - 1] and j > 0:
                _add(ev, "sf space: a descent in a LIST's slack, accepted")
        elif lf["kind"] == "len" and j < n0 and int(lf["a"][j + 1]) < int(lf["a"][j]):
            _add(ev, "sf refuse: a COUNT leaf's offsets decrease")
            bad = True
    if v_off[0] != 0 or np.any(np.diff(v_off) < 0) or v_off[nrows] > v_cap:
        _add(ev, "sf refuse: row offsets")
        bad = True
    nv = min(int(v_off[nrows]), v_cap)
    if v_off[0] == 0 and nv > 1:
        desc = np.flatnonzero(v[1:nv] <= v[:nv - 1]) + 1
        for t in desc:
            r = _lower_bound(v_off, nrows + 1, t + 1) - 1
            if v_off[r] != t:
                _add(ev, "sf refuse: a row descends")
                bad = True
    if int(v_off[nrows]) < v_cap and int(v_off[nrows]) // EN_TILE != (v_cap - 1) // EN_TILE:
        _add(ev, "sf space: v_off[nrows] below v_cap across a tile edge")
    launches = sp.launches(d0_cap)
    if bad:
        if host:
            return SfOut(ERR_ARG, None, None, None, None, None, None, launches)
        return SfOut(OK, ERR_ARG, 0, None, None, None, None, launches)
    # sf_eval_kernel
    keep = np.zeros(d0_cap, np.int64)
    if n0:
        x = d0[:n0]
        hold = np.array([_holds(lf, None, x, n0) for lf in I["leaves"]]).reshape(nl, n0)
        if any(lf["kind"] != "list" and any(int(lf["a"][j + 1]) - int(lf["a"][j]) >= 1 << 32 for j in range(n0))
               for lf in I["leaves"] if lf["kind"] == "len"):
            _add(ev, "sf space: a count of 2^32 or more")
        cols, inv = np.unique(hold, axis=1, return_inverse=True)
        res = []
        for c in range(cols.shape[1]):
            r, closes = _walk(prog, cols[:, c], mut, ev)
            _walk_events(prog, closes, ev)
            res.append(r)
        if None in res:
            return SfOut(OK, None if host else OK, None, None, None, None, None, launches)
        keep[:n0] = np.array(res, np.int64)[np.asarray(inv).reshape(-1)]
    if n0 < d0_cap and word is not None:   # the slack's verdicts over the padded leaf arrays
        hold = np.array([_holds(lf, None, d0, d0_cap) for lf in I["leaves"]]).reshape(nl, d0_cap)
        if any(_walk(prog, hold[:, i], mut, set())[0] == 1 for i in range(n0, min(d0_cap, n0 + 8))):
            _add(ev, "sf eval: slack D0 values that hold, not evaluated")
    if len(prog) == K["SGF_MAX_NODES"]:
        _add(ev, "sf eval: a program of the node limit")
    used = {w0 for w0, _ in prog if not w0 & NODE}
    if nl == K["SGF_MAX_LEAVES"] and len(used) == nl - 1:
        _add(ev, "sf eval: a leaf table of the leaf limit, one entry never evaluated")
    # cascade's level kernels over one NEW node
    S = _State()
    for f, val in (("vb", 0), ("vcap", v_cap), ("ob", 0), ("nrows", nrows), ("db", 0), ("ndest", n0), ("hb", 0),
                   ("nhv", 0), ("mode", NEW), ("ordered", 1), ("first", case.count), ("offset", case.offset)):
        setattr(S, f, np.array([val], np.int64))
    S.bad = False
    S.V, S.VO, S.D = v, v_off, d0
    S.ND = np.full(d0_cap, POISON, np.uint64)
    S.NDE = np.zeros(1, np.int64)
    S.OV = np.full(max(v_cap, 1), POISON, np.uint64)
    S.OO = np.zeros(nrows + 1, np.int64)
    L = {"a": 0, "b": 1, "depth": None, "va": 0, "nv": v_cap, "da": 0, "nd": d0_cap, "oa": 0, "no": nrows + 1}
    kx = _scan(keep, n0, ev, None, mut)
    kx = np.concatenate([kx, np.full(d0_cap - n0, BIG, np.int64)])
    fv, rw = _filter_kernel(S, L, keep, kx, None, mut)
    n1 = int(S.NDE[0])
    for e, name in ((0, "sf d1: empty"), (2048, "sf d1: 2048 values"), (2049, "sf d1: 2049 values")):
        if n1 == e:
            _add(ev, name)
    wv = int(v_off[nrows])
    fx = _scan(fv, wv, None, None, mut)
    fv = _page_kernel(S, L, fv, rw, fx, None, mut)
    fy = _scan(fv, wv, None, None, mut)
    _compact_kernel(S, {**L, "nv": 0} if call.counts_only else L, fv, fy, mut, values=not call.counts_only)
    # sf_mark_kernel, the mark scan, sf_out_kernel
    d1 = S.ND[:n1]
    paged = case.count != 0 or case.offset != 0
    mark = np.zeros(d0_cap, np.int64)
    if not paged or "sf_mark marks all of D1 when paged" in mut:
        mark[:n1] = 1
        if not paged:
            _add(ev, "sf d2: unpaged")
    if paged:
        hit = np.searchsorted(d1, v[np.flatnonzero(fv[:v_cap])], "left")
        mark[hit] = 1
        if n1 and not np.all(np.isin(np.arange(n1), hit)):
            _add(ev, "sf d2: paged, a D1 value no kept row holds")
    mx = _scan(mark, n1, None, None, mut)
    dest = np.full(d0_cap, POISON, np.uint64)
    t = np.flatnonzero(mark[:n1])
    dest[mx[t]] = d1[t]
    dl = int(mx[n1])
    counts = (S.OO[1:] - S.OO[:-1]) & 0xFFFFFFFF
    out = None if call.counts_only else S.OV
    return SfOut(OK, None if host else OK, dl, dest, out, S.OO.copy(), counts, launches)


def sf_malformed(case: SfCase, call: SfCall) -> bool:
    """The inputs break dgx.h's rules: a length word over its room, D0 or a LIST that does not strictly ascend, COUNT
    offsets or row offsets that decrease, row offsets that do not start at 0 or end past v_cap, a row that does not
    strictly ascend."""
    I = sf_inputs(case, call)
    n0 = I["d0_cap"] if I["d0_word"] is None else I["d0_word"] & 0xFFFFFFFF
    if n0 > I["d0_cap"] or np.any(I["d0"][1:n0] <= I["d0"][:max(n0 - 1, 0)]):
        return True
    for lf in I["leaves"]:
        if lf["kind"] == "list":
            n = lf["room"] if lf["word"] is None else lf["word"] & 0xFFFFFFFF
            if n > lf["room"] or np.any(lf["p"][1:n] <= lf["p"][:max(n - 1, 0)]):
                return True
        elif lf["kind"] == "len" and np.any(lf["a"][1:n0 + 1].astype(object) < lf["a"][:n0].astype(object)):
            return True
    o = I["v_off"].astype(np.int64)
    if o[0] != 0 or np.any(np.diff(o) < 0) or o[-1] > I["v_cap"]:
        return True
    rows = (I["v"][o[r]:o[r + 1]] for r in range(I["nrows"]))
    return any(np.any(row[1:] <= row[:-1]) for row in rows)


def sf_oracle_args(case: SfCase, call: SfCall):
    """(tree, leaves, d0, rows, count, offset) of the call as sg_filter_oracle takes them: the first |D0| values, each
    LIST's first word-length uids, the rows the offsets cut."""
    I = sf_inputs(case, call)
    n0 = I["d0_cap"] if I["d0_word"] is None else I["d0_word"] & 0xFFFFFFFF
    leaves = []
    for lf, orig in zip(I["leaves"], case.leaves):
        if lf["kind"] == "list":
            n = lf["room"] if lf["word"] is None else lf["word"] & 0xFFFFFFFF
            leaves.append(("list", lf["p"][:n]))
        else:
            leaves.append((lf["kind"], lf["cmp"], lf["thr"], lf["a"][:n0 + (lf["kind"] == "len")]))
    o = I["v_off"].astype(np.int64)
    rows = [I["v"][o[r]:o[r + 1]] for r in range(I["nrows"])]
    return case.tree, leaves, I["d0"][:n0], rows, case.count, case.offset


def sf_expected(case: SfCase, call: SfCall):
    """None for a refused call, else sg_filter_oracle's (rows, counts, dest)."""
    import sg_filter_oracle as so

    if sf_malformed(case, call):
        return None
    return so.sg_filter(*sf_oracle_args(case, call))


def sf_agrees(o: SfOut, w, case: SfCase, call: SfCall) -> bool:
    host = call.form == "host"
    if w is None:
        return (o.rc, o.sync) == ((ERR_ARG, None) if host else (OK, ERR_ARG)) and (host or o.dest_len == 0)
    rows, counts, dest = w
    if (o.rc, o.sync) != ((OK, None) if host else (OK, OK)):
        return False
    nrows = len(rows)
    off = np.zeros(nrows + 1, np.int64)
    np.cumsum([r.size for r in rows], out=off[1:])
    if not (o.dest_len == dest.size and np.array_equal(o.dest[:dest.size], dest) and
            np.array_equal(o.counts, counts.astype(np.int64)) and np.array_equal(o.out_off, off)):
        return False
    return call.counts_only or np.array_equal(o.out[:off[-1]], np.concatenate(rows + [np.zeros(0, np.uint64)]))


# ---- fixtures ---------------------------------------------------------------------------------------------------------

CcFix = namedtuple("CcFix", "name cases events kills")
SfFix = namedtuple("SfFix", "name cases calls events kills")
SF_CALLS = (SfCall("host", False), SfCall("dev", False), SfCall("dev_words", False), SfCall("dev_words", True))

C = CC_CASCADE | CC_CHECKED
U = np.uint64


def _u(a):
    return np.asarray(a, np.uint64)


def _node(parent, flags=0, dest=(), rows=(), has_val=(), first=0, offset=0, counts_len=0):
    return CascadeNode(parent, flags, first, offset, counts_len, _u(dest), [_u(r) for r in rows], has_val)


def _rows_of(lens, start=1, step=3):
    """Strictly ascending rows of the given lengths, each starting again from `start` (rows may share uids)."""
    return [start + step * np.arange(n, dtype=np.uint64) for n in lens]


def _straddle(total, first, offset):
    """A level of `total` value slots: a root holding 3 rows' parents, one NEW child whose middle row straddles slot
    EN_TILE; the child's dest drops every 7th uid, so its rows lose values to the filter."""
    lens = [1000, total - 1001, 1]
    rows = _rows_of(lens)
    allv = np.unique(np.concatenate(rows))
    dest = allv[allv % U(7) != U(1)]
    root = _node(-1, CC_CASCADE, [10, 20, 30], [[10, 20, 30]])
    return [root, _node(0, C, dest, rows, first=first, offset=offset)]


def _chain(depth, empty=(), refuse_at=None):
    """A chain of depth + 1 nodes; the nodes at the depths in `empty` have no dest and empty rows (a level without
    work); the node at refuse_at gets a dest that descends."""
    nodes, dest = [], _u([5, 9])
    for d in range(depth + 1):
        parent_dest = nodes[-1].dest if nodes else _u([1])
        if d in empty:
            mine = _u([])
        elif d == refuse_at:
            mine = _u([9, 5])
        else:
            mine = dest
        rows = [np.intersect1d(mine, dest) if mine.size and d != refuse_at else _u([]) for _ in parent_dest]
        nodes.append(_node(d - 1, C if d else CC_CASCADE, mine, rows if nodes else [mine]))
    return nodes


def _forest(nn, every=97):
    """nn roots, mostly empty: every `every`th holds a dest and one row; every 5th holds an empty row."""
    nodes = []
    for k in range(nn):
        if k % every == 3:
            nodes.append(_node(-1, CC_CASCADE, [k + 1, k + 2], [[k + 1, k + 2]], first=1 if k % 2 else 0))
        else:
            nodes.append(_node(-1, 0, [], [[]] if k % 5 == 0 else []))
    return nodes


def cc_fixtures():
    fx = []
    pages = [(100, 850), (-200, 0), (-2**31, 0), (2**31 - 1, 0), (5, 10**6), (50, -3), (0, 900)]
    fx.append(CcFix("value slots across a tile edge",
                    [cc_case(_straddle(T, f, o)) for T in (2047, 2048, 2049, 4097) for f, o in pages],
                    {"cc page: kept values on both sides of a tile edge",
                     "cc page: the page cut on both sides of a tile edge", "cc page: a negative first inside the row",
                     "cc page: a negative first past the row, clamped", "cc page: first reaches past the row",
                     "cc page: an offset past the row", "cc page: a negative offset", "cc page: an offset only",
                     "cc page: first cuts inside the row", "cc scan: value flags over 2 tiles with a carry",
                     "cc space: a level's values in 3 or more tiles", "cc page: a row's survivors fewer than its values"},
                    {"row rank relative to the level", "page on the pre-filter length", "row search at p",
                     "scans without tile carry", "negative count clamp dropped"}))

    def dest_edge(nd):
        # one level of two CASCADE nodes: A holds 1000 dest values, B the rest, straddling dest slot EN_TILE; a
        # checked child of each empties every third row, so every third dest is pruned
        root = _node(-1, CC_CASCADE, [1, 2], [[1, 2]])
        da = 1 + np.arange(1000, dtype=np.uint64)
        db = 1 + np.arange(nd - 1000, dtype=np.uint64)
        a = _node(0, C, da, [da, []])
        b = _node(0, C, db, [[], db])
        ca = _node(1, C, [7], [[7] if i % 3 else [] for i in range(1000)])
        cb = _node(3, C, [7], [[7] if i % 3 else [] for i in range(nd - 1000)])
        return [root, a, ca, b, cb]

    fx.append(CcFix("dest slots across a tile edge", [cc_case(dest_edge(nd)) for nd in (2047, 2048, 2049)],
                    {"cc keep: a later node's kept dest compacted across a tile edge", "cc scan: keep flags over 2 tiles with a carry",
                     "cc keep: a dest pruned"},
                    {"dest rank not relative to its node", "scans without tile carry"}))

    def cta_level(lens_a, gap_nodes):
        # a level of: zero-slot nodes (first), node A with rows of lens_a (empty rows included), a zero-slot node
        # (between), node B whose first value slot sits on a CTA edge, zero-slot nodes (last)
        root = _node(-1, CC_CASCADE, [1, 2, 3, 4], [[1, 2, 3, 4]])
        ra = _rows_of(lens_a)
        allv = np.unique(np.concatenate([r for r in ra if r.size]))
        nodes = [root]
        for _ in range(gap_nodes):
            nodes.append(_node(0, C, [], [[], [], [], []][:0], []))
        nodes.append(_node(0, C | CC_FILTERED, allv[allv % U(5) != U(4)], ra, [1, 0, 1, 0], first=2, offset=1))
        nodes.append(_node(0, CC_CHECKED, [], [], []))
        nodes.append(_node(0, C, [4, 7, 10], _rows_of([3, 0, 3, 1]), [0, 1, 1, 1], first=-1))
        nodes.append(_node(0, CC_CHECKED, [], [], []))
        return nodes

    fx.append(CcFix("rows, nodes and empty rows on CTA edges",
                    [cc_case(cta_level([255, 1, 0, 0], 1)), cc_case(cta_level([256, 0, 0, 3], 2)),
                     cc_case(cta_level([257, 0, 255, 0], 1)), cc_case(cta_level([2046, 0, 0, 2], 1))],
                    {"cc space: a zero-slot node first in a level's value slots",
                     "cc space: a zero-slot node between value slots",
                     "cc space: a zero-slot node last in a level's value slots",
                     "cc space: a zero-slot node first in a level's dest slots",
                     "cc space: a zero-slot node last in a level's dest slots",
                     "cc space: a zero-slot node first in a level's has_val slots",
                     "cc space: a zero-slot node between has_val slots",
                     "cc space: a zero-slot node last in a level's has_val slots",
                     "cc space: a node's first value slot on a CTA edge",
                     "cc space: a node's first value slot on a tile edge", "cc space: a row boundary on a CTA edge", "cc space: a row of 256 values",
                     "cc space: empty rows sharing an offset on a CTA edge",
                     "cc filter: a row after empty rows starts on a CTA edge"},
                    {"node_of takes the first of equal bases", "row search at p"}))

    def dest_between():
        root = _node(-1, CC_CASCADE, [1, 2, 3], [[1, 2, 3]])
        return [root, _node(0, C, [5, 6], [[5], [6], []]), _node(0, C, [], [[], [], []], [1, 0, 0]),
                _node(0, C, [2, 3], [[2], [], [3]])]

    def dest_on_edge(pad):
        root = _node(-1, CC_CASCADE, [1, 2], [[1, 2]])
        da = 1 + np.arange(pad, dtype=np.uint64)
        return [root, _node(0, C, da, [da[:-1], []]), _node(0, CC_CHECKED, [], [[], []]),
                _node(0, C, [3, 4], [[], [3, 4]])]

    fx.append(CcFix("zero-slot dest nodes and dest on edges",
                    [cc_case(dest_between()), cc_case(dest_on_edge(256)), cc_case(dest_on_edge(2048))],
                    {"cc space: a zero-slot node between dest slots", "cc space: a node's first dest slot on a CTA edge",
                     "cc space: a node's first dest slot on a tile edge",
                     "cc keep: a dest that descends across a node edge"},
                    {"dest order across node edges"}))

    deep = _chain(K["CC_MAX_DEPTH"] - 1, empty={20, 21, 40})
    rootless = _chain(5, empty={0})
    fx.append(CcFix("levels without work and a depth-63 chain", [cc_case(deep), cc_case(rootless)],
                    {"cc plan: a level without work between levels with work", "cc plan: the root level without work",
                     "cc plan: a node at depth kCcMaxDepth - 1", "cc plan: 2 to 63 levels with work"}, set()))

    fx.append(CcFix("forests of 1 023 to 65 535 nodes",
                    [cc_case(_forest(n)) for n in (1023, 1024, 1025, K["CC_MAX_NODES"] - 1)],
                    {"cc scan: node-order counts in 1 tile", "cc scan: node-order counts over 2 tiles",
                     "cc scan: node-order counts over 64 tiles", "cc plan: a forest of 2^16 - 1 nodes"},
                    {"count scan over NN"}))

    def prune(pad):
        # P (NEW, 6 dest) at level 1 with checked children at level 2: c1 with 3 rows, 4 has_val and counts_len 5;
        # c2 NEW, whose row 1 straddles the level's tile edge and is emptied by c2's own filter (its dest lacks it);
        # c3 not checked (KEEP); c4 FILTERED (OLD); an ORDERED node with descending rows; a CASCADE node without a
        # checked child.  `pad` values in a KEEP node in front put c2's row 1 on the tile edge.
        root = _node(-1, CC_CASCADE, [1], [[1]])
        d = [10, 11, 12, 13, 14, 15]
        P = _node(0, C, d, [d])
        lone = _node(0, CC_CASCADE | CC_CHECKED, [3], [[3]])
        kp = _node(1, 0, [], [list(range(100, 100 + pad))] + [[] for _ in range(5)])
        c1 = _node(1, CC_CHECKED, [7], [[7], [7], [7]], [0, 0, 0, 1], counts_len=5)
        row1 = list(range(200, 220))
        c2 = _node(1, C, [7, 300], [[7], row1, [300], [7], [7], [300, 301]][:6])
        c3 = _node(1, 0, [7], [[7]] * 6)
        c4 = _node(1, CC_FILTERED | CC_CHECKED, [7], [[7, 8]] * 6, [1] * 6)
        c5 = _node(1, CC_ORDERED | CC_CHECKED, [7, 8], [[8, 7]] * 6, [1] * 6)
        c6 = _node(2, C, [], [[]])
        return [root, P, kp, c1, c2, c3, c4, c5, lone, c6]

    def page_cut_child():
        root = _node(-1, CC_CASCADE, [1], [[1]])
        P = _node(0, C, [10, 11, 12], [[10, 11, 12]])
        c = _node(1, C, [20, 21, 22], [[20, 21, 22], [20], [21, 22]], offset=1)
        return [root, P, c]

    fx.append(CcFix("prune edges", [cc_case(prune(pad)) for pad in (2030, 1)] + [cc_case(page_cut_child())],
                    {"cc keep: a checked child with nrows == i", "cc keep: a checked child with nhv == i",
                     "cc keep: kept by counts_len == i + 1", "cc keep: pruned at i == counts_len",
                     "cc keep: a child row emptied by the child's own filter",
                     "cc keep: a CASCADE node without a checked child",
                     "cc filter: KEEP, OLD and NEW nodes in one level", "cc filter: an ORDERED row that descends", "cc filter: a value dropped by OLD",
                     "cc filter: a value dropped by NEW", "cc keep: a child row emptied by the child's page cut"},
                    {"prune reads the gathered rows"}))

    def slack_room():
        root = _node(-1, CC_CASCADE, [1, 2], [[1, 2]])
        rows = _rows_of([1500, 300])
        allv = np.unique(np.concatenate(rows))
        return cc_case([root, _node(0, C, allv, rows, first=-400), _node(0, C | CC_FILTERED, [4], [[4], [4]])],
                       slack={1: np.repeat(allv[:50], 60), 2: np.full(3000, 4)})

    def descend_rows():
        root = _node(-1, CC_CASCADE, [1, 2], [[1, 2]])
        return cc_case([root, _node(0, C, [2, 5, 9], [[5, 9], [2, 5]], first=1)])

    fx.append(CcFix("device slack and descents across row edges", [slack_room(), descend_rows()],
                    {"cc space: a device value room with slack across a tile edge",
                     "cc filter: the slack of a value room", "cc filter: a row that descends from the row before"}, set()))

    def refuse_dest(at, depth):
        nodes = _chain(depth)
        last = nodes[-1]
        d = np.arange(1, at + 60, dtype=np.uint64) * U(2)
        d[at] = d[at - 1]
        nodes[-1] = _node(last.parent, last.flags, d, [d[:3]] * len(nodes[-2].dest) if depth else [d])
        return cc_case(nodes)

    def refuse_row(at, ordered=False):
        root = _node(-1, CC_CASCADE, [1], [[1]])
        r = np.arange(1, at + 60, dtype=np.uint64) * U(3)
        r[at] = r[at - 1] - U(1)
        return cc_case([root, _node(0, C | (CC_ORDERED if ordered else 0), np.unique(r), [r])])

    def refuse_off(at, kind):
        # a second root of 40 rows whose broken offset lands on gather slot `at`, after a root of empty rows
        r = {"offset start": 0, "offset decrease": 2, "offset past room": 40}[kind]
        first = _node(-1, 0, [], [[]] * (at - r - 1))
        off = np.arange(41, dtype=np.uint64)
        if kind == "offset start":
            off = off + U(1)
        elif kind == "offset decrease":
            off[2] = 0
        else:
            off[-1] = 41
        return cc_case([first, _node(-1, CC_CASCADE, [5], [[5]] * 40)], v_off={1: off})

    cases = [refuse_dest(255, 0), refuse_dest(EN_TILE, 0), refuse_dest(255, 40), refuse_dest(EN_TILE, 1),
             refuse_row(255), refuse_row(EN_TILE), refuse_row(255, True)]
    cases += [refuse_off(at, kind) for kind in REFUSALS[2:] for at in (255, EN_TILE)]
    fx.append(CcFix("every refusal on a CTA and a tile edge", cases,
                    {f"cc refuse: {k} {w}" for k in REFUSALS for w in WHERE} |
                    {"cc refuse: at the root level", "cc refuse: at a level 32 or more deep"}, set()))
    return fx


def _lst(u):
    return ("list", _u(u))


def _d0_case(n0, slack):
    """|D0| = n0 over uids 2, 4, ...; the tree AND(LIST of every uid but those = 6 mod 8, NOT(COUNT c_i == 3)), rows
    over D0 and outside it, `slack` D0 values past |D0| that hold under the tree (device form with a length word)."""
    d0 = 2 * np.arange(1, n0 + 1, dtype=np.uint64)
    top = int(d0[-1]) if n0 else 0
    sl = np.arange(top + 2, top + 2 + 2 * slack, 2, dtype=np.uint64)
    allu = np.concatenate([d0, sl])
    la = allu[allu % U(8) != U(6)]
    cnt = (np.arange(n0) % 5).astype(np.uint32)
    rows = [d0[i::7] for i in range(7)] + [np.arange(1, 50, dtype=np.uint64)]
    return sf_case(("and", [0, ("not", 1)]), [_lst(la), ("count", "eq", 3, cnt)], d0, rows, d0_slack=sl,
                   list_slack=())


def _fx_truth():
    """Every tree of the shapes below over 3 LIST leaves; D0 = 1..8 with leaf i holding u + 1 iff bit i of u is set."""
    leaves = [_lst([u + 1 for u in range(8) if u >> i & 1]) for i in range(3)]
    atoms = [0, 1, 2, ("not", 0), ("not", 1)]
    shapes = list(atoms)
    for op in ("and", "or"):
        for k in (1, 2, 3):
            for combo in itertools.permutations(atoms[:3] + [("not", 2)], k):
                shapes.append((op, list(combo)))
    for o1, o2 in itertools.product(("and", "or"), repeat=2):
        shapes.append((o1, [(o2, [0, 1]), 2]))
        shapes.append((o1, [2, (o2, [0, ("not", 1)])]))
        shapes.append(("not", (o1, [(o2, [1, 2]), ("not", 0)])))
    d0 = np.arange(1, 9, dtype=np.uint64)
    rows = [d0, _u([2, 3, 5, 8]), _u([])]
    return [sf_case(s, leaves, d0, rows, count=c, offset=o) for s in shapes for c, o in ((0, 0), (2, 1))]


def _nested(depth, ops):
    """A chain of `depth` op nodes (cycled from ops) over leaf 0.  At even depths an AND gets leaf 3 (every D0 value)
    and an OR leaf 4 (none) as a first child, so the chain is always its last child; at odd depths it has one child."""
    t = 0
    for d in range(depth):
        op = ops[d % len(ops)]
        if op == "not":
            t = ("not", t)
        elif d % 2:
            t = (op, [t])
        else:
            t = (op, [3 if op == "and" else 4, t])
    return t


def sf_fixtures():
    fx = []
    fx.append(SfFix("|D0| on CTA and tile edges", [_d0_case(n, 2048) for n in (255, 256, 257, 2047, 2048, 2049, 4097)],
                    SF_CALLS,
                    {f"sf space: |D0| of {n}" for n in (255, 256, 257, 2047, 2048, 2049, 4097)} |
                    {"sf space: a length word below d0_cap by a tile",
                     "sf eval: slack D0 values that hold, not evaluated", "sf out: counts-only"},
                    {"|D0| read as d0_cap", "scans without tile carry"}))

    d0 = np.arange(1, 301, dtype=np.uint64)
    base = dict(tree=("or", [0, 1]), leaves=[_lst(d0[::2]), ("count", "gt", 1, (np.arange(300) % 3).astype(np.uint32))])
    rows_many = [d0[i % 300:i % 300 + 3] for i in range(400)]
    fx.append(SfFix("values and rows", [
        sf_case(d0=d0, rows=[d0[:200], d0[100:], d0[5:6]], v_slack=np.resize(d0, 2900), count=2,
                **base),
        sf_case(d0=d0, rows=rows_many, **base), sf_case(d0=d0, rows=[], count=3, **base)], SF_CALLS,
        {"sf space: v_off[nrows] below v_cap across a tile edge", "sf space: nrows above d0_cap", "sf space: no rows"},
        set()))

    def d1_case(n1, paged):
        d0 = np.arange(1, 3001, dtype=np.uint64)
        keep = d0[:n1]
        rows = [d0[:1500:3], d0[1000:3000:2], d0[2990:]]
        return sf_case(0, [_lst(keep)], d0, rows, count=2 if paged else 0, offset=1 if paged else 0)

    fx.append(SfFix("D1 of 0, 2 048 and 2 049", [d1_case(n, p) for n in (0, 2048, 2049) for p in (False, True)],
                    SF_CALLS, {"sf d1: empty", "sf d1: 2048 values", "sf d1: 2049 values", "sf d2: unpaged",
                               "sf d2: paged, a D1 value no kept row holds"},
                    {"sf_mark marks all of D1 when paged"}))

    d0 = np.arange(1, 256, dtype=np.uint64)
    cnt = (np.arange(255) % 4).astype(np.uint32)
    off = np.concatenate([[0], np.cumsum(np.arange(255) % 3)]).astype(np.uint64)
    rows = [d0[::2], d0[1::5]]
    # slots: COUNT over counts (none), LIST of room 0 (slot 0), COUNT over off (slots 1-255), LIST from slot 256
    ok_leaves = [("count", "ge", 2, cnt), _lst([]), ("len", "lt", 2, off), _lst(d0[::3]), ("count", "le", 1, cnt),
                 _lst(d0[::4]), ("count", "eq", 0, cnt)]
    tree = ("or", [("and", [0, 3]), ("and", [2, ("not", 1)]), 4, ("and", [5, 6])])

    def broken(j, at):
        lv = list(ok_leaves)
        u = _u(lv[j][1]).copy()
        u[at] = u[at - 1]
        lv[j] = ("list", u)
        return sf_case(tree, lv, d0, rows)

    over = sf_case(tree, ok_leaves, d0, rows, list_words=[0, 10**6, 64], list_slack=[3, 2, 1])
    slack_desc = sf_case(tree, ok_leaves, d0, rows, list_words=[0, 85, 64], list_slack=[3, 2, 1])
    first_cnt = sf_case(("and", [1, 0]), [("count", "gt", 0, cnt), _lst([5, 5, 6])], d0, rows)
    fx.append(SfFix("the leaf slot space", [sf_case(tree, ok_leaves, d0, rows), broken(3, 1), broken(3, 84),
                                            over, slack_desc, first_cnt], SF_CALLS,
                    {"sf space: a LIST leaf of room 0", "sf space: a zero-slot leaf first",
                     "sf space: a zero-slot leaf between others", "sf space: a zero-slot leaf last",
                     "sf space: a leaf boundary on a CTA edge", "sf refuse: a LIST descends at its first checked slot",
                     "sf refuse: a LIST descends at its last checked slot", "sf refuse: a length word over its room",
                     "sf space: a descent in a LIST's slack, accepted",
                     "sf space: check slots past d0_cap, v_cap and nrows"},
                    {"leaf search takes the first of an equal sb"}))

    d0 = np.arange(10, 16, dtype=np.uint64)
    big = [0, 2**32 - 1, 2**32 - 1 + 2**32, 2**33 - 1 + 2**32 + 1, 2**34, 2**34, 2**34 + 1]
    offb = _u(big)
    cases = [sf_case(("or", [0, ("not", 1)]), [("len", cmp, thr, offb), ("len", "ge", -1, offb)], d0,
                     [d0, d0[::2]]) for cmp in ("le", "ge", "lt", "gt", "eq")
             for thr in (2**32 - 1, 2**32, 2**32 + 1, -5)]
    fx.append(SfFix("counts of 2^32 and more", cases, SF_CALLS, {"sf space: a count of 2^32 or more"}, set()))

    d0 = np.arange(1, 41, dtype=np.uint64)
    rows = [d0[::3], d0[1::2]]
    lv = [_lst(d0[::2]), _lst(d0[1::4]), _lst(d0[::5]), _lst(d0), _lst([])]
    maxd = K["SGF_MAX_DEPTH"]
    chains = [_nested(maxd, ["and"]), _nested(maxd, ["or"]), _nested(maxd, ["not"]), _nested(maxd - 1, ["not"]),
              _nested(maxd, ["and", "not", "or"]), ("not", ("not", ("not", 0))), ("and", [0]), ("or", [1]),
              ("or", [("and", [0, 1]), 2]), ("and", [("or", [1, 0]), ("not", 2)]), ("and", [0, ("or", [1, 2])])]
    n_lim = K["SGF_MAX_NODES"]
    many = [_lst(d0[j % 40:j % 40 + 1 + j % 3]) for j in range(K["SGF_MAX_LEAVES"])]
    wide = ("or", list(range(n_lim - 1)))
    fx.append(SfFix("the walk", [sf_case(t, lv, d0, rows, count=c) for t in chains for c in (0, 1)] +
                    [sf_case(wide, many, d0, rows)], SF_CALLS[:3],
                    {"sf eval: one leaf closes 64 levels", "sf eval: one leaf closes 2 to 63 levels",
                     "sf eval: an odd chain of NOTs closed by one leaf",
                     "sf eval: an even chain of NOTs closed by one leaf", "sf eval: an AND of one child", "sf eval: an OR of one child",
                     "sf eval: an AND stopped by a miss before its last child",
                     "sf eval: an OR stopped by a hit before its last child",
                     "sf eval: an AND decided by a miss at its last child",
                     "sf eval: an OR decided by a hit at its last child", "sf eval: a program of the node limit",
                     "sf eval: a leaf table of the leaf limit, one entry never evaluated"},
                    {"eval without pc != end", "NOT decoded as OR"}))

    fx.append(SfFix("a truth table over small trees", _fx_truth(), SF_CALLS[:2],
                    {"sf truth: leaf i holds u + 1 iff bit i of u is set", "sf eval: the walk ends at a leaf root",
                     "sf eval: the close loop goes on to a next child"},
                    {"eval without pc != end", "NOT decoded as OR"}))

    d0 = np.arange(1, 600, dtype=np.uint64)
    rows = [d0[:300], d0[250:]]
    lv = [_lst(d0[::2]), ("len", "gt", 0, np.concatenate([[0], np.cumsum(np.arange(599) % 2)]).astype(np.uint64))]
    desc_d0 = d0.copy()
    desc_d0[256] = desc_d0[255]
    bad_off = lv[1][3].copy()
    bad_off[300] = 0
    bad_row = [d0[:300].copy(), d0[250:]]
    bad_row[0][255] = bad_row[0][254]
    fx.append(SfFix("device-side refusals", [
        sf_case(("and", [0, 1]), lv, desc_d0, rows),
        sf_case(("and", [0, 1]), [lv[0], ("len", "gt", 0, bad_off)], d0, rows),
        sf_case(("and", [0, 1]), lv, d0, bad_row),
        sf_case(("and", [0, 1]), lv, d0, rows, v_off=[0, 300, 300 + 349 + 5000]),
        sf_case(("and", [0, 1]), lv, d0, rows, d0_word=601, d0_slack=[700])], SF_CALLS,
        {"sf refuse: D0 descends", "sf refuse: a COUNT leaf's offsets decrease", "sf refuse: a row descends",
         "sf refuse: row offsets", "sf refuse: D0's length word over d0_cap"}, set()))
    return fx


def all_fixtures():
    return cc_fixtures() + sf_fixtures()


def outcomes(f, mut=frozenset()):
    """(per case and call: the model's outcome), the events the fixture reaches."""
    ev: set = set()
    if isinstance(f, CcFix):
        return [[cc_run(c, form, mut, ev) for form in c.forms] for c in f.cases], ev
    res = [[sf_run(c, call, mut, ev) for call in f.calls] for c in f.cases]
    if f.name == "a truth table over small trees":
        _add(ev, "sf truth: leaf i holds u + 1 iff bit i of u is set")
    return res, ev
