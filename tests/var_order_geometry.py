"""Host model of orderasc / orderdesc by a value variable (var_order_kernel.cuh, dgx_api.cu vo_run: dgx_var_order and
dgx_dev_var_order), with fixtures aimed at every tier, split, chunk, pass, page and refusal boundary.

One call is restated in exact integer arithmetic: vo_check_kernel's refusals with the thread and CTA that detects each;
vo_gather_kernel's U and W flags and the two position scans, vo_compact_kernel's U, W, `uoff` and `woff`; the order
keys (int64 with its sign bit flipped, float64's order-preserving bits with -0.0 on +0.0, complemented for desc); both
radix sorts through radix_geometry.radix_sort with `tiles` taken from v_cap (the device form's slack gives trailing
empty tiles) and the row sort's result read from buffer `pr & 1`; vo_tier_kernel's row flags and its bool-first
refusal; each row's tier (tier 1, tier 2 on one thread, tier 2 on a CTA of the `2 * SMs` grid); Go's pdqsort driven
by the device's own frame loop (vo_advance / vo_after), recording every helper that runs and the deepest frame stack
per row; for CTA rows, every partition worked chunk by chunk as vo_coop_partition does it (the left count `m`, the
pair count, each chunk's block ranks, the chunk each pair's two sides fall in); the page ranges through
cascade_geometry._page_range (the kernel calls cc_page_range); the output slots, the dest marks and the new dest.
The launch count is built from the kernels vo_run launches around the two sorts (FRONT, BACK) and the sorts' own
passes, and tests/test_var_order_geometry.py holds it to var_order_plan.py, which counts vo_run's count_launches.

What the kernels decide is named as *events*; fixtures name the events they must reach, and the model refuses a name
that is not registered in EVENTS.  The model also carries named *mutants* (MUTANTS), each a plausible slip in one
kernel; a fixture names the mutants it kills, and tests/test_var_order_geometry.py checks that the mutated model's
output differs from the restatement's (var_order_oracle.c) on it.  No mutated kernel is built.  Two slips are invisible
by design and so are not mutants: where the thread / CTA threshold lies (both run the same partition), and tier 1
against tier 2 on distinct keys (the order is unique).  The tests assert that invisibility instead.  So is tier 2 at
`n >= 12` rather than `n > 12`: a tied row of 12 runs insertionSort in pdqsort, which is stable under a strict weak
order, so it equals the stable radix order; the visible slip at that edge is the other side, tier 2 only at `n > 13`.

Edges the kernels have that no fixture reaches at test scale:
  - totals of 2^32 values, rows or dest values, which both forms refuse at the call;
  - four row passes: nrows > 2^24 needs about 270 MB of offsets and values per call;
  - VO_STACK_CTA (32 frames) and VO_STACK_THREAD (13) themselves: a frame is pushed for the larger side while the
    smaller runs, so the depth grows only through balanced partitions.  A seeded search over 1 400 long rows of eight
    kinds (SEARCH_KINDS) reached 7 frames on thread rows of 4 096 entries and 8 on CTA rows of up to 8 193; the
    fixtures hold those depths and tests/test_var_order_geometry.py checks the bound on random tied rows;
  - partitionEqual with m = 0: its pivot is no greater than the entry before the range, which bounds the range, so
    m = 0 needs that entry and the pivot equal and no other entry equal to them; the search never met it;
  - partitionEqual with 256 or 257 pairs (0 and 1 are reached): its pairs are the entries greater than the pivot
    among the first m of the range, a count that lands on 256 or 257 by chance only; 1 400 searched rows and 2 567
    more of few distinct values never met it;
  - partialInsertionSort's left shift running below its range's start (Go's `j >= 1` bound): it needs a comparator
    that is not a strict weak order to rank an entry of a later range below the pivot before it, and to reach that
    range with wasBalanced, wasPartitioned and an increasing hint.  The search never met it, so the slip of bounding
    the shift at `a` has no fixture and is not listed in MUTANTS;
  - which CTA of the grid pulls which long row, and the look-back order of the multi-tile scans: the scheduler
    chooses both.  Fixtures with more long rows than CTAs make a second pull certain but cannot choose its CTA.  The
    long rows there hold different values, each after a short row, so a CTA that sorted the wrong row would write a
    wrong answer whichever CTA pulled it (the mutant "CTA sorts row i").  A CTA's pair slots written without the
    row's offset (`P.pairs` for `P.pairs + b0`) are a race between CTAs, not a deterministic answer, and so no
    mutant: its outcome depends on the schedule.

The constants and the statements the model restates are read from the CUDA sources as text, so a rewrite fails here
loudly instead of leaving the fixtures aimed at stale edges.  tests/test_var_order_geometry.py checks the fixtures on
the CPU; tests/test_gpu_var_order_edges.py runs them through the kernels.
"""
from __future__ import annotations

import os
import re
import struct
from collections import namedtuple

import numpy as np

import cascade_geometry as cg
import radix_geometry as rg
import var_order_plan as vp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")
T_INT, T_FLOAT, T_BOOL, T_NIL = 1, 2, 3, 4
GO_TID = {T_INT: 2, T_FLOAT: 3, T_BOOL: 4, T_NIL: 0}
SIGN = 1 << 63
U64 = (1 << 64) - 1
H100_SMS = 132


def _src(fn):
    with open(os.path.join(CSRC, fn)) as f:
        return f.read()


def _one(pat, text, what):
    m = re.search(pat, text)
    if not m:
        raise ValueError(f"{what} changed: restate it in the order-by-variable model (tests/var_order_geometry.py)")
    return m


def _fn(name, text):
    """The body of the function or kernel `name` (a definition starting a line, through its closing brace)."""
    head = r"(?ms)^(?:static |__global__ |__device__ |extern \"C\" )[^\n]*\b"
    return _one(head + name + r"\(.*?\n\}\n", text, name).group(0)


K_FILE, API = "var_order_kernel.cuh", "dgx_api.cu"
# (file, function or None for the whole file, statement as a regex, what it restates)
STATEMENTS = [
    (API, "vo_run", r"vo_cta_kernel<<<\(unsigned\)\(2 \* g_num_sms\), VO_NT, 0, l->stream>>>\(P\);", "the CTA grid"),
    (API, "vo_run", r"tiles = \(vc \+ GB_TILE - 1\) / GB_TILE", "the radix tiles over v_cap"),
    (API, "vo_run", r"P\.S = rp\[pr & 1\];", "the row sort's result buffer"),
    (API, "vo_run", r"vo_check_kernel<<<gb_grid\(std::max<uint64_t>\(\{dcap, M\.n, nrows \+ 1, v_cap\}\)\), 256, 0, "
     r"l->stream>>>\(P\);\s*vo_gather_kernel<<<[^\n]*\n\s*scan\(P\.uf, [^\n]*\n\s*scan\(P\.wf, [^\n]*\n\s*"
     r"vo_compact_kernel<<<[^\n]*\n\s*CK\(cudaGetLastError\(\)\);\s*count_launches\(l, 5\);",
     "the launches before the sorts"),
    (API, "vo_run", r"vo_rowkey_kernel<<<gb_grid\(v_cap\), 256, 0, l->stream>>>\(P, ep\[0\], ek\[1\], ep\[1\]\);"
     r"(?s:.*?)P\.S = rp\[pr & 1\];\s*vo_tier_kernel<<<[^\n]*\n\s*vo_rows_kernel<<<[^\n]*\n\s*vo_cta_kernel<<<[^\n]*\n"
     r"\s*scan\(P\.plen, [^\n]*\n\s*vo_write_kernel<<<[^\n]*\n\s*scan\(P\.mark, [^\n]*\n\s*vo_dest_kernel<<<[^\n]*\n"
     r"\s*CK\(cudaGetLastError\(\)\);\s*count_launches\(l, 8\);", "the launches after the key sort"),
    (API, "vo_row_passes", r"return \(gb_bits\(nrows \? nrows - 1 : 0\) \+ GB_DIGIT_BITS - 1\) / GB_DIGIT_BITS;",
     "the row sort's key width"),
    (K_FILE, "vo_rows_kernel",
     r"if \(n > 1 && \(\(f & VO_MIXED\) \|\| \(\(f & VO_TIE\) && n > \(u64\)VO_MAX_INSERTION\)\)\) \{",
     "the tier-2 test"),
    (K_FILE, "vo_rows_kernel", r"if \(n > VO_CTA_MIN\) \{", "the thread / CTA split"),
    (K_FILE, "vo_rows_kernel", r"const u64 len = n \? n : P\.uoff\[r \+ 1\] - P\.uoff\[r\];", "the paged length"),
    (K_FILE, "vo_order_key", r"if \(tag == VO_INT\) \{\s*k = w \^ kSign;", "the int order key"),
    (K_FILE, "vo_order_key", r"if \(w == kSign\) w = 0;\s*k = \(w & kSign\) \? ~w : \(w \| kSign\);",
     "the float order key"),
    (K_FILE, "vo_order_key", r"return desc \? ~k : k;", "the desc complement"),
    (K_FILE, "vo_is_nan", r"return tag == VO_FLOAT && \(w & 0x7ff0000000000000ull\) == 0x7ff0000000000000ull && "
     r"\(w & 0x000fffffffffffffull\);", "vo_is_nan"),
    (K_FILE, "vo_tier_kernel", r"if \(\(tag != VO_INT && tag != VO_FLOAT\) \|\| tag != ft \|\| "
     r"vo_is_nan\(tag, P\.wword\[p\]\)\) f \|= VO_MIXED;", "the MIXED flag"),
    (K_FILE, "vo_tier_kernel", r"if \(t > first && P\.okey\[P\.S\[t - 1\]\] == P\.okey\[p\]\) f \|= VO_TIE;",
     "the tie test"),
    (K_FILE, "vo_tier_kernel", r"if \(t < P\.nrows && P\.woff\[t \+ 1\] > P\.woff\[t\] && "
     r"P\.wtag\[P\.woff\[t\]\] == VO_BOOL\) vo_refuse\(P\);", "the bool-first refusal"),
    (K_FILE, "vo_less", r"if \(a\.tag == VO_FLOAT\) return vo_f64\(a\.w\) < \(double\)\(long long\)b\.w;\s*"
     r"return \(double\)\(long long\)a\.w < vo_f64\(b\.w\);", "int against float"),
    (K_FILE, "vo_coop_partition", r"auto left = \[&\]\(long i\) \{ return eq \? !vo_Less\(pv, d\.at\(i\), d\.desc\) : "
     r"vo_Less\(d\.at\(i\), pv, d\.desc\); \};", "the left test"),
    (K_FILE, "vo_coop_partition", r"if \(g\) pairs\[s \+ rk\] = \(u32\)i;\s*s \+= tot;", "the left part's pairs"),
    (K_FILE, "vo_coop_partition", r"if \(g\) d\.swap\(pairs\[s - 1 - \(seen \+ rk\)\], j\);\s*seen \+= tot;",
     "the pair swap"),
    (K_FILE, "vo_coop_partition", r"\*mid = eq \? l1 \+ 1 : l1;", "the cooperative mid"),
    (K_FILE, "vo_cta_kernel", r"vo_after\(s_f, s_st, s_top, kind, mid, np == 0\);", "alreadyPartitioned"),
    (K_FILE, "vo_partial_insertion_sort", r"for \(long k = i - 1; k >= 1; k--\) \{", "the left shift's bound"),
    (K_FILE, "vo_break_patterns", r"const long idx = a \+ \(length / 4\) \* 2 - 1;", "breakPatterns' index"),
    (K_FILE, "vo_write_kernel", r"if \(P\.woff\[r \+ 1\] == wb\) x = P\.U\[P\.uoff\[r\] \+ i\];\s*"
     r"else if \(P\.rflag\[r\] & VO_TIER2\) x = P\.wuid\[wb \+ i\];\s*else x = P\.wuid\[P\.S\[wb \+ i\]\];",
     "the write's three sources"),
]


def read_constants() -> dict:
    kern, api, gbk = _src(K_FILE), _src(API), _src("groupby_kernel.cuh")
    K = {k: int(_one(r"constexpr \w+ VO_%s = (\d+);" % k, kern, f"VO_{k}").group(1))
         for k in ("MAX_INSERTION", "CTA_MIN", "NT", "STACK_THREAD", "STACK_CTA", "KEY_PASSES")}
    m = _one(r"constexpr int GB_NT = (\d+), GB_VT = (\d+), GB_TILE = GB_NT \* GB_VT;", gbk, "GB_TILE")
    K["GB_TILE"] = int(m.group(1)) * int(m.group(2))
    text = {K_FILE: kern, API: api}
    for fn, func, pat, what in STATEMENTS:
        _one(pat, _fn(func, text[fn]) if func else text[fn], what)
    if K["GB_TILE"] != rg.TILE or K["KEY_PASSES"] != vp.K["KEY_PASSES"]:
        raise ValueError("the radix or plan model disagrees: restate it in the order-by-variable model")
    return K


K = read_constants()
MAXI, CTA_MIN, NT, TILE = K["MAX_INSERTION"], K["CTA_MIN"], K["NT"], K["GB_TILE"]

MUTANTS = {
    "tier 2 only at n > 13": "a tied row of 13 taken as tier 1 (`n > VO_MAX_INSERTION + 1`)",
    "pairs from the left": "pairs[seen + rk]: the k-th misplaced entry from the left of the right part",
    "chunk offset not carried": "pairs[rk]: the left part's chunks each written from slot 0",
    "partitionEqual returns l1": "*mid = l1 for partitionEqual too",
    "alreadyPartitioned as m == 0": "vo_after(..., m == 0) instead of no pair",
    "-0.0 not folded": "the order key without `if (w == kSign) w = 0`",
    "canonical NaN only": "vo_is_nan recognising only 0x7ff8000000000000",
    "bool-first after sorting": "the bool-first refusal reading the row's first entry after the sort",
    "no desc complement for floats": "a float's order key not complemented under desc",
    "int against float exactly": "int64 against float64 compared exactly, not through float64(int64)",
    "row sort result from buffer 0": "P.S = rp[0] whatever the row sort's pass parity",
    "tier 1 read in place": "vo_write_kernel reading a tier-1 row's W in pre-sort order",
    "W row paged on U's length": "a row with W paged on |U| instead of |W|",
    "breakPatterns index off by one": "breakPatterns' idx = a + (length / 4) * 2",
    "CTA sorts row i": "vo_cta_kernel's pull i sorting row i instead of longrows[i]",
}

# ---- events -----------------------------------------------------------------------------------------------------------

WHERE = ("in a CTA's last thread", "in a CTA's first thread")
REFUSALS = ("dest order", "key order", "tag", "offset decrease", "row order", "bool first")
KINDS = ("partition", "partitionEqual")
PAGES = ("no page", "negative first inside", "negative first clamped", "offset past the row", "first only",
         "offset only", "first and offset inside", "first past the end", "negative offset")
EVENTS = {
    "tier: W empty, U empty", "tier: W empty, U non-empty", "tier: a row of n = 1",
    "tier: tied row of 12 (tier 1)", "tier: tied row of 13 (tier 2)", "tier: distinct floats, n > 12 (tier 1)",
    "tier: MIXED by one entry of a second tag", "tier: MIXED by a NaN with the sign bit",
    "tier: MIXED by a non-canonical NaN",
    "tier: MIXED by a bool after the first entry", "tier: a +-0.0 tie at n = 13",
    "split: a thread row of 4096", "split: a CTA row of 4097", "split: long and short tier-2 rows in one warp",
    "split: a CTA pulls a second row",
    "driver: heapSort on a CTA row", "driver: partialInsertionSort succeeds on a CTA row",
    "driver: partialInsertionSort fails after its fifth step on a CTA row", "driver: reverseRange on a CTA row",
    "driver: breakPatterns on a CTA row",
    "driver: stack depth 7 or more on a thread row", "driver: stack depth 8 or more on a CTA row",
    "coop: a pair with both sides past their phase's first chunk", "coop: right part's last chunk holds one entry",
    "coop: partitionEqual over an all-equal range",
    "radix: trailing empty tiles (v_cap past |W| by a tile)", "radix: keys differ only in the top byte",
    "radix: keys differ only in the bottom byte",
    "cmp: int 2^53 + 1 against float 2^53", "cmp: INT64_MAX against float 2^63",
    "key: INT64_MIN", "key: INT64_MAX", "key: +Inf", "key: -Inf", "key: the largest subnormal", "key: -0.0 and +0.0",
    "write: output slots 255", "write: output slots 256", "write: output slots 257",
    "write: dest mark at 0", "write: dest mark at nd - 1", "write: new dest empty",
    "call: length words with bits above 32, over slack",
} | {f"tier: {e} under desc" for e in ("tied row of 13 (tier 2)", "MIXED by one entry of a second tag",
                                        "a +-0.0 tie at n = 13", "distinct floats, n > 12 (tier 1)")} \
  | {f"split: {k} long rows = 2*SMs {d}" for k in ("tied",) for d in ("- 1", "", "+ 1")} \
  | {f"coop: m = {e} ({k})" for e in ("0", "n - 1", "0 mod 256", "1 mod 256", "255 mod 256") for k in KINDS
     if (e, k) != ("0", "partitionEqual")} \
  | {f"coop: {p} pairs (partition)" for p in (0, 1, 256, 257)} \
  | {f"coop: {p} pairs (partitionEqual)" for p in (0, 1)} \
  | {f"radix: |W| = {n}, every row tier 1" for n in rg.N_EDGES} \
  | {f"radix: nrows = {n}, {p} row passes" for n, p in ((1, 0), (256, 1), (257, 2), (65536, 2), (65537, 3))} \
  | {f"page: {p} on a {w} row" for p in PAGES for w in ("W", "U-only")} \
  | {f"refuse: {r} {w}" for r in REFUSALS for w in WHERE}


def _add(ev, name):
    if name not in EVENTS:
        raise KeyError(f"event {name!r} is not registered in var_order_geometry.EVENTS")
    ev.add(name)


# ---- byValue.Less -----------------------------------------------------------------------------------------------------

def f64(w):
    return struct.unpack("<d", struct.pack("<Q", int(w)))[0]


def i64(w):
    w = int(w)
    return w - (1 << 64) if w & SIGN else w


def entry(tag, w, uid):
    """One W entry as the sort sees it: (tag, word, its Python value, uid)."""
    tag, w = int(tag), int(w)
    return (tag, w, i64(w) if tag == T_INT else f64(w) if tag == T_FLOAT else w, int(uid))


def make_less(desc, mut):
    exact = "int against float exactly" in mut

    def less(a, b):  # types.less with mismatchedLess
        ta, tb = a[0], b[0]
        if ta != tb:
            if ta > T_FLOAT or tb > T_FLOAT:
                return GO_TID[ta] < GO_TID[tb]
            if exact:
                return a[2] < b[2]      # Python compares int with float exactly
            return a[2] < float(b[2]) if ta == T_FLOAT else float(a[2]) < b[2]
        if ta == T_INT or ta == T_FLOAT:
            return a[2] < b[2]
        return False

    def Less(a, b):
        an, bn = a[0] == T_NIL, b[0] == T_NIL
        if an and bn:
            return desc
        if an:
            return False
        if bn:
            return True
        if a[0] == b[0] and (a[2] == b[2] if a[0] == T_FLOAT else a[1] == b[1]):
            return False
        lt = less(a, b)
        return (not lt) if desc else lt
    return Less


def order_key(tag, w, desc, mut=frozenset()):
    k = 0
    if tag == T_INT:
        k = w ^ SIGN
    elif tag == T_FLOAT:
        if w == SIGN and "-0.0 not folded" not in mut:
            w = 0
        k = (~w & U64) if w & SIGN else (w | SIGN)
        if "no desc complement for floats" in mut:
            return k
    return (~k & U64) if desc else k


def is_nan(tag, w, mut=frozenset()):
    if "canonical NaN only" in mut:
        return tag == T_FLOAT and w == 0x7FF8000000000000
    return tag == T_FLOAT and (w & 0x7FF0000000000000) == 0x7FF0000000000000 and bool(w & 0x000FFFFFFFFFFFFF)


# ---- Go's pdqsort over the device's frame loop -----------------------------------------------------------------------

class Row:
    """One row of W (Go's data[0 .. n)) with the statistics of its sort."""

    def __init__(self, entries, desc, mut, coop):
        self.e = list(entries)
        self.L = make_less(desc, mut)
        self.mut, self.coop = mut, coop
        self.pairs = [0] * max(len(self.e), 1)    # P.pairs + b0: stale slots survive between partitions
        self.helpers, self.depth, self.parts = set(), 0, []

    def less(self, i, j):
        return self.L(self.e[i], self.e[j])

    def swap(self, i, j):
        e = self.e
        e[i], e[j] = e[j], e[i]


def _insertion_sort(d, a, b):
    for i in range(a + 1, b):
        j = i
        while j > a and d.less(j, j - 1):
            d.swap(j, j - 1)
            j -= 1


def _sift_down(d, lo, hi, first):
    root = lo
    while True:
        child = 2 * root + 1
        if child >= hi:
            return
        if child + 1 < hi and d.less(first + child, first + child + 1):
            child += 1
        if not d.less(first + root, first + child):
            return
        d.swap(first + root, first + child)
        root = child


def _heap_sort(d, a, b):
    first, lo, hi = a, 0, b - a
    for i in range((hi - 1) // 2, -1, -1):
        _sift_down(d, i, hi, first)
    for i in range(hi - 1, -1, -1):
        d.swap(first, first + i)
        _sift_down(d, lo, i, first)


def partition_seq(d, a, b):
    """Go's partition with the pivot at a: (mid, alreadyPartitioned), before the final swap."""
    i, j = a + 1, b - 1
    while i <= j and d.less(i, a):
        i += 1
    while i <= j and not d.less(j, a):
        j -= 1
    if i > j:
        return j, True
    d.swap(i, j)
    i, j = i + 1, j - 1
    while True:
        while i <= j and d.less(i, a):
            i += 1
        while i <= j and not d.less(j, a):
            j -= 1
        if i > j:
            return j, False
        d.swap(i, j)
        i, j = i + 1, j - 1


def partition_equal_seq(d, a, b):
    i, j = a + 1, b - 1
    while True:
        while i <= j and not d.less(a, i):
            i += 1
        while i <= j and d.less(a, j):
            j -= 1
        if i > j:
            return i
        d.swap(i, j)
        i, j = i + 1, j - 1


Part = namedtuple("Part", "kind a b m pairs chunks1 chunks2 cross")


def partition_coop(d, a, b, eq, mut=frozenset()):
    """vo_coop_partition: (mid, pair count, Part).  Chunks are VO_NT entries; a chunk's flags are ballots taken
    before any of its swaps, and its ranks are block ranks in thread order."""
    pv, e, L = d.e[a], d.e, d.L
    left = (lambda i: not L(pv, e[i])) if eq else (lambda i: L(e[i], pv))
    m = sum(1 for i in range(a + 1, b) if left(i))
    l1 = a + m
    s, chunks1, where1 = 0, [], {}
    for ci, c0 in enumerate(range(a + 1, l1 + 1, NT)):
        g = [i for i in range(c0, min(c0 + NT, l1 + 1)) if not left(i)]
        for rk, i in enumerate(g):
            slot = rk if "chunk offset not carried" in mut else s + rk
            d.pairs[slot] = i
            where1[slot] = ci
        chunks1.append(len(g))
        s += len(g)
    seen, chunks2, cross = 0, [], False
    for ci, c0 in enumerate(range(l1 + 1, b, NT)):
        g = [j for j in range(c0, min(c0 + NT, b)) if left(j)]
        for rk, j in enumerate(g):
            slot = seen + rk if "pairs from the left" in mut else s - 1 - (seen + rk)
            if ci > 0 and where1.get(slot, 0) > 0:
                cross = True
            d.swap(d.pairs[slot], j)
        chunks2.append(len(g))
        seen += len(g)
    mid = l1 if (not eq or "partitionEqual returns l1" in mut) else l1 + 1
    return mid, s, Part("partitionEqual" if eq else "partition", a, b, m, s, tuple(chunks1), tuple(chunks2), cross)


def _bits_len(x):
    return x.bit_length()


def _break_patterns(d, a, b):
    length = b - a
    if length >= 8:
        d.helpers.add("breakPatterns")
        rnd = length
        modulus = 1 << _bits_len(length)
        idx = a + (length // 4) * 2 - (0 if "breakPatterns index off by one" in d.mut else 1)
        for i in range(3):
            rnd ^= (rnd << 13) & U64
            rnd ^= rnd >> 7
            rnd ^= (rnd << 17) & U64
            other = rnd & (modulus - 1)
            if other >= length:
                other -= length
            d.swap(idx - 1 + i, a + other)


def _choose_pivot(d, a, b):
    l = b - a
    swaps = [0]

    def order2(x, y):
        if d.less(y, x):
            swaps[0] += 1
            return y, x
        return x, y

    def median(x, y, z):
        x, y = order2(x, y)
        y, z = order2(y, z)
        x, y = order2(x, y)
        return y

    i, j, k = a + l // 4 * 1, a + l // 4 * 2, a + l // 4 * 3
    if l >= 8:
        if l >= 50:
            i = median(i - 1, i, i + 1)
            j = median(j - 1, j, j + 1)
            k = median(k - 1, k, k + 1)
        j = median(i, j, k)
    hint = 1 if swaps[0] == 0 else 2 if swaps[0] == 12 else 0
    return j, hint


def _reverse_range(d, a, b):
    d.helpers.add("reverseRange")
    i, j = a, b - 1
    while i < j:
        d.swap(i, j)
        i, j = i + 1, j - 1


def _partial_insertion_sort(d, a, b):
    i = a + 1
    for step in range(5):
        while i < b and not d.less(i, i - 1):
            i += 1
        if i == b:
            d.helpers.add("partialInsertionSort ok")
            return True
        if b - a < 50:
            return False
        d.swap(i, i - 1)
        if i - a >= 2:
            for k in range(i - 1, 0, -1):   # Go's bound: down to 1, not to a
                if not d.less(k, k - 1):
                    break
                d.swap(k, k - 1)
        if b - i >= 2:
            for k in range(i + 1, b):
                if not d.less(k, k - 1):
                    break
                d.swap(k, k - 1)
    d.helpers.add("partialInsertionSort failed after 5 steps")
    return False


def _advance(d, f, st):
    """vo_advance: runs the loop to the next partition of [f[0], f[1]) (the pivot swapped to f[0]); "done" at the end.
    f = [a, b, limit, wasBalanced, wasPartitioned]."""
    while True:
        a, b = f[0], f[1]
        length = b - a
        ret = False
        if length <= MAXI:
            _insertion_sort(d, a, b)
            ret = True
        elif f[2] == 0:
            d.helpers.add("heapSort")
            _heap_sort(d, a, b)
            ret = True
        else:
            if not f[3]:
                _break_patterns(d, a, b)
                f[2] -= 1
            pivot, hint = _choose_pivot(d, a, b)
            if hint == 2:
                _reverse_range(d, a, b)
                pivot = (b - 1) - (pivot - a)
                hint = 1
            if f[3] and f[4] and hint == 1 and _partial_insertion_sort(d, a, b):
                ret = True
            else:
                kind = "partitionEqual" if a > 0 and not d.less(a - 1, pivot) else "partition"
                d.swap(a, pivot)
                return kind
        if ret:
            if not st:
                return "done"
            f[:] = st.pop()


def _after(f, st, kind, mid, already):
    if kind == "partitionEqual":
        f[0] = mid
        return
    a, b, length = f[0], f[1], f[1] - f[0]
    f[4] = int(already)
    left, right, thr = mid - a, b - mid, length // 8
    if left < right:
        f[3] = int(left >= thr)
        st.append([mid + 1, b, f[2], f[3], f[4]])
        f[:] = [a, mid, f[2], 1, 1]
    else:
        f[3] = int(right >= thr)
        st.append([a, mid, f[2], f[3], f[4]])
        f[:] = [mid + 1, b, f[2], 1, 1]


def pdqsort(d):
    """sort.Sort over the device's frame loop: on one thread (d.coop false) or one CTA (true)."""
    n = len(d.e)
    if n <= 1:
        return d
    st, f = [], [0, n, _bits_len(n), 1, 1]
    while True:
        kind = _advance(d, f, st)
        if kind == "done":
            return d
        a, b = f[0], f[1]
        if d.coop:
            mid, npairs, part = partition_coop(d, a, b, kind == "partitionEqual", d.mut)
            d.parts.append(part)
            already = (part.m == 0) if "alreadyPartitioned as m == 0" in d.mut else npairs == 0
        elif kind == "partition":
            mid, already = partition_seq(d, a, b)
        else:
            mid, already = partition_equal_seq(d, a, b), False
        if kind == "partition":
            d.swap(mid, a)
        _after(f, st, kind, mid, already)
        d.depth = max(d.depth, len(st))


# ---- one call ---------------------------------------------------------------------------------------------------------

Call = namedtuple("Call", "form slack words")      # form "host" / "dev"; slack garbage slots; lengths from words
HOST, DEV, DEV_SLACK = Call("host", 0, False), Call("dev", 0, False), Call("dev", 3, True)
Fix = namedtuple("Fix", "name case events kills calls mutate")
Out = namedtuple("Out", "refused rows dest launches tiers rows_info")
GARBAGE_D, GARBAGE_M = 0x33 << 36, 0x5A << 40      # what the GPU test puts above a length word's low 32 bits


def map_arrays(m):
    """(keys, words, tags or None, mtype) of a fixture's map: (keys, int64 / float64 values) or tagged."""
    if len(m) == 3:
        return (np.asarray(m[0], np.uint64), np.asarray(m[1], np.uint64), np.asarray(m[2], np.uint8), 0)
    vals = np.asarray(m[1])
    return (np.asarray(m[0], np.uint64), vals.view(np.uint64), None, T_INT if vals.dtype == np.int64 else T_FLOAT)


def csr(rows):
    off = np.zeros(len(rows) + 1, np.uint64)
    np.cumsum([len(r) for r in rows], out=off[1:])
    v = np.concatenate([np.asarray(r, np.uint64) for r in rows]) if int(off[-1]) else np.zeros(0, np.uint64)
    return v, off


def arrays(case, call, mutate=None):
    """What the kernels see, built as tests/test_gpu_var_order.dev_call builds it: dest with `slack` slots of 3 past
    it when its length is a word; the values with `slack` slots of 9; the map with `slack` entries (keys and words 7,
    tags 9) past it when its length is a word.  mutate(a) breaks the inputs before that."""
    m, desc, dest, rows, count, offset = case
    d = np.asarray(dest, np.uint64)
    v, v_off = csr(rows)
    slack = call.slack if call.form == "dev" else 0
    a = {"dest": np.concatenate([d, np.full(slack if call.words else 0, 3, np.uint64)]),
         "v": np.concatenate([v, np.full(slack, 9, np.uint64)]), "v_off": v_off.copy(), "map": m}
    if mutate:
        MUTATE[mutate](a)
    k, w, t, mtype = map_arrays(a["map"])
    n = k.size
    pad = slack if call.words else 0
    a["key"] = np.concatenate([k, np.full(pad, 7, np.uint64)])
    a["word"] = np.concatenate([w, np.full(pad, 7, np.uint64)])
    a["tag"] = None if t is None else np.concatenate([t, np.full(pad, 9, np.uint8)])
    a["mtype"] = mtype
    a["dlen"] = (d.size | GARBAGE_D) if call.words else None
    a["mlen"] = (n | GARBAGE_M) if call.words else None
    return a


def _word_len(w, room):
    if w is None:
        return room, False
    n = w & 0xFFFFFFFF
    return (0, True) if n > room else (n, False)


def _refuse(ev, refused, kind, t):
    refused.append((kind, t))
    if kind in REFUSALS and t > 0:
        if t % 256 == 255:
            _add(ev, f"refuse: {kind} {WHERE[0]}")
        elif t % 256 == 0:
            _add(ev, f"refuse: {kind} {WHERE[1]}")


def check(a, ev):
    """vo_check_kernel: [(refusal, thread)], nd, nm, m."""
    refused = []
    dest, key, tag, v, v_off = a["dest"], a["key"], a["tag"], a["v"], a["v_off"]
    nd, dover = _word_len(a["dlen"], dest.size)
    nm, mover = _word_len(a["mlen"], key.size)
    nrows, v_cap = v_off.size - 1, v.size
    m = int(v_off[nrows])
    if dover or mover or m > v_cap:
        refused.append(("room", 0))
    for t in np.nonzero(dest[:nd][:-1] >= dest[:nd][1:])[0] + 1 if nd > 1 else ():
        _refuse(ev, refused, "dest order", int(t))
    for t in np.nonzero(key[:nm][:-1] >= key[:nm][1:])[0] + 1 if nm > 1 else ():
        _refuse(ev, refused, "key order", int(t))
    if tag is not None:
        for t in np.nonzero((tag[:nm] < T_INT) | (tag[:nm] > T_NIL))[0]:
            _refuse(ev, refused, "tag", int(t))
    if v_off[0] != 0:
        refused.append(("offset start", 0))
    for t in np.nonzero(v_off[1:] < v_off[:-1])[0] + 1:
        _refuse(ev, refused, "offset decrease", int(t))
    if m <= v_cap and v_off[0] == 0 and m > 1:
        for t in np.nonzero(v[:m - 1] >= v[1:m])[0] + 1:
            r = int(np.searchsorted(v_off, t, side="right")) - 1      # vo_row_of: lower_bound(v_off, t + 1) - 1
            if int(v_off[r]) != t:
                _refuse(ev, refused, "row order", int(t))
    return refused, nd, nm, m


def _page_event(count, offset, n):
    if count == 0 and offset == 0:
        return "no page"
    if count < 0:
        return "negative first clamped" if -count > n else "negative first inside"
    if offset < 0:
        return "negative offset"
    if offset > n:
        return "offset past the row"
    if count == 0:
        return "offset only"
    if offset == 0:
        return "first only" if count < n else "first past the end"
    return "first and offset inside" if offset + count < n else "first past the end"


_RADIX = {}


def _radix(key, pay, tiles, width):
    """radix_geometry.radix_sort, remembered by its inputs: a fixture's calls and the invisibility runs sort the same
    keys again."""
    h = (hash(np.asarray(key, np.uint64).tobytes()), hash(np.asarray(pay, np.int64).tobytes()), tiles, width)
    if h not in _RADIX:
        if len(_RADIX) > 64:
            _RADIX.clear()
        _RADIX[h] = rg.radix_sort(key, pay, tiles, width, set())
    return _RADIX[h]


# vo_run's launches besides the two radix sorts, in order (matched as text in STATEMENTS)
FRONT = ("vo_check_kernel", "vo_gather_kernel", "scan of the U flags", "scan of the W flags", "vo_compact_kernel")
BACK = ("vo_rowkey_kernel", "vo_tier_kernel", "vo_rows_kernel", "vo_cta_kernel", "scan of the page lengths",
        "vo_write_kernel", "scan of the dest marks", "vo_dest_kernel")


def launch_count(rbits):
    """A call's launches: FRONT, the order-key sort (64 bits), BACK's row-key kernel, the row sort (rbits bits), the
    rest of BACK.  A refused call launches them all: each kernel returns early on the bad flag."""
    return len(FRONT) + rg.K["SORT_PER_PASS"] * (rg.npasses(64) + rg.npasses(rbits)) + len(BACK)


def run(case, call=HOST, sms=H100_SMS, mut=frozenset(), ev=None, mutate=None, cta_min=CTA_MIN, tier2_all=False):
    """One call of the model: Out, with the refusals (empty when the call runs), the rows and new dest, the launches,
    each row's tier ("U", 1, "thread", "cta") and per tier-2 row (helpers, depth, partitions)."""
    ev = set() if ev is None else ev
    m_, desc, _, _, count, offset = case
    desc = bool(desc)
    a = arrays(case, call, mutate)
    dest, v, v_off = a["dest"], a["v"], a["v_off"]
    nrows = v_off.size - 1
    rbits = (nrows - 1).bit_length() if nrows > 1 else 0      # the row sort's key: rows 0 .. nrows - 1
    launches = launch_count(rbits)
    if dest.size == 0 or nrows == 0:   # both forms return before any launch: every row empty, so is the new dest
        return Out([], [np.zeros(0, np.uint64)] * nrows, np.zeros(0, np.uint64), 0, [], {})
    refused, nd, nm, m = check(a, ev)
    if call.words:
        _add(ev, "call: length words with bits above 32, over slack")
    if refused:
        return Out(refused, None, None, launches, None, None)
    # gather and compact
    vals = v[:m]
    dset, keys = dest[:nd], a["key"][:nm]
    di = np.searchsorted(dset, vals)
    uf = (di < nd) & (dset[np.minimum(di, max(nd - 1, 0))] == vals) if nd else np.zeros(m, bool)
    mj = np.searchsorted(keys, vals)
    wf = uf & (mj < nm) & (keys[np.minimum(mj, max(nm - 1, 0))] == vals) if nm else np.zeros(m, bool)
    ux = np.concatenate([[0], np.cumsum(uf)]).astype(np.int64)
    wx = np.concatenate([[0], np.cumsum(wf)]).astype(np.int64)
    U = vals[uf]
    uoff, woff = ux[v_off.astype(np.int64)], wx[v_off.astype(np.int64)]
    j = mj[wf]
    wuid, wword = vals[wf], a["word"][j]
    wtag = a["tag"][j].astype(np.int64) if a["tag"] is not None else np.full(j.size, a["mtype"], np.int64)
    W = wuid.size
    wrow = np.repeat(np.arange(nrows, dtype=np.int64), np.diff(woff))
    okey = np.array([order_key(int(t), int(w), desc, mut) for t, w in zip(wtag, wword)], np.uint64)
    # the two radix sorts; the row sort's result is in buffer pr & 1
    tiles = -(-max(v.size, 1) // TILE)
    s1 = _radix(okey, np.arange(W, dtype=np.int64), tiles, 64)
    rk = wrow[s1.pay]
    s2 = _radix(rk, s1.pay, tiles, rbits)
    pr = s2.passes
    S = s2.pay
    if "row sort result from buffer 0" in mut and pr & 1:
        S = _radix(rk, s1.pay, tiles, 8 * (pr - 1)).pay
    launches = len(FRONT) + s1.launches + s2.launches + len(BACK)
    if W:
        if tiles > -(-W // TILE):
            _add(ev, "radix: trailing empty tiles (v_cap past |W| by a tile)")
        sk = s1.key.astype(object)
        for x, y in zip(sk[:-1], sk[1:]):
            d_ = int(x) ^ int(y)
            if d_ and d_ < 256:
                _add(ev, "radix: keys differ only in the bottom byte")
            if d_ >> 56 and not d_ & ((1 << 56) - 1):
                _add(ev, "radix: keys differ only in the top byte")
    if nrows in (1, 256, 257, 65536, 65537):
        _add(ev, f"radix: nrows = {nrows}, {pr} row passes")
    # vo_tier_kernel
    flags = np.zeros(nrows, np.int64)
    if W:
        p = S
        r = wrow[p]
        first = woff[r]
        tg, ft = wtag[p], wtag[first]
        nan = np.array([is_nan(int(t), int(w), mut) for t, w in zip(tg, wword[p])], bool)
        mixed = (tg > T_FLOAT) | (tg != ft) | nan
        t_ = np.arange(W)
        tie = np.zeros(W, bool)
        tie[1:] = okey[p[:-1]] == okey[p[1:]]
        tie &= t_ > first
        np.bitwise_or.at(flags, r[mixed], 2)
        np.bitwise_or.at(flags, r[tie], 1)
    n_w = np.diff(woff)
    if "bool-first after sorting" not in mut:
        bad = [r for r in range(nrows) if n_w[r] and wtag[woff[r]] == T_BOOL]
        if bad:
            _refuse(ev, [], "bool first", bad[0])
            return Out([("bool first", r) for r in bad], None, None, launches, None, None)
    # vo_rows_kernel and vo_cta_kernel
    tier2_at = MAXI + 1 if "tier 2 only at n > 13" in mut else MAXI
    rows_out, tiers, info, longrows, perms = [], [], {}, [], {}
    cache = {}
    for r in range(nrows):
        b0, n = int(woff[r]), int(n_w[r])
        f = int(flags[r])
        two = n > 1 and (f & 2 or (f & 1 and n > tier2_at) or (tier2_all and not f & 2))
        if n == 0:
            tiers.append("U")
            row = U[uoff[r]:uoff[r + 1]]
        elif not two:
            tiers.append(1)
            src = wuid[b0:b0 + n] if "tier 1 read in place" in mut else wuid[S[b0:b0 + n]]
            row = src
        else:
            coop = n > cta_min
            tiers.append("cta" if coop else "thread")
            if coop:
                longrows.append(r)
            perm, helpers, depth, parts, first_tag = _sorted(cache, wtag[b0:b0 + n], wword[b0:b0 + n], desc, mut,
                                                             coop)
            perms[r] = perm
            info[r] = (helpers, depth, parts)
            row = wuid[b0:b0 + n][perm]
            if "bool-first after sorting" in mut and first_tag == T_BOOL:
                return Out([("bool first", r)], None, None, launches, None, None)
        if "bool-first after sorting" in mut and tiers[-1] == 1 and n and wtag[S[b0]] == T_BOOL:
            return Out([("bool first", r)], None, None, launches, None, None)
        rows_out.append(np.asarray(row, np.uint64))
    if "CTA sorts row i" in mut:
        _cta_row_i(rows_out, longrows, tiers, perms, cache, woff, wtag, wword, wuid, S, desc, mut)
    _tier_events(ev, case, n_w, uoff, flags, tiers, wtag, wword, woff, info, longrows, sms, desc, okey, tier2_at)
    if W in rg.N_EDGES and all(t in (1, "U") for t in tiers):
        _add(ev, f"radix: |W| = {W}, every row tier 1")
    # page and write
    out_rows = []
    for r in range(nrows):
        n = int(n_w[r])
        ln = n if n else int(uoff[r + 1] - uoff[r])
        if "W row paged on U's length" in mut and n:
            ln = int(uoff[r + 1] - uoff[r])
        s, e = cg._page_range(count, offset, ln)
        e = min(e, n) if n and "W row paged on U's length" in mut else e
        if ln or n:
            _add(ev, f"page: {_page_event(count, offset, ln)} on a {'W' if n else 'U-only'} row")
        out_rows.append(rows_out[r][s:e])
    K_out = sum(x.size for x in out_rows)
    if K_out in (255, 256, 257):
        _add(ev, f"write: output slots {K_out}")
    marks = np.zeros(nd, bool)
    if K_out:
        allv = np.concatenate(out_rows)
        marks[np.searchsorted(dset, allv)] = True
    if nd and marks[0]:
        _add(ev, "write: dest mark at 0")
    if nd and marks[nd - 1]:
        _add(ev, "write: dest mark at nd - 1")
    if not marks.any():
        _add(ev, "write: new dest empty")
    return Out([], out_rows, dset[marks].copy(), launches, tiers, info)


def _sorted(cache, tags, words, desc, mut, coop):
    """Go's sort of one row's W: (the permutation of its positions, helpers, deepest stack, partitions, the first tag
    after the sort).  Rows of equal values sort to one permutation of their positions, so it is kept by content."""
    sig = (np.asarray(tags).tobytes(), np.asarray(words, np.uint64).tobytes(), desc, coop)
    if sig not in cache:
        d = Row([entry(t, w, i)[:3] + (i,) for i, (t, w) in enumerate(zip(tags, words))], desc, mut, coop)
        pdqsort(d)
        cache[sig] = (np.array([e[3] for e in d.e], np.int64), d.helpers, d.depth, d.parts,
                      d.e[0][0] if len(d.e) else None)
    return cache[sig]


def _cta_row_i(rows_out, longrows, tiers, perms, cache, woff, wtag, wword, wuid, S, desc, mut):
    """The mutant "CTA sorts row i": pull i sorts row i's W in place, whatever its tier, and the long rows past the
    first len(longrows) rows stay in their pre-sort order.  Which CTA makes which pull does not enter."""
    pulled = set(range(len(longrows)))
    for r in longrows:
        if r not in pulled:
            b0, n = int(woff[r]), int(woff[r + 1] - woff[r])
            rows_out[r] = wuid[b0:b0 + n].copy()
    for r in pulled - set(longrows):
        b0, n = int(woff[r]), int(woff[r + 1] - woff[r])
        if n <= 1:
            continue
        cur = perms.get(r, np.arange(n))          # W's positions as the row holds them now
        p2 = _sorted(cache, wtag[b0:b0 + n][cur], wword[b0:b0 + n][cur], desc, mut, True)[0]
        now = cur[p2]
        if tiers[r] == 1:                           # read through the radix payload over the re-sorted W
            rows_out[r] = wuid[b0 + now][S[b0:b0 + n] - b0]
        else:
            rows_out[r] = wuid[b0 + now]


def _tier_events(ev, case, n_w, uoff, flags, tiers, wtag, wword, woff, info, longrows, sms, desc, okey, tier2_at):
    nu = np.diff(uoff)
    sfx = " under desc" if desc else ""
    for r, t in enumerate(tiers):
        n, f = int(n_w[r]), int(flags[r])
        b0 = int(woff[r])
        tags, words = wtag[b0:b0 + n], wword[b0:b0 + n]
        if n == 0:
            _add(ev, "tier: W empty, U non-empty" if nu[r] else "tier: W empty, U empty")
            continue
        if n == 1:
            _add(ev, "tier: a row of n = 1")
        if n == 12 and f == 1 and t == 1:
            _add(ev, "tier: tied row of 12 (tier 1)")
        if n == 13 and f == 1 and t != 1:
            if _pm0_tie(tags, words):
                _add(ev, "tier: a +-0.0 tie at n = 13" + sfx)
            else:
                _add(ev, "tier: tied row of 13 (tier 2)" + sfx)
        if n > MAXI and f == 0 and t == 1 and np.all(tags == T_FLOAT):
            _add(ev, "tier: distinct floats, n > 12 (tier 1)" + sfx)
        if f & 2:
            if np.all(tags <= T_FLOAT) and np.count_nonzero(tags != tags[0]) == 1:
                _add(ev, "tier: MIXED by one entry of a second tag" + sfx)
            for x, w in zip(tags, words):
                if is_nan(int(x), int(w)) and int(w) & SIGN:
                    _add(ev, "tier: MIXED by a NaN with the sign bit")
                if is_nan(int(x), int(w)) and int(w) & ~SIGN & U64 != 0x7FF8000000000000:
                    _add(ev, "tier: MIXED by a non-canonical NaN")
            if T_BOOL in tags[1:].tolist() and tags[0] != T_BOOL:
                _add(ev, "tier: MIXED by a bool after the first entry")
        vals = {(int(x), int(w)) for x, w in zip(tags, words)}
        if t == 1 or t in ("thread", "cta"):
            for (x, w), name in ((T_INT, SIGN), "key: INT64_MIN"), ((T_INT, SIGN - 1), "key: INT64_MAX"), \
                    ((T_FLOAT, 0x7FF0000000000000), "key: +Inf"), ((T_FLOAT, 0xFFF0000000000000), "key: -Inf"), \
                    ((T_FLOAT, 0x000FFFFFFFFFFFFF), "key: the largest subnormal"):
                if (x, w) in vals:
                    _add(ev, name)
            if (T_FLOAT, 0) in vals and (T_FLOAT, SIGN) in vals and n > MAXI:
                _add(ev, "key: -0.0 and +0.0")
        if t in ("thread", "cta"):
            if (T_INT, (1 << 53) + 1) in vals and (T_FLOAT, 0x4340000000000000) in vals:
                _add(ev, "cmp: int 2^53 + 1 against float 2^53")
            if (T_INT, SIGN - 1) in vals and (T_FLOAT, 0x43E0000000000000) in vals:
                _add(ev, "cmp: INT64_MAX against float 2^63")
        if t == "thread" and n == CTA_MIN:
            _add(ev, "split: a thread row of 4096")
        if t == "cta" and n == CTA_MIN + 1:
            _add(ev, "split: a CTA row of 4097")
        if r in info:
            helpers, depth, parts = info[r]
            if t == "thread" and depth >= 7:
                _add(ev, "driver: stack depth 7 or more on a thread row")
            if t == "cta":
                if depth >= 8:
                    _add(ev, "driver: stack depth 8 or more on a CTA row")
                for h, name in (("heapSort", "heapSort"), ("partialInsertionSort ok", "partialInsertionSort succeeds"),
                                ("partialInsertionSort failed after 5 steps",
                                 "partialInsertionSort fails after its fifth step"),
                                ("reverseRange", "reverseRange"), ("breakPatterns", "breakPatterns")):
                    if h in helpers:
                        _add(ev, f"driver: {name} on a CTA row")
                for p in parts:
                    _part_events(ev, p)
    for w0 in range(0, len(tiers), 32):
        ts = tiers[w0:w0 + 32]
        if "cta" in ts and "thread" in ts:
            _add(ev, "split: long and short tier-2 rows in one warp")
    G = 2 * sms
    if len(longrows) > G:
        _add(ev, "split: a CTA pulls a second row")
    for d, name in ((-1, "- 1"), (0, ""), (1, "+ 1")):
        if longrows and len(longrows) == G + d:
            _add(ev, f"split: tied long rows = 2*SMs {name}")


def _pm0_tie(tags, words):
    s = {(int(x), int(w)) for x, w in zip(tags, words)}
    return (T_FLOAT, 0) in s and (T_FLOAT, SIGN) in s


def _part_events(ev, p):
    n = p.b - p.a
    k = p.kind
    if p.m == 0 and k == "partition":
        _add(ev, "coop: m = 0 (partition)")
    if p.m == n - 1:
        _add(ev, f"coop: m = n - 1 ({k})")
        if k == "partitionEqual":
            _add(ev, "coop: partitionEqual over an all-equal range")
    if p.m >= 256:
        for r in (0, 1, 255):
            if p.m % 256 == r:
                _add(ev, f"coop: m = {r} mod 256 ({k})")
    if p.pairs in ((0, 1, 256, 257) if k == "partition" else (0, 1)):
        _add(ev, f"coop: {p.pairs} pairs ({k})")
    if p.cross:
        _add(ev, "coop: a pair with both sides past their phase's first chunk")
    if (p.b - (p.a + p.m + 1)) % NT == 1:
        _add(ev, "coop: right part's last chunk holds one entry")


# ---- mutations of the inputs for refusal fixtures ---------------------------------------------------------------------

def _swap_at(name, t):
    def f(a):
        x = a[name]
        x[t - 1], x[t] = x[t], x[t - 1]
    return f


def _map_swap(t):
    def f(a):
        k, w = a["map"][:2]
        k = np.asarray(k, np.uint64).copy()
        k[t - 1], k[t] = k[t], k[t - 1]
        a["map"] = (k, w) + tuple(a["map"][2:])
    return f


def _map_tag(t, tag):
    def f(a):
        k, w = a["map"][:2]
        w = np.asarray(w).view(np.uint64)
        tags = np.full(np.asarray(k).size, T_INT, np.uint8)
        tags[t] = tag
        a["map"] = (k, w, tags)
    return f


def _off_dec(t):
    def f(a):
        a["v_off"][t - 1] = a["v_off"][t] + 1
    return f


MUTATE = {}
for _t in (255, 256):
    MUTATE[f"dest order at {_t}"] = _swap_at("dest", _t)
    MUTATE[f"key order at {_t}"] = _map_swap(_t)
    MUTATE[f"tag at {_t}"] = _map_tag(_t, 5)
    MUTATE[f"offset decrease at {_t}"] = _off_dec(_t)
    MUTATE[f"row order at {_t}"] = _swap_at("v", _t)
    MUTATE[f"bool first at {_t}"] = _map_tag(2 * _t, T_BOOL)   # row _t of two-entry rows starts at key 2 * _t


# ---- fixtures ---------------------------------------------------------------------------------------------------------

def _u(x):
    return np.asarray(x, np.uint64)


def imap(keys, vals):
    return _u(keys), np.asarray(vals, np.int64)


def fmap(keys, vals):
    return _u(keys), np.asarray(vals, np.float64)


def tmap(keys, tags, words):
    return _u(keys), _u(words), np.asarray(tags, np.uint8)


def fw(x):
    return int(np.array([x], np.float64).view(np.uint64)[0])


def iw(x):
    return int(np.array([x], np.int64).view(np.uint64)[0])


DEFAULT = (HOST, DEV, DEV_SLACK)


def _fx(name, case, events, kills=(), calls=DEFAULT, mutate=None):
    return Fix(name, case, frozenset(events), frozenset(kills), calls, mutate)


GRID_VARIANTS = 5


def grid_rows(seed, nlong, n, desc=False):
    """nlong long tied rows of n entries, each after a short row, over one int map.  The long rows take their values
    (0..99) from GRID_VARIANTS seeded variants in rotation, so a CTA that sorts the wrong row writes a wrong answer.
    The short rows rotate through an empty row, a row without W (no map entry), a tier-1 row of 3 to 7 distinct values
    and a tied tier-2 row of 20 on a thread, so a long row's pull index is never its row index."""
    rng = np.random.default_rng(seed)
    variants = [rng.integers(0, 100, n) for _ in range(GRID_VARIANTS)]
    L = nlong * n
    t1, tied, uo = (np.arange(L + 1 + 20 * i, L + 21 + 20 * i, dtype=np.uint64) for i in range(3))
    keys = np.concatenate([np.arange(1, L + 1, dtype=np.uint64), t1, tied])
    vals = np.concatenate([np.concatenate([variants[j % GRID_VARIANTS] for j in range(nlong)]),
                           rng.permutation(20) * 3 - 7, rng.integers(0, 3, 20)])
    rows = []
    for j in range(nlong):
        rows.append([np.zeros(0, np.uint64), uo[:5 + j % 7], t1[:3 + j % 5], tied][j % 4])
        rows.append(np.arange(j * n + 1, (j + 1) * n + 1, dtype=np.uint64))
    return (imap(keys, vals), desc, np.arange(1, L + 61, dtype=np.uint64), rows, 0, 0)


SEARCH_KINDS = ("ties", "nan", "nil", "runs", "few", "mixed", "wide", "nilruns")


def search_row(seed, n, kind, desc):
    """One seeded long row for the cooperative-partition and driver fixtures: (map, rows) over keys 1..n."""
    rng = np.random.default_rng(seed)
    keys = np.arange(1, n + 1, dtype=np.uint64)
    if kind == "ties":
        m = imap(keys, rng.integers(0, int(rng.integers(2, 200)), n))
    elif kind == "few":
        m = imap(keys, rng.integers(0, 3, n))
    elif kind == "nan":
        w = np.where(rng.random(n) < rng.uniform(0.05, 0.5), np.nan, rng.integers(0, 50, n).astype(np.float64))
        m = fmap(keys, w)
    elif kind == "nil":
        tags = np.where(rng.random(n) < rng.uniform(0.2, 1.0), T_NIL, T_INT).astype(np.uint8)
        words = np.where(tags == T_INT, rng.integers(0, 30, n), 0).astype(np.uint64)
        tags[0] = T_INT
        m = tmap(keys, tags, words)
    elif kind == "runs":   # sorted runs with a few displaced entries: partialInsertionSort and reverseRange
        x = np.sort(rng.integers(0, int(rng.integers(50, 5000)), n))
        if rng.random() < 0.5:
            x = x[::-1].copy()
        for _ in range(int(rng.integers(1, 8))):
            i, j = rng.integers(0, n, 2)
            x[i], x[j] = x[j], x[i]
        m = imap(keys, x)
    elif kind == "wide":   # a few ties among nearly distinct values: the deepest frame stacks
        m = imap(keys, rng.integers(0, n - int(rng.integers(1, 64)), n))
    elif kind == "nilruns":   # ascending ints with runs of nils: Less(nil, nil) under desc reaches below a range
        tags = np.where((np.arange(n) // int(rng.integers(3, 40))) % int(rng.integers(2, 6)) == 0, T_NIL, T_INT)
        tags = tags.astype(np.uint8)
        tags[0] = T_INT
        words = np.where(tags == T_INT, np.sort(rng.integers(0, 10 * n, n)), 0).astype(np.uint64)
        m = tmap(keys, tags, words)
    else:   # ints and floats mixed, bools after the first
        tags = rng.choice([T_INT, T_FLOAT, T_BOOL], size=n, p=[0.45, 0.45, 0.1]).astype(np.uint8)
        tags[0] = T_INT
        ints = rng.integers(0, 20, n)
        words = np.where(tags == T_INT, ints.astype(np.uint64),
                         np.where(tags == T_FLOAT, (ints + 0.5).astype(np.float64).view(np.uint64),
                                  (ints & 1).astype(np.uint64)))
        m = tmap(keys, tags, words)
    return (m, desc, keys, [keys], 0, 0)


# (seed, n, kind, desc, events, kills): long rows found by a seeded search over search_row, frozen here
SEARCHED = [
    (57, 4352, 'runs', True,
     {'coop: 0 pairs (partitionEqual)', 'coop: 1 pairs (partitionEqual)'},
     {'pairs from the left', 'chunk offset not carried', 'partitionEqual returns l1', 'alreadyPartitioned as m == 0',
      'breakPatterns index off by one'}),
    (743, 4097, 'nilruns', False,
     {'coop: 1 pairs (partition)', 'coop: m = 255 mod 256 (partitionEqual)',
      "coop: right part's last chunk holds one entry", 'driver: reverseRange on a CTA row'},
     {'pairs from the left', 'chunk offset not carried', 'alreadyPartitioned as m == 0',
      'breakPatterns index off by one'}),
    (42, 4352, 'ties', True,
     {'coop: m = 0 mod 256 (partition)', 'coop: m = 1 mod 256 (partitionEqual)'},
     {'pairs from the left', 'chunk offset not carried', 'partitionEqual returns l1',
      'breakPatterns index off by one'}),
    (529, 4097, 'nan', False,
     {'coop: m = 0 mod 256 (partitionEqual)'},
     {'pairs from the left', 'chunk offset not carried', 'partitionEqual returns l1',
      'breakPatterns index off by one'}),
    (494, 4096, 'wide', True,
     {'driver: stack depth 7 or more on a thread row'},
     {'breakPatterns index off by one'}),
    (447, 8193, 'nilruns', True,
     {'coop: 1 pairs (partition)', 'coop: m = 0 mod 256 (partition)', 'coop: m = 255 mod 256 (partition)',
      'coop: m = n - 1 (partition)', "coop: right part's last chunk holds one entry",
      'driver: heapSort on a CTA row', 'driver: reverseRange on a CTA row',
      'driver: stack depth 8 or more on a CTA row'},
     {'pairs from the left', 'chunk offset not carried', 'breakPatterns index off by one'}),
    (223, 4097, 'nan', True,
     {'coop: 256 pairs (partition)', 'coop: m = n - 1 (partition)', 'driver: heapSort on a CTA row',
      'driver: reverseRange on a CTA row'},
     {'pairs from the left', 'chunk offset not carried', 'partitionEqual returns l1',
      'breakPatterns index off by one'}),
    (368, 4097, 'nil', True,
     {'coop: 257 pairs (partition)', 'coop: m = 0 mod 256 (partition)', 'coop: m = n - 1 (partition)',
      'driver: heapSort on a CTA row', 'driver: reverseRange on a CTA row'},
     {'pairs from the left', 'chunk offset not carried', 'partitionEqual returns l1',
      'breakPatterns index off by one'}),
]


def fixtures(sms=H100_SMS):
    F = []
    rng = np.random.default_rng(16)
    # tiers
    k = np.arange(1, 41, dtype=np.uint64)
    tie12 = np.array([3, 1, 3, 2, 1, 3, 2, 2, 1, 3, 1, 2], np.int64)
    tie13 = np.array([3, 1, 3, 2, 1, 3, 2, 2, 1, 3, 1, 2, 1], np.int64)
    for desc in (False, True):
        d = " desc" if desc else ""
        F.append(_fx(f"tiers: tied rows of 12 and 13{d}",
                     (imap(k[:25], np.concatenate([tie12, tie13])), desc, k[:25], [k[:12], k[12:25]], 0, 0),
                     {"tier: tied row of 12 (tier 1)",
                      "tier: tied row of 13 (tier 2)" + (" under desc" if desc else "")},
                     {"tier 2 only at n > 13"}))
        pm = np.array([0.0, -0.0, 1.5, -0.0, 0.0, 0.0, -1.0, -0.0, 2.0, 0.0, -0.0, 1.5, 0.0])
        F.append(_fx(f"tiers: a +-0.0 tie at n = 13{d}", (fmap(k[:13], pm), desc, k[:13], [k[:13], k[:2]], 0, 0),
                     {"key: -0.0 and +0.0", "tier: a +-0.0 tie at n = 13" + (" under desc" if desc else "")},
                     () if desc else {"-0.0 not folded"}))
        dk = rng.permutation(30).astype(np.float64) * 0.75 - 7.0
        F.append(_fx(f"tiers: distinct floats, n = 30{d}", (fmap(k[:30], dk), desc, k[:30], [k[:30], k[5:9]], 0, 0),
                     {"tier: distinct floats, n > 12 (tier 1)" + (" under desc" if desc else "")},
                     {"no desc complement for floats"} if desc else {"tier 1 read in place"}))
        ints = np.array([5, 2, 9, 2, 7, 1, 8, 3], np.int64)
        tags = [T_INT] * 8
        words = [iw(x) for x in ints]
        tags[5], words[5] = T_FLOAT, fw(2.0)
        F.append(_fx(f"tiers: MIXED by a second tag{d}", (tmap(k[:8], tags, words), desc, k[:8], [k[:8]], 0, 0),
                     {"tier: MIXED by one entry of a second tag" + (" under desc" if desc else "")}))
    nan_neg, nan_pay = 0xFFF8000000000000, 0x7FF0000000000001
    vals = [3.0, 0.0, 1.0, 2.0, 5.0, 4.0]
    words = [fw(x) for x in vals]
    words[1] = nan_neg
    F.append(_fx("tiers: a NaN with the sign bit", (tmap(k[:6], [T_FLOAT] * 6, words), False, k[:6], [k[:6]], 0, 0),
                 {"tier: MIXED by a NaN with the sign bit"}, {"canonical NaN only"}))
    words = [fw(x) for x in vals]
    words[2] = nan_pay
    F.append(_fx("tiers: a non-canonical NaN", (tmap(k[:6], [T_FLOAT] * 6, words), True, k[:6], [k[:6]], 0, 0),
                 {"tier: MIXED by a non-canonical NaN"}, {"canonical NaN only"}))
    F.append(_fx("tiers: a bool after the first entry, desc",
                 (tmap(k[:5], [T_INT, T_BOOL, T_INT, T_INT, T_FLOAT], [iw(4), 1, iw(2), iw(9), fw(3.5)]), True, k[:5],
                  [k[:5]], 0, 0), {"tier: MIXED by a bool after the first entry"}, {"bool-first after sorting"}))
    # comparisons and order-key extremes
    big = 1 << 53
    tags = [T_INT, T_FLOAT, T_INT, T_FLOAT, T_INT, T_INT, T_FLOAT]
    words = [iw(big + 1), fw(float(big)), iw(big - 1), fw(float(big) + 2), iw((1 << 63) - 1), iw(5), fw(2.0 ** 63)]
    F.append(_fx("cmp: int against float at 2^53 and 2^63",
                 (tmap(k[:7], tags, words), False, k[:7], [k[:7], k[:7]], 0, 0),
                 {"cmp: int 2^53 + 1 against float 2^53", "cmp: INT64_MAX against float 2^63"},
                 {"int against float exactly"}))
    ext_i = np.array([-(1 << 63), (1 << 63) - 1, 0, -1, 1, 255, 256, -(1 << 63) + 1, 1 << 56, 0x7F << 56], np.int64)
    F.append(_fx("key: int extremes and one-byte differences",
                 (imap(k[:10], ext_i), False, k[:10], [k[:10]], 0, 0),
                 {"key: INT64_MIN", "key: INT64_MAX", "radix: keys differ only in the bottom byte",
                  "radix: keys differ only in the top byte"}))
    ext_f = [np.inf, -np.inf, 5e-324 * (2 ** 52 - 1), -0.0, 0.0, 1.0, -1.0, 5e-324, 1e308, -1e-308, 0.5, 2.0, 3.0,
             -0.0]
    F.append(_fx("key: float extremes in a tied tier-2 row",
                 (fmap(k[:14], ext_f), True, k[:14], [k[:14], k[:6]], 0, 0),
                 {"key: +Inf", "key: -Inf", "key: the largest subnormal", "key: -0.0 and +0.0"},
                 {"-0.0 not folded"}))
    # radix: |W| around tile edges, one row of distinct ints; v_cap past |W|
    for n in rg.N_EDGES:
        keys = np.arange(1, n + 1, dtype=np.uint64)
        vals = rng.permutation(n).astype(np.int64) - n // 2
        calls = DEFAULT + ((Call("dev", TILE + 5, True),) if n == rg.N_EDGES[0] else ())
        ev = {f"radix: |W| = {n}, every row tier 1"} | ({"radix: trailing empty tiles (v_cap past |W| by a tile)"}
                                     if n == rg.N_EDGES[0] else set())
        F.append(_fx(f"radix: |W| = {n}", (imap(keys, vals), n % 2 == 1, keys, [keys[:n // 3], keys[n // 3:]], 0, 0),
                     ev, {"tier 1 read in place", "row sort result from buffer 0"}, calls=calls))
    # row passes
    for nrows, desc in ((256, True), (257, False), (65536, True), (65537, False)):
        F.append(_fx(f"radix: nrows = {nrows}", _many_rows(rng, nrows, desc),
                     {f"radix: nrows = {nrows}, {vp.row_passes(nrows)} row passes"},
                     {"row sort result from buffer 0"} if vp.row_passes(nrows) & 1 else (),
                     calls=(HOST, DEV_SLACK)))
    # the split
    G = 2 * sms
    for d, name in ((-1, "- 1"), (0, ""), (1, "+ 1")):
        ev = {f"split: tied long rows = 2*SMs {name}", "split: long and short tier-2 rows in one warp",
              "tier: W empty, U empty", "tier: W empty, U non-empty"} \
            | ({"split: a CTA pulls a second row"} if d > 0 else set())
        F.append(_fx(f"split: 2*SMs {name} long rows", grid_rows(7 + d, G + d, CTA_MIN + 4, desc=d == 0), ev,
                     {"CTA sorts row i"}, calls=(HOST, DEV_SLACK)))
    # page and write
    F.extend(_page_fixtures(rng))
    # refusals
    base_k = np.arange(1, 601, dtype=np.uint64)
    base = (imap(base_k, base_k.astype(np.int64) % 7), False, base_k, [base_k[:300], base_k[250:]], 0, 0)
    for kind in REFUSALS:
        for t, w in ((255, WHERE[0]), (256, WHERE[1])):
            case = base
            if kind in ("offset decrease", "bool first"):   # t is a row: 257 and more rows
                rows = [base_k[i:i + 2] for i in range(0, 600, 2)]
                case = (base[0], False, base_k, rows, 0, 0)
            F.append(_fx(f"refuse: {kind} at {t}", case, {f"refuse: {kind} {w}"}, calls=(HOST, DEV, DEV_SLACK),
                         mutate=f"{kind} at {t}"))
    for seed, n, kind, desc, events, kills in SEARCHED:
        events = events | ({"split: a thread row of 4096"} if n == CTA_MIN else set()) \
            | ({"split: a CTA row of 4097"} if n == CTA_MIN + 1 else set())
        F.append(_fx(f"coop: {kind} row {n} seed {seed}{' desc' if desc else ''}", search_row(seed, n, kind, desc),
                     events, kills, calls=(HOST, DEV_SLACK)))
    return F


def _many_rows(rng, nrows, desc):
    """nrows rows over one int map: most of 0 to 3 entries with distinct values (tier 1), every 97th a tied row of
    20 (tier 2), the first and last rows non-empty."""
    U = np.arange(1, 4 * nrows + 41, dtype=np.uint64)
    vals = rng.permutation(U.size).astype(np.int64)
    tied = rng.integers(0, 3, U.size)
    rows = []
    for r in range(nrows):
        if r % 97 == 50 or (nrows == 1):
            rows.append(U[rng.choice(U.size - 20, 1)[0]:][:20])
        else:
            c = int(rng.integers(1 if r in (0, nrows - 1) else 0, 4))
            rows.append(np.sort(rng.choice(U, size=c, replace=False)))
    vals = np.where(np.isin(np.arange(U.size), np.arange(0, U.size, 3)), tied, vals)
    return (imap(U, vals), desc, U, rows, 0, 0)


def _page_fixtures(rng):
    F = []
    keys = np.arange(1, 301, dtype=np.uint64)
    mk = keys[::2]                          # half the values have a map entry
    m = imap(mk, (mk.astype(np.int64) * 7919) % 101)
    # a W row of 20 (40 values), a row of 20 without W (even keys), a W row of 100 (200 values)
    rows = [keys[:40], keys[40:80:2] + 1, keys[100:300]]
    # "no page" is reached by every unpaged fixture; (30, 15) is past the end of 20 and inside 100
    pages = {"negative first inside": (-5, 0), "negative first clamped": (-500, 0), "offset past the row": (0, 250),
             "first only": (7, 0), "offset only": (0, 3), "first and offset inside": (4, 6),
             "first past the end": (30, 15), "negative offset": (5, -2)}
    for p, (c, o) in pages.items():
        want = {f"page: {p} on a W row", f"page: {p} on a U-only row"}
        F.append(_fx(f"page: {p}", (m, False, keys, rows, c, o), want,
                     {"W row paged on U's length"} if p == "negative first inside" else ()))
    # output slot counts 255..257 and the dest marks; dest 0 and nd - 1 marked; an empty new dest
    for K_ in (255, 256, 257):
        ks = np.arange(1, 400, dtype=np.uint64)
        row = np.concatenate([ks[:K_ - 1], ks[-1:]])     # dest's first and last value among the output
        F.append(_fx(f"write: {K_} output slots", (imap(ks, rng.permutation(ks.size)), K_ == 256, ks, [row, []], 0, 0),
                     {f"write: output slots {K_}", "write: dest mark at 0", "write: dest mark at nd - 1"}))
    return F


def outcomes(f: Fix, sms=H100_SMS, mut=frozenset(), calls=None):
    """(outs per call, events) of a fixture."""
    ev = set()
    outs = [run(f.case, c, sms, mut, ev, f.mutate) for c in (f.calls if calls is None else calls)]
    return outs, ev
