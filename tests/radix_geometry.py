"""Host model of libdgx's stable LSD radix sort (groupby_kernel.cuh gb_hist_kernel / gb_scatter_kernel, dgx_api.cu
gb_sort) and of the two ops built on it: @groupby (dgx_groupby_uid, dgx_dev_groupby_uid) and value variables
(valvar_kernel.cuh: dgx_var_propagate, dgx_dev_var_propagate, dgx_var_level_agg, dgx_dev_var_level_agg), with fixtures
aimed at every tile, round, warp, digit, pass, range and segment boundary.

One radix pass over n items in `tiles` tiles of GB_TILE = GB_NT * GB_VT items: item r * GB_NT + x of a tile belongs to
thread x of round r, so a tile's order is (round, warp, lane).  gb_hist_kernel writes tile t's count of digit d at
hist[d * tiles + t]; scan_u64_kernel scans the GB_RADIX * tiles entries digit-major in ceil(GB_RADIX * tiles / EN_TILE)
CTAs, so hoff[d * tiles + t] is where tile t's first item of digit d goes.  gb_scatter_kernel adds, per round, the
counts of the digit in the tile's earlier rounds (s_base), in the round's earlier warps (s_warp) and in the warp's
lower lanes (__match_any_sync, lanemask_lt).  `tiles` is ceil(max(e_cap, 1) / GB_TILE) for @groupby (the host form sets
e_cap = E) and vv_rtiles(max(v_cap, 1)) for a value-variable level, so trailing empty tiles exist whenever the capacity
exceeds the item count.  The model restates all of it in exact integer arithmetic and returns, for every sort, every
pass's digits, tiles, rounds, warps and match groups, each digit's tile span, the hist-scan CTA count and the launches,
together with what the ops compute from the sorted items: the groups, member lists and group order of @groupby, and
for value variables Go's ranges (width nrows / 4, the last range taking the rest), the segment and rank heads packed
in one u64, vv_fold_kernel's ordered float fold (eight gathered ahead, the same order), the warp-segmented int sum with
one atomicAdd per run, vv_combine_kernel's ascending merge of a rank's ranges, and la_fold_kernel's ballot / shuffle
fold of every row in rounds of 32 lanes.

What the kernels decide is named as *events*; fixtures name the events they must reach, and the model refuses a name
that is not registered in EVENTS.  The model also carries named *mutants* (MUTANTS), each a plausible slip in one of
those kernels; a fixture names the mutants it kills, and tests/test_radix_geometry.py checks that the mutated model's
output differs from the oracle's on it, which is what shows the GPU test would catch that class of bug.  No mutated
kernel is built.

Edges the kernels have that no fixture reaches at test scale:
  - @groupby P1 = 7 or 8: b_p + b_d > 48 (b_p, b_d <= 32) needs at least npar > 2^23 with ndest > 2^24 (or the
    reverse), about 200 MB of parent offsets and dest values per call;
  - @groupby P2 = 7 or 8: b_p + b_s > 48, the same through npar and nrows (about 200 MB of parent and row offsets);
  - a fifth value-variable pass: b_d + 2 > 32 needs ndest > 2^30, 8 GB of dest values;
  - counts of 2^32 and more, which the ops refuse on the host (kGbMax, kVvMax);
  - which CTA of the hist scan publishes its prefix first: the look-back's order is the scheduler's, the fixtures of 9
    and more tiles make a multi-CTA scan possible but cannot choose its order.

The constants and the statements the model restates are read from the CUDA sources as text, so a rewrite fails here
loudly instead of leaving the fixtures aimed at stale edges.  tests/test_radix_geometry.py checks the fixtures on the
CPU; tests/test_gpu_radix_edges.py runs them through the kernels.
"""
from __future__ import annotations

import os
import re
from collections import namedtuple

import numpy as np

import groupby_plan as gp
import valvar_plan as vp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")
OK, ERR_ARG, ERR_CAP = 0, -3, -4
U64 = (1 << 64) - 1
FMAX = float(np.finfo(np.float64).max)
TINY = 2.0 ** -53          # 1.0 + TINY ties back to 1.0; TINY + TINY is exact: sums of these reveal their order


def _src(fn):
    with open(os.path.join(CSRC, fn)) as f:
        return f.read()


def _one(pat, text, what):
    m = re.search(pat, text)
    if not m:
        raise ValueError(f"{what} changed: restate it in the radix model (tests/radix_geometry.py)")
    return m


def _fn(name, text):
    """The body of the function or kernel `name` (a definition starting a line, through its closing brace)."""
    head = r"(?ms)^(?:static |__global__ |__device__ |extern \"C\" )[^\n]*\b"
    return _one(head + name + r"\(.*?\n\}\n", text, name).group(0)


# (file, function or None for the whole file, statement as a regex, what it restates)
STATEMENTS = [
    ("groupby_kernel.cuh", "gb_hist_kernel", r"const u64 t0 = \(u64\)blockIdx\.x \* GB_TILE;", "a tile's first item"),
    ("groupby_kernel.cuh", "gb_hist_kernel", r"const u64 e = t0 \+ \(u64\)r \* GB_NT \+ tid;", "the tile mapping"),
    ("groupby_kernel.cuh", "gb_hist_kernel", r"hist\[\(u64\)tid \* tiles \+ blockIdx\.x\] = cnt\[tid\];",
     "the digit-major hist layout"),
    ("groupby_kernel.cuh", "gb_scatter_kernel", r"s_base\[tid\] = hoff\[\(u64\)tid \* tiles \+ blockIdx\.x\];",
     "the scatter's bases"),
    ("groupby_kernel.cuh", "gb_scatter_kernel", r"for \(int r = 0; r < GB_VT; \+\+r\) \{", "the rounds in order"),
    ("groupby_kernel.cuh", "gb_scatter_kernel", r"const u64 e = t0 \+ \(u64\)r \* GB_NT \+ tid;",
     "the scatter's tile mapping"),
    ("groupby_kernel.cuh", "gb_scatter_kernel", r"const u32 same = __match_any_sync\(0xffffffffu, d\);",
     "the warp's digit groups"),
    ("groupby_kernel.cuh", "gb_scatter_kernel", r"const u32 rank = __popc\(same & lanemask_lt\(\)\);",
     "the rank inside a warp"),
    ("groupby_kernel.cuh", "gb_scatter_kernel",
     r"for \(int w = 0; w < GB_WARPS; \+\+w\) \{\s*const u32 c = s_warp\[w\]\[tid\];\s*s_warp\[w\]\[tid\] = run;"
     r"\s*run \+= c;", "the warps' exclusive offsets"),
    ("groupby_kernel.cuh", "gb_scatter_kernel", r"const u64 pos = s_base\[d\] \+ s_warp\[wid\]\[d\] \+ rank;",
     "the scatter position"),
    ("groupby_kernel.cuh", "gb_scatter_kernel", r"s_base\[tid\] \+= run;", "the round's hand-off"),
    ("groupby_kernel.cuh", "gb_expand_kernel", r"P\.ek\[k\] = \(\(u64\)P\.ppar\[j\] << P\.b_d\) \| r;",
     "the edge key"),
    ("groupby_kernel.cuh", "gb_gkeys_kernel", r"gk\[g\] = \(\(P\.ek\[s\] >> P\.b_d\) << P\.b_s\) \| "
     r"\(P\.gstart\[g \+ 1\] - s\);", "the group order key"),
    ("dgx_api.cu", "gb_sort", r"hn = \(uint64_t\)GB_RADIX \* tiles, ht = \(hn \+ EN_TILE - 1\) / EN_TILE;",
     "the hist scan's CTAs"),
    ("dgx_api.cu", "gb_sort", r"for \(uint32_t q = 0; q < passes; \+\+q\) \{\s*const int a = q & 1;"
     r"\s*const u32 shift = q \* GB_DIGIT_BITS;", "the passes"),
    ("dgx_api.cu", "gb_back", r"const uint64_t ec = std::max<uint64_t>\(P\.e_cap, 1\);", "groupby's room"),
    ("dgx_api.cu", "gb_back", r"P\.tiles = \(ec \+ GB_TILE - 1\) / GB_TILE;", "groupby's tiles"),
    ("dgx_api.cu", "dgx_groupby_uid", r"P\.e_cap = P\.grp_cap = P\.mem_cap = E;", "the host form's e_cap"),
    ("dgx_api.cu", "vv_rtiles", r"return std::max<uint64_t>\(1, \(n \+ GB_TILE - 1\) / GB_TILE\);", "vv_rtiles"),
    ("dgx_api.cu", "vv_run", r"const uint64_t c = std::max<uint64_t>\(V\.v_cap, 1\), tv = scan_tiles\(c\);",
     "a level's capacity"),
    ("dgx_api.cu", "vv_run", r"P\.tiles = vv_rtiles\(c\);", "a level's tiles"),
    ("dgx_api.cu", "vv_run", r"u32\* ticket = tickets \+ kVvTickets \* k;", "a level's tickets"),
    ("valvar_kernel.cuh", "vv_range", r"const u64 w = nrows / VV_RANGES;", "vv_range's width"),
    ("valvar_kernel.cuh", "vv_range", r"if \(w == 0\) return VV_RANGES - 1;", "vv_range for nrows < 4"),
    ("valvar_kernel.cuh", "vv_range", r"const u64 q = r / w;\s*return q < VV_RANGES - 1 \? \(u32\)q : VV_RANGES - 1;",
     "vv_range's last range"),
    ("valvar_kernel.cuh", "vv_flags_kernel", r"P\.ek_raw\[t\] = \(d << VV_RANGE_BITS\) \| vv_range\(r, P\.nrows\);",
     "the level's sort key"),
    ("valvar_kernel.cuh", "vv_heads_kernel", r"P\.head\[k\] = \(u64\)\(key != prev\) \| \(\(u64\)\(\(key >> "
     r"VV_RANGE_BITS\) != \(prev >> VV_RANGE_BITS\)\) << 32\);", "the packed heads"),
    ("valvar_kernel.cuh", "vv_fold_kernel", r"u64 acc = vv_first\(__ldg\(P\.mv \+ P\.ep\[a\]\), fl\);",
     "the fold's first item"),
    ("valvar_kernel.cuh", "vv_fold_kernel", r"for \(; k \+ 8 <= b; k \+= 8\) \{", "the fold's eight-ahead loop"),
    ("valvar_kernel.cuh", "vv_fold_kernel", r"for \(int j = 0; j < 8; \+\+j\) acc = vv_add\(c\[j\], acc, fl\);",
     "the fold's adds"),
    ("valvar_kernel.cuh", "vv_fold_kernel", r"for \(; k < b; \+\+k\) acc = vv_add\(__ldg\(P\.mv \+ __ldg\(P\.ep \+ k\)\), "
     r"acc, fl\);", "the fold's tail"),
    ("valvar_kernel.cuh", "vv_sum_items", r"if \(lane >= d && sy == seg\) x \+= y;", "the segmented scan"),
    ("valvar_kernel.cuh", "vv_sum_items", r"if \(ok && \(lane == 31 \|\| next != seg\)\) atomicAdd\(",
     "the atomicAdd per run"),
    ("valvar_kernel.cuh", "vv_combine_kernel", r"for \(u64 q = s \+ 1; q < S && !\(P\.head\[P\.sstart\[q\]\] >> 32\); "
     r"\+\+q\) acc = vv_add\(acc, P\.part\[q\], P\.is_float\);", "the ascending combine"),
    ("valvar_kernel.cuh", "vv_clamp", r"if \(x != x\) return 0\.0;", "Value()'s clamp"),
    ("valvar_kernel.cuh", "la_fold_kernel", r"for \(u64 base = a; base < b; base \+= 32\) \{", "la_fold's rounds"),
    ("valvar_kernel.cuh", "la_fold_kernel", r"for \(u32 m = __ballot_sync\(0xffffffffu, present\); m; m &= m - 1\) \{"
     r"\s*const u64 xi = __shfl_sync\(0xffffffffu, x, __ffs\(m\) - 1\);"
     r"\s*acc = cnt \? va_apply\(acc, xi, fn, fl\) : xi;", "la_fold's lanes, low to high"),
    ("valvar_kernel.cuh", "va_apply", r"return \(fn == kVaMin\) == lt \? acc : x;", "va_apply's min / max"),
]


def read_constants() -> dict:
    api, gbk, vvk, enc = (_src(f) for f in ("dgx_api.cu", "groupby_kernel.cuh", "valvar_kernel.cuh",
                                            "encode_kernel.cuh"))
    K = dict(gp.read_constants(api, gbk))
    K.update({k: v for k, v in vp.read_constants(api, vvk).items() if k not in K})
    m = _one(r"constexpr int EN_NT = (\d+), EN_VT = (\d+), EN_TILE = EN_NT \* EN_VT;", enc, "EN_TILE")
    K["EN_TILE"] = int(m.group(1)) * int(m.group(2))
    K["VV_RANGES"] = int(_one(r"constexpr int VV_RANGES = (\d+), VV_RANGE_BITS = \d+;", vvk, "VV_RANGES").group(1))
    K["kVvTickets"] = int(_one(r"constexpr size_t kVvTickets = (\d+);", api, "kVvTickets").group(1))
    K["GB_TICKETS"] = int(_one(r"ws\.zeroed\(tickets, (\d+)\);", _fn("gb_front", api), "groupby's tickets").group(1))
    if K["VV_RANGES"] != 1 << K["RANGE_BITS"]:
        raise ValueError("VV_RANGES is not 2^VV_RANGE_BITS: restate it in the radix model (tests/radix_geometry.py)")
    text = {"dgx_api.cu": api, "groupby_kernel.cuh": gbk, "valvar_kernel.cuh": vvk}
    for fn, func, pat, what in STATEMENTS:
        _one(pat, _fn(func, text[fn]) if func else text[fn], what)
    return K


K = read_constants()
NT, VT, RADIX, DB = K["GB_NT"], K["GB_VT"], K["RADIX"], K["DIGIT_BITS"]
TILE, EN_TILE, WARP = NT * VT, K["EN_TILE"], 32
RB, NRANGE = K["RANGE_BITS"], K["VV_RANGES"]

MUTANTS = {
    "ranks reversed in a warp": "__match_any_sync ranks counted from the high lane",
    "rounds reversed in a tile": "a tile's rounds scattered from the last",
    "tile-major hist": "hist[t * GB_RADIX + d]: the scan no longer orders digits first",
    "one pass fewer": "the pass count floor(width / 8) instead of the ceiling",
    "fold from the end": "a float segment folded from its last item",
    "fold without its tail": "vv_fold_kernel without `for (; k < b; ++k)`: items past the last group of eight dropped",
    "range width rounded up": "vv_range's width ceil(nrows / 4)",
    "ranges combined descending": "a rank's ranges merged from the last",
    "scan without the segment test": "the int warp scan adding across segments (no `sy == seg`)",
    "la lanes high to low": "la_fold taking a round's present lanes from lane 31 down",
}

# ---- events -----------------------------------------------------------------------------------------------------------

N_EDGES = tuple(k * TILE + d for k in (1, 2) for d in (-1, 0, 1))   # n = 2048k - 1, 2048k, 2048k + 1
EVENTS = {
    "sort: n = 0 over tiles > 0", "sort: trailing empty tiles",
    "sort: last tile ends mid-warp", "sort: last tile ends mid-round on a warp edge",
    "sort: last tile ends on a round edge",
    "sort: hist scan of exactly EN_TILE entries (8 tiles)", "sort: hist scan of one tile more, two CTAs",
    "sort: a warp whose 32 lanes share a digit", "sort: a warp of 32 distinct digits",
    "sort: a tile holding all 256 digits", "sort: one digit's items in 3 or more tiles",
    "sort: a pass in which every item has one digit", "sort: key width 8k with the all-ones key",
    "sort: key width 8k + 1, the last pass sorts one bit", "sort: no pass (key width 0)",
    "gb: a group's edges in 3 or more tiles of sort 1", "gb: equal-size groups of one parent over a tile edge in sort 2",
    "gb: a group of size nrows, nrows a power of two", "gb: parent npar - 1 = 2^b_p - 1 used",
    "gb: dest rank ndest - 1 used", "gb: npar = 1", "gb: ndest = 1",
    "gb: parents without groups first, last and between", "gb: device e_cap = E",
    "gb: device e_cap with whole empty tiles", "gb: device e_cap one short at E = 2049",
    "gb: no edge, device form", "gb: counts only",
    "vv: nrows < 4", "vv: a rank holding ranges {0,1,2,3}", "vv: a rank holding ranges {0,3}",
    "vv: a rank holding ranges {1}", "vv: a rank holding ranges {3}",
    "vv: a float segment spanning tiles", "vv: a sparse map, tiles sized by v_cap",
    "vv: levels of three different pass counts", "vv: device v_cap past v_off[nrows]", "vv: out_cap one short",
    "vv: no contributing value",
    "int: a segment crossing lane 31 to 0", "int: a segment crossing a CTA edge", "int: a whole warp in one segment",
    "int: 32 one-item segments in a warp", "int: a wrapping segment sum",
    "la: nrows = 8k - 1", "la: nrows = 8k + 1", "la: only lane 0 present", "la: only lane 31 present",
    "la: alternating lanes present", "la: NaN first (min / max)", "la: NaN after the first (min / max)",
    "la: out_cap one short",
} | {f"sort: n = {n}" for n in N_EDGES} \
  | {f"gb: P1 = {p}" for p in range(0, 7)} | {f"gb: P2 = {p}" for p in range(1, 7)} \
  | {f"vv: P = {p}" for p in range(1, 5)} \
  | {f"vv: nrows = 4w + {i}, contributing rows at every range edge" for i in range(4)} \
  | {f"vv: a float segment of {n} items" for n in (1, 2, 8, 9, 16, 17)} \
  | {f"la: a row of {n} values" for n in (0, 1, 31, 32, 33, 63, 64, 65)}


def _add(ev, name):
    if name not in EVENTS:
        raise KeyError(f"event {name!r} is not registered in radix_geometry.EVENTS")
    ev.add(name)


# ---- the sort ---------------------------------------------------------------------------------------------------------

def _cumcount(g):
    """Per item: its rank among the earlier items of its group, and its group's size (g: int64 group ids)."""
    n = g.size
    if n == 0:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    order = np.argsort(g, kind="stable")
    gs = g[order]
    start = np.r_[True, gs[1:] != gs[:-1]]
    idx = np.arange(n)
    first = np.maximum.accumulate(np.where(start, idx, 0))
    rank = np.empty(n, np.int64)
    rank[order] = idx - first
    ends = np.r_[np.nonzero(start)[0], n]
    size = np.empty(n, np.int64)
    size[order] = np.repeat(np.diff(ends), np.diff(ends))
    return rank, size


def npasses(width: int, mut=frozenset()) -> int:
    return width // DB if "one pass fewer" in mut else -(-width // DB)


Pass = namedtuple("Pass", "shift digit tile round warp lane match lrank hist span")
Sort = namedtuple("Sort", "n tiles passes hist_ctas key pay steps launches")


def radix_sort(key, pay, tiles, width, ev, mut=frozenset()) -> Sort:
    """gb_sort over n = key.size items in `tiles` tiles, npasses(width) passes; the result is where the last pass
    leaves it.  Each step records the pass's digits, the (tile, round, warp, lane) of every item, its
    __match_any_sync group size and rank, the hist and each digit's [first, last] tile."""
    key = np.asarray(key, np.uint64)
    pay = np.asarray(pay)
    n = key.size
    assert tiles >= max(1, -(-n // TILE))
    passes = npasses(width, mut)
    hn = RADIX * tiles
    ctas = -(-hn // EN_TILE)
    if passes == 0:  # gb_sort launches nothing: none of the sort's edges is reached
        _add(ev, "sort: no pass (key width 0)")
    elif n == 0:
        _add(ev, "sort: n = 0 over tiles > 0")
    else:
        if tiles > -(-n // TILE):
            _add(ev, "sort: trailing empty tiles")
        if n in N_EDGES:
            _add(ev, f"sort: n = {n}")
        rem = n % TILE
        if rem % WARP:
            _add(ev, "sort: last tile ends mid-warp")
        elif rem % NT:
            _add(ev, "sort: last tile ends mid-round on a warp edge")
        elif rem:
            _add(ev, "sort: last tile ends on a round edge")
        if width % DB == 0 and width and np.any(key == np.uint64((1 << width) - 1)):
            _add(ev, "sort: key width 8k with the all-ones key")
        if width % DB == 1:
            _add(ev, "sort: key width 8k + 1, the last pass sorts one bit")
    if passes and hn == EN_TILE:
        _add(ev, "sort: hist scan of exactly EN_TILE entries (8 tiles)")
    if passes and hn == EN_TILE + RADIX and ctas == 2:
        _add(ev, "sort: hist scan of one tile more, two CTAs")
    e = np.arange(n, dtype=np.int64)
    t, gr, w, lane = e // TILE, e // NT, e // WARP, e % WARP
    steps = []
    for q in range(passes):
        d = ((key >> np.uint64(q * DB)) & np.uint64(RADIX - 1)).astype(np.int64)
        lr, msz = _cumcount(w * RADIX + d)          # __match_any_sync: rank and popc(same)
        rr, rsz = _cumcount(gr * RADIX + d)         # rank inside the round: warp offset + lane rank
        tr, tsz = _cumcount(t * RADIX + d)          # rank inside the tile: round base + the above
        warp_off, round_off = rr - lr, tr - rr
        span = np.full((RADIX, 2), -1, np.int64)    # each digit's first and last tile
        if n:
            u, i0 = np.unique(d, return_index=True)
            _, i1 = np.unique(d[::-1], return_index=True)
            span[u, 0], span[u, 1] = t[i0], t[n - 1 - i1]
            if np.any(msz == WARP):
                _add(ev, "sort: a warp whose 32 lanes share a digit")
            if np.any(np.bincount(w[lr == 0]) == WARP):
                _add(ev, "sort: a warp of 32 distinct digits")
            if np.any(np.bincount(t[tr == 0], minlength=tiles) == RADIX):
                _add(ev, "sort: a tile holding all 256 digits")
            if np.any(span[:, 1] - span[:, 0] >= 2):
                _add(ev, "sort: one digit's items in 3 or more tiles")
            if n > TILE and np.all(d == d[0]):
                _add(ev, "sort: a pass in which every item has one digit")
        if "ranks reversed in a warp" in mut:
            lr = msz - 1 - lr
        if "rounds reversed in a tile" in mut:
            round_off = tsz - round_off - rsz
        idx = t * RADIX + d if "tile-major hist" in mut else d * tiles + t
        hist = np.bincount(idx, minlength=hn).astype(np.int64)
        hoff = np.concatenate([[0], np.cumsum(hist)[:-1]])
        pos = hoff[idx] + round_off + warp_off + lr
        assert np.array_equal(np.sort(pos), e), "the scatter is not a permutation"
        ko, po = np.empty_like(key), np.empty_like(pay)
        ko[pos], po[pos] = key, pay
        steps.append(Pass(q * DB, d, t, (e % TILE) // NT, w, lane, msz, lr, hist, span))
        key, pay = ko, po
    return Sort(n, tiles, passes, ctas, key, pay, steps, K["SORT_PER_PASS"] * passes)


# ---- @groupby ----------------------------------------------------------------------------------------------------------

GbCall = namedtuple("GbCall", "form members e_cap")   # form "host" / "dev"; e_cap None: E
GbOut = namedtuple("GbOut", "rc sync G E keys grp_off mem_off members launches sorts")


def gb_plan(nrows, ndest, npar, mut=frozenset()):
    b_p, b_d, b_s = gp.bits(npar - 1), gp.bits(ndest - 1 if ndest else 0), gp.bits(nrows)
    return b_p, b_d, b_s, npasses(b_p + b_d, mut), npasses(b_p + b_s, mut)


def gb_edges(src, v, v_off, par, par_off):
    """The expand kernel's edges in (parent, source) order: (parent, row, value) per edge."""
    npar, nrows = par_off.size - 1, v_off.size - 1
    PV = int(par_off[-1])
    ppar = np.repeat(np.arange(npar, dtype=np.int64), np.diff(par_off.astype(np.int64)))
    x = par[:PV]
    i = np.minimum(np.searchsorted(src[:nrows], x), nrows - 1)   # nrows > 0
    hit = src[i] == x
    lens = np.where(hit, np.diff(v_off.astype(np.int64))[i], 0)
    E = int(lens.sum())
    j = np.repeat(np.arange(PV, dtype=np.int64), lens)
    eoff = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
    k = np.arange(E, dtype=np.int64) - eoff[j]
    row = i[j].astype(np.int64)
    return ppar[j], row, v[v_off[row].astype(np.int64) + k] if E else np.zeros(0, np.uint64)


def groupby(fx, call: GbCall, mut=frozenset(), ev=None) -> GbOut:
    ev = set() if ev is None else ev
    src, v, v_off, par, par_off, dest = fx.src, fx.v, fx.v_off, fx.par, fx.par_off, fx.dest
    nrows, npar, ndest = v_off.size - 1, par_off.size - 1, dest.size
    M, PV = int(v_off[-1]), int(par_off[-1])
    b_p, b_d, b_s, p1, p2 = gb_plan(nrows, ndest, npar, mut)
    empty = GbOut(OK, OK, 0, 0, np.zeros(0, np.uint64), np.zeros(npar + 1, np.uint64), np.zeros(1, np.uint64),
                  np.zeros(0, np.uint64), 0, ())
    if npar == 0 or M == 0 or PV == 0 or nrows == 0:
        return empty
    if npar == 1:
        _add(ev, "gb: npar = 1")
    if ndest == 1:
        _add(ev, "gb: ndest = 1")
    if not call.members:
        _add(ev, "gb: counts only")
    full = gp.K["FRONT"] + gp.K["BACK"] + gp.K["SORT_PER_PASS"] * (p1 + p2)
    assert 1 + p1 + 1 + p2 + 1 <= K["GB_TICKETS"]
    ppar, row, val = gb_edges(src, v, v_off, par, par_off)
    E = row.size
    if E == 0 and call.form == "host":
        return empty._replace(launches=gp.K["FRONT"])
    e_cap = E if call.form == "host" or call.e_cap is None else call.e_cap
    tiles = -(-max(e_cap, 1) // TILE)
    if call.form == "dev":
        if e_cap == E:
            _add(ev, "gb: device e_cap = E")
        elif e_cap > E and tiles > -(-max(E, 1) // TILE):
            _add(ev, "gb: device e_cap with whole empty tiles")
        if E == 0:
            _add(ev, "gb: no edge, device form")
    if E > e_cap:
        if E == 2049 and e_cap == 2048:
            _add(ev, "gb: device e_cap one short at E = 2049")
        return GbOut(OK, ERR_CAP, 0, E, None, None, None, None, full, ())
    if not mut:
        _add(ev, f"gb: P1 = {p1}")
        _add(ev, f"gb: P2 = {p2}")
    r = np.searchsorted(dest, val).astype(np.uint64)
    assert np.all(dest[np.minimum(r, ndest - 1).astype(np.int64)] == val), "a value outside dest is refused"
    ek = (ppar.astype(np.uint64) << np.uint64(b_d)) | r
    if E:
        if np.any(r == ndest - 1):
            _add(ev, "gb: dest rank ndest - 1 used")
        if npar - 1 == (1 << b_p) - 1 and np.any(ppar == npar - 1) and npar > 1:
            _add(ev, "gb: parent npar - 1 = 2^b_p - 1 used")
        gid = np.unique(ek, return_inverse=True)[1].astype(np.int64)
        tiles_per_key = np.bincount(np.unique(gid * (tiles + 1) + np.arange(E) // TILE) // (tiles + 1))
        if np.any(tiles_per_key >= 3):
            _add(ev, "gb: a group's edges in 3 or more tiles of sort 1")
    s1 = radix_sort(ek, row.astype(np.uint32), tiles, b_p + b_d, ev, mut)
    eks, eps = s1.key, s1.pay.astype(np.int64)
    head = np.r_[True, eks[1:] != eks[:-1]] if E else np.zeros(0, bool)
    gstart = np.nonzero(head)[0]
    G = gstart.size
    size = np.diff(np.r_[gstart, E]).astype(np.uint64)
    gk = ((eks[gstart] >> np.uint64(b_d)) << np.uint64(b_s)) | size
    if G > TILE:
        gpar = eks[gstart] >> np.uint64(b_d)
        for p in np.unique(gpar):
            sel = np.nonzero(gpar == p)[0]
            for s in np.unique(size[sel]):
                at = sel[size[sel] == s]
                if at.size > 1 and at[0] // TILE != at[-1] // TILE:
                    _add(ev, "gb: equal-size groups of one parent over a tile edge in sort 2")
    if np.any(size == nrows) and (nrows & (nrows - 1)) == 0:
        _add(ev, "gb: a group of size nrows, nrows a power of two")
    s2 = radix_sort(gk, np.arange(G, dtype=np.uint32), tiles, b_p + b_s, ev, mut)
    gks, gps = s2.key, s2.pay.astype(np.int64)
    gsz = size[gps]
    moff = np.concatenate([[0], np.cumsum(gsz)]).astype(np.uint64)
    mask = np.uint64((1 << b_d) - 1)
    keys = dest[(eks[gstart[gps]] & mask).astype(np.int64)] if G else np.zeros(0, np.uint64)
    grp_off = np.searchsorted(gks >> np.uint64(b_s), np.arange(npar + 1, dtype=np.uint64), "left").astype(np.uint64)
    gcount = np.diff(grp_off.astype(np.int64))
    nz = np.nonzero(gcount)[0]
    if nz.size and gcount[0] == 0 and gcount[-1] == 0 and np.any(gcount[nz[0]:nz[-1]] == 0):
        _add(ev, "gb: parents without groups first, last and between")
    inv = np.empty(G, np.int64)
    inv[gps] = np.arange(G)
    g_of = np.cumsum(head) - 1
    members = np.empty(E, np.uint64)
    members[moff[inv[g_of]].astype(np.int64) + np.arange(E) - gstart[g_of]] = src[eps]
    return GbOut(OK, OK, G, E, keys, grp_off, moff, members if call.members else None, full, (s1, s2))


GbFix = namedtuple("GbFix", "name src v v_off par par_off dest calls events kills")


def gb_oracle(fx):
    """groupby_oracle.c's (keys, grp_off, mem_off, members) for the fixture."""
    import groupby_oracle as gbo

    # The restatement walks every row for every parent.  A parent row without a value owns no group, so it runs over
    # the rows that hold one and the others are spread back into grp_off (the sparse fixtures have 2^20 parents).
    _, row, _ = gb_edges(fx.src, fx.v, fx.v_off, fx.par, fx.par_off)
    cap = max(row.size, 1)
    keys, agg, mem = (np.empty(cap, np.uint64) for _ in range(3))
    npar = fx.par_off.size - 1
    lens = np.diff(fx.par_off.astype(np.int64))
    used = np.nonzero(lens)[0]
    u_off = np.zeros(used.size + 1, np.uint64)
    np.cumsum(lens[used], out=u_off[1:])
    g_used, mem_off = np.empty(used.size + 1, np.uint64), np.empty(cap + 1, np.uint64)
    b = [x if x.size else np.zeros(1, np.uint64) for x in (fx.src, fx.v, fx.par)]
    n = gbo.lib().orc_groupby_uid(b[0].ctypes.data, fx.v_off.size - 1, b[1].ctypes.data, fx.v_off.ctypes.data,
                                  b[2].ctypes.data, u_off.ctypes.data, used.size, keys.ctypes.data, agg.ctypes.data,
                                  g_used.ctypes.data, mem_off.ctypes.data, mem.ctypes.data)
    g_used[used.size] = n
    cnt = np.zeros(npar, np.int64)
    cnt[used] = np.diff(g_used.astype(np.int64))
    grp_off = np.zeros(npar + 1, np.uint64)
    np.cumsum(cnt, out=grp_off[1:])
    return keys[:n].copy(), grp_off, mem_off[:n + 1].copy(), mem[:int(mem_off[n])].copy()


# ---- value variables ---------------------------------------------------------------------------------------------------

VvCall = namedtuple("VvCall", "form v_caps out_cap")     # v_caps None: v_off[nrows] per level; out_cap None: exact
VvOut = namedtuple("VvOut", "rc sync n keys vals launches sorts")
Level = namedtuple("Level", "src v v_off dest")


def vv_range(r, nrows, mut=frozenset()):
    w = -(-nrows // NRANGE) if "range width rounded up" in mut else nrows // NRANGE
    if w == 0:
        return np.full(np.shape(r), NRANGE - 1, np.int64)
    return np.minimum(np.asarray(r, np.int64) // w, NRANGE - 1)


def _f(w):
    return np.asarray(w, np.uint64).view(np.float64)


def _clamp(x):
    x = np.where(np.isnan(x), 0.0, x)
    return np.where(x == np.inf, FMAX, np.where(x == -np.inf, -FMAX, x))


def _add_w(a, b, is_float):
    """vv_add: clamp(a + b) for floats, a wrapping add for ints, on u64 words."""
    if not is_float:
        return a + b
    with np.errstate(over="ignore", invalid="ignore"):
        return _clamp(_f(a) + _f(b)).view(np.uint64)


def _seq_fold(vals, starts, lens, step, first=None):
    """acc = first(vals[start]), then acc = step(acc, vals[start + i]) for i = 1 .. len - 1, every segment at once."""
    S = starts.size
    out = np.zeros(S, vals.dtype)
    if S == 0:
        return out
    order = np.argsort(-lens, kind="stable")
    st, ln = starts[order], lens[order]
    acc = vals[st].copy() if first is None else first(vals[st])
    for i in range(1, int(ln.max()) if ln.size else 0):
        c = int(np.searchsorted(-ln, -i, "left"))   # segments longer than i: a prefix of the order
        acc[:c] = step(acc[:c], vals[st[:c] + i])
    out[order] = acc
    return out


def _int_parts(x, seg, S, mut, ev):
    """vv_sum_items: per item a Hillis-Steele scan across its warp (limited to its segment's run unless mutated), and
    one wrapping atomicAdd per run end into the segment's part."""
    E = x.size
    k = np.arange(E)
    lane = k % WARP
    wstart = k - lane
    sstart_of = np.maximum.accumulate(np.where(np.r_[True, seg[1:] != seg[:-1]], k, 0)) if E else k
    gs = wstart if "scan without the segment test" in mut else np.maximum(wstart, sstart_of)
    cs = np.concatenate([[np.uint64(0)], np.cumsum(x, dtype=np.uint64)])
    inc = cs[k + 1] - cs[gs]
    nxt = np.r_[seg[1:], -1]
    run_end = (lane == WARP - 1) | (nxt != seg)
    part = np.zeros(S, np.uint64)
    np.add.at(part, seg[run_end], inc[run_end])
    if E:
        lens = np.bincount(seg, minlength=S)
        cross = (lane[:-1] == WARP - 1) & (seg[:-1] == seg[1:])
        if np.any(cross):
            _add(ev, "int: a segment crossing lane 31 to 0")
        if np.any((k[:-1] % NT == NT - 1) & (seg[:-1] == seg[1:])):
            _add(ev, "int: a segment crossing a CTA edge")
        full = E // WARP
        if full:
            ws = seg[:full * WARP].reshape(full, WARP)
            if np.any(np.all(ws == ws[:, :1], axis=1)):
                _add(ev, "int: a whole warp in one segment")
            one = lens[ws] == 1
            if np.any(np.all(one, axis=1)):
                _add(ev, "int: 32 one-item segments in a warp")
        starts = np.nonzero(np.r_[True, seg[1:] != seg[:-1]])[0]
        fs = np.add.reduceat(x.view(np.int64).astype(np.float64), starts)
        if np.any(np.abs(fs) >= 2.0 ** 63):
            _add(ev, "int: a wrapping segment sum")
    return part


def propagate(fx, words, is_float, call: VvCall, mut=frozenset(), ev=None) -> VvOut:
    """The levels of vv_run over the map (fx.keys, words); the outputs the last level writes."""
    ev = set() if ev is None else ev
    mk, mv = np.asarray(fx.keys, np.uint64), np.asarray(words, np.uint64)
    if mk.size == 0:
        return VvOut(OK, OK, 0, np.zeros(0, np.uint64), np.zeros(0, np.uint64), 0, ())
    launches, sorts, passes_of = 0, [], []
    nl = len(fx.levels)
    for li, L in enumerate(fx.levels):
        nrows, M, ndest = L.v_off.size - 1, int(L.v_off[-1]), L.dest.size
        v_cap = M if call.form == "host" or call.v_caps is None else call.v_caps[li]
        if v_cap > M:
            _add(ev, "vv: device v_cap past v_off[nrows]")
        b_d = gp.bits(ndest - 1 if ndest else 0)
        passes = npasses(b_d + RB, mut)
        assert 2 + passes <= K["kVvTickets"]
        passes_of.append(passes)
        if not mut:
            _add(ev, f"vv: P = {passes}")
        launches += K["LEVEL"] + K["SORT_PER_PASS"] * passes
        tiles = max(1, -(-max(v_cap, 1) // TILE))
        r = np.repeat(np.arange(nrows, dtype=np.int64), np.diff(L.v_off.astype(np.int64)))
        d = np.searchsorted(L.dest, L.v[:M]).astype(np.int64)
        j = np.searchsorted(mk, L.src[r]) if M else np.zeros(0, np.int64)
        hit = (j < mk.size) & (mk[np.minimum(j, mk.size - 1)] == L.src[r]) if M else np.zeros(0, bool)
        rng = vv_range(r, nrows, mut)
        if nrows < NRANGE:
            _add(ev, "vv: nrows < 4")
        elif hit.any():
            w = nrows // NRANGE
            edges = {w - 1, w, 2 * w, 3 * w - 1, 3 * w, nrows - 1}
            if edges <= set(r[hit].tolist()):
                _add(ev, f"vv: nrows = 4w + {nrows % NRANGE}, contributing rows at every range edge")
        ek = (d[hit].astype(np.uint64) << np.uint64(RB)) | rng[hit].astype(np.uint64)
        ep = j[hit].astype(np.uint32)
        E = ek.size
        if E == 0:
            _add(ev, "vv: no contributing value")
        elif 4 * E <= M and tiles > -(-E // TILE):
            _add(ev, "vv: a sparse map, tiles sized by v_cap")
        s = radix_sort(ek, ep, tiles, b_d + RB, ev, mut)
        sorts.append(s)
        eks, eps = s.key, s.pay.astype(np.int64)
        prev = np.r_[np.uint64(U64), eks[:-1]] if E else eks
        seg_head = eks != prev
        rank_head = (eks >> np.uint64(RB)) != (prev >> np.uint64(RB))
        if E:
            seg_head[0] = rank_head[0] = True
        sstart = np.nonzero(seg_head)[0]
        S = sstart.size
        slen = np.diff(np.r_[sstart, E])
        x = mv[eps]
        if is_float:
            # vv_fold_kernel: acc = clamp(first), then acc = clamp(c + acc); the eight-ahead gather keeps this order
            xs, st = (x[::-1].copy(), E - sstart - slen) if "fold from the end" in mut else (x, sstart)
            fl = 1 + (slen - 1) // 8 * 8 if "fold without its tail" in mut else slen
            part = _seq_fold(xs, st, fl, lambda a, c: _add_w(c, a, True),
                             first=lambda c: _clamp(_f(c)).view(np.uint64))
            if S:
                for n_ in (1, 2, 8, 9, 16, 17):
                    if np.any(slen == n_):
                        _add(ev, f"vv: a float segment of {n_} items")
                if np.any(sstart // TILE != (sstart + slen - 1) // TILE):
                    _add(ev, "vv: a float segment spanning tiles")
        else:
            seg = np.cumsum(seg_head) - 1
            part = _int_parts(x, seg, S, mut, ev)
        # vv_combine_kernel: per rank, its segments' parts in ascending (mutant: descending) range order
        rstart = np.nonzero(rank_head[sstart])[0] if S else np.zeros(0, np.int64)
        G = rstart.size
        nseg = np.diff(np.r_[rstart, S])
        rmask = np.zeros(G, np.int64)
        if S:
            srng = (eks[sstart] & np.uint64(NRANGE - 1)).astype(np.int64)
            np.bitwise_or.at(rmask, np.repeat(np.arange(G), nseg), 1 << srng)
        for m_, name in ((0b1111, "{0,1,2,3}"), (0b1001, "{0,3}"), (0b0010, "{1}"), (0b1000, "{3}")):
            if np.any(rmask == m_):
                _add(ev, f"vv: a rank holding ranges {name}")
        if "ranges combined descending" in mut:
            order = np.concatenate([np.arange(a, a + c)[::-1] for a, c in zip(rstart, nseg)]) if G else rstart
            pv = part[order]
        else:
            pv = part
        vals = _seq_fold(pv, rstart, nseg, lambda a, c: _add_w(a, c, is_float))
        nkeys = L.dest[(eks[sstart[rstart]] >> np.uint64(RB)).astype(np.int64)] if G else np.zeros(0, np.uint64)
        mk, mv = nkeys, vals
    if len(set(passes_of)) >= 3:
        _add(ev, "vv: levels of three different pass counts")
    out_cap = mk.size if call.out_cap is None else call.out_cap
    if mk.size > out_cap:
        if out_cap == mk.size - 1:
            _add(ev, "vv: out_cap one short")
        return VvOut(ERR_CAP if call.form == "host" else OK, ERR_CAP, mk.size, None, None, launches, tuple(sorts))
    return VvOut(OK, OK, mk.size, mk, mv, launches, tuple(sorts))


VvFix = namedtuple("VvFix", "name keys vals levels calls events kills")   # vals: int64 / float64 arrays


def vv_oracle(fx, vals):
    import valvar_oracle as vo

    k, v = vo.propagate_csr(fx.keys, vals, [(L.src, L.v, L.v_off) for L in fx.levels])
    return k, np.asarray(v).view(np.uint64)


# ---- level aggregation ------------------------------------------------------------------------------------------------

LaCall = namedtuple("LaCall", "form v_cap out_cap")
LaFix = namedtuple("LaFix", "name keys vals src v v_off fns calls events kills")
FNS = {"min": 0, "max": 1, "sum": 2, "avg": 3}


def level_agg(fx, words, is_float, fn, call: LaCall, mut=frozenset(), ev=None) -> VvOut:
    """la_run: a warp per row, lanes look their value up, the present ones folded in rounds of 32 in lane order."""
    ev = set() if ev is None else ev
    mk, mv = np.asarray(fx.keys, np.uint64), np.asarray(words, np.uint64)
    nrows, M = fx.v_off.size - 1, int(fx.v_off[-1])
    v_cap = M if call.form == "host" or call.v_cap is None else call.v_cap
    if mk.size == 0 or nrows == 0 or v_cap == 0 or M == 0 and call.form == "host":
        return VvOut(OK, OK, 0, np.zeros(0, np.uint64), np.zeros(0, np.uint64), 0, ())
    rlen = np.diff(fx.v_off.astype(np.int64))
    for n_ in (0, 1, 31, 32, 33, 63, 64, 65):
        if np.any(rlen == n_):
            _add(ev, f"la: a row of {n_} values")
    if nrows % 8 == 7:
        _add(ev, "la: nrows = 8k - 1")
    if nrows % 8 == 1 and nrows > 8:
        _add(ev, "la: nrows = 8k + 1")
    r = np.repeat(np.arange(nrows, dtype=np.int64), rlen)
    pos = np.arange(M, dtype=np.int64) - fx.v_off[r].astype(np.int64)
    rnd, lane = pos // WARP, pos % WARP
    j = np.searchsorted(mk, fx.v[:M])
    present = (j < mk.size) & (mk[np.minimum(j, mk.size - 1)] == fx.v[:M])
    if present.any():
        rr = r[present] * (int(rnd.max()) + 1) + rnd[present]
        u, inv = np.unique(rr, return_inverse=True)
        masks = np.zeros(u.size, np.uint64)
        np.bitwise_or.at(masks, inv, np.uint64(1) << lane[present].astype(np.uint64))
        for m_, name in ((1, "la: only lane 0 present"), (1 << 31, "la: only lane 31 present"),
                         (0x55555555, "la: alternating lanes present"), (0xAAAAAAAA, "la: alternating lanes present")):
            if np.any(masks == np.uint64(m_)):
                _add(ev, name)
    lk = WARP - 1 - lane if "la lanes high to low" in mut else lane
    order = np.lexsort((lk, rnd, r))
    order = order[present[order]]
    x, rows = mv[j[order]], r[order]
    cnt = np.bincount(rows, minlength=nrows)
    has = np.nonzero(cnt)[0]
    starts = np.concatenate([[0], np.cumsum(cnt[has])[:-1]]).astype(np.int64)
    f = FNS[fn]
    if is_float and f in (0, 1) and x.size:
        nan = np.isnan(_f(x))
        if np.any(nan[starts] & (cnt[has] > 1)):
            _add(ev, "la: NaN first (min / max)")
        first = np.zeros(x.size, bool)
        first[starts] = True
        if np.any(nan & ~first):
            _add(ev, "la: NaN after the first (min / max)")

    def step(acc, c):
        if f in (0, 1):
            lt = _f(acc) < _f(c) if is_float else acc.view(np.int64) < c.view(np.int64)
            return np.where(lt, acc, c) if f == 0 else np.where(lt, c, acc)
        if is_float:
            with np.errstate(over="ignore", invalid="ignore"):
                return (_f(acc) + _f(c)).view(np.uint64)
        return acc + c

    acc = _seq_fold(x, starts, cnt[has], step)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        if f == 3:
            s = _f(acc) if is_float else acc.view(np.int64).astype(np.float64)
            acc = _clamp(s / cnt[has].astype(np.float64)).view(np.uint64)
        elif is_float:
            acc = _clamp(_f(acc)).view(np.uint64)
    G = has.size
    out_cap = G if call.out_cap is None else call.out_cap
    if G > out_cap:
        if out_cap == G - 1:
            _add(ev, "la: out_cap one short")
        return VvOut(ERR_CAP if call.form == "host" else OK, ERR_CAP, G, None, None, K["AGG"], ())
    return VvOut(OK, OK, G, fx.src[has], acc, K["AGG"], ())


def la_oracle(fx, vals, fn):
    import valvar_oracle as vo

    k, v = vo.level_agg_csr(fn, fx.keys, vals, fx.src, fx.v, fx.v_off)
    return k, np.asarray(v).view(np.uint64)


# ---- fixture builders -------------------------------------------------------------------------------------------------

def csr(rows):
    rows = [np.ascontiguousarray(np.asarray(r, np.uint64)) for r in rows]
    off = np.zeros(len(rows) + 1, np.uint64)
    if rows:
        np.cumsum([r.size for r in rows], out=off[1:])
    return (np.concatenate(rows) if int(off[-1]) else np.zeros(0, np.uint64)), off


def _u(x):
    return np.ascontiguousarray(np.asarray(x, np.uint64))


GB_DEFAULT = (GbCall("host", True, None), GbCall("host", False, None), GbCall("dev", True, None),
              GbCall("dev", False, None))


def _gb(name, parents, src, rows, dest, events, kills=(), calls=GB_DEFAULT):
    v, v_off = csr(rows)
    par, par_off = parents if isinstance(parents, tuple) else csr(parents)
    return GbFix(name, _u(src), v, v_off, _u(par), _u(par_off), _u(dest), tuple(calls), set(events), set(kills))


def _sparse_parents(npar, used):
    """npar parent rows, empty but for used = {p: ascending values}: (par, par_off) built in O(npar)."""
    cnt = np.zeros(npar, np.int64)
    for p, vals in used.items():
        cnt[p] = len(vals)
    off = np.zeros(npar + 1, np.uint64)
    np.cumsum(cnt, out=off[1:])
    par = np.concatenate([np.asarray(used[p], np.uint64) for p in sorted(used)])
    return par, off


def gb_fixtures():
    rng = np.random.default_rng(9100)
    fx = []
    src = np.arange(1, 20_000, dtype=np.uint64) * 3
    d64 = np.arange(64, dtype=np.uint64) * 5 + 7
    # sort 1 of 2047 edges in one pass; sort 2 puts 63 groups of 32 in one warp-wide tie
    s = src[:2047]
    fx.append(_gb("E = 2047, 64 keys", [s], s, [[d64[(i * 7) % 64]] for i in range(2047)], d64,
                  {"sort: n = 2047", "sort: last tile ends mid-warp", "gb: P1 = 1", "gb: P2 = 2"},
                  {"ranks reversed in a warp", "rounds reversed in a tile"}))
    d256 = np.arange(256, dtype=np.uint64) * 11 + 1
    s = src[:2048]
    fx.append(_gb("E = 2048, every digit in the tile", [s], s, [[d256[i % 256]] for i in range(2048)], d256,
                  {"sort: n = 2048", "sort: a tile holding all 256 digits", "sort: a warp of 32 distinct digits",
                   "sort: key width 8k with the all-ones key", "gb: dest rank ndest - 1 used"}))
    s = src[:2049]
    d40 = np.arange(40, dtype=np.uint64) * 13 + 2
    rows = [[d40[int(x)]] for x in rng.integers(0, 40, 2049)]
    calls = GB_DEFAULT + (GbCall("dev", True, 2048), GbCall("dev", True, 2049 + 3 * TILE),
                          GbCall("dev", False, 2049 + 3 * TILE))
    fx.append(_gb("E = 2049, e_cap exact, one short and with empty tiles", [s, []], s, rows, d40,
                  {"sort: n = 2049", "gb: device e_cap one short at E = 2049", "gb: device e_cap with whole empty tiles",
                   "sort: trailing empty tiles", "gb: device e_cap = E"}, {"rounds reversed in a tile"}, calls))
    s = src[:4095]
    d9 = np.arange(9, dtype=np.uint64) * 17 + 3
    rows = [[d9[0]] if i < 32 or i % 3 == 0 else [d9[1 + i % 8]] for i in range(4095)]
    fx.append(_gb("E = 4095, a warp of one key", [s], s, rows, d9,
                  {"sort: n = 4095", "sort: a warp whose 32 lanes share a digit"},
                  {"ranks reversed in a warp", "rounds reversed in a tile"}))
    s = src[:4096]
    # an empty second parent: b_p = 1, so sort 1 runs one pass over the 4 096 edges
    fx.append(_gb("E = 4096, one group of nrows = 2^12", [s, []], s, [[99]] * 4096, [99],
                  {"sort: n = 4096", "gb: a group of size nrows, nrows a power of two", "gb: ndest = 1"},
                  {"ranks reversed in a warp", "rounds reversed in a tile"}))
    s = src[:300]
    fx.append(_gb("npar = 1, ndest = 1: sort 1 has no pass", [s], s, [[99]] * 300, [99],
                  {"gb: P1 = 0", "sort: no pass (key width 0)", "gb: npar = 1", "gb: ndest = 1"}))
    s = src[:4097]
    d300 = np.arange(300, dtype=np.uint64) * 7 + 5
    fx.append(_gb("E = 4097, 300 keys over 3 tiles", [s], s, [[d300[int(x)]] for x in rng.integers(0, 300, 4097)],
                  d300, {"sort: n = 4097", "sort: one digit's items in 3 or more tiles",
                         "gb: a group's edges in 3 or more tiles of sort 1",
                         "sort: key width 8k + 1, the last pass sorts one bit"},
                  {"tile-major hist", "one pass fewer", "ranks reversed in a warp", "rounds reversed in a tile"}))
    s = src[:4098]
    d2049 = np.arange(2049, dtype=np.uint64) * 3 + 1
    fx.append(_gb("2049 groups of 2, ties over a tile edge in sort 2", [s], s, [[d2049[i // 2]] for i in range(4098)],
                  d2049, {"gb: equal-size groups of one parent over a tile edge in sort 2",
                          "sort: a pass in which every item has one digit"},
                  {"rounds reversed in a tile", "ranks reversed in a warp"}))
    s = src[:200]
    fx.append(_gb("P1 = 1, P2 = 1", [s[::2]], s, [np.sort(rng.choice(d64, 3, replace=False)) for _ in range(200)],
                  d64, {"gb: P2 = 1"}, {"ranks reversed in a warp"}))
    fx.append(_gb("no edge reaches a parent", [[5, 8], []], s, [[d64[0]]] * 200, d64,
                  {"gb: no edge, device form", "sort: n = 0 over tiles > 0"},
                  calls=GB_DEFAULT + (GbCall("dev", True, 5000),)))
    # the pass counts: large npar / ndest, few edges; parents and dest values mostly unused
    for name, npar, ndest, nrows, used, events, kills in (
            ("P1 = 3: npar 2^8, ndest 2^12 + 1", 256, (1 << 12) + 1, 3000, (15, 16, 255), {
                "gb: P1 = 3", "gb: P2 = 3", "gb: parent npar - 1 = 2^b_p - 1 used",
                "sort: last tile ends mid-round on a warp edge"}, {"one pass fewer"}),
            ("P1 = 4: npar 2^12, ndest 2^20, the all-ones key", 1 << 12, 1 << 20, 8192, (1023, 1024, 4095), {
                "gb: P1 = 4", "gb: P2 = 4", "sort: last tile ends on a round edge"}, {"one pass fewer"}),
            ("P1 = 5, P2 = 5: npar 2^16 + 1, ndest 2^15 + 1, nrows 2^15", (1 << 16) + 1, (1 << 15) + 1, 1 << 15,
             (0, 1 << 15, 1 << 16), {"gb: P1 = 5", "gb: P2 = 5"}, {"ranks reversed in a warp"}),
            ("P1 = 6, P2 = 6: npar and ndest 2^20 + 1, nrows 2^19", (1 << 20) + 1, (1 << 20) + 1, 1 << 19,
             (7, 9, 1 << 19), {"gb: P1 = 6", "gb: P2 = 6", "gb: parents without groups first, last and between"},
             {"ranks reversed in a warp"})):
        dest = np.arange(ndest, dtype=np.uint64) * 2 + 1
        srcp = np.arange(nrows, dtype=np.uint64) * 5 + 2
        # E per fixture: 96 (mid-round on a warp edge), 512 (a round edge), else a few hundred
        E = {3000: 96, 8192: 512, 1 << 15: 90}.get(nrows, 600)
        per = -(-E // len(used))
        lens, vals = np.zeros(nrows, np.int64), np.zeros(nrows, np.uint64)
        par = {}
        for k, p in enumerate(used):
            take = np.arange(k * per, min((k + 1) * per, E))
            par[p] = srcp[take]
            lens[take] = 1  # one value per row, the slice's last one the largest rank
            vals[take] = dest[rng.integers(0, ndest - 1, take.size)]
            vals[take[-1]] = dest[ndest - 1]
        v_off = np.zeros(nrows + 1, np.uint64)
        np.cumsum(lens, out=v_off[1:])
        fx.append(GbFix(name, srcp, vals[lens > 0], v_off, *_sparse_parents(npar, par), dest, GB_DEFAULT,
                        events | {"gb: dest rank ndest - 1 used"}, kills))
    return fx


VV_DEFAULT = (VvCall("host", None, None), VvCall("dev", None, None))


def _lv(src, rows, dest):
    v, v_off = csr(rows)
    return Level(_u(src), v, v_off, _u(dest))


def _vv(name, keys, vals, levels, events, kills=(), calls=VV_DEFAULT):
    return VvFix(name, _u(keys), tuple(vals), tuple(levels), tuple(calls), set(events), set(kills))


def _marked(n, first):
    """n float64 values: 1.0 where `first` (a boolean mask) is set, TINY elsewhere (sums that reveal their order)."""
    return np.where(first, 1.0, TINY)


def _counted(n):
    """n float64 values k / 8, k = 1 .. 13: every partial sum is exact, so a segment's sum counts its items."""
    return (np.arange(n) % 13 + 1) / 8.0


def _ints(rng, n):
    return rng.integers(1 << 61, 1 << 62, n, dtype=np.int64) * rng.choice([-1, 1], n)


def vv_fixtures():
    rng = np.random.default_rng(9200)
    fx = []
    # Go's ranges at nrows = 4w + i: rows at every range edge contribute; ranks holding {0,1,2,3}, {0,3}, {1}, {3}
    for i in range(4):
        nrows = 20 + i
        w = nrows // 4
        src = np.arange(1, nrows + 1, dtype=np.uint64) * 10
        dest = np.array([100, 200, 300, 400], np.uint64)
        rows = [[100] for _ in range(nrows)]
        rows[0], rows[nrows - 1] = [100, 200], [200, 100]
        for r in range(w, 2 * w):
            rows[r] = [300, 100]
        rows[3 * w] = [400, 100]
        vals = _marked(nrows, np.arange(nrows) == 0 if i == 0 else np.arange(nrows) % w == 0)
        ev = {f"vv: nrows = 4w + {i}, contributing rows at every range edge"}
        kills = {"range width rounded up"} if i else {"ranges combined descending", "fold from the end"}
        if i == 0:
            ev |= {"vv: a rank holding ranges {0,1,2,3}", "vv: a rank holding ranges {0,3}",
                   "vv: a rank holding ranges {1}", "vv: a rank holding ranges {3}", "vv: out_cap one short"}
        calls = VV_DEFAULT + ((VvCall("host", None, 3), VvCall("dev", None, 3)) if i == 0 else ())
        fx.append(_vv(f"nrows = {nrows}: rows at Go's range edges", src, (vals, _ints(rng, nrows)),
                      [_lv(src, rows, dest)], ev, kills, calls))
    # nrows < 4: one range; width 8 with the all-ones key (rank 63, range 3)
    src = np.array([5, 6, 7], np.uint64)
    d64 = np.arange(64, dtype=np.uint64) + 1000
    fx.append(_vv("nrows = 3, the all-ones key", src, (np.array([1.0, TINY, TINY]), np.array([3, -4, 5], np.int64)),
                  [_lv(src, [[1063, 1000], [1063], [1063, 1001]], d64)],
                  {"vv: nrows < 4", "sort: key width 8k with the all-ones key", "vv: P = 1"}, {"fold from the end"}))
    # float segments of 1, 2, 8, 9, 16 and 17 items (range 0 of nrows = 68)
    nrows = 68
    src = np.arange(1, nrows + 1, dtype=np.uint64)
    lens = (1, 2, 8, 9, 16, 17)
    dest = np.arange(len(lens) + 1, dtype=np.uint64) + 500
    rows = [[int(dest[k]) for k, L in enumerate(lens) if r < L] or [int(dest[-1])] for r in range(nrows)]
    # 1.0 after three TINY values (row 3), and a companion map whose sums count the items
    fx.append(_vv("float segments of 1 to 17 items", src, (_marked(nrows, np.arange(nrows) == 3), _counted(nrows)),
                  [_lv(src, rows, dest)], {f"vv: a float segment of {L} items" for L in lens},
                  {"fold from the end", "fold without its tail"}))
    # a float segment over tiles: 6 000 rows, three dests interleaved, 1.0 at the middle row of every segment (a
    # reorder that moves an item across it changes the sum), and a companion map whose sums count the items
    nrows = 6000
    src = np.arange(1, nrows + 1, dtype=np.uint64) * 2
    dest = np.array([7, 8, 9], np.uint64)
    rr = np.arange(nrows)
    first = np.zeros(nrows, bool)
    for q in range(4):
        for d in range(3):
            seg = np.nonzero((rr // 1500 == q) & (rr % 3 == d))[0]
            first[seg[seg.size // 2]] = True
    fx.append(_vv("float segments over tiles", src, (_marked(nrows, first), _counted(nrows)),
                  [_lv(src, [[int(dest[r % 3])] for r in rr], dest)],
                  {"vv: a float segment spanning tiles"},
                  {"ranks reversed in a warp", "rounds reversed in a tile", "tile-major hist", "fold from the end",
                   "fold without its tail"}))
    # int segments at warp and CTA edges: sorted, 32 one-item segments, then 64 items (two whole warps), then 204 over
    # item 255 | 256; the rest in ranges 1-3
    nrows = 1200
    src = np.arange(1, nrows + 1, dtype=np.uint64)
    dest = np.arange(40, dtype=np.uint64) + 3000
    tgt = np.where(rr[:nrows] < 32, rr[:nrows], np.where(rr[:nrows] < 96, 32, np.where(rr[:nrows] < 300, 33,
                                                                                         34 + rr[:nrows] % 6)))
    fx.append(_vv("int segments at warp and CTA edges", src,
                  (np.full(nrows, 3 << 61, np.int64) * np.where(rr[:nrows] % 2, 1, -1) + rr[:nrows],),
                  [_lv(src, [[int(dest[t])] for t in tgt], dest)],
                  {"int: a segment crossing lane 31 to 0", "int: a segment crossing a CTA edge",
                   "int: a whole warp in one segment", "int: 32 one-item segments in a warp",
                   "int: a wrapping segment sum"}, {"scan without the segment test"}))
    # a sparse map: 16 384 values, 40 contributing; tiles from v_cap: 8 (a hist scan of EN_TILE), 9 with v_cap + 1
    nrows = 4096
    src = np.arange(1, nrows + 1, dtype=np.uint64) * 3
    dest = np.arange(500, dtype=np.uint64) * 7 + 1
    rows = [np.sort(rng.choice(dest, 4, replace=False)) for _ in range(nrows)]
    keys = src[::103][:10]
    fx.append(_vv("a sparse map over 8 and 9 tiles", keys, (_marked(10, np.arange(10) < 2), _ints(rng, 10)),
                  [_lv(src, rows, dest)],
                  {"vv: a sparse map, tiles sized by v_cap", "sort: hist scan of exactly EN_TILE entries (8 tiles)",
                   "sort: hist scan of one tile more, two CTAs", "vv: device v_cap past v_off[nrows]"},
                  calls=VV_DEFAULT + (VvCall("dev", (4 * nrows + 1,), None),)))
    fx.append(_vv("a map reaching no row", [1, 2], (np.array([1.0, 2.0]),), [_lv(src, rows, dest)],
                  {"vv: no contributing value", "sort: n = 0 over tiles > 0"}))
    # three levels of 1, 4 and 2 passes: the maps ping-pong, each level on its own tickets
    s1 = np.arange(1, 41, dtype=np.uint64)
    d1 = np.arange(60, dtype=np.uint64) * 2 + 100
    big = (1 << 22) + 1
    d2 = np.arange(big, dtype=np.uint64) * 3 + 1000
    d3 = np.arange(1000, dtype=np.uint64) + (1 << 40)
    L1 = _lv(s1, [d1[rng.choice(60, 3, replace=False)] for _ in range(40)], d1)
    L2 = _lv(d1, [np.r_[d2[rng.integers(0, big - 1, 2)], d2[-1:]] for _ in range(60)], d2)
    used2 = np.unique(L2.v)
    used2 = used2[:used2.size // 4 * 4]   # keep the range-edge events to their own fixtures
    L3 = _lv(used2, [d3[rng.choice(1000, 5, replace=False)] for _ in range(used2.size)], d3)
    fx.append(_vv("levels of 1, 4 and 2 passes", s1, (_marked(40, np.arange(40) % 7 == 0),),
                  [L1, L2, L3], {"vv: levels of three different pass counts", "vv: P = 4", "vv: P = 2",
                                 "sort: key width 8k + 1, the last pass sorts one bit"}))
    d3b = np.arange((1 << 14) + 1, dtype=np.uint64) * 5 + 9
    src = np.arange(1, 301, dtype=np.uint64)
    fx.append(_vv("P = 3: ndest 2^14 + 1", src, (_marked(300, np.arange(300) % 50 == 0),),
                  [_lv(src, [d3b[[int(rng.integers(0, 1 << 14)), 1 << 14]] for _ in range(300)], d3b)],
                  {"vv: P = 3"}, {"ranks reversed in a warp"}))
    return fx


LA_DEFAULT = (LaCall("host", None, None), LaCall("dev", None, None))


def _la(name, keys, vals, src, rows, events, kills=(), calls=LA_DEFAULT, fns=tuple(FNS)):
    v, v_off = csr(rows)
    return LaFix(name, _u(keys), tuple(vals), _u(src), v, v_off, fns, tuple(calls), set(events), set(kills))


def la_fixtures():
    rng = np.random.default_rng(9300)
    fx = []
    # rows of 0 to 65 values, every value in the map; each row's first value 1.0, the rest TINY
    lens = (0, 1, 31, 32, 33, 63, 64, 65, 5, 40, 2, 96, 3, 7, 70)       # 15 rows: nrows = 8k - 1
    rows, vals, u = [], [], 1
    for L in lens:
        rows.append(np.arange(u, u + L, dtype=np.uint64))
        vals += [1.0] + [TINY] * (L - 1) if L else []
        u += L
    keys = np.arange(1, u, dtype=np.uint64)
    fx.append(_la("rows of 0 to 65 values", keys, (np.array(vals), _ints(rng, keys.size)),
                  np.arange(len(lens), dtype=np.uint64) * 4 + 1, rows,
                  {f"la: a row of {n} values" for n in (0, 1, 31, 32, 33, 63, 64, 65)} | {"la: nrows = 8k - 1"},
                  {"la lanes high to low"}))
    # present masks of lane 0, lane 31 and alternating lanes; NaN first and later; 17 rows: nrows = 8k + 1
    nrows = 17
    rows = [np.arange(100 * r + 1, 100 * r + 1 + 64, dtype=np.uint64) for r in range(nrows)]
    present = []
    for r in range(nrows):
        m = np.zeros(64, bool)
        if r == 0:
            m[0] = m[32] = True
        elif r == 1:
            m[31] = m[63] = True
        elif r == 2:
            m[::2] = True
        else:
            m[rng.choice(64, int(rng.integers(1, 64)), replace=False)] = True
        present.append(rows[r][m])
    keys = np.concatenate(present)
    fv = rng.normal(0, 10, keys.size)
    fv[0], fv[2] = np.nan, np.nan          # row 0: NaN first (lane 0 of round 0)
    off = np.cumsum([0] + [p.size for p in present])
    fv[off[3] + 1] = np.nan                # row 3: NaN after the first
    fv[off[2]:off[3]] = np.where(np.arange(off[3] - off[2]) == 0, 1.0, TINY)
    fx.append(_la("present masks and NaNs", keys, (fv, _ints(rng, keys.size)),
                  np.arange(nrows, dtype=np.uint64) + 7, rows,
                  {"la: only lane 0 present", "la: only lane 31 present", "la: alternating lanes present",
                   "la: NaN first (min / max)", "la: NaN after the first (min / max)", "la: nrows = 8k + 1",
                   "la: out_cap one short"}, {"la lanes high to low"},
                  LA_DEFAULT + (LaCall("host", None, 16), LaCall("dev", None, 16), LaCall("dev", 17 * 64 + 50, None))))
    return fx


def all_fixtures():
    return gb_fixtures() + vv_fixtures() + la_fixtures()


def outcomes(f, mut=frozenset()):
    """(per call and value array and function: the model's outcome), the events the fixture reaches."""
    ev: set = set()
    outs = []
    for c in f.calls:
        if isinstance(f, GbFix):
            outs.append(groupby(f, c, mut, ev))
        elif isinstance(f, VvFix):
            outs.append([propagate(f, x.view(np.uint64), x.dtype == np.float64, c, mut, ev) for x in f.vals])
        else:
            outs.append([[level_agg(f, x.view(np.uint64), x.dtype == np.float64, fn, c, mut, ev) for fn in f.fns]
                         for x in f.vals])
    return outs, ev
