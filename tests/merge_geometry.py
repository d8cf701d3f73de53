"""Host model of MergeSorted (dgx_api.cu merge_runs_impl and the multiway pipeline of merge_multi.cuh /
merge_tile32.cuh), and seeded fixtures aimed at its geometry edges.

The model restates, step for step and with exact integer arithmetic:
  - the path and launch plan: pairwise tree / single-pass multiway / groups of <= MM_K runs merged again;
  - the multiway geometry: sample counts and positions, the distinct splitters, every run's bounds, every tile's
    interior / exact decision, lo, hi, engine (32-bit keys or 64-bit values) and largest key;
  - the rounds of the tile engines (t32_tile, mm_levels_tile): per round every run's take, the padded size, whether the
    tile fits, the bound, how many merged values are final, how far every run advances, and whether the value written
    last has more copies waiting (the carry a round hands to the next).
The constants are read from the CUDA sources, so a tuning change moves the model with it, and a renamed or moved
constant fails here loudly instead of leaving the fixtures aimed at stale boundaries.

Fixture builders return runs plus the geometry they are meant to reach; tests/test_merge_geometry.py checks on the
CPU that each one still reaches it, tests/test_gpu_merge_edges.py runs them through the kernels.
"""
from __future__ import annotations

import os
import re
from collections import namedtuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")
U64_MAX = (1 << 64) - 1
_SOURCES = ("merge_multi.cuh", "merge_tile32.cuh", "merge_kernel.cuh", "dgx_api.cu")
_NAMES = ("MM_K", "MM_NT", "MM_C", "MM_VT", "MM_STRIDE", "T_NT", "T_VT", "T_C", "T_INF", "M_NT", "M_VT", "M_T",
          "g_merge_multi_min")


def read_constants() -> dict:
    """`constexpr <type> NAME = <expr>;` of the merge sources, evaluated (C casts and integer suffixes stripped)."""
    exprs = {}
    for fn in _SOURCES:
        with open(os.path.join(CSRC, fn)) as f:
            for name, expr in re.findall(r"\bconstexpr\s+[\w:]+\s+(\w+)\s*=\s*([^;]+);", f.read()):
                exprs.setdefault(name, expr)
    vals: dict = {}

    def ev(name):
        if name not in vals:
            if name not in exprs:
                raise KeyError(f"constexpr {name} not found in {', '.join(_SOURCES)}: the merge model needs it")
            e = re.sub(r"\((?:u64|u32|int|size_t)\)", "", exprs[name])
            e = re.sub(r"\b(?:size_t|u64|u32|int)\s*\(", "(", e)
            e = re.sub(r"\b(0[xX][0-9a-fA-F]+|\d+)[uUlL]*\b", r"\1", e).replace("/", "//")
            for ref in re.findall(r"\b[A-Za-z_]\w*\b", e):
                if not re.fullmatch(r"0[xX][0-9a-fA-F]+", ref):
                    ev(ref)
            vals[name] = int(eval(e, {"__builtins__": {}}, dict(vals)))  # noqa: S307 -- our own sources
        return vals[name]

    return {n: ev(n) for n in _NAMES}


K = read_constants()
MM_K, MM_C, MM_VT, MM_STRIDE = K["MM_K"], K["MM_C"], K["MM_VT"], K["MM_STRIDE"]
T_C, T_VT, T_INF, M_T = K["T_C"], K["T_VT"], K["T_INF"], K["M_T"]
MERGE_MULTI_MIN = K["g_merge_multi_min"]


# ---- path and launch plan (merge_runs_impl) ----------------------------------------------------------------------

def tree_launches(k):
    """merge_tree_impl: one merge_kernel launch per level; a single run still takes one (in-run de-duplication)."""
    levels = 0
    while k > 1:
        k, levels = (k + 1) // 2, levels + 1
    return max(levels, 1)


def ntarget_of(total):
    """merge_multi_impl: about one sample per 512 values, at most 2^24 samples."""
    return min(max(total // 512, 1), 1 << 24)


def sample_counts(ub):
    """Samples per run: floor(ub_j * ntarget / total) (soff of merge_multi_impl), from the runs' upper bounds."""
    total = sum(int(u) for u in ub)
    nt = ntarget_of(total)
    return [int(u) * nt // total for u in ub]


Plan = namedtuple("Plan", "path launches parts")  # parts: the group plans then the plan of the merged groups


def merge_plan(lens) -> Plan:
    """Plan of merge_runs_impl for non-empty runs with these lengths (upper bounds at a grouped level)."""
    lens = [int(n) for n in lens]
    k, total = len(lens), sum(lens)
    if 3 <= k <= MM_K and total >= MERGE_MULTI_MIN:
        # msample, the tree over the non-empty sample runs, mplan2, mmerge3, mscan, mcompact
        return Plan("multiway", 5 + tree_launches(sum(1 for s in sample_counts(lens) if s)), ())
    ngroups = -(-k // MM_K)
    if k <= MM_K or total // ngroups < 4 * MERGE_MULTI_MIN:
        return Plan("tree", tree_launches(k), ())
    gsz = -(-k // ngroups)
    parts = [merge_plan(lens[b:b + gsz]) for b in range(0, k, gsz)]
    top = merge_plan([sum(lens[b:b + gsz]) for b in range(0, k, gsz)])
    return Plan("grouped", sum(p.launches for p in parts) + top.launches, tuple(parts) + (top,))


def describe(plan: Plan) -> str:
    """'grouped[multiway x64, tree x1 -> grouped[multiway x2 -> tree]]'"""
    if plan.path != "grouped":
        return plan.path
    counts: dict = {}
    for p in plan.parts[:-1]:
        d = describe(p)
        counts[d] = counts.get(d, 0) + 1
    return "grouped[" + ", ".join(f"{d} x{n}" for d, n in counts.items()) + " -> " + describe(plan.parts[-1]) + "]"


# ---- multiway geometry ----------------------------------------------------------------------------------------------

Round = namedtuple("Round", "takes need np fits bound nsafe adv carry_in carry_out")
Tile = namedtuple("Tile", "b interior exact lo hi wide start end total max_key rounds out")
Geometry = namedtuple("Geometry", "total ntarget soff samples splitters nsplit ns S bounds tiles")


def sample_positions(n, s):
    """msample_kernel: sample r of a run of n values with s samples sits at (r + 1) * n / (s + 1)."""
    return [(r + 1) * n // (s + 1) for r in range(s)]


def _u64(x):
    return np.asarray(x, dtype=np.uint64)


def simulate_rounds(slices, wide):
    """t32_tile (wide=False) / mm_levels_tile (wide=True) on one tile's slices: the rounds and the distinct output."""
    C, VT = (MM_C, MM_VT) if wide else (T_C, T_VT)
    k = len(slices)
    cur = [0] * k
    end = [int(s.size) for s in slices]
    have_last, last = False, 0
    rounds, out = [], []
    while True:
        rem = [end[j] - cur[j] for j in range(k)]
        total_rem = sum(rem)
        if total_rem == 0:
            break
        need = sum(-(-r // VT) * VT for r in rem)
        fits = need <= C
        takes, bnds = [], []
        for j in range(k):
            if fits:
                t = rem[j]
            elif rem[j] > 0:
                t = min(max(rem[j] * (C - VT * MM_K) // total_rem, 1), rem[j])
                if t < rem[j]:
                    bnds.append(int(slices[j][cur[j] + t - 1]))
            else:
                t = 0
            takes.append(t)
        bound = min(bnds) if bnds else U64_MAX
        chunk = np.sort(np.concatenate([slices[j][cur[j]:cur[j] + takes[j]] for j in range(k)]))
        nsafe = chunk.size if fits else int(np.searchsorted(chunk, np.uint64(bound), side="right"))
        safe = chunk[:nsafe]
        carry_in = bool(have_last and nsafe > 0 and int(safe[0]) == last)
        if nsafe:
            keep = np.ones(nsafe, dtype=bool)
            keep[1:] = safe[1:] != safe[:-1]
            keep[0] = not carry_in
            out.append(safe[keep])
            have_last, last = True, int(safe[-1])
        adv = []
        for j in range(k):
            a = takes[j] if fits else int(np.searchsorted(slices[j][cur[j]:cur[j] + takes[j]], np.uint64(bound), side="right"))
            adv.append(a)
            cur[j] += a
        carry_out = have_last and any(cur[j] < end[j] and int(slices[j][cur[j]]) == last for j in range(k))
        rounds.append(Round(takes, need, sum(-(-t // VT) * VT for t in takes), fits, bound, nsafe, adv, carry_in,
                            carry_out))
        if fits:
            break
    return rounds, (np.concatenate(out) if out else np.zeros(0, np.uint64))


def multiway_geometry(runs, ub=None, rounds=True) -> Geometry:
    """The geometry merge_multi_impl gives these runs (ub: the lengths the host plans with; actual lengths otherwise)."""
    runs = [_u64(r) for r in runs]
    ub = [int(r.size) for r in runs] if ub is None else [int(u) for u in ub]
    k, total = len(runs), sum(ub)
    s = sample_counts(ub)
    soff = np.concatenate([[0], np.cumsum(s)]).astype(np.int64)
    samples = []
    for r, sj in zip(runs, s):
        n = int(r.size)
        samples.append(r[sample_positions(n, sj)] if n else np.full(sj, U64_MAX, np.uint64))
    allsamp = np.concatenate(samples) if samples else np.zeros(0, np.uint64)
    splitters = np.unique(allsamp)  # the merge tree over the sample runs de-duplicates
    nsplit = int(splitters.size)
    ns = nsplit // MM_STRIDE
    S = [None] + [int(splitters[b * MM_STRIDE - 1]) for b in range(1, ns + 1)]
    bounds = []
    for r in runs:
        n = int(r.size)
        bj = [0] + [int(np.searchsorted(r, np.uint64(S[b]), side="left")) if n else 0 for b in range(1, ns + 1)] + [n]
        bounds.append(bj)
    tiles = []
    for b in range(ns + 1):
        interior = 1 <= b < ns
        start = [bounds[j][b] for j in range(k)]
        end = [bounds[j][b + 1] for j in range(k)]
        lo = hi = 0
        exact = not interior
        if interior:
            lo, hi = S[b], S[b + 1] - 1
            exact = hi - lo >= T_INF
        slices = [runs[j][start[j]:end[j]] for j in range(k)]
        tot = sum(e - c for c, e in zip(start, end))
        if exact:
            lo = min((int(x[0]) for x in slices if x.size), default=U64_MAX)
            hi = max((int(x[-1]) for x in slices if x.size), default=0)
        wide = (hi - lo) % (1 << 64) >= T_INF
        vmax = max((int(x[-1]) for x in slices if x.size), default=None)
        max_key = None if (vmax is None or wide) else vmax - lo
        rs, out = simulate_rounds(slices, wide) if (rounds and tot) else ([], np.zeros(0, np.uint64))
        tiles.append(Tile(b, interior, exact, lo, hi, wide, start, end, tot, max_key, rs, out))
    return Geometry(total, ntarget_of(total), soff, samples, splitters, nsplit, ns, S, bounds, tiles)


def model_output(geo: Geometry):
    return np.concatenate([t.out for t in geo.tiles]) if geo.tiles else np.zeros(0, np.uint64)


# ---- pairwise tree: where a merge_kernel tile's predecessor comes from ----------------------------------------------

def tree_tile_preds(a, b):
    """First level of the tree on runs (a, b): for every merge-path tile boundary d0 = t * M_T inside the merged pair,
    'B' when the value at d0 repeats the one at d0 - 1, that one comes from b and a holds no copy of it (only
    b[bi0 - 1] tells the tile its first value is a repeat), 'A' when only a's predecessor does, '' otherwise."""
    a, b = _u64(a), _u64(b)
    # merged order with ties to a: value-major, a before b
    vals = np.concatenate([a, b])
    side = np.concatenate([np.zeros(a.size, np.int8), np.ones(b.size, np.int8)])
    order = np.lexsort((side, vals))
    vals, side = vals[order], side[order]
    kinds = []
    for d0 in range(M_T, vals.size, M_T):
        v = vals[d0 - 1]
        if vals[d0] != v:
            kinds.append("")
        elif side[d0 - 1] == 1:
            # every copy in a precedes the copies in b; a's predecessor is a copy only when a holds v
            ai0 = int(np.sum(side[:d0] == 0))
            kinds.append("B" if ai0 == 0 or a[ai0 - 1] != v else "")
        else:
            kinds.append("A")
    return kinds


# ---- fixture builders -----------------------------------------------------------------------------------------------

Fixture = namedtuple("Fixture", "name runs expect")


def _fill(rng, lo, hi, n):
    """n sorted values in [lo, hi] (0 <= lo <= hi <= 2^64 - 1)."""
    return np.sort(rng.integers(lo, hi, n, dtype=np.uint64, endpoint=True)) if n > 0 else np.zeros(0, np.uint64)


def targeted_tile(rng, counts, low, high, where, lo, top, next_split=None, dup=False, low_floor=None,
                  high_ceiling=None):
    """Runs whose tile `where` ('first' | 'interior' | 'last') holds exactly counts[j] values of run j, smallest lo,
    largest top; an interior or first tile ends at next_split, the value of the first sample above it.

    Sample positions depend only on the run lengths low[j] + counts[j] + high[j], so they are fixed first.  The samples
    below the tile get low_floor..lo-1 values, so many distinct ones that the tile starts at a boundary (10b - 1
    distinct values below it); the samples inside take MM_STRIDE levels lo = L0 < L1 < ... (MM_STRIDE - 1 for the
    first tile, at most MM_STRIDE for the last); the samples above start at next_split.  The values between samples
    are drawn between their neighbours (dup: repeats of the level before them), so each run's slice of the tile is
    exactly counts[j] long.  Returns (runs, b)."""
    k = len(counts)
    lens = [low[j] + counts[j] + high[j] for j in range(k)]
    s = sample_counts(lens)
    pos = [sample_positions(lens[j], s[j]) for j in range(k)]
    vals = [[None] * lens[j] for j in range(k)]  # Python ints, np.uint64 at the end
    low_slots = sorted((r, j) for j in range(k) for r, q in enumerate(pos[j]) if q < low[j])
    tile_slots = sorted(((q - low[j]) / counts[j], j, q) for j in range(k) for q in pos[j]
                        if low[j] <= q < low[j] + counts[j])
    high_slots = sorted((r, j) for j in range(k) for r, q in enumerate(pos[j]) if q >= low[j] + counts[j])
    if where == "first":
        assert not low_slots and all(x == 0 for x in low), "the first tile has nothing below it"
        b, nl = 0, MM_STRIDE - 1
    else:
        assert len(low_slots) >= MM_STRIDE - 1, "too few samples below the tile"
        dlow = (len(low_slots) + 1) // MM_STRIDE * MM_STRIDE - 1
        b, nl = (dlow + 1) // MM_STRIDE, MM_STRIDE
        if where == "last":
            assert not high_slots and all(x == 0 for x in high)
            nl = min(MM_STRIDE, len(tile_slots))
        low_floor = max(0, lo - (1 << 30)) if low_floor is None else low_floor
        extra = len(low_slots) - dlow
        step = (lo - 1 - low_floor) // (dlow + 1)
        assert step >= 1
        for i, (r, j) in enumerate(low_slots):
            vals[j][pos[j][r]] = low_floor + step * (1 + max(0, i - extra))
    if where != "last":
        assert high_slots and next_split is not None and next_split > top
        high_ceiling = min(U64_MAX, next_split + (1 << 30)) if high_ceiling is None else high_ceiling
        hstep = max(1, (high_ceiling - next_split) // (len(high_slots) + 1))
        for i, (r, j) in enumerate(high_slots):
            vals[j][pos[j][r]] = next_split + hstep * i
    assert len(tile_slots) >= nl, f"{len(tile_slots)} samples inside the tile, {nl} levels wanted"
    lstep = max(1, (top - lo) // (2 * nl))
    levels = [lo + i * lstep for i in range(nl)]
    assert levels[-1] <= top
    for i, (_, j, q) in enumerate(tile_slots):
        vals[j][q] = levels[i * nl // len(tile_slots)]
    runs = []
    for j in range(k):
        v = vals[j]
        t0, t1 = low[j], low[j] + counts[j]
        # the gaps between fixed values: each region filled between its neighbours, clamped to its region's range
        fixed = [q for q in range(lens[j]) if v[q] is not None]
        edges = [-1] + fixed + [lens[j]]
        for e0, e1 in zip(edges[:-1], edges[1:]):
            if e1 - e0 <= 1:
                continue
            for r0, r1, rlo, rhi in ((0, t0, low_floor if where != "first" else 0, lo - 1),
                                     (t0, t1, lo, top),
                                     (t1, lens[j], next_split if where != "last" else 0, high_ceiling or 0)):
                a, z = max(e0 + 1, r0), min(e1, r1)
                if a >= z:
                    continue
                left = v[e0] if e0 >= r0 and e0 >= 0 else rlo
                right = v[e1] if e1 < r1 else rhi
                if dup and r0 == t0:
                    fill = np.full(z - a, left, np.uint64)
                else:
                    fill = _fill(rng, left, right, z - a)
                for q, x in zip(range(a, z), fill):
                    v[q] = int(x)
        runs.append(v)
    # the tile's extremes: lo (already a level-0 sample, or forced here) and top at a non-sample position
    spos = [set(p) for p in pos]
    j = max((j for j in range(k) if counts[j] and (low[j] + counts[j] - 1) not in spos[j]),
            key=lambda j: counts[j], default=None)
    assert j is not None, "every run's last tile value is a sample"
    runs[j][low[j] + counts[j] - 1] = top
    if where == "first":
        j0 = next(j for j in range(k) if counts[j])
        runs[j0][0] = lo
    out = [np.array(r, dtype=np.uint64) for r in runs]
    for r in out:
        assert r.size < 2 or bool(np.all(r[1:] >= r[:-1])), "builder produced an unsorted run"
    return out, b


def _spread(total, k):
    return [total // k + (1 if j < total % k else 0) for j in range(k)]


def _around(k, tile_counts, where, rest=300_000):
    """low / high region lengths for a tile of these counts inside ~rest values over k runs."""
    side = _spread(max(rest - sum(tile_counts), 0), k)
    if where == "first":
        return [0] * k, side
    if where == "last":
        return side, [0] * k
    return [x // 2 for x in side], [x - x // 2 for x in side]


def tile_fixture(name, seed, counts, where, lo, top, next_split=None, dup=False, **expect):
    rng = np.random.default_rng(seed)
    low, high = _around(len(counts), counts, where)
    runs, b = targeted_tile(rng, counts, low, high, where, lo, top, next_split, dup)
    return Fixture(name, runs, dict(expect, tile=b, counts=list(counts), lo=lo, top=top, where=where))


G32 = 1 << 32


def span_fixtures():
    """Items 1-3: tile spans at the edge between the 32-bit and the 64-bit engine, decided both ways."""
    fx = []
    base = (5 << 32) + 12_345
    c = [2_600, 2_100, 2_300]
    # 1. interior, narrow by its splitter gap (2^32 - 1), a value at S(b+1) - 1: key 0xFFFFFFFE
    fx.append(tile_fixture("interior gap 2^32-1, key 0xFFFFFFFE", 101, c, "interior", base, base + G32 - 2,
                           base + G32 - 1, exact=False, wide=False, max_key=T_INF - 1))
    # 2. interior, splitter gap >= 2^32: decided by the real min / max
    for i, span in enumerate((G32 - 2, G32 - 1, G32)):
        fx.append(tile_fixture(f"interior exact span {span:#x}", 110 + i, c, "interior", base, base + span,
                               base + max(G32, span + 1), exact=True, wide=span >= T_INF,
                               max_key=None if span >= T_INF else span))
    # 3. first tile from 0, last tile to 2^64 - 1
    for i, span in enumerate((G32 - 2, G32 - 1, G32)):
        fx.append(tile_fixture(f"first tile 0..{span:#x}", 120 + i, c, "first", 0, span, span + 1 + (1 << 20),
                               exact=True, wide=span >= T_INF, max_key=None if span >= T_INF else span))
        fx.append(tile_fixture(f"last tile ..2^64-1 span {span:#x}", 130 + i, c, "last", U64_MAX - span, U64_MAX,
                               exact=True, wide=span >= T_INF, max_key=None if span >= T_INF else span))
    return fx


def _padded_counts(VT, C, extra_slot):
    """Three runs whose slots pad to exactly C (extra_slot False, raw total C) or to C + VT with a raw total below C."""
    if not extra_slot:
        q = C // VT
        return [VT * (q // 4)] * 3 + [VT * (q - 3 * (q // 4))]
    q = (C + VT) // VT - 3
    return [VT * (q // 3) + 1, VT * (q // 3) + 1, VT * (q - 2 * (q // 3)) + 1]


def round_fixtures():
    """Items 4-5: a tile that exactly fills one round, one that overflows it by one padded slot, and one whose rounds
    end on a value that has copies left in partly loaded runs -- in each engine."""
    fx = []
    lo32 = (3 << 32) + 777
    for wide, C, VT in ((False, T_C, T_VT), (True, MM_C, MM_VT)):
        eng = "64-bit" if wide else "32-bit"
        # narrow: an interior tile; wide: the last tile, 2^33 wide (a 4096-value tile holds too few samples for ten
        # distinct interior levels)
        where, top, nxt = ("last", U64_MAX - 12_345, None) if wide else ("interior", lo32 + (1 << 24), lo32 + (1 << 25))
        lo = top - (1 << 33) if wide else lo32
        c = _padded_counts(VT, C, False)
        fx.append(tile_fixture(f"{eng} padded {C}: one round", 200 + wide, c, where, lo, top, nxt, wide=wide,
                               rounds_min=1, rounds_max=1, need=C, raw=sum(c)))
        c = _padded_counts(VT, C, True)
        assert sum(c) <= C and sum(-(-x // VT) * VT for x in c) == C + VT
        fx.append(tile_fixture(f"{eng} padded {C + VT}: rounds", 210 + wide, c, where, lo, top, nxt, wide=wide,
                               rounds_min=2, need=C + VT, raw=sum(c)))
        c = [2_600] * 6
        fx.append(tile_fixture(f"{eng} bound value carried across rounds", 220 + wide, c, where, lo, top, nxt,
                               dup=True, wide=wide, rounds_min=3, carry=True))
    return fx


def one_value_fixtures():
    """Item 6: one distinct value over 64 runs of 2^18 values in total: one tile, dozens of rounds."""
    n = MERGE_MULTI_MIN // MM_K
    return [Fixture(f"one value {v:#x}", [np.full(n, v, np.uint64)] * MM_K, dict(one_value=v))
            for v in (0, G32 - 1, U64_MAX)]


def zero_sample_fixture(seed=300):
    """Item 7: runs too short for a sample next to large runs; one inside one tile, one below the first splitter, one
    above the last, one across many tiles."""
    import gen

    rng = np.random.default_rng(seed)
    big = [gen.zipf_gaps(rng, n, start=1 << 20) for n in (120_000, 90_000, 70_000)]
    small_lens = [1, 7, 300, 511, 64]
    lens = [b.size for b in big] + small_lens
    s = sample_counts(lens)
    assert s[3:] == [0] * len(small_lens), s
    # splitters come from the big runs' samples only: the small runs' values can be chosen after them
    geo = multiway_geometry(big + [np.zeros(n, np.uint64) for n in small_lens], ub=lens, rounds=False)
    S, ns = geo.S, geo.ns
    mid = ns // 2
    inside = _fill(rng, S[mid], S[mid + 1] - 1, small_lens[0] + 0)
    below = _fill(rng, 0, S[1] - 1, small_lens[1])
    above = _fill(rng, S[ns], S[ns] + (1 << 22), small_lens[2])
    across = np.sort(rng.choice(np.concatenate(big), small_lens[3], replace=False))
    inside2 = _fill(rng, S[mid + 2], S[mid + 3] - 1, small_lens[4])
    return Fixture("runs without samples", big + [inside, below, above, across, inside2],
                   dict(zero_samples=len(small_lens), inside_tiles=(mid, mid + 2)))


def zipf_slices(rng, lens, master_len=None):
    """Lists cut from one Zipf-gap master at random offsets: cheap at any k, overlapping, so values repeat across lists."""
    import gen

    m = gen.zipf_gaps(rng, master_len or max(4 * max(lens), 1 << 20))
    offs = rng.integers(0, m.size - max(lens) + 1, len(lens))
    return [m[o:o + n] for o, n in zip(offs, lens)]


THRESHOLDS = {  # name -> (k, total, path)
    "k=3 below the multiway minimum": (3, MERGE_MULTI_MIN - 1, "tree"),
    "k=3 at the multiway minimum": (3, MERGE_MULTI_MIN, "multiway"),
    "k=64 below the multiway minimum": (64, MERGE_MULTI_MIN - 1, "tree"),
    "k=64 at the multiway minimum": (64, MERGE_MULTI_MIN, "multiway"),
    "k=65 below the grouping minimum": (65, 2 * 4 * MERGE_MULTI_MIN - 1, "tree"),
    "k=65 at the grouping minimum": (65, 2 * 4 * MERGE_MULTI_MIN, "grouped"),
    "k=4096 grouped then multiway": (4096, 64 * 4 * MERGE_MULTI_MIN, "grouped"),
    "k=4097 grouped twice": (4097, 65 * 4 * MERGE_MULTI_MIN, "grouped"),
}
THRESHOLD_PLANS = {  # what the levels below the top one are expected to be
    "k=4096 grouped then multiway": "grouped[multiway x64 -> multiway]",
    "k=4097 grouped twice": "grouped[multiway x64, tree x1 -> grouped[multiway x2 -> tree]]",
}


def threshold_fixture(name, seed=400):
    k, total, _ = THRESHOLDS[name]
    rng = np.random.default_rng(seed)
    return Fixture(name, zipf_slices(rng, _spread(total, k), master_len=1 << 22), dict(threshold=name))


def tree_pair(rng, n, every=M_T, how=("B", "A", "split"), lo_edge=True):
    """Two runs whose merge (ties to A) has a run of equal values across every `every`-th merged position, in turn all
    from B (B's predecessor alone says the tile starts with a repeat), all from A, and split between the end of A's
    copies and the start of B's; 0 first and 2^64 - 1 last in both when lo_edge."""
    import gen

    v = gen.zipf_gaps(rng, n, start=1)
    side = rng.integers(0, 2, n).astype(np.int8)
    for t, d0 in enumerate(range(every, n - every // 2, every)):
        a, z = d0 - int(rng.integers(2, 40)), d0 + int(rng.integers(1, 40))
        v[a:z] = v[a]
        kind = how[t % len(how)]
        side[a:z] = 1 if kind == "B" else 0
        if kind == "split":
            side[d0 - 1:z] = 1  # A's copies end just before d0 - 1, B's run across it
    if lo_edge:
        v[:5] = 0
        v[-5:] = U64_MAX
        side[:5] = [0, 0, 1, 1, 1]
        side[-5:] = [0, 0, 0, 1, 1]
    return v[side == 0], v[side == 1]


def tree_fixtures(seed=500):
    """Item 9: the pairwise tree at sizes and edges its random tests do not reach."""
    import gen

    rng = np.random.default_rng(seed)
    fx = []
    a, b = tree_pair(rng, 3_000_000)
    fx.append(Fixture("tree k=2 runs across every tile edge", [a, b], dict(tree_pairs=[(a, b)])))
    one = gen.zipf_gaps(rng, 2_500_000)
    for d0 in range(M_T, one.size - 100, M_T):
        one[d0 - 3:d0 + 2] = one[d0 - 3]
    one[:3], one[-3:] = 0, U64_MAX
    fx.append(Fixture("tree k=1 repeats across every tile edge", [one], {}))
    fx.append(Fixture("tree one side empty", [np.zeros(0, np.uint64), a[:200_000], np.zeros(0, np.uint64)], {}))
    fx.append(Fixture("tree 0 and 2^64-1 only", [np.array([0, 0, U64_MAX], np.uint64), np.array([0, U64_MAX, U64_MAX],
                                                                                                np.uint64)], {}))
    for k in (3, 5, 9, 17, 33):
        runs = []
        for i in range((k + 1) // 2):
            x, y = tree_pair(rng, (MERGE_MULTI_MIN - 1) // k * 2 - 64, lo_edge=i == 0)
            runs += [x, y]
        runs = runs[:k]
        assert sum(r.size for r in runs) < MERGE_MULTI_MIN
        fx.append(Fixture(f"tree k={k}", runs, dict(tree_pairs=[(runs[i], runs[i + 1]) for i in range(0, k - 1, 2)])))
    return fx


def all_fixtures():
    return span_fixtures() + round_fixtures() + one_value_fixtures() + [zero_sample_fixture()]
