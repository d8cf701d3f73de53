"""Host model of the filter pipeline (dgx_api.cu filter_batch_impl and the kernels of filter_pipe.cuh), and seeded
fixtures aimed at its tile, staging and deferral edges.

The model restates, step for step and with exact integer arithmetic:
  - the batch plan: each intersection query's lists in stable length order (the driving list A first; u for
    Difference), kmax, the tile geometry (VA, tile size), slice_cap, grp, tiles per query, whether the batch is deep
    (sampled, with a deferred tail) and the launches it makes;
  - filter_sample_kernel: the 256 samples of A, their hits in lists 1..min(k - 2, 31), the depth counts and k_eff;
  - per tile: a0, na, prev, has_prev, the slice bounds r0 / r1 of every streamed filter list, the 16-byte head of A
    and of each slice, the staged words, their prefix sums, which lists fit and the leading run that is staged;
  - per consumer warp: rows, repeated values, the 32-bit fast-path predicate and, step by step, the branch the chain
    takes (fast: two rows x two lists, rows x one list, one row x 3 / 2 / 1 lists, the ladder fallback, an empty
    slice; 64-bit: staged lists row pairs, one row x up to three staged lists, a list searched in HBM), the windows
    lift32m picks, duplicate ranks (cand_rank), the survivors after each step and the re-packed row count;
  - filter_tail_kernel: the intermediate (mid / mid_off), every survivor's duplicate rank and the deferred lists.
The survivors are exact set arithmetic, so the model also produces each query's result, which tests compare with
the oracle.  What the kernels decide is named as *events*; fixtures name the events they must reach.

The constants are read from the CUDA sources and the slice_cap statement of filter_batch_impl is matched as text, so
a tuning change moves the model with it and a renamed constant or a rewritten statement fails here loudly instead
of leaving the fixtures aimed at stale boundaries.

tests/test_filter_geometry.py checks the fixtures on the CPU; tests/test_gpu_filter_edges.py runs them through the
kernels.
"""
from __future__ import annotations

import os
import re
from collections import namedtuple

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dgraph_b200", "csrc")
U64_MAX = (1 << 64) - 1
G32 = 1 << 32
_NAMES = ("P_CW", "P_MAXL", "P_SAMPLES", "P_DEFER_DIV", "P_SAMPLE_MIN_A", "P_SAMPLE_LISTS", "P_TAIL_NT")
OP_INTERSECT, OP_DIFFERENCE = 0, 1


def _src(fn):
    with open(os.path.join(CSRC, fn)) as f:
        return f.read()


def read_constants() -> dict:
    """The named constants of filter_pipe.cuh, the tile size of p_tile_size and the batch geometry of
    filter_batch_impl (VA choice, staged-list count, slice_cap formula, grp)."""
    pipe, api = _src("filter_pipe.cuh"), _src("dgx_api.cu")
    exprs = dict(re.findall(r"\bconstexpr\s+[\w:]+\s+(\w+)\s*=\s*([^;]+);", pipe))
    vals = {}
    for name in _NAMES:
        if name not in exprs:
            raise KeyError(f"constexpr {name} not found in filter_pipe.cuh: the filter model needs it")
        e = re.sub(r"\b(0[xX][0-9a-fA-F]+|\d+)[uUlL]*\b", r"\1", exprs[name]).strip()
        if not re.fullmatch(r"[0-9xXa-fA-F]+", e):
            raise ValueError(f"{name} = {exprs[name]}: not a literal")
        vals[name] = int(e, 0)
    m = re.search(r"constexpr int p_tile_size\(int va\) \{ return P_CW \* 32 \* va; \}", pipe)
    if not m:
        raise ValueError("p_tile_size(va) is no longer P_CW * 32 * va: restate the tile size in the filter model")
    m = re.search(r"const int pipe_va = kmax <= (\d+) \? (\d) : (\d);", api)
    if not m:
        raise ValueError("filter_batch_impl's tile-geometry choice (pipe_va) not found: restate it in the filter model")
    vals["VA_KMAX"], vals["VA_NARROW"], vals["VA_WIDE"] = (int(x) for x in m.groups())
    m = re.search(r"const size_t nl = std::min<size_t>\(std::max<size_t>\(kmax - 1, 1\), P_MAXL\);\s*"
                  r"const size_t TA = \(size_t\)tile_sz;.*?"
                  r"size_t cap = \(TA \+ TA / (\d+)\) \* nl \* \(kmax <= (\d+) \? (\d+) : 1\);\s*"
                  r"cap = std::min<size_t>\(std::max<size_t>\(cap, TA \+ TA / (\d+)\), (\d+)\) & ~size_t\(1\);", api, re.S)
    if not m:
        raise ValueError("filter_batch_impl's slice_cap statement changed: restate it in the filter model "
                         "(tests/filter_geometry.py) before aiming fixtures at it")
    div, kmax2, mult, div2, top = (int(x) for x in m.groups())
    if div != div2:
        raise ValueError("slice_cap: two different TA fractions")
    vals["CAP_DIV"], vals["CAP_KMAX"], vals["CAP_MULT"], vals["CAP_MAX"] = div, kmax2, mult, top
    m = re.search(r"PP\.grp = kmax >= (\d+) \? 1u : 2u;", api)
    if not m:
        raise ValueError("filter_batch_impl's grp choice not found")
    vals["GRP_KMAX"] = int(m.group(1))
    return vals


K = read_constants()
P_CW, P_MAXL, P_SAMPLES, P_DEFER_DIV = K["P_CW"], K["P_MAXL"], K["P_SAMPLES"], K["P_DEFER_DIV"]
P_SAMPLE_MIN_A, P_SAMPLE_LISTS, P_TAIL_NT = K["P_SAMPLE_MIN_A"], K["P_SAMPLE_LISTS"], K["P_TAIL_NT"]


def tile_size(va):
    return P_CW * 32 * va


def geometry(kmax):
    """(VA, tile size, slice_cap, grp) of a batch whose widest query has kmax lists (filter_batch_impl)."""
    va = K["VA_NARROW"] if kmax <= K["VA_KMAX"] else K["VA_WIDE"]
    ta = tile_size(va)
    nl = min(max(kmax - 1, 1), P_MAXL)
    cap = (ta + ta // K["CAP_DIV"]) * nl * (K["CAP_MULT"] if kmax <= K["CAP_KMAX"] else 1)
    cap = min(max(cap, ta + ta // K["CAP_DIV"]), K["CAP_MAX"]) & ~1
    grp = 1 if kmax >= K["GRP_KMAX"] else 2
    return va, ta, cap, grp


# ---- the batch ------------------------------------------------------------------------------------------------------

def _u64(x):
    return np.ascontiguousarray(np.asarray(x, dtype=np.uint64))


Query = namedtuple("Query", "k order lists offs lenA ntiles")
Plan = namedtuple("Plan", "op kmax va ta slice_cap grp deep launches queries npairs")


def plan_batch(queries, op=OP_INTERSECT, resident=False, offsets=None) -> Plan:
    """queries: per query its lists in caller order; offsets: per query the element offset of each list on the device
    (its parity is the 16-byte head), 0 when None."""
    kmax = max(1, max(len(q) for q in queries))
    va, ta, cap, grp = geometry(kmax)
    qs, sample_any, npairs = [], False, 0
    for qi, q in enumerate(queries):
        k = len(q)
        assert k >= 1 and (op == OP_INTERSECT or k == 2)
        order = list(range(k))
        if op == OP_INTERSECT:
            order.sort(key=lambda i: len(q[i]))  # list.sort is stable, as std::stable_sort
        offs = [0] * k if offsets is None else list(offsets[qi])
        lists = [_u64(q[i]) for i in order]
        lenA = int(lists[0].size)
        nt = max(1, -(-lenA // ta))
        qs.append(Query(k, order, lists, [offs[i] for i in order], lenA, nt))
        sample_any |= k >= 3 and lenA >= P_SAMPLE_MIN_A
        npairs += nt * (k - 1)
    deep = op == OP_INTERSECT and resident and sample_any
    launches = 1 + (1 if npairs else 0) + 1 + (2 if deep else 0)
    return Plan(op, kmax, va, ta, cap, grp, deep, launches, qs, npairs)


# ---- filter_sample_kernel -------------------------------------------------------------------------------------------

def sample_keff(q: Query, events=None):
    """k_eff of one query of a deep batch, and the alive counts after each split point."""
    k, A, lenA = q.k, q.lists[0], q.lenA
    nj = 0 if (k < 3 or lenA < P_SAMPLE_MIN_A) else min(k - 2, P_SAMPLE_LISTS)
    if nj == 0:
        return k, []
    x = A[np.arange(P_SAMPLES, dtype=np.int64) * lenA // P_SAMPLES]
    depth = np.full(P_SAMPLES, nj, np.int64)  # lists 1..depth all hit
    for j in range(nj, 0, -1):
        L = q.lists[j]
        p = np.searchsorted(L, x, side="left")
        hit = (p < L.size) & (L[np.minimum(p, max(L.size - 1, 0))] == x) if L.size else np.zeros(P_SAMPLES, bool)
        depth = np.where(hit, depth, j - 1)
    ke, alive, seq = k, P_SAMPLES, []
    for jj in range(1, nj + 1):
        alive -= int(np.sum(depth == jj - 1))
        seq.append(alive)
        if alive * P_DEFER_DIV < P_SAMPLES:
            ke = 1 + jj
            break
    if events is not None:
        _add(events, "sample.taken")
        thr = P_SAMPLES // P_DEFER_DIV
        if any(a == thr for a in seq):
            _add(events, "sample.alive_eq_threshold")
        if ke < k:
            _add(events, "sample.defer")
            if ke == 2:
                _add(events, "sample.defer_j1")
            else:
                _add(events, "sample.defer_later")
            if ke - 1 == k - 2:
                _add(events, "sample.defer_last_split")
            if seq[-1] == thr - 1:
                _add(events, "sample.alive_one_below_threshold")
        if k - 2 > P_SAMPLE_LISTS:
            _add(events, "sample.nj_capped")
        if k - 2 == P_SAMPLE_LISTS:
            _add(events, "sample.nj_full")
    return ke, seq


# ---- lift32m: the 32-bit window search --------------------------------------------------------------------------------

def lift32m(s, l2, x, live, events=None, path=None):
    """Hit mask of the low words x (any shape) in the staged slice s (uint32, n >= P = 2^l2) as lift32m finds it:
    three pivots choose one of four windows of P values, then log2 P lifting steps.  live: lanes whose result is
    used (events are recorded for those only); path: the ladder that called it ("pair" or "group"), which names the
    pivot and window events (none for the rows x one list ladder)."""
    n, P = int(s.size), 1 << l2
    assert P <= n, (P, n)
    y = n - P
    d = (y + 2) // 3
    s1, s2 = min(d, y), min(2 * d, y)
    p0, p1, p2 = s[P - 1], s[s1 + P - 1], s[s2 + P - 1]
    st = np.zeros(x.shape, np.int64)
    st = np.where(p0 < x, s1, st)
    st = np.where(p1 < x, s2, st)
    st = np.where(p2 < x, y, st)
    st0 = st
    h = P >> 1
    while h:
        st = np.where(s[st + h - 1] < x, st + h, st)
        h >>= 1
    hit = s[st] == x
    if events is not None and np.any(live):
        xl, w0 = x[live], st0[live]
        win = np.select([(p0 >= xl), (p1 >= xl), (p2 >= xl)], [0, 1, 2], 3)
        for i, pv in enumerate((p0, p1, p2) if path else ()):
            if np.any(xl == pv):
                _add(events, f"fast.{path}.x_on_pivot{i}")
        for wi in range(4 if path else 0):
            m = win == wi
            if np.any(xl[m] == s[w0[m]]):
                _add(events, f"fast.{path}.x_window{wi}_first")
            if np.any(xl[m] == s[w0[m] + P - 1]):
                _add(events, f"fast.{path}.x_window{wi}_last")
        if np.any(xl < s[0]):
            _add(events, "fast.x_below_slice")
        if np.any(xl > s[-1]):
            _add(events, "fast.x_above_slice")
        hl = hit[live]
        if np.any(hl & (xl == 0)):
            _add(events, "fast.hit_low_0")
        if np.any(hl & (xl == 0xFFFFFFFF)):
            _add(events, "fast.hit_low_ffffffff")
    return hit


def window_gaps(n, l2):
    """Largest gap between neighbouring windows of lift32m on a slice of n values (<= P: the windows cover it)."""
    P = 1 << l2
    y = n - P
    d = (y + 2) // 3
    s1, s2 = min(d, y), min(2 * d, y)
    return max(s1, s2 - s1, y - s2)


# ---- one tile ---------------------------------------------------------------------------------------------------------

Stage = namedtuple("Stage", "r0 r1 n64 head words incl fits nstaged headA")


def stage_tile(plan: Plan, q: Query, a0, na, keff, events):
    """filter_plan_kernel's bounds and the TMA warp's layout of one tile."""
    A, cap = q.lists[0], plan.slice_cap
    km1 = keff - 1
    r0, r1, n64, head, words, incl, fits = [], [], [], [], [], [], []
    run = 0
    for j in range(1, keff):
        L = q.lists[j]
        if na:
            a, b = int(np.searchsorted(L, A[a0], "left")), int(np.searchsorted(L, A[a0 + na - 1], "right"))
        else:
            a = b = 0
        r0.append(a)
        r1.append(b)
        mine = j - 1 < P_MAXL
        n = b - a
        hd = (q.offs[j] + a) & 1 if mine else 0
        w = ((n + hd + 1) & ~1) if (mine and n <= cap) else 0
        run += w
        n64.append(n)
        head.append(hd)
        words.append(w)
        incl.append(run)
        fits.append(mine and n <= cap and run <= cap)
    nstaged = 0
    while nstaged < len(fits) and fits[nstaged]:
        nstaged += 1
    nstaged = min(nstaged, km1, P_MAXL)
    headA = ((q.offs[0] + a0) & 1) if na else 0
    if na:
        if headA:
            _add(events, "stage.headA1")
        lim = min(km1, P_MAXL)
        if any(head[j] and j < nstaged for j in range(lim)):
            _add(events, "stage.head1")
        if any(incl[j] == cap for j in range(nstaged)):
            _add(events, "stage.exact_fit")
        if nstaged < lim:
            j = nstaged
            before = incl[j - 1] if j else 0
            if n64[j] > cap:
                _add(events, "stage.slice_over_cap")
            elif n64[j] + head[j] + before == cap + 1:
                _add(events, "stage.one_word_over")
            if any(fits[jj] for jj in range(j + 1, lim)):
                _add(events, "stage.leading_run_cut")
        if km1 > P_MAXL:
            _add(events, "stage.beyond_maxl")
        if km1 and nstaged == km1:
            _add(events, "stage.all_staged")
    return Stage(r0, r1, n64, head, words, incl, fits, nstaged, headA)


def _rank(cand, idx, x, has_prev, prev, A, a0):
    """cand_rank: copies of x before tile position idx, plus those before the tile when the run reaches its start."""
    s = idx
    while s > 0 and int(cand[s - 1]) == x:
        s -= 1
    r = idx - s
    if s == 0 and has_prev and prev == x:
        r += a0 - int(np.searchsorted(A[:a0], np.uint64(x), "left"))
    return r, s == 0 and has_prev and prev == x


def simulate_tile(plan: Plan, q: Query, tix, keff, events):
    """Survivors of one tile (values in tile order) after the query's first keff lists, as the consumer warps
    produce them."""
    VA, TA, op = plan.va, plan.ta, plan.op
    WC = 32 * VA
    A, lenA = q.lists[0], q.lenA
    a0 = tix * TA
    na = min(TA, lenA - a0) if a0 < lenA else 0
    km1 = keff - 1
    st = stage_tile(plan, q, a0, na, keff, events)
    nstaged = min(st.nstaged, km1)
    cand = A[a0:a0 + na]
    has_prev = a0 > 0 and na > 0
    prev = int(A[a0 - 1]) if has_prev else 0
    keep_hits = op == OP_INTERSECT
    slices = [q.lists[j + 1][st.r0[j]:st.r1[j]] for j in range(km1)]
    lo_words = [s.astype(np.uint32) for s in slices]  # low 32 bits (astype wraps)
    fast_tile = na > 0 and (int(cand[0]) >> 32) == (int(cand[na - 1]) >> 32)
    if na and not fast_tile:
        _add(events, "tile.straddle_2^32")
        if (int(cand[na - 2]) >> 32 if na > 1 else -1) == int(cand[0]) >> 32:
            _add(events, "tile.last_alone_crosses")
        if na > 1 and int(cand[1]) >> 32 == int(cand[na - 1]) >> 32:
            _add(events, "tile.first_alone_below")
    if na and has_prev and (prev >> 32) != (int(cand[0]) >> 32) and fast_tile:
        _add(events, "tile.starts_on_new_upper_word")
    if na and int(cand[na - 1]) == U64_MAX:
        _add(events, "tile.holds_2^64-1")
    out, kinds = [], set()
    for w in range(P_CW):
        wn = na - WC * w
        rows = 0 if wn <= 0 else (VA if wn >= WC else (wn + 31) >> 5)
        if na:
            _add(events, f"warp.va{VA}.rows{rows}")
        idx = WC * w + np.arange(32)[None, :] + 32 * np.arange(VA)[:, None]  # (VA, 32): tile position of (row, lane)
        valid = idx < na
        c = np.zeros((VA, 32), np.uint64)
        c[valid] = cand[idx[valid]]
        alive = valid.copy()
        dup = np.zeros((VA, 32), bool)
        for i, l in zip(*np.nonzero(valid)):
            t_ = int(idx[i, l])
            before = int(cand[t_ - 1]) if t_ > 0 else prev
            if (t_ > 0 or has_prev) and before == int(c[i, l]):
                dup[i, l] = True
        warp_dup = bool(dup.any())
        fast = (not warp_dup) and nstaged == km1 and na > 0 and fast_tile
        if rows == 0:
            continue
        kinds.add("fast" if fast else "wide")
        live = [int(alive.sum())]
        t = 0
        if warp_dup:
            _add(events, "wide.dup_warp")
        if fast:
            _add(events, "fast.warp")
            hiword = int(cand[0]) >> 32
            x = (c & np.uint64(0xFFFFFFFF)).astype(np.uint32)
            while t < km1 and rows > 0:
                n = [int(s.size) for s in slices]
                rmask = np.arange(VA)[:, None] < rows
                if (rows == 2 and t >= 1 and t + 1 < km1 and n[t] and n[t + 1]
                        and max(n[t], n[t + 1]) <= 3 << (min(n[t], n[t + 1]).bit_length() - 1)):
                    l2 = min(n[t], n[t + 1]).bit_length() - 1
                    _add(events, "fast.pair")
                    if max(n[t], n[t + 1]) == 3 << l2:
                        _add(events, "fast.pair_n_3P")
                    m = alive & rmask
                    h0 = lift32m(lo_words[t], l2, x[:2], m[:2], events, "pair")
                    h1 = lift32m(lo_words[t + 1], l2, x[:2], m[:2], events, "pair")
                    if l2 >= 10:
                        _add(events, "fast.pair_l2_ge_10")
                    hit = np.zeros_like(alive)
                    hit[:2] = h0 & h1
                    alive &= hit
                    t += 2
                elif rows >= 2:
                    if (rows == 2 and t >= 1 and t + 1 < km1 and n[t] and n[t + 1]):
                        _add(events, "fast.pair_refused_ratio")
                        r = max(n[t], n[t + 1]) / (1 << (min(n[t], n[t + 1]).bit_length() - 1))
                        if r > 4:
                            _add(events, "fast.pair_refused_n_gt_4P")
                        elif r == 4:
                            _add(events, "fast.pair_refused_n_eq_4P")
                    _add(events, "fast.rows_x1")
                    if rows > 2:
                        _add(events, "fast.rows_x1.all_rows")
                    hit = np.zeros_like(alive)
                    if n[t]:
                        hit = lift32m(lo_words[t], n[t].bit_length() - 1, x, alive & rmask, events) & rmask
                    else:
                        _add(events, f"{'' if keep_hits else 'diff.'}fast.empty_slice.rows")
                    alive &= hit if keep_hits else ~hit
                    t += 1
                else:
                    g = min(km1 - t, 3)
                    nn = [n[t + j] if j < g else n[t] for j in range(3)]
                    nmin, nmax = min(nn), max(nn)
                    m0 = alive[0]
                    if nmin == 0:
                        _add(events, f"{'' if keep_hits else 'diff.'}fast.empty_slice.g{nn.index(0)}")
                        ok = np.zeros(32, bool) if keep_hits else np.ones(32, bool)
                        g = g if keep_hits else 1
                    else:
                        l2 = nmin.bit_length() - 1
                        if nmax > 3 << l2:
                            _add(events, "fast.ladder_fallback")
                            g, l2 = 1, nn[0].bit_length() - 1
                        _add(events, f"fast.g{g}")
                        hs = [lift32m(lo_words[t + j], l2, x[0], m0, events, "group") for j in range(g)]
                        ok = np.logical_and.reduce(hs)
                        if g == 1 and not keep_hits:
                            ok = ~hs[0]
                    alive[0] &= ok
                    alive[1:] = False
                    t += g
                if t < km1 and rows == 1:
                    if not alive[0].any():
                        rows, alive[:] = 0, False
                elif t < km1:
                    m = alive & (np.arange(VA)[:, None] < rows)
                    tot = int(m.sum())
                    nrows = (tot + 31) >> 5
                    if nrows == 0:
                        rows, alive[:] = 0, False
                    elif nrows < rows:
                        vals = x[m]  # row-major: row i lanes 0..31, then row i + 1
                        x = np.zeros_like(x)
                        x.reshape(-1)[:tot] = vals
                        alive = (np.arange(VA * 32).reshape(VA, 32) < tot)
                        rows = nrows
                        _add(events, "fast.repack")
                live.append(int(alive.sum()) if rows else 0)
            c = (np.uint64(hiword) << np.uint64(32)) | x.astype(np.uint64)
            t = km1
        def search(j, rmask):
            """phit / the HBM search of list j for the alive candidates of the rows in rmask: the position is the
            lower bound of x in the slice [r0, r1) of list j, plus the duplicate rank (cand_rank) for repeated
            values; a hit reads list j there (shared memory for a staged slice, HBM past it)"""
            B, a, b = q.lists[j + 1], st.r0[j], st.r1[j]
            m = alive & rmask
            g = a + np.searchsorted(B[a:b], c, "left")
            for i, l in zip(*np.nonzero(m & dup)):
                r, from_prev = _rank(cand, int(WC * w + l + 32 * i), int(c[i, l]), has_prev, prev, A, a0)
                _add(events, "dup.rank")
                if from_prev:
                    _add(events, "dup.run_from_prev_tile")
                g[i, l] += r
                if g[i, l] >= b:
                    _add(events, "dup.rank_past_slice")
                if g[i, l] >= B.size:
                    _add(events, "dup.rank_past_list")
            h = g < B.size
            h[h] = B[g[h]] == c[h]
            return m & (h if keep_hits else ~h)

        all_rows = np.ones((VA, 32), bool)
        while t < km1 and rows > 0:
            if t < nstaged:
                if rows >= 2 or t + 1 >= nstaged:
                    if rows >= 2:
                        _add(events, "wide.staged_rows")
                    else:
                        _add(events, "wide.staged_one")
                    if slices[t].size == 0:
                        _add(events, "wide.empty_slice")
                        if keep_hits:
                            alive[:], rows = False, 0
                    else:
                        alive = search(t, np.arange(VA)[:, None] < ((rows + 1) & ~1))
                    t += 1
                else:
                    nl = 3 if nstaged - t >= 3 else 2
                    _add(events, f"wide.row_g{nl}")
                    if any(slices[t + j].size == 0 for j in range(nl)) and keep_hits:
                        _add(events, "wide.empty_slice")
                        alive[:], rows = False, 0
                    else:
                        row0 = np.arange(VA)[:, None] == 0
                        alive &= row0
                        for j in range(nl):
                            if slices[t + j].size:
                                alive = search(t + j, row0)
                    t += nl
            else:
                _add(events, "wide.hbm_list")
                if t >= P_MAXL:
                    _add(events, "wide.hbm_list_beyond_maxl")
                alive = search(t, all_rows)
                t += 1
            if t < km1:
                if not warp_dup:
                    m = alive & (np.arange(VA)[:, None] < rows)
                    tot = int(m.sum())
                    nrows = (tot + 31) >> 5
                    if nrows == 0:
                        rows, alive[:] = 0, False
                    elif nrows < rows:
                        vals = c[m]
                        c = np.zeros_like(c)
                        c.reshape(-1)[:tot] = vals
                        alive = (np.arange(VA * 32).reshape(VA, 32) < tot)
                        rows = nrows
                elif not alive.any():
                    rows = 0
            live.append(int(alive.sum()) if rows else 0)
        if rows == 0:
            alive[:] = False
        if _has_run(live, (64, 33, 32, 0)) and fast:
            _add(events, "fast.live_64_33_32_0")
        out.append(c[alive])  # row-major = tile order
    if kinds == {"fast", "wide"}:
        _add(events, "wide.mixed_tile")
    return np.concatenate(out) if out else np.zeros(0, np.uint64)


def _add(events, name):
    """Record an event; every name is registered in EVENTS."""
    assert name in EVENTS, f"event {name!r} is not registered in EVENTS"
    events.add(name)


def device_offsets(queries, offsets):
    """Element offsets of every list when a batch's lists are laid out back to back in one 256-byte-aligned device
    buffer, each padded to the parity its fixture chose (the layout of the device-form tests)."""
    out, pos = [], 0
    for q, oq in zip(queries, offsets):
        row = []
        for l, o in zip(q, oq):
            pos += (pos + o) & 1
            row.append(pos)
            pos += int(np.asarray(l).size)
        out.append(row)
    return out, pos


def deferring_queries(plan: Plan):
    """Queries of a batch that the sample defers (what dgx_filter_tail_queries counts for it)."""
    return sum(sample_keff(q)[0] < q.k for q in plan.queries) if plan.deep else 0


def _has_run(seq, pat):
    return any(tuple(seq[i:i + len(pat)]) == pat for i in range(len(seq) - len(pat) + 1))


# ---- the whole batch ------------------------------------------------------------------------------------------------

Run = namedtuple("Run", "plan keff mids mid_off results events tail_queries")


def simulate(queries, op=OP_INTERSECT, resident=False, offsets=None) -> Run:
    plan = plan_batch(queries, op, resident, offsets)
    ev = set()
    _add(ev, f"batch.va{plan.va}")
    ks = {q.k for q in plan.queries}
    if ks & {1, 2} and max(ks) >= 3:
        _add(ev, "batch.mixed_k")
    if ks == {1}:
        _add(ev, "batch.k1_only")
    if op == OP_DIFFERENCE:
        _add(ev, "batch.difference")
    keff = []
    for q in plan.queries:
        ke = sample_keff(q, ev)[0] if plan.deep else q.k
        keff.append(ke)
    if plan.deep:
        _add(ev, "batch.deep")
        if any(q.k >= 3 and q.lenA == P_SAMPLE_MIN_A - 1 for q in plan.queries):
            _add(ev, "sample.lenA_one_below_min")
        if any(q.k >= 3 and q.lenA == P_SAMPLE_MIN_A for q in plan.queries):
            _add(ev, "sample.lenA_at_min")
    mids = []
    for q, ke in zip(plan.queries, keff):
        if q.lenA == 0:
            _add(ev, "query.empty_A")
        if any(a != b for a, b in zip(q.order, range(q.k))):
            _add(ev, "query.reordered")
        parts = [simulate_tile(plan, q, t, ke, ev) for t in range(q.ntiles)]
        mids.append(np.concatenate(parts))
    deferred = [ke < q.k for q, ke in zip(plan.queries, keff)]
    mid_off = np.concatenate([[0], np.cumsum([m.size for m in mids])]).astype(np.int64)
    if not any(deferred):
        return Run(plan, keff, mids, None, mids, ev, 0)
    # filter_tail_kernel: the batch's survivors went to mid; every value of a deferring query is tested against the
    # lists after k_eff with its duplicate rank among the copies in its query's range
    _add(ev, "tail.ran")
    m = int(mid_off[-1])
    inner = [int(o) for o in mid_off[1:-1]]
    if any(o % P_TAIL_NT == 0 and 0 < o < m for o in inner):
        _add(ev, "tail.mid_off_on_chunk_edge")
    if plan.queries[0].lenA == 0 or mids[0].size == 0:
        _add(ev, "tail.leading_empty")
    if mids[-1].size == 0:
        _add(ev, "tail.trailing_empty")
    res = []
    for q, ke, mv in zip(plan.queries, keff, mids):
        if ke == q.k:
            res.append(mv)
            continue
        keep = np.ones(mv.size, bool)
        first = np.searchsorted(mv, mv, "left")
        r = np.arange(mv.size) - first
        if np.any(r > 0):
            _add(ev, "tail.dup_rank")
        first_only = np.ones(mv.size, bool)
        for j in range(ke, q.k):
            L = q.lists[j]
            lb = np.searchsorted(L, mv, "left")
            g = lb + r
            ok = g < L.size
            ok[ok] = L[g[ok]] == mv[ok]
            keep &= ok
            ok0 = lb < L.size
            ok0[ok0] = L[lb[ok0]] == mv[ok0]
            first_only &= ok0
        if np.any(first_only & ~keep):
            _add(ev, "tail.rank_drops_copy")  # a deferred list holds fewer copies of a value than the intermediate
        res.append(mv[keep])
    return Run(plan, keff, mids, mid_off, res, ev, sum(deferred))


# ---- the oracle's rule ------------------------------------------------------------------------------------------------

def has_dups(lists):
    return any(l.size > 1 and bool(np.any(l[1:] == l[:-1])) for l in map(_u64, lists))


def oracle_result(orc, lists, op):
    """The oracle's answer for one query.  With repeated values the rule is the two-pointer IntersectWith's
    multiset-min over the lists in length order (the reference's IntersectSorted chain switches to variants that
    keep fewer copies), and multiset difference."""
    lists = [_u64(l) for l in lists]
    if op == OP_DIFFERENCE:
        return orc.difference(lists[0], lists[1])
    if len(lists) == 1:
        return lists[0].copy()
    if has_dups(lists):
        ls = sorted(lists, key=len)
        w = ls[0]
        for l in ls[1:]:
            w = orc.intersect_with_lin(w, l)
        return w
    if len(lists) == 2:
        return orc.intersect_with(lists[0], lists[1])
    return orc.intersect_sorted(lists)


# ---- fixture builders -----------------------------------------------------------------------------------------------
#
# A fixture is one batch: its queries (lists in caller order), the operation, the element offset of every list on the
# device (the parity of the 16-byte head of its slices), whether it is aimed at a resident-inputs lane (the only one
# that samples and defers), and the events the model must see it reach there.

Fixture = namedtuple("Fixture", "name queries op offsets resident events tail")


def fixture(name, queries, events, op=OP_INTERSECT, offsets=None, resident=False, tail=None):
    queries = [[_u64(l) for l in q] for q in queries]
    offsets = offsets or [[0] * len(q) for q in queries]
    return Fixture(name, queries, op, offsets, resident, frozenset(events), tail)


def _pick(rng, pool, n):
    pool = np.asarray(pool, np.uint64)
    assert n <= pool.size, (n, pool.size)
    return np.sort(rng.choice(pool, n, replace=False)) if n else np.zeros(0, np.uint64)


def tile_list(rng, A, inside, keep, n_in, below=3, above=3, gap=1):
    """A filter list whose slice of the tile [A[0], A[-1]] holds exactly n_in values: `keep` of A's values (the
    candidates that can survive) and the rest drawn from `inside` (values in the tile range not in A); `below` values
    under the tile (they set r0) and `above` over it."""
    lo, hi = int(A[0]), int(A[-1])
    keep = _u64(keep)
    rest = _pick(rng, inside, n_in - keep.size)
    under = np.array([lo - gap * (below - i) for i in range(below)], np.uint64) if below else np.zeros(0, np.uint64)
    over = np.array([hi + gap * (i + 1) for i in range(above)], np.uint64) if above else np.zeros(0, np.uint64)
    return np.sort(np.concatenate([under, keep, rest, over]))


def spaced(base, n, stride):
    return np.uint64(base) + np.uint64(stride) * np.arange(n, dtype=np.uint64)


def holes(A, stride):
    """Every value strictly between A's values (A spaced by stride)."""
    return (A[:-1, None] + np.arange(1, stride, dtype=np.uint64)[None, :]).reshape(-1)


def ordered(lists, base_len):
    """Pad lists 1.. with values far above everything so that their total lengths are strictly increasing and above
    base_len: the stable length sort then keeps the order the fixture built."""
    top = max(int(l[-1]) for l in lists if l.size) if any(l.size for l in lists) else 0
    out, need = [lists[0]], base_len + 1
    for j, l in enumerate(lists[1:]):
        pad = max(0, need - l.size)
        ext = spaced(top + 1_000_000 * (j + 1) + 1, pad, 3)
        l2 = np.sort(np.concatenate([l, ext]))
        out.append(l2)
        need = l2.size + 1
    return out


EDGE_SIZES = (1, 31, 32, 33, 63, 64, 65, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025)


def warp_edge_fixtures(seed=1):
    """|A| at every warp-row and tile edge of both geometries: k = 2 (VA = 4, 1024-value tiles) and k = 3 (VA = 2)."""
    import gen

    fx = []
    for k in (2, 3):
        rng = np.random.default_rng(seed + k)
        qs = []
        for n in EDGE_SIZES:
            master = gen.zipf_gaps(rng, 2 * n + 64, start=1 + (n << 32))
            A = _pick(rng, master, n)
            qs.append([A] + [np.union1d(gen.thin(rng, master, 0.75), gen.thin(rng, A, 0.9)) for _ in range(k - 1)])
        va = 4 if k == 2 else 2
        fx.append(fixture(f"warp and tile edges, k={k}", qs, {f"warp.va{va}.rows{r}" for r in range(1, va + 1)}
                          | {"fast.warp", f"batch.va{va}"}))
    return fx


def batch_geometry_fixtures(seed=10):
    import gen

    rng = np.random.default_rng(seed)
    qs, ones = [], []
    for i, k in enumerate((1, 2, 3, 1, 2, 5, 2, 1)):
        master = gen.zipf_gaps(rng, 6000, start=1 + (i << 40))
        A = gen.thin(rng, master, 0.3)
        qs.append([A] + [np.union1d(gen.thin(rng, master, 0.6), gen.thin(rng, A, 0.8)) for _ in range(k - 1)])
        if k == 1:
            ones.append([A])
    qs.append([np.zeros(0, np.uint64), gen.zipf_gaps(rng, 50), gen.zipf_gaps(rng, 70)])
    return [fixture("batch of k = 1, 2, 3 and 5: 2-list queries in 512-value tiles", qs,
                    {"batch.mixed_k", "batch.va2", "query.empty_A", "fast.warp"}),
            fixture("batch of one-list queries", ones + [[np.zeros(0, np.uint64)]], {"batch.k1_only"})]


def maxl_fixtures(seed=20):
    """k = 9, 10 and 17: filter lists 9 and up are searched in HBM; kmax >= 9 sets slice_cap to 8 staged lists."""
    import gen

    rng = np.random.default_rng(seed)
    qs = []
    for k in (9, 10, 17):
        master = gen.zipf_gaps(rng, 8000)
        A = gen.thin(rng, master, 0.4)
        qs.append([A] + [np.union1d(gen.thin(rng, master, 0.3), gen.thin(rng, A, 0.97)) for _ in range(k - 1)])
    fx = [fixture("k = 9, 10, 17: lists past P_MAXL in HBM", qs,
                  {"stage.beyond_maxl", "wide.hbm_list_beyond_maxl", "batch.va2"})]
    fx.append(fixture("k = 9 alone: eight filter lists, as many as a stage holds", [qs[0]], {"batch.va2"}))
    fx.append(fixture("k = 10 alone", [qs[1]], {"stage.beyond_maxl", "wide.hbm_list_beyond_maxl"}))
    return fx


def staging_fixtures(seed=30):
    """Slices at the stage capacity: exactly slice_cap words with head 0 and 1, one word over, a slice over the cap,
    a run of slices filling the stage with the next one word over, a long first slice cutting the leading run."""
    rng = np.random.default_rng(seed)
    fx = []
    # 2-list batch: one filter list, slice_cap = 2.25 tile widths
    _, ta, cap, _ = geometry(2)
    qs, offs = [], []
    for i, (n_in, head, what) in enumerate(((cap, 0, "exact"), (cap, 1, "over by its head"), (cap - 1, 1, "exact, head 1"),
                                            (cap + 1, 0, "over"), (5000, 0, "HBM"))):
        A = spaced((i + 1) << 36, ta, 16)
        L = tile_list(rng, A, holes(A, 16), _pick(rng, A, int(0.8 * ta)), n_in, below=4)
        qs.append([A, L])
        offs.append([0, head])  # r0 = 4: the head is the list's own offset parity
    fx.append(fixture("2-list slices at slice_cap", qs,
                      {"stage.exact_fit", "stage.one_word_over", "stage.slice_over_cap", "stage.head1", "wide.hbm_list",
                       "fast.warp", "batch.va4"}, offsets=offs))
    # 4-list batch: three staged lists share slice_cap
    _, ta, cap, _ = geometry(4)
    qs, offs = [], []
    half = cap // 2
    for i, (ns, hs) in enumerate((((half, half, 1), (0, 0, 0)),          # 1..2 fill the stage, 3 one word over
                                  ((cap - 1, 1, 60), (1, 0, 0)),         # 1 fills it with its head, 2 one word over
                                  ((cap + 72, 100, 100), (0, 0, 0)),     # a long first slice cuts the leading run
                                  ((300, 400, 500), (1, 1, 0)))):        # everything staged, heads 1 (A's too)
        A = spaced((i + 1) << 36, ta, 32)
        inside = holes(A, 32)
        ls = [tile_list(rng, A, inside, _pick(rng, A, min(n, int(0.9 * ta)) if j == 0 else int(0.5 * min(n, ta))), n,
                        below=2) for j, n in enumerate(ns)]
        qs.append(ordered([A] + ls, A.size))
        offs.append([i // 3] + list(hs))
    fx.append(fixture("4-list slices sharing the stage", qs,
                      {"stage.exact_fit", "stage.one_word_over", "stage.leading_run_cut", "stage.slice_over_cap",
                       "stage.all_staged", "stage.head1", "stage.headA1", "wide.hbm_list"}, offsets=offs))
    return fx


def pair_queries(rng, kmax):
    """Two rows x two lists: the second and third filter lists of a k = 4 query have slice lengths P and n for n in
    P, 2P - 1, 2P, 3P, 3P + 1, 4P, 4P + 1, 5P, for every P whose slices still fit the stage of a batch whose widest
    query has kmax lists.  Every value of the longer slice is a candidate where the tile allows it, so every pivot
    and window edge is searched; the short slice holds the values at positions P..2P - 1 of the long one, the first
    gap the windows would leave past n = 4P."""
    _, ta, cap, _ = geometry(kmax)
    qs = []
    P = 1
    while True:
        ns = sorted({P, 2 * P - 1, 2 * P, 3 * P, 3 * P + 1, 4 * P, 4 * P + 1, 5 * P})
        ns = [n for n in ns if ta + ((P + 1) & ~1) + ((n + 1) & ~1) <= cap]
        if not ns:
            break
        for n in ns:
            i = len(qs)
            A = spaced(((i + 7) << 33) + (1 << 20), ta, 8)
            inside = holes(A, 8)
            L1 = tile_list(rng, A, inside, A, ta, below=2)
            if n <= ta:
                long_in = _pick(rng, A, n)
            else:
                long_in = np.sort(np.concatenate([A, _pick(rng, inside, n - ta)]))
            L3 = tile_list(rng, A, inside, long_in, n, below=2)
            short_in = long_in[P:2 * P] if n >= 2 * P else long_in[:P]
            L2 = tile_list(rng, A, inside, short_in, P, below=2)
            qs.append(ordered([A, L1, L2, L3], ta))
        P *= 2
    return qs


# x on each pivot, and on the first and last element of the window it chooses.  The last window starts at n - P <=
# s2 + P - 1 (the windows touch or overlap while n <= 4P), so its first element is never above pivot 2 and x equal to
# it always chooses an earlier window: that event cannot occur.
WINDOW_EVENTS = ("x_on_pivot0", "x_on_pivot1", "x_on_pivot2") + tuple(
    f"x_window{w}_{end}" for w in range(4) for end in ("first", "last") if (w, end) != (3, "first"))


def pair_fixtures(seed=40):
    """The pair path in the stage of a 4-list batch (slice_cap 1728) and of a batch whose widest query has 9 lists
    (8 staged lists, slice_cap 4608, P up to 1024); a small k = 9 query sets that batch's geometry."""
    rng = np.random.default_rng(seed)
    ev = {"fast.pair", "fast.pair_n_3P", "fast.pair_refused_ratio", "fast.pair_refused_n_eq_4P",
          "fast.pair_refused_n_gt_4P"} | {f"fast.pair.{e}" for e in WINDOW_EVENTS}
    wide = spaced(1 << 50, 40, 4)
    nine = [wide] + [np.union1d(wide, spaced((1 << 50) + 1, 50 + j, 4)) for j in range(8)]
    return [fixture("pair path: slice lengths P..5P, 4-list stage", pair_queries(rng, 4), ev),
            fixture("pair path: slice lengths P..5P, 8-list stage", pair_queries(rng, 9) + [nine],
                    ev | {"fast.pair_l2_ge_10"})]


def group_fixtures(seed=50):
    """One row (|A| = 32) x three lists, and the cases that break the group up: lengths P..3P in one ladder, a length
    past 3P (one list, then two), and an empty slice at each position of the group; the same empty slices in the rows
    x one list path; Difference, where an empty slice keeps everything."""
    rng = np.random.default_rng(seed)
    _, ta, cap, _ = geometry(4)
    fx, qs = [], []
    for P in (1, 2, 8, 32, 128):
        for ns in ((P, P, P), (P, 2 * P, 3 * P), (3 * P, P, 2 * P), (P, 3 * P, 3 * P + 1), (3 * P + 1, P, P),
                   (P + 1, 2 * P + 1, 3 * P), (2 * P - 1, P, 3 * P), (P, 2 * P - 1, 2 * P - 1)):
            A = spaced(((len(qs) + 3) << 34) + 5, 32, 64)
            inside = holes(A, 64)
            # a slice of at most 32 values is made of candidates only: every pivot and window edge is searched
            ls = [tile_list(rng, A, inside, _pick(rng, A, n if n <= A.size else 24), n, below=1) for n in ns]
            qs.append(ordered([A] + ls, 32))
    fx.append(fixture("one row x three lists", qs, {"fast.g3", "fast.g2", "fast.g1", "fast.ladder_fallback",
                                                    "warp.va2.rows1"} | {f"fast.group.{e}" for e in WINDOW_EVENTS}))
    qs = []
    for pos in range(3):
        A = spaced(((pos + 1) << 34) + 5, 32, 64)
        inside = holes(A, 64)
        ls = [tile_list(rng, A, inside, _pick(rng, A, 20), 40, below=1) for _ in range(3)]
        ls[pos] = np.concatenate([spaced(1, 3, 1), spaced(int(A[-1]) + 1, 50, 1)])  # nothing inside the tile
        qs.append(ordered([A] + ls, 32))
    for pos in range(2):  # rows x one list: t = 0, and t = 1 after a list that keeps every candidate
        A = spaced(((pos + 9) << 34) + 5, ta, 64)
        inside = holes(A, 64)
        ls = [tile_list(rng, A, inside, A, ta, below=1), tile_list(rng, A, inside, _pick(rng, A, 400), 500, below=1),
              tile_list(rng, A, inside, _pick(rng, A, 300), 500, below=1)]
        ls[pos] = np.concatenate([spaced(1, 3, 1), spaced(int(A[-1]) + 1, 2 * ta, 1)])
        qs.append(ordered([A] + ls, ta))
    fx.append(fixture("empty slices in the chain", qs, {"fast.empty_slice.g0", "fast.empty_slice.g1",
                                                        "fast.empty_slice.g2", "fast.empty_slice.rows"}))
    qs = []
    for n in (20, 32, 33, 1024, 1500):
        u = spaced((n << 34) + 5, n, 64)
        v = np.concatenate([spaced(1, 3, 1), spaced(int(u[-1]) + 1, 10, 1)])
        qs.append([u, v])
        v2 = tile_list(rng, u, holes(u, 64), _pick(rng, u, n // 2), n // 2 + 7, below=1)
        qs.append([u, v2])
    fx.append(fixture("Difference with empty slices", qs, {"diff.fast.empty_slice.g0", "diff.fast.empty_slice.rows",
                                                           "batch.difference", "fast.rows_x1.all_rows"},
                      op=OP_DIFFERENCE))
    return fx


def survivor_fixture(seed=60):
    """A warp whose survivors go 64 -> 33 -> 32 -> 0 with lists still to come."""
    rng = np.random.default_rng(seed)
    A = spaced((5 << 33) + 9, 64, 64)
    inside = holes(A, 64)
    k33 = _pick(rng, A, 33)
    k32 = _pick(rng, k33, 32)
    ls = [tile_list(rng, A, inside, k33, 40, below=1), tile_list(rng, A, inside, k32, 40, below=1),
          tile_list(rng, A, inside, [], 200, below=1), tile_list(rng, A, inside, _pick(rng, A, 8), 10, below=1),
          tile_list(rng, A, inside, _pick(rng, A, 8), 10, below=1)]
    return fixture("survivors 64 -> 33 -> 32 -> 0", [ordered([A] + ls, 64)],
                   {"fast.live_64_33_32_0", "fast.repack", "fast.ladder_fallback"})


def upper_word_fixtures(seed=70):
    """Tiles around a multiple of 2^32: the last value alone across, the first alone below, tiles on either side,
    and a tile of one upper word holding low words 0 and 0xFFFFFFFF up to 2^64 - 1."""
    rng = np.random.default_rng(seed)
    fx = []
    for k in (2, 3):
        _, ta, _, _ = geometry(k)
        qs = []
        hi = 7 << 32
        cases = [np.concatenate([spaced(hi - 2 * (ta - 1), ta - 1, 2), [hi + 3]]),               # last alone across
                 np.concatenate([[hi - 5], spaced(hi + 1, ta - 1, 2)]),                            # first alone below
                 np.concatenate([spaced(hi - 2 * ta, ta, 2), spaced(hi, ta, 2)]),                  # tiles either side
                 np.concatenate([[U64_MAX - 0xFFFFFFFF], spaced(U64_MAX - 2 * (ta - 2), ta - 1, 2)]),  # low 0 .. 2^64-1
                 np.concatenate([spaced(hi + 0xFFFFFFFF - 4 * (ta - 1), ta, 4), [(8 << 32)]])]    # low 0xFFFFFFFF
        for A in cases:
            A = _u64(A)
            pool = np.setdiff1d(np.concatenate([A + np.uint64(1), A[1:] - np.uint64(1)]), A)
            keep = np.union1d(_pick(rng, A, int(0.7 * A.size)), [A[0], A[-1]])
            ls = [np.union1d(keep, _pick(rng, pool, A.size // 3)) for _ in range(k - 1)]
            if A[-1] != np.uint64(U64_MAX):
                ls = [np.union1d(l, [A[-1] + np.uint64(1)]) for l in ls]
            qs.append(ordered([A] + ls, A.size) if A[-1] != np.uint64(U64_MAX) else
                      [A] + [np.union1d(l, A[:1] - np.uint64(np.arange(1, 3 + j))) for j, l in enumerate(ls)])
        fx.append(fixture(f"upper words, k={k}", qs, {"tile.straddle_2^32", "tile.last_alone_crosses",
                                                      "tile.first_alone_below", "tile.starts_on_new_upper_word",
                                                      "tile.holds_2^64-1", "fast.hit_low_0", "fast.hit_low_ffffffff"}))
    return fx


def dup_fixtures(seed=80):
    """Repeated values: warps with and without them in one tile, a run from the previous tile, runs longer than a
    tile in A and in a filter list, ranks past the staged slice and past the list, Difference with more and fewer
    copies in u than in v."""
    rng = np.random.default_rng(seed)
    fx = []
    for k in (2, 3):
        _, ta, _, _ = geometry(k)
        qs = []
        # one repeated value in warp 3 only
        A = spaced((3 << 32) + 11, ta, 4)
        A[3 * 32 * (ta // 256) + 5] = A[3 * 32 * (ta // 256) + 4]
        A = np.sort(A)
        qs.append(ordered([A] + [np.union1d(_pick(rng, A, int(0.8 * ta)), _pick(rng, holes(A, 4), ta // 4))
                                 for _ in range(k - 1)], ta))
        # a run of 10 from the previous tile; the lists hold 7 and 9 copies
        base = spaced(1 << 33, 2 * ta, 4)
        x = base[ta - 5]
        A = np.sort(np.concatenate([np.delete(base, np.arange(ta - 5, ta + 5)), np.full(10, x, np.uint64)]))
        L = [np.sort(np.concatenate([np.setdiff1d(_pick(rng, base, ta + 100), [x]), np.full(c, x, np.uint64)]))
             for c in (7, 9)[:k - 1]]
        qs.append(ordered([A] + L, A.size))
        # a run longer than a tile in A (1.5 tiles) and in the lists (1.3 and 1.4 tiles)
        x = np.uint64((5 << 33) + 77)
        A = np.sort(np.concatenate([spaced((5 << 33) + 1, 50, 1), np.full(3 * ta // 2, x, np.uint64),
                                    spaced((5 << 33) + 100, 300, 1)]))
        L = [np.sort(np.concatenate([spaced((5 << 33) + 1, 60, 1), np.full(int(c * ta), x, np.uint64),
                                     spaced((5 << 33) + 100, 400, 1)])) for c in (1.3, 1.4)[:k - 1]]
        qs.append(ordered([A] + L, A.size))
        # the tile's last value has 6 copies at its end; the lists hold 3, and end with them
        x = np.uint64((6 << 33) + 4 * ta)
        A = np.sort(np.concatenate([spaced(6 << 33, ta - 6, 4), np.full(6, x, np.uint64)]))
        L = [np.sort(np.concatenate([_pick(rng, A[:-6], ta // 2), spaced((6 << 33) + 1, ta, 4), np.full(3, x, np.uint64)]))
             for _ in range(k - 1)]
        qs.append([A] + L)
        # a repeated value, and a list with nothing inside the tile (empty staged slice on the 64-bit path)
        A = np.sort(np.concatenate([spaced(7 << 33, 40, 8), [(7 << 33) + 8]]))
        L = [np.union1d(A, spaced((7 << 33) + 1, 100, 8)), np.concatenate([spaced(1, 5, 1), spaced(8 << 33, 200, 1)])]
        qs.append(ordered([A] + L[::-1][:k - 1], A.size))
        fx.append(fixture(f"duplicates, k={k}", qs, {"wide.dup_warp", "wide.mixed_tile", "dup.run_from_prev_tile",
                                                     "dup.rank_past_slice", "dup.rank_past_list", "wide.empty_slice"}))
    # Difference: more copies in u than in v, and fewer, across a tile edge
    qs = []
    for cu, cv in ((5, 3), (2, 4), (1300, 700), (700, 1300)):
        x = np.uint64((9 << 33) + 1000)
        u = np.sort(np.concatenate([spaced(9 << 33, 900, 1), np.full(cu, x, np.uint64), spaced((9 << 33) + 2000, 300, 1)]))
        v = np.sort(np.concatenate([spaced((9 << 33) + 500, 100, 3), np.full(cv, x, np.uint64)]))
        qs.append([u, v])
    fx.append(fixture("Difference with repeated values", qs, {"wide.dup_warp", "dup.rank", "dup.run_from_prev_tile"},
                      op=OP_DIFFERENCE))
    return fx


# ---- deferral (resident-inputs lanes) ---------------------------------------------------------------------------------

def _sample_pos(n):
    return np.arange(P_SAMPLES, dtype=np.int64) * n // P_SAMPLES


def defer_query(rng, n, hits, p=0.5, base=1 << 34, dup_every=0):
    """A of n values (stride 4) and filter lists that hold exactly the samples listed in hits[j] (indices 0..255;
    None: all of them) plus a p share of A's other values and filler between A's values; list j + 1 is longer than
    list j.  dup_every: every such value of A is repeated (three copies), and the lists hold one to three."""
    A = spaced(base, n, 4)
    sp = _sample_pos(n)
    other = np.setdiff1d(np.arange(n), sp)
    lists = []
    for j, h in enumerate(hits):
        hs = sp if h is None else sp[np.asarray(sorted(h), np.int64)] if len(h) else np.zeros(0, np.int64)
        # samples and other values are disjoint, and so are A's values and the filler between them (stride 4,
        # offsets 1..3 from distinct values): sorted concatenations are the unions
        sel = np.sort(np.concatenate([hs, other[rng.random(other.size) < p]]))
        L = A[sel]
        fill = n + 1000 * (j + 1) - L.size
        L = np.sort(np.concatenate([L, (A[rng.choice(n, max(fill, 0) // 3 + 1, replace=False), None]
                                        + np.arange(1, 4, dtype=np.uint64)[None, :]).reshape(-1)]))
        lists.append(L)
    if dup_every:
        rep = np.zeros(n, np.int64)
        rep[other[::dup_every]] = 2
        A = np.repeat(A, 1 + rep)
        lists = [np.sort(np.concatenate([L, np.repeat(L[::dup_every], rng.integers(0, 3, L[::dup_every].size))]))
                 for L in lists]
    return ordered([A] + lists, A.size)


def defer_fixtures(seed=90):
    rng = np.random.default_rng(seed)
    N = P_SAMPLE_MIN_A
    thr = P_SAMPLES // P_DEFER_DIV
    few = lambda c: list(range(0, 256, 256 // c))[:c]  # noqa: E731
    fx = [fixture("|A| = 65535 against 65536", [defer_query(rng, N - 1, [[], None], p=0.02),
                                               defer_query(rng, N, [[], None], p=0.02, base=1 << 36)],
                  {"sample.lenA_one_below_min", "sample.lenA_at_min", "sample.defer_j1"}, resident=True, tail=1)]
    for alive in (thr, thr - 1):
        fx.append(fixture(f"k = 3: {alive} samples alive after list 1", [defer_query(rng, N, [few(alive), None])],
                          {"sample.alive_eq_threshold"} if alive == thr else {"sample.defer_j1",
                                                                             "sample.alive_one_below_threshold"},
                          resident=True, tail=int(alive < thr)))
        fx.append(fixture(f"k = 5: {alive} samples alive after list 1", [
            defer_query(rng, N, [few(alive), few(thr), few(thr), None], p=0.9)],
            {"sample.alive_eq_threshold"} if alive == thr else {"sample.defer_j1"}, resident=True, tail=int(alive < thr)))
        fx.append(fixture(f"k = 5: {alive} samples alive after list 3", [
            defer_query(rng, N, [None, None, few(alive), None], p=0.9)],
            {"sample.alive_eq_threshold"} if alive == thr else {"sample.defer_last_split"}, resident=True,
            tail=int(alive < thr)))
    for k in (P_SAMPLE_LISTS + 2, P_SAMPLE_LISTS + 3):
        hits = [None] * P_SAMPLE_LISTS + [[]] + [None] * (k - 2 - P_SAMPLE_LISTS)
        fx.append(fixture(f"k = {k}: list {P_SAMPLE_LISTS + 1} is never a split point",
                          [defer_query(rng, N, hits, p=0.97)],
                          {"sample.nj_full"} if k == P_SAMPLE_LISTS + 2 else {"sample.nj_capped"}, resident=True, tail=0))
    return fx


def _intersect_k2(rng, n_res, base):
    """A 2-list query whose result has exactly n_res values."""
    A = spaced(base, max(n_res, 1) + 40, 4)
    keep = A[:n_res]
    B = np.union1d(keep, A[n_res:] + np.uint64(1))
    B = np.union1d(B, spaced(int(A[-1]) + 10, 50, 1))
    return [A, B]


def multiset_min(lists):
    """The r-th copy of x in lists[0] survives iff every other list holds more than r copies of it (the rule the
    pipeline and the tail apply): each value min(counts) times."""
    vals, cnt = np.unique(_u64(lists[0]), return_counts=True)
    for l in lists[1:]:
        v2, c2 = np.unique(_u64(l), return_counts=True)
        keep = np.isin(vals, v2)
        vals, cnt = vals[keep], np.minimum(cnt[keep], c2[np.searchsorted(v2, vals[keep])])
    return np.repeat(vals, cnt)


def pipeline_count(q, resident):
    """Values one query leaves in the intermediate of a deep batch: the survivors of its first k_eff lists."""
    pq = plan_batch([q], resident=resident).queries[0]
    ke = sample_keff(pq)[0]
    return int(multiset_min(pq.lists[:ke]).size)


def deep_mix_fixture(seed=100):
    """A deep batch: leading and trailing queries with an empty A, 2-list queries sized so that mid_off lands on
    multiples of 256, a deferring query with repeated values, a dense query that defers nothing."""
    rng = np.random.default_rng(seed)
    N = P_SAMPLE_MIN_A
    empty_lead = [np.zeros(0, np.uint64), spaced(1, 10, 1), spaced(1, 20, 1)]
    two = _intersect_k2(rng, 2 * P_TAIL_NT, 1 << 40)
    deferring = defer_query(rng, N + 3000, [[], None, None], p=0.02, base=1 << 41, dup_every=5)
    # values with 4 copies in A and the streamed list, 2 and 3 in the deferred ones: the tail keeps 2 by rank
    xs = deferring[0][1001:30000:997]
    xs = xs[np.sum(deferring[0][None, :] == xs[:, None], axis=1) == 1]
    deferring = [np.sort(np.concatenate([l[~np.isin(l, xs)], np.repeat(xs, c)])) for l, c in zip(deferring, (4, 4, 2, 3))]
    deferring = ordered(deferring, deferring[0].size)
    dense = defer_query(rng, N, [None, None], p=0.95, base=1 << 42)
    m = sum(pipeline_count(q, resident=True) for q in (empty_lead, two, deferring, dense))
    fill = (-m) % P_TAIL_NT + P_TAIL_NT
    tail2 = _intersect_k2(rng, fill, 1 << 43)
    empty_trail = [np.zeros(0, np.uint64), spaced(5, 30, 1), spaced(5, 40, 1), spaced(5, 50, 1)]
    qs = [empty_lead, two, deferring, dense, tail2, empty_trail]
    return fixture("deep batch: empty, 2-list, deferring with repeats, dense, 2-list, empty", qs,
                   {"batch.deep", "tail.ran", "tail.mid_off_on_chunk_edge", "tail.leading_empty", "tail.trailing_empty",
                    "tail.dup_rank", "tail.rank_drops_copy", "query.empty_A", "sample.defer_j1"}, resident=True,
                   tail=1)


def all_fixtures():
    return (warp_edge_fixtures() + batch_geometry_fixtures() + maxl_fixtures() + staging_fixtures() + pair_fixtures()
            + group_fixtures() + [survivor_fixture()] + upper_word_fixtures() + dup_fixtures() + defer_fixtures()
            + [deep_mix_fixture()])


# Every event the model can name, in one table: _add refuses a name missing here, and every name here must be reached
# by some fixture.
EVENTS = frozenset(f"""
batch.va2 batch.va4 batch.mixed_k batch.k1_only batch.difference batch.deep query.empty_A query.reordered
warp.va4.rows0 warp.va2.rows0 warp.va4.rows1 warp.va4.rows2 warp.va4.rows3 warp.va4.rows4 warp.va2.rows1 warp.va2.rows2
stage.exact_fit stage.one_word_over stage.slice_over_cap stage.head1 stage.headA1 stage.leading_run_cut
stage.beyond_maxl stage.all_staged
fast.warp fast.pair fast.pair_n_3P fast.pair_refused_ratio fast.pair_refused_n_eq_4P fast.pair_refused_n_gt_4P
fast.rows_x1 fast.rows_x1.all_rows fast.g3 fast.g2 fast.g1 fast.ladder_fallback fast.repack
fast.empty_slice.g0 fast.empty_slice.g1 fast.empty_slice.g2 fast.empty_slice.rows
diff.fast.empty_slice.g0 diff.fast.empty_slice.rows
fast.x_below_slice fast.x_above_slice fast.pair_l2_ge_10
fast.hit_low_0 fast.hit_low_ffffffff fast.live_64_33_32_0
tile.straddle_2^32 tile.last_alone_crosses tile.first_alone_below tile.starts_on_new_upper_word tile.holds_2^64-1
wide.dup_warp wide.mixed_tile wide.staged_rows wide.staged_one wide.row_g2 wide.row_g3 wide.hbm_list
wide.hbm_list_beyond_maxl wide.empty_slice
dup.rank dup.run_from_prev_tile dup.rank_past_slice dup.rank_past_list
sample.taken sample.alive_eq_threshold sample.alive_one_below_threshold sample.defer sample.defer_j1
sample.defer_later sample.defer_last_split sample.nj_full sample.nj_capped sample.lenA_one_below_min sample.lenA_at_min
tail.ran tail.mid_off_on_chunk_edge tail.leading_empty tail.trailing_empty tail.dup_rank tail.rank_drops_copy
{' '.join(f"fast.{path}.{e}" for path in ("pair", "group") for e in WINDOW_EVENTS)}
""".split())
