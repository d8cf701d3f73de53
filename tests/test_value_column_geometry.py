"""The value-column model (tests/value_column_geometry.py) on the CPU: every event reached and every fixture needed,
the model equal to the restatements (match_oracle.c, regex_oracle.py, compare_oracle.c) on every fixture and on
seeded random cases, the launch counts, every mutant killed by the fixtures that name it, a rewritten statement
refused, and rx_load's read set inside the column at every alignment."""
import functools
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import value_column_geometry as vg  # noqa: E402

SMS = vg.H100_SMS


@functools.lru_cache(maxsize=None)
def fixtures():
    return {f.name: f for f in vg.fixtures(SMS)}


@functools.lru_cache(maxsize=None)
def model(name, form, mut=None):
    return vg.run(fixtures()[name], form, SMS, mut)


def _algo():
    from dgraph_b200 import algo

    return algo


def str_col(case):
    return _algo().StrColumn(case["uids"], case["values"])


def val_col(case):
    algo = _algo()
    bad = case.get("bad")
    return algo.ValColumn(case.get("typ", vg.T_STR), case["uids"], case["values"], bad)


def _nc(case, form):
    word = case.get("word") if form == "lane" else None
    n = len(case["cands"])
    raw = n if word is None else word & 0xFFFFFFFF
    return raw if raw <= n else 0


def oracle(case, form):
    """The restatements' answer to one fixture call, in the model's result shape."""
    import compare_oracle as co
    import match_oracle as mo
    import regex_oracle as ro

    kind = case["kind"]
    if kind == "rows":
        col = val_col(case)
        out = []
        for op, args in case["calls"]:
            rows = co.compare_rows(col, op, args, case["rows"], case["row_arg"])
            off = [0]
            for r in rows:
                off.append(off[-1] + len(r))
            out.append(("ok", tuple(off), tuple(int(x) for r in rows for x in r)))
        return tuple(out)
    cands = np.asarray(case["cands"], np.uint64)[:_nc(case, form)]
    if kind == "match":
        return (("ok", [int(x) for x in mo.match(str_col(case), case["query"], case["max"], uids=cands)], None),)
    if kind == "regex":
        col = str_col(case)
        if col.bytes.size > 200_000:
            want = by_re(col, case["pattern"], cands)
        else:
            want = ro.regex_match(col, ro.Prog(case["pattern"], case.get("fold", False)), cands)
        return (("ok", [int(x) for x in want], None),)
    col = val_col(case)
    out = []
    ccap = len(case["cands"])
    for op, args in case["calls"]:
        r = co.compare_uids(col, op, args, cands)
        if r is None:
            out.append(("refused",))
            continue
        counts = [int(c) for c in r[1][:cands.size]] + [None] * (ccap - cands.size)
        out.append(("ok", [int(x) for x in r[0]], tuple(counts)))
    return tuple(out)


def by_re(col, pat, cands):
    """matchRegex for an ASCII pattern over values without '\\n', by Python's re: the large fixtures' checker."""
    rx = re.compile(pat.encode())
    pos = {int(u): i for i, u in enumerate(col.uid)}
    data, bo, vo = col.bytes.tobytes(), col.byte_off, col.val_off
    out = []
    for u in cands:
        i = pos.get(int(u))
        if i is not None and any(bo[j + 1] > bo[j] and rx.search(data[int(bo[j]):int(bo[j + 1])])
                                 for j in range(int(vo[i]), int(vo[i + 1]))):
            out.append(int(u))
    return out


REFUSING = {"fe.refuse_count_word", "fe.col_refuse_past_ccap", "fe.byte_refuse_last_value",
            "fe.cand_refuse_last_thread", "cmp.bad_only_in_later_stride", "idx.refused"}


def test_statements_pinned_and_launches():
    vg.check_sources()
    assert vg.LAUNCHES == {"match": 5, "regex": 5, "cmp": 5, "rows": 4}


@pytest.mark.parametrize("fn,old,new", [
    ("regex_kernel.cuh", "if (g * 16 >= sp.clo && g * 16 + 16 <= sp.chi) return __ldg(sp.seg + g);",
     "if (g * 16 + 16 <= sp.chi) return __ldg(sp.seg + g);"),
    ("regex_kernel.cuh", "constexpr u64 RX_LONG_BYTES = 4096;", "constexpr u64 RX_LONG_BYTES = 4095;"),
    ("match_kernel.cuh", "const u32 owner = (W - 1) & 31;", "const u32 owner = (W - 1) >> 5;"),
    ("compare_kernel.cuh", "if (P.counts && t < F.words[FZ_W_N]) P.counts[t] = P.hits[t];",
     "if (P.counts) P.counts[t] = P.hits[t];"),
    ("dgx_api.cu", "rx_long_kernel<<<(unsigned)(2 * g_num_sms), RX_NT, 0, l->stream>>>(P);",
     "rx_long_kernel<<<(unsigned)(4 * g_num_sms), RX_NT, 0, l->stream>>>(P);"),
])
def test_rewrite_refused(fn, old, new):
    text = vg._src(fn)
    assert text.count(old) == 1
    with pytest.raises(ValueError, match="restate it in the value-column model"):
        vg.check_sources({fn: text.replace(old, new)})


def test_events_reached_and_fixtures_needed():
    fx = fixtures()
    reached = {}
    for name, f in fx.items():
        evs = set()
        for form in vg.forms(f.case):
            r, ev, oob = model(name, form)
            assert r[0] != "fault" and not oob, name
            evs |= ev
        assert f.events <= evs, (name, f.events - evs)
        assert set(f.kills) <= set(vg.MUTANTS), name
        reached[name] = evs
    allev = set().union(*reached.values())
    assert allev == vg.EVENTS, sorted(vg.EVENTS - allev)
    for name, evs in reached.items():
        others = set().union(*(e for n, e in reached.items() if n != name))
        assert evs - others, f"{name} reaches no event another fixture does not"


def test_model_equals_oracles_on_fixtures():
    for name, f in fixtures().items():
        for form in vg.forms(f.case):
            r, _, _ = model(name, form)
            if f.events & REFUSING:
                assert all(x[0] == "refused" for x in r), (name, form)
                continue
            if "broken" in f.case:
                continue
            assert r == oracle(f.case, form), (name, form)


def test_mutants_killed():
    killed = set()
    for name, f in fixtures().items():
        for mut in f.kills:
            diff = False
            for form in vg.forms(f.case):
                r0 = model(name, form)
                r1 = model(name, form, mut)
                diff = diff or r1[0] != r0[0] or r1[2] != r0[2]
            assert diff, (name, mut)
            killed.add(mut)
    assert killed == set(vg.MUTANTS), sorted(set(vg.MUTANTS) - killed)


def test_first_segment_whole_is_a_read_past_the_column():
    # results cannot show it: the read-set invariant does
    r0, _, oob0 = model("align_rx_a_5", "lane")
    r1, _, oob1 = model("align_rx_a_5", "lane", "first segment whole")
    assert r0 == r1 and not oob0 and oob1


def test_table_patterns():
    for nt, pat in vg.TABLE_PATTERNS.items():
        _, _, _, ns, nc = vg.dfa(pat)
        assert ns * nc == nt
        assert vg.smem_plan(ns, nc)[0] == (nt <= vg.RX_SMEM_TABLE // 2)
    assert vg.TABLE_PATTERNS.keys() == {16383, 16384, 16385}


def test_smem_size_never_decides():
    # rx_run's `smem <= 48 * 1024`: with 2 nt <= RX_SMEM_TABLE and nstates <= 4096 (DGX_REGEX_MAX_STATES) it holds
    worst = 0
    for ns in range(1, 4097):
        nc = min(256, vg.RX_SMEM_TABLE // (2 * ns))
        if nc == 0:
            continue
        ok, table_fits, smem = vg.smem_plan(ns, nc)
        assert table_fits and ok
        worst = max(worst, smem)
    assert worst <= 48 * 1024


def test_warp_tier_threshold_is_invisible():
    # the thread tier and the warp tier compute the same answer, so where the 4096-byte split lies cannot show
    rng = np.random.default_rng(5)
    for pat in ("needle", "^ab", "b$", "a.b"):
        cls, trans, term, ns, nc = vg.dfa(pat)
        D = vg.Dfa(cls, trans, term)
        for _ in range(40):
            ln = int(rng.integers(1, 700))
            data = bytes(rng.choice(np.frombuffer(b"needlab\nx", np.uint8), ln))
            clo = int(rng.integers(0, 16))
            rd = vg.Reader(data, clo)
            lo, hi = clo, clo + ln
            assert vg.rx_thread(vg.Events(), D, rd, lo, hi) == vg.rx_warp(vg.Events(), D, rd, lo, hi, None) == \
                vg.plain_walk(D, rd, lo, hi)
            assert not rd.oob


@pytest.mark.parametrize("kind", ["thread", "warp", "cmp"])
def test_read_set_every_alignment(kind):
    """rx_load's loads for every column base offset 0-15, column size 0-80 and value inside: every byte read lies in
    the column, and a segment takes the byte path exactly when part of it lies outside."""
    for whole_first, want_ok in ((False, True), (True, False)):
        ok = True
        for clo in range(16):
            for nbytes in range(81):
                chi = clo + nbytes
                for b0 in range(nbytes):
                    for ln in range(1, nbytes - b0 + 1):
                        lo, hi = clo + b0, clo + b0 + ln
                        segs = vg.segs_read(clo, nbytes, lo, hi, kind, alen=ln if kind == "cmp" else None)
                        if kind == "warp":
                            assert sorted(segs) == list(vg.segs_read(clo, nbytes, lo, hi, "thread"))
                        for g in segs:
                            a, b, whole = vg.rx_load(clo, chi, g, whole_first)
                            inside = a >= clo and b <= chi
                            if whole_first:
                                ok = ok and inside
                                continue
                            assert inside, (clo, nbytes, b0, ln, g)
                            assert whole == (g * 16 >= clo and g * 16 + 16 <= chi)
                            assert a <= max(lo, g * 16) and b >= min(hi, g * 16 + 16)
            if whole_first and not ok:
                break
        assert ok == want_ok


def test_cmp_bytes_reads_the_argument_below_its_length():
    class Arg(bytes):
        def __getitem__(self, i):
            assert 0 <= i < len(self)
            return bytes.__getitem__(self, i)

    rng = np.random.default_rng(9)
    for _ in range(3000):
        data = bytes(rng.choice(np.frombuffer(b"ab", np.uint8), int(rng.integers(0, 60))))
        clo = int(rng.integers(0, 16))
        b0 = int(rng.integers(0, len(data) + 1))
        ln = int(rng.integers(0, len(data) - b0 + 1))
        a = Arg(bytes(rng.choice(np.frombuffer(b"ab", np.uint8), int(rng.integers(0, 40)))))
        rd = vg.Reader(data, clo)
        C = vg.Cmp(vg.Events(), vg.T_STR, "le", [(0, 0, a)], rd, None)
        v = data[b0:b0 + ln]
        assert C.cmp_bytes(clo + b0, clo + b0 + ln, a) == (v > a) - (v < a)
        assert not rd.oob


# ---------------------------------------------------------------------------------------------------------------
# seeded random cases
PATTERNS = ["ab", "^a", "b$", "a.b", "[ab]x", "x|é", "a+b", "(?i)AB", "^$", "a\\nb"]


def _random_case(rng, kind):
    n = int(rng.integers(0, 10))
    uids = sorted(rng.choice(np.arange(1, 40), n, replace=False).tolist())
    alpha = np.frombuffer(b"ab\nx\xc3\xa9", np.uint8)
    if kind in ("match", "regex") or rng.random() < 0.4:
        typ = vg.T_STR
        values = [[bytes(rng.choice(alpha, int(rng.integers(0, 40)))) for _ in range(int(rng.integers(0, 3)))]
                  for _ in uids]
        if kind == "regex" and uids and rng.random() < 0.1:
            values[0].append(bytes(rng.choice(alpha, int(rng.integers(4090, 4200)))))
    else:
        typ = int(rng.choice([vg.T_INT, vg.T_FLOAT]))
        pool = [-3, 0, 2, 7] if typ == vg.T_INT else [-1.5, -0.0, 0.0, 2.0, float("nan")]
        values = [[pool[int(rng.integers(0, len(pool)))] for _ in range(int(rng.integers(0, 3)))] for _ in uids]
    cands = sorted(set(rng.choice(np.arange(1, 42), int(rng.integers(0, 12))).tolist()))
    case = dict(kind=kind, typ=typ, uids=uids, values=values, cands=cands, shift=int(rng.integers(0, 16)))
    if cands and rng.random() < 0.3:
        case["word"] = int(rng.integers(0, len(cands) + 1)) | (int(rng.integers(0, 4)) << 32)
        case["cands"] = cands + sorted(rng.choice(np.arange(1, 42), int(rng.integers(0, 4))).tolist(), reverse=True)
    if kind == "match":
        case["query"] = bytes(rng.choice(alpha, int(rng.choice([int(rng.integers(0, 8)), 70]))))
        case["max"] = int(rng.integers(0, 4))
    elif kind == "regex":
        case["pattern"] = PATTERNS[int(rng.integers(0, len(PATTERNS)))]
    else:
        if typ == vg.T_STR:
            args = [bytes(rng.choice(alpha, int(rng.integers(0, 6)))) for _ in range(3)]
        else:
            args = [pool[int(rng.integers(0, len(pool)))] for _ in range(3)]
        op = ["le", "ge", "lt", "gt", "eq", "between"][int(rng.integers(0, 6))]
        case["calls"] = [(op, args[:2] if op == "between" else args if op == "eq" else args[:1])]
        if kind == "rows":
            rows = [sorted(rng.choice(np.arange(1, 42), int(rng.integers(0, 6))).tolist()) for _ in
                    range(int(rng.integers(1, 5)))]
            case["rows"] = rows
            case["row_arg"] = [vg.NO_ARG if rng.random() < 0.3 else 0 for _ in rows]
            case.pop("word", None)
    return case


@pytest.mark.parametrize("kind,count", [("match", 1500), ("regex", 1000), ("cmp", 1500), ("rows", 800)])
def test_model_equals_oracles_on_random_cases(kind, count):
    for seed in range(count):
        rng = np.random.default_rng(9_100_000 + 10_000 * ["match", "regex", "cmp", "rows"].index(kind) + seed)
        case = _random_case(rng, kind)
        f = vg.Fixture(f"random {kind} {seed}", case, frozenset(), frozenset())
        for form in vg.forms(case):
            r, _, oob = vg.run(f, form, SMS)
            assert not oob, (kind, seed)
            assert r == oracle(case, form), (kind, seed, form)
