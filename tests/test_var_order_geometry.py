"""The host model of orderasc / orderdesc by a value variable (tests/var_order_geometry.py), on the CPU: the constants
and the matched statements parse and a rewritten one is an error; every fixture of tests/test_gpu_var_order_edges.py
reaches the events it names, the fixtures together reach every registered event and each one reaches one no other
does; the model equals the line-by-line restatement (var_order_oracle.c) on every fixture and on seeded random cases,
and its launches equal the plan model's; the cooperative partition equals Go's sequential Hoare loop; the split and
the tiers are invisible where the design says they are.  Each named mutant of the model differs from the restatement
on the fixtures aimed at it: that is what shows the GPU test would catch the slip.  A fixture that drifts off its edge
fails here, before any GPU run."""
import functools
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen_var_order as gv  # noqa: E402
import var_order_geometry as vg  # noqa: E402
import var_order_oracle as vo  # noqa: E402
import var_order_plan as vp  # noqa: E402

FIXTURES = {f.name: f for f in vg.fixtures()}
OTHER_SMS = 78   # a grid of another size: the 2*SMs fixtures move with it


@functools.lru_cache(maxsize=None)
def run(name):
    return vg.outcomes(FIXTURES[name])


@functools.lru_cache(maxsize=None)
def want(name):
    """The restatement's (rows, dest), or None for a refused call."""
    f = FIXTURES[name]
    if f.mutate is not None:
        return None
    return vo.var_order(*f.case)


def same(out, exp):
    if exp is None:
        return bool(out.refused)
    if out.refused:
        return False
    return (len(out.rows) == len(exp[0]) and all(np.array_equal(a, b) for a, b in zip(out.rows, exp[0]))
            and np.array_equal(out.dest, exp[1]))


def test_constants():
    K = vg.K
    assert (K["MAX_INSERTION"], K["CTA_MIN"], K["NT"], K["STACK_THREAD"], K["STACK_CTA"]) == (12, 4096, 256, 13, 32)
    assert (K["KEY_PASSES"], K["GB_TILE"]) == (8, 2048)
    # the pdqsort stacks cover the rows they sort: floor(log2 n) frames at most
    assert (vg.CTA_MIN).bit_length() <= K["STACK_THREAD"] and 32 <= K["STACK_CTA"]


def _rewrite(text, func, pat):
    """The first space of the statement's match inside its function doubled: the same code, no longer the restated
    text."""
    body = vg._fn(func, text)
    s = re.search(pat, body).group(0)
    return text.replace(body, body.replace(s, s.replace(" ", "  ", 1), 1), 1)


@pytest.mark.parametrize("fn, func, pat, what", vg.STATEMENTS, ids=[s[3] for s in vg.STATEMENTS])
def test_a_rewritten_statement_fails(monkeypatch, fn, func, pat, what):
    real = vg._src
    assert re.search(pat, real(fn)), what
    monkeypatch.setattr(vg, "_src", lambda f: _rewrite(real(f), func, pat) if f == fn else real(f))
    with pytest.raises(ValueError, match=re.escape(f"{what} changed: restate it in the order-by-variable model")):
        vg.read_constants()


@pytest.mark.parametrize("what, to, err", [
    ("constexpr u64 VO_CTA_MIN = 4096;", "constexpr u64 VO_CTA_MIN = 4 * 1024;", "VO_CTA_MIN"),
    ("constexpr int VO_NT = 256;", "constexpr int VO_NT = 2 * 128;", "VO_NT"),
    ("constexpr long VO_MAX_INSERTION = 12;", "constexpr long VO_MAX_INSERTION = 6 * 2;", "VO_MAX_INSERTION"),
])
def test_a_rewritten_constant_fails(monkeypatch, what, to, err):
    real = vg._src
    assert what in real(vg.K_FILE)
    monkeypatch.setattr(vg, "_src", lambda f: real(f).replace(what, to) if f == vg.K_FILE else real(f))
    with pytest.raises(ValueError, match=re.escape(err)):
        vg.read_constants()


@pytest.mark.parametrize("name", list(FIXTURES))
def test_fixture_reaches_its_events(name):
    missing = FIXTURES[name].events - run(name)[1]
    assert not missing, f"{name}: does not reach {sorted(missing)}"


def test_every_event_is_reached():
    reached = set().union(*(run(n)[1] for n in FIXTURES))
    assert not vg.EVENTS - reached, f"no fixture reaches {sorted(vg.EVENTS - reached)}"


def test_every_fixture_is_needed():
    """Each fixture reaches an event no other fixture reaches: deleting any one leaves an event unreached."""
    for name in FIXTURES:
        others = set().union(*(run(n)[1] for n in FIXTURES if n != name))
        assert run(name)[1] - others, f"{name}: every event it reaches is reached by another fixture"


def test_every_event_name_in_the_model_is_registered():
    src = open(vg.__file__).read()
    assert len(re.findall(r"\bev\.add\(", src)) == 1, "events are recorded through _add only"
    for is_f, text in re.findall(r"_add\(ev, (f?)\"([^\"]*)\"", src):
        if not is_f:
            assert text in vg.EVENTS, f"{text!r} is recorded but not registered"
            continue
        pat = "".join(".+" if i % 2 else re.escape(part) for i, part in enumerate(re.split(r"[{}]", text)))
        assert any(re.fullmatch(pat, e) for e in vg.EVENTS), f"f-string {text!r} matches no registered event"


def test_a_fixture_moved_off_its_edge_fails():
    """The 4 097-entry row shrunk to 4 096 runs on a thread: the CTA event is gone.  The same for a tied row of 13
    shrunk to 12, and for 2*SMs + 1 long rows on a grid one SM larger."""
    ev = set()
    vg.run(vg.grid_rows(1, 1, vg.CTA_MIN), ev=ev)
    assert "split: a CTA row of 4097" not in ev and "split: a thread row of 4096" in ev
    f = FIXTURES["tiers: tied rows of 12 and 13"]
    m, desc, dest, rows, c, o = f.case
    ev = set()
    vg.run((m, desc, dest, [rows[0], rows[1][:12]], c, o), ev=ev)
    assert "tier: tied row of 13 (tier 2)" not in ev
    ev = set()
    vg.run(FIXTURES["split: 2*SMs + 1 long rows"].case, sms=vg.H100_SMS + 1, ev=ev)
    assert "split: a CTA pulls a second row" not in ev


@pytest.mark.parametrize("name", list(FIXTURES))
def test_model_equals_oracle(name):
    """Every call of the fixture (host form, device form with and without slack and length words)."""
    for c, o in zip(FIXTURES[name].calls, run(name)[0]):
        assert same(o, want(name)), (name, c)


@pytest.mark.parametrize("name", list(FIXTURES))
def test_launches_match_the_plan(name):
    f = FIXTURES[name]
    for c, o in zip(f.calls, run(name)[0]):
        dest_room = len(f.case[2]) + (c.slack if c.form == "dev" and c.words else 0)
        assert o.launches == vp.launches(dest_room, len(f.case[3])), (name, c)


def test_grid_fixtures_follow_the_sm_count():
    """The model takes the SM count: on a 78-SM part the 2*SMs fixtures hold 155, 156 and 157 long rows and reach
    the same split events."""
    for f in vg.fixtures(OTHER_SMS):
        if "2*SMs" not in f.name:
            continue
        nlong = sum(len(r) > vg.CTA_MIN for r in f.case[3])
        assert nlong in (2 * OTHER_SMS - 1, 2 * OTHER_SMS, 2 * OTHER_SMS + 1) and len(f.case[3]) == 2 * nlong
        ev = set()
        vg.run(f.case, sms=OTHER_SMS, ev=ev)
        assert f.events <= ev, f.name


def test_model_random_cases():
    """gen_var_order's random cases, 2 000 of them, through the host form and the device form with slack and length
    words: the model is the restatement."""
    rng = np.random.default_rng(1600)
    for it in range(2000):
        case = gv.random_case(rng)
        if case[0] is None:
            continue
        try:
            exp = vo.var_order(*case)
        except vo.NotSortable:
            exp = None
        call = vg.DEV_SLACK if it & 1 else vg.HOST
        assert same(vg.run(case, call), exp), it


def _range(rng, n):
    kind = rng.integers(0, 6)
    if kind == 0:
        return [vg.entry(vg.T_INT, vg.iw(x), 0) for x in rng.integers(0, int(rng.integers(1, 40)), n)]
    if kind == 1:
        return [vg.entry(vg.T_FLOAT, vg.fw(x), 0) for x in
                np.where(rng.random(n) < 0.3, np.nan, rng.integers(0, 20, n).astype(np.float64))]
    if kind == 2:
        return [vg.entry(vg.T_NIL if rng.random() < 0.5 else vg.T_INT, int(rng.integers(0, 9)), 0) for _ in range(n)]
    if kind == 3:
        return [vg.entry(vg.T_BOOL if rng.random() < 0.2 else vg.T_INT, int(rng.integers(0, 2)), 0) for _ in range(n)]
    if kind == 4:
        t = rng.choice([vg.T_INT, vg.T_FLOAT, vg.T_NIL, vg.T_BOOL], n)
        return [vg.entry(int(x), vg.fw(float(rng.integers(0, 5))) if x == vg.T_FLOAT else int(rng.integers(0, 5)), 0)
                for x in t]
    return [vg.entry(vg.T_INT, vg.iw(x), 0) for x in rng.permutation(n)]


def test_cooperative_partition_is_the_hoare_loop():
    """On 1 000 random ranges, NaN, nils under desc, bools and mixed tags included, and on every partition the
    fixtures' CTA rows run: the chunked partition leaves the array, mid and alreadyPartitioned of Go's loop."""
    rng = np.random.default_rng(1601)
    for it in range(1000):
        n = int(rng.choice([13, 50, 257, 258, 513, 700, 1100]))
        es = [(t, w, v, i) for i, (t, w, v, _) in enumerate(_range(rng, n))]
        desc, eq = bool(rng.integers(2)), bool(rng.integers(2))
        a = int(rng.integers(0, 4))
        b = n - int(rng.integers(0, 4))
        p = int(rng.integers(a, b))
        seq, coop = vg.Row(es, desc, frozenset(), False), vg.Row(es, desc, frozenset(), True)
        for d in (seq, coop):
            d.swap(a, p)
        if eq:
            m_seq, already = vg.partition_equal_seq(seq, a, b), None
        else:
            m_seq, already = vg.partition_seq(seq, a, b)
        m_coop, npairs, _ = vg.partition_coop(coop, a, b, eq)
        assert m_seq == m_coop and seq.e == coop.e, it
        if not eq:
            assert already == (npairs == 0), it


def test_fixture_partitions_match_the_hoare_loop():
    """Every CTA row of every fixture sorted with the sequential partition on a thread gives the same row."""
    for name, f in FIXTURES.items():
        o = run(name)[0][0]
        if o.refused or not any(t == "cta" for t in o.tiers):
            continue
        o2 = vg.run(f.case, cta_min=1 << 31)
        assert same(o2, want(name)), name


@pytest.mark.parametrize("cta_min", [12, 256, 1 << 31])
def test_the_split_is_invisible(cta_min):
    """Moving VO_CTA_MIN leaves every fixture's output unchanged: both sides run Go's partition."""
    for name, f in FIXTURES.items():
        if f.mutate is not None or (cta_min == 12 and len(f.case[2]) > 100_000):
            continue
        assert same(vg.run(f.case, cta_min=cta_min), want(name)), name


def test_tier_1_on_distinct_keys_is_invisible():
    """Every MIXED-free row sent to tier 2 gives the same output: a tier-1 row's order is the only correct one."""
    for name, f in FIXTURES.items():
        if f.mutate is None:
            assert same(vg.run(f.case, tier2_all=True), want(name)), name


def test_tier_2_from_12_is_invisible():
    """Tier 2 at n >= 12 instead of n > 12 is no slip: a tied row of 12 runs insertionSort, stable like the radix."""
    rng = np.random.default_rng(1602)
    keys = np.arange(1, 13, dtype=np.uint64)
    for _ in range(200):
        case = (vg.imap(keys, rng.integers(0, 3, 12)), bool(rng.integers(2)), keys, [keys], 0, 0)
        assert same(vg.run(case, tier2_all=True), vo.var_order(*case))


def test_the_stack_bound():
    """The deepest frame stack of every fixture row and of random tied rows of 4 096 entries stays far below
    VO_STACK_THREAD / VO_STACK_CTA."""
    deepest = {"thread": 0, "cta": 0}
    for name in FIXTURES:
        for o in run(name)[0]:
            for r, (_, depth, _) in (o.rows_info or {}).items():
                deepest[o.tiers[r]] = max(deepest[o.tiers[r]], depth)
    rng = np.random.default_rng(1603)
    keys = np.arange(1, vg.CTA_MIN + 1, dtype=np.uint64)
    for _ in range(20):
        case = (vg.imap(keys, rng.integers(0, int(rng.integers(2, 4000)), keys.size)), False, keys, [keys], 0, 0)
        o = vg.run(case)
        deepest["thread"] = max(deepest["thread"], o.rows_info[0][1])
    assert deepest["thread"] >= 7 and deepest["cta"] >= 8
    assert deepest["thread"] < vg.K["STACK_THREAD"] and deepest["cta"] < vg.K["STACK_CTA"], deepest


def test_every_mutant_is_aimed_at():
    named = set().union(*(f.kills for f in FIXTURES.values()))
    assert named == set(vg.MUTANTS), f"no fixture kills {sorted(set(vg.MUTANTS) - named)}"


@pytest.mark.parametrize("name, mutant", [(n, m) for n, f in FIXTURES.items() for m in sorted(f.kills)])
def test_the_mutant_differs_from_the_oracle(name, mutant):
    """The model with one slip gives a different output on the fixture aimed at it (host form)."""
    f = FIXTURES[name]
    o = vg.run(f.case, vg.HOST, mut=frozenset([mutant]), mutate=f.mutate)
    assert not same(o, want(name)), f"{name}: the mutant {mutant!r} gives the restatement's output"
