"""The host model of the radix sort and of the ops built on it (tests/radix_geometry.py), on the CPU: the constants and
the matched statements parse and a rewritten one is an error; every fixture of tests/test_gpu_radix_edges.py reaches
the events it names, the fixtures together reach every registered event and each one reaches one no other does; the
model equals the line-by-line restatements (groupby_oracle.c, valvar_oracle.c) on every fixture and on seeded random
cases, and its launches equal the plan models'.  Each named mutant of the model differs from the oracle on the
fixtures aimed at it: that is what shows the GPU test would catch the slip.  A fixture that drifts off its edge fails
here, before any GPU run."""
import functools
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen_groupby as gg  # noqa: E402
import gen_valvar as gv  # noqa: E402
import groupby_plan as gp  # noqa: E402
import radix_geometry as rg  # noqa: E402
import valvar_plan as vp  # noqa: E402

FIXTURES = {f.name: f for f in rg.all_fixtures()}


@functools.lru_cache(maxsize=None)
def run(name, mut=frozenset()):
    return rg.outcomes(FIXTURES[name], mut)


@functools.lru_cache(maxsize=None)
def want(name):
    """The oracle's outputs: groupby (keys, grp_off, mem_off, members); per value array (and function) (keys, words)."""
    f = FIXTURES[name]
    if isinstance(f, rg.GbFix):
        return rg.gb_oracle(f)
    if isinstance(f, rg.VvFix):
        return [rg.vv_oracle(f, x) for x in f.vals]
    return [[rg.la_oracle(f, x, fn) for fn in f.fns] for x in f.vals]


def results(name, outs):
    """The outputs of the fixture's first call (host form, exact room) as comparable tuples."""
    f, o = FIXTURES[name], outs[0]
    if isinstance(f, rg.GbFix):
        return [(o.keys, o.grp_off, o.mem_off, o.members)]
    if isinstance(f, rg.VvFix):
        return [(x.keys, x.vals) for x in o]
    return [(y.keys, y.vals) for x in o for y in x]


def wanted(name):
    w, f = want(name), FIXTURES[name]
    if isinstance(f, rg.GbFix):
        return [w]
    if isinstance(f, rg.VvFix):
        return w
    return [y for x in w for y in x]


def same(got, exp):
    return all(a is not None and np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(got, exp))


def test_constants():
    K = rg.K
    assert (K["GB_NT"], K["GB_VT"], K["RADIX"], K["DIGIT_BITS"], K["EN_TILE"]) == (256, 8, 256, 8, 2048)
    assert (K["VV_RANGES"], K["RANGE_BITS"], K["kVvTickets"], K["GB_TICKETS"]) == (4, 2, 8, 32)
    assert (K["SORT_PER_PASS"], K["FRONT"], K["BACK"], K["LEVEL"], K["AGG"]) == (3, 3, 8, 9, 4)
    # the largest pass counts fit the tickets: a level takes 2 + P, groupby 3 + P1 + P2
    assert 2 + rg.npasses(32 + rg.RB) <= K["kVvTickets"] and 3 + 2 * rg.npasses(64) <= K["GB_TICKETS"]


def _rewrite(text, func, pat):
    """The first space of the statement's match inside its function doubled: the same code, no longer the restated
    text."""
    body = rg._fn(func, text)
    s = re.search(pat, body).group(0)
    return text.replace(body, body.replace(s, s.replace(" ", "  ", 1), 1), 1)


@pytest.mark.parametrize("fn, func, pat, what", rg.STATEMENTS, ids=[s[3] for s in rg.STATEMENTS])
def test_a_rewritten_statement_fails(monkeypatch, fn, func, pat, what):
    real = rg._src
    assert re.search(pat, real(fn)), what
    monkeypatch.setattr(rg, "_src", lambda f: _rewrite(real(f), func, pat) if f == fn else real(f))
    with pytest.raises(ValueError, match=re.escape(f"{what} changed: restate it in the radix model")):
        rg.read_constants()


@pytest.mark.parametrize("fn, what, to, err", [
    ("dgx_api.cu", "constexpr size_t kVvTickets = 8;", "constexpr size_t kVvTickets = 2 * 4;", "kVvTickets"),
    ("encode_kernel.cuh", "EN_TILE = EN_NT * EN_VT;", "EN_TILE = EN_VT * EN_NT;", "EN_TILE"),
    ("valvar_kernel.cuh", "VV_RANGES = 4, VV_RANGE_BITS = 2;", "VV_RANGES = 4, VV_RBITS = 2;", "the range bits"),
    ("groupby_kernel.cuh", "GB_RADIX = 256, GB_DIGIT_BITS = 8;", "GB_RADIX = 256, GB_BITS = 8;", "the radix digit"),
])
def test_a_rewritten_constant_fails(monkeypatch, fn, what, to, err):
    real = rg._src
    assert what in real(fn)
    monkeypatch.setattr(rg, "_src", lambda f: real(f).replace(what, to) if f == fn else real(f))
    with pytest.raises(ValueError, match=re.escape(err)):
        rg.read_constants()


@pytest.mark.parametrize("name", list(FIXTURES))
def test_fixture_reaches_its_events(name):
    missing = FIXTURES[name].events - run(name)[1]
    assert not missing, f"{name}: does not reach {sorted(missing)}"


def test_every_event_is_reached():
    reached = set().union(*(run(n)[1] for n in FIXTURES))
    assert not rg.EVENTS - reached, f"no fixture reaches {sorted(rg.EVENTS - reached)}"


def test_every_fixture_is_needed():
    """Each fixture reaches an event no other fixture reaches: deleting any one leaves an event unreached."""
    for name in FIXTURES:
        others = set().union(*(run(n)[1] for n in FIXTURES if n != name))
        assert run(name)[1] - others, f"{name}: every event it reaches is reached by another fixture"


def test_a_sort_without_a_pass_reaches_no_sort_edge():
    """gb_sort launches nothing at key width 0, so 4 096 items over 9 tiles reach no size, tile or hist-scan event."""
    ev = set()
    s = rg.radix_sort(np.zeros(4096, np.uint64), np.arange(4096, dtype=np.uint32), 9, 0, ev)
    assert ev == {"sort: no pass (key width 0)"} and s.launches == 0 and s.passes == 0


def test_every_event_name_in_the_model_is_registered():
    src = open(rg.__file__).read()
    assert len(re.findall(r"\bev\.add\(", src)) == 1, "events are recorded through _add only"
    for is_f, text in re.findall(r"_add\(ev, (f?)\"([^\"]*)\"", src):
        if not is_f:
            assert text in rg.EVENTS, f"{text!r} is recorded but not registered"
            continue
        pat = "".join(".+" if i % 2 else re.escape(part) for i, part in enumerate(re.split(r"[{}]", text)))
        assert any(re.fullmatch(pat, e) for e in rg.EVENTS), f"f-string {text!r} matches no registered event"
    for text in re.findall(r"\"((?:sort|gb|vv|int|la): [^\"]*)\"", src):
        if "{" not in text:
            assert text in rg.EVENTS, f"{text!r} is named in the model but not registered"


@pytest.mark.parametrize("name", list(FIXTURES))
def test_model_equals_oracle(name):
    """Every call of the fixture: DGX_OK calls give the oracle's outputs, over-capacity calls only the sizes."""
    f = FIXTURES[name]
    exp = wanted(name)
    for c, o in zip(f.calls, run(name)[0]):
        flat = [o] if isinstance(f, rg.GbFix) else o if isinstance(f, rg.VvFix) else [y for x in o for y in x]
        for got, w in zip(flat, exp):
            if got.sync != rg.OK:
                assert got.sync == rg.ERR_CAP and got.keys is None, (name, c)
                continue
            if isinstance(f, rg.GbFix):
                assert (got.G, got.E) == (w[0].size, w[3].size), (name, c)
                res = (got.keys, got.grp_off, got.mem_off) + ((got.members,) if c.members else ())
                assert same(res, w[:3] + ((w[3],) if c.members else ())), (name, c)
            else:
                assert got.n == w[0].size and same((got.keys, got.vals), w), (name, c)


@pytest.mark.parametrize("name", list(FIXTURES))
def test_launches_match_the_plans(name):
    f = FIXTURES[name]
    for c, o in zip(f.calls, run(name)[0]):
        if isinstance(f, rg.GbFix):
            E = int(rg.gb_edges(f.src, f.v, f.v_off, f.par, f.par_off)[1].size) if f.v_off.size > 1 else 0
            assert o.launches == gp.launches(f.v_off.size - 1, f.dest.size, f.par_off.size - 1, int(f.v_off[-1]),
                                             int(f.par_off[-1]), E, c.form == "dev"), (name, c)
        elif isinstance(f, rg.VvFix):
            for x in o:
                assert x.launches == vp.propagate_launches(f.keys.size, [L.dest.size for L in f.levels]), (name, c)
                assert x.launches == sum(s.launches for s in x.sorts) + rg.K["LEVEL"] * len(f.levels)
        else:
            vals = int(f.v_off[-1]) if c.form == "host" or c.v_cap is None else c.v_cap
            for y in (y for x in o for y in x):
                assert y.launches == vp.level_agg_launches(f.keys.size, f.v_off.size - 1, vals), (name, c)


def test_every_mutant_is_aimed_at():
    named = set().union(*(f.kills for f in FIXTURES.values()))
    assert named == set(rg.MUTANTS), f"no fixture kills {sorted(set(rg.MUTANTS) - named)}"


@pytest.mark.parametrize("name, mutant", [(n, m) for n, f in FIXTURES.items() for m in sorted(f.kills)])
def test_the_mutant_differs_from_the_oracle(name, mutant):
    """The model with one slip gives a different output on the fixture aimed at it (host form, exact room)."""
    f = FIXTURES[name]
    outs = rg.outcomes(f._replace(calls=f.calls[:1]), frozenset([mutant]))[0]
    got, exp = results(name, outs), wanted(name)
    assert not all(same(g, w) for g, w in zip(got, exp)), f"{name}: the mutant {mutant!r} gives the oracle's output"


def test_model_random_groupby():
    """gen_groupby's cases at every kind, and wider ones over several tiles: the model is the oracle."""
    rng = np.random.default_rng(9400)
    for it in range(120):
        kind = ["small", "high", "mixed", "hub"][it % 4]
        if it % 10 == 9:
            parents, src, rows, dest = gg.case(rng, kind, nrows=int(rng.integers(500, 3000)), npar=3, nd=400)
        else:
            parents, src, rows, dest = gg.case(rng, kind)
        f = rg._gb(f"random {it}", parents, src, rows, dest, set())
        w = rg.gb_oracle(f)
        for c in (rg.GbCall("host", True, None), rg.GbCall("dev", True, None)):
            o = rg.groupby(f, c)
            assert o.G == w[0].size and same((o.keys, o.grp_off, o.mem_off, o.members), w), (it, c)


def test_model_random_paths():
    """gen_valvar's paths, int and float maps: the model's propagation and aggregation are the oracle's."""
    rng = np.random.default_rng(9500)
    for it in range(60):
        lv = gv.path(rng, int(rng.integers(1, 4)), int(rng.integers(1, 80)), hi=int(rng.integers(3, 3000)),
                     avg_deg=float(rng.uniform(0.5, 40)), unordered=bool(rng.integers(2)), repeats=bool(rng.integers(2)))
        levels = [rg._lv(s, r, d) for s, r, d in lv]
        for kind in ("int", "wild", "dyadic"):
            k, v = gv.value_map(rng, lv[0][0], rng.random(), kind)
            f = rg.VvFix("random", rg._u(k), (v,), tuple(levels), (), set(), set())
            o = rg.propagate(f, v.view(np.uint64), v.dtype == np.float64, rg.VV_DEFAULT[0])
            assert same((o.keys, o.vals), rg.vv_oracle(f, v)), (it, kind)
            s, r, d = lv[-1]
            k2, v2 = gv.value_map(rng, d if d.size else s, rng.random(), kind)
            a = rg._la("random", k2, (v2,), s, r, set())
            for fn in rg.FNS:
                o = rg.level_agg(a, v2.view(np.uint64), v2.dtype == np.float64, fn, rg.LA_DEFAULT[0])
                assert same((o.keys, o.vals), rg.la_oracle(a, v2, fn)), (it, kind, fn)
