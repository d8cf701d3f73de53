"""The host model of regexp()'s and math()'s tree evaluators (tests/tree_geometry.py), on the CPU: the constants and the
matched statements parse and a rewritten one is an error; every fixture of tests/test_gpu_tree_edges.py reaches the
events it names, the fixtures together reach every registered event and each one reaches one no other does; the model
equals the restatements (trigram_oracle.c and gen_trigram's set formula, math_oracle.c and gen_math's formula) on
every fixture and on seeded random cases, and its launches equal the plan models'.  Each named mutant of the model
differs from the oracle on the fixtures aimed at it: that is what shows the GPU test would catch the slip."""
import functools
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen_math as gm  # noqa: E402
import gen_trigram as gt  # noqa: E402
import math_plan as mp  # noqa: E402
import tree_geometry as tg  # noqa: E402
import trigram_plan as tp  # noqa: E402

FIXTURES = {f.name: f for f in tg.all_fixtures()}


@functools.lru_cache(maxsize=None)
def run(name, mut=frozenset()):
    return tg.outcomes(FIXTURES[name], mut)


@functools.lru_cache(maxsize=None)
def expected(name):
    """Per case and call: the oracle's answer in the model's terms."""
    f = FIXTURES[name]
    if isinstance(f, tg.TgFix):
        return [[tg.tg_expected(c, call) for call in f.calls] for c in f.cases]
    return [tg.mt_expected(c) for c in f.cases]


def agrees(name, outs):
    """Every call of the fixture gives the oracle's answer: return codes, sync codes and the values written."""
    f = FIXTURES[name]
    for k, (c, per) in enumerate(zip(f.cases, outs)):
        for call, o in zip(f.calls, per):
            if isinstance(f, tg.TgFix):
                rc, sync, vals = expected(name)[k][f.calls.index(call)]
                if (o.rc, o.sync) != (rc, sync):
                    return False
                if vals is not None and not (o.n == vals.size and np.array_equal(o.out, vals)):
                    return False
            elif not mt_agrees(expected(name)[k], c, call, o):
                return False
    return True


def mt_agrees(w, c, call, o):
    dev = call.form == "dev"
    if w is None:
        return (o.rc, o.sync, o.info, o.keys) == ((tg.OK, tg.ERR_ARG) if dev else (tg.ERR_ARG, None)) + (None, None)
    kind, k, words, tags = w
    n = k.size
    info = n | {"none": 0, "map": 1, "const": 2}[kind] << 32 | (
        int(np.bitwise_or.reduce(1 << tags.astype(np.int64))) if n else 0) << 40
    if o.info != info:
        return False
    if call.out_cap is not None and n > call.out_cap:
        return (o.rc, o.sync, o.keys) == ((tg.OK, tg.ERR_CAP) if dev else (tg.ERR_CAP, None)) + (None,)
    return (o.rc, o.sync) == ((tg.OK, tg.OK) if dev else (tg.OK, None)) and all(
        a is not None and np.array_equal(a, b) for a, b in ((o.keys, k), (o.words, words), (o.tags, tags)))


def test_constants():
    K = tg.K
    assert (K["TG_NT"], K["CP_NT"] * K["CP_VT"], K["EN_TILE"], K["GRID_NT"]) == (1024, 2048, 2048, 256)
    assert (K["MAX_NODES"], K["MAX_LEAVES"], K["TG_MAX_DEPTH"]) == (64, 16, 32)
    assert (K["TG_MAX_NODES"], K["TG_MAX_LEAVES"], K["TG_MAX_REFS"]) == (1 << 16, 1 << 16, 1 << 20)


def _rewrite(text, func, pat):
    """The first space of the statement's match doubled: the same code, no longer the restated text."""
    body = tg._fn(func, text) if func else text
    s = re.search(pat, body).group(0)
    return text.replace(body, body.replace(s, s.replace(" ", "  ", 1), 1), 1)


@pytest.mark.parametrize("fn, func, pat, what", tg.STATEMENTS, ids=[f"{s[1]}: {s[3]}" for s in tg.STATEMENTS])
def test_a_rewritten_statement_fails(monkeypatch, fn, func, pat, what):
    real = tg._src
    assert re.search(pat, real(fn)), what
    monkeypatch.setattr(tg, "_src", lambda f: _rewrite(real(f), func, pat) if f == fn else real(f))
    with pytest.raises(ValueError, match=re.escape("restate it in the tree model")):
        tg.read_constants()


@pytest.mark.parametrize("fn, what, to", [
    ("trigram_kernel.cuh", "constexpr int TG_NT = 1024;", "constexpr int TG_NT = 2 * 512;"),
    ("compressed_kernel.cuh", "CP_TILE = CP_NT * CP_VT;", "CP_TILE = CP_VT * CP_NT;"),
    ("encode_kernel.cuh", "EN_TILE = EN_NT * EN_VT;", "EN_TILE = EN_VT * EN_NT;"),
    ("dgx.h", "#define DGX_MATH_MAX_NODES 64", "#define DGX_MATH_MAX_NODES (32 * 2)"),
    ("math_kernel.cuh", "MT_MAX_NODES = 64, MT_MAX_LEAVES = 16;", "MT_MAX_NODES = 64, MT_MAX_LEAVES = 32;"),
    ("math_kernel.cuh", "__launch_bounds__(256) mt_write_kernel", "__launch_bounds__(512) mt_write_kernel"),
])
def test_a_rewritten_constant_fails(monkeypatch, fn, what, to):
    real = tg._src
    assert what in real(fn)
    monkeypatch.setattr(tg, "_src", lambda f: real(f).replace(what, to) if f == fn else real(f))
    with pytest.raises(ValueError, match=re.escape("restate it in the tree model")):
        tg.read_constants()


@pytest.mark.parametrize("name", list(FIXTURES))
def test_fixture_reaches_its_events(name):
    missing = FIXTURES[name].events - run(name)[1]
    assert not missing, f"{name}: does not reach {sorted(missing)}"


def test_every_event_is_reached():
    reached = set().union(*(run(n)[1] for n in FIXTURES))
    assert not tg.EVENTS - reached, f"no fixture reaches {sorted(tg.EVENTS - reached)}"


def test_every_fixture_is_needed():
    """Each fixture reaches an event no other fixture reaches: deleting any one leaves an event unreached."""
    for name in FIXTURES:
        others = set().union(*(run(n)[1] for n in FIXTURES if n != name))
        assert run(name)[1] - others, f"{name}: every event it reaches is reached by another fixture"


def test_every_event_name_in_the_model_is_registered():
    src = open(tg.__file__).read()
    assert len(re.findall(r"\bev\.add\(", src)) == 1, "events are recorded through _add only"
    for is_f, text in re.findall(r"_add\(ev, (f?)\"([^\"]*)\"", src):
        if not is_f:
            assert text in tg.EVENTS, f"{text!r} is recorded but not registered"
            continue
        pat = "".join(".+" if i % 2 else re.escape(part) for i, part in enumerate(re.split(r"[{}]", text)))
        assert any(re.fullmatch(pat, e) for e in tg.EVENTS), f"f-string {text!r} matches no registered event"
    for text in re.findall(r"\"((?:tg|mt) [a-z]+: [^\"]*)\"", src):
        if "{" not in text:
            assert text in tg.EVENTS, f"{text!r} is named in the model but not registered"


@pytest.mark.parametrize("name", [n for n, f in FIXTURES.items() if isinstance(f, tg.TgFix)])
def test_trigram_oracles_agree(name):
    """trigram_oracle.c (uidsForRegex line by line) and gen_trigram's set formula give one answer on every case."""
    for c in FIXTURES[name].cases:
        assert np.array_equal(tg.tg_oracle(c), gt.want(*c)), name


@pytest.mark.parametrize("name", [n for n, f in FIXTURES.items() if isinstance(f, tg.MtFix)])
def test_math_oracles_agree(name):
    """math_oracle.c (evalMathTree line by line) and gen_math's formula give one answer on every case."""
    for c in FIXTURES[name].cases:
        if tg.mt_malformed(c):
            continue
        w, g = tg.mt_expected(c), gm.formula(*c)
        assert (w is None) == (g is None), name
        if w is not None:
            assert w[0] == g[0] and all(np.array_equal(a, b) for a, b in zip(w[1:], g[1:])), name


@pytest.mark.parametrize("name", list(FIXTURES))
def test_model_equals_oracle(name):
    assert agrees(name, run(name)[0]), name


@pytest.mark.parametrize("name", list(FIXTURES))
def test_launches_match_the_plans(name):
    f = FIXTURES[name]
    for c, per in zip(f.cases, run(name)[0]):
        for call, o in zip(f.calls, per):
            if isinstance(f, tg.TgFix):
                npacks = tg.tg_npacks(c.leaves)
                lb = [gt.leaf_bound(lf) for lf in c.leaves]
                p = tp.plan(c.tree, lb, tg.tg_cap(tp.plan(c.tree, lb), call))
                if o.rc == tg.OK:
                    assert o.launches == tp.launches(p, npacks), (name, call)
                else:
                    assert o.launches == 0, (name, call)
            else:
                cap = sum(r[2] for r in tg.mt_room(c, call))
                dev_ran = call.form == "dev" or o.rc == tg.OK
                assert o.launches == (mp.launches(cap) if dev_ran else 0), (name, call)


def test_every_mutant_is_aimed_at():
    named = set().union(*(f.kills for f in FIXTURES.values()))
    assert named == set(tg.MUTANTS), f"no fixture kills {sorted(set(tg.MUTANTS) - named)}"


@pytest.mark.parametrize("name, mutant", [(n, m) for n, f in FIXTURES.items() for m in sorted(f.kills)])
def test_the_mutant_differs_from_the_oracle(name, mutant):
    """The model with one slip gives a different answer on the fixture aimed at it."""
    assert not agrees(name, run(name, frozenset([mutant]))[0]), f"{name}: the mutant {mutant!r} gives the oracle's output"


def test_model_random_trigram():
    """gen_trigram's random trees and leaves: the model is the oracle in both forms."""
    for seed in range(150):
        rng = np.random.default_rng(61_000 + seed)
        universe = int(rng.choice([300, 5000]))
        after = [0, universe // 2][seed % 2]
        nleaves = int(rng.integers(1, 12))
        leaves = gt.random_leaves(rng, nleaves, universe, str(rng.choice(["mixed", "probe", "iterate"])), after=after)
        order = [j for j, lf in enumerate(leaves) if lf[0] == "pack"] + [j for j, lf in enumerate(leaves)
                                                                         if lf[0] == "list"]
        ren = {j: k for k, j in enumerate(order)}
        tree = [(op, [ren[j] for j in ls], subs) for op, ls, subs in
                gt.random_tree(rng, nleaves, int(rng.integers(1, 10)), max_depth=int(rng.choice([2, 6, 32])))]
        case = tg.TgCase(tree, [leaves[j] for j in order], after)
        want = tg.tg_oracle(case)
        assert np.array_equal(want, gt.want(*case)), seed
        for call in tg.TG_DEFAULT:
            o = tg.tg_run(case, call)
            assert o.rc == tg.OK and o.n == want.size and np.array_equal(o.out, want), (seed, call)


def test_model_random_math():
    """gen_math's random programs: the model is the oracle (refusals included) in both forms."""
    rng = np.random.default_rng(62_000)
    refused = 0
    for it in range(300):
        case = tg.MtCase(*gm.case(rng, max_depth=5))
        w = tg.mt_expected(case)
        refused += w is None
        for call in tg.MT_DEFAULT:
            assert mt_agrees(w, case, call, tg.mt_run(case, call)), (it, call)
    assert refused > 0
