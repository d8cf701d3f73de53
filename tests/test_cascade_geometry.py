"""The host model of @cascade's level kernels and @filter's evaluator (tests/cascade_geometry.py), on the CPU: the
constants and the matched statements parse and a rewritten one is an error; every fixture of
tests/test_gpu_cascade_edges.py reaches the events it names, the fixtures together reach every registered event and
each one reaches one no other does; the model equals the restatements (cascade_oracle.c and gen_cascade's formula,
sg_filter_oracle.c and gen_sg_filter's formula) on every fixture and on seeded random cases, and its launches equal the
plan models'.  Each named mutant of the model differs from the oracle on the fixtures aimed at it: that is what shows
the GPU test would catch the slip."""
import functools
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import cascade_geometry as cg  # noqa: E402
import cascade_oracle as co  # noqa: E402
import cascade_plan as cp  # noqa: E402
import gen_cascade as gc  # noqa: E402
import gen_sg_filter as gs  # noqa: E402
import sg_filter_oracle as so  # noqa: E402
import sg_filter_plan as sp  # noqa: E402

FIXTURES = {f.name: f for f in cg.all_fixtures()}


@functools.lru_cache(maxsize=None)
def run(name, mut=frozenset()):
    return cg.outcomes(FIXTURES[name], mut)


@functools.lru_cache(maxsize=None)
def expected(name):
    """Per case and call: the oracle's answer in the model's terms."""
    f = FIXTURES[name]
    if isinstance(f, cg.CcFix):
        return [[cg.cc_expected(c, form) for form in c.forms] for c in f.cases]
    return [[cg.sf_expected(c, call) for call in f.calls] for c in f.cases]


def agrees(name, outs):
    """Every call of the fixture gives the oracle's answer: return codes, sync codes and the values written."""
    f = FIXTURES[name]
    for c, per, want in zip(f.cases, outs, expected(name)):
        if isinstance(f, cg.CcFix):
            if not all(cg.cc_agrees(o, w, form) for o, w, form in zip(per, want, c.forms)):
                return False
        elif not all(cg.sf_agrees(o, w, c, call) for o, w, call in zip(per, want, f.calls)):
            return False
    return True


def test_constants():
    K = cg.K
    assert (K["EN_NT"], K["EN_VT"], K["EN_TILE"], K["GRID_NT"]) == (256, 8, 2048, 256)
    assert (K["CC_MAX_NODES"], K["CC_MAX_DEPTH"]) == (1 << 16, 64) and K["CC_MAX_DEPTH"] == cp.K["MAX_DEPTH"]
    assert (K["SGF_MAX_NODES"], K["SGF_MAX_LEAVES"], K["SGF_MAX_DEPTH"]) == (1024, 1024, 64)
    assert all(K["SGF_" + k] == sp.K[k] for k in ("MAX_NODES", "MAX_LEAVES", "MAX_DEPTH"))


def _rewrite(text, func, pat):
    """The first space of the statement's match doubled: the same code, no longer the restated text."""
    body = cg._fn(func, text) if func else text
    s = re.search(pat, body).group(0)
    return text.replace(body, body.replace(s, s.replace(" ", "  ", 1), 1), 1)


@pytest.mark.parametrize("fn, func, pat, what", cg.STATEMENTS, ids=[f"{s[1]}: {s[3]}" for s in cg.STATEMENTS])
def test_a_rewritten_statement_fails(monkeypatch, fn, func, pat, what):
    real = cg._src
    assert re.search(pat, real(fn)), what
    monkeypatch.setattr(cg, "_src", lambda f: _rewrite(real(f), func, pat) if f == fn else real(f))
    with pytest.raises(ValueError, match=re.escape("restate it in the cascade model")):
        cg.read_constants()


@pytest.mark.parametrize("fn, what, to", [
    ("encode_kernel.cuh", "EN_TILE = EN_NT * EN_VT;", "EN_TILE = EN_VT * EN_NT;"),
    ("dgx_api.cu", "kCcMaxNodes = size_t(1) << 16;", "kCcMaxNodes = size_t(65536);"),
    ("dgx_api.cu", "constexpr uint32_t kCcMaxDepth = 64;", "constexpr uint32_t kCcMaxDepth = 32 * 2;"),
    ("dgx.h", "#define DGX_SGF_MAX_LEAVES 1024", "#define DGX_SGF_MAX_LEAVES (1 << 10)"),
    ("cascade_kernel.cuh", "__launch_bounds__(256) cc_page_kernel", "__launch_bounds__(512) cc_page_kernel"),
    ("sg_filter_kernel.cuh", "__launch_bounds__(256) sf_eval_kernel", "__launch_bounds__(128) sf_eval_kernel"),
])
def test_a_rewritten_constant_fails(monkeypatch, fn, what, to):
    real = cg._src
    assert what in real(fn)
    monkeypatch.setattr(cg, "_src", lambda f: real(f).replace(what, to) if f == fn else real(f))
    with pytest.raises(ValueError, match=re.escape("restate it in the cascade model")):
        cg.read_constants()


@pytest.mark.parametrize("name", list(FIXTURES))
def test_fixture_reaches_its_events(name):
    missing = FIXTURES[name].events - run(name)[1]
    assert not missing, f"{name}: does not reach {sorted(missing)}"


def test_every_event_is_reached():
    reached = set().union(*(run(n)[1] for n in FIXTURES))
    assert not cg.EVENTS - reached, f"no fixture reaches {sorted(cg.EVENTS - reached)}"


def test_every_fixture_is_needed():
    """Each fixture reaches an event no other fixture reaches: deleting any one leaves an event unreached."""
    for name in FIXTURES:
        others = set().union(*(run(n)[1] for n in FIXTURES if n != name))
        assert run(name)[1] - others, f"{name}: every event it reaches is reached by another fixture"


def test_every_event_name_in_the_model_is_registered():
    src = open(cg.__file__).read()
    assert len(re.findall(r"\bev\.add\(", src)) == 1, "events are recorded through _add only"
    for is_f, text in re.findall(r"_add\(ev, (f?)\"([^\"]*)\"", src):
        if not is_f:
            assert text in cg.EVENTS, f"{text!r} is recorded but not registered"
            continue
        pat = "".join(".+" if i % 2 else re.escape(part) for i, part in enumerate(re.split(r"[{}]", text)))
        assert any(re.fullmatch(pat, e) for e in cg.EVENTS), f"f-string {text!r} matches no registered event"
    for text in re.findall(r"\"((?:cc|sf) [a-z0-9]+: [^\"]*)\"", src):
        if "{" not in text:
            assert text in cg.EVENTS, f"{text!r} is named in the model but not registered"


@pytest.mark.parametrize("name", [n for n, f in FIXTURES.items() if isinstance(f, cg.CcFix)])
def test_cascade_oracles_agree(name):
    """cascade_oracle.c (populateVarMap line by line) and gen_cascade's formula give one answer on every case."""
    for c in FIXTURES[name].cases:
        if cg.cc_malformed(c, "dev"):
            continue
        rows, dests = co.cascade(c.nodes)
        frows, fdests = gc.formula(c.nodes)
        assert all(np.array_equal(a, b) for a, b in zip(dests, fdests)), name
        assert all(len(x) == len(y) and all(np.array_equal(u, v) for u, v in zip(x, y))
                   for x, y in zip(rows, frows)), name


@pytest.mark.parametrize("name", [n for n, f in FIXTURES.items() if isinstance(f, cg.SfFix)])
def test_sg_filter_oracles_agree(name):
    """sg_filter_oracle.c (ProcessGraph's filter block line by line) and gen_sg_filter's per-D0 formula give one
    answer on every call of every case."""
    f = FIXTURES[name]
    for c in f.cases:
        for call in f.calls:
            if cg.sf_malformed(c, call):
                continue
            args = cg.sf_oracle_args(c, call)
            rows, counts, dest = so.sg_filter(*args)
            frows, fcounts, fdest = gs.formula(*args)
            assert [r.tolist() for r in rows] == frows and counts.tolist() == fcounts and dest.tolist() == fdest, \
                (name, call)


@pytest.mark.parametrize("name", list(FIXTURES))
def test_model_equals_oracle(name):
    assert agrees(name, run(name)[0]), name


@pytest.mark.parametrize("name", list(FIXTURES))
def test_launches_match_the_plans(name):
    f = FIXTURES[name]
    for c, per in zip(f.cases, run(name)[0]):
        if isinstance(f, cg.CcFix):
            for form, o in zip(c.forms, per):
                src = cg.cc_inputs(c, form)
                assert o.launches == cp.launches(gc.levels_with_work(c.nodes, [s[3] for s in src])), (name, form)
        else:
            for call, o in zip(f.calls, per):
                assert o.launches == sp.launches(cg.sf_inputs(c, call)["d0_cap"]), (name, call)


def test_every_mutant_is_aimed_at():
    named = set().union(*(f.kills for f in FIXTURES.values()))
    assert named == set(cg.MUTANTS), f"no fixture kills {sorted(set(cg.MUTANTS) - named)}"


@pytest.mark.parametrize("name, mutant", [(n, m) for n, f in FIXTURES.items() for m in sorted(f.kills)])
def test_the_mutant_differs_from_the_oracle(name, mutant):
    """The model with one slip gives a different answer on the fixture aimed at it."""
    assert not agrees(name, run(name, frozenset([mutant]))[0]), f"{name}: the mutant {mutant!r} gives the oracle's output"


def test_model_random_cascade():
    """gen_cascade's random forests: the model is the oracle in both forms, with random value rooms."""
    rng = np.random.default_rng(71_000)
    for it in range(150):
        f = gc.random_forest(rng)
        slack = {k: rng.integers(1, 50, int(rng.integers(0, 4))).astype(np.uint64) for k in range(len(f))}
        case = cg.cc_case(f, slack=slack)
        for form in case.forms:
            assert cg.cc_agrees(cg.cc_run(case, form), cg.cc_expected(case, form), form), (it, form)


def test_model_random_sg_filter():
    """gen_sg_filter's random cases: the model is the oracle in every form and in counts-only mode."""
    rng = np.random.default_rng(72_000)
    for it in range(300):
        case = cg.sf_case(*gs.random_case(rng), d0_slack=rng.integers(1, 9, int(rng.integers(0, 3))).astype(np.uint64),
                          v_slack=rng.integers(1, 9, int(rng.integers(0, 3))).astype(np.uint64))
        for call in cg.SF_CALLS:
            if call.form == "dev_words" and case.d0_slack.size and case.d0.size and \
                    case.d0_slack[0] <= case.d0[-1]:
                case = case._replace(d0_slack=case.d0_slack + case.d0[-1])
            w = cg.sf_expected(case, call)
            assert cg.sf_agrees(cg.sf_run(case, call), w, case, call), (it, call)
