"""The host model of the filter pipeline (tests/filter_geometry.py), on the CPU: the constants and the slice_cap
statement parse, every fixture of tests/test_gpu_filter_edges.py reaches the events it names, the fixtures together
reach every branch the model names, and the model's results equal the oracle's.  A fixture that drifts off its edge
(a constant changed, a builder edited) fails here, before any GPU run."""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import filter_geometry as fg  # noqa: E402

FIXTURES = {f.name: f for f in fg.all_fixtures()}
_RUNS = {}


def run(name):
    if name not in _RUNS:
        f = FIXTURES[name]
        _RUNS[name] = fg.simulate(f.queries, f.op, f.resident, f.offsets)
    return _RUNS[name]


def test_constants_and_slice_cap_statement():
    assert (fg.P_CW, fg.P_MAXL, fg.P_SAMPLES, fg.P_DEFER_DIV) == (8, 8, 256, 32)
    assert (fg.P_SAMPLE_MIN_A, fg.P_SAMPLE_LISTS, fg.P_TAIL_NT) == (65536, 31, 256)
    # (VA, tile, slice_cap, grp) by kmax, derived by hand from filter_batch_impl
    assert fg.geometry(1) == (4, 1024, 2304, 2)
    assert fg.geometry(2) == (4, 1024, 2304, 2)
    assert fg.geometry(3) == (2, 512, 1152, 2)
    assert fg.geometry(4) == (2, 512, 1728, 1)
    assert fg.geometry(8) == (2, 512, 4032, 1)
    assert fg.geometry(9) == fg.geometry(40) == (2, 512, 4608, 1)


def test_constants_fail_loudly(monkeypatch):
    """A rewritten slice_cap statement or a renamed constant is an error, not a silently different model."""
    real = fg._src

    def edited(fn, what, to):
        return lambda f: real(f).replace(what, to) if f == fn else real(f)

    monkeypatch.setattr(fg, "_src", edited("dgx_api.cu", "(TA + TA / 8) * nl", "(TA + TA / 4) * nl"))
    with pytest.raises(ValueError, match="slice_cap"):
        fg.read_constants()
    monkeypatch.setattr(fg, "_src", edited("filter_pipe.cuh", "P_DEFER_DIV =", "P_DEFER_DIVISOR ="))
    with pytest.raises(KeyError, match="P_DEFER_DIV"):
        fg.read_constants()
    monkeypatch.setattr(fg, "_src", edited("dgx_api.cu", "kmax <= 2 ? 4 : 2", "kmax <= 3 ? 4 : 2"))
    assert fg.read_constants()["VA_KMAX"] == 3  # moved with the source


@pytest.mark.parametrize("name", list(FIXTURES))
def test_fixture_reaches_its_events(name):
    f, r = FIXTURES[name], run(name)
    missing = f.events - r.events
    assert not missing, f"{name}: does not reach {sorted(missing)}"
    if f.tail is not None:
        assert r.tail_queries == f.tail, (r.tail_queries, r.keff)
    print(f"{name}: {len(f.queries)} queries, va={r.plan.va} slice_cap={r.plan.slice_cap} deep={r.plan.deep} "
          f"launches={r.plan.launches} keff={r.keff} tail={r.tail_queries}")


def test_every_event_is_reached():
    reached = set().union(*(run(n).events for n in FIXTURES))
    missing = fg.EVENTS - reached
    assert not missing, f"no fixture reaches {sorted(missing)}"


def test_every_event_name_in_the_model_is_registered():
    """Every name the model's source can record is in EVENTS (literal, or an f-string whose every expansion the table
    must list at least once), so a new branch name without a fixture fails test_every_event_is_reached."""
    src = open(fg.__file__).read()
    assert len(re.findall(r"\b(?:events|ev)\.add\(", src)) == 1, "events are recorded through _add only"
    calls = re.findall(r"_add\(\w+, (f?)\"([^\"]*)\"\)", src)
    assert len(calls) == src.count("_add(") - 1, "an _add call with a computed name"  # minus the definition
    for is_f, text in calls:
        if not is_f:
            assert text in fg.EVENTS, f"{text!r} is recorded but not registered"
            continue
        pat = "".join(".+" if i % 2 else re.escape(part) for i, part in enumerate(re.split(r"[{}]", text)))
        assert any(re.fullmatch(pat, e) for e in fg.EVENTS), f"f-string {text!r} matches no registered event"


@pytest.mark.parametrize("name", list(FIXTURES))
def test_fixture_events_under_device_placement(name):
    """The device-form tests lay every batch out back to back in one buffer (fg.device_offsets); placed so, each
    fixture still reaches its events on the lane it is aimed at, and the GPU tests' launch and deferral counts come
    from the same plan as the model's."""
    f = FIXTURES[name]
    offs, _ = fg.device_offsets(f.queries, f.offsets)
    assert all(o % 2 == c % 2 for ro, rc in zip(offs, f.offsets) for o, c in zip(ro, rc))
    r = fg.simulate(f.queries, f.op, f.resident, offs)
    missing = f.events - r.events
    assert not missing, f"{name}: placed as on the device, the batch does not reach {sorted(missing)}"
    for resident in (False, True):
        plan = fg.plan_batch(f.queries, f.op, resident, offs)
        rr = r if resident == f.resident else fg.simulate(f.queries, f.op, resident, offs)
        assert plan.launches == rr.plan.launches and fg.deferring_queries(plan) == rr.tail_queries


@pytest.mark.parametrize("name", list(FIXTURES))
def test_model_equals_oracle(orc, name):
    f, r = FIXTURES[name], run(name)
    for qi, (q, got) in enumerate(zip(f.queries, r.results)):
        want = fg.oracle_result(orc, q, f.op)
        assert np.array_equal(got, want), f"{name}: query {qi}: model {got.size} values, oracle {want.size}"


def test_windows_cover_slices_up_to_4P():
    """lift32m's four windows leave no gap while n <= 4P (the pair path allows n <= 3P), and leave one past it."""
    for l2 in range(0, 9):
        P = 1 << l2
        for n in range(P, 4 * P + 1):
            assert fg.window_gaps(n, l2) <= P, (P, n)
        assert fg.window_gaps(4 * P + 1, l2) > P or P == 1


def test_lift32m_is_a_lower_bound_up_to_4P():
    """The model's lift32m finds every value of a slice and no value outside it, for every n in P..4P."""
    rng = np.random.default_rng(3)
    for l2 in range(0, 7):
        P = 1 << l2
        for n in range(P, 4 * P + 1):
            s = np.sort(rng.choice(np.arange(1, 10 * n + 10, 2, dtype=np.uint32), n, replace=False))
            x = np.concatenate([s, s + np.uint32(1), [0, 0xFFFFFFFF]]).astype(np.uint32)
            hit = fg.lift32m(s, l2, x, np.ones(x.size, bool))
            assert np.array_equal(hit, np.isin(x, s)), (P, n)
        if P >= 2:  # past 4P a value in the first gap is missed
            n = 5 * P
            s = np.arange(1, 2 * n, 2, dtype=np.uint32)
            assert not fg.lift32m(s, l2, s, np.ones(n, bool)).all(), P


def _random_batch(rng):
    import gen

    nq = int(rng.integers(1, 5))
    qs = []
    for _ in range(nq):
        k = int(rng.integers(1, 7))
        master = gen.zipf_gaps(rng, int(rng.integers(50, 3000)), start=int(rng.choice([1, (1 << 32) - 700, 1 << 60])))
        if rng.random() < 0.3:
            master = np.sort(np.concatenate([master, master[:: int(rng.integers(3, 20))]]))
        qs.append([gen.thin(rng, master, float(p)) for p in rng.uniform(0.2, 1.0, k)])
    offs = [[int(x) for x in rng.integers(0, 2, len(q))] for q in qs]
    return qs, offs


def test_model_random_batches(orc):
    """The model against the oracle on random batches: repeated values, values around 2^32, head parities."""
    rng = np.random.default_rng(11)
    for it in range(60):
        qs, offs = _random_batch(rng)
        r = fg.simulate(qs, offsets=offs)
        for q, got in zip(qs, r.results):
            assert np.array_equal(got, fg.oracle_result(orc, q, fg.OP_INTERSECT)), it
        pairs = [q[:2] for q in qs if len(q) >= 2]
        if pairs:
            r = fg.simulate(pairs, fg.OP_DIFFERENCE)
            for q, got in zip(pairs, r.results):
                assert np.array_equal(got, orc.difference(q[0], q[1])), it
