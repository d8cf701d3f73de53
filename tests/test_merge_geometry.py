"""The host model of MergeSorted's plan and multiway geometry (tests/merge_geometry.py), on the CPU: every fixture of
tests/test_gpu_merge_edges.py still reaches the geometry it is aimed at, and the model keeps its invariants on the
fixtures and on random inputs.  A fixture that drifts off its edge (a constant changed, a builder edited) fails here,
before any GPU run."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import merge_geometry as mg  # noqa: E402

FIXTURES = {f.name: f for f in mg.all_fixtures()}


def check_invariants(runs, geo):
    """What every multiway plan must satisfy, whatever the input."""
    allsamp = np.concatenate(geo.samples) if geo.samples else np.zeros(0, np.uint64)
    want = np.unique(allsamp)[mg.MM_STRIDE - 1::mg.MM_STRIDE]
    assert [int(x) for x in want] == geo.S[1:], "boundary b is distinct sample b * MM_STRIDE - 1"
    for j, r in enumerate(runs):
        bj = geo.bounds[j]
        assert bj[0] == 0 and bj[-1] == r.size and all(x <= y for x, y in zip(bj, bj[1:])), f"run {j}: pieces {bj}"
    prev_max = None
    for t in geo.tiles:
        vals = [r[c:e] for r, c, e in zip(runs, t.start, t.end) if e > c]
        if not vals:
            continue
        lo, hi = min(int(v[0]) for v in vals), max(int(v[-1]) for v in vals)
        assert prev_max is None or lo > prev_max, f"tile {t.b}: a value shares two tiles"
        prev_max = hi
        if t.interior:
            assert t.lo <= lo and hi <= t.hi, f"tile {t.b}: values outside [S(b), S(b+1))"
        if not t.wide:
            assert hi - t.lo < mg.T_INF, f"tile {t.b}: key {hi - t.lo:#x} in the 32-bit engine"
        adv = np.sum([r.adv for r in t.rounds], axis=0)
        assert list(adv) == [e - c for c, e in zip(t.start, t.end)], f"tile {t.b}: rounds end before the runs do"
        for r in t.rounds:
            assert r.np <= (mg.MM_C if t.wide else mg.T_C), f"tile {t.b}: a round overflows shared memory"
    got = mg.model_output(geo)
    want = np.unique(np.concatenate(runs)) if runs else np.zeros(0, np.uint64)
    assert np.array_equal(got, want), "the modelled tiles do not add up to the sorted union"


def target_tile(f, geo):
    t = geo.tiles[f.expect["tile"]]
    where = f.expect["where"]
    assert (t.b == 0) == (where == "first") and (t.b == geo.ns) == (where == "last"), (where, t.b, geo.ns)
    assert [e - c for c, e in zip(t.start, t.end)] == f.expect["counts"]
    assert (where == "first" and t.lo == f.expect["lo"]) or where != "first"
    return t


@pytest.mark.parametrize("name", list(FIXTURES))
def test_fixture_reaches_its_geometry(name):
    f = FIXTURES[name]
    runs = [r for r in f.runs if r.size]
    geo = mg.multiway_geometry(runs)
    check_invariants(runs, geo)
    e = f.expect
    plan = mg.merge_plan([r.size for r in runs])
    assert plan.path == "multiway", (name, plan)
    if "tile" in e:
        t = target_tile(f, geo)
        assert t.exact == e.get("exact", t.exact) and t.wide == e["wide"], (t.exact, t.wide)
        real_max = max(int(r[c:e_][-1]) for r, c, e_ in zip(runs, t.start, t.end) if e_ > c)
        real_min = min(int(r[c]) for r, c, e_ in zip(runs, t.start, t.end) if e_ > c)
        assert real_max == e["top"] and real_min == e["lo"]
        if "max_key" in e:
            assert t.max_key == e["max_key"], (t.max_key, e["max_key"])
        if "need" in e:
            assert t.rounds[0].need == e["need"] and t.total == e["raw"], (t.rounds[0].need, t.total)
        nr = len(t.rounds)
        assert e.get("rounds_min", 1) <= nr <= e.get("rounds_max", nr), nr
        if e.get("carry"):
            assert any(r.carry_in for r in t.rounds), "no round starts on the value the previous one ended with"
        print(f"{name}: tile {t.b}/{geo.ns} lo={t.lo:#x} hi={t.hi:#x} exact={t.exact} wide={t.wide} "
              f"max_key={t.max_key if t.max_key is None else hex(t.max_key)} padded={t.rounds[0].need} rounds={nr} "
              f"carries={sum(r.carry_in for r in t.rounds)}")
    if "one_value" in e:
        assert geo.ns == 0 and len(geo.tiles) == 1
        t = geo.tiles[0]
        assert not t.wide and t.max_key == 0 and len(t.rounds) >= 30
        assert all(r.nsafe == sum(r.takes) for r in t.rounds), "a value above the bound"
        assert sum(r.carry_in for r in t.rounds) == len(t.rounds) - 1
        print(f"{name}: one tile, {len(t.rounds)} rounds")
    if "zero_samples" in e:
        s = mg.sample_counts([r.size for r in runs])
        z = [j for j, x in enumerate(s) if x == 0]
        assert len(z) == e["zero_samples"]
        for j in z:
            tiles = [t.b for t in geo.tiles if t.end[j] > t.start[j]]
            print(f"{name}: run {j} ({runs[j].size} values, no sample) in tiles {tiles[0]}..{tiles[-1]}")
        pieces = {j: [t.b for t in geo.tiles if t.end[j] > t.start[j]] for j in z}
        assert pieces[z[0]] == [e["inside_tiles"][0]] and pieces[z[4]] == [e["inside_tiles"][1]]
        assert pieces[z[1]] == [0] and pieces[z[2]] == [geo.ns] and len(pieces[z[3]]) > 10


def test_span_fixtures_pin_both_sides_of_the_engine_choice():
    """The spans straddle hi - lo = 0xFFFFFFFF in every way a tile's span is decided."""
    seen = {(f.expect["where"], f.expect.get("exact"), f.expect["wide"]) for f in mg.span_fixtures()}
    assert ("interior", False, False) in seen and ("interior", True, False) in seen and ("interior", True, True) in seen
    assert {("first", True, False), ("first", True, True), ("last", True, False), ("last", True, True)} <= seen


@pytest.mark.parametrize("name", list(mg.THRESHOLDS))
def test_threshold_plans(name):
    k, total, path = mg.THRESHOLDS[name]
    lens = mg._spread(total, k)
    plan = mg.merge_plan(lens)
    assert plan.path == path, (name, mg.describe(plan))
    if name in mg.THRESHOLD_PLANS:
        assert mg.describe(plan) == mg.THRESHOLD_PLANS[name], mg.describe(plan)
    print(f"{name}: {mg.describe(plan)}, {plan.launches} launches")


def test_grouping_below_its_minimum_stays_on_the_tree():
    assert mg.merge_plan(mg._spread(64 * 4 * mg.MERGE_MULTI_MIN - 1, 4096)).path == "tree"
    assert mg.merge_plan(mg._spread(65 * 4 * mg.MERGE_MULTI_MIN - 1, 4097)).path == "tree"


def test_threshold_fixture_lengths():
    for name in ("k=3 at the multiway minimum", "k=65 at the grouping minimum"):
        f = mg.threshold_fixture(name)
        k, total, _ = mg.THRESHOLDS[name]
        assert len(f.runs) == k and sum(r.size for r in f.runs) == total


def test_tree_fixtures_reach_their_tile_edges():
    for f in mg.tree_fixtures():
        runs = [r for r in f.runs if r.size]
        assert mg.merge_plan([r.size for r in runs]).path == "tree", f.name
        for a, b in f.expect.get("tree_pairs", ()):
            kinds = mg.tree_tile_preds(a, b)
            nb, na = kinds.count("B"), kinds.count("A")
            print(f"{f.name}: {len(kinds)} tile edges, {nb} where only B's predecessor is a repeat, {na} from A")
            assert nb >= len(kinds) // 4 and na >= len(kinds) // 4, (nb, na, len(kinds))
    ks = sorted(len([r for r in f.runs if r.size]) for f in mg.tree_fixtures())
    assert {mg.tree_launches(k) % 2 for k in ks} == {0, 1}, "both parities of the tree's ping-pong"


def test_merge_plan_matches_merge_runs_impl_examples():
    """Hand-derived plans: multiway = msample + the sample tree + 4; grouping recurses."""
    assert mg.merge_plan([100_000] * 3) == ("multiway", 5 + 2, ())
    assert mg.merge_plan([10] * 2).launches == 1 and mg.merge_plan([10]).launches == 1
    assert mg.merge_plan([5] * 5).launches == 3
    p = mg.merge_plan([40_000] * 65)
    assert p.path == "grouped" and mg.describe(p) == "grouped[multiway x2 -> tree]" and p.launches == (5 + 6) + (5 + 5) + 1  # groups of 33 and 32 runs


def _random_runs(rng):
    k = int(rng.integers(1, 20))
    lens = [int(x) for x in rng.choice([0, 1, 3, 200, 700, 3_000, 9_000, 30_000], k)]
    runs = []
    for n in lens:
        hi = int(rng.choice([50, 5_000, 1 << 20, 1 << 34, 1 << 63]))
        base = int(rng.choice([0, (1 << 32) - 3_000, (1 << 64) - (1 << 35)])) if hi < (1 << 63) else 0
        runs.append(np.sort(rng.integers(0, hi, n, dtype=np.uint64)) + np.uint64(base))
    return [r for r in runs if r.size]


def test_model_invariants_random():
    rng = np.random.default_rng(600)
    for it in range(250):
        runs = _random_runs(rng)
        if not runs:
            continue
        geo = mg.multiway_geometry(runs)
        check_invariants(runs, geo)
