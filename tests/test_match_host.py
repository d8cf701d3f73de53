"""match() on the CPU: the line-by-line restatement (match_oracle.c) against the independent formula (gen_match.py) on
seeded random cases and the published answers, the branch choice and every argument dgx_match refuses before it needs
a device."""
import numpy as np
import pytest

import gen_match as gm
import gen_trigram as gt
import match_cases as mc
import match_oracle as mo


def test_oracle_equals_formula_random():
    # 3 000 cases weighted to invalid and truncated UTF-8, literal U+FFFD, 2-4 byte runes, empty values and queries,
    # max of 0 / the length difference / 2^31 - 1, list values whose first fails and a later one passes, and
    # candidates without a value
    seen = {"empty query": 0, "max 0": 0, "max i32": 0, "later value": 0, "absent": 0, "kept": 0}
    for seed in range(3000):
        rng = np.random.default_rng(900_000 + seed)
        uids, values, q, mx, cands = gm.random_case(rng)
        col = mc.column(uids, values)
        got = mo.match(col, q, mx, uids=cands)
        vo = mc.values_of(uids, values)
        want = gm.formula(vo, q, mx, cands)
        assert got.tolist() == want, (seed, q, mx)
        seen["empty query"] += not q
        seen["max 0"] += mx == 0
        seen["max i32"] += mx == gm.MAX_I32
        seen["absent"] += any(int(u) not in vo for u in cands)
        seen["kept"] += len(want)
        for u in want:
            vs = vo[u]
            seen["later value"] += not (vs[0] and gm.distance(vs[0], q) <= mx)
    assert all(v > 20 for v in seen.values()), seen


def test_levenshtein_tricky_bytes():
    for a in gm.TRICKY:
        for b in gm.TRICKY:
            assert mo.levenshtein(a, b) == gm.distance(a, b), (a, b)
    # Go's one U+FFFD per invalid byte, not Python's maximal subpart
    assert mo.levenshtein(b"\xe2\x82", b"") == 2 and mo.levenshtein(b"\xf0\x9f", b"") == 2
    assert mo.levenshtein(b"\xe2\x82", "��".encode()) == 0
    assert len(gm.runes(b"\xe2\x82")) == 2 != len(b"\xe2\x82".decode("utf-8", "replace"))


def test_golden_distances():
    g, _ = mc.golden()
    for a, b, d in g["distance"]:
        assert mo.levenshtein(a, b) == d and gm.distance(a.encode(), b.encode()) == d, (a, b)


def test_golden_queries_restatement_and_formula():
    g, cols = mc.golden()
    for case in g["cases"]:
        uids, vals = cols[case["pred"]]
        col = mc.column(uids, vals)
        q = case["query"].encode()
        after = case["after"]
        # a list leaf is a row pl.Uids already read from after
        leaves = [("list", lf[1][lf[1] > np.uint64(after)]) for lf in mc.trigram_leaves(mc.trigram_index(uids, vals), q)]
        got = mo.match(col, q, case["max"], leaves=gt.to_oracle(leaves), after=after)
        first = case["first"] or len(got)
        assert got[:first].tolist() == case["want"], case["test"]
        cands = np.unique(np.concatenate([gt.leaf_set(lf, after) for lf in leaves] or [np.zeros(0, np.uint64)]))
        want = gm.formula(mc.values_of(uids, vals), q, case["max"], cands)
        assert want[:first] == case["want"], case["test"]


def test_trigram_branch_packs_and_layers_restatement():
    # the restatement's uidsForMatch over pack leaves with layers and after_uid equals the formula over leaf_set
    for seed in range(200):
        rng = np.random.default_rng(70_000 + seed)
        uids, values, q, mx, _ = gm.random_case(rng, nuids=60, universe=120)
        after = int(rng.choice([0, 30, 119]))
        leaves = gt.random_leaves(rng, int(rng.integers(0, 6)), 120, "mixed", after=after)
        col = mc.column(uids, values)
        got = mo.match(col, q, mx, leaves=gt.to_oracle(leaves), after=after)
        cands = np.unique(np.concatenate([gt.leaf_set(lf, after) for lf in leaves] or [np.zeros(0, np.uint64)]))
        assert got.tolist() == gm.formula(mc.values_of(uids, values), q, mx, cands), seed


@pytest.mark.parametrize("name,kw,want_rc,on_device", mc.error_cases(), ids=[c[0] for c in mc.error_cases()])
def test_argument_errors(name, kw, want_rc, on_device):
    if on_device:
        pytest.skip("found on the device: tests/test_gpu_match.py")
    r = mc.Raw(**kw)
    rc, out, n = r.host(0, 64)
    assert rc == want_rc and n == mc.SENTINEL and np.all(out == np.uint64(mc.SENTINEL)), name


def test_out_cap_is_the_branchs_bound():
    col = mc.column([3, 5, 9], [[b"abc"], [b"abd"], [b"x"]])
    leaves = [("list", np.array([3, 5, 9], np.uint64)), ("list", np.array([5, 7], np.uint64))]
    # nuids > 0: the UidList branch, bound nuids, whatever the leaves
    r = mc.Raw(col, "abc", 1, uids=[3, 5], leaves=leaves)
    rc, out, n = r.host(0, 1)
    assert rc == mc.ERR_CAP and n == mc.SENTINEL and np.all(out == np.uint64(mc.SENTINEL))
    # nuids == 0: the leaves, bound 3 + 2
    r = mc.Raw(col, "abc", 1, uids=[], leaves=leaves)
    rc, out, n = r.host(0, 4)
    assert rc == mc.ERR_CAP and n == mc.SENTINEL
    # nuids == 0 and no leaf (a query under 3 bytes): no candidate, no device
    r = mc.Raw(col, "ab", 1, uids=[])
    rc, out, n = r.host(0, 0)
    assert (rc, n) == (mc.OK, 0) and np.all(out == np.uint64(mc.SENTINEL))
    # empty leaves only: bound 0
    r = mc.Raw(col, "abc", 1, leaves=[("list", np.zeros(0, np.uint64)), ("pack", None, None, 0)])
    rc, out, n = r.host(0, 0)
    assert (rc, n) == (mc.OK, 0)


def test_launch_plan():
    # 5 launches after the candidates whatever the sizes; the trigram stages of one OR node before them
    rng = np.random.default_rng(3)
    lv = gt.random_leaves(rng, 6, 5000, "mixed", p_list=0.5)
    one_list = [("list", np.array([1, 2], np.uint64))]
    assert mc.launches([], 7) == 5
    assert mc.launches([], 0) == 0
    assert mc.launches([("list", np.zeros(0, np.uint64))], 0) == 0
    assert mc.launches(one_list, 0) == 2 + 5  # tg_leaves, tg_gather (the result), then the match stages
    npk = sum(1 for lf in lv if lf[0] == "pack")
    assert mc.launches(lv, 0) > 2 + 5 + (5 if npk else 0)  # two or more driving leaves add the merge
