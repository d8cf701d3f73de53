"""uidsForRegex on the CPU: the line-by-line restatement (trigram_oracle.c) against the set formula the device
computes, the host plan (trigram_plan.py), the hand-written trees of regexp patterns on a small index, and every
argument dgx_trigram_query refuses before it needs a device."""
import re

import numpy as np
import pytest

import gen_trigram as gt
import trigram_oracle as tgo
import trigram_plan as tp
from trigram_cases import ERR_ARG, ERR_CAP, OK, SENTINEL, Raw, error_cases

AFTERS = ("zero", "median", "max")


def _after(kind, universe):
    return {"zero": 0, "median": universe // 2, "max": gt.U64}[kind]


def _case(seed, branch, after_kind, universe=240):
    rng = np.random.default_rng(seed)
    after = _after(after_kind, universe)
    nleaves = int(rng.integers(1, 9))
    leaves = gt.random_leaves(rng, nleaves, universe, branch, after=after)
    tree = gt.random_tree(rng, nleaves, int(rng.integers(1, 8)), max_depth=int(rng.choice([3, 8])))
    return tree, leaves, after


@pytest.mark.parametrize("branch", ["compressed", "probe", "iterate", "mixed"])
def test_oracle_equals_formula(branch):
    # 800 trees per branch, each at after 0, the median uid and 2^64 - 1: with "compressed" / "probe" / "iterate" every
    # filtered read of a pack leaf below an AND takes that branch of List.Uids, and all give the formula's set
    n_and_sub = 0
    for seed in range(800):
        for ak in AFTERS:
            tree, leaves, after = _case(seed, branch, ak)
            got = tgo.uids_for_regex(tree, gt.to_oracle(leaves), after)
            assert np.array_equal(got, gt.want(tree, leaves, after)), (branch, seed, ak, tree)
        n_and_sub += any(op == gt.QAND and subs for op, _, subs in tree)
    assert n_and_sub > 150  # filtered reads below an AND's running result are common, not incidental


def test_branches_are_taken():
    # the branch rule of a filtered read (posting/list.go:1795-1822) as the oracle restates it, on one AND sub
    universe = 100
    a = np.arange(1, 60, dtype=np.uint64)
    mut = (np.array([2, 70], np.uint64), np.array([1, 0], np.uint8))
    for approx in (0, 1 << 40):  # iterate, probe
        tree = [(gt.QAND, [0], [1]), (gt.QAND, [1], [])]
        for after in (0, 30):  # a list leaf is a pl.Uids read: above after
            leaves = [("list", a[a > after]), ("pack", np.arange(1, universe, 2, dtype=np.uint64), mut, approx)]
            got = tgo.uids_for_regex(tree, gt.to_oracle(leaves), after)
            assert np.array_equal(got, gt.want(tree, leaves, after))


def test_plan_driving_set_covers_result():
    for seed in range(1500):
        tree, leaves, after = _case(10_000 + seed, "mixed", AFTERS[seed % 3])
        bounds = [gt.leaf_bound(lf) for lf in leaves]
        p = tp.plan(tree, bounds)
        assert p.rc == OK
        res = gt.want(tree, leaves, after)
        assert res.size <= p.root_bound
        if p.root_bound == 0:
            assert res.size == 0
            continue
        cover = np.unique(np.concatenate([gt.leaf_set(leaves[j], after) for j in p.drive] + [np.zeros(0, np.uint64)]))
        assert np.all(np.isin(res, cover)), (seed, tree)
        assert p.dcap <= p.root_bound
        if p.all_or:  # the candidates are the result
            assert np.array_equal(cover, res)


def test_plan_launches():
    b = [10, 20, 30]
    star = [(gt.QOR, [0, 1, 2], [])]
    assert tp.launches(tp.plan(star, b), npacks=3) == tp.K["ROWS"] + 2 + tp.K["MERGE"] + 1
    assert tp.launches(tp.plan([(gt.QOR, [1], [])], b), npacks=0) == 2
    assert tp.launches(tp.plan([(gt.QAND, [0, 1, 2], [])], b), npacks=3) == tp.K["ROWS"] + 4
    assert tp.launches(tp.plan([(gt.QOR, [], [])], b), npacks=3) == 0
    big = tp.plan([(gt.QAND, [0], [1]), (gt.QOR, [1, 2], [])], [3 << 20, 3 << 19, 1 << 19])
    assert big.drive == [1, 2] and big.dcap == 1 << 21
    assert tp.launches(big, npacks=3) == tp.K["ROWS"] + 4 + tp.K["MERGE"] + 10  # 1024 tiles: ten tree levels


def test_patterns_on_small_index():
    idx = gt.TrigramIndex(seed=7, n_nodes=3000, n_words=600)
    texts = [" ".join(idx.words_of_node(i)) for i in range(idx.n_nodes)]
    tris_of = [set().union(*[gt.trigrams(w) for w in idx.words_of_node(i)]) for i in range(idx.n_nodes)]
    for pat, nodes in gt.PATTERNS.items():
        tree, tris = gt.tree_of_pattern(nodes)
        leaves = [("list", idx.posting(t)) for t in tris]
        got = tgo.uids_for_regex(tree, gt.to_oracle(leaves), 0)
        assert np.array_equal(got, gt.want(tree, leaves, 0)), pat
        implied = np.array([i + 1 for i in range(idx.n_nodes) if gt.eval_on_value(nodes, tris_of[i])], np.uint64)
        assert np.array_equal(got, implied), pat
        matching = np.array([i + 1 for i, s in enumerate(texts) if re.search(pat, s)], np.uint64)
        assert matching.size > 0, pat  # the index holds a value the pattern matches
        assert np.all(np.isin(matching, got)), pat  # the trigram query never drops a match
        assert got.size < idx.n_nodes, pat


@pytest.mark.parametrize("name,kw,want_rc", error_cases(), ids=[c[0] for c in error_cases()])
def test_refused_before_anything_is_copied(name, kw, want_rc):
    # the checks run on the host before a device is needed, with out untouched; the plan model agrees
    r = Raw(**kw)
    rc, out, n = r.host(0, 64)
    assert rc == want_rc, name
    assert np.all(out == np.uint64(SENTINEL)) and n == SENTINEL
    bounds = [(0 if (m is None) else len(m[0])) for m in r.muts] + [int(x) for x in np.diff(r.list_off.astype(np.int64))]
    if name not in ("list_off decreasing", "list_off[0] != 0", "mut_off decreasing", "DGX_MUT_VALUE"):
        assert tp.plan(kw["tree"], bounds).rc == ERR_ARG, name


def test_cap_and_empty_root_need_no_device():
    a, b = np.array([1, 4, 9], np.uint64), np.array([4, 5], np.uint64)
    r = Raw([(gt.QOR, [0, 1], [])], lists=[a, b])
    rc, out, n = r.host(0, 4)  # root bound 5
    assert rc == ERR_CAP and np.all(out == np.uint64(SENTINEL))
    assert tp.plan(r.tree, [3, 2], out_cap=4).rc == ERR_CAP
    e = Raw([(gt.QAND, [0], [1]), (gt.QOR, [], [])], lists=[a])
    rc, out, n = e.host(0, 0)
    assert rc == OK and n == 0
