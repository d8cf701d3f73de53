"""@recurse on the host (no GPU): the line-by-line restatement of expandRecurse's per-sg step (recurse_oracle.c) against
the independent numpy formula (gen_recurse.Formula) over random recursions, the reference's recurse tests restated at
the uid level on the friend / follow fixture, and the launch plan model."""
from __future__ import annotations

import json
import os

import numpy as np
import pytest

import gen_recurse as gr
import recurse_oracle as ro
import recurse_plan

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "recurse_friend_follow.json")


def oracle_step(reach, ids):
    def step(attr, src, rows, dest):
        return reach.step(ids.setdefault(attr, len(ids) + 1), src, rows, dest)
    return step


def fixture():
    with open(GOLDEN) as f:
        d = json.load(f)
    graph = {}
    for p, e in d["edges"].items():
        if e:
            fr, to = zip(*e)
            graph[p] = gr.Pred.from_edges(1003, fr, to)
    return d, graph


def run_oracle(graph, preds, depth, roots=(1,), **kw):
    reach = ro.Reach()
    return gr.recurse(graph, list(roots), preds, depth, oracle_step(reach, {}), **kw)


def random_case(rng):
    n = int(rng.integers(1, 40))
    preds = [f"p{i}" for i in range(int(rng.integers(1, 4)))]
    graph = gr.random_graph(rng, n, preds, mean_deg=float(rng.uniform(0.5, 4)), self_loops=bool(rng.random() < 0.7))
    roots = rng.choice(np.arange(1, n + 1), size=int(rng.integers(1, min(n, 4) + 1)), replace=False)
    filters = {p: rng.choice(np.arange(1, n + 1), size=int(rng.integers(0, n + 1)), replace=False)
               for p in preds if rng.random() < 0.4}
    return graph, roots, preds, int(rng.integers(1, 9)), filters


@pytest.mark.parametrize("seed", range(8))
def test_restatement_equals_formula(seed):
    rng = np.random.default_rng(1400 + seed)
    for _ in range(400):
        graph, roots, preds, depth, filters = random_case(rng)
        reach, ids = ro.Reach(), {}
        formula = gr.Formula()
        a, na, _ = gr.recurse(graph, roots, preds, depth, oracle_step(reach, ids), filters=filters)
        b, nb, _ = gr.recurse(graph, roots, preds, depth, formula.step, filters=filters)
        assert na == nb and len(a) == len(b)
        for x, y in zip(a, b):
            assert (x.level, x.pos, x.attr, x.kept) == (y.level, y.pos, y.attr, y.kept)
            assert np.array_equal(x.dest_uids, y.dest_uids)
            assert all(np.array_equal(r, s) for r, s in zip(x.kept_rows, y.kept_rows))
        for p, i in ids.items():
            f0, t0 = reach.edges(i)
            f1, t1 = formula.edges(p)
            assert np.array_equal(f0, f1) and np.array_equal(t0, t1)


def test_restatement_edge_limit_and_loop():
    rng = np.random.default_rng(7)
    graph = gr.random_graph(rng, 30, ["a", "b"], mean_deg=3)
    root = int(np.argmax(np.diff(graph["a"].ptr)))
    _, total, err = run_oracle(graph, ["a", "b"], 8, roots=[root])
    assert not err and total > 4
    steps, n, err = run_oracle(graph, ["a", "b"], 8, roots=[root], limit=total // 2)
    assert err and n > total // 2
    # loop: true counts len(SrcUIDs) x the matrix's values per sg (:112-115) and keeps every edge
    steps, n, _ = gr.recurse(graph, [root], ["a"], 3, None, allow_loop=True)
    assert n > 0
    assert n == sum(len(s.src) * sum(len(r) for r in s.rows) for s in steps)


def test_friend_follow_example():
    d, graph = fixture()
    c = d["cases"]["friend_follow"]
    steps, n, err = run_oracle(graph, c["preds"], c["depth"])
    assert not err and n == c["edges"] and max(s.level for s in steps) == c["levels"]
    lvl2 = [s for s in steps if s.level == 2]
    third = lvl2[2]
    assert third.attr == c["level2_third"]["attr"] and third.src.tolist() == c["level2_third"]["src"]
    assert third.kept == c["level2_third"]["kept"] and third.rows[1].tolist() == [24]
    for attr, want in c["union"].items():
        assert gr.merge_sorted([s.dest_uids for s in steps if s.attr == attr]).tolist() == want


def names_of(d, uids):
    return [d["names"][str(u)] for u in sorted(int(x) for x in uids) if str(u) in d["names"]]


def tree(d, steps, depth, uid, parent, k):
    """The JSON node of uid at node depth k (the root is 0): its name, which the level k + 1 fetches, and for every sg
    expanded from `parent` the kept values of its row."""
    node = {}
    if k < depth and str(uid) in d["names"]:
        node["name"] = d["names"][str(uid)]
    for i, s in enumerate(steps):
        if s.parent != parent:
            continue
        hit = np.flatnonzero(s.src == uid)
        if not hit.size:
            continue
        kids = [tree(d, steps, depth, int(v), i, k + 1) for v in s.kept_rows[int(hit[0])]]
        kids = [x for x in kids if x]
        if kids:
            node[s.attr] = kids
    return node


@pytest.mark.parametrize("name", ["TestRecurseQuery", "TestRecurseQueryLimitDepth1"])
def test_reference_trees(name):
    d, graph = fixture()
    c = d["cases"][name]
    steps, n, err = run_oracle(graph, c["preds"], c["depth"])
    assert not err
    assert tree(d, steps, c["depth"], 1, None, 0) == c["tree"]
    if "rows" in c:
        friend = [s for s in steps if s.attr == "friend"]
        assert [[s.src.tolist(), [r.tolist() for r in s.kept_rows]] for s in friend] == c["rows"]
        assert n == c["edges"] and max(s.level for s in steps) == c["levels"]


def test_reference_variables():
    d, graph = fixture()
    c = d["cases"]["TestRecurseVariable2"]
    steps, _, _ = run_oracle(graph, c["preds"], c["depth"])
    var = {a: gr.merge_sorted([s.dest_uids for s in steps if s.attr == a]) for a in c["preds"]}
    assert names_of(d, var["follow"]) == c["me"] and names_of(d, var["friend"]) == c["me2"]
    c = d["cases"]["TestRecurseVariable"]
    steps, _, _ = run_oracle(graph, c["preds"], c["depth"])
    assert names_of(d, gr.merge_sorted([s.dest_uids for s in steps])) == c["me"]
    c = d["cases"]["TestRecurseQueryLimitDepth2"]
    steps, _, _ = run_oracle(graph, c["preds"], c["depth"])
    assert [s.kept_rows[0].tolist() for s in steps if s.level == 1 and s.attr == "friend"] == [c["friend_uids"]]


def test_launch_plan():
    K = recurse_plan.K
    assert (K["FRONT"], K["BACK"]) == (5, 2)
    assert recurse_plan.launches(0, 100) == 0 and recurse_plan.launches(5, 0) == 0
    base = K["FRONT"] + K["MERGE"] + K["BACK"]
    assert recurse_plan.launches(1, 1) == base + 1
    assert recurse_plan.launches(10 ** 6, 2048) == base + 1
    assert recurse_plan.launches(1, 2049) == base + 1 and recurse_plan.launches(1, 3 * 2048) == base + 2
    with pytest.raises(ValueError):
        api = recurse_plan._src("dgx_api.cu").replace("count_launches(l, 2);\n    return DGX_OK;\n}\n\n// The checks",
                                                      "count_launches(l, 3);\n    return DGX_OK;\n}\n\n// The checks")
        recurse_plan.read_constants(api.replace("rc_commit_kernel<<<1, 1, 0, l->stream>>>(P);", ""))
