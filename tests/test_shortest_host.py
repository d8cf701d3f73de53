"""shortest() without weights on the host (no GPU): the line-by-line restatement of expandOut + shortestPath
(shortest_oracle.c) against the independent numpy formula (gen_shortest.Formula) over random searches and several
neighbour orders, the argument checks of dgx_path_create / dgx_path_expand, and the launch plan model."""
from __future__ import annotations

import ctypes as C
import json
import os

import numpy as np
import pytest

import gen_shortest as gs
import shortest_oracle as so
import shortest_plan

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "shortest_path_follow.json")
SEEDS = (0x9E3779B97F4A7C15, 12345, 0xDEADBEEF)  # neighbour orders: Go's map iteration


def check_against_restatement(g, frm, to, hops, seed):
    f = gs.Formula(frm, to)
    lv = gs.search(g, frm, to, hops, f.expand)
    r = so.run(g, frm, to, hops, seed)
    L = f.to_level
    reached = to in r.dist
    assert reached == bool(L), "reachability"
    disc = [0] * (max(r.levels, len(lv)) + 2)
    for u, (h, _, _) in r.dist.items():
        if u != frm and h < len(disc):
            disc[h] += 1
    if L:
        assert r.dist[to][0] == L, "To's level"
        assert r.levels in (L, L + 1), "Go runs L levels, or L + 1 when a hop-L item pops before To"
        assert len(lv) == L
        assert len(r.path) == L + 1
    else:
        assert r.levels == len(lv), "levels run without To"
    k = len(lv)
    assert [st[0] for _, _, st in lv] == r.level_edges[:k], "numEdges of every level"
    assert [len(sgs) for sgs, _, _ in lv] == r.level_sgs[:k], "exec sgs of every level"
    assert [st[1] for _, _, st in lv] == disc[1:k + 1], "nodes discovered at every level"
    if L:
        uids, attrs = f.path()
        assert uids[0] == frm and uids[-1] == to and len(uids) == L + 1
        for i in range(L):  # admissible: a kept edge of the restatement's adjacency, at the restatement's levels
            e = (int(uids[i]), int(uids[i + 1]))
            assert e in r.adj, f"hop {i} is not an edge"
            assert r.adj[e] == int(attrs[i]), f"hop {i}'s attr is not adjacencyMap's last writer"
            assert r.dist[int(uids[i + 1])][0] == i + 1, f"hop {i + 1} is not at its BFS level"
    return L


@pytest.mark.parametrize("part", range(6))
def test_restatement_equals_formula(part):
    rng = np.random.default_rng(1600 + part)
    reached = 0
    for _ in range(500):
        g, frm, to, hops = gs.random_case(rng)
        for seed in SEEDS:
            reached += bool(check_against_restatement(g, frm, to, hops, seed))
    assert reached > 250, "the generator reaches To often enough to test paths"


def test_multi_predicate_overrides_and_depth():
    # 1 -> 2 over both predicates: the later child's attr wins; 2 -> 3 only over p1; depth 1 stops before 3
    p0 = gs.pred_from_edges(5, [1], [2])
    p1 = gs.pred_from_edges(5, [1, 2], [2, 3])
    g = gs.Graph(5, [p0, p1], [(0, None), (1, None)])
    for seed in SEEDS:
        assert check_against_restatement(g, 1, 3, None, seed) == 2
        assert check_against_restatement(g, 1, 3, 1, seed) == 0
    f = gs.Formula(1, 3)
    lv = gs.search(g, 1, 3, None, f.expand)
    assert [st for _, _, st in lv] == [(2, 1, 0), (2, 1, 2)]  # (1, 2) and (2, 3) count once per sg holding them
    assert f.path()[1].tolist() == [1, 1]


def test_self_loops_and_unreachable():
    g = gs.Graph(6, [gs.pred_from_edges(6, [1, 1, 2, 2, 4], [1, 2, 2, 3, 5])], [(0, None)])
    for seed in SEEDS:
        assert check_against_restatement(g, 1, 5, None, seed) == 0
        assert check_against_restatement(g, 1, 3, None, seed) == 2



def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(_golden()["cases"]))
def test_reference_queries(name):
    """The reference's shortest-path tests at the uid and attr level: the formula's path and hop attrs, the weight and
    the names of `me`, and the restatement agreeing with the formula under every neighbour order."""
    d = _golden()
    want = d["cases"][name]
    g, frm, to, preds = gs.fixture_case(d, name)
    f = gs.Formula(frm, to)
    gs.search(g, frm, to, None, f.expand)
    uids, attrs = f.path()
    assert uids.tolist() == want["path"]
    assert [preds[a] for a in attrs.tolist()] == want["attrs"]
    assert (f.to_level or None) == want["weight"]
    assert [d["names"][str(u)] for u in uids.tolist()] == want["me"]
    for seed in SEEDS:
        assert check_against_restatement(g, frm, to, None, seed) == max(len(want["path"]) - 1, 0)
        r = so.run(g, frm, to, None, seed)
        assert r.path.tolist() == want["path"]
        assert [preds[r.dist[int(v)][2]] for v in r.path[1:]] == want["attrs"], "Go's dist attrs"

def _lib():
    from dgraph_b200 import _lib
    return _lib


def test_create_refusals_need_no_device():
    L = _lib()
    h = C.c_void_p()
    for frm, to in ((0, 5), (5, 0), (7, 7)):
        assert L.load().dgx_path_create(frm, to, C.byref(h)) == L.DGX_ERR_ARG
        assert not h.value
    assert L.load().dgx_path_create(1, 2, None) == L.DGX_ERR_ARG


def test_expand_argument_errors_leave_outputs_untouched():
    L = _lib()
    lib = L.load()

    def call(sgs, mutate=None, next_cap=None, null_next=False):
        arrs = list(__import__("dgraph_b200.algo", fromlist=["x"]).path_level_arrays(sgs))
        if mutate:
            mutate(arrs)
        lv = L.PathLevel(len(sgs), *[a.ctypes.data for a in arrs])
        d = int(arrs[5][-1])
        nxt, off = np.full(8, 7, np.uint64), np.full(len(sgs) + 1, 7, np.uint64)
        st = L.PathStats(7, 7, 7)
        rc = lib.dgx_path_expand(None, C.byref(lv), None if null_next else nxt.ctypes.data, off.ctypes.data,
                                 d if next_cap is None else next_cap, C.byref(st))
        assert (nxt == 7).all() and (off == 7).all() and (st.edges, st.discovered, st.to_level) == (7, 7, 7)
        return rc, lib.dgx_last_error().decode()

    sgs = [(0, [1, 2], [[3, 4], [4]], [3, 4]), (1, [1], [[5]], [5])]
    rc, msg = call(sgs)
    assert rc == L.DGX_ERR_ARG and "null path search" in msg  # a well-formed level reaches the search check

    def bump(i, k, v):
        def f(a):
            a[i][k] = v
        return f

    assert call(sgs, bump(1, 0, 1))[0] == L.DGX_ERR_ARG             # src_off[0] != 0
    assert call(sgs, bump(1, 1, 3))[0] == L.DGX_ERR_ARG             # src_off decreases
    assert call(sgs, bump(3, 1, 0))[0] == L.DGX_ERR_ARG             # v_off decreases
    assert call(sgs, bump(3, 0, 1))[0] == L.DGX_ERR_ARG             # v_off[0] != 0
    assert call(sgs, bump(5, 1, 3))[0] == L.DGX_ERR_ARG             # dest_off decreases
    assert call(sgs, bump(1, 2, 1 << 32))[0] == L.DGX_ERR_ARG       # 2^32 rows
    assert call(sgs, next_cap=2)[0] == L.DGX_ERR_CAP                # next_cap below dest_off[nsg]
    assert call(sgs, null_next=True)[0] == L.DGX_ERR_ARG
    lv = L.PathLevel(0, *[np.zeros(2, np.uint64).ctypes.data] * 7)
    assert lib.dgx_path_expand(None, C.byref(lv), None, np.zeros(1, np.uint64).ctypes.data, 0,
                               C.byref(L.PathStats())) == L.DGX_ERR_ARG  # no sg


def test_launch_plan():
    K = shortest_plan.K
    assert K["FRONT"] == 5 and K["BACK"] == 6 and K["WALK"] == 1
    base = shortest_plan.launches(1, 1)
    assert base == 11 + 2 * (K["MERGE"] + 1)
    # the sg count never enters; rows and values only through the merges' sample trees
    assert shortest_plan.launches(10, 10) == base
    assert shortest_plan.launches(1, 4 * K["XM_T"]) == base + 1
    assert shortest_plan.launches(4 * K["XM_T"], 4 * K["XM_T"]) == base + 2
