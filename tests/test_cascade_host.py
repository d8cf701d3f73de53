"""@cascade on the host (no GPU): the line-by-line restatement of populateVarMap's cascade path (cascade_oracle.c)
against the independent numpy formula (gen_cascade.formula) over random forests, the argument and capacity errors
dgx_cascade refuses before it needs a device, and the launch plan model."""
from __future__ import annotations

import ctypes as C
import json
import os

import numpy as np
import pytest

import cascade_oracle as co
import cascade_plan
import gen_cascade as gc
from dgraph_b200 import _lib
from dgraph_b200.algo import CC_CASCADE, CC_CHECKED, CC_ORDERED, CC_SKIP, CascadeNode, cascade_arrays, cascade_tree

GUARD = np.uint64(0xA5A5A5A5DEADBEEF)


def same(a, b):
    (ra, da), (rb, db) = a, b
    return (len(ra) == len(rb) and all(np.array_equal(x, y) for x, y in zip(da, db)) and
            all(len(x) == len(y) and all(np.array_equal(u, v) for u, v in zip(x, y)) for x, y in zip(ra, rb)))


@pytest.mark.parametrize("seed", range(8))
def test_restatement_equals_formula(seed):
    rng = np.random.default_rng(1500 + seed)
    for _ in range(400):
        f = gc.random_forest(rng)
        assert same(co.cascade(f), gc.formula(f))


def test_page_range_matches_restatement():
    # a root with first / offset is filtered by its dest and paged; its one row of n values shows PageRange(first,
    # offset, n) through the restatement, against the closed form
    for n in range(0, 6):
        for first in [0, 1, 2, 5, 7, -1, -3, -6, -2**31, 2**31 - 1]:
            for offset in [0, 1, 3, 6, -1, -2**31, 2**31 - 1]:
                d = np.arange(1, n + 1, dtype=np.uint64)
                rows, _ = co.cascade([CascadeNode(-1, CC_CASCADE, first, offset, 0, d, [d])])
                s, e = gc.page_range(first, offset, n)
                assert rows[0][0].tolist() == d[s:e].tolist(), (n, first, offset)


def host_call(a, out_cap=None, dest_cap=None, tree=None, **arr):
    """dgx_cascade over the arrays of cascade_arrays (any replaced through arr; None passes NULL), with guard words
    in and past every output.  Returns (rc, out, out_off, dest_out, dest_off)."""
    m, nd = int(a["v_off"][-1]), int(a["dest_off"][-1])
    out = np.full(max(m, 1) + 4, GUARD, np.uint64)
    dout = np.full(max(nd, 1) + 4, GUARD, np.uint64)
    out_off = np.full(int(a["row_off"][-1]) + 5, GUARD, np.uint64)
    a = dict(a, **arr)
    dest_off = np.full(a["nnodes"] + 5, GUARD, np.uint64)
    t = cascade_tree(a) if tree is None else tree
    p = lambda k: None if a[k] is None else a[k].ctypes.data  # noqa: E731
    rc = _lib.load().dgx_cascade(C.byref(t), p("v"), p("v_off"), p("row_off"), p("dest"), p("dest_off"),
                                 p("has_val"), p("hv_off"), out.ctypes.data, out_off.ctypes.data,
                                 m if out_cap is None else out_cap, dout.ctypes.data, dest_off.ctypes.data,
                                 nd if dest_cap is None else dest_cap)
    return rc, out, out_off, dout, dest_off


def untouched(*arrs):
    return all(bool(np.all(x == GUARD)) for x in arrs)


def small_forest():
    d = np.array([1, 2, 3], np.uint64)
    return [CascadeNode(-1, CC_CASCADE, 0, 0, 0, d, [d]),
            CascadeNode(0, CC_CASCADE | CC_CHECKED, 0, 0, 0, np.array([5, 6], np.uint64),
                        [[5], [], [6]], [0, 1]),
            CascadeNode(1, CC_CHECKED, 0, 0, 0, np.array([9], np.uint64), [[9], []])]


def test_argument_errors_leave_outputs_untouched():
    a = cascade_arrays(small_forest())
    ARG, CAP = _lib.DGX_ERR_ARG, _lib.DGX_ERR_CAP

    def refused(code, **kw):
        rc, *outs = host_call(a, **kw)
        assert rc == code, (_lib.load().dgx_last_error(), kw.keys())
        assert untouched(*outs)

    bad = a["parent"].copy()
    bad[2] = 2
    refused(ARG, parent=bad)
    bad = a["flags"].copy()
    bad[1] |= 32
    refused(ARG, flags=bad)
    bad = a["flags"].copy()
    bad[1] |= CC_SKIP  # a SKIP node with a child
    refused(ARG, flags=bad)
    bad = a["row_off"].copy()
    bad[0] = 1
    refused(ARG, row_off=bad)
    bad = a["v_off"].copy()
    bad[2] = bad[1] - 1  # decreasing
    refused(ARG, v_off=bad)
    bad = a["dest_off"].copy()
    bad[1] = 7
    refused(ARG, dest_off=bad)
    bad = a["hv_off"].copy()
    bad[2] = bad[3] + 1
    refused(ARG, hv_off=bad)
    big = a["v_off"].copy()
    big[-1] = 1 << 32  # 2^32 values in all: refused before v is read
    refused(ARG, v_off=big)
    for k in ("v", "dest", "has_val", "row_off", "v_off", "dest_off", "hv_off"):
        refused(ARG, **{k: None})
    refused(ARG, tree=_lib.CascadeTree(1 << 16, *[a[k].ctypes.data for k in ("parent", "flags", "first", "offset",
                                                                             "counts_len")]))
    refused(ARG, tree=_lib.CascadeTree(3, None, a["flags"].ctypes.data, a["first"].ctypes.data,
                                       a["offset"].ctypes.data, a["counts_len"].ctypes.data))
    refused(CAP, out_cap=int(a["v_off"][-1]) - 1)
    refused(CAP, dest_cap=int(a["dest_off"][-1]) - 1)
    rc = _lib.load().dgx_cascade(None, *[None] * 8, None, 0, None, None, 0)
    assert rc == ARG


def test_depth_limit():
    depth = cascade_plan.K["MAX_DEPTH"]
    chain = [CascadeNode(k - 1, 0) for k in range(depth + 1)]  # depths 0 .. depth
    rc, *outs = host_call(cascade_arrays(chain))
    assert rc == _lib.DGX_ERR_ARG and untouched(*outs)


def test_no_device_needed_without_work():
    # an empty forest, and a forest with no dest value and no row value, write zero offsets without a device
    a = cascade_arrays([])
    out_off, dest_off = np.full(2, GUARD, np.uint64), np.full(2, GUARD, np.uint64)
    rc = _lib.load().dgx_cascade(C.byref(cascade_tree(a)), *[None] * 7, None, out_off.ctypes.data, 0, None,
                                 dest_off.ctypes.data, 0)
    assert rc == 0 and out_off[0] == 0 and dest_off[0] == 0 and out_off[1] == GUARD and dest_off[1] == GUARD
    f = [CascadeNode(-1, CC_CASCADE, 2, 1, 0, [], [[]]), CascadeNode(0, CC_CASCADE | CC_CHECKED, 0, 0, 0, [], [],
                                                                      [1, 0])]
    rc, out, out_off, dout, dest_off = host_call(cascade_arrays(f))
    assert rc == 0 and out_off[:2].tolist() == [0, 0] and dest_off[:3].tolist() == [0, 0, 0]
    assert untouched(out, dout, out_off[2:], dest_off[3:])


def test_launch_plan():
    K = cascade_plan.K
    assert (K["A"], K["B"]) == (4, 7)
    assert cascade_plan.launches(0) == 0 and cascade_plan.launches(1) == 11 and cascade_plan.launches(8) == 60
    api = cascade_plan._src("dgx_api.cu")
    with pytest.raises(ValueError):
        cascade_plan.read_constants(api.replace("count_launches(l, 4 + 7 * (int)D);", "count_launches(l, 5 + 7 * (int)D);"))
    with pytest.raises(ValueError):
        cascade_plan.read_constants(api.replace("        cc_page_kernel<<<gb_grid(L.nv), 256, 0, l->stream>>>(P, L);\n",
                                                ""))
    f = gc.random_forest(np.random.default_rng(3))
    assert 1 <= gc.levels_with_work(f) <= 8


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cascade_person.json")


def golden_forest(d, case):
    """The forest of one reference query over the fixture: a root from its func (uid order, or the name order of
    orderasc: name as ORDERED rows), a value predicate as a node with has_val only, friend as a node with its rows and
    DestUIDs, @cascade (__all__) reaching every node below it, first / offset inside a cascade as Cascade.First /
    Offset.  Returns (nodes, each node's spec)."""
    adj = {}
    for f, t in d["friend"]:
        adj.setdefault(f, []).append(t)
    has = {p: set(u) for p, u in d["has"].items()}
    r = case["root"]
    func = r["func"]
    row = d[func] if isinstance(func, str) else func
    dest = sorted(row)
    flags = (CC_CASCADE if r["cascade"] else 0) | (CC_ORDERED if row != dest else 0)
    nodes = [CascadeNode(-1, flags, r.get("first", 0), r.get("offset", 0), 0, dest, [row])]
    specs = [{"pred": "me"}]

    def add(spec, parent, cascade):
        pdest = nodes[parent].dest.tolist()
        casc = cascade or spec.get("cascade", False)
        flags = (CC_CASCADE if casc else 0) | (CC_CHECKED if cascade else 0)
        first, offset = (spec.get("first", 0), spec.get("offset", 0)) if casc else (0, 0)
        if spec["pred"] == "friend":
            rows = [sorted(adj.get(u, [])) for u in pdest]
            nd = CascadeNode(parent, flags, first, offset, 0, sorted({x for r in rows for x in r}), rows)
        else:
            nd = CascadeNode(parent, flags, 0, 0, 0, [], [], [int(u in has[spec["pred"]]) for u in pdest])
        k = len(nodes)
        nodes.append(nd)
        specs.append(spec)
        for c in spec.get("children", []):
            add(c, k, casc)

    for c in case["children"]:
        add(c, 0, r["cascade"])
    return nodes, specs


def render(nodes, specs, rows, dests):
    """The result as uids, the way the JSON output nests it: the root's row restricted to its DestUIDs, then under
    each uid the row of each uid predicate that is not empty."""
    kids = [[k for k, nd in enumerate(nodes) if nd.parent == p] for p in range(len(nodes))]

    def obj(k, u):
        o = {"uid": int(u)}
        i = nodes[k].dest.tolist().index(u)
        for c in kids[k]:
            if specs[c]["pred"] == "friend" and i < len(rows[c]) and rows[c][i].size:
                o["friend"] = [obj(c, x) for x in rows[c][i].tolist()]
        return o

    final = set(dests[0].tolist())
    return [obj(0, u) for u in rows[0][0].tolist() if u in final]


@pytest.mark.parametrize("name", ["TestCascadeDirective", "TestCascadeWithPaginationDeep",
                                  "TestCascadeWithPaginationAtRoot", "TestCascadeWithPaginationAndOffsetZero",
                                  "TestCascadeWithSort", "TestCascadeRepeatedMultipleLevels"])
def test_reference_queries(name):
    with open(GOLDEN) as f:
        d = json.load(f)
    nodes, specs = golden_forest(d, d["cases"][name])
    got = co.cascade(nodes)
    assert same(got, gc.formula(nodes))
    assert render(nodes, specs, *got) == d["cases"][name]["want"]
