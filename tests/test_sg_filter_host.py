"""@filter and first / offset on the host (no GPU): the line-by-line restatement of ProcessGraph's filter block
(sg_filter_oracle.c) against the independent per-D0 formula (gen_sg_filter.formula) over random trees, every argument
and capacity error dgx_sg_filter refuses before it needs a device, and the launch plan model."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import gen_sg_filter as gs
import sg_filter_golden as sgg
import sg_filter_oracle as so
import sg_filter_plan as sp
from dgraph_b200 import _lib
from dgraph_b200.algo import SubgraphFilter, sg_filter_flat, sg_filter_leaf_arrays, sg_filter_tree

GUARD = np.uint64(0xA5A5A5A5DEADBEEF)


def agree(a, b):
    return ([r.tolist() for r in a[0]] == [list(map(int, r)) for r in b[0]] and a[1].tolist() == list(b[1]) and
            a[2].tolist() == list(map(int, b[2])))


@pytest.mark.parametrize("seed", range(10))
def test_restatement_equals_formula(seed):
    rng = np.random.default_rng(1800 + seed)
    for _ in range(400):
        case = gs.random_case(rng)
        assert agree(so.sg_filter(*case), gs.formula(*case)), case


@pytest.mark.parametrize("label,case,counts_only,want", sgg.cases(), ids=[c[0] for c in sgg.cases()])
def test_reference_answers(label, case, counts_only, want):
    # the published answers of the reference's @filter tests, through the restatement and the formula
    for got in (so.sg_filter(*case), gs.formula(*case)):
        assert sgg.check(got, want), label


def test_reference_answers_catch_a_wrong_resolution():
    # the fixture tells a COUNT leaf read the wrong way round apart: has(friend) as "no friend" fails the answer
    label, case, _, want = [c for c in sgg.cases() if c[0] == "TestHasFuncAtRootFilter"][0]
    tree, leaves, *rest = case
    flipped = [("count", "le", 0, leaves[0][3])]
    assert not sgg.check(so.sg_filter(tree, flipped, *rest), want)


def test_count_leaf_arrays_must_match_d0():
    # the library copies n0 counts or n0 + 1 offsets: a shorter array is refused before the call
    d0 = np.array([2, 4, 6], np.uint64)
    for lf in (("count", "gt", 0, np.zeros(2, np.uint32)), ("len", "gt", 0, np.zeros(3, np.uint64)),
               ("count", "gt", 0, np.zeros(0, np.uint32))):
        with pytest.raises(ValueError, match="expected"):
            sg_filter_leaf_arrays([lf], d0.size)
        with pytest.raises(ValueError, match="expected"):
            SubgraphFilter(0, [lf], d0, [d0])
    sg_filter_leaf_arrays([("count", "gt", 0, np.zeros(0, np.uint32)), ("len", "gt", 0, np.zeros(1, np.uint64))], 0)


def test_page_range_edges():
    # one row of n values, every value in D0 and kept: the row shows PageRange(count, offset, n) through the
    # restatement, against the slice rule of the formula
    for n in range(0, 6):
        d = np.arange(1, n + 1, dtype=np.uint64)
        for count in [0, 1, 2, 5, 7, -1, -3, -6, -2**31, 2**31 - 1]:
            for offset in [0, 1, 3, 6, -1, -2**31, 2**31 - 1]:
                case = (0, [("list", d)], d, [d], count, offset)
                rows, counts, dest = so.sg_filter(*case)
                want = gs.page(d.tolist(), count, offset)
                assert rows[0].tolist() == want and counts.tolist() == [len(want)], (n, count, offset)
                assert dest.tolist() == (d.tolist() if count == 0 and offset == 0 else want)


def test_traps():
    d0 = np.array([2, 4, 6], np.uint64)
    # a literal reaching outside D0 counts only inside it; a row value outside D0 never survives
    rows, _, dest = so.sg_filter(0, [("list", np.array([1, 4, 9], np.uint64))], d0, [np.array([1, 4, 9], np.uint64)])
    assert dest.tolist() == [4] and rows[0].tolist() == [4]
    # NOT of an empty leaf is D0; nested NOT is the leaf
    assert so.sg_filter(("not", 0), [("list", [])], d0, [])[2].tolist() == [2, 4, 6]
    assert so.sg_filter(("not", ("not", 0)), [("list", [4])], d0, [])[2].tolist() == [4]
    # an empty D0: every output is empty, whatever the leaves
    r = so.sg_filter(("not", 0), [("list", [])], np.zeros(0, np.uint64), [np.array([1, 2], np.uint64)], 1, 0)
    assert r[0][0].tolist() == [] and r[1].tolist() == [0] and r[2].tolist() == []


def call(case, counts_only=False, dest_cap=None, out_cap=None, tree=None, leaves=None, nleaves=None, **ptr):
    """dgx_sg_filter with guard words; ptr replaces an argument with None (NULL).  Returns (rc, outputs untouched)."""
    t_, lv, d0, rows, count, offset = case
    f = sg_filter_flat(t_)
    d0 = np.ascontiguousarray(np.asarray(d0, np.uint64))
    keep, tab = sg_filter_leaf_arrays(lv, d0.size)
    v = np.concatenate([np.asarray(r, np.uint64) for r in rows] + [np.zeros(1, np.uint64)])
    v_off = ptr.pop("v_off_arr", None)
    if v_off is None:
        v_off = np.zeros(len(rows) + 1, np.uint64)
        np.cumsum([len(r) for r in rows], out=v_off[1:])
    nrows, m = len(rows), int(v_off[-1])
    dest = np.full(max(d0.size, 1) + 4, GUARD, np.uint64)
    out = np.full(max(m, 1) + 4, GUARD, np.uint64)
    oo = np.full(nrows + 5, GUARD, np.uint64)
    cnt = np.full(nrows + 4, 0xA5A5A5A5, np.uint32)
    n = C.c_size_t(12345)
    t = sg_filter_tree(f) if tree is None else tree
    args = {"d0": d0.ctypes.data if d0.size else None, "v": v.ctypes.data, "v_off": v_off.ctypes.data,
            "dest": dest.ctypes.data, "len": C.byref(n), "out": None if counts_only else out.ctypes.data,
            "oo": oo.ctypes.data, "cnt": cnt.ctypes.data}
    args.update(ptr)
    rc = _lib.load().dgx_sg_filter(C.byref(t) if t is not False else None, tab if leaves is None else leaves,
                                   len(lv) if nleaves is None else nleaves, args["d0"], d0.size, args["v"],
                                   args["v_off"], nrows, count, offset, args["dest"],
                                   d0.size if dest_cap is None else dest_cap, args["len"], args["out"], args["oo"],
                                   m if out_cap is None else out_cap, args["cnt"])
    del keep
    untouched = (np.all(dest == GUARD) and np.all(out == GUARD) and np.all(oo == GUARD) and np.all(cnt == 0xA5A5A5A5)
                 and n.value == 12345)
    return rc, untouched


BASE = (("or", [("and", [0, 1]), ("not", 2)]),
        [("list", np.array([1, 4, 6, 9], np.uint64)), ("count", "gt", 1, np.array([0, 2, 3, 1], np.uint32)),
         ("len", "ge", 1, np.array([0, 1, 1, 3, 3], np.uint64))],
        np.array([2, 4, 6, 8], np.uint64), [np.array([2, 4], np.uint64), np.array([6, 8, 9], np.uint64)], 1, 0)


def flat_tree(op, parent, leaf):
    a = {"op": np.array(op, np.uint8), "parent": np.array(parent, np.uint32), "leaf": np.array(leaf, np.uint32)}
    return a, _lib.SgFilterTree(len(op), a["op"].ctypes.data, a["parent"].ctypes.data, a["leaf"].ctypes.data)


def test_argument_and_capacity_errors():
    ARG, CAP = _lib.DGX_ERR_ARG, _lib.DGX_ERR_CAP
    assert call(BASE, dest_cap=3) == (CAP, True)
    assert call(BASE, out_cap=4) == (CAP, True)
    for k in ("len", "v_off", "oo", "cnt", "dest", "d0", "v"):
        assert call(BASE, **{k: None}) == (ARG, True), k
    assert call(BASE, tree=False) == (ARG, True)
    u32 = 0xFFFFFFFF
    bad_trees = [([], [], []),                      # no node
                 ([9], [u32], [0]),                 # unknown op
                 ([1, 0, 0], [u32, 2, 0], [0, 0, 0]),  # a parent above its child
                 ([0, 0], [u32, 0], [0, 0]),        # a leaf as parent
                 ([3, 0, 0], [u32, 0, 0], [0, 0, 1]),  # NOT with two children
                 ([1], [u32], [0]),                 # AND without children
                 ([0], [u32], [7]),                 # a leaf index past the leaves
                 ([3] * 66 + [0], [u32] + list(range(66)), [0] * 67)]  # deeper than 64
    for op, par, lf in bad_trees:
        keep, t = flat_tree(op, par, lf)
        assert call(BASE, tree=t) == (ARG, True), op[:4]
    keep, t = flat_tree([3] * 64 + [0], [u32] + list(range(64)), [0] * 65)  # depth 64 is allowed
    assert call(BASE, tree=t)[0] != ARG
    # leaves: unknown kind, COUNT with both or neither array, unknown cmp, a null LIST with uids
    L = _lib.SgFilterLeaf
    cnt = np.zeros(4, np.uint32)
    off = np.zeros(5, np.uint64)
    for lf in (L(5, 0, 0, None, 0, None, None, None), L(1, 0, 0, None, 0, None, cnt.ctypes.data, off.ctypes.data),
               L(1, 0, 0, None, 0, None, None, None), L(1, 7, 0, None, 0, None, cnt.ctypes.data, None),
               L(0, 0, 0, None, 3, None, None, None), L(0, 0, 0, off.ctypes.data, 3, off.ctypes.data, None, None)):
        tab = (L * 3)(lf, lf, lf)
        assert call(BASE, leaves=tab) == (ARG, True)
    assert call(BASE, nleaves=2000) == (ARG, True)
    # row offsets not starting at 0 or decreasing
    assert call(BASE, v_off_arr=np.array([1, 2, 5], np.uint64)) == (ARG, True)
    assert call(BASE, v_off_arr=np.array([0, 3, 2], np.uint64)) == (ARG, True)
    # counts-only mode needs no value room
    assert call(BASE, counts_only=True, out_cap=0)[0] != CAP


def test_empty_d0_needs_no_device():
    case = (("not", 0), [("list", [])], np.zeros(0, np.uint64), [np.array([3, 5], np.uint64), np.zeros(0)], 2, 1)
    f = sg_filter_flat(case[0])
    keep, tab = sg_filter_leaf_arrays(case[1], 0)
    v = np.array([3, 5], np.uint64)
    v_off = np.array([0, 2, 2], np.uint64)
    oo = np.full(3, GUARD, np.uint64)
    cnt = np.full(2, 7, np.uint32)
    n = C.c_size_t(9)
    t = sg_filter_tree(f)
    rc = _lib.load().dgx_sg_filter(C.byref(t), tab, 1, None, 0, v.ctypes.data, v_off.ctypes.data, 2, 2, 1, None, 0,
                                   C.byref(n), None, oo.ctypes.data, 0, cnt.ctypes.data)
    assert rc == _lib.DGX_OK and n.value == 0 and oo.tolist() == [0, 0, 0] and cnt.tolist() == [0, 0]


def test_launch_plan_model():
    assert sp.K["LAUNCHES"] == 11 and sp.launches(0) == 0 and sp.launches(1) == sp.launches(10**7) == 11
    assert (sp.K["MAX_NODES"], sp.K["MAX_LEAVES"], sp.K["MAX_DEPTH"]) == (1024, 1024, 64)
    api = open(sp.os.path.join(sp.CSRC, "dgx_api.cu")).read()
    with pytest.raises(ValueError, match="restate"):
        sp.read_constants(api.replace("count_launches(l, 11);", "count_launches(l, 12);"))
    with pytest.raises(ValueError, match="restate"):
        sp.read_constants(api.replace("sf_out_kernel<<<", "sf_out2_kernel<<<"))
