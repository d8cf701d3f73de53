"""@groupby over one uid attribute on the CPU: the line-by-line restatement (groupby_oracle.c) against the numpy
formula (gen_groupby.py) on random cases, the reference's known answers, and the plan model's reading of the sources.
No GPU needed."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen_groupby as gg  # noqa: E402
import groupby_oracle as gbo  # noqa: E402
import groupby_plan as gp  # noqa: E402

U64_MAX = gg.U64_MAX
FRIEND_SRC = [1, 23, 31]  # query/common_test.go:513-519: 1 -> {23, 24, 25, 31, 101}, 31 -> {24}, 23 -> {1}
FRIEND_ROWS = [[23, 24, 25, 31, 101], [1], [24]]


def _same(a, b):
    for x, y, name in zip(a, b, ("keys", "counts", "grp_off", "mem_off", "members")):
        assert np.array_equal(np.asarray(x, np.uint64), np.asarray(y, np.uint64)), name


@pytest.mark.parametrize("kind", ["small", "high", "mixed", "hub"])
def test_oracle_equals_formula(kind):
    rng = np.random.default_rng({"small": 1, "high": 2, "mixed": 3, "hub": 4}[kind])
    for _ in range(800):
        parents, src, rows, dest = gg.case(rng, kind)
        _same(gbo.groupby_uid(parents, src, rows), gg.groupby_uid(parents, src, rows))


def test_one_and_many_parents_and_empty_rows():
    rng = np.random.default_rng(5)
    for npar in (0, 1, 64):
        for nrows in (0, 1, 300):
            parents, src, rows, dest = gg.case(rng, "mixed", nrows=nrows, npar=npar, nd=50)
            _same(gbo.groupby_uid(parents, src, rows), gg.groupby_uid(parents, src, rows))


def test_friends_multiple_parents():
    """TestGroupByFriendsMultipleParents (query/query0_test.go:1798-1816)."""
    keys, counts, grp_off, mem_off, mem = gbo.groupby_uid([[23, 24, 25, 31, 101], [1], [24]], FRIEND_SRC, FRIEND_ROWS)
    groups = [[(int(keys[g]), mem[mem_off[g]:mem_off[g + 1]].tolist()) for g in range(grp_off[p], grp_off[p + 1])]
              for p in range(3)]
    assert groups[0] == [(1, [23]), (24, [31])]
    assert groups[1] == [(23, [1]), (24, [1]), (25, [1]), (31, [1]), (101, [1])]
    assert groups[2] == []
    assert counts.tolist() == [1] * 7


def test_friends_multiple_parents_var():
    """TestGroupByFriendsMultipleParentsVar (query/query0_test.go:1818-1836): fillGroupedVars, one parent = SrcUIDs."""
    assert gbo.grouped_vars(FRIEND_SRC, FRIEND_ROWS) == {24: 2, 1: 1, 23: 1, 25: 1, 31: 1, 101: 1}
    keys, counts, _, mem_off, mem = gbo.groupby_uid([FRIEND_SRC], FRIEND_SRC, FRIEND_ROWS)
    g = keys.tolist().index(24)
    assert mem[mem_off[g]:mem_off[g + 1]].tolist() == [1, 31]
    assert keys[-1] == 24  # the largest group orders last


def test_uids_at_the_ends():
    src = [0, 5, U64_MAX]
    rows = [[U64_MAX], [0, U64_MAX], [0]]
    want = gg.groupby_uid([[0, U64_MAX], src], src, rows)
    _same(gbo.groupby_uid([[0, U64_MAX], src], src, rows), want)
    assert want[0].tolist() == [0, U64_MAX, 0, U64_MAX]


def test_plan_constants_and_formula():
    K = gp.K
    assert K["FRONT"] == 3 and K["BACK"] == 8 and K["SORT_PER_PASS"] == 3 and K["DIGIT_BITS"] == 8
    assert gp.plan(1, 1, 1) == {"b_p": 0, "b_d": 0, "b_s": 1, "p1": 0, "p2": 1}
    # a pass per 8 bits of key: 1e6 rows and destinations under one parent sort 20-bit keys twice
    assert gp.plan(10 ** 6, 10 ** 6, 1)["p1"] == 3 and gp.plan(10 ** 6, 10 ** 6, 1)["p2"] == 3
    assert gp.launches(10, 10, 10, 5, 5, 5) == 11 + 3 * (1 + 1)
    assert gp.launches(10, 10, 0, 5, 5, 5) == 0 and gp.launches(10, 10, 3, 5, 5, 0) == 3
    # the launch count does not depend on the number of parents, rows or edges at the same key widths
    assert len({gp.launches(n, 200, n, 10 * n, 10 * n, 7 * n) for n in (129, 200, 255)}) == 1


def test_plan_rewrites_raise():
    api, kern = gp._src("dgx_api.cu"), gp._src("groupby_kernel.cuh")
    for a, b in (("g.b_s = gb_bits(nrows);", "g.b_s = gb_bits(nrows + 1);"),
                 ("gb_heads_kernel<<<", "gb_heads_kernel<<<1, 1>>>(P); gb_heads_kernel<<<"),
                 ("gb_scatter_kernel<<<", "gb_scatter_kernel("),
                 ("GB_RADIX = 256, GB_DIGIT_BITS = 8;", "GB_RADIX = 256, GB_DIGIT_BITS = 4;")):
        assert (a in api) != (a in kern), a
        with pytest.raises(ValueError):
            gp.read_constants(api.replace(a, b), kern.replace(a, b))
