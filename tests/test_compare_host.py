"""The compare functions on the host side (no GPU): the line-by-line restatement (compare_oracle.c) against the
independent formula (gen_compare.py) on seeded cases, the pinned Go corners, CompareRowArgs for Go's three cases of
handleCompareFunction, and every refusal dgx_compare_uids / dgx_compare_rows make before anything is copied."""
import ctypes as C

import numpy as np
import pytest

import compare_oracle as co
import gen_compare as gc
from dgraph_b200 import _lib, algo

NAN, INF = float("nan"), float("inf")


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("seed", range(4))
def test_restatement_matches_formula(seed):
    rng = np.random.default_rng(1000 + seed)
    for _ in range(1500):
        typ, uids, values, bad, op, args, cands = gc.rand_case(rng)
        col = gc.column(typ, uids, values, bad)
        assert _same(co.compare_uids(col, op, args, cands), gc.compare_uids(typ, uids, values, bad, op, args, cands)), \
            (typ, op, args, values, bad, cands)
        rows = [np.asarray(rng.permutation(cands)[: int(rng.integers(0, cands.size + 1))], np.uint64)
                for _ in range(int(rng.integers(0, 4)))]
        span = 2 if op == "between" else 1
        ra = [int(rng.integers(0, len(args) - span + 1)) if rng.random() < 0.7 else algo.CMP_NO_ARG for _ in rows]
        want = gc.compare_rows(typ, uids, values, bad, op, args, rows, ra)
        got = co.compare_rows(col, op, args, rows, ra)
        assert [g.tolist() for g in got] == [w.tolist() for w in want], (typ, op, args, values, rows, ra)


def _one(typ, op, args, vals):
    col = algo.ValColumn(typ, np.arange(1, len(vals) + 1), [[v] for v in vals])
    return co.compare_uids(col, op, args, np.arange(1, len(vals) + 1, dtype=np.uint64))[0].tolist()


def test_go_corners():
    F = algo.VAL_FLOAT64
    vals = [NAN, -0.0, 0.0, 1.0]
    # a NaN value satisfies ge, le and between, not gt, lt or eq
    assert _one(F, "ge", [0.5], vals) == [1, 4]
    assert _one(F, "le", [0.5], vals) == [1, 2, 3]
    assert _one(F, "between", [0.5, 2.0], vals) == [1, 4]
    assert _one(F, "gt", [0.5], vals) == [4] and _one(F, "lt", [0.5], vals) == [2, 3] and _one(F, "eq", [NAN], vals) == []
    # a NaN argument makes ge / le true for every value and gt / lt / eq false
    assert _one(F, "ge", [NAN], vals) == _one(F, "le", [NAN], vals) == [1, 2, 3, 4]
    assert _one(F, "gt", [NAN], vals) == _one(F, "lt", [NAN], vals) == []
    assert _one(F, "eq", [-0.0], vals) == [2, 3]
    # between with a > b is empty
    assert _one(F, "between", [2.0, 0.5], [1.0, 1.5]) == []
    assert _one(algo.VAL_STRING, "between", ["Alice", ""], ["Alice", "Bob", ""]) == []
    # int64: signed order
    assert _one(algo.VAL_INT64, "lt", [0], [-2 ** 63, 2 ** 63 - 1, 0]) == [1]
    # datetime: the instant, seconds then nanoseconds; before 1970 negative
    T = algo.VAL_DATETIME
    assert _one(T, "lt", [(0, 0)], [(-14516064000, 0), (0, 1), (-1, 999999999)]) == [1, 3]
    assert _one(T, "eq", [(5, 7)], [(5, 7), (5, 8)]) == [1]
    # bool: only eq
    for op in ("ge", "le", "gt", "lt"):
        assert _one(algo.VAL_BOOL, op, [True], [True, False]) == []
    assert _one(algo.VAL_BOOL, "eq", [False], [True, False]) == [2]
    # strings: bytewise unsigned, a proper prefix less, NUL and high bytes
    S = algo.VAL_STRING
    assert _one(S, "lt", ["ab"], [b"a", b"ab", b"ab\x00", b"\xff", b""]) == [1, 5]
    assert _one(S, "gt", [b"\x7f"], [b"\x80", b"\x7f", b"\x7f\x00"]) == [1, 3]
    assert _one(S, "eq", [""], [b"", b"\x00"]) == [1]


def test_list_values_and_errors():
    col = algo.ValColumn(algo.VAL_INT64, [1, 2, 3], [[5, 5, 9], [1], []], bad=[[False, False, False], [True], []])
    # eq with several arguments: break after the first hit, so a value counts once; k matching values append k times
    dest, rl = co.compare_uids(col, "eq", [5, 9, 5], [1, 3])
    assert dest.tolist() == [1] and rl.tolist() == [3, 0]
    # a conversion error on a candidate's value fails the task; off the candidates it is never read
    assert co.compare_uids(col, "ge", [0], [1, 2]) is None
    # the index path skips it
    assert [r.tolist() for r in co.compare_rows(col, "ge", [0], [[2, 1]], [0])] == [[1]]


def test_row_args_go_cases():
    assert algo.CompareRowArgs("eq", 3, 3).tolist() == [0, 1, 2]
    # an earlier argument without a token still pairs row r with eqTokens[r]
    assert algo.CompareRowArgs("eq", 2, 3).tolist() == [0, 1]
    with pytest.raises(ValueError):
        algo.CompareRowArgs("eq", 4, 3)  # Go would index past eqTokens
    NO = algo.CMP_NO_ARG
    assert algo.CompareRowArgs("between", 4).tolist() == [0, NO, NO, 0]
    assert algo.CompareRowArgs("between", 1).tolist() == [0]
    assert algo.CompareRowArgs("ge", 3, 1, True).tolist() == [0, NO, NO]
    assert algo.CompareRowArgs("lt", 3, 1, False).tolist() == [NO, NO, NO]
    assert algo.CompareRowArgs("le", 0, 1, True).tolist() == []


def _refused(fn, code=_lib.DGX_ERR_ARG):
    with pytest.raises(_lib.DgxError) as e:
        fn()
    assert e.value.code == code


def test_refusals_before_copy():
    col = algo.ValColumn(algo.VAL_INT64, [1, 2], [[1], [2]])
    u = [1, 2]
    _refused(lambda: algo.CompareUids(col, 6, [1], u))                      # unknown op
    _refused(lambda: algo.CompareUids(col, "ge", [1, 2], u))                # one argument
    _refused(lambda: algo.CompareUids(col, "ge", [], u))
    _refused(lambda: algo.CompareUids(col, "eq", [], u))                    # at least one
    _refused(lambda: algo.CompareUids(col, "between", [1], u))              # exactly two
    _refused(lambda: algo.CompareUids(col, "between", [1, 2, 3], u))
    t = algo.ValColumn(algo.VAL_DATETIME, [1], [[(0, 0)]])
    _refused(lambda: algo.CompareUids(t, "ge", [(0, 10 ** 9)], [1]))        # argument nanoseconds
    bad_type = algo.ValColumn.from_arrays(7, [1], [0, 1], np.zeros(1, np.uint64))
    _refused(lambda: algo.CompareUids(bad_type, "ge", algo.ValArgs(algo.VAL_INT64, [1]), [1]))
    dec = algo.ValColumn.from_arrays(algo.VAL_INT64, [1, 2], [0, 2, 1], np.zeros(2, np.int64))
    _refused(lambda: algo.CompareUids(dec, "ge", [1], u))                   # column offsets decreasing
    short = algo.ValColumn.from_arrays(algo.VAL_INT64, [1, 2], [0, 1, 1], np.zeros(2, np.int64))
    short.val_off[-1] = 1
    cs = short.struct()
    cs.nvals = 2
    a = algo.ValArgs(algo.VAL_INT64, [1])
    ast = a.struct()
    uu = np.asarray(u, np.uint64)
    out = np.empty(2, np.uint64)
    n = C.c_size_t(0)
    L = _lib.load()
    assert L.dgx_compare_uids(1, C.byref(ast), C.byref(cs), uu.ctypes.data, 2, out.ctypes.data, 2, C.byref(n),
                              None) == _lib.DGX_ERR_ARG                     # val_off[n] != nvals
    assert L.dgx_compare_uids(1, C.byref(ast), C.byref(col.struct()), uu.ctypes.data, 2, out.ctypes.data, 1,
                              C.byref(n), None) == _lib.DGX_ERR_CAP        # out_cap below nuids
    assert L.dgx_compare_uids(1, None, C.byref(col.struct()), uu.ctypes.data, 2, out.ctypes.data, 2, C.byref(n),
                              None) == _lib.DGX_ERR_ARG                     # null arguments
    nul = col.struct()
    nul.word = None
    assert L.dgx_compare_uids(1, C.byref(ast), C.byref(nul), uu.ctypes.data, 2, out.ctypes.data, 2, C.byref(n),
                              None) == _lib.DGX_ERR_ARG                     # null column words
    s = algo.ValColumn(algo.VAL_STRING, [1], [[b"x"]])
    ss = s.struct()
    ss.str = None
    sa = algo.ValArgs(algo.VAL_STRING, ["x"]).struct()
    assert L.dgx_compare_uids(1, C.byref(sa), C.byref(ss), uu.ctypes.data, 1, out.ctypes.data, 2, C.byref(n),
                              None) == _lib.DGX_ERR_ARG                     # a string column without its str
    # the rows form: row_arg past the arguments, v_off, out_cap
    _refused(lambda: algo.CompareRows(col, "ge", [1], [[1, 2]], [1]))
    _refused(lambda: algo.CompareRows(col, "between", [1, 2], [[1, 2]], [1]))
    _refused(lambda: algo.CompareRows(col, "eq", [1, 2], [[1], [2]], [0, 2]))
    v = np.asarray([1, 2], np.uint64)
    ra = np.zeros(2, np.uint32)
    oo = np.zeros(3, np.uint64)
    cst = col.struct()
    for off, cap, code in (([1, 1, 2], 2, _lib.DGX_ERR_ARG), ([0, 2, 1], 2, _lib.DGX_ERR_ARG),
                           ([0, 1, 2], 1, _lib.DGX_ERR_CAP)):
        vo = np.asarray(off, np.uint64)
        assert L.dgx_compare_rows(1, C.byref(ast), C.byref(cst), v.ctypes.data, vo.ctypes.data, 2, ra.ctypes.data,
                                  out.ctypes.data, oo.ctypes.data, cap) == code
    assert L.dgx_compare_rows(1, C.byref(ast), C.byref(cst), v.ctypes.data, np.zeros(1, np.uint64).ctypes.data, 2,
                              None, out.ctypes.data, oo.ctypes.data, 2) == _lib.DGX_ERR_ARG  # null row_arg


def test_empty_calls_need_no_device():
    col = algo.ValColumn(algo.VAL_INT64, [1], [[1]])
    got, cnt = algo.CompareUids(col, "ge", [0], [], counts=True)
    assert got.Uids.size == 0 and cnt.size == 0
    assert algo.CompareRows(col, "ge", [0], [], []) == []


def test_golden_cases_on_the_restatement():
    """The published answers (tests/golden/compare_common.json) on the restatement and on the formula."""
    import compare_golden as cg

    G = cg.load()
    assert len(G["cases"]) == 36
    for c in G["cases"]:
        if c["path"] == "value":
            col, op, args, cands = cg.value_case(G, c)
            dest, rl = co.compare_uids(col, op, args, cands)
            assert dest.tolist() == c["want"], c["query"]
            typ, uids, values = col.type, *cg.column(G, c["pred"])[1:]
            assert gc.compare_uids(typ, uids, values, None, op, args, cands)[0].tolist() == c["want"]
        else:
            col, op, args, rows, ra = cg.index_case(G, c)
            got = co.compare_rows(col, op, args, rows, ra)
            assert cg.merged(got).tolist() == c["want"], c["query"]
            _, uids, values = cg.column(G, c["pred"])
            assert cg.merged(gc.compare_rows(col.type, uids, values, None, op, args, rows, ra)).tolist() == c["want"]


def test_golden_index_rows_take_go_cases():
    """The tokenizer-built rows hit each of Go's three row cases: between's rows 0 and last, row 0 when the first token
    is the argument's, and eq's one row per argument."""
    import compare_golden as cg

    G = cg.load()
    seen = set()
    for c in G["cases"]:
        if c["path"] != "index":
            continue
        _, op, _, rows, ra = cg.index_case(G, c)
        if op == "between" and len(rows) >= 3:
            assert ra[0] == 0 and ra[-1] == 0 and (ra[1:-1] == algo.CMP_NO_ARG).all()
            seen.add("between")
        if op in ("le", "lt", "gt") and len(rows) and ra[0] == 0:
            seen.add("first")
        if op == "eq":
            assert ra.tolist() == list(range(len(rows)))
            seen.add("eq")
    assert seen == {"between", "first", "eq"}
