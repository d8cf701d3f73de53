"""orderasc / orderdesc by a predicate on the host side (no GPU): the line-by-line restatement (pred_order_oracle.c)
against the independent formula (gen_pred_order.py) on seeded cases, against the order-by-variable restatement where
both apply, the launch plan, and every refusal dgx_pred_order makes before anything is copied."""
import ctypes as C

import numpy as np
import pytest

import gen_pred_order as gp
import pred_order_oracle as po
import pred_order_plan as pp
import var_order_oracle as vo
from dgraph_b200 import _lib, algo

NAN = float("nan")


@pytest.mark.parametrize("seed", range(6))
def test_restatement_matches_formula(seed):
    """6 000 seeded cases over the four types, weighted to ties, +-0, NaN, int64 extremes, pre-1970 datetimes, shared
    string prefixes, bad values and uids outside the column or dest."""
    rng = np.random.default_rng(2300 + seed)
    for _ in range(1000):
        case = gp.random_case(rng)
        got = po.pred_order(*case)
        full = po.pred_order(*case[:4]) if case[4] or case[5] else None
        gp.check(case, got[0], got[1], None if full is None else full[0])


@pytest.mark.parametrize("typ", [algo.VAL_INT64, algo.VAL_FLOAT64])
def test_restatement_matches_var_order_on_full_columns(typ):
    """With every U uid holding a value, sortWithoutIndex and sortAndPaginateUsingVar run the same comparator and the
    same driver: 1 000 seeded tied rows per type give the same answer."""
    rng = np.random.default_rng(77 + typ)
    for _ in range(1000):
        n = int(rng.integers(1, 300))
        uids = np.arange(1, n + 1, dtype=np.uint64) * 3
        if typ == algo.VAL_INT64:
            vals = rng.integers(-4, 4, n).astype(np.int64)
        else:
            vals = rng.choice(np.array([0.0, -0.0, 1.5, -2.0, NAN, np.inf]), n)
        col = algo.ValColumn(typ, uids, [[v] for v in vals.tolist()])
        rows = [np.sort(rng.choice(uids, int(rng.integers(0, n + 1)), replace=False)) for _ in range(3)]
        desc = bool(rng.random() < 0.5)
        count, offset = (0, 0) if rng.random() < 0.5 else (int(rng.integers(0, 20)), int(rng.integers(0, 20)))
        a = po.pred_order(col, desc, uids, rows, count, offset)
        b = vo.var_order((uids, vals), desc, uids, rows, count, offset)
        assert [r.tolist() for r in a[0]] == [r.tolist() for r in b[0]]
        assert a[1].tolist() == b[1].tolist()


def test_go_corners():
    s = algo.ValColumn(algo.VAL_STRING, [1, 2, 3, 4, 5, 6],
                       [[b"ab"], [b"ab\0"], [b""], [b"abcdefghB"], [b"abcdefghA"], [b"\xff"]])
    rows, dest = po.pred_order(s, False, [1, 2, 3, 4, 5, 6, 7], [[1, 2, 3, 4, 5, 6, 7]])
    assert rows[0].tolist() == [3, 1, 2, 5, 4, 6, 7]  # a proper prefix first, bytes unsigned, the null last
    rows, _ = po.pred_order(s, True, [1, 2, 3, 4, 5, 6, 7], [[1, 2, 3, 4, 5, 6, 7]])
    assert rows[0].tolist() == [6, 4, 5, 2, 1, 3, 7]  # desc: nulls still last
    t = algo.ValColumn(algo.VAL_DATETIME, [1, 2, 3], [[(-1, 5)], [(-1, 4)], [(-2, 999_999_999)]])
    assert po.pred_order(t, False, [1, 2, 3], [[1, 2, 3]])[0][0].tolist() == [3, 2, 1]
    b = algo.ValColumn(algo.VAL_INT64, [1, 2, 3], [[5], [1], [3]], bad=[[False], [True], [False]])
    rows, dest = po.pred_order(b, False, [1, 2, 3, 4], [[4, 3, 2, 1][::-1]], count=2, offset=1)
    assert rows[0].tolist() == [1, 2] and dest.tolist() == [1, 2]  # [3, 1, 2, 4] paged: the bad value is a null
    with pytest.raises(po.ListPredicate):
        po.pred_order(algo.ValColumn(algo.VAL_INT64, [1], [[1, 2]]), False, [1], [[1]])
    with pytest.raises(po.NegativeCount):
        po.pred_order(b, False, [1], [[1]], count=-1)


def test_launch_plan():
    assert pp.launches(algo.VAL_INT64, 1) == 38
    assert pp.launches(algo.VAL_STRING, 256) == 41
    assert pp.launches(algo.VAL_DATETIME, 257) == 57
    assert pp.launches(algo.VAL_FLOAT64, 65537) == 47


def _refused(fn, code=_lib.DGX_ERR_ARG):
    with pytest.raises(_lib.DgxError) as e:
        fn()
    assert e.value.code == code


def test_refusals_before_copy():
    col = algo.ValColumn(algo.VAL_INT64, [1, 2], [[1], [2]])
    _refused(lambda: algo.OrderByPred(algo.ValColumn(algo.VAL_BOOL, [1], [[True]]), False, [1], [[1]]))  # bool
    _refused(lambda: algo.OrderByPred(algo.ValColumn.from_arrays(7, [1], [0, 1], np.zeros(1, np.uint64)), False,
                                      [1], [[1]]))                                   # unknown type
    _refused(lambda: algo.OrderByPred(col, False, [1, 2], [[1, 2]], count=-1))     # negative count
    dec = algo.ValColumn.from_arrays(algo.VAL_INT64, [1, 2], [0, 2, 1], np.zeros(2, np.int64))
    _refused(lambda: algo.OrderByPred(dec, False, [1], [[1]]))                      # column offsets decreasing
    L = _lib.load()
    cs = col.struct()
    d = np.asarray([1, 2], np.uint64)
    v = np.asarray([1, 2], np.uint64)
    out = np.empty(2, np.uint64)
    oo = np.zeros(3, np.uint64)
    dout = np.empty(2, np.uint64)
    n = C.c_size_t(0)

    def call(cst=cs, dest=d.ctypes.data, nd=2, vo_=None, nrows=2, out_cap=2, dest_cap=2, vv=v.ctypes.data,
             o=out.ctypes.data, dl=C.byref(n)):
        off = np.asarray([0, 1, 2] if vo_ is None else vo_, np.uint64)
        return L.dgx_pred_order(C.byref(cst) if cst is not None else None, 0, dest, nd, vv, off.ctypes.data, nrows,
                                0, 0, o, oo.ctypes.data, out_cap, dout.ctypes.data, dest_cap, dl)

    assert call(cst=None) == _lib.DGX_ERR_ARG                        # null column
    assert call(nd=1 << 32) == _lib.DGX_ERR_ARG                      # a size of 2^32
    assert call(nrows=1 << 32) == _lib.DGX_ERR_ARG
    assert call(vo_=[1, 1, 2]) == _lib.DGX_ERR_ARG                   # v_off not starting at 0
    assert call(vo_=[0, 2, 1]) == _lib.DGX_ERR_ARG                   # v_off decreasing
    assert call(out_cap=1) == _lib.DGX_ERR_CAP                       # out_cap below v_off[nrows]
    assert call(dest_cap=1) == _lib.DGX_ERR_CAP                      # dest_cap below ndest
    assert call(dest=None) == _lib.DGX_ERR_ARG                       # null arrays
    assert call(vv=None) == _lib.DGX_ERR_ARG
    assert call(o=None) == _lib.DGX_ERR_ARG
    assert call(dl=None) == _lib.DGX_ERR_ARG
    nul = col.struct()
    nul.word = None
    assert call(cst=nul) == _lib.DGX_ERR_ARG                         # null column words
    big = col.struct()
    big.n = 1 << 32
    assert call(cst=big) == _lib.DGX_ERR_ARG                         # column size of 2^32
    t = algo.ValColumn(algo.VAL_DATETIME, [1], [[(0, 0)]]).struct()
    t.nsec = None
    assert call(cst=t) == _lib.DGX_ERR_ARG                           # datetime without nanoseconds
    s = algo.ValColumn(algo.VAL_STRING, [1], [[b"x"]]).struct()
    s.str = None
    assert call(cst=s) == _lib.DGX_ERR_ARG                           # a string column without its str


def test_empty_calls_need_no_device():
    col = algo.ValColumn(algo.VAL_STRING, [1], [["a"]])
    rows, dest = algo.OrderByPred(col, True, [], [[1, 2], []])
    assert [r.tolist() for r in rows] == [[], []] and dest.Uids.size == 0
    rows, dest = algo.OrderByPred(col, False, [1], [])
    assert rows == [] and dest.Uids.size == 0


def test_golden_published_answers():
    """The published answers of the reference tests in tests/golden/pred_order_common.json, on the restatement and
    the formula (every qualifying row has distinct values, so the formula names the answer)."""
    import pred_order_golden as pg

    cs = pg.cases()
    assert len(cs) == 5
    for label, case, want in cs:
        rows, dest = po.pred_order(*case)
        assert rows[0].tolist() == want.tolist(), label
        assert dest.tolist() == sorted(want.tolist()), label
        frows, fdest = gp.formula(*case)
        assert frows[0].tolist() == want.tolist() and fdest.tolist() == sorted(want.tolist()), label
