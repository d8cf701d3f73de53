"""orderasc / orderdesc by a predicate on the device (dgx_pred_order and dgx_dev_pred_order): both forms against the
line-by-line restatement (pred_order_oracle.c), bit for bit, with guard words past every output, on seeded cases of
each type; tied string and datetime rows on threads and on the CTA path (rows of more than 4 096 entries); int and
float columns with no nulls against dgx_var_order on the equivalent map, device against device; a dgx_dev_sg_filter ->
dgx_dev_pred_order chain with no host read; every device-side refusal; launches per call against the plan
(pred_order_plan.py).  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen_pred_order as gp  # noqa: E402
import pred_order_oracle as po  # noqa: E402
import pred_order_plan as pp  # noqa: E402
import var_order_oracle as vo  # noqa: E402
from dgraph_b200 import _lib, algo  # noqa: E402

pytestmark = pytest.mark.gpu

OK, ERR_ARG, ERR_CAP = 0, -3, -4
SENT = 0xDEADBEEFCAFEF00D
GUARD = 4
T_INT, T_FLOAT, T_TIME, T_STR = algo.VAL_INT64, algo.VAL_FLOAT64, algo.VAL_DATETIME, algo.VAL_STRING


@pytest.fixture(scope="module")
def lib():
    L = _lib.load()
    _lib.check(L.dgx_init(-1))
    return L


@pytest.fixture(scope="module")
def lane(lib):
    import torch

    stream = torch.cuda.Stream()
    ln = lib.dgx_lane_create(0, C.c_void_p(stream.cuda_stream))
    assert ln
    yield ln
    lib.dgx_lane_destroy(ln)


def _t(a, dtype=np.uint64):
    import torch

    a = np.ascontiguousarray(np.asarray(a, dtype))
    if a.size == 0:
        a = np.zeros(1, dtype)
    if dtype == np.uint64:
        return torch.from_numpy(a.view(np.int64).copy()).cuda()
    if dtype == np.uint32:
        return torch.from_numpy(a.view(np.int32).copy()).cuda()
    return torch.from_numpy(a.copy()).cuda()


def _h(t, n, dtype=np.uint64):
    a = t.cpu().numpy()[:n]
    return a.view(np.uint64).copy() if dtype == np.uint64 else a.copy()


def sent(n):
    import torch

    return torch.full((max(n, 1),), SENT - (1 << 64), dtype=torch.int64, device="cuda")


def csr(rows):
    off = np.zeros(len(rows) + 1, np.uint64)
    np.cumsum([len(r) for r in rows], out=off[1:])
    v = np.concatenate([np.asarray(r, np.uint64) for r in rows]) if int(off[-1]) else np.zeros(0, np.uint64)
    return v, off


class DevCol:
    """A resident copy of a ValColumn: the struct dgx_dev_pred_order takes, arrays in device memory."""

    def __init__(self, col):
        self.keep = []

        def d(a, dt=None):
            if a is None:
                return None
            t = _t(a, dt or a.dtype.type)
            self.keep.append(t)
            return t.data_ptr()

        if col.type == T_STR:
            s = col.str
            self.s = _lib.StrColumn(d(s.uid) if s.uid.size else None, d(s.val_off), d(s.byte_off), d(s.bytes),
                                    s.uid.size, s.byte_off.size - 1, int(s.byte_off[-1]))
            self.struct = _lib.ValColumn(col.type, None, None, None, None, d(col.bad), C.pointer(self.s), 0, 0)
        else:
            self.struct = _lib.ValColumn(col.type, d(col.uid) if col.uid.size else None, d(col.val_off),
                                         d(col.word), d(col.nsec), d(col.bad), None, col.uid.size,
                                         int(col.val_off[-1]))


def want(case):
    try:
        return po.pred_order(*case)
    except (po.ListPredicate, po.NegativeCount, po.NotSortable) as e:
        return type(e)


def same(got, exp):
    (gr, gd), (er, ed) = got, exp
    return len(gr) == len(er) and all(np.array_equal(x, y) for x, y in zip(gr, er)) and np.array_equal(gd, ed)


def host_call(lib, case):
    """dgx_pred_order with guard words past every output: (rc, (rows, dest) or None, guards intact, launches)."""
    col, desc, dest, rows, count, offset = case
    d = np.ascontiguousarray(np.asarray(dest, np.uint64))
    v, v_off = csr(rows)
    v = v if v.size else np.zeros(1, np.uint64)
    nrows, M = len(rows), int(v_off[-1])
    out = np.full(M + GUARD, SENT, np.uint64)
    oo = np.full(nrows + 1 + GUARD, SENT, np.uint64)
    dout = np.full(d.size + GUARD, SENT, np.uint64)
    n = C.c_size_t(SENT)
    cs = col.struct()
    l0 = _lib.stats()["kernel_launches"]
    rc = lib.dgx_pred_order(C.byref(cs), int(desc), (d if d.size else np.zeros(1, np.uint64)).ctypes.data, d.size,
                            v.ctypes.data, v_off.ctypes.data, nrows, count, offset, out.ctypes.data, oo.ctypes.data,
                            M, dout.ctypes.data, d.size, C.byref(n))
    nl = _lib.stats()["kernel_launches"] - l0
    guards = np.all(out[M:] == SENT) and np.all(oo[nrows + 1:] == SENT) and np.all(dout[d.size:] == SENT)
    if rc != OK:
        return rc, None, guards and np.all(out == SENT) and np.all(dout == SENT), nl
    K = int(oo[nrows])
    guards = guards and np.all(out[K:] == SENT) and np.all(dout[n.value:] == SENT)
    return rc, ([out[int(oo[i]):int(oo[i + 1])].copy() for i in range(nrows)], dout[:n.value].copy()), guards, nl


def dev_call(lib, lane, case, slack=0, len_word=False, mutate=None, dcol=None):
    """dgx_dev_pred_order with `slack` garbage slots past dest (its length then from a device word) and the values.
    mutate(arrays) may break the inputs before upload.  Returns (rc, sync rc, dest length word, (rows, dest) or None,
    launches, guards intact)."""
    col, desc, dest, rows, count, offset = case
    d = np.asarray(dest, np.uint64)
    v, v_off = csr(rows)
    a = {"dest": np.concatenate([d, np.full(slack if len_word else 0, 3, np.uint64)]),
         "v": np.concatenate([v, np.full(slack, 9, np.uint64)]), "v_off": v_off.copy()}
    if mutate:
        mutate(a)
    nrows, ndest, vcap = len(rows), a["dest"].size, a["v"].size
    dc = dcol or DevCol(col)
    dd, vv, oo_in = _t(a["dest"]), _t(a["v"]), _t(a["v_off"])
    dw = _t(np.array([d.size | (0x33 << 36)], np.uint64)) if len_word else None
    out, oo, dout, dlen = sent(vcap + GUARD), sent(nrows + 1 + GUARD), sent(ndest + GUARD), sent(1)
    l0 = lib.dgx_lane_launches(lane)
    rc = lib.dgx_dev_pred_order(lane, C.byref(dc.struct), int(desc), dd.data_ptr(), ndest,
                                dw.data_ptr() if dw is not None else None, vv.data_ptr(), oo_in.data_ptr(), nrows,
                                vcap, count, offset, out.data_ptr(), oo.data_ptr(), vcap, dout.data_ptr(), ndest,
                                dlen.data_ptr())
    src = lib.dgx_lane_sync(lane) if rc == OK else None
    nl = lib.dgx_lane_launches(lane) - l0
    o, off, de, L = _h(out, vcap + GUARD), _h(oo, nrows + 1 + GUARD), _h(dout, ndest + GUARD), int(_h(dlen, 1)[0])
    guards = np.all(o[vcap:] == SENT) and np.all(off[nrows + 1:] == SENT) and np.all(de[ndest:] == SENT)
    if rc != OK or src != OK:
        guards = guards and np.all(o == SENT) and np.all(off == SENT) and np.all(de == SENT)
        return rc, src, L, None, nl, guards
    K = int(off[nrows])
    guards = guards and np.all(o[K:] == SENT) and np.all(de[L:] == SENT)
    return rc, src, L, ([o[int(off[i]):int(off[i + 1])].copy() for i in range(nrows)], de[:L].copy()), nl, guards


def run_both(lib, lane, case, **kw):
    """Both forms against the restatement, launches against the plan; returns the restatement's answer."""
    exp = want(case)
    col = case[0]
    live = len(case[2]) > 0 and len(case[3]) > 0
    rc, got, g, nl = host_call(lib, case)
    assert g
    if isinstance(exp, type):
        assert rc == ERR_ARG
    else:
        assert rc == OK and same(got, exp), case
        assert nl == (pp.launches(col.type, len(case[3])) if live else 0)
    rc, src, L, got, nl, g = dev_call(lib, lane, case, **kw)
    assert rc == OK and g
    if isinstance(exp, type):
        assert src == ERR_ARG and L == 0
    else:
        assert src == OK and same(got, exp), case
        ndev = len(case[2]) + (kw.get("slack", 0) if kw.get("len_word") else 0)
        assert nl == (pp.launches(col.type, len(case[3])) if ndev and len(case[3]) else 0)
    return exp


@pytest.mark.parametrize("typ", [T_INT, T_FLOAT, T_TIME, T_STR])
def test_random_cases(lib, lane, typ):
    rng = np.random.default_rng(4100 + typ)
    for i in range(60):
        case = gp.random_case(rng, typ)
        kw = {"slack": int(rng.integers(0, 5)), "len_word": bool(rng.random() < 0.3)} if i % 2 else {}
        run_both(lib, lane, case, **kw)


def _tied_string_col(rng, uids, distinct, prefix=b"shared-prefix-"):
    names = [prefix + b"%06d" % k for k in rng.integers(0, distinct, uids.size)]
    return algo.ValColumn(T_STR, uids, [[x] for x in names])


def _tied_time_col(rng, uids, distinct):
    s = rng.integers(-10, distinct - 10, uids.size)
    ns = rng.choice([0, 1, 999_999_999], uids.size)
    return algo.ValColumn(T_TIME, uids, [[(int(a), int(b))] for a, b in zip(s, ns)])


@pytest.mark.parametrize("kind", ["string", "datetime"])
@pytest.mark.parametrize("n", [13, 300, 4096, 4097, 20000])
def test_tied_rows_on_threads_and_ctas(lib, lane, kind, n):
    """Tied rows of 13 (tier 2 on a thread), 4 096 (the longest thread row), 4 097 and 20 000 (a CTA each), with nulls
    and bad values, both directions; a second row keeps the call mixed."""
    rng = np.random.default_rng(n)
    uids = np.arange(1, n + 1, dtype=np.uint64) * 2
    col = _tied_string_col(rng, uids, 50) if kind == "string" else _tied_time_col(rng, uids, 30)
    col.bad = (rng.random(uids.size) < 0.05).astype(np.uint8)
    rows = [np.concatenate([uids, uids[-1:] + 1]), uids[:7]]
    for desc in (False, True):
        for count, offset in ((0, 0), (1000, 3)):
            exp = run_both(lib, lane, (col, desc, uids, rows, count, offset))
            assert not isinstance(exp, type)


def test_strings_past_their_prefix(lib, lane):
    """Distinct strings that share their first 8 bytes (tier 2 at any length), proper prefixes, empty and high bytes."""
    rng = np.random.default_rng(9)
    vals = [b"", b"ab", b"ab\0", b"ab\0\0", b"abcdefgh", b"abcdefgh\0", b"abcdefghA", b"abcdefghB", b"\xff", b"\x80",
            b"\xff\xff\xff\xff\xff\xff\xff\xff\x01", b"\xff\xff\xff\xff\xff\xff\xff\xff"]
    vals += [b"0123456789abcdef" + bytes([k]) * int(rng.integers(0, 40)) for k in range(200)]
    uids = np.arange(1, len(vals) + 1, dtype=np.uint64)
    order = rng.permutation(len(vals))
    col = algo.ValColumn(T_STR, uids, [[vals[k]] for k in order])
    for desc in (False, True):
        run_both(lib, lane, (col, desc, uids, [uids, uids[:5], uids[::-3][::-1]], 0, 0))


@pytest.mark.parametrize("typ", [T_INT, T_FLOAT])
def test_matches_var_order_device_to_device(lib, lane, typ):
    """A column with every uid holding a value orders as dgx_var_order orders the same map."""
    rng = np.random.default_rng(31 + typ)
    n = 6000
    uids = np.arange(1, n + 1, dtype=np.uint64)
    vals = (rng.integers(-5, 5, n).astype(np.int64) if typ == T_INT
            else rng.choice(np.array([0.0, -0.0, 1.5, np.nan, -np.inf]), n))
    col = algo.ValColumn(typ, uids, [[x] for x in vals.tolist()])
    rows = [uids, np.sort(rng.choice(uids, 500, replace=False)), uids[:12]]
    for desc in (False, True):
        a = algo.OrderByPred(col, desc, uids, rows, 100, 7)
        b = algo.OrderByVar((uids, vals), desc, uids, rows, 100, 7)
        assert all(np.array_equal(x, y) for x, y in zip(a[0], b[0])) and np.array_equal(a[1].Uids, b[1].Uids)
        rc, src, L, got, nl, g = dev_call(lib, lane, (col, desc, uids, rows, 100, 7))
        assert rc == OK and src == OK and g
        assert all(np.array_equal(x, y) for x, y in zip(got[0], b[0])) and np.array_equal(got[1], b[1].Uids)


def test_device_chain(lib, lane):
    """Rows -> dgx_dev_sg_filter (its new dest's length a device word) -> dgx_dev_pred_order over a resident string
    column, no host read between the calls."""
    from dgraph_b200.algo import sg_filter_flat, sg_filter_leaf_arrays, sg_filter_tree

    rng = np.random.default_rng(5)
    U = np.arange(1, 3001, dtype=np.uint64)
    d0 = U[rng.random(U.size) < 0.8]
    rows = [np.sort(rng.choice(d0, size=int(rng.integers(0, 400)), replace=False)) for _ in range(30)]
    flt = np.sort(rng.choice(d0, size=d0.size // 2, replace=False))
    in_col = np.sort(rng.choice(U, size=2000, replace=False))
    col = _tied_string_col(rng, in_col, 40, b"n")
    fs = set(flt.tolist())
    f_rows = [np.array([x for x in r if x in fs], np.uint64) for r in rows]
    f_dest = np.array(sorted(set(d0.tolist()) & fs), np.uint64)
    exp_rows, exp_dest = po.pred_order(col, True, f_dest, f_rows, 5, 1)
    f = sg_filter_flat(0)
    keep_l, tab = sg_filter_leaf_arrays([("list", flt)], d0.size)
    t_flt = _t(flt)
    tab[0].uids = t_flt.data_ptr()
    v, v_off = csr(rows)
    d_d0, d_v, d_vo = _t(d0), _t(v), _t(v_off)
    nrows = len(rows)
    s_dest, s_len, s_out, s_off, s_cnt = sent(d0.size), sent(1), sent(v.size), sent(nrows + 1), sent(nrows)
    t = sg_filter_tree(f)
    assert lib.dgx_dev_sg_filter(lane, C.byref(t), tab, 1, d_d0.data_ptr(), d0.size, None, d_v.data_ptr(),
                                 d_vo.data_ptr(), nrows, v.size, 0, 0, s_dest.data_ptr(), d0.size, s_len.data_ptr(),
                                 s_out.data_ptr(), s_off.data_ptr(), v.size, s_cnt.data_ptr()) == OK
    dc = DevCol(col)
    o_out, o_off, o_dest, o_len = sent(v.size), sent(nrows + 1), sent(d0.size), sent(1)
    l0 = lib.dgx_lane_launches(lane)
    algo.dev_order_by_pred(lane, dc.struct, True, s_dest.data_ptr(), d0.size, s_out.data_ptr(), s_off.data_ptr(),
                           nrows, v.size, o_out.data_ptr(), o_off.data_ptr(), v.size, o_dest.data_ptr(), d0.size,
                           o_len.data_ptr(), 5, 1, d_ndest=s_len.data_ptr())
    assert lib.dgx_lane_launches(lane) - l0 == pp.launches(T_STR, nrows)
    assert lib.dgx_lane_sync(lane) == OK
    off = _h(o_off, nrows + 1)
    out = _h(o_out, int(off[-1]))
    assert all(np.array_equal(out[int(off[i]):int(off[i + 1])], exp_rows[i]) for i in range(nrows))
    assert np.array_equal(_h(o_dest, int(_h(o_len, 1)[0])), exp_dest)
    del keep_l


def test_device_refusals(lib, lane):
    """Each refusal found on the device surfaces at dgx_lane_sync with the length word 0 and nothing else written."""
    uids = np.arange(1, 9, dtype=np.uint64)
    col = algo.ValColumn(T_INT, uids, [[int(x) % 3] for x in uids])
    base = (col, False, uids, [uids[:4], uids[4:]], 0, 0)

    def dest_desc(a):
        a["dest"][[0, 1]] = a["dest"][[1, 0]]

    def row_desc(a):
        a["v"][[1, 2]] = a["v"][[2, 1]]

    def off_start(a):
        a["v_off"][0] = 1

    def off_past(a):
        a["v_off"][-1] = a["v"].size + 1

    def off_dec(a):
        a["v_off"][1] = a["v_off"][2] + 1

    for mut in (dest_desc, row_desc, off_start, off_past, off_dec):
        rc, src, L, got, nl, g = dev_call(lib, lane, base, mutate=mut)
        assert rc == OK and src == ERR_ARG and L == 0 and g, mut.__name__
    cols = {
        "column uids": algo.ValColumn.from_arrays(T_INT, uids[::-1].copy(), np.arange(9, dtype=np.uint64),
                                                  np.zeros(8, np.int64)),
        "list value": algo.ValColumn(T_INT, uids, [[1, 2]] + [[1]] * 7),
        "nanoseconds": algo.ValColumn(T_TIME, uids, [[(0, 10 ** 9)]] + [[(0, 0)]] * 7),
    }
    for name, c in cols.items():
        rc, src, L, got, nl, g = dev_call(lib, lane, (c,) + base[1:])
        assert rc == OK and src == ERR_ARG and L == 0 and g, name
        rc, got, g, nl = host_call(lib, (c,) + base[1:])
        assert rc == ERR_ARG and g, name
    # a bad value, or a list value outside U, is not read
    ok = algo.ValColumn(T_TIME, uids, [[(0, 10 ** 9)]] + [[(0, 0)]] * 7, bad=[[True]] + [[False]] * 7)
    run_both(lib, lane, (ok, False, uids, [uids], 0, 0))
    run_both(lib, lane, (cols["list value"], False, uids[1:], [uids], 0, 0))
    # a dest length word past its room
    dc = DevCol(col)
    dd, vv, oo_in = _t(uids), _t(uids), _t(np.array([0, 8], np.uint64))
    dw = _t(np.array([9], np.uint64))
    out, oo, dout, dlen = sent(8), sent(2), sent(8), sent(1)
    assert lib.dgx_dev_pred_order(lane, C.byref(dc.struct), 0, dd.data_ptr(), 8, dw.data_ptr(), vv.data_ptr(),
                                  oo_in.data_ptr(), 1, 8, 0, 0, out.data_ptr(), oo.data_ptr(), 8, dout.data_ptr(), 8,
                                  dlen.data_ptr()) == OK
    assert lib.dgx_lane_sync(lane) == ERR_ARG and int(_h(dlen, 1)[0]) == 0
    # refusals at the call
    assert lib.dgx_dev_pred_order(lane, C.byref(dc.struct), 0, dd.data_ptr(), 8, None, vv.data_ptr(),
                                  oo_in.data_ptr(), 1, 8, -1, 0, out.data_ptr(), oo.data_ptr(), 8, dout.data_ptr(), 8,
                                  dlen.data_ptr()) == ERR_ARG
    assert lib.dgx_dev_pred_order(lane, C.byref(dc.struct), 0, dd.data_ptr(), 8, None, vv.data_ptr(),
                                  oo_in.data_ptr(), 1, 8, 0, 0, out.data_ptr(), oo.data_ptr(), 7, dout.data_ptr(), 8,
                                  dlen.data_ptr()) == ERR_CAP
    assert lib.dgx_lane_sync(lane) == OK


def test_launches_constant(lib, lane):
    """Launches per call depend on the type and nrows alone, not on the values, ties or column size."""
    rng = np.random.default_rng(3)
    for typ in (T_INT, T_TIME, T_STR):
        for nrows in (1, 256, 257):
            counts = set()
            for n in (10, 1000):
                uids = np.arange(1, n + 1, dtype=np.uint64)
                case = gp.random_case(rng, typ)
                col = case[0]
                rows = [uids[: int(rng.integers(0, n + 1))] for _ in range(nrows)]
                rc, src, L, got, nl, g = dev_call(lib, lane, (col, True, uids, rows, 0, 0))
                assert rc == OK and src == OK
                counts.add(nl)
            assert counts == {pp.launches(typ, nrows)}, (typ, nrows, counts)


def test_golden_published_answers(lib, lane):
    """The published answers of tests/golden/pred_order_common.json on both forms (and the restatement)."""
    import pred_order_golden as pg

    for label, case, want in pg.cases():
        exp = run_both(lib, lane, case)
        assert exp[0][0].tolist() == want.tolist(), label


def test_device_column_offset_refusals(lib, lane):
    """A resident column's offsets are checked on the device alone: val_off not ending at nvals, a decreasing
    val_off and a decreasing byte_off each surface at dgx_lane_sync with nothing written but the length word."""
    uids = np.arange(1, 9, dtype=np.uint64)
    base = (False, uids, [uids], 0, 0)
    ints = algo.ValColumn(T_INT, uids, [[int(x)] for x in uids])
    short = algo.ValColumn.from_arrays(T_INT, uids, ints.val_off.copy(), ints.word.view(np.int64))
    short.val_off[-1] = 7  # val_off[n] != nvals
    dec = algo.ValColumn.from_arrays(T_INT, uids, ints.val_off.copy(), ints.word.view(np.int64))
    dec.val_off[3], dec.val_off[4] = 4, 3
    strs = algo.ValColumn(T_STR, uids, [[b"v%d" % int(x)] for x in uids])
    sb = algo.StrColumn.from_csr(strs.str.uid, strs.str.val_off, strs.str.byte_off.copy(), strs.str.bytes)
    sb.byte_off[2], sb.byte_off[3] = sb.byte_off[3], sb.byte_off[2]  # byte_off decreasing
    bstr = algo.ValColumn.from_arrays(T_STR, str_col=sb)
    for name, c in (("val_off[n] != nvals", short), ("val_off decreasing", dec), ("byte_off decreasing", bstr)):
        dc = DevCol(c)
        if name == "val_off[n] != nvals":
            dc.struct.nvals = 8
        rc, src, L, got, nl, g = dev_call(lib, lane, (c,) + base, dcol=dc)
        assert rc == OK and src == ERR_ARG and L == 0 and g, name


def test_device_v_cap_of_2_32_refused(lib, lane):
    uids = np.arange(1, 5, dtype=np.uint64)
    dc = DevCol(algo.ValColumn(T_INT, uids, [[1]] * 4))
    dd, vv, oo_in = _t(uids), _t(uids), _t(np.array([0, 4], np.uint64))
    out, oo, dout, dlen = sent(8), sent(2), sent(8), sent(1)
    assert lib.dgx_dev_pred_order(lane, C.byref(dc.struct), 0, dd.data_ptr(), 4, None, vv.data_ptr(),
                                  oo_in.data_ptr(), 1, 1 << 32, 0, 0, out.data_ptr(), oo.data_ptr(), 1 << 32,
                                  dout.data_ptr(), 4, dlen.data_ptr()) == ERR_ARG
    assert lib.dgx_lane_sync(lane) == OK and int(_h(dlen, 1)[0]) == SENT
