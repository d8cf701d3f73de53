"""The compare functions on the device (dgx_compare_uids / dgx_compare_rows and their lane forms): every result
compared in full with the line-by-line restatement (compare_oracle.c), with guard words after every output, and
launches with the plan.  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import threading

import numpy as np
import pytest

import compare_oracle as co
import gen_compare as gc
from dgraph_b200 import _lib, algo

pytestmark = pytest.mark.gpu
GUARD = np.uint64(0xDEADBEEFCAFEF00D)
NO = algo.CMP_NO_ARG


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


def _dev(a):
    import torch

    a = np.ascontiguousarray(a)
    if a.dtype == np.uint64:
        a = a.view(np.int64)
    elif a.dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(a.copy()).cuda()


class DevCol:
    """A resident copy of a ValColumn: the struct dgx_dev_compare_* take, arrays in device memory."""

    def __init__(self, col: algo.ValColumn):
        self.keep = []

        def d(a):
            if a is None:
                return None
            t = _dev(a)
            self.keep.append(t)
            return t.data_ptr()

        self.s = None
        if col.type == algo.VAL_STRING:
            s = col.str
            self.s = _lib.StrColumn(d(s.uid) if s.uid.size else None, d(s.val_off), d(s.byte_off), d(s.bytes),
                                    s.uid.size, s.byte_off.size - 1, int(s.byte_off[-1]))
            self.struct = _lib.ValColumn(col.type, None, None, None, None, d(col.bad), C.pointer(self.s), 0, 0)
        else:
            self.struct = _lib.ValColumn(col.type, d(col.uid) if col.uid.size else None, d(col.val_off), d(col.word),
                                         d(col.nsec), d(col.bad), None, col.uid.size, int(col.val_off[-1]))


def _sync(lib, lane):
    return lib.dgx_lane_sync(lane)


def dev_uids(lib, lane, col, op, args, cands, dcol=None, count_word=None):
    """The lane form with guard words after d_out and d_counts; returns (dest, counts) or the sync's status."""
    import torch

    dcol = dcol or DevCol(col)
    a = args if isinstance(args, algo.ValArgs) else algo.ValArgs(col.type, args)
    u = np.asarray(cands, np.uint64)
    n = u.size
    du = _dev(np.concatenate([u, [GUARD]]).astype(np.uint64))
    out = _dev(np.full(n + 4, GUARD, np.uint64))
    cnt = _dev(np.full(n + 4, 0xA5A5A5A5, np.uint32))
    olen = _dev(np.full(1, GUARD, np.uint64))
    dn = None
    if count_word is not None:
        dn = _dev(np.asarray([count_word], np.uint64))
    algo.dev_compare_uids(lane, dcol.struct, op, a, du.data_ptr(), n, out.data_ptr(), n, olen.data_ptr(),
                          d_nuids=dn.data_ptr() if dn is not None else None, d_counts=cnt.data_ptr())
    rc = _sync(lib, lane)
    torch.cuda.synchronize()
    o = out.cpu().numpy().view(np.uint64)
    c = cnt.cpu().numpy().view(np.uint32)
    L = int(olen.cpu().numpy().view(np.uint64)[0])
    if rc:
        return rc, L, o, c
    assert (o[L:] == GUARD).all() and (c[n:] == 0xA5A5A5A5).all()
    return o[:L].copy(), c[:n].copy()


def dev_rows(lib, lane, col, op, args, rows, row_arg, dcol=None, v_off=None, v_cap=None):
    import torch

    dcol = dcol or DevCol(col)
    a = args if isinstance(args, algo.ValArgs) else algo.ValArgs(col.type, args)
    off = np.zeros(len(rows) + 1, np.uint64)
    np.cumsum([len(r) for r in rows], out=off[1:])
    if v_off is not None:
        off = np.asarray(v_off, np.uint64)
    M = int(off[-1]) if v_cap is None else v_cap
    v = np.concatenate([np.asarray(r, np.uint64) for r in rows] + [np.full(2, GUARD, np.uint64)])
    dv, doff = _dev(v), _dev(off)
    out = _dev(np.full(M + 4, GUARD, np.uint64))
    oo = _dev(np.full(len(rows) + 3, GUARD, np.uint64))
    algo.dev_compare_rows(lane, dcol.struct, op, a, dv.data_ptr(), doff.data_ptr(), len(rows), M, row_arg,
                          out.data_ptr(), oo.data_ptr(), M)
    rc = _sync(lib, lane)
    torch.cuda.synchronize()
    o = out.cpu().numpy().view(np.uint64)
    f = oo.cpu().numpy().view(np.uint64)
    if rc:
        return rc, o, f
    n = len(rows)
    assert (f[n + 1:] == GUARD).all() and (o[int(f[n]):] == GUARD).all()
    return [o[int(f[i]):int(f[i + 1])].copy() for i in range(n)]


def check_uids(lib, lane, col, op, args, cands):
    want = co.compare_uids(col, op, args, cands)
    if want is None:
        with pytest.raises(_lib.DgxError) as e:
            algo.CompareUids(col, op, args, cands)
        assert e.value.code == _lib.DGX_ERR_ARG
        r = dev_uids(lib, lane, col, op, args, cands)
        assert r[0] == _lib.DGX_ERR_ARG and r[1] == 0
        assert (r[2] == GUARD).all() and (r[3] == 0xA5A5A5A5).all()
        return None
    got, cnt = algo.CompareUids(col, op, args, cands, counts=True)
    assert np.array_equal(got.Uids, want[0]) and np.array_equal(cnt, want[1])
    d, dc = dev_uids(lib, lane, col, op, args, cands)
    assert np.array_equal(d, want[0]) and np.array_equal(dc, want[1])
    return want


def check_rows(lib, lane, col, op, args, rows, row_arg):
    want = co.compare_rows(col, op, args, rows, row_arg)
    got = algo.CompareRows(col, op, args, rows, row_arg)
    assert [g.tolist() for g in got] == [w.tolist() for w in want]
    d = dev_rows(lib, lane, col, op, args, rows, row_arg)
    assert [g.tolist() for g in d] == [w.tolist() for w in want]
    return want


@pytest.mark.parametrize("typ", gc.TYPES)
@pytest.mark.parametrize("op", gc.OPS)
def test_every_type_and_op(lib, lane, typ, op):
    rng = np.random.default_rng(typ * 10 + gc.OPS.index(op))
    for _ in range(25):
        typ_, uids, values, bad, op_, args, cands = gc.rand_case(rng, typ, op)
        col = gc.column(typ, uids, values, bad)
        check_uids(lib, lane, col, op, args, cands)
        rows = [np.sort(rng.choice(np.arange(1, 60, dtype=np.uint64), int(rng.integers(0, 8)), replace=False))
                for _ in range(int(rng.integers(1, 5)))]
        ra = [int(rng.integers(0, len(args) - (1 if op == "between" else 0))) if rng.random() < 0.7 else NO
              for _ in rows]
        check_rows(lib, lane, col, op, args, rows, ra)


def test_float_and_bool_corners(lib, lane):
    nan, inf = float("nan"), float("inf")
    vals = [nan, -0.0, 0.0, inf, -inf, 1.0, -1.0]
    col = algo.ValColumn(algo.VAL_FLOAT64, np.arange(1, 8), [[v] for v in vals])
    cands = np.arange(1, 8, dtype=np.uint64)
    for op in ("ge", "le", "gt", "lt", "eq"):
        for a in (nan, 0.0, -0.0, inf, -inf, 1.0):
            check_uids(lib, lane, col, op, [a], cands)
    for a, b in ((0.0, 1.0), (nan, 0.0), (1.0, 0.0), (-0.0, 0.0), (-inf, inf)):
        check_uids(lib, lane, col, "between", [a, b], cands)
    # a NaN value passes ge, le and between, not gt, lt or eq; -0 equals +0
    assert algo.CompareUids(col, "ge", [5.0], cands).Uids.tolist() == [1, 4]
    assert algo.CompareUids(col, "eq", [-0.0], cands).Uids.tolist() == [2, 3]
    assert algo.CompareUids(col, "ge", [nan], cands).Uids.tolist() == list(range(1, 8))
    b = algo.ValColumn(algo.VAL_BOOL, [1, 2, 3], [[True], [False], [True, False]])
    for op in gc.OPS:
        args = [True, False] if op == "between" else [True]
        w = check_uids(lib, lane, b, op, args, [1, 2, 3])
        assert (w[0].tolist() == [1, 3]) if op == "eq" else w[0].size == 0


def test_strings_around_vector_edges(lib, lane):
    rng = np.random.default_rng(7)
    base = bytes(rng.integers(0, 256, 70).astype(np.uint8))
    vals, args = [], []
    for L in (0, 1, 15, 16, 17, 31, 32, 33, 47, 48, 63, 64, 65):
        v = base[:L]
        vals.append([v, v + b"\x00", v[:-1] + b"\xff" if L else b"\xff"])
    for L in (0, 15, 16, 17, 32, 33, 64):
        args.append(base[:L])
    col = algo.ValColumn(algo.VAL_STRING, np.arange(1, len(vals) + 1), vals)
    cands = np.arange(1, len(vals) + 1, dtype=np.uint64)
    for a in args:
        for op in ("ge", "le", "gt", "lt", "eq"):
            check_uids(lib, lane, col, op, [a], cands)
    check_uids(lib, lane, col, "eq", args + args, cands)
    check_uids(lib, lane, col, "between", [b"", base[:33]], cands)
    # a column whose first and last bytes are a value's: every offset of the column base inside a 16-byte segment
    for shift in range(0, 17):
        data = bytes(rng.integers(0, 256, shift + 40).astype(np.uint8))
        offs = np.asarray([0, shift, shift + 17, shift + 40], np.uint64)
        sc = algo.StrColumn.from_csr([1, 2, 3], [0, 1, 2, 3], offs, np.frombuffer(data, np.uint8))
        vc = algo.ValColumn.from_arrays(algo.VAL_STRING, str_col=sc)
        for a in (data[:shift], data[shift:shift + 17], data[shift + 17:], data[-1:], b""):
            check_uids(lib, lane, vc, "eq", [a], [1, 2, 3])
            check_uids(lib, lane, vc, "ge", [a], [1, 2, 3])


def test_long_strings(lib, lane):
    big = bytes(np.random.default_rng(3).integers(97, 99, 1 << 20).astype(np.uint8))
    vals = [[big], [big[:-1] + b"z"], [big + b"a"], [big[: 1 << 19]]]
    col = algo.ValColumn(algo.VAL_STRING, [1, 2, 3, 4], vals)
    for op in ("eq", "ge", "lt"):
        check_uids(lib, lane, col, op, [big], [1, 2, 3, 4])


def test_eq_many_arguments(lib, lane):
    rng = np.random.default_rng(11)
    for typ in (algo.VAL_INT64, algo.VAL_FLOAT64, algo.VAL_DATETIME, algo.VAL_STRING):
        uids = np.arange(1, 3001, dtype=np.uint64)
        values = [[gc.rand_value(rng, typ) for _ in range(int(rng.integers(0, 3)))] for _ in uids]
        col = algo.ValColumn(typ, uids, values)
        stored = [v for vs in values for v in vs]
        for k in (1, 2, 10000):
            args = [stored[i] for i in rng.integers(0, len(stored), k // 2 + 1)] + \
                   [gc.rand_value(rng, typ) for _ in range(k - k // 2 - 1)]
            if typ == algo.VAL_FLOAT64 and k > 1:
                args[1] = float("nan")
            check_uids(lib, lane, col, "eq", args, uids[::2])


def test_list_hub_row_lengths(lib, lane):
    vals = [[int(x) for x in np.arange(20000) % 100], [5], [7, 7, 7]]
    col = algo.ValColumn(algo.VAL_INT64, [10, 20, 30], vals)
    w = check_uids(lib, lane, col, "ge", [50], [10, 20, 30])
    assert w[1].tolist() == [10000, 0, 0]
    w = check_uids(lib, lane, col, "eq", [7, 7, 5, 99], [10, 20, 30])
    assert w[1].tolist() == [600, 1, 3]


def test_bad_values(lib, lane):
    col = algo.ValColumn(algo.VAL_INT64, [1, 2, 3], [[1], [2, 3], [4]], bad=[[False], [False, True], [False]])
    assert check_uids(lib, lane, col, "ge", [0], [1, 2]) is None  # a candidate owns a bad value: Go's error
    w = check_uids(lib, lane, col, "ge", [0], [1, 3])  # off the candidates: ignored
    assert w[0].tolist() == [1, 3]
    # the index path skips a bad value
    rows = check_rows(lib, lane, col, "ge", [3], [[1, 2, 3]], [0])
    assert rows[0].tolist() == [3]


def test_row_args(lib, lane):
    col = algo.ValColumn(algo.VAL_FLOAT64, [1, 2, 3, 4, 5], [[0.5], [1.5], [2.5], [3.5], [float("nan")]])
    ra = algo.CompareRowArgs("between", 1)
    assert ra.tolist() == [0]
    assert check_rows(lib, lane, col, "between", [1.0, 3.0], [[1, 2, 3, 5]], ra)[0].tolist() == [2, 3, 5]
    ra = algo.CompareRowArgs("between", 3)
    check_rows(lib, lane, col, "between", [1.0, 3.0], [[1, 2], [], [3, 4, 5]], ra)
    check_rows(lib, lane, col, "eq", [0.5, 2.5, 9.0], [[1, 2], [3], []], algo.CompareRowArgs("eq", 3, 3))
    check_rows(lib, lane, col, "ge", [2.0], [[1, 2, 3], [4, 5]], algo.CompareRowArgs("ge", 2, 1, True))
    check_rows(lib, lane, col, "ge", [2.0], [[3, 1], [4, 5]], algo.CompareRowArgs("ge", 2, 1, False))


def test_device_refusals(lib, lane):
    col = algo.ValColumn(algo.VAL_INT64, [1, 2, 3], [[1], [2], [3]])
    r = dev_uids(lib, lane, col, "ge", [0], [2, 1])  # unordered candidates
    assert r[0] == _lib.DGX_ERR_ARG and r[1] == 0 and (r[2] == GUARD).all()
    r = dev_uids(lib, lane, col, "ge", [0], [1, 2], count_word=3)  # a count word past its room
    assert r[0] == _lib.DGX_ERR_ARG and r[1] == 0
    unordered = algo.ValColumn.from_arrays(algo.VAL_INT64, [2, 1, 3], [0, 1, 2, 3], np.asarray([1, 2, 3], np.int64))
    r = dev_uids(lib, lane, unordered, "ge", [0], [1, 2])
    assert r[0] == _lib.DGX_ERR_ARG
    r = dev_rows(lib, lane, unordered, "ge", [0], [[1, 2]], [0])
    assert r[0] == _lib.DGX_ERR_ARG and (r[2][:2] == 0).all() and (r[1] == GUARD).all()
    offs = algo.ValColumn.from_arrays(algo.VAL_INT64, [1, 2, 3], [0, 2, 1, 3], np.asarray([1, 2, 3], np.int64))
    assert dev_uids(lib, lane, offs, "ge", [0], [1, 2])[0] == _lib.DGX_ERR_ARG
    r = dev_rows(lib, lane, col, "ge", [0], [[1, 2], [3]], [0, 0], v_off=[0, 2, 1])  # v_off decreasing
    assert r[0] == _lib.DGX_ERR_ARG and (r[2][:3] == 0).all()
    r = dev_rows(lib, lane, col, "ge", [0], [[1, 2], [3]], [0, 0], v_off=[0, 2, 3], v_cap=2)  # past v_cap
    assert r[0] == _lib.DGX_ERR_ARG
    t = algo.ValColumn(algo.VAL_DATETIME, [1], [[(0, 10 ** 9)]])
    assert dev_uids(lib, lane, t, "ge", [(0, 0)], [1])[0] == _lib.DGX_ERR_ARG
    # the lane is usable after every refusal
    d, c = dev_uids(lib, lane, col, "ge", [2], [1, 2, 3])
    assert d.tolist() == [2, 3] and c.tolist() == [0, 1, 1]


def test_launches_constant(lib, lane):
    rng = np.random.default_rng(5)
    got_u, got_r = set(), set()
    for n in (1, 100, 100000):
        uids = np.arange(1, n + 1, dtype=np.uint64)
        col = algo.ValColumn.from_arrays(algo.VAL_INT64, uids, np.arange(n + 1, dtype=np.uint64),
                                         rng.integers(-5, 5, n).astype(np.int64))
        dcol = DevCol(col)
        l0 = lib.dgx_lane_launches(lane)
        dev_uids(lib, lane, col, "eq", list(range(min(n, 50))), uids, dcol=dcol)
        got_u.add(lib.dgx_lane_launches(lane) - l0)
        l0 = lib.dgx_lane_launches(lane)
        dev_rows(lib, lane, col, "ge", [0], [uids, uids[:3]], [0, NO], dcol=dcol)
        got_r.add(lib.dgx_lane_launches(lane) - l0)
    assert got_u == {5} and got_r == {4}


def test_concurrent_callers(lib):
    rng = np.random.default_rng(9)
    cases = [gc.rand_case(rng, nuids=200) for _ in range(16)]
    wants = [co.compare_uids(gc.column(*c[:4]), c[4], c[5], c[6]) for c in cases]
    errs = []

    def work(t):
        try:
            for i in range(t, len(cases), 4):
                typ, uids, values, bad, op, args, cands = cases[i]
                col = gc.column(typ, uids, values, bad)
                if wants[i] is None:
                    with pytest.raises(_lib.DgxError):
                        algo.CompareUids(col, op, args, cands)
                else:
                    got, cnt = algo.CompareUids(col, op, args, cands, counts=True)
                    assert np.array_equal(got.Uids, wants[i][0]) and np.array_equal(cnt, wants[i][1])
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs


def test_large(lib, lane):
    rng = np.random.default_rng(13)
    n = 10 ** 8
    uids = np.arange(1, 2 * n, 2, dtype=np.uint64)
    word = rng.integers(-10 ** 6, 10 ** 6, n).astype(np.int64)
    col = algo.ValColumn.from_arrays(algo.VAL_INT64, uids, np.arange(n + 1, dtype=np.uint64), word)
    cands = np.sort(rng.choice(2 * n, 2 * 10 ** 7, replace=False).astype(np.uint64) + 1)
    got, cnt = algo.CompareUids(col, "ge", [0], cands, counts=True)
    want = co.compare_uids(col, "ge", [0], cands)
    assert np.array_equal(got.Uids, want[0]) and np.array_equal(cnt, want[1])
    d, dc = dev_uids(lib, lane, col, "ge", [0], cands)
    assert np.array_equal(d, want[0]) and np.array_equal(dc, want[1])


def test_device_chains(lib, lane):
    import torch

    # index rows -> dgx_dev_compare_rows (between on rows 0 and last) -> dgx_dev_merge_sorted_matrix
    rng = np.random.default_rng(17)
    uids = np.arange(1, 2001, dtype=np.uint64)
    vals = rng.normal(0, 10, uids.size)
    col = algo.ValColumn(algo.VAL_FLOAT64, uids, [[float(v)] for v in vals])
    buckets = np.floor(vals).astype(np.int64)
    keys = np.arange(-3, 4)
    rows = [uids[buckets == k] for k in keys]
    ra = algo.CompareRowArgs("between", len(rows))
    args = [-2.5, 3.5]
    want_rows = co.compare_rows(col, "between", args, rows, ra)
    want = np.unique(np.concatenate(want_rows)).astype(np.uint64)
    assert np.array_equal(want, uids[(vals >= -2.5) & (vals <= 3.5)])
    dcol = DevCol(col)
    off = np.zeros(len(rows) + 1, np.uint64)
    np.cumsum([len(r) for r in rows], out=off[1:])
    M = int(off[-1])
    dv, doff = _dev(np.concatenate(rows)), _dev(off)
    out, oo = _dev(np.zeros(M, np.uint64)), _dev(np.zeros(len(rows) + 1, np.uint64))
    dest, dlen = _dev(np.zeros(M + 1, np.uint64)), _dev(np.zeros(1, np.uint64))
    algo.dev_compare_rows(lane, dcol.struct, "between", algo.ValArgs(algo.VAL_FLOAT64, args), dv.data_ptr(),
                          doff.data_ptr(), len(rows), M, ra, out.data_ptr(), oo.data_ptr(), M)
    _lib.check(lib.dgx_dev_merge_sorted_matrix(lane, out.data_ptr(), oo.data_ptr(), len(rows), M, dest.data_ptr(), M,
                                               dlen.data_ptr()))
    # DestUIDs -> dgx_dev_compare_uids (le) -> dgx_dev_compare_uids (ge), every count in a device word
    d2, l2 = _dev(np.zeros(M + 1, np.uint64)), _dev(np.zeros(1, np.uint64))
    d3, l3 = _dev(np.zeros(M + 1, np.uint64)), _dev(np.zeros(1, np.uint64))
    algo.dev_compare_uids(lane, dcol.struct, "le", algo.ValArgs(algo.VAL_FLOAT64, [1.0]), dest.data_ptr(), M,
                          d2.data_ptr(), M, l2.data_ptr(), d_nuids=dlen.data_ptr())
    algo.dev_compare_uids(lane, dcol.struct, "ge", algo.ValArgs(algo.VAL_FLOAT64, [-1.0]), d2.data_ptr(), M,
                          d3.data_ptr(), M, l3.data_ptr(), d_nuids=l2.data_ptr())
    _lib.check(lib.dgx_lane_sync(lane))
    torch.cuda.synchronize()
    n1 = int(dlen.cpu().numpy().view(np.uint64)[0])
    assert np.array_equal(dest.cpu().numpy().view(np.uint64)[:n1], want)
    n3 = int(l3.cpu().numpy().view(np.uint64)[0])
    w3 = want[(vals[(want - 1).astype(np.int64)] <= 1.0) & (vals[(want - 1).astype(np.int64)] >= -1.0)]
    assert np.array_equal(d3.cpu().numpy().view(np.uint64)[:n3], w3)


def test_rows_device_refusals_guard_reads(lib, lane):
    """The rows path refuses, writing zero offsets and no value, where a read would leave its arrays: v_off not starting
    at 0 (the row search would land before row_arg) and a column refused by the lookup (its val_off past nvals or
    decreasing, so the value loop would read past the words)."""
    col = algo.ValColumn(algo.VAL_INT64, [1, 2, 3], [[1], [2], [3]])
    rows = [[1, 2], [3]]
    r = dev_rows(lib, lane, col, "ge", [0], rows, [0, 0], v_off=[1, 2, 3], v_cap=3)
    assert r[0] == _lib.DGX_ERR_ARG and (r[2][:3] == 0).all() and (r[1] == GUARD).all()
    for val_off in ([0, 1, 2, 9], [0, 3, 1, 3]):
        bad = algo.ValColumn.from_arrays(algo.VAL_INT64, [1, 2, 3], val_off, np.asarray([1, 2, 3], np.int64))
        dcol = DevCol(bad)
        dcol.struct.nvals = 3
        r = dev_rows(lib, lane, bad, "ge", [0], rows, [0, 0], dcol=dcol)
        assert r[0] == _lib.DGX_ERR_ARG and (r[2][:3] == 0).all() and (r[1] == GUARD).all()
        r = dev_uids(lib, lane, bad, "ge", [0], [1, 2, 3], dcol=dcol)
        assert r[0] == _lib.DGX_ERR_ARG and r[1] == 0 and (r[2] == GUARD).all()
    s = algo.StrColumn.from_csr([1, 2], [0, 1, 2], [0, 9, 4], np.frombuffer(b"abcd", np.uint8))
    sc = algo.ValColumn.from_arrays(algo.VAL_STRING, str_col=s)
    dcol = DevCol(sc)
    dcol.s.nbytes = 4
    r = dev_rows(lib, lane, sc, "ge", [b"a"], [[1, 2]], [0], dcol=dcol)  # byte offsets past nbytes
    assert r[0] == _lib.DGX_ERR_ARG and (r[2][:2] == 0).all()
    d, c = dev_uids(lib, lane, col, "ge", [2], [1, 2, 3])  # the lane is usable afterwards
    assert d.tolist() == [2, 3]


def test_golden_cases(lib, lane):
    """The published answers of tests/golden/compare_common.json through both forms of both entry points."""
    import compare_golden as cg

    G = cg.load()
    for c in G["cases"]:
        if c["path"] == "value":
            col, op, args, cands = cg.value_case(G, c)
            assert check_uids(lib, lane, col, op, args, cands)[0].tolist() == c["want"], c["query"]
        else:
            col, op, args, rows, ra = cg.index_case(G, c)
            if not rows:
                assert algo.CompareRows(col, op, args, rows, ra) == [] and c["want"] == []
                continue
            assert cg.merged(check_rows(lib, lane, col, op, args, rows, ra)).tolist() == c["want"], c["query"]


def test_golden_index_chain(lib, lane):
    """TestBetweenFloat and TestDateTimeQuery's index rows -> dgx_dev_compare_rows -> dgx_dev_merge_sorted_matrix, every
    length in a device word, against the published DestUIDs."""
    import torch

    import compare_golden as cg

    G = cg.load()
    n = 0
    for c in G["cases"]:
        if c["path"] != "index":
            continue
        col, op, args, rows, ra = cg.index_case(G, c)
        off = np.zeros(len(rows) + 1, np.uint64)
        np.cumsum([len(r) for r in rows], out=off[1:])
        if not int(off[-1]):  # no index key in range, or eq's one empty row: the answer is empty without a call
            assert c["want"] == []
            continue
        dcol = DevCol(col)
        M = max(int(off[-1]), 1)
        dv = _dev(np.concatenate(rows + [np.zeros(1, np.uint64)]))
        doff = _dev(off)
        out, oo = _dev(np.zeros(M, np.uint64)), _dev(np.zeros(len(rows) + 1, np.uint64))
        dest, dlen = _dev(np.full(M + 1, GUARD, np.uint64)), _dev(np.zeros(1, np.uint64))
        algo.dev_compare_rows(lane, dcol.struct, op, algo.ValArgs(col.type, args), dv.data_ptr(), doff.data_ptr(),
                              len(rows), int(off[-1]), ra, out.data_ptr(), oo.data_ptr(), M)
        _lib.check(lib.dgx_dev_merge_sorted_matrix(lane, out.data_ptr(), oo.data_ptr(), len(rows), int(off[-1]),
                                                   dest.data_ptr(), M, dlen.data_ptr()))
        _lib.check(lib.dgx_lane_sync(lane))
        torch.cuda.synchronize()
        k = int(dlen.cpu().numpy().view(np.uint64)[0])
        d = dest.cpu().numpy().view(np.uint64)
        assert d[:k].tolist() == c["want"] and (d[k:] == GUARD).all(), c["query"]
        n += 1
    assert n == 11


def test_sg_filter_compare_var_order_chain(lib, lane):
    """dgx_dev_sg_filter's new dest -> dgx_dev_compare_uids (its count the filter's length word) ->
    dgx_dev_var_order over the filter's rows, no host read between the calls."""
    import torch

    import var_order_oracle as vo
    from dgraph_b200.algo import sg_filter_flat, sg_filter_leaf_arrays, sg_filter_tree

    rng = np.random.default_rng(31)
    U = np.arange(1, 4001, dtype=np.uint64)
    d0 = U[rng.random(U.size) < 0.8]
    rows = [np.sort(rng.choice(d0, size=int(rng.integers(0, 300)), replace=False)) for _ in range(20)]
    flt = np.sort(rng.choice(d0, size=d0.size // 2, replace=False))
    col = algo.ValColumn(algo.VAL_FLOAT64, U, [[float(x)] for x in rng.normal(0, 1, U.size)])
    mk = np.sort(rng.choice(U, size=2500, replace=False))
    mv = rng.integers(-20, 20, mk.size).astype(np.int64)
    # the host answer: the filter, the comparison over its dest, then the order over its rows
    fs = set(flt.tolist())
    f_rows = [np.array([x for x in r if x in fs], np.uint64) for r in rows]
    f_dest = np.array(sorted(set(d0.tolist()) & fs), np.uint64)
    kept, _ = co.compare_uids(col, "ge", [0.25], f_dest)
    exp_rows, exp_dest = vo.var_order((mk, mv), False, kept, f_rows, 0, 0)
    # device
    f = sg_filter_flat(0)
    keep_l, tab = sg_filter_leaf_arrays([("list", flt)], d0.size)
    t_flt = _dev(flt)
    tab[0].uids = t_flt.data_ptr()
    v = np.concatenate(rows)
    v_off = np.zeros(len(rows) + 1, np.uint64)
    np.cumsum([len(r) for r in rows], out=v_off[1:])
    d_d0, d_v, d_vo = _dev(d0), _dev(v), _dev(v_off)
    nrows, nd = len(rows), d0.size
    s_dest, s_len = _dev(np.zeros(nd, np.uint64)), _dev(np.zeros(1, np.uint64))
    s_out, s_off, s_cnt = _dev(np.zeros(v.size, np.uint64)), _dev(np.zeros(nrows + 1, np.uint64)), \
        _dev(np.zeros(nrows, np.uint32))
    t = sg_filter_tree(f)
    _lib.check(lib.dgx_dev_sg_filter(lane, C.byref(t), tab, 1, d_d0.data_ptr(), nd, None, d_v.data_ptr(),
                                     d_vo.data_ptr(), nrows, v.size, 0, 0, s_dest.data_ptr(), nd, s_len.data_ptr(),
                                     s_out.data_ptr(), s_off.data_ptr(), v.size, s_cnt.data_ptr()))
    dcol = DevCol(col)
    c_out, c_len = _dev(np.zeros(nd, np.uint64)), _dev(np.zeros(1, np.uint64))
    algo.dev_compare_uids(lane, dcol.struct, "ge", algo.ValArgs(algo.VAL_FLOAT64, [0.25]), s_dest.data_ptr(), nd,
                          c_out.data_ptr(), nd, c_len.data_ptr(), d_nuids=s_len.data_ptr())
    d_mk, d_mv = _dev(mk), _dev(mv.view(np.uint64))
    var = _lib.MathLeaf(d_mk.data_ptr(), d_mv.data_ptr(), None, None, mk.size, algo.VAL_INT64, 0)
    o_out, o_off = _dev(np.zeros(v.size, np.uint64)), _dev(np.zeros(nrows + 1, np.uint64))
    o_dest, o_len = _dev(np.zeros(nd, np.uint64)), _dev(np.zeros(1, np.uint64))
    _lib.check(lib.dgx_dev_var_order(lane, C.byref(var), 0, c_out.data_ptr(), nd, c_len.data_ptr(), s_out.data_ptr(),
                                     s_off.data_ptr(), nrows, v.size, 0, 0, o_out.data_ptr(), o_off.data_ptr(), v.size,
                                     o_dest.data_ptr(), nd, o_len.data_ptr()))
    _lib.check(lib.dgx_lane_sync(lane))
    torch.cuda.synchronize()
    k = int(c_len.cpu().numpy().view(np.uint64)[0])
    assert np.array_equal(c_out.cpu().numpy().view(np.uint64)[:k], kept)
    off = o_off.cpu().numpy().view(np.uint64)
    out = o_out.cpu().numpy().view(np.uint64)
    assert [out[int(off[i]):int(off[i + 1])].tolist() for i in range(nrows)] == [r.tolist() for r in exp_rows]
    nl = int(o_len.cpu().numpy().view(np.uint64)[0])
    assert o_dest.cpu().numpy().view(np.uint64)[:nl].tolist() == np.asarray(exp_dest).tolist()
