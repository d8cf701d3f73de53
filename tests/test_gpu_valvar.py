"""Value variables on the device (dgx_var_propagate / dgx_var_level_agg and their device forms): every result compared
bit for bit with the line-by-line restatement (valvar_oracle.c, Go's chunks finishing in index order), guard words past
every output, launches with the plan model (valvar_plan.py).  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen_valvar as gv  # noqa: E402
import valvar_oracle as vo  # noqa: E402
import valvar_plan as vp  # noqa: E402

pytestmark = pytest.mark.gpu

OK, ERR_ARG, ERR_CAP = 0, -3, -4
SENT = 0xDEADBEEFCAFEF00D
GUARD = 4
FNS = ("min", "max", "sum", "avg")


@pytest.fixture(scope="module")
def lib():
    from dgraph_b200 import _lib

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


def _words(vals):
    v = np.ascontiguousarray(vals)
    return (2 if v.dtype == np.float64 else 1), v.view(np.uint64)


def _b(x):
    x = np.ascontiguousarray(x, np.uint64)
    return x if x.size else np.zeros(1, np.uint64)


def _csr(rows):
    off = np.zeros(len(rows) + 1, np.uint64)
    np.cumsum([len(r) for r in rows], out=off[1:])
    return (np.concatenate([np.asarray(r, np.uint64) for r in rows]) if int(off[-1]) else np.zeros(1, np.uint64)), off


def _up(x):
    import torch

    return torch.from_numpy(np.ascontiguousarray(_b(x)).view(np.int64).copy()).cuda()


def _sent(n):
    import torch

    return torch.full((n,), SENT - (1 << 64), dtype=torch.int64, device="cuda")


def _h(t):
    return t.cpu().numpy().view(np.uint64)


class Path:
    """A propagation's inputs as flat arrays, per level (src, v, v_off, dest)."""

    def __init__(self, keys, vals, levels):
        self.keys, self.vals = np.asarray(keys, np.uint64), np.asarray(vals)
        self.typ, self.w = _words(self.vals)
        self.levels = [(np.asarray(s, np.uint64), *_csr(r), np.asarray(d, np.uint64)) for s, r, d in levels]
        self.rows = [(s, r) for s, r, _ in levels]

    def want(self):
        return vo.propagate(self.keys, self.vals, self.rows)


def _check(got_n, ok, ov, want, cap):
    k, v = want
    assert got_n == k.size
    assert np.array_equal(ok[:got_n], k) and np.array_equal(ov[:got_n], np.asarray(v).view(np.uint64))
    assert (ok[got_n:] == SENT).all() and (ov[got_n:] == SENT).all()
    assert ok.size == cap + GUARD


def prop_host(lib, p: Path, cap):
    from dgraph_b200 import _lib

    keep = [(_b(s), _b(v), o, _b(d)) for s, v, o, d in p.levels]
    lv = (_lib.VarLevel * len(keep))()
    for i, (s, v, o, d) in enumerate(keep):
        lv[i] = _lib.VarLevel(s.ctypes.data, o.ctypes.data, v.ctypes.data, d.ctypes.data, o.size - 1, 0,
                              p.levels[i][3].size)
    ok, ov = np.full(cap + GUARD, SENT, np.uint64), np.full(cap + GUARD, SENT, np.uint64)
    n = C.c_size_t(7)
    rc = lib.dgx_var_propagate(p.typ, _b(p.keys).ctypes.data, _b(p.w).ctypes.data, p.keys.size, lv, len(keep),
                               ok.ctypes.data, ov.ctypes.data, cap, C.byref(n))
    return rc, n.value, ok, ov


def prop_dev(lib, lane, p: Path, cap, v_caps=None, levels=None):
    """(rc of the call, rc of the sync, d_out_len, ok, ov, launches).  levels: device (src, v, v_off, dest, ndest)
    tuples to use instead of uploading p's."""
    import torch

    from dgraph_b200 import _lib

    dl = levels or [(_up(s), _up(v), _up(o), _up(d), d.size) for s, v, o, d in p.levels]
    lv = (_lib.VarLevel * len(dl))()
    for i, (s, v, o, d, nd) in enumerate(dl):
        vc = v_caps[i] if v_caps else int(p.levels[i][2][-1])
        lv[i] = _lib.VarLevel(s.data_ptr(), o.data_ptr(), v.data_ptr(), d.data_ptr(), p.levels[i][2].size - 1, vc, nd)
    dk, dv = _up(p.keys), _up(p.w)
    ok, ov, dn = _sent(cap + GUARD), _sent(cap + GUARD), _sent(1)
    torch.cuda.synchronize()
    l0 = lib.dgx_lane_launches(lane)
    rc = lib.dgx_dev_var_propagate(lane, p.typ, dk.data_ptr(), dv.data_ptr(), p.keys.size, lv, len(dl), ok.data_ptr(),
                                   ov.data_ptr(), cap, dn.data_ptr())
    src = lib.dgx_lane_sync(lane)
    return rc, src, int(_h(dn)[0]), _h(ok), _h(ov), lib.dgx_lane_launches(lane) - l0


def both_prop(lib, lane, p: Path, want=None):
    want = p.want() if want is None else want
    cap = max(p.levels[-1][3].size, 1)
    rc, n, ok, ov = prop_host(lib, p, cap)
    assert rc == OK, lib.dgx_last_error()
    _check(n, ok, ov, want, cap)
    rc, src, n, ok, ov, launches = prop_dev(lib, lane, p, cap)
    assert rc == OK and src == OK, lib.dgx_last_error()
    _check(n, ok, ov, want, cap)
    assert launches == vp.propagate_launches(p.keys.size, [d.size for _, _, _, d in p.levels])


class Agg:
    def __init__(self, fn, keys, vals, src, rows):
        self.fn, self.keys, self.vals = fn, np.asarray(keys, np.uint64), np.asarray(vals)
        self.typ, self.w = _words(self.vals)
        self.src, self.rows = np.asarray(src, np.uint64), rows
        self.v, self.v_off = _csr(rows)

    def want(self):
        return vo.level_agg(self.fn, self.keys, self.vals, self.src, self.rows)


def agg_host(lib, a: Agg, cap):
    ok, ov = np.full(cap + GUARD, SENT, np.uint64), np.full(cap + GUARD, SENT, np.uint64)
    n = C.c_size_t(7)
    rc = lib.dgx_var_level_agg(a.typ, vo.AGG[a.fn], _b(a.keys).ctypes.data, _b(a.w).ctypes.data, a.keys.size,
                               _b(a.src).ctypes.data, len(a.rows), a.v_off.ctypes.data, a.v.ctypes.data,
                               ok.ctypes.data, ov.ctypes.data, cap, C.byref(n))
    return rc, n.value, ok, ov


def agg_dev(lib, lane, a: Agg, cap, v_cap=None):
    import torch

    t = [_up(x) for x in (a.keys, a.w, a.src, a.v_off, a.v)]
    ok, ov, dn = _sent(cap + GUARD), _sent(cap + GUARD), _sent(1)
    torch.cuda.synchronize()
    l0 = lib.dgx_lane_launches(lane)
    rc = lib.dgx_dev_var_level_agg(lane, a.typ, vo.AGG[a.fn], t[0].data_ptr(), t[1].data_ptr(), a.keys.size,
                                   t[2].data_ptr(), len(a.rows), t[3].data_ptr(), t[4].data_ptr(),
                                   int(a.v_off[-1]) if v_cap is None else v_cap, ok.data_ptr(), ov.data_ptr(), cap,
                                   dn.data_ptr())
    src = lib.dgx_lane_sync(lane)
    return rc, src, int(_h(dn)[0]), _h(ok), _h(ov), lib.dgx_lane_launches(lane) - l0


def both_agg(lib, lane, a: Agg):
    want = a.want()
    cap = max(len(a.rows), 1)
    rc, n, ok, ov = agg_host(lib, a, cap)
    assert rc == OK, lib.dgx_last_error()
    _check(n, ok, ov, want, cap)
    rc, src, n, ok, ov, launches = agg_dev(lib, lane, a, cap)
    assert rc == OK and src == OK, lib.dgx_last_error()
    _check(n, ok, ov, want, cap)
    assert launches == vp.level_agg_launches(a.keys.size, len(a.rows), int(a.v_off[-1]))


# ---- propagation -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["int", "wild", "dyadic"])
def test_random_paths(lib, lane, kind):
    rng = np.random.default_rng(["int", "wild", "dyadic"].index(kind) + 1)
    for _ in range(40):
        lv = gv.path(rng, int(rng.integers(1, 5)), int(rng.integers(1, 60)), hi=int(rng.integers(3, 300)),
                     avg_deg=float(rng.uniform(0.5, 6)), unordered=bool(rng.integers(2)),
                     repeats=bool(rng.integers(2)))
        k, v = gv.value_map(rng, lv[0][0], rng.random(), kind)
        p = Path(k, v, lv)
        want = p.want()
        if kind != "wild":
            f = gv.formula_propagate(k, v, lv)
            assert np.array_equal(f[0], want[0]) and np.array_equal(f[1].view(np.uint64), want[1].view(np.uint64))
        both_prop(lib, lane, p, want)


def test_few_rows_and_overflow(lib, lane):
    f = np.finfo(np.float64).max
    for nrows in (1, 2, 3, 4, 5, 8):
        keys = np.arange(1, nrows + 1, dtype=np.uint64)
        for vals in (np.full(nrows, f), np.array([f, -f, np.nan, np.inf, -np.inf, -0.0, 0.0, 1.0])[:nrows],
                     np.full(nrows, np.iinfo(np.int64).max, np.int64)):
            rows = [[100, 101, 100] for _ in range(nrows)]
            both_prop(lib, lane, Path(keys, vals, [(keys, rows, [100, 101])]))
    # overflow inside a range, then across the merge: ranges {1,2} {3,4} {5,6} {7,8}
    k = np.arange(1, 9, dtype=np.uint64)
    v = np.array([f, f, -f, np.nan, f, 1.0, -f, -f])
    p = Path(k, v, [(k, [[20], [20], [20], [21], [20, 21], [21], [20], [20]], [20, 21])])
    both_prop(lib, lane, p)


def test_hub_of_a_million_edges(lib, lane):
    rng = np.random.default_rng(5)
    n = 10 ** 6
    src = np.arange(1, n + 1, dtype=np.uint64) * 2
    hub = np.uint64(7)
    rows = [np.array([hub, 9 + 2 * (i % 1000)], np.uint64) if i % 3 else np.array([hub], np.uint64) for i in range(n)]
    dest = np.unique(np.concatenate(rows))
    for kind in ("int", "wild"):
        k, v = gv.value_map(rng, src, 0.9, kind)
        both_prop(lib, lane, Path(k, v, [(src, rows, dest)]))


@pytest.mark.parametrize("form", ["host", "dev"])
def test_refusals_write_nothing(lib, lane, form):
    keys, vals = np.array([1, 2, 3], np.uint64), np.array([1, 2, 3], np.int64)
    src, rows, dest = np.array([1, 2, 3], np.uint64), [[5], [6], [5, 6]], np.array([5, 6], np.uint64)
    cases = {
        "map keys": (np.array([1, 3, 2], np.uint64), src, rows, dest),
        "src": (keys, np.array([1, 3, 2], np.uint64), rows, dest),
        "dest": (keys, src, rows, np.array([6, 5], np.uint64)),
        "value not in dest": (keys, src, [[5], [7], [5]], dest),
        "second level dest": None,
    }
    for name, c in cases.items():
        if c is None:
            p = Path(keys, vals, [(src, rows, dest), (dest, [[9], [9]], [9, 8])])
        else:
            p = Path(c[0], vals, [(c[1], c[2], c[3])])
        if form == "host":
            rc, n, ok, ov = prop_host(lib, p, 4)
            assert rc == ERR_ARG and n == 7, name
        else:
            rc, src_rc, n, ok, ov, _ = prop_dev(lib, lane, p, 4)
            assert rc == OK and src_rc == ERR_ARG and n == SENT, name
        assert (ok == SENT).all() and (ov == SENT).all(), name
    if form == "dev":  # the offsets are the device's to check: past v_cap, not from 0, decreasing
        p = Path(keys, vals, [(src, rows, dest)])
        rc, src_rc, n, ok, ov, _ = prop_dev(lib, lane, p, 4, v_caps=[3])
        assert rc == OK and src_rc == ERR_ARG and n == SENT and (ok == SENT).all()
        assert lib.dgx_lane_sync(lane) == OK  # the refusal bit is cleared by the sync that reported it
        for name, off in (("from 1", [1, 1, 2, 4]), ("decreasing", [0, 2, 1, 4])):
            p.levels[0] = (p.levels[0][0], p.levels[0][1], np.asarray(off, np.uint64), p.levels[0][3])
            rc, src_rc, n, ok, ov, _ = prop_dev(lib, lane, p, 4, v_caps=[4])
            assert rc == OK and src_rc == ERR_ARG and n == SENT, name
            assert (ok == SENT).all() and (ov == SENT).all(), name


def test_capacity(lib, lane):
    keys = np.arange(1, 6, dtype=np.uint64)
    p = Path(keys, np.arange(5, dtype=np.int64), [(keys, [[10], [11], [12], [13], [14]], [10, 11, 12, 13, 14])])
    rc, n, ok, ov = prop_host(lib, p, 4)
    assert rc == ERR_CAP and n == 5 and (ok == SENT).all() and (ov == SENT).all()
    rc, src, n, ok, ov, _ = prop_dev(lib, lane, p, 4)
    assert rc == OK and src == ERR_CAP and n == 5 and (ok == SENT).all() and (ov == SENT).all()
    rc, n, ok, ov = prop_host(lib, p, 5)
    assert rc == OK and n == 5


def test_launches_do_not_grow_with_rows_values_or_maps(lib, lane):
    rng = np.random.default_rng(9)
    counts = []
    for scale in (1, 10):
        lv = []
        src = np.arange(1, 200 * scale + 1, dtype=np.uint64)
        for ndest in (60, 250, 3000):  # 1, 2 and 2 radix passes, whatever the scale
            universe = np.arange(10 ** 6, 10 ** 6 + ndest, dtype=np.uint64)
            rows = [rng.choice(universe, size=int(rng.integers(0, 6 * scale))) for _ in range(src.size)]
            rows[0] = universe  # every dest value is used
            lv.append((src, rows, universe))
            src = universe
        k, v = gv.value_map(rng, lv[0][0], 0.8, "dyadic")
        p = Path(k, v, lv)
        cap = 3000
        rc, s, n, ok, ov, launches = prop_dev(lib, lane, p, cap)
        assert rc == OK and s == OK
        _check(n, ok, ov, p.want(), cap)
        assert launches == vp.propagate_launches(k.size, [60, 250, 3000])
        counts.append(launches)
    assert counts[0] == counts[1]


# ---- level aggregation -----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["int", "wild", "dyadic"])
def test_level_agg_random(lib, lane, kind):
    rng = np.random.default_rng(20 + ["int", "wild", "dyadic"].index(kind))
    for _ in range(12):
        s, r, d = gv.path(rng, 1, int(rng.integers(1, 200)), hi=int(rng.integers(3, 400)),
                          avg_deg=float(rng.uniform(0.5, 60)), repeats=bool(rng.integers(2)))[0]
        k, v = gv.value_map(rng, d if d.size else s, rng.random(), kind)
        for fn in FNS:
            both_agg(lib, lane, Agg(fn, k, v, s, r))


def test_level_agg_ties_and_long_rows(lib, lane):
    k = np.arange(1, 7, dtype=np.uint64)
    for v in (np.array([0.0, -0.0, np.nan, 1.0, np.inf, -np.inf]), np.array([3, 3, -1, -1, 5, 5], np.int64)):
        rows = [[1, 2], [2, 1], [3, 4], [4, 3], [5, 6, 1], list(range(1, 7)) * 30, [], [9]]
        for fn in FNS:
            both_agg(lib, lane, Agg(fn, k, v, np.arange(10, 18, dtype=np.uint64), rows))


def test_level_agg_refusals_and_capacity(lib, lane):
    k, v = np.array([1, 2], np.uint64), np.array([1, 2], np.int64)
    for name, a in {"map keys": Agg("sum", [2, 1], v, [5, 6], [[1], [2]]),
                    "src": Agg("sum", k, v, [6, 5], [[1], [2]])}.items():
        rc, n, ok, ov = agg_host(lib, a, 4)
        assert rc == ERR_ARG and n == 7 and (ok == SENT).all(), name
        rc, s, n, ok, ov, _ = agg_dev(lib, lane, a, 4)
        assert rc == OK and s == ERR_ARG and n == SENT and (ok == SENT).all() and (ov == SENT).all(), name
    a = Agg("max", k, v, [5, 6], [[1], [2]])
    rc, s, n, ok, ov, _ = agg_dev(lib, lane, a, 4, v_cap=1)
    assert rc == OK and s == ERR_ARG and n == SENT
    for name, off in (("from 1", [1, 1, 2]), ("decreasing", [0, 2, 1])):
        b = Agg("max", k, v, [5, 6], [[1], [2]])
        b.v_off = np.asarray(off, np.uint64)
        rc, s, n, ok, ov, _ = agg_dev(lib, lane, b, 4, v_cap=2)
        assert rc == OK and s == ERR_ARG and n == SENT and (ok == SENT).all() and (ov == SENT).all(), name
    rc, n, ok, ov = agg_host(lib, a, 1)
    assert rc == ERR_CAP and n == 2 and (ok == SENT).all()
    rc, s, n, ok, ov, _ = agg_dev(lib, lane, a, 1)
    assert rc == OK and s == ERR_CAP and n == 2 and (ok == SENT).all() and (ov == SENT).all()


# ---- chains, threads, size -------------------------------------------------------------------------------------------

def test_device_chain_from_unfiltered_rows(lib, lane):
    """A level whose rows come from dgx_dev_list_uids_unfiltered_rows and whose dest is their
    dgx_dev_merge_sorted_matrix, with no copy of rows or dest to the host.  ndest is an exact host size, as the header
    says: the caller reads the merge's length word (here it is known from the test data)."""
    import torch

    from dgraph_b200 import codec, pb
    from oracle import pyoracle as orc

    rng = np.random.default_rng(31)
    nrows = 60
    src = np.unique(rng.integers(1, 10 ** 6, 300, dtype=np.uint64))[:nrows]
    lists = [np.unique(rng.integers(1, 4000, int(rng.integers(0, 200)), dtype=np.uint64)) for _ in range(nrows)]
    tab = (C.c_void_p * nrows)()
    handles, keep = [], []
    for i, l in enumerate(lists):
        if l.size == 0:
            continue
        op = orc.encode(l, 256)
        pk = pb.UidPack(op.block_size, op.base, op.num_uids, op.delta_off, op.deltas).normalized()
        view = codec.view_of(pk)
        keep.append((pk, view))
        h = C.c_void_p()
        assert lib.dgx_dev_pack_upload(lane, C.byref(view), C.byref(h)) == OK
        handles.append(h)
        tab[i] = h.value
    m = int(sum(l.size for l in lists))
    mut_off = np.zeros(nrows + 1, np.uint64)
    d_rows = torch.zeros(m + 1, dtype=torch.int64, device="cuda")
    d_off = torch.zeros(nrows + 1, dtype=torch.int64, device="cuda")
    d_dest = torch.zeros(m + 1, dtype=torch.int64, device="cuda")
    d_dlen = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.dgx_dev_list_uids_unfiltered_rows(lane, tab, nrows, None, None, mut_off.ctypes.data, 0, 0,
                                                 d_rows.data_ptr(), m, d_off.data_ptr()) == OK
    assert lib.dgx_dev_merge_sorted_matrix(lane, d_rows.data_ptr(), d_off.data_ptr(), nrows, m, d_dest.data_ptr(), m,
                                           d_dlen.data_ptr()) == OK
    dest = np.unique(np.concatenate(lists))
    k, v = gv.value_map(rng, src, 0.6, "wild")
    p = Path(k, v, [(src, lists, dest)])
    rc, s, n, ok, ov, _ = prop_dev(lib, lane, p, dest.size,
                                   levels=[(_up(src), d_rows, d_off, d_dest, dest.size)], v_caps=[m])
    assert rc == OK and s == OK, lib.dgx_last_error()
    _check(n, ok, ov, p.want(), dest.size)
    k2, v2 = gv.value_map(rng, dest, 0.5, "int")
    a = Agg("sum", k2, v2, src, lists)
    t = [_up(x) for x in (k2, v2.view(np.uint64), src)]
    ok, ov, dn = _sent(nrows + GUARD), _sent(nrows + GUARD), _sent(1)
    assert lib.dgx_dev_var_level_agg(lane, 1, 2, t[0].data_ptr(), t[1].data_ptr(), k2.size, t[2].data_ptr(), nrows,
                                     d_off.data_ptr(), d_rows.data_ptr(), m, ok.data_ptr(), ov.data_ptr(), nrows,
                                     dn.data_ptr()) == OK
    assert lib.dgx_lane_sync(lane) == OK
    _check(int(_h(dn)[0]), _h(ok), _h(ov), a.want(), nrows)
    for h_ in handles:
        lib.dgx_dev_pack_free(h_)


def test_concurrent_callers(lib):
    rng = np.random.default_rng(41)
    cases = []
    for _ in range(16):
        lv = gv.path(rng, 2, 80, hi=200, avg_deg=4.0)
        cases.append(Path(*gv.value_map(rng, lv[0][0], 0.7, "wild"), lv))
    errors = []

    def worker(w):
        try:
            for p in cases[w::4]:
                cap = max(p.levels[-1][3].size, 1)
                rc, n, ok, ov = prop_host(lib, p, cap)
                assert rc == OK
                _check(n, ok, ov, p.want(), cap)
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=worker, args=(w,)) for w in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


def test_c17_sized_calls(lib, lane):
    """C17b's shape: 1e6 rows and about 2e7 values of the C13 matrix, a map over most destinations, every function,
    and the same matrix as one propagation level (its most popular destination is a hub of about 1e6 in-edges)."""
    import gen_groupby as gg

    rng = np.random.default_rng(13)
    src, v, v_off, dest = gg.c13_rows(rng)
    rows = np.split(v, v_off[1:-1].astype(np.int64))
    for kind in ("int", "wild"):
        k, vals = gv.value_map(rng, dest, 0.9, kind)
        for fn in FNS:
            both_agg(lib, lane, Agg(fn, k, vals, src, rows))
        k, vals = gv.value_map(rng, src, 0.9, kind)
        both_prop(lib, lane, Path(k, vals, [(src, rows, dest)]))


def test_reference_answers_on_the_fixture(lib):
    """The reference's nine value-variable tests on query/common_test.go's data, through algo.PropagateVar and
    algo.LevelAgg."""
    import valvar_golden as vg

    from dgraph_b200 import algo

    vg.check(vg.replay(algo.PropagateVar, algo.LevelAgg))
