"""orderasc / orderdesc by a value variable on the device (dgx_var_order and dgx_dev_var_order): random cases and
shaped calls against the line-by-line restatement (var_order_oracle.c), bit for bit, with guard words past every
output; tier-1-only, tier-2-only and mixed calls; rows of 12 and 13 tied entries; long tied rows on the CTA path that
reach partitionEqual, breakPatterns, partialInsertionSort, reverseRange and heapSort; every device-side refusal; the
launch count against the plan model (var_order_plan.py) as rows, values and ties grow 100-fold; a device chain from
@filter through math() and the order into @cascade; concurrent callers and a C20a-sized call.  Runs on an H100 only
(`pytest -m gpu`)."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen_var_order as gv  # noqa: E402
import var_order_golden as vg  # noqa: E402
import var_order_oracle as vo  # noqa: E402
import var_order_plan as vp  # noqa: E402

pytestmark = pytest.mark.gpu

OK, ERR_ARG, ERR_CAP = 0, -3, -4
SENT = 0xDEADBEEFCAFEF00D
GUARD = 4


@pytest.fixture(scope="module")
def lib():
    from dgraph_b200 import _lib

    L = _lib.load()
    _lib.check(L.dgx_init(-1))
    return L


def new_lane(lib):
    import torch

    stream = torch.cuda.Stream()
    ln = lib.dgx_lane_create(0, C.c_void_p(stream.cuda_stream))
    assert ln
    return ln, stream


@pytest.fixture(scope="module")
def lane(lib):
    ln, _ = new_lane(lib)
    yield ln
    lib.dgx_lane_destroy(ln)


def _t(a, dtype=np.uint64):
    import torch

    a = np.ascontiguousarray(np.asarray(a, dtype))
    if a.size == 0:
        a = np.zeros(1, dtype)
    if dtype == np.uint64:
        return torch.from_numpy(a.view(np.int64)).cuda()
    return torch.from_numpy(a).cuda()


def _h(t, n, dtype=np.uint64):
    a = t.cpu().numpy()[:n]
    return a.view(np.uint64).copy() if dtype == np.uint64 else a.copy()


def sent(n):
    import torch

    return torch.full((n,), SENT - (1 << 64), dtype=torch.int64, device="cuda")


def csr(rows):
    off = np.zeros(len(rows) + 1, np.uint64)
    np.cumsum([len(r) for r in rows], out=off[1:])
    v = np.concatenate([np.asarray(r, np.uint64) for r in rows]) if int(off[-1]) else np.zeros(0, np.uint64)
    return v, off


def want(case):
    """The restatement's (rows, dest), or the error class."""
    try:
        return vo.var_order(*case)
    except (vo.NilMap, vo.NotSortable) as e:
        return type(e)


def same(got, exp):
    (gr, gd), (er, ed) = got, exp
    return len(gr) == len(er) and all(np.array_equal(x, y) for x, y in zip(gr, er)) and np.array_equal(gd, ed)


def launches(lib):
    from dgraph_b200 import _lib

    return _lib.stats()["kernel_launches"]


def host_call(lib, case, out_cap=None, dest_cap=None):
    """dgx_var_order with guard words past every output.  Returns (rc, (rows, dest) or None, guards intact, launches)."""
    from dgraph_b200.algo import var_order_leaf

    m, desc, dest, rows, count, offset = case
    keep, leaf = var_order_leaf(m)
    d = np.ascontiguousarray(np.asarray(dest, np.uint64))
    v, v_off = csr(rows)
    v = v if v.size else np.zeros(1, np.uint64)
    nrows, M = len(rows), int(v_off[-1])
    out_cap = M if out_cap is None else out_cap
    dest_cap = d.size if dest_cap is None else dest_cap
    out = np.full(out_cap + GUARD, SENT, np.uint64)
    oo = np.full(nrows + 1 + GUARD, SENT, np.uint64)
    dout = np.full(dest_cap + GUARD, SENT, np.uint64)
    n = C.c_size_t(SENT)
    l0 = launches(lib)
    rc = lib.dgx_var_order(C.byref(leaf), int(desc), (d if d.size else np.zeros(1, np.uint64)).ctypes.data, d.size,
                           v.ctypes.data, v_off.ctypes.data, nrows, count, offset, out.ctypes.data, oo.ctypes.data,
                           out_cap, dout.ctypes.data, dest_cap, C.byref(n))
    nl = launches(lib) - l0
    del keep
    guards = np.all(out[out_cap:] == SENT) and np.all(oo[nrows + 1:] == SENT) and np.all(dout[dest_cap:] == SENT)
    if rc != OK:
        return rc, None, guards and np.all(out == SENT) and np.all(dout == SENT), nl, n.value
    K = int(oo[nrows])
    guards = guards and np.all(out[K:] == SENT) and np.all(dout[n.value:] == SENT)
    return rc, ([out[int(oo[i]):int(oo[i + 1])].copy() for i in range(nrows)], dout[:n.value].copy()), guards, nl, n.value


def dev_leaf(m, slack=0, len_word=False):
    """(kept tensors, MathLeaf over device arrays) of a map, with `slack` garbage entries past it when its count comes
    from a device word."""
    from dgraph_b200 import _lib

    k, w, t, nil = vo.map_arrays(m)
    typed = m is not None and len(m) == 2
    n = k.size
    pad = slack if len_word else 0
    kk = _t(np.concatenate([k, np.full(pad, 7, np.uint64)]))
    ww = _t(np.concatenate([w, np.full(pad, 7, np.uint64)]))
    keep = [kk, ww]
    tag_p = None
    if not typed and m is not None:
        tt = _t(np.concatenate([t, np.full(pad, 9, np.uint8)]), np.uint8)
        keep.append(tt)
        tag_p = tt.data_ptr()
    d_len = None
    if len_word:
        lw = _t(np.array([n | (0x5A << 40)], np.uint64))
        keep.append(lw)
        d_len = lw.data_ptr()
    typ = (vo.T_INT if np.asarray(m[1]).dtype == np.int64 else vo.T_FLOAT) if typed else vo.T_INT
    leaf = _lib.MathLeaf(kk.data_ptr(), ww.data_ptr(), tag_p, d_len, n + pad, typ, nil)
    return keep, leaf


def dev_call(lib, lane, case, slack=0, len_words=False, mutate=None):
    """dgx_dev_var_order with `slack` garbage slots past dest, the values and the map (their lengths then from device
    words when len_words).  mutate(arrays) may break the inputs before upload.  Returns (rc, sync rc, dest length word,
    (rows, dest) or None, launches, guards intact)."""
    m, desc, dest, rows, count, offset = case
    d = np.asarray(dest, np.uint64)
    v, v_off = csr(rows)
    a = {"dest": np.concatenate([d, np.full(slack if len_words else 0, 3, np.uint64)]),
         "v": np.concatenate([v, np.full(slack, 9, np.uint64)]), "v_off": v_off.copy(), "map": m}
    if mutate:
        mutate(a)
    nrows, ndest, vcap = len(rows), a["dest"].size, a["v"].size
    keep, leaf = dev_leaf(a["map"], slack, len_words)
    dd, vv, oo_in = _t(a["dest"]), _t(a["v"]), _t(a["v_off"])
    dw = _t(np.array([d.size | (0x33 << 36)], np.uint64)) if len_words else None
    out, oo, dout, dlen = sent(vcap + GUARD), sent(nrows + 1 + GUARD), sent(ndest + GUARD), sent(1)
    l0 = lib.dgx_lane_launches(lane)
    rc = lib.dgx_dev_var_order(lane, C.byref(leaf), int(desc), dd.data_ptr(), ndest,
                               dw.data_ptr() if dw is not None else None, vv.data_ptr(), oo_in.data_ptr(), nrows, vcap,
                               count, offset, out.data_ptr(), oo.data_ptr(), vcap, dout.data_ptr(), ndest,
                               dlen.data_ptr())
    src = lib.dgx_lane_sync(lane) if rc == OK else None
    nl = lib.dgx_lane_launches(lane) - l0
    del keep
    o, off, de, L = _h(out, vcap + GUARD), _h(oo, nrows + 1 + GUARD), _h(dout, ndest + GUARD), int(_h(dlen, 1)[0])
    guards = np.all(o[vcap:] == SENT) and np.all(off[nrows + 1:] == SENT) and np.all(de[ndest:] == SENT)
    if rc != OK or src != OK:
        guards = guards and np.all(o == SENT) and np.all(off == SENT) and np.all(de == SENT)
        return rc, src, L, None, nl, guards
    K = int(off[nrows])
    guards = guards and np.all(o[K:] == SENT) and np.all(de[L:] == SENT)
    return rc, src, L, ([o[int(off[i]):int(off[i + 1])].copy() for i in range(nrows)], de[:L].copy()), nl, guards


def run_both(lib, lane, case, **kw):
    """Both forms against the restatement; returns the restatement's answer."""
    exp = want(case)
    rc, got, g, nl, _ = host_call(lib, case)
    assert g
    if isinstance(exp, type):
        assert rc == ERR_ARG
    else:
        assert rc == OK and same(got, exp)
        assert nl == vp.launches(len(case[2]), len(case[3]))
    rc, src, L, got, nl, g = dev_call(lib, lane, case, **kw)
    assert rc == OK and g
    if isinstance(exp, type):
        assert src == ERR_ARG and L == 0
    else:
        assert src == OK and same(got, exp), case
        assert nl == vp.launches(len(case[2]) + (kw.get("slack", 0) if kw.get("len_words") else 0), len(case[3]))
    return exp


@pytest.mark.parametrize("seed", range(4))
def test_random_cases(lib, lane, seed):
    rng = np.random.default_rng(2000 + seed)
    for i in range(60):
        case = gv.random_case(rng)
        if case[0] is None:
            continue
        run_both(lib, lane, case, slack=int(rng.integers(0, 4)), len_words=bool(i & 1))


@pytest.mark.parametrize("label,case,want", vg.cases(), ids=[c[0] for c in vg.cases()])
def test_reference_answers(lib, lane, label, case, want):
    from dgraph_b200 import _lib
    from dgraph_b200.algo import OrderByVar

    if want == "nil":
        with pytest.raises(_lib.DgxError, match="used before definition"):
            OrderByVar(*case)
        return
    rows, dest = OrderByVar(*case)
    assert vg.check(rows, dest.Uids, want), label
    exp = run_both(lib, lane, case)
    assert vg.check(*exp, want)


def int_map(keys, vals):
    return np.asarray(keys, np.uint64), np.asarray(vals, np.int64)


def float_map(keys, vals):
    return np.asarray(keys, np.uint64), np.asarray(vals, np.float64)


def test_tier_mixes(lib, lane):
    rng = np.random.default_rng(7)
    U = np.arange(1, 5001, dtype=np.uint64)
    dest = U[rng.random(U.size) < 0.9]
    rows = [np.sort(rng.choice(U, size=int(rng.integers(0, 600)), replace=False)) for _ in range(40)]
    distinct = float_map(U, rng.permutation(U.size).astype(np.float64) - 2000.5)
    tied = int_map(U, rng.integers(0, 5, U.size))
    mixed_k, mixed_w, mixed_t = gv.random_map(rng, U.tolist(), "math")
    mixed_t = np.where(mixed_t == gv.T_BOOL, gv.T_NIL, mixed_t).astype(np.uint8)
    for m in (distinct, tied, (mixed_k, np.where(mixed_t == gv.T_NIL, 0, mixed_w).astype(np.uint64), mixed_t)):
        for desc in (False, True):
            for count, offset in ((0, 0), (10, 0), (-7, 0), (3, 5), (0, 10000)):
                run_both(lib, lane, (m, desc, dest, rows, count, offset))
    # one call holding tier-1 rows (distinct keys), tier-2 rows (ties past 12) and rows without W
    keys = U[:3000]
    vals = np.where(keys < 1500, keys.astype(np.int64) * 7, (keys.astype(np.int64) % 3))
    run_both(lib, lane, (int_map(keys, vals), True, dest, rows, 5, 2))


def test_rows_of_12_and_13(lib, lane):
    for n in (11, 12, 13, 14):
        keys = np.arange(1, n + 1, dtype=np.uint64)
        for vals in (np.zeros(n, np.int64), np.arange(n, dtype=np.int64) % 3, np.arange(n, dtype=np.int64)[::-1] % 2):
            for desc in (False, True):
                run_both(lib, lane, (int_map(keys, vals), desc, keys, [keys, keys[::2]], 0, 0))


def long_row_case(kind, n=20000, desc=False):
    rng = np.random.default_rng(n)
    keys = np.arange(1, n + 1, dtype=np.uint64)
    if kind == "ties":
        m = int_map(keys, rng.integers(0, 100, n))
    elif kind == "nil":  # two nils compare as desc: an inconsistent comparator that runs pdqsort into heapSort
        m = (keys, np.zeros(n, np.uint64), np.full(n, gv.T_NIL, np.uint8))
    elif kind == "dec":  # strictly decreasing but for one tie at the end: reverseRange, then partialInsertionSort
        m = int_map(keys, np.concatenate([np.arange(n - 1, 0, -1), [1]]).astype(np.int64))
    elif kind == "nan":
        w = np.where(rng.random(n) < 0.3, np.nan, rng.integers(0, 50, n).astype(np.float64))
        m = float_map(keys, w)
    else:
        raise ValueError(kind)
    return (m, desc, keys, [keys], 0, 0)


@pytest.mark.parametrize("kind,desc", [("ties", False), ("ties", True), ("nil", True), ("dec", False), ("nan", True),
                                       ("nan", False)])
def test_long_tied_row_takes_the_cta_path(lib, lane, kind, desc):
    case = long_row_case(kind, desc=desc)
    assert len(case[3][0]) > vp.K["CTA_MIN"]
    vo.stats()
    run_both(lib, lane, case)
    st = vo.stats()
    if kind != "dec":
        assert st["partition"] + st["partition_equal"] > 0
    if kind == "ties":
        assert st["partition_equal"] and st["partial_insertion_ok"]
    if kind == "nil":
        assert st["heap"] and st["break_patterns"]
    if kind == "dec":
        assert st["reverse"]


def test_device_refusals(lib, lane):
    keys = np.arange(1, 41, dtype=np.uint64)
    base = (int_map(keys, keys.astype(np.int64) % 4), False, keys, [keys[:20], keys[10:]], 0, 0)
    assert dev_call(lib, lane, base)[1] == OK

    def dest_desc(a):
        a["dest"][5], a["dest"][6] = a["dest"][6], a["dest"][5]

    def keys_desc(a):
        k, w = a["map"]
        k = k.copy()
        k[3], k[4] = k[4], k[3]
        a["map"] = (k, w)

    def row_desc(a):
        a["v"][2], a["v"][3] = a["v"][3], a["v"][2]

    def off_start(a):
        a["v_off"][0] = 1

    def off_past(a):
        a["v_off"][-1] = a["v"].size + 1

    def off_dec(a):
        a["v_off"][1] = a["v_off"][2] + 1

    def bad_tag(a):
        k, w = a["map"]
        a["map"] = (k, w.view(np.uint64), np.where(np.arange(k.size) == 7, 5, gv.T_INT).astype(np.uint8))

    def bool_first(a):
        k, w = a["map"]
        a["map"] = (k, w.view(np.uint64), np.where(np.arange(k.size) == 10, gv.T_BOOL, gv.T_INT).astype(np.uint8))

    for mut in (dest_desc, keys_desc, row_desc, off_start, off_past, off_dec, bad_tag, bool_first):
        rc, src, L, got, nl, g = dev_call(lib, lane, base, mutate=mut)
        assert rc == OK and src == ERR_ARG and L == 0 and got is None and g, mut.__name__
    # a bool that is not a row's first W entry is sorted, not refused
    def bool_later(a):
        k, w = a["map"]
        a["map"] = (k, w.view(np.uint64), np.where(np.arange(k.size) == 12, gv.T_BOOL, gv.T_INT).astype(np.uint8))
    assert dev_call(lib, lane, base, mutate=bool_later)[1] == OK
    # length words past their rooms
    import torch
    from dgraph_b200 import _lib
    keep, leaf = dev_leaf(base[0])
    v, v_off = csr(base[3])
    dd, vv, oo_in = _t(keys), _t(v), _t(v_off)
    out, oo, dout, dlen = sent(v.size), sent(3), sent(keys.size), sent(1)
    for over in ("dest", "map"):
        w = _t(np.array([keys.size + 1], np.uint64))
        lf = _lib.MathLeaf(leaf.key, leaf.word, None, w.data_ptr() if over == "map" else None, keys.size, 1, 0)
        rc = lib.dgx_dev_var_order(lane, C.byref(lf), 0, dd.data_ptr(), keys.size,
                                   w.data_ptr() if over == "dest" else None, vv.data_ptr(), oo_in.data_ptr(), 2, v.size,
                                   0, 0, out.data_ptr(), oo.data_ptr(), v.size, dout.data_ptr(), keys.size,
                                   dlen.data_ptr())
        assert rc == OK and lib.dgx_lane_sync(lane) == ERR_ARG and int(_h(dlen, 1)[0]) == 0, over
    torch.cuda.synchronize()
    del keep


def test_device_argument_and_capacity_errors(lib, lane):
    from dgraph_b200 import _lib

    keys = np.arange(1, 9, dtype=np.uint64)
    keep, leaf = dev_leaf(int_map(keys, keys.astype(np.int64)))
    dd, vv, oo_in = _t(keys), _t(keys), _t(np.array([0, 8], np.uint64))
    out, oo, dout, dlen = sent(8), sent(2), sent(8), sent(1)

    def call(lf=leaf, out_cap=8, dest_cap=8, nrows=1, d_v_off=oo_in.data_ptr()):
        return lib.dgx_dev_var_order(lane, C.byref(lf) if lf is not None else None, 0, dd.data_ptr(), 8, None,
                                     vv.data_ptr(), d_v_off, nrows, 8, 0, 0, out.data_ptr(), oo.data_ptr(), out_cap,
                                     dout.data_ptr(), dest_cap, dlen.data_ptr())

    assert call() == OK and lib.dgx_lane_sync(lane) == OK
    out.fill_(SENT - (1 << 64))
    nil = _lib.MathLeaf(None, None, None, None, 0, 1, 1)
    assert call(lf=nil) == ERR_ARG and call(lf=None) == ERR_ARG
    assert call(lf=_lib.MathLeaf(leaf.key, leaf.word, None, None, 8, 3, 0)) == ERR_ARG
    assert call(out_cap=7) == ERR_CAP and call(dest_cap=7) == ERR_CAP
    assert call(nrows=1 << 32) == ERR_ARG and call(d_v_off=None) == ERR_ARG
    assert np.all(_h(out, 8) == SENT)
    del keep


def test_launches_constant(lib, lane):
    """The launch count depends on nrows' bit width alone: rows, values, ties and the map grow 100-fold."""
    rng = np.random.default_rng(11)
    for nrows in (1, 2, 256, 257):
        counts = set()
        for scale in (1, 10, 100):
            n = 50 * scale
            U = np.arange(1, n * 4, dtype=np.uint64)
            rows = [np.sort(rng.choice(U, size=min(U.size, int(rng.integers(0, 3 * scale + 1))), replace=False))
                    for _ in range(nrows)]
            vals = rng.integers(0, max(1, 100 // scale), U.size)
            case = (int_map(U, vals), bool(scale & 1), U, rows, 3, 1)
            exp = want(case)
            rc, got, g, nl, _ = host_call(lib, case)
            assert rc == OK and g and same(got, exp)
            counts.add(nl)
            rc, src, L, got, dl, g = dev_call(lib, lane, case)
            assert src == OK and same(got, exp)
            counts.add(dl)
        assert counts == {vp.launches(1, nrows)}, (nrows, counts)


def test_device_chain(lib, lane):
    """Unfiltered rows -> dgx_dev_sg_filter (count = offset = 0) -> dgx_dev_math_eval over a device map ->
    dgx_dev_var_order with first: 3 -> dgx_dev_cascade with DGX_CASCADE_ORDERED, no host read between the calls."""
    import torch

    from dgraph_b200 import _lib
    from dgraph_b200.algo import EvalMath, math_program, sg_filter_flat, sg_filter_leaf_arrays, sg_filter_tree

    rng = np.random.default_rng(5)
    U = np.arange(1, 3001, dtype=np.uint64)
    d0 = U[rng.random(U.size) < 0.8]
    rows = [np.sort(rng.choice(d0, size=int(rng.integers(0, 400)), replace=False)) for _ in range(30)]
    flt = np.sort(rng.choice(d0, size=d0.size // 2, replace=False))
    mk = np.sort(rng.choice(U, size=2000, replace=False))
    mv = rng.integers(-20, 20, mk.size).astype(np.int64)
    # the host answer: filter, math (s * 2 + 1), order, then cascade's filter of the ordered rows by their dest
    f_rows = [np.array([x for x in r if x in set(flt.tolist())], np.uint64) for r in rows]
    f_dest = np.array(sorted(set(d0.tolist()) & set(flt.tolist())), np.uint64)
    tree = ("+", ("*", ("var", "s"), ("const", 2)), ("const", 1))
    kind, ek, ew, et = EvalMath(tree, {"s": (mk, mv)})
    exp_rows, exp_dest = vo.var_order((ek, ew, et), True, f_dest, f_rows, 3, 0)
    # device
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
    names = {}
    prog = math_program(tree, names)
    d_mk, d_mv = _t(mk), _t(mv.view(np.uint64))
    ml = (_lib.MathLeaf * 1)(_lib.MathLeaf(d_mk.data_ptr(), d_mv.data_ptr(), None, None, mk.size, 1, 0))
    cap = mk.size + 1
    m_key, m_word = sent(cap), sent(cap)
    m_tag = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    m_info = sent(1)
    assert lib.dgx_dev_math_eval(lane, (_lib.MathNode * len(prog))(*prog), len(prog), ml, 1, None, 0,
                                 m_key.data_ptr(), m_word.data_ptr(), m_tag.data_ptr(), cap, m_info.data_ptr()) == OK
    var = _lib.MathLeaf(m_key.data_ptr(), m_word.data_ptr(), m_tag.data_ptr(), m_info.data_ptr(), cap, 1, 0)
    o_out, o_off, o_dest, o_len = sent(v.size), sent(nrows + 1), sent(d0.size), sent(1)
    l0 = lib.dgx_lane_launches(lane)
    assert lib.dgx_dev_var_order(lane, C.byref(var), 1, s_dest.data_ptr(), d0.size, s_len.data_ptr(), s_out.data_ptr(),
                                 s_off.data_ptr(), nrows, v.size, 3, 0, o_out.data_ptr(), o_off.data_ptr(), v.size,
                                 o_dest.data_ptr(), d0.size, o_len.data_ptr()) == OK
    assert lib.dgx_lane_launches(lane) - l0 == vp.launches(d0.size, nrows)
    # @cascade over the ordered node: one root, FILTERED | ORDERED, its rows filtered by its own dest (order kept)
    tr_parent, tr_flags = np.array([0xFFFFFFFF], np.uint32), np.array([4 | 8], np.uint8)
    tr_first, tr_off, tr_cl = np.zeros(1, np.int32), np.zeros(1, np.int32), np.zeros(1, np.uint64)
    ctree = _lib.CascadeTree(1, tr_parent.ctypes.data, tr_flags.ctypes.data, tr_first.ctypes.data, tr_off.ctypes.data,
                             tr_cl.ctypes.data)
    assert lib.dgx_lane_sync(lane) == OK
    n_dest = int(_h(o_len, 1)[0])  # cascade's node takes an exact dest length
    node = (_lib.CascadeNode * 1)(_lib.CascadeNode(o_out.data_ptr(), o_off.data_ptr(), nrows, v.size,
                                                   o_dest.data_ptr(), n_dest, None, 0))
    c_out, c_off, c_dest, c_doff, c_sizes = sent(v.size), sent(nrows + 1), sent(max(n_dest, 1)), sent(2), sent(2)
    assert lib.dgx_dev_cascade(lane, C.byref(ctree), node, c_out.data_ptr(), c_off.data_ptr(), v.size,
                               c_dest.data_ptr(), c_doff.data_ptr(), max(n_dest, 1), c_sizes.data_ptr()) == OK
    assert lib.dgx_lane_sync(lane) == OK
    off = _h(c_off, nrows + 1)
    out = _h(c_out, int(off[-1]))
    got_rows = [out[int(off[i]):int(off[i + 1])] for i in range(nrows)]
    assert all(np.array_equal(a, b) for a, b in zip(got_rows, exp_rows))
    assert np.array_equal(_h(c_dest, n_dest), exp_dest)
    del keep_l


def test_concurrent_callers(lib):
    rng = np.random.default_rng(9)
    cases = [gv.random_case(rng, max_rows=20, max_len=300, universe=600) for _ in range(24)]
    cases = [c for c in cases if c[0] is not None]
    exp = [want(c) for c in cases]
    errors = []

    def work(idx):
        try:
            for i in idx:
                rc, got, g, _, _ = host_call(lib, cases[i])
                ok = g and ((rc == ERR_ARG) if isinstance(exp[i], type) else (rc == OK and same(got, exp[i])))
                if not ok:
                    errors.append(i)
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    th = [threading.Thread(target=work, args=(list(range(k, len(cases), 4)),)) for k in range(4)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors


def test_c20a_sized_call(lib):
    """C20a's shape: 10 000 rows, about 1e7 values, an int map over about 90 % of dest with values in 0..99, first: 10."""
    from dgraph_b200.algo import OrderByVar

    rng = np.random.default_rng(20)
    N = 3_000_000
    U = np.arange(1, N + 1, dtype=np.uint64)
    dest = U[rng.random(N) < 0.95]
    mk = dest[rng.random(dest.size) < 0.9]
    m = int_map(mk, rng.integers(0, 100, mk.size))
    lens = rng.integers(500, 1500, 10_000)
    rows = [np.unique(rng.integers(1, N + 1, int(k)).astype(np.uint64)) for k in lens]
    exp_rows, exp_dest = vo.var_order(m, True, dest, rows, 10, 0)
    got_rows, got_dest = OrderByVar(m, True, dest, rows, 10, 0)
    assert all(np.array_equal(a, b) for a, b in zip(got_rows, exp_rows))
    assert np.array_equal(got_dest.Uids, exp_dest)
