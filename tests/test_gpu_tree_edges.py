"""regexp()'s and math()'s tree evaluators at their chunk, CTA and tile edges (fixtures and host model:
tests/tree_geometry.py): 1 023 to 3 073 driving leaves, leaf tables past TG_NT with the pack / list split at 1023, 1024
and 1025, value flags past TG_NT, empty driving rows and row boundaries on CTA edges, dcap far above the rows, the
three paths, an exhaustive truth table of small trees, depth-32 chains, compactions of 2 047 to 4 097 candidates; U
lengths at the warp, CTA and tile edges with absent root keys, promotion from the first or last CTA, refusal counts
across CTAs, the COND over nil rule, rooms of 0, count words below the room, 2^64 - 1 keys, constants over ranges and
the program limits.

Every case runs through the host form (dgx_trigram_query, dgx_math_eval) and the device form (dgx_dev_trigram_query,
dgx_dev_math_eval) as the fixture names it.  Return codes, the lane's sync code, the length and info words and the
device form's launches equal the model's; the outputs equal the oracle's bit for bit (math words as u64); nothing is
written past an output, and a refused or over-capacity call writes only what the library documents.  Runs on an H100
only (`pytest -m gpu`)."""
import ctypes as C
import functools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen_trigram as gt  # noqa: E402
import tree_geometry as tg  # noqa: E402
from trigram_cases import SENTINEL, Raw  # noqa: E402

pytestmark = pytest.mark.gpu

SENT = 0xDEADBEEFCAFEF00D
GUARD = 4
FIXTURES = {f.name: f for f in tg.all_fixtures()}
TG = [(n, k) for n, f in FIXTURES.items() if isinstance(f, tg.TgFix) for k in range(len(f.cases))
      if len(f.cases) < 50] + [(n, None) for n, f in FIXTURES.items() if isinstance(f, tg.TgFix) and len(f.cases) >= 50]
MT = [(n, k) for n, f in FIXTURES.items() if isinstance(f, tg.MtFix) for k in range(len(f.cases))]


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


@functools.lru_cache(maxsize=None)
def model(name):
    return tg.outcomes(FIXTURES[name])[0]


# ---- regexp() ---------------------------------------------------------------------------------------------------------

def raw_of(case):
    npacks = tg.tg_npacks(case.leaves)
    al = gt.to_algo(case.leaves)
    return Raw(case.tree, packs=[a[0] for a in al[:npacks]], muts=[a[1] for a in al[:npacks]], lists=al[npacks:])


def tg_dev(lib, lane, raw, after, cap):
    """dgx_dev_trigram_query: (rc, sync rc, out with its guard words, the length word, launches)."""
    import torch

    from dgraph_b200 import codec

    tab = (C.c_void_p * max(raw.npacks, 1))()
    handles = []
    try:
        for i, p in enumerate(raw.packs):
            if p is None or p.nblocks == 0:
                continue
            h = C.c_void_p()
            assert lib.dgx_dev_pack_upload(lane, C.byref(codec.view_of(p.normalized())), C.byref(h)) == tg.OK
            handles.append(h)
            tab[i] = h.value
        d_mu = torch.from_numpy(raw.mu.view(np.int64)).cuda()
        d_mf = torch.from_numpy(raw.mf).cuda()
        d_lists = torch.from_numpy(raw.lists.view(np.int64)).cuda()
        d_len = torch.full((1,), -7, dtype=torch.int64, device="cuda")
        d_out = torch.full((max(cap, 1) + GUARD,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        l0 = lib.dgx_lane_launches(lane)
        rc = lib.dgx_dev_trigram_query(
            lane, C.byref(raw.qt), tab, raw.npacks, C.c_void_p(d_mu.data_ptr()), C.c_void_p(d_mf.data_ptr()),
            raw.mut_off.ctypes.data, C.c_void_p(d_lists.data_ptr()), raw.list_off.ctypes.data, raw.nlists, after,
            C.c_void_p(d_out.data_ptr()), cap, C.c_void_p(d_len.data_ptr()))
        nl = lib.dgx_lane_launches(lane) - l0
        rs = lib.dgx_lane_sync(lane) if rc == tg.OK else None
        return rc, rs, d_out.cpu().numpy().view(np.uint64), int(d_len.cpu().numpy().view(np.uint64)[0]), nl
    finally:
        for h in handles:
            lib.dgx_dev_pack_free(h)


def tg_check(lib, lane, name, k):
    f = FIXTURES[name]
    case, outs = f.cases[k], model(name)[k]
    raw = raw_of(case)
    lb = [gt.leaf_bound(lf) for lf in case.leaves]
    for call, o in zip(f.calls, outs):
        what = (name, k, call)
        rc, sync, want = tg.tg_expected(case, call)
        assert (o.rc, o.sync) == (rc, sync), what
        cap = tg.tg_cap(tg.tp.plan(case.tree, lb), call)
        if call.form == "host":
            got_rc, out, n = raw.host(case.after, cap)
            assert got_rc == o.rc, what
            if o.rc != tg.OK:
                assert n == SENTINEL and np.all(out == np.uint64(SENTINEL)), what
                continue
        else:
            got_rc, rs, out, n, nl = tg_dev(lib, lane, raw, case.after, cap)
            assert (got_rc, rs) == (o.rc, o.sync), what
            if o.rc != tg.OK:
                assert nl == 0 and n == (-7 & gt.U64) and np.all(out == np.uint64(SENTINEL)), what
                continue
            assert nl == o.launches, what
        assert n == want.size == o.n, what
        if o.sync == tg.ERR_ARG:                  # a value flag found on the device: nothing written
            assert np.all(out == np.uint64(SENTINEL)), what
            continue
        assert np.array_equal(out[:n], want), what
        assert np.all(out[n:] == np.uint64(SENTINEL)), what


@pytest.mark.parametrize("name, k", TG, ids=[f"{n}-{k}" if k is not None else n for n, k in TG])
def test_trigram_edges(lib, lane, name, k):
    for j in ([k] if k is not None else range(len(FIXTURES[name].cases))):
        tg_check(lib, lane, name, j)


# ---- math() -----------------------------------------------------------------------------------------------------------

def _b(x, dt=np.uint64):
    x = np.ascontiguousarray(x, dt)
    return x if x.size else np.zeros(1, dt)


def _up(x, dt=np.uint64):
    import torch

    return torch.from_numpy(_b(x, dt).view(np.int64 if dt == np.uint64 else np.uint8).copy()).cuda()


def _h(t):
    a = t.cpu().numpy()
    return a.view(np.uint64) if a.dtype == np.int64 else a


def _prepared(case):
    from dgraph_b200 import algo

    names = {}
    nodes = algo.math_program(case.tree, names)
    leaves = [None] * len(names)
    for nm, j in names.items():
        leaves[j] = algo.math_leaf_arrays(case.maps.get(nm))
    return nodes, leaves, names


def mt_host(lib, case, cap):
    from dgraph_b200 import _lib

    nodes, leaves, _ = _prepared(case)
    lv = (_lib.MathLeaf * max(len(leaves), 1))()
    for j, (k, w, t, typ, nil) in enumerate(leaves):
        lv[j] = _lib.MathLeaf(k.ctypes.data, w.ctypes.data, None if t is None else t.ctypes.data, None,
                              0 if nil else k.size, typ, nil)
    r = None if case.range is None else _b(case.range)
    ok, ow = np.full(cap + GUARD, SENT, np.uint64), np.full(cap + GUARD, SENT, np.uint64)
    ot = np.full(cap + GUARD, 0xAB, np.uint8)
    info = C.c_uint64(SENT)
    prog = (_lib.MathNode * len(nodes))(*nodes)
    rc = lib.dgx_math_eval(prog, len(nodes), lv, len(leaves), None if r is None else r.ctypes.data,
                           0 if case.range is None else len(case.range), ok.ctypes.data, ow.ctypes.data,
                           ot.ctypes.data, cap, C.byref(info))
    return rc, None, info.value, ok, ow, ot, None


def mt_dev(lib, lane, case, call, cap):
    """Every leaf in a room of the model's size (spare entries hold 5), its count in a device word."""
    import torch

    from dgraph_b200 import _lib

    nodes, leaves, names = _prepared(case)
    rooms = {nm: room for nm, _, room in tg.mt_room(case, call)}
    keep = []
    lv = (_lib.MathLeaf * max(len(leaves), 1))()
    for nm, j in names.items():
        k, w, t, typ, nil = leaves[j]
        n = 0 if nil else k.size
        room = rooms[nm]
        pad = lambda a, dt: np.concatenate([np.asarray(a[:n], dt), np.full(room - n, 5, dt)])  # noqa: E731
        dk, dw = _up(pad(k, np.uint64)), _up(pad(w, np.uint64))
        dt_ = None if t is None else _up(pad(t, np.uint8), np.uint8)
        dn = _up(np.array([n], np.uint64))
        keep += [dk, dw, dt_, dn]
        lv[j] = _lib.MathLeaf(dk.data_ptr(), dw.data_ptr(), None if dt_ is None else dt_.data_ptr(),
                              None if nil else dn.data_ptr(), 0 if nil else room, typ, nil)
    dr = None if case.range is None else _up(case.range)
    ok = torch.full((cap + GUARD,), SENT - (1 << 64), dtype=torch.int64, device="cuda")
    ow = ok.clone()
    ot = torch.full((cap + GUARD,), 0xAB, dtype=torch.uint8, device="cuda")
    di = torch.full((1,), SENT - (1 << 64), dtype=torch.int64, device="cuda")
    prog = (_lib.MathNode * len(nodes))(*nodes)
    torch.cuda.synchronize()
    l0 = lib.dgx_lane_launches(lane)
    rc = lib.dgx_dev_math_eval(lane, prog, len(nodes), lv, len(leaves), None if dr is None else dr.data_ptr(),
                               0 if case.range is None else len(case.range), ok.data_ptr(), ow.data_ptr(),
                               ot.data_ptr(), cap, di.data_ptr())
    nl = lib.dgx_lane_launches(lane) - l0
    src = lib.dgx_lane_sync(lane)
    return rc, src, int(_h(di)[0]), _h(ok), _h(ow), _h(ot), nl


@pytest.mark.parametrize("name, k", MT, ids=[f"{n}-{k}" for n, k in MT])
def test_math_edges(lib, lane, name, k):
    f = FIXTURES[name]
    case, outs = f.cases[k], model(name)[k]
    w = tg.mt_expected(case)
    for call, o in zip(f.calls, outs):
        what = (name, k, call)
        cap = call.out_cap if call.out_cap is not None else \
            max(sum(r[1] for r in tg.mt_room(case, call)) + 1, len(case.range) if case.range is not None else 1)
        if call.form == "host":
            rc, src, info, ok, ow, ot, nl = mt_host(lib, case, cap)
        else:
            rc, src, info, ok, ow, ot, nl = mt_dev(lib, lane, case, call, cap)
            assert nl == o.launches, what
        assert (rc, src) == (o.rc, o.sync), what
        assert info == (SENT if o.info is None else o.info), what
        if o.keys is None:                       # refused or over capacity: the entries are untouched
            assert (ok == SENT).all() and (ow == SENT).all() and (ot == 0xAB).all(), what
            continue
        kind, keys, words, tags = w
        n = keys.size
        assert info & 0xFFFFFFFF == n and (info >> 32) & 0xFF == {"none": 0, "map": 1, "const": 2}[kind], what
        assert np.array_equal(ok[:n], keys) and np.array_equal(ow[:n], words) and np.array_equal(ot[:n], tags), what
        assert (ok[n:] == SENT).all() and (ow[n:] == SENT).all() and (ot[n:] == 0xAB).all(), what
