"""The edge fixtures of tests/value_column_geometry.py through match(), the regexp() value test and the compare
functions on the device, both library forms: dgx_match / dgx_dev_match, dgx_regex_match / dgx_dev_regex_match,
dgx_compare_uids / dgx_dev_compare_uids and dgx_compare_rows / dgx_dev_compare_rows.  The fixtures include lane-form
string columns whose bytes start at offset 1 .. 15 of a segment, long-tier and warp-tier queues of 2*SMs*8 - 1,
2*SMs*8, 2*SMs*8 + 1 and 2 * 2*SMs*8 + 1 items and pair counts on both sides of 8*SMs*256 for the device it runs on,
DFAs of 16 383, 16 384 and 16 385 table entries, the warp tier's chunk edges, count words below the room and with
bits above 32, column refusals past the candidates, zero-count runs at the tile edges and the index path's slot
space.  Each call is checked bit for bit against the model (which tests/test_value_column_geometry.py holds equal to
the restatements), with guard words past the output, the counts and the row offsets, and its launches counted.
Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import functools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import value_column_geometry as vg  # noqa: E402

pytestmark = pytest.mark.gpu

OK, ERR_ARG = 0, -3
SENT = 0xDEADBEEFCAFEF00D
CSENT = 0xA5A5A5A5
GUARD = 4


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
def sms():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


@functools.lru_cache(maxsize=None)
def fixtures():
    """The fixtures built for this device's SM count: the stride fixtures follow it."""
    return {f.name: f for f in vg.fixtures(sms())}


def _names():
    return [f.name for f in vg.fixtures()]


@functools.lru_cache(maxsize=None)
def want(name, form):
    r, _, oob = vg.run(fixtures()[name], form, sms())
    assert r[0] != "fault" and not oob
    return r


def _t(a, dtype=np.uint64):
    import torch

    a = np.ascontiguousarray(np.asarray(a, dtype))
    if a.size == 0:
        a = np.zeros(1, dtype)
    if dtype == np.uint64:
        a = a.view(np.int64)
    elif dtype == np.uint32:
        a = a.view(np.int32)
    return torch.from_numpy(a.copy()).cuda()


def _h(t, dtype=np.uint64):
    return t.cpu().numpy().view(dtype).copy()


def _filled(n, v, dtype=np.uint64):
    return _t(np.full(max(n, 1), v, dtype), dtype)


class DevStr:
    """A resident string column, its bytes at offset `shift` of a 16-byte-aligned device buffer."""

    def __init__(self, col, shift):
        from dgraph_b200 import _lib

        nb = int(col.byte_off[-1])
        buf = np.full(nb + shift + 32, 0xEE, np.uint8)
        buf[shift:shift + nb] = col.bytes[:nb]
        self.t = [_t(col.uid), _t(col.val_off), _t(col.byte_off), _t(buf, np.uint8)]
        assert self.t[3].data_ptr() % 16 == 0
        self.s = _lib.StrColumn(self.t[0].data_ptr() if col.uid.size else None, self.t[1].data_ptr(),
                                self.t[2].data_ptr(), self.t[3].data_ptr() + shift, col.uid.size,
                                col.byte_off.size - 1, nb)


class DevVal:
    def __init__(self, col, shift):
        from dgraph_b200 import _lib

        self.keep = []

        def d(a, dtype=np.uint64):
            if a is None:
                return None
            t = _t(a, dtype)
            self.keep.append(t)
            return t.data_ptr()

        if col.type == vg.T_STR:
            self.str = DevStr(col.str, shift)
            self.s = _lib.ValColumn(col.type, None, None, None, None, d(col.bad, np.uint8), C.pointer(self.str.s), 0,
                                    0)
        else:
            self.s = _lib.ValColumn(col.type, d(col.uid) if col.uid.size else None, d(col.val_off), d(col.word),
                                    d(col.nsec, np.uint32), d(col.bad, np.uint8), None, col.uid.size,
                                    int(col.val_off[-1]))


def columns(case):
    """The fixture's algo column, with the broken arrays a lane-form fixture hands over."""
    from dgraph_b200 import algo

    typ = case.get("typ", vg.T_STR)
    if case["kind"] in ("match", "regex"):
        col = algo.StrColumn(case["uids"], case["values"])
        for k, v in case.get("broken", {}).items():
            setattr(col, k, np.asarray(v, np.uint64))
        return col
    return algo.ValColumn(typ, case["uids"], case["values"], case.get("bad"))


def host_call(lib, f, op=None, args=None):
    """The host form: (rc, result in the model's shape, launches)."""
    from dgraph_b200 import _lib, algo

    case = f.case
    col = columns(case)
    l0 = _lib.stats()["kernel_launches"]
    try:
        if case["kind"] == "match":
            r = ("ok", [int(x) for x in algo.MatchFuzzy(col, case["query"], case["max"], uids=case["cands"]).Uids],
                 None)
        elif case["kind"] == "regex":
            prog = algo.RegexProg(case["pattern"], case.get("fold", False))
            r = ("ok", [int(x) for x in algo.MatchRegex(col, prog, uids=case["cands"]).Uids], None)
        elif case["kind"] == "cmp":
            got, cnt = algo.CompareUids(col, op, algo.ValArgs(col.type, args), case["cands"], counts=True)
            r = ("ok", [int(x) for x in got.Uids], tuple(int(c) for c in cnt))
        else:
            rows = algo.CompareRows(col, op, algo.ValArgs(col.type, args), case["rows"], case["row_arg"])
            off = [0]
            for x in rows:
                off.append(off[-1] + len(x))
            r = ("ok", tuple(off), tuple(int(x) for x in np.concatenate(rows + [np.zeros(0, np.uint64)])))
        rc = OK
    except _lib.DgxError as e:
        rc, r = e.code, None
    return rc, r, _lib.stats()["kernel_launches"] - l0


def lane_uids(lib, lane, f, op=None, args=None):
    """The lane form over a UidList with its count word: (rc, sync rc, result or None, guards intact, launches)."""
    import torch

    from dgraph_b200 import algo

    case = f.case
    col = columns(case)
    shift = case.get("shift", 0)
    cands = np.asarray(case["cands"], np.uint64)
    ccap = cands.size
    du = _t(np.concatenate([cands, np.full(GUARD, SENT, np.uint64)]))
    out, olen = _filled(ccap + GUARD, SENT), _filled(1, SENT)
    cnt = _filled(ccap + GUARD, CSENT, np.uint32)
    dn = _t([case["word"]]) if case.get("word") is not None else None
    dnp = dn.data_ptr() if dn is not None else None
    dc = DevVal(col, shift) if case["kind"] == "cmp" else DevStr(col, shift)
    torch.cuda.synchronize()
    l0 = lib.dgx_lane_launches(lane)
    rc = OK
    try:
        if case["kind"] == "match":
            algo.dev_match(lane, dc.s, case["query"], case["max"], out.data_ptr(), ccap, olen.data_ptr(),
                           d_uids=du.data_ptr(), nuids=ccap, d_nuids=dnp)
        elif case["kind"] == "regex":
            prog = algo.RegexProg(case["pattern"], case.get("fold", False))
            algo.dev_match_regex(lane, dc.s, prog, out.data_ptr(), ccap, olen.data_ptr(), d_uids=du.data_ptr(),
                                 nuids=ccap, d_nuids=dnp)
        else:
            algo.dev_compare_uids(lane, dc.s, op, algo.ValArgs(col.type, args), du.data_ptr(), ccap, out.data_ptr(),
                                  ccap, olen.data_ptr(), d_nuids=dnp, d_counts=cnt.data_ptr())
    except Exception as e:  # noqa: BLE001
        rc = e.code
    nl = lib.dgx_lane_launches(lane) - l0
    src = lib.dgx_lane_sync(lane) if rc == OK else None
    torch.cuda.synchronize()
    o, n, c = _h(out), int(_h(olen)[0]), _h(cnt, np.uint32)
    msg = lib.dgx_last_error() if src not in (None, OK) else b""
    if src != OK:
        return rc, src, None, np.all(o == SENT) and np.all(c == CSENT) and n == 0, nl, msg
    guards = np.all(o[n:] == SENT) and np.all(c[ccap:] == CSENT)
    counts = None
    if case["kind"] == "cmp":
        counts = tuple(None if int(x) == CSENT else int(x) for x in c[:ccap])
    return rc, src, ("ok", [int(x) for x in o[:n]], counts), guards, nl, msg


def lane_rows(lib, lane, f, op, args):
    import torch

    from dgraph_b200 import algo

    case = f.case
    col = columns(case)
    rows = case["rows"]
    off = np.zeros(len(rows) + 1, np.uint64)
    np.cumsum([len(r) for r in rows], out=off[1:])
    M = int(off[-1])
    v_cap = case.get("v_cap") if case.get("v_cap") is not None else M
    v = np.concatenate([np.asarray(r, np.uint64) for r in rows] + [np.zeros(0, np.uint64)])
    v = np.concatenate([v, np.full(max(v_cap - v.size, 0), 7, np.uint64), np.full(GUARD, SENT, np.uint64)])
    dv, doff = _t(v), _t(off)
    out, oo = _filled(v_cap + GUARD, SENT), _filled(len(rows) + 1 + GUARD, SENT)
    dc = DevVal(col, case.get("shift", 0))
    torch.cuda.synchronize()
    l0 = lib.dgx_lane_launches(lane)
    algo.dev_compare_rows(lane, dc.s, op, algo.ValArgs(col.type, args), dv.data_ptr(), doff.data_ptr(), len(rows),
                          v_cap, case["row_arg"], out.data_ptr(), oo.data_ptr(), v_cap)
    nl = lib.dgx_lane_launches(lane) - l0
    src = lib.dgx_lane_sync(lane)
    torch.cuda.synchronize()
    o, fo = _h(out), _h(oo)
    nr = len(rows)
    guards = np.all(fo[nr + 1:] == SENT)
    if src != OK:
        return src, None, guards and np.all(fo[:nr + 1] == 0) and np.all(o == SENT), nl
    K = int(fo[nr])
    guards = guards and np.all(o[K:] == SENT)
    return src, ("ok", tuple(int(x) for x in fo[:nr + 1]), tuple(int(x) for x in o[:K])), guards, nl


def _calls(case):
    return case["calls"] if case["kind"] in ("cmp", "rows") else [(None, None)]


@pytest.mark.parametrize("name", _names())
def test_fixture(lib, lane, name):
    f = fixtures()[name]
    kind = f.case["kind"]
    for form in vg.forms(f.case):
        exp = want(name, form)
        for (op, args), e in zip(_calls(f.case), exp):
            if form == "host":
                rc, got, nl = host_call(lib, f, op, args)
                if e[0] == "refused":
                    assert rc == ERR_ARG, (name, form, op)
                    continue
                assert rc == OK and got == e, (name, form, op)
                assert nl == vg.LAUNCHES[kind], (name, form, op, nl)
                continue
            if kind == "rows":
                src, got, guards, nl = lane_rows(lib, lane, f, op, args)
                assert guards, (name, form, op)
                assert nl == vg.LAUNCHES[kind], (name, form, op, nl)
                if e[0] == "refused":
                    assert src == ERR_ARG, (name, form, op)
                    continue
                assert src == OK and got == e, (name, form, op)
                continue
            rc, src, got, guards, nl, msg = lane_uids(lib, lane, f, op, args)
            assert rc == OK and guards, (name, form, op)
            assert nl == vg.LAUNCHES[kind], (name, form, op, nl)
            if e[0] == "refused":
                assert src == ERR_ARG, (name, form, op)
                assert (b"compare function" if kind == "cmp" else b"match()") in msg, msg
                continue
            assert src == OK and got == e, (name, form, op)
