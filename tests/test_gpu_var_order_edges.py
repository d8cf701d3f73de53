"""The edge fixtures of tests/var_order_geometry.py through dgx_var_order and dgx_dev_var_order on the device: tier
edges (rows of 12 and 13, +-0.0, NaN forms, bools, mixed tags, under asc and desc), the thread / CTA split at 4 096 /
4 097 entries and 2*SMs - 1, 2*SMs and 2*SMs + 1 long rows for the device it runs on, the cooperative partition's
chunk edges and the pdqsort driver's helpers on CTA rows found by a seeded search, |W| and row-pass edges of the two
radix sorts, every PageRange branch, output slot and dest-mark edges, and every refusal in a CTA's last and next
CTA's first thread.  Each call is checked bit for bit against the line-by-line restatement (var_order_oracle.c, which
tests/test_var_order_geometry.py holds equal to the model), with guard words past every output, and its launches
against the plan model.  The device form runs with and without slack and length words.  Runs on an H100 only
(`pytest -m gpu`)."""
import ctypes as C
import functools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import var_order_geometry as vg  # noqa: E402
import var_order_oracle as vo  # noqa: E402
import var_order_plan as vp  # noqa: E402

pytestmark = pytest.mark.gpu

OK, ERR_ARG = 0, -3
SENT = 0xDEADBEEFCAFEF00D
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
def fixtures():
    """The fixtures built for this device's SM count: the 2*SMs fixtures follow it."""
    import torch

    return {f.name: f for f in vg.fixtures(torch.cuda.get_device_properties(0).multi_processor_count)}


def _names():
    return [f.name for f in vg.fixtures()]


@functools.lru_cache(maxsize=None)
def want(name):
    f = fixtures()[name]
    return None if f.mutate is not None else vo.var_order(*f.case)


def _t(a, dtype=np.uint64):
    import torch

    a = np.ascontiguousarray(np.asarray(a, dtype))
    if a.size == 0:
        a = np.zeros(1, dtype)
    return torch.from_numpy(a.view(np.int64) if dtype == np.uint64 else a).cuda()


def _h(t, n):
    return t.cpu().numpy()[:n].view(np.uint64).copy()


def sent(n):
    import torch

    return torch.full((max(n, 1),), SENT - (1 << 64), dtype=torch.int64, device="cuda")


def same(rows, dest, exp):
    return (len(rows) == len(exp[0]) and all(np.array_equal(a, b) for a, b in zip(rows, exp[0]))
            and np.array_equal(dest, exp[1]))


def host_call(lib, f):
    """dgx_var_order over the fixture's (possibly broken) inputs, with guard words past every output."""
    from dgraph_b200 import _lib
    from dgraph_b200.algo import var_order_leaf

    a = vg.arrays(f.case, vg.HOST, f.mutate)
    keep, leaf = var_order_leaf(a["map"])
    d, v, v_off = a["dest"], a["v"], a["v_off"]
    nrows, M = v_off.size - 1, int(v_off[-1])
    out = np.full(M + GUARD, SENT, np.uint64)
    oo = np.full(nrows + 1 + GUARD, SENT, np.uint64)
    dout = np.full(d.size + GUARD, SENT, np.uint64)
    n = C.c_size_t(SENT)
    l0 = _lib.stats()["kernel_launches"]
    rc = lib.dgx_var_order(C.byref(leaf), int(f.case[1]), (d if d.size else np.zeros(1, np.uint64)).ctypes.data,
                           d.size, (v if v.size else np.zeros(1, np.uint64)).ctypes.data, v_off.ctypes.data, nrows,
                           f.case[4], f.case[5], out.ctypes.data, oo.ctypes.data, M, dout.ctypes.data, d.size,
                           C.byref(n))
    nl = _lib.stats()["kernel_launches"] - l0
    del keep
    guards = np.all(out[M:] == SENT) and np.all(oo[nrows + 1:] == SENT) and np.all(dout[d.size:] == SENT)
    if rc != OK:
        return rc, None, guards and np.all(out == SENT) and np.all(dout == SENT), nl
    K = int(oo[nrows])
    guards = guards and np.all(out[K:] == SENT) and np.all(dout[n.value:] == SENT)
    return rc, ([out[int(oo[i]):int(oo[i + 1])].copy() for i in range(nrows)], dout[:n.value].copy()), guards, nl


def dev_call(lib, lane, f, call):
    """dgx_dev_var_order over vg.arrays' device layout: slack past dest, the values and the map, their lengths from
    words with garbage above bit 32 when call.words.  Returns (rc, sync rc, dest length word, (rows, dest) or None,
    launches, guards intact)."""
    from dgraph_b200 import _lib

    a = vg.arrays(f.case, call, f.mutate)
    dest, v, v_off = a["dest"], a["v"], a["v_off"]
    nrows, ndest, vcap = v_off.size - 1, dest.size, v.size
    keep = [_t(a["key"]), _t(a["word"])]
    tag_p = None
    if a["tag"] is not None:
        keep.append(_t(a["tag"], np.uint8))
        tag_p = keep[-1].data_ptr()
    mlen = None
    if a["mlen"] is not None:
        keep.append(_t(np.array([a["mlen"]], np.uint64)))
        mlen = keep[-1].data_ptr()
    leaf = _lib.MathLeaf(keep[0].data_ptr(), keep[1].data_ptr(), tag_p, mlen, a["key"].size, a["mtype"] or vg.T_INT,
                         0)
    dd, vv, oo_in = _t(dest), _t(v), _t(v_off)
    dw = _t(np.array([a["dlen"]], np.uint64)) if a["dlen"] is not None else None
    out, oo, dout, dlen = sent(vcap + GUARD), sent(nrows + 1 + GUARD), sent(ndest + GUARD), sent(1)
    l0 = lib.dgx_lane_launches(lane)
    rc = lib.dgx_dev_var_order(lane, C.byref(leaf), int(f.case[1]), dd.data_ptr(), ndest,
                               dw.data_ptr() if dw is not None else None, vv.data_ptr(), oo_in.data_ptr(), nrows, vcap,
                               f.case[4], f.case[5], out.data_ptr(), oo.data_ptr(), vcap, dout.data_ptr(), ndest,
                               dlen.data_ptr())
    src = lib.dgx_lane_sync(lane) if rc == OK else None
    nl = lib.dgx_lane_launches(lane) - l0
    o, off, de, L = _h(out, vcap + GUARD), _h(oo, nrows + 1 + GUARD), _h(dout, ndest + GUARD), int(_h(dlen, 1)[0])
    del keep
    guards = np.all(o[vcap:] == SENT) and np.all(off[nrows + 1:] == SENT) and np.all(de[ndest:] == SENT)
    if rc != OK or src != OK:
        guards = guards and np.all(o == SENT) and np.all(off == SENT) and np.all(de == SENT)
        return rc, src, L, None, nl, guards
    K = int(off[nrows])
    guards = guards and np.all(o[K:] == SENT) and np.all(de[L:] == SENT)
    return rc, src, L, ([o[int(off[i]):int(off[i + 1])].copy() for i in range(nrows)], de[:L].copy()), nl, guards


@pytest.mark.parametrize("name", _names())
def test_fixture(lib, lane, name):
    f = fixtures()[name]
    exp = want(name)
    nrows = len(f.case[3])
    for call in f.calls:
        if call.form == "host":
            rc, got, guards, nl = host_call(lib, f)
            assert guards, (name, call)
            if exp is None:
                assert rc == ERR_ARG, (name, call)
                continue
            assert rc == OK and same(*got, exp), (name, call)
            assert nl == vp.launches(len(f.case[2]), nrows), (name, call)
            continue
        rc, src, L, got, nl, guards = dev_call(lib, lane, f, call)
        assert rc == OK and guards, (name, call)
        if exp is None:
            assert src == ERR_ARG and L == 0, (name, call)
            continue
        assert src == OK and L == exp[1].size and same(*got, exp), (name, call)
        room = len(f.case[2]) + (call.slack if call.words else 0)
        assert nl == vp.launches(room, nrows), (name, call)
