"""The UidPack readers at the edges of their block walk (fixtures and host model: tests/pack_geometry.py), bit-exact
against the oracle: windows of exactly D_WB bytes and one byte past it from a win0 misaligned by 0 and 15, runs cut at
lanes 1 and 31, partial batches, packs of 1 to 129 blocks in one job table, blocks of 0 to 65 groups, the slow path
at lanes 0 and 31, hand-built blocks (no delta bytes, deltas of 0xFFFFFFFF past 2^32, trailing bytes past the
window), the seeks of decode, the range choice, `after` and the slices of IntersectCompressedWith, the units of the
matrix form, and the seek block, the First cut and the mutable entries of unfiltered List.Uids.

Every fixture runs through its reader's host form with anonymous packs, with named packs (the second call hits the
cache) and, for the row forms, with flat pack images with and without a 16-byte gap; then through the device form on
a lane, whose launch count is checked against the model, and once more with out_cap one value short (DGX_ERR_CAP,
nothing written at or past out_cap).  The decode fixtures also run through the zero-copy route in one subprocess.
Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import functools
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import pack_geometry as pg  # noqa: E402
from test_gpu_parity import eq, pack_images  # noqa: E402
from test_pack_geometry import oracle_result  # noqa: E402

pytestmark = pytest.mark.gpu

ERR_CAP = -4
FILL = -0x2152411035014FF3  # 0xDEADBEEFCAFEB00D as int64
FILL_U = FILL & ((1 << 64) - 1)

FIXTURES = {f.name: f for f in pg.all_fixtures()}
NAMES = list(FIXTURES)
DEVICE = [n for n in NAMES if FIXTURES[n].kind != "batch"]


@pytest.fixture(scope="module")
def dgx():
    import dgraph_b200
    from dgraph_b200 import _lib

    lib = _lib.load()
    _lib.check(lib.dgx_init(-1))
    _lib.check(lib.dgx_cache_configure(1 << 30))
    return dgraph_b200


@functools.lru_cache(maxsize=None)
def want(name):
    from oracle import pyoracle

    return oracle_result(pyoracle, FIXTURES[name])


@functools.lru_cache(maxsize=None)
def plan(name):
    return pg.simulate(FIXTURES[name])


def upk(dgx, pk):
    """The model's pack as a dgraph_b200 UidPack over the same arrays (None for a NULL pack)."""
    return None if pk is None else dgx.pb.UidPack(*pk.arrays())


def keys_of(name, n):
    k = zlib.crc32(name.encode())
    return [(k, 100 + i) for i in range(n)]


def _u(x):
    return np.ascontiguousarray(np.asarray(x, dtype=np.uint64))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _launched(fn):
    from dgraph_b200 import _lib

    k0 = _lib.stats()["kernel_launches"]
    res = fn()
    return res, _lib.stats()["kernel_launches"] - k0


def _rows(out, off):
    return [out[int(off[i]):int(off[i + 1])] for i in range(len(off) - 1)]


# ---- host forms -------------------------------------------------------------------------------------------------------

def _host_runs(dgx, f, name):
    """(route, result) of every host route of the fixture; the result has the shape of oracle_result."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    a = f.args
    if f.kind == "decode":
        pk, seek, _ = a
        got, n = _launched(lambda: dgx.codec.Decode(upk(dgx, pk), seek))
        assert n == plan(name).launches, (n, plan(name).launches)
        yield "Decode", got
        return
    if f.kind == "batch":
        packs = [upk(dgx, p) for p in a[0]]
        merged = dgx.algo.MergeSortedPacked(packs)
        yield "MergeSortedPacked", [dgx.codec.Decode(merged, 0)]
        return
    if f.kind == "icw":
        pk, after, v = a
        o = dgx.pb.List(None)
        _, n = _launched(lambda: dgx.algo.IntersectCompressedWith(upk(dgx, pk), after, dgx.pb.List(_u(v)), o))
        assert n == plan(name).launches, (n, plan(name).launches)
        yield "IntersectCompressedWith", o.Uids
        for k in range(2):
            out, off = dgx.algo.IntersectCompressedWithRows([upk(dgx, pk)], after, _u(v), keys_of(name, 1))
            yield f"rows, named pack, call {k}", out
        return
    if f.kind == "rows":
        packs, after, v = a
        up = [upk(dgx, p) for p in packs]
        out, off = dgx.algo.IntersectCompressedWithRows(up, after, _u(v))
        yield "rows", _rows(out, off)
        for k in range(2):
            out, off = dgx.algo.IntersectCompressedWithRows(up, after, _u(v), keys_of(name, len(packs)))
            yield f"rows, named packs, call {k}", _rows(out, off)
        vv = _u(v)
        cap = sum(min(vv.size, dgx.codec.ExactLen(p)) for p in up if p is not None)
        for gaps in ((), tuple(range(len(packs)))):
            with pack_images(up, gaps) as refs:
                out = np.empty(max(cap, 1), np.uint64)
                off = np.zeros(len(packs) + 1, np.uint64)
                _lib.check(lib.dgx_intersect_compressed_rows(refs, len(packs), after, _p(vv), vv.size, _p(out),
                                                             _p(off), cap))
                yield f"rows, images, gaps {bool(gaps)}", _rows(out, off)
        return
    if f.kind == "mx":
        pk, rows = a
        rows = [_u(r) for r in rows]
        out, off = dgx.algo.IntersectCompressedWithMatrix(upk(dgx, pk), rows)
        yield "matrix", _rows(out, off)
        for k in range(2):
            out, off = dgx.algo.IntersectCompressedWithMatrix(upk(dgx, pk), rows, keys_of(name, 1)[0])
            yield f"matrix, named pack, call {k}", _rows(out, off)
        return
    rows, after, first = a
    up = [upk(dgx, p) for p, _, _ in rows]
    muts = [(mu, mf) for _, mu, mf in rows]
    out, off = dgx.algo.ListUidsUnfilteredRows(up, muts, after, first)
    counts = dgx.algo.ListCountRows(up, muts, after)
    yield "unfiltered rows and counts", list(zip(_rows(out, off), counts.tolist()))
    for k in range(2):
        out, off = dgx.algo.ListUidsUnfilteredRows(up, muts, after, first, keys_of(name, len(rows)))
        yield f"unfiltered rows, named packs, call {k}", list(zip(_rows(out, off), counts.tolist()))
    mu, mf, mut_off = dgx.algo._mut_csr(muts)
    cap = sum(len(w) for w, _ in want(name))
    for gaps in ((), tuple(range(len(rows)))):
        with pack_images(up, gaps) as refs:
            out = np.empty(max(cap, 1), np.uint64)
            off = np.zeros(len(rows) + 1, np.uint64)
            _lib.check(lib.dgx_list_uids_unfiltered_rows(refs, len(rows), _p(mu), _p(mf), _p(mut_off), after, first,
                                                         _p(out), _p(off), cap))
            yield f"unfiltered rows, images, gaps {bool(gaps)}", list(zip(_rows(out, off), counts.tolist()))


def _check(f, got, w, what):
    if f.kind in ("decode", "icw"):
        eq(got, w, what)
    elif f.kind == "batch":
        eq(got[0], np.unique(np.concatenate([x for x in w if x.size] or [np.zeros(0, np.uint64)])), what)
    elif f.kind == "luu":
        assert len(got) == len(w)
        for i, ((g, gc), (ww, wc)) in enumerate(zip(got, w)):
            eq(g, ww, f"{what}: row {i}")
            assert gc == wc, f"{what}: row {i}: count {gc}, want {wc}"
    else:
        assert len(got) == len(w)
        for i, (g, ww) in enumerate(zip(got, w)):
            eq(g, ww, f"{what}: row {i}")


@pytest.mark.parametrize("name", NAMES)
def test_host_forms(dgx, name):
    f, w = FIXTURES[name], want(name)
    for route, got in _host_runs(dgx, f, name):
        _check(f, got, w, f"{name}: {route}")


# ---- the device form --------------------------------------------------------------------------------------------------

class Lane:
    def __init__(self):
        import torch

        from dgraph_b200 import _lib

        self.lib = _lib.load()
        self.stream = torch.cuda.Stream()
        self.h = self.lib.dgx_lane_create(0, C.c_void_p(self.stream.cuda_stream))
        assert self.h
        self.handles = {}

    def pack(self, dgx, pk):
        """The pack uploaded once per lane (dgx_dev_pack_upload); None for a NULL pack."""
        from dgraph_b200 import _lib

        if pk is None:
            return None
        if id(pk) not in self.handles:
            p = upk(dgx, pk).normalized()
            view = dgx.codec.view_of(p)
            h = C.c_void_p()
            _lib.check(self.lib.dgx_dev_pack_upload(self.h, C.byref(view), C.byref(h)))
            self.handles[id(pk)] = (h, p, pk)
        return self.handles[id(pk)][0]

    def close(self):
        for h, _, _ in self.handles.values():
            self.lib.dgx_dev_pack_free(h)
        self.lib.dgx_lane_destroy(self.h)


@pytest.fixture(scope="module")
def lane(dgx):
    ln = Lane()
    yield ln
    ln.close()


def _dev(t):
    import torch

    return torch.from_numpy(np.ascontiguousarray(t).view(np.int64) if t.dtype == np.uint64 else t).cuda()


def dev_call(dgx, lane, name, cap):
    """The fixture's device form with out_cap = cap.  Returns (rc, out words from the output's start, offsets or
    length, counts or None, launches)."""
    import torch

    f = FIXTURES[name]
    lib = lane.lib
    buf = torch.full((cap + 72,), FILL, dtype=torch.int64, device="cuda")
    assert buf.data_ptr() % 256 == 0
    word = f.args[2] if f.kind == "decode" else 0
    d_out = buf.data_ptr() + 8 * word
    keep = []
    if f.kind == "decode":
        pk, seek, _ = f.args
        meta = torch.full((2,), 7, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        l0 = lib.dgx_lane_launches(lane.h)
        rc = lib.dgx_dev_decode(lane.h, lane.pack(dgx, pk), seek, C.c_void_p(d_out), cap, C.c_void_p(meta.data_ptr()))
        res = (meta, None)
    elif f.kind in ("icw", "rows"):
        packs, after, v = ([f.args[0]], f.args[1], f.args[2]) if f.kind == "icw" else f.args
        tab = (C.c_void_p * len(packs))(*[lane.pack(dgx, p) for p in packs])
        vv = _u(v)
        d_v = _dev(vv if vv.size else np.zeros(1, np.uint64))
        off = torch.full((len(packs) + 1,), 7, dtype=torch.int64, device="cuda")
        keep += [d_v]
        torch.cuda.synchronize()
        l0 = lib.dgx_lane_launches(lane.h)
        rc = lib.dgx_dev_intersect_compressed_rows(lane.h, tab, len(packs), after, C.c_void_p(d_v.data_ptr()), vv.size,
                                                   C.c_void_p(d_out), cap, C.c_void_p(off.data_ptr()))
        res = (off, None)
    elif f.kind == "mx":
        pk, rows = f.args
        v_off = np.zeros(len(rows) + 1, np.uint64)
        np.cumsum([len(r) for r in rows], out=v_off[1:])
        v = np.concatenate([_u(r) for r in rows] + [np.zeros(1, np.uint64)])
        d_v = _dev(v)
        off = torch.full((len(rows) + 1,), 7, dtype=torch.int64, device="cuda")
        keep += [d_v, v_off]
        torch.cuda.synchronize()
        l0 = lib.dgx_lane_launches(lane.h)
        rc = lib.dgx_dev_intersect_compressed_matrix(lane.h, lane.pack(dgx, pk), C.c_void_p(d_v.data_ptr()), _p(v_off),
                                                     len(rows), C.c_void_p(d_out), cap, C.c_void_p(off.data_ptr()))
        res = (off, None)
    else:
        rows, after, first = f.args
        mu, mf, mut_off = dgx.algo._mut_csr([(m_, f_) for _, m_, f_ in rows])
        tab = (C.c_void_p * len(rows))(*[lane.pack(dgx, p) for p, _, _ in rows])
        d_mu, d_mf = _dev(mu), _dev(mf)
        off = torch.full((len(rows) + 1,), 7, dtype=torch.int64, device="cuda")
        cnt = torch.full((len(rows),), 9, dtype=torch.int32, device="cuda")
        keep += [d_mu, d_mf, mut_off]
        torch.cuda.synchronize()
        l0 = lib.dgx_lane_launches(lane.h)
        rc = lib.dgx_dev_list_uids_unfiltered_rows(lane.h, tab, len(rows), C.c_void_p(d_mu.data_ptr()),
                                                   C.c_void_p(d_mf.data_ptr()), _p(mut_off), after, first,
                                                   C.c_void_p(d_out), cap, C.c_void_p(off.data_ptr()))
        l1 = lib.dgx_lane_launches(lane.h)
        if rc == 0:
            rc = lib.dgx_dev_list_count_rows(lane.h, tab, len(rows), C.c_void_p(d_mu.data_ptr()),
                                             C.c_void_p(d_mf.data_ptr()), _p(mut_off), after,
                                             C.c_void_p(cnt.data_ptr()))
        res = (off, cnt)
        launches = (l1 - l0, lib.dgx_lane_launches(lane.h) - l1)
    if f.kind != "luu":
        launches = lib.dgx_lane_launches(lane.h) - l0
    sync = lib.dgx_lane_sync(lane.h) if rc == 0 else rc
    out = buf.cpu().numpy().view(np.uint64)[word:]
    return sync, out, res[0].cpu().numpy().view(np.uint64), (None if res[1] is None else res[1].cpu().numpy()), launches


def _total(f, w):
    if f.kind in ("decode", "icw"):
        return len(w)
    if f.kind == "luu":
        return sum(len(x) for x, _ in w)
    return sum(len(x) for x in w)


def _model_launches(f, r):
    if f.kind == "icw":  # the device form of one pack is the rows form
        return 6 if len(f.args[2]) and f.args[0].nb else 0
    if f.kind == "luu":
        return (r.launches, r.count_launches)
    return r.launches


@pytest.mark.parametrize("name", DEVICE)
def test_device_form(dgx, lane, name):
    f, w, r = FIXTURES[name], want(name), plan(name)
    total = _total(f, w)
    sync, out, off, cnt, launches = dev_call(dgx, lane, name, total)
    assert sync == 0, f"{name}: lane sync {sync}"
    assert launches == _model_launches(f, r), f"{name}: {launches} launches, the model plans {_model_launches(f, r)}"
    if f.kind == "decode":
        assert int(off[0]) == total, (int(off[0]), total)
        eq(out[:total], w, name)
    elif f.kind == "icw":
        assert off.tolist() == [0, total]
        eq(out[:total], w, name)
    else:
        rows = w if f.kind != "luu" else [x for x, _ in w]
        eq(off, np.concatenate([[0], np.cumsum([len(x) for x in rows])]), f"{name}: out_off")
        for i, x in enumerate(rows):
            eq(out[int(off[i]):int(off[i + 1])], x, f"{name}: row {i}")
        if f.kind == "luu":
            assert cnt.tolist() == [c for _, c in w], f"{name}: counts"
    assert (out[total:total + 64] == FILL_U).all(), f"{name}: written past the result"


@pytest.mark.parametrize("name", DEVICE)
def test_out_cap_one_short(dgx, lane, name):
    """out_cap one value short of the result: DGX_ERR_CAP at the sync and nothing written at or past out_cap."""
    f, w = FIXTURES[name], want(name)
    total = _total(f, w)
    if total == 0:
        pytest.skip("empty result")
    sync, out, _, _, _ = dev_call(dgx, lane, name, total - 1)
    assert sync == ERR_CAP, f"{name}: sync {sync}"
    assert (out[total - 1:total + 63] == FILL_U).all(), f"{name}: a value was written at or past out_cap"


def test_decode_zero_copy():
    """The decode fixtures through DGX_ZERO_COPY=1 (pinned pack images decoded in place by decode_batch_kernel), in
    one subprocess because libdgx reads its knobs once: IntersectSorted of a pack with itself is the pack decoded."""
    code = r'''
import os, sys
import numpy as np
sys.path.insert(0, os.getcwd()); sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
import ctypes as C
import dgraph_b200
from dgraph_b200 import _lib
import pack_geometry as pg
from test_gpu_parity import eq, pack_images
from test_gpu_round2 import sorted_packed
_lib.check(_lib.load().dgx_init(-1))
n = 0
for f in pg.all_fixtures():
    if f.kind != "decode" or f.args[1] != 0:
        continue
    pk = f.args[0]
    p = dgraph_b200.pb.UidPack(*pk.arrays())
    with pack_images([p, p], (1,)) as refs:
        got, _ = sorted_packed(refs, 2, len(pk.flat))
    eq(got, np.asarray(pk.flat, np.uint64), f.name)
    n += 1
assert n >= 5, n
print("ZERO_COPY_OK")
'''
    env = dict(os.environ, DGX_ZERO_COPY="1")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, env=env,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert "ZERO_COPY_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]
