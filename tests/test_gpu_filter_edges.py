"""The filter pipeline at the edges of its tile, staging and deferral plan (fixtures and host model:
tests/filter_geometry.py), bit-exact against the oracle: warp-row and tile edges of both tile geometries, batches
mixing 1-, 2- and wide queries, the P_MAXL boundary, slices that fill the stage or overflow it by one word, every
branch of the 32-bit fast path's ladders and the window pivots, tiles around multiples of 2^32, repeated values
(ranks from the previous tile, past the staged slice, in Difference), and the sample's deferral threshold with the
tail kernel behind it.  Every fixture runs through the host forms and through dgx_dev_filter_batch on a lane
without and a lane with resident inputs (the only one that samples and defers), with its lists placed at the element
offsets it chose; launches and deferred queries are checked against the model.  Runs on an H100 only
(`pytest -m gpu`)."""
import ctypes as C
import functools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import filter_geometry as fg  # noqa: E402
from test_gpu_parity import L, eq  # noqa: E402

pytestmark = pytest.mark.gpu

ERR_CAP = -4
FILL = -0x2152411035014FF3  # 0xDEADBEEFCAFEB00D as int64

FIXTURES = {f.name: f for f in fg.all_fixtures()}


@pytest.fixture(scope="module")
def dgx():
    import dgraph_b200
    from dgraph_b200 import _lib

    _lib.check(_lib.load().dgx_init(-1))
    return dgraph_b200


@functools.lru_cache(maxsize=None)
def want(name):
    from oracle import pyoracle as orc

    f = FIXTURES[name]
    return [fg.oracle_result(orc, q, f.op) for q in f.queries]


# ---- host forms -------------------------------------------------------------------------------------------------------

def _launched(fn):
    from dgraph_b200 import _lib

    k0 = _lib.stats()["kernel_launches"]
    res = fn()
    return res, _lib.stats()["kernel_launches"] - k0


@pytest.mark.parametrize("name", list(FIXTURES))
def test_host_forms(dgx, name):
    """dgx_intersect_sorted / dgx_intersect2 / dgx_difference per query (lists in their own allocations), and
    dgx_intersect_batch when every query has two lists (pair i at a_off[i] / b_off[i] inside one upload)."""
    f, ws = FIXTURES[name], want(name)
    for qi, (q, w) in enumerate(zip(f.queries, ws)):
        what = f"{name}: query {qi} (k={len(q)}, |A|={min(l.size for l in q)})"
        plan = fg.plan_batch([q], f.op)
        if f.op == fg.OP_DIFFERENCE:
            got, n = _launched(lambda: dgx.algo.Difference(L(dgx, q[0]), L(dgx, q[1])).Uids)
        else:
            got, n = _launched(lambda: dgx.algo.IntersectSorted([L(dgx, l) for l in q]).Uids)
            if len(q) == 2:
                o = dgx.pb.List(None)
                dgx.algo.IntersectWith(L(dgx, q[0]), L(dgx, q[1]), o)
                eq(o.Uids, w, what + " IntersectWith")
        eq(got, w, what)
        assert n == plan.launches, f"{what}: {n} launches, the model plans {plan.launches}"
    if f.op == fg.OP_INTERSECT and all(len(q) == 2 for q in f.queries):
        a_off = np.concatenate([[0], np.cumsum([q[0].size for q in f.queries])]).astype(np.uint64)
        b_off = np.concatenate([[0], np.cumsum([q[1].size for q in f.queries])]).astype(np.uint64)
        a = np.concatenate([q[0] for q in f.queries])
        b = np.concatenate([q[1] for q in f.queries])
        plan = fg.plan_batch(f.queries, f.op)
        (out, out_off), n = _launched(lambda: dgx.algo.IntersectBatch(a, a_off, b, b_off))
        eq(out_off, np.concatenate([[0], np.cumsum([w.size for w in ws])]), f"{name}: IntersectBatch out_off")
        for i, w in enumerate(ws):
            eq(out[int(out_off[i]):int(out_off[i + 1])], w, f"{name}: IntersectBatch pair {i}")
        assert n == plan.launches, (n, plan.launches)


# ---- the device form --------------------------------------------------------------------------------------------------

class Lane:
    def __init__(self, resident):
        import torch

        from dgraph_b200 import _lib

        self.lib = _lib.load()
        self.stream = torch.cuda.Stream()
        self.h = self.lib.dgx_lane_create(0, C.c_void_p(self.stream.cuda_stream))
        assert self.h
        _lib.check(self.lib.dgx_lane_set_resident_inputs(self.h, 1 if resident else 0))

    def close(self):
        self.lib.dgx_lane_destroy(self.h)


@pytest.fixture(scope="module")
def lanes(dgx):
    ls = {False: Lane(False), True: Lane(True)}
    yield ls
    for lane in ls.values():
        lane.close()


class DevBatch:
    """The batch's lists back to back in one device buffer at the element offsets fg.device_offsets gives (each list
    at the parity its fixture chose; the buffer itself is 256-byte aligned).  tests/test_filter_geometry.py checks
    that the fixtures reach their events placed so."""

    def __init__(self, f):
        import torch

        self.offsets, size = fg.device_offsets(f.queries, f.offsets)
        buf = np.zeros(size + 2, np.uint64)
        offs = [p for row in self.offsets for p in row]
        flat = [l for q in f.queries for l in q]
        for p, l in zip(offs, flat):
            buf[p:p + l.size] = l
        self.buf = torch.from_numpy(buf.view(np.int64)).cuda()
        base = self.buf.data_ptr()
        assert base % 256 == 0
        self.ptrs = (C.c_void_p * len(flat))(*[base + 8 * p for p in offs])
        self.lens = (C.c_size_t * len(flat))(*[l.size for l in flat])
        koff = np.concatenate([[0], np.cumsum([len(q) for q in f.queries])])
        self.koff = (C.c_size_t * len(koff))(*[int(x) for x in koff])
        self.nq = len(f.queries)


def dev_filter(lane, f, d, cap):
    import torch

    out = torch.full((cap + 64,), FILL, dtype=torch.int64, device="cuda")
    off = torch.full((d.nq + 1,), 7, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    l0 = lane.lib.dgx_lane_launches(lane.h)
    rc = lane.lib.dgx_dev_filter_batch(lane.h, f.op, d.ptrs, d.lens, d.koff, d.nq, C.c_void_p(out.data_ptr()), cap,
                                       C.c_void_p(off.data_ptr()))
    return rc, out, off, lane.lib.dgx_lane_launches(lane.h) - l0


@pytest.mark.parametrize("resident", [False, True], ids=["streaming lane", "resident lane"])
@pytest.mark.parametrize("name", list(FIXTURES))
def test_device_form(dgx, lanes, name, resident):
    from dgraph_b200 import _lib

    f, ws = FIXTURES[name], want(name)
    lane = lanes[resident]
    d = DevBatch(f)
    plan = fg.plan_batch(f.queries, f.op, resident, d.offsets)
    total = sum(w.size for w in ws)
    _lib.check(lane.lib.dgx_lane_sync(lane.h))
    t0 = lane.lib.dgx_filter_tail_queries(lane.h)
    rc, out, off, launches = dev_filter(lane, f, d, total)
    _lib.check(rc)
    _lib.check(lane.lib.dgx_lane_sync(lane.h))
    tail = lane.lib.dgx_filter_tail_queries(lane.h) - t0
    ho, hoff = out.cpu().numpy(), off.cpu().numpy().view(np.uint64)
    eq(hoff, np.concatenate([[0], np.cumsum([w.size for w in ws])]), f"{name}: out_off")
    for qi, w in enumerate(ws):
        eq(ho[int(hoff[qi]):int(hoff[qi + 1])].view(np.uint64), w, f"{name}: query {qi} (k={len(f.queries[qi])})")
    assert (ho[total:] == FILL).all(), f"{name}: {int((ho[total:] != FILL).sum())} words written past the result"
    assert launches == plan.launches, f"{name}: {launches} launches, the model plans {plan.launches}"
    ndef = fg.deferring_queries(plan)
    assert tail == ndef, f"{name}: {tail} deferred queries, the model's sample defers {ndef}"
    if f.tail is not None and resident:
        assert tail == f.tail


OUT_CAP_CASES = [n for n, f in FIXTURES.items() if f.resident and len(f.queries) > 2] + [
    "2-list slices at slice_cap", "duplicates, k=3", "Difference with repeated values"]


@pytest.mark.parametrize("resident", [False, True], ids=["streaming lane", "resident lane"])
@pytest.mark.parametrize("name", OUT_CAP_CASES)
def test_out_cap_one_short(dgx, lanes, name, resident):
    """out_cap one value short of the result: DGX_ERR_CAP at the sync, nothing written at or past out_cap; the lane
    then serves the same batch with the exact capacity."""
    from dgraph_b200 import _lib

    f, ws = FIXTURES[name], want(name)
    lane = lanes[resident]
    d = DevBatch(f)
    total = sum(w.size for w in ws)
    assert total > 0
    _lib.check(lane.lib.dgx_lane_sync(lane.h))
    rc, out, off, _ = dev_filter(lane, f, d, total - 1)
    _lib.check(rc)
    assert lane.lib.dgx_lane_sync(lane.h) == ERR_CAP
    ho = out.cpu().numpy()
    assert (ho[total - 1:] == FILL).all(), f"{name}: a value was written at or past out_cap"
    rc, out, off, _ = dev_filter(lane, f, d, total)
    _lib.check(rc)
    _lib.check(lane.lib.dgx_lane_sync(lane.h))
    hoff = off.cpu().numpy().view(np.uint64)
    ho = out.cpu().numpy()
    for qi, w in enumerate(ws):
        eq(ho[int(hoff[qi]):int(hoff[qi + 1])].view(np.uint64), w, f"{name}: query {qi} after the refusal")
