"""MergeSorted at the edges of its geometry (fixtures and host model: tests/merge_geometry.py), bit-exact against the
oracle: tile spans around 2^32 decided by splitter gaps and by real extremes, rounds that exactly fill or overflow shared
memory in both tile engines, values carried from one round to the next, runs without samples, the path thresholds
(tree / multiway / grouped / grouped twice), the pairwise tree's tile edges; the device form on one GPU; the packed form
through the grouped path and with more blocks than dgx_encode_bound plans for.  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import functools
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import merge_geometry as mg  # noqa: E402
from test_gpu_parity import L, eq, to_pack  # noqa: E402
from test_gpu_round2 import same_pack  # noqa: E402

pytestmark = pytest.mark.gpu

ERR_CAP = -4
FILL = -0x2152411035014FF3  # 0xDEADBEEFCAFEB00D as int64


@pytest.fixture(scope="module")
def dgx():
    import dgraph_b200
    from dgraph_b200 import _lib

    _lib.check(_lib.load().dgx_init(-1))
    return dgraph_b200


GEOMETRY = {f.name: f for f in mg.all_fixtures()}
TREE = {f.name: f for f in mg.tree_fixtures()}
CASES = list(GEOMETRY) + list(mg.THRESHOLDS) + list(TREE)


@functools.lru_cache(maxsize=None)
def case(name):
    """(runs, oracle result, plan) of a fixture, built once per module."""
    from oracle import pyoracle as orc

    if name in GEOMETRY:
        runs = GEOMETRY[name].runs
    elif name in TREE:
        runs = TREE[name].runs
    else:
        runs = mg.threshold_fixture(name).runs
    return runs, orc.merge_sorted(runs), mg.merge_plan([r.size for r in runs if r.size])


@pytest.mark.parametrize("name", CASES)
def test_host_form(dgx, name):
    from dgraph_b200 import _lib

    runs, want, plan = case(name)
    if name in mg.THRESHOLDS:
        assert plan.path == mg.THRESHOLDS[name][2]
    k0 = _lib.stats()["kernel_launches"]
    got = dgx.algo.MergeSorted([L(dgx, r) for r in runs]).Uids
    launches = _lib.stats()["kernel_launches"] - k0
    print(f"{name}: k={len(runs)} values={sum(r.size for r in runs)} {mg.describe(plan)}, {launches} launches")
    eq(got, want, name)
    assert launches == plan.launches, f"{name}: {launches} launches, {mg.describe(plan)} makes {plan.launches}"


# ---- the device form ------------------------------------------------------------------------------------------------

class Lane:
    def __init__(self):
        import torch

        from dgraph_b200 import _lib

        self.lib = _lib.load()
        self.stream = torch.cuda.Stream()
        self.h = self.lib.dgx_lane_create(0, C.c_void_p(self.stream.cuda_stream))
        assert self.h

    def launches(self):
        return self.lib.dgx_lane_launches(self.h)

    def sync(self):
        return self.lib.dgx_lane_sync(self.h)

    def close(self):
        self.lib.dgx_lane_destroy(self.h)


class DevLists:
    """The runs back to back in one device buffer, a pointer per run (NULL for an empty one)."""

    def __init__(self, runs):
        import torch

        self.lens = [int(r.size) for r in runs]
        self.total = sum(self.lens)
        cat = np.concatenate([np.asarray(r, np.uint64) for r in runs] + [np.zeros(1, np.uint64)])
        self.buf = torch.from_numpy(cat.view(np.int64)).cuda()
        offs = np.concatenate([[0], np.cumsum(self.lens)])
        base = self.buf.data_ptr()
        self.ptrs = (C.c_void_p * max(len(runs), 1))(*[base + 8 * int(o) if n else None for o, n in zip(offs, self.lens)])
        self.c_lens = (C.c_size_t * max(len(runs), 1))(*self.lens)


def dev_out(n):
    import torch

    return torch.full((n + 64,), FILL, dtype=torch.int64, device="cuda"), torch.full((1,), 7, dtype=torch.int64, device="cuda")


def dev_merge(lane, lists, d_out, d_len, cap):
    return lane.lib.dgx_dev_merge_sorted(lane.h, lists.ptrs, lists.c_lens, len(lists.lens), C.c_void_p(d_out.data_ptr()),
                                         cap, C.c_void_p(d_len.data_ptr()))


def check_out(d_out, d_len, want, what):
    n = int(d_len.item())
    out = d_out.cpu().numpy()
    eq(out[:n].view(np.uint64), want, what)
    # the final pass of these paths writes only the result: the rest of the buffer, out_cap included, keeps its fill
    assert (out[n:] == FILL).all(), f"{what}: {int((out[n:] != FILL).sum())} words written past out_len"


DEVICE_CASES = {  # one fixture of each path whose last pass writes straight into d_out
    "tree": "tree k=2 runs across every tile edge",
    "multiway": "32-bit padded 7695: rounds",
    "grouped": "k=65 at the grouping minimum",
    "grouped twice": "k=4097 grouped twice",
}


@pytest.mark.parametrize("path", list(DEVICE_CASES))
def test_device_form(dgx, path):
    import torch

    from dgraph_b200 import _lib

    name = DEVICE_CASES[path]
    runs, want, plan = case(name)
    assert mg.describe(plan).startswith(path.split()[0])
    lane = Lane()
    try:
        lists = DevLists(runs)
        d_out, d_len = dev_out(lists.total)
        torch.cuda.synchronize()
        l0 = lane.launches()
        _lib.check(dev_merge(lane, lists, d_out, d_len, lists.total))
        _lib.check(lane.sync())
        assert lane.launches() - l0 == plan.launches, (lane.launches() - l0, mg.describe(plan))
        check_out(d_out, d_len, want, f"{name} (device)")
        # one value short of the inputs' total: refused before anything is queued
        l0 = lane.launches()
        assert dev_merge(lane, lists, d_out, d_len, lists.total - 1) == ERR_CAP
        assert lane.launches() == l0
        _lib.check(lane.sync())
        # all inputs empty: length 0, no kernel
        empty = DevLists([np.zeros(0, np.uint64)] * 3)
        e_out, e_len = dev_out(0)
        torch.cuda.synchronize()
        _lib.check(dev_merge(lane, empty, e_out, e_len, 0))
        _lib.check(lane.sync())
        assert int(e_len.item()) == 0 and lane.launches() == l0
        # two calls back to back on the lane, one sync for both; the lane still works after the refusal above
        sub = DevLists(runs[:2])
        from oracle import pyoracle as orc

        want2 = orc.merge_sorted(runs[:2])
        d_out.fill_(FILL)
        d_out2, d_len2 = dev_out(sub.total)
        torch.cuda.synchronize()
        _lib.check(dev_merge(lane, lists, d_out, d_len, lists.total))
        _lib.check(dev_merge(lane, sub, d_out2, d_len2, sub.total))
        _lib.check(lane.sync())
        check_out(d_out, d_len, want, f"{name} (first of two)")
        check_out(d_out2, d_len2, want2, f"{name} (second of two)")
    finally:
        lane.close()


# ---- MergeSortedPacked ----------------------------------------------------------------------------------------------

def test_packed_grouped(dgx, orc):
    """Packs of block sizes 10, 256 and 1000, decoded on the device, merged through the grouped path, encoded."""
    rng = np.random.default_rng(700)
    lens = mg._spread(2 * 4 * mg.MERGE_MULTI_MIN + 5_000, 66)
    lists = mg.zipf_slices(rng, lens, master_len=1 << 22)
    assert mg.merge_plan(lens).path == "grouped"
    packs = [to_pack(dgx, orc.encode(l, (10, 256, 1000)[i % 3])) for i, l in enumerate(lists)]
    want = orc.merge_sorted(lists)
    for bs in (256, 10):
        same_pack(dgx.algo.MergeSortedPacked(packs, bs), orc.encode(want, bs), f"grouped packed merge bs={bs}")


def test_packed_more_blocks_than_the_bound(dgx, orc):
    """A result whose uids all differ in their upper 32 bits: a block each, far more than dgx_encode_bound's 64 spare
    blocks.  The first call reports DGX_ERR_CAP and the exact block count; the call again with the sizes it returned
    succeeds."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(701)
    u = (np.arange(1, 6_001, dtype=np.uint64) << np.uint64(32)) + rng.integers(0, 1 << 32, 6_000, dtype=np.uint64)
    lists = [u[0::3], u[1::3], np.sort(np.concatenate([u[2::3], u[::50]]))]
    want = orc.encode(orc.merge_sorted(lists), 256)
    refs, keep = dgx.algo._refs_of([to_pack(dgx, orc.encode(l, 256)) for l in lists])
    total = sum(l.size for l in lists)
    nb_cap, db_cap = C.c_size_t(0), C.c_size_t(0)
    lib.dgx_encode_bound(total, 256, C.byref(nb_cap), C.byref(db_cap))
    assert want.nblocks > nb_cap.value

    def call(nb, db):
        arrs = (np.zeros(max(nb, 1), np.uint64), np.zeros(max(nb, 1), np.uint32), np.zeros(nb + 1, np.uint64),
                np.zeros(max(db, 1), np.uint8))
        n, d, view = C.c_size_t(nb), C.c_size_t(db), _lib.PackView()
        rc = lib.dgx_merge_sorted_packed(refs, len(lists), 256, *[C.c_void_p(a.ctypes.data) for a in arrs], C.byref(n),
                                         C.byref(d), C.byref(view))
        return rc, n.value, d.value, arrs

    rc, nb, db, _ = call(nb_cap.value, db_cap.value)
    assert rc == ERR_CAP and nb == want.nblocks, (rc, nb, want.nblocks)
    rc, nb, db, (base, num, doff, deltas) = call(nb, db)
    _lib.check(rc)
    assert nb == want.nblocks and db == want.deltas.size
    eq(base[:nb], want.base, "base")
    assert np.array_equal(num[:nb], want.num_uids) and np.array_equal(doff[:nb + 1], want.delta_off)
    assert np.array_equal(deltas[:db], want.deltas)
    # the wrapper's own retry loop reaches the same pack
    same_pack(dgx.algo.MergeSortedPacked([to_pack(dgx, orc.encode(l, 256)) for l in lists]), want, "MergeSortedPacked")


# ---- threads --------------------------------------------------------------------------------------------------------

def test_threads_multiway_and_tree(dgx):
    names = ["32-bit bound value carried across rounds", "tree k=5", "64-bit padded 4104: rounds", "tree k=9"]
    jobs = [case(n) for n in names]
    errs = []

    def work(t):
        try:
            for it in range(3):
                runs, want, _ = jobs[(t + it) % len(jobs)]
                eq(dgx.algo.MergeSorted([L(dgx, r) for r in runs]).Uids, want, f"thread {t} {names[(t + it) % 4]}")
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs[0]
