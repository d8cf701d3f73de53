"""MergeSorted over the rows of a uid matrix (dgx_merge_sorted_matrix / dgx_dev_merge_sorted_matrix): every result
bit-exact against the oracle's MergeSorted of the same rows and, where noted, against dgx_merge_sorted given one
pointer per row.  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen  # noqa: E402
import gen_merge  # noqa: E402
from test_gpu_parity import eq, to_pack  # noqa: E402

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_CAP = -3, -4
GUARD = 0xDEADBEEFCAFEF00D


@pytest.fixture(scope="module")
def dgx():
    import dgraph_b200
    from dgraph_b200 import _lib

    lib = _lib.load()
    _lib.check(lib.dgx_init(-1))
    return dgraph_b200


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def u64(rows):
    return [np.ascontiguousarray(np.asarray(r, np.uint64)) for r in rows]


def check(dgx, orc, rows, what, per_row=True):
    rows = u64(rows)
    got = dgx.algo.MergeSortedMatrix(rows).Uids
    eq(got, orc.merge_sorted(rows), f"{what} vs oracle")
    if per_row:
        eq(got, dgx.algo.MergeSorted([dgx.pb.List(r) for r in rows]).Uids, f"{what} vs dgx_merge_sorted")
    return got


REF_TABLES = {  # algo/uidlist_test.go TestMergeSorted1..10, each input a matrix
    1: [[55]],
    2: [[1, 3, 6, 8, 10], [2, 4, 5, 7, 15]],
    3: [[1, 3, 6, 8, 10], []],
    4: [[], [1, 3, 6, 8, 10]],
    5: [[], []],
    6: [[11, 13, 16, 18, 20], [12, 14, 15, 15, 16, 16, 17, 25], [1, 2]],
    7: [[5, 6, 7], [3, 4], [1, 2], []],
    8: [],
    9: [[1, 1, 1]],
    10: [[1, 2, 3, 3, 6], [4, 8, 9]],
}


@pytest.mark.parametrize("case", sorted(REF_TABLES))
def test_reference_tables(dgx, orc, case):
    check(dgx, orc, REF_TABLES[case], f"TestMergeSorted{case}")


def _random_rows(rng, master, sizes):
    return [np.sort(rng.choice(master, int(s), replace=False)) if s else np.zeros(0, np.uint64) for s in sizes]


@pytest.mark.parametrize("shape", ["tiny", "huge", "mix"])
def test_random_matrices(dgx, orc, shape):
    rng = np.random.default_rng({"tiny": 11, "huge": 12, "mix": 13}[shape])
    master = gen.zipf_gaps(rng, 3_000_000)
    if shape == "tiny":
        sizes = rng.integers(0, 6, 30_000)
    elif shape == "huge":
        sizes = [1_500_000, 900_000, 2_000_000]
    else:
        sizes = np.concatenate([rng.integers(0, 40, 5_000), [700_000, 3, 250_000], rng.integers(100, 5_000, 300)])
        rng.shuffle(sizes)
    check(dgx, orc, _random_rows(rng, master, sizes), shape, per_row=shape != "tiny")


def test_duplicates_inside_and_across_rows(dgx, orc):
    rng = np.random.default_rng(14)
    base = gen.zipf_gaps(rng, 200_000)
    rows = []
    for _ in range(3_000):
        r = np.sort(rng.choice(base[:20_000], int(rng.integers(1, 60))))  # with replacement: repeats inside a row
        rows.append(r)
    check(dgx, orc, rows, "duplicates")


def test_identical_rows_and_hub(dgx, orc):
    rng = np.random.default_rng(15)
    row = gen.zipf_gaps(rng, 5_000)
    check(dgx, orc, [row] * 1_000, "identical rows", per_row=False)
    master = gen.zipf_gaps(rng, 1_000_000)
    hub = master[master.size // 3]
    rows = [np.union1d(np.sort(rng.choice(master, int(rng.integers(1, 33)), replace=False)), [hub]) for _ in range(20_000)]
    got = check(dgx, orc, rows, "hub", per_row=False)
    assert hub in got


def test_values_around_2_32_and_2_63(dgx, orc):
    top = np.uint64(2**64 - 1)
    rows = [
        np.arange(2**32 - 3000, 2**32 + 3000, 7, dtype=np.uint64),
        np.arange(2**32 - 1, 2**32 + 2, dtype=np.uint64),
        np.array([0, 2**63 - 1, 2**63, 2**63 + 1, 2**64 - 2, 2**64 - 1], np.uint64),
        np.array([top, top], np.uint64),
        np.arange(2**64 - 5000, 2**64 - 1, 3, dtype=np.uint64),
        np.arange(5 * 2**32 - 100, 5 * 2**32 + 100, dtype=np.uint64),
        np.zeros(0, np.uint64),
    ]
    got = check(dgx, orc, rows, "high values")
    assert int(got[-1]) == 2**64 - 1


def test_single_row_in_row_dedup(dgx, orc):
    rng = np.random.default_rng(16)
    r = np.sort(rng.integers(0, 50_000, 300_000).astype(np.uint64))
    check(dgx, orc, [r], "single row")


def test_overflow_path_forced(dgx, orc):
    """Rows of one tile each (2048 uids): uid 0 of every row and every 32nd after it are the samples, so the 31 uids of
    every row in between all fall into one bucket between two splitters -- 300 x 31 values, more than shared memory."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    rows = []
    for r in range(300):
        cluster = (1 << 40) + r * 31 + np.arange(31, dtype=np.uint64)
        high = (1 << 50) + np.uint64(r * 2016) + np.arange(2016, dtype=np.uint64)
        rows.append(np.concatenate([np.array([r + 1], np.uint64), cluster, high]))
    before = lib.dgx_merge_matrix_overflows(None)
    check(dgx, orc, rows, "adversarial")
    assert lib.dgx_merge_matrix_overflows(None) > before, "the overflow path did not run"


def test_descending_row_refused(dgx):
    from dgraph_b200 import _lib

    lib = _lib.load()
    v, off = gen_merge.csr(u64([[1, 2, 3], [10, 9], [4, 5, 5, 6]]))
    out = np.full(v.size, GUARD, np.uint64)
    n = C.c_size_t(12345)
    assert lib.dgx_merge_sorted_matrix(_p(v), _p(off), 3, _p(out), out.size, C.byref(n)) == ERR_ARG
    assert (out == np.uint64(GUARD)).all() and n.value == 12345
    # a repeated value is not a descent
    _lib.check(lib.dgx_merge_sorted_matrix(_p(v[5:]), _p(np.array([0, 4], np.uint64)), 1, _p(out), 4, C.byref(n)))
    eq(out[: n.value], [4, 5, 6], "repeat")


def test_host_cap(dgx, orc):
    from dgraph_b200 import _lib

    lib = _lib.load()
    rows = u64([[1, 2, 3], [2, 3, 4], [9]])
    v, off = gen_merge.csr(rows)
    out = np.full(v.size, GUARD, np.uint64)
    n = C.c_size_t(0)
    assert lib.dgx_merge_sorted_matrix(_p(v), _p(off), 3, _p(out), 4, C.byref(n)) == ERR_CAP
    _lib.check(lib.dgx_merge_sorted_matrix(_p(v), _p(off), 3, _p(out), 5, C.byref(n)))
    eq(out[: n.value], orc.merge_sorted(rows), "exact cap")


def _lane():
    import torch

    from dgraph_b200 import _lib

    stream = torch.cuda.Stream()
    lane = _lib.load().dgx_lane_create(0, C.c_void_p(stream.cuda_stream))
    assert lane
    return lane, stream


def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a).view(np.int64)).cuda()


def test_device_form_cap_order_and_bound(dgx, orc):
    import torch

    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(17)
    master = gen.zipf_gaps(rng, 400_000)
    rows = _random_rows(rng, master, rng.integers(0, 300, 2_000))
    want = orc.merge_sorted(rows)
    v, off = gen_merge.csr(rows)
    lane, _ = _lane()
    try:
        d_v, d_off = _dev(v), _dev(off)
        d_out = torch.full((v.size + 1,), -7, dtype=torch.int64, device="cuda")
        d_len = torch.zeros(1, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        args = lambda cap, vcap: (lane, C.c_void_p(d_v.data_ptr()), C.c_void_p(d_off.data_ptr()), len(rows), vcap,  # noqa: E731
                                  C.c_void_p(d_out.data_ptr()), cap, C.c_void_p(d_len.data_ptr()))
        _lib.check(lib.dgx_dev_merge_sorted_matrix(*args(v.size, v.size + 100)))
        _lib.check(lib.dgx_lane_sync(lane))
        n = int(d_len.item())
        eq(d_out.cpu().numpy().view(np.uint64)[:n], want, "device form")
        # one short: nothing past out_cap, DGX_ERR_CAP at the sync
        d_out.fill_(-7)
        torch.cuda.synchronize()
        _lib.check(lib.dgx_dev_merge_sorted_matrix(*args(want.size - 1, v.size)))
        assert lib.dgx_lane_sync(lane) == ERR_CAP
        assert int(d_out[want.size - 1].item()) == -7 and int(d_out[want.size].item()) == -7
        _lib.check(lib.dgx_lane_sync(lane))
        # d_v_off[nrows] > v_cap: DGX_ERR_CAP
        _lib.check(lib.dgx_dev_merge_sorted_matrix(*args(v.size, v.size - 1)))
        assert lib.dgx_lane_sync(lane) == ERR_CAP
        # a descending row: DGX_ERR_ARG at the sync
        bad = v.copy()
        r = next(i for i in range(len(rows)) if rows[i].size >= 2)
        bad[int(off[r])], bad[int(off[r]) + 1] = bad[int(off[r]) + 1], bad[int(off[r])]
        d_v.copy_(_dev(bad))
        torch.cuda.synchronize()
        _lib.check(lib.dgx_dev_merge_sorted_matrix(*args(v.size, v.size)))
        assert lib.dgx_lane_sync(lane) == ERR_ARG
        _lib.check(lib.dgx_lane_sync(lane))
    finally:
        lib.dgx_lane_destroy(lane)


def test_device_form_chained_after_rows(dgx, orc):
    """dgx_dev_intersect_compressed_rows -> dgx_dev_merge_sorted_matrix on one lane, no host round trip in between."""
    import torch

    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(18)
    master = gen.zipf_gaps(rng, 2_000_000)
    lists = [gen.thin(rng, master, p) for p in rng.uniform(0.001, 0.3, 40)] + [master[:1]]
    ops = [orc.encode(l, 256) for l in lists]
    v = gen.thin(rng, master, 0.05)
    after = int(master[master.size // 5])
    lane, _ = _lane()
    handles = []
    try:
        for op in ops:
            p = to_pack(dgx, op).normalized()
            view = dgx.codec.view_of(p)
            h = C.c_void_p()
            _lib.check(lib.dgx_dev_pack_upload(lane, C.byref(view), C.byref(h)))
            handles.append(h)
        tab = (C.c_void_p * len(handles))(*[h.value for h in handles])
        rows = [orc.intersect_compressed_with(op, after, v) for op in ops]
        cap = sum(min(v.size, l.size) for l in lists)
        d_v = _dev(v)
        d_rows = torch.zeros(cap + 1, dtype=torch.int64, device="cuda")
        d_off = torch.zeros(len(handles) + 1, dtype=torch.int64, device="cuda")
        d_out = torch.zeros(cap + 1, dtype=torch.int64, device="cuda")
        d_len = torch.zeros(1, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        _lib.check(lib.dgx_dev_intersect_compressed_rows(lane, tab, len(handles), after, C.c_void_p(d_v.data_ptr()), v.size,
                                                         C.c_void_p(d_rows.data_ptr()), cap, C.c_void_p(d_off.data_ptr())))
        _lib.check(lib.dgx_dev_merge_sorted_matrix(lane, C.c_void_p(d_rows.data_ptr()), C.c_void_p(d_off.data_ptr()),
                                                   len(handles), cap, C.c_void_p(d_out.data_ptr()), cap,
                                                   C.c_void_p(d_len.data_ptr())))
        _lib.check(lib.dgx_lane_sync(lane))
        n = int(d_len.item())
        eq(d_out.cpu().numpy().view(np.uint64)[:n], orc.merge_sorted(rows), "chained")
    finally:
        for h in handles:
            lib.dgx_dev_pack_free(h)
        lib.dgx_lane_destroy(lane)


def test_launch_count_independent_of_rows(dgx, orc):
    from dgraph_b200 import _lib

    rng = np.random.default_rng(19)
    master = gen.zipf_gaps(rng, 2_000_000)
    deltas = []
    for nrows in (10, 10_000):
        rows = _random_rows(rng, master, [100_000 // nrows] * nrows)
        k0 = _lib.stats()["kernel_launches"]
        got = dgx.algo.MergeSortedMatrix(rows).Uids
        deltas.append(_lib.stats()["kernel_launches"] - k0)
        eq(got, orc.merge_sorted(rows), f"{nrows} rows")
    assert deltas[0] == deltas[1], f"launches for 10 rows {deltas[0]} != for 10 000 rows {deltas[1]}"


def test_concurrent_threads(dgx, orc):
    rng = np.random.default_rng(20)
    master = gen.zipf_gaps(rng, 1_000_000)
    jobs = [_random_rows(rng, master, rng.integers(0, 400, 1_500)) for _ in range(8)]
    wants = [orc.merge_sorted(j) for j in jobs]
    got = [None] * 8
    errs = []

    def work(t):
        try:
            for _ in range(3):
                got[t] = dgx.algo.MergeSortedMatrix(jobs[t]).Uids
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs
    for t in range(8):
        eq(got[t], wants[t], f"thread {t}")


def test_full_c8b(dgx, orc):
    v, off = gen_merge.c8b()
    rows = gen_merge.rows_of(v, off)
    got = dgx.algo.MergeSortedMatrix(rows).Uids
    eq(got, orc.merge_sorted(rows), "C8b")
