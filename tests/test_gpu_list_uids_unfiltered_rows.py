"""List.Uids without a filter, and the count, over a task's rows (dgx_list_uids_unfiltered_rows / dgx_list_count_rows
and their device forms): every row compared in full with the line-by-line restatement
(list_uids_unfiltered_oracle.c).  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen  # noqa: E402
import gen_mut  # noqa: E402
import gen_rows  # noqa: E402
import list_uids_unfiltered_oracle as luo  # noqa: E402
from gen_mut import MUT_DEL, MUT_VALUE  # noqa: E402
from test_gpu_parity import eq, pack_images, to_pack  # noqa: E402

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_CAP = -3, -4
MAX = 2**64 - 1
MAXI32 = 2**31 - 1
NONE = (np.zeros(0, np.uint64), np.zeros(0, np.uint8))
FIRSTS = (0, MAXI32, 1, 10, 255, 256, 257, -1, -5)


@pytest.fixture(scope="module")
def dgx():
    import dgraph_b200
    from dgraph_b200 import _lib

    lib = _lib.load()
    _lib.check(lib.dgx_init(-1))
    return dgraph_b200


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def rows_of(out, off):
    return [out[int(off[i]): int(off[i + 1])] for i in range(off.size - 1)]


class Row:
    """One key of a task: its immutable layer (uids, block size), resolved mutable layer and delete-all bit."""

    def __init__(self, orc, dgx, uids, mut=NONE, bs=256, delete_all=False):
        self.uids = None if uids is None else np.asarray(uids, np.uint64)
        self.mut, self.delete_all = mut, delete_all
        self.op = None if self.uids is None or self.uids.size == 0 else orc.encode(self.uids, bs)
        self.pack = None if self.op is None or delete_all else to_pack(dgx, self.op)

    def want(self, after, first=0):
        return luo.list_uids_unfiltered(None if self.delete_all else self.op, self.mut[0], self.mut[1], after, first)

    def count(self, after):
        return luo.list_count(None if self.delete_all else self.op, self.mut[0], self.mut[1], after)


def check(dgx, rows, after, first, what, keys=None):
    out, off = dgx.algo.ListUidsUnfilteredRows([r.pack for r in rows], [r.mut for r in rows], after, first, keys)
    assert off.size == len(rows) + 1 and int(off[0]) == 0
    for i, (g, r) in enumerate(zip(rows_of(out, off), rows)):
        eq(g, r.want(after, first), f"{what}: after {after} first {first} row {i}")
    return out, off


def check_counts(dgx, rows, after, what, keys=None):
    got = dgx.algo.ListCountRows([r.pack for r in rows], [r.mut for r in rows], after, keys)
    assert got.dtype == np.uint32 and got.size == len(rows)
    want = [r.count(after) for r in rows]
    assert got.tolist() == want, f"{what}: after {after} counts differ"
    return got


def c6_rows(orc, dgx, rng, n_rows=300):
    """C6-shaped rows, 30 % of them with a layer of about 1 % of their length, every eleventh layered row a delete-all
    row; then a NULL row, an empty-layer row with entries only, and rows at BlockSize 10 and 5000."""
    master, lists, _ = gen_rows.c6_inputs(n_rows=n_rows, n_master=2_000_000, lo=100, hi=100_000, p_v=0.02)
    rows = []
    for i, u in enumerate(lists):
        if rng.random() >= 0.3:
            rows.append(Row(orc, dgx, u))
            continue
        rows.append(Row(orc, dgx, u, gen_mut.layer(rng, u, master, max(1, u.size // 100)), delete_all=i % 11 == 0))
    rows += [Row(orc, dgx, None), Row(orc, dgx, None, gen_mut.layer(rng, lists[0], master, 50)),
             Row(orc, dgx, lists[1], gen_mut.layer(rng, lists[1], master, 80), bs=10),
             Row(orc, dgx, lists[2], gen_mut.layer(rng, lists[2], master, 80), bs=5000)]
    return master, rows


def insert_cut(rows, after):
    """A First that cuts some row inside its inserts: one past the position of a layered row's first insert."""
    for r in rows:
        if r.mut[0].size == 0 or r.delete_all or r.uids is None:
            continue
        full = r.want(after)
        ins = np.nonzero(np.isin(full, r.mut[0]) & ~np.isin(full, r.uids))[0]
        if ins.size:
            return int(ins[ins.size // 2]) + 1
    raise AssertionError("no layered row inserts above after")


def test_c6_mix_every_after_and_first(dgx, orc):
    rng = np.random.default_rng(1101)
    master, rows = c6_rows(orc, dgx, rng)
    assert any(r.delete_all for r in rows) and any(r.pack is None and not r.delete_all for r in rows)
    big = next(r for r in rows if r.op is not None and r.op.nblocks > 4 and not r.delete_all)
    base = int(big.op.base[2])
    afters = (0, base, base - 1, int(master[master.size // 2]), MAX)
    for after in afters:
        cut = insert_cut(rows, after) if after != MAX else 3
        for first in FIRSTS + (cut,):
            out, off = check(dgx, rows, after, first, "c6 mix")
            if first == MAXI32:
                counts = check_counts(dgx, rows, after, "c6 mix")
                assert np.array_equal(counts.astype(np.uint64), np.diff(off)), "counts differ from the row lengths"


def test_layer_free_rows_equal_decode(dgx, orc):
    """A row without a layer is the pack decoded from after + 1 (Decoder.Seek(after, SeekCurrent))."""
    rng = np.random.default_rng(1102)
    master = gen.zipf_gaps(rng, 1_000_000, start=1000)
    lists = [gen.thin(rng, master, p) for p in (0.5, 0.01, 0.2, 0.0005)] + [master[:1], master[-300:]]
    rows = [Row(orc, dgx, u, bs=bs) for u, bs in zip(lists, (256, 256, 10, 256, 256, 5000))]
    for after in (0, int(master[0]), int(lists[0][lists[0].size // 3]), int(rows[0].op.base[5]) - 1,
                  int(master[-1]) - 1, int(master[-1])):
        out, off = check(dgx, rows, after, 0, "layer-free")
        for i, (g, r) in enumerate(zip(rows_of(out, off), rows)):
            eq(g, dgx.codec.Decode(r.pack, after + 1), f"after {after} row {i} vs Decode")


def test_pack_kinds(dgx, orc):
    """Named packs as cache misses then hits, pack images, NULL packs and an empty pack view, in one batch."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(1103)
    master = gen.zipf_gaps(rng, 500_000, start=10)
    lists = [gen.thin(rng, master, p) for p in (0.3, 0.05, 0.6)]
    rows = [Row(orc, dgx, u, gen_mut.layer(rng, u, master, 40) if i != 2 else NONE) for i, u in enumerate(lists)]
    rows.append(Row(orc, dgx, None, gen_mut.layer(rng, lists[0], master, 30)))
    after = int(master[master.size // 2])
    keys = [(11_100 + i, 3) for i in range(len(rows))]
    lib.dgx_cache_clear()
    st = _lib.CacheStats()
    try:
        for rep in range(2):
            lib.dgx_cache_get_stats(C.byref(st))
            h0 = st.hits
            check(dgx, rows, after, 100, f"named rep {rep}", keys)
            lib.dgx_cache_get_stats(C.byref(st))
            assert (st.hits - h0 >= 3) == (rep == 1), "the second call must hit the three named packs"
            check_counts(dgx, rows, after, f"named rep {rep}", keys)
    finally:
        lib.dgx_cache_clear()
    # the same rows as flat images, plus an empty pack view (nblocks 0), which is an empty layer
    muts = [r.mut for r in rows] + [gen_mut.layer(rng, lists[1], master, 20)]
    mut_off = np.zeros(len(muts) + 1, np.uint64)
    np.cumsum([m[0].size for m in muts], out=mut_off[1:])
    mu = np.concatenate([m[0] for m in muts])
    mf = np.concatenate([m[1] for m in muts])
    wants = [r.want(after) for r in rows] + [luo.list_uids_unfiltered(None, muts[-1][0], muts[-1][1], after)]
    need = sum(w.size for w in wants)
    out = np.full(need + 8, 7, np.uint64)
    off = np.zeros(len(muts) + 1, np.uint64)
    counts = np.zeros(len(muts), np.uint32)
    with pack_images([r.pack for r in rows] + [None]) as refs:
        empty = _lib.PackView()
        refs[len(rows)].pack = C.pointer(empty)
        _lib.check(lib.dgx_list_uids_unfiltered_rows(refs, len(muts), _p(mu), _p(mf), _p(mut_off), after, 0, _p(out),
                                                     _p(off), need))
        _lib.check(lib.dgx_list_count_rows(refs, len(muts), _p(mu), _p(mf), _p(mut_off), after, _p(counts)))
    for i, g in enumerate(rows_of(out, off)):
        eq(g, wants[i], f"image row {i}")
    assert counts.tolist() == [w.size for w in wants]
    assert (out[need:] == 7).all()


def _raw(dgx, rows, mut_off, mu, mf, after, first, out, off, cap, counts=None):
    from dgraph_b200 import _lib

    lib = _lib.load()
    refs, keep = dgx.algo._refs_of([r.pack for r in rows])
    if counts is not None:
        return lib.dgx_list_count_rows(refs, len(rows), _p(mu), _p(mf), _p(mut_off), after, _p(counts))
    return lib.dgx_list_uids_unfiltered_rows(refs, len(rows), _p(mu), _p(mf), _p(mut_off), after, first, _p(out),
                                             _p(off), cap)


def test_capacity_and_device_checked_errors(dgx, orc):
    rng = np.random.default_rng(1104)
    master = gen.zipf_gaps(rng, 200_000, start=10)
    lists = [gen.thin(rng, master, p) for p in (0.4, 0.2)]
    rows = [Row(orc, dgx, u, gen_mut.layer(rng, u, master, 30)) for u in lists]
    mu = np.concatenate([r.mut[0] for r in rows])
    mf = np.concatenate([r.mut[1] for r in rows])
    mut_off = np.array([0, rows[0].mut[0].size, mu.size], np.uint64)
    for first in (0, 300):
        wants = [r.want(0, first) for r in rows]
        need = sum(w.size for w in wants)
        out = np.full(need + 4, 7, np.uint64)
        off = np.zeros(3, np.uint64)
        assert _raw(dgx, rows, mut_off, mu, mf, 0, first, out, off, need) == 0  # exact
        for i, g in enumerate(rows_of(out, off)):
            eq(g, wants[i], f"first {first}: exact cap row {i}")
        out[:] = 7
        assert _raw(dgx, rows, mut_off, mu, mf, 0, first, out, off, need - 1) == ERR_CAP  # one short
        assert (out == 7).all()
    # device-checked: order, uid 0, unknown flag bits, a pack that starts at uid 0; rows and counts are emptied
    k = int(mut_off[1]) + 3
    bad_order = mu.copy()
    bad_order[k] = bad_order[k - 1]
    bad_zero = mu.copy()
    bad_zero[0] = 0
    bad_flag = mf.copy()
    bad_flag[k] = 4
    zrows = [Row(orc, dgx, np.concatenate([[0], lists[0]]).astype(np.uint64), rows[0].mut), rows[1]]
    for what, (rs, m2, f2) in {"order": (rows, bad_order, mf), "zero": (rows, bad_zero, mf),
                               "flags": (rows, mu, bad_flag), "pack at uid 0": (zrows, mu, mf)}.items():
        out[:] = 7
        off[:] = 9
        assert _raw(dgx, rs, mut_off, m2, f2, 0, 0, out, off, out.size) == ERR_ARG, what
        assert (out == 7).all() and (off == 0).all(), what
        counts = np.full(2, 9, np.uint32)
        assert _raw(dgx, rs, mut_off, m2, f2, 0, 0, None, None, 0, counts) == ERR_ARG, what
        assert (counts == 0).all(), what
    # an entry at or below after is still checked
    assert _raw(dgx, rows, mut_off, bad_zero, mf, MAX, 0, out, off, out.size) == ERR_ARG


def test_device_form(dgx, orc):
    import torch

    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(1105)
    master = gen.zipf_gaps(rng, 1_000_000, start=10)
    lists = [gen.thin(rng, master, p) for p in (0.5, 0.001, 0.2, 0.1)]
    rows = [Row(orc, dgx, lists[0], gen_mut.layer(rng, lists[0], master, 300)),
            Row(orc, dgx, lists[1]),
            Row(orc, dgx, lists[2], gen_mut.layer(rng, lists[2], master, 300), bs=10),
            Row(orc, dgx, None, gen_mut.layer(rng, lists[3], master, 100)),
            Row(orc, dgx, lists[3], gen_mut.layer(rng, lists[3], master, 200), delete_all=True)]
    after, first = int(master[master.size // 3]), 5000
    mut_off = np.zeros(len(rows) + 1, np.uint64)
    np.cumsum([r.mut[0].size for r in rows], out=mut_off[1:])
    mu = np.concatenate([r.mut[0] for r in rows])
    mf = np.concatenate([r.mut[1] for r in rows])
    wants = [r.want(after, first) for r in rows]
    need = sum(w.size for w in wants)
    stream = torch.cuda.Stream()
    lane = lib.dgx_lane_create(0, C.c_void_p(stream.cuda_stream))
    assert lane
    handles = []
    try:
        tab = (C.c_void_p * len(rows))()
        for i, r in enumerate(rows):
            if r.pack is None:
                continue
            view = dgx.codec.view_of(r.pack.normalized())
            h = C.c_void_p()
            _lib.check(lib.dgx_dev_pack_upload(lane, C.byref(view), C.byref(h)))
            handles.append(h)
            tab[i] = h.value
        d_mu = torch.from_numpy(mu.view(np.int64)).cuda()
        d_mf = torch.from_numpy(mf).cuda()
        d_out = torch.full((need + 1,), -7, dtype=torch.int64, device="cuda")
        d_off = torch.zeros(len(rows) + 1, dtype=torch.int64, device="cuda")
        d_cnt = torch.full((len(rows),), 9, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()

        def run(d_mu_, cap):
            return lib.dgx_dev_list_uids_unfiltered_rows(lane, tab, len(rows), C.c_void_p(d_mu_.data_ptr()),
                                                         C.c_void_p(d_mf.data_ptr()), _p(mut_off), after, first,
                                                         C.c_void_p(d_out.data_ptr()), cap, C.c_void_p(d_off.data_ptr()))

        def run_counts(d_mu_):
            return lib.dgx_dev_list_count_rows(lane, tab, len(rows), C.c_void_p(d_mu_.data_ptr()),
                                               C.c_void_p(d_mf.data_ptr()), _p(mut_off), after,
                                               C.c_void_p(d_cnt.data_ptr()))
        _lib.check(run(d_mu, need))
        _lib.check(run_counts(d_mu))
        _lib.check(lib.dgx_lane_sync(lane))
        out = d_out.cpu().numpy().view(np.uint64)
        off = d_off.cpu().numpy().view(np.uint64)
        for i, g in enumerate(rows_of(out, off)):
            eq(g, wants[i], f"device row {i}")
        assert int(out[need]) == (-7 & MAX)
        assert d_cnt.cpu().numpy().view(np.uint32).tolist() == [r.count(after) for r in rows]
        # one short: nothing is written and the sync reports DGX_ERR_CAP
        d_out.fill_(-7)
        torch.cuda.synchronize()
        _lib.check(run(d_mu, need - 1))
        assert lib.dgx_lane_sync(lane) == ERR_CAP
        assert bool((d_out == -7).all())
        # entries out of order: reported at the sync, d_out untouched, offsets and counts zeroed
        bad = mu.copy()
        bad[[3, 4]] = bad[[4, 3]]
        d_bad = torch.from_numpy(bad.view(np.int64)).cuda()
        torch.cuda.synchronize()
        _lib.check(run(d_bad, need))
        assert lib.dgx_lane_sync(lane) == ERR_ARG
        assert b"mutable layer" in lib.dgx_last_error()
        assert bool((d_out == -7).all()) and bool((d_off == 0).all())
        _lib.check(run_counts(d_bad))
        assert lib.dgx_lane_sync(lane) == ERR_ARG
        assert bool((d_cnt == 0).all())
        _lib.check(lib.dgx_lane_sync(lane))
    finally:
        for h in handles:
            lib.dgx_dev_pack_free(h)
        lib.dgx_lane_destroy(lane)


def test_launch_count_independent_of_rows(dgx, orc):
    from dgraph_b200 import _lib

    rng = np.random.default_rng(1106)
    master = gen.zipf_gaps(rng, 2_000_000)
    sizes = rng.integers(1, 3000, 10_000)
    starts = rng.integers(0, master.size - 3000, 10_000)
    rows = []
    for i, (s, n) in enumerate(zip(starts, sizes)):
        u = master[s: s + n]
        rows.append(Row(orc, dgx, u, gen_mut.layer(rng, u, master, int(n) // 50 + 1) if i % 2 else NONE))
    after = int(master[master.size // 2])
    deltas, cdeltas = [], []
    for n in (10, 10_000):
        k0 = _lib.stats()["kernel_launches"]
        out, off = dgx.algo.ListUidsUnfilteredRows([r.pack for r in rows[:n]], [r.mut for r in rows[:n]], after, 0)
        deltas.append(_lib.stats()["kernel_launches"] - k0)
        k0 = _lib.stats()["kernel_launches"]
        counts = dgx.algo.ListCountRows([r.pack for r in rows[:n]], [r.mut for r in rows[:n]], after)
        cdeltas.append(_lib.stats()["kernel_launches"] - k0)
        assert np.array_equal(counts.astype(np.uint64), np.diff(off))
        got = rows_of(out, off)
        for i in range(0, n, max(1, n // 200)):
            eq(got[i], rows[i].want(after), f"{n} rows: row {i}")
    assert deltas[0] == deltas[1] == 5, f"launches for 10 rows {deltas[0]}, for 10 000 rows {deltas[1]}"
    assert cdeltas[0] == cdeltas[1] == 3, f"count launches for 10 rows {cdeltas[0]}, for 10 000 rows {cdeltas[1]}"


def test_concurrent_threads(dgx, orc):
    rng = np.random.default_rng(1107)
    master = gen.zipf_gaps(rng, 600_000)
    lists = [gen.thin(rng, master, p) for p in (0.5, 0.2, 0.05, 0.3, 0.6, 0.1)]
    rows = [Row(orc, dgx, u, gen_mut.layer(rng, u, master, 100) if i % 3 else NONE) for i, u in enumerate(lists)]
    errs = []

    def work(t):
        try:
            r = np.random.default_rng(300 + t)
            for _ in range(5):
                sel = r.choice(len(rows), 4, replace=False).tolist()  # overlapping named packs across threads
                after = int(master[int(r.integers(0, master.size))]) if r.random() < 0.5 else 0
                first = FIRSTS[int(r.integers(0, len(FIRSTS)))]
                keys = [(11_500 + i, 1) for i in sel]
                check(dgx, [rows[i] for i in sel], after, first, f"thread {t}", keys)
                check_counts(dgx, [rows[i] for i in sel], after, f"thread {t}", keys)
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errs, errs[0]
    from dgraph_b200 import _lib

    _lib.load().dgx_cache_clear()


def test_uids_near_2_32_and_2_64(dgx, orc):
    rng = np.random.default_rng(1108)
    near32 = np.arange(2**32 - 30_000, 2**32 + 30_000, 3, dtype=np.uint64)
    near64 = np.arange(MAX - 40_000, MAX, 2, dtype=np.uint64)  # below 2^64 - 1
    pool = np.concatenate([near32, near64, np.array([MAX], np.uint64)])
    lists = [gen.thin(rng, near32, 0.5), gen.thin(rng, near64, 0.5),
             np.concatenate([gen.thin(rng, near32, 0.3), gen.thin(rng, near64, 0.3)]), np.append(near64[::7], MAX)]
    rows = [Row(orc, dgx, u, gen_mut.layer(rng, u, pool, 200)) for u in lists] + [Row(orc, dgx, u) for u in lists]
    rows.append(Row(orc, dgx, None, (np.array([2**32 - 1, 2**32, MAX - 1, MAX], np.uint64),
                                     np.array([0, MUT_VALUE, MUT_DEL, 0], np.uint8))))
    for after in (0, 2**32 - 1, 2**32, int(near64[near64.size // 2]), MAX - 1, MAX):
        for first in (0, 1, 257, -1):
            check(dgx, rows, after, first, "near 2^64")
        check_counts(dgx, rows, after, "near 2^64")
