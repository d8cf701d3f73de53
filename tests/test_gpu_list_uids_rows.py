"""List.Uids over a task's rows with mutable layers (dgx_list_uids_rows / dgx_dev_list_uids_rows): every row compared in
full with the line-by-line List.Uids restatement (list_uids_oracle.c).  Runs on an H100 only (`pytest -m gpu`)."""
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
import list_uids_oracle as luo  # noqa: E402
from gen_mut import COMPRESSED, ITERATE, MUT_VALUE, PROBE  # noqa: E402
from test_gpu_parity import eq, pack_images, to_pack  # noqa: E402

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_CAP = -3, -4
MAX = 2**64 - 1
NONE = (np.zeros(0, np.uint64), np.zeros(0, np.uint8))


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
    """One key of a task: its immutable layer (uids, block size), branch, resolved mutable layer, delete-all bit."""

    def __init__(self, orc, dgx, uids, mode, mut=NONE, bs=256, delete_all=False):
        self.uids = None if uids is None else np.asarray(uids, np.uint64)
        self.mode, self.mut, self.delete_all = mode, mut, delete_all
        self.op = None if self.uids is None or self.uids.size == 0 else orc.encode(self.uids, bs)
        self.pack = None if self.op is None or delete_all else to_pack(dgx, self.op)

    def want(self, orc, after, v):
        op = None if self.delete_all else self.op
        if self.mode == COMPRESSED and (op is None or after > int(self.uids[-1])):
            return np.zeros(0, np.uint64)  # the reference's Bin branch indexes past the blocks there (DESIGN section 5)
        return luo.list_uids(op, self.mode, self.mut[0], self.mut[1], after, v)


def call(dgx, rows, after, v, keys=None):
    return dgx.algo.ListUidsRows([r.pack for r in rows], [r.mode for r in rows],
                                 [None if r.mode == COMPRESSED else r.mut for r in rows], after, v, keys)


def check(dgx, orc, rows, after, v, what, keys=None):
    out, off = call(dgx, rows, after, v, keys)
    assert off.size == len(rows) + 1 and int(off[0]) == 0
    for i, (g, r) in enumerate(zip(rows_of(out, off), rows)):
        eq(g, r.want(orc, after, v), f"{what}: after {after} row {i} mode {r.mode}")
    return out, off


def c6_rows(orc, dgx, rng, n_rows=300):
    """C6-shaped rows, 30 % of them with a layer of about 1 % of their length; modes by the ApproxLen rule, every third
    layered row forced to probe, every eleventh a delete-all row."""
    master, lists, v = gen_rows.c6_inputs(n_rows=n_rows, n_master=2_000_000, lo=100, hi=100_000, p_v=0.02)
    rows = []
    for i, u in enumerate(lists):
        if rng.random() >= 0.3:
            rows.append(Row(orc, dgx, u, COMPRESSED))
            continue
        mut = gen_mut.layer(rng, u, master, max(1, u.size // 100))
        approx = orc.approx_len(orc.encode(u, 256))
        mode = PROBE if i % 3 == 0 else gen_mut.mode_of(approx, v.size, True)
        rows.append(Row(orc, dgx, u, mode, mut, delete_all=i % 11 == 0))
    rows += [Row(orc, dgx, None, COMPRESSED), Row(orc, dgx, None, ITERATE, gen_mut.layer(rng, v, master, 50)),
             Row(orc, dgx, None, PROBE, gen_mut.layer(rng, v, master, 50))]
    return master, rows, v


def test_random_mix_all_modes(dgx, orc):
    rng = np.random.default_rng(90)
    master, rows, v = c6_rows(orc, dgx, rng)
    assert {r.mode for r in rows} == {COMPRESSED, PROBE, ITERATE} and any(r.delete_all for r in rows)
    for after in (0, int(v[v.size // 2]), MAX):
        check(dgx, orc, rows, after, v, "c6 mix")


def test_compressed_rows_equal_intersect_compressed_rows(dgx, orc):
    rng = np.random.default_rng(91)
    master = gen.zipf_gaps(rng, 1_000_000, start=1000)
    lists = [gen.thin(rng, master, p) for p in (0.5, 0.01, 0.2, 0.0005)] + [master[:1], master[-300:]]
    rows = [Row(orc, dgx, u, COMPRESSED, bs=bs) for u, bs in zip(lists, (256, 256, 7, 256, 256, 5000))]
    rows.insert(2, Row(orc, dgx, None, COMPRESSED))
    v = gen.thin(rng, master, 0.05)
    inside = int(v[v.size // 3])
    for after in (0, inside, inside + 1, int(master[-1]) + 1):
        out, off = check(dgx, orc, rows, after, v, "compressed")
        o2, f2 = dgx.algo.IntersectCompressedWithRows([r.pack for r in rows], after, v)
        assert np.array_equal(off, f2) and np.array_equal(out, o2), f"after {after}: differs from the rows call"


def test_pack_kinds(dgx, orc):
    """Named packs as cache misses then hits, pack images, NULL packs and an empty pack view, in one batch."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(92)
    master = gen.zipf_gaps(rng, 500_000, start=10)
    v = gen.thin(rng, master, 0.05)
    lists = [gen.thin(rng, master, p) for p in (0.3, 0.05, 0.6)]
    modes = (PROBE, ITERATE, COMPRESSED)
    rows = [Row(orc, dgx, u, md, gen_mut.layer(rng, u, master, 40) if md else NONE) for u, md in zip(lists, modes)]
    rows.append(Row(orc, dgx, None, ITERATE, gen_mut.layer(rng, v, master, 30)))
    after = int(v[v.size // 2])
    keys = [(9100 + i, 3) for i in range(len(rows))]
    lib.dgx_cache_clear()
    st = _lib.CacheStats()
    try:
        for rep in range(2):
            lib.dgx_cache_get_stats(C.byref(st))
            h0 = st.hits
            check(dgx, orc, rows, after, v, f"named rep {rep}", keys)
            lib.dgx_cache_get_stats(C.byref(st))
            assert (st.hits - h0 >= 3) == (rep == 1), "the second call must hit the three named packs"
    finally:
        lib.dgx_cache_clear()
    # the same rows as flat images, plus an empty pack view (nblocks 0), which is an empty layer
    mode = np.array([r.mode for r in rows] + [ITERATE], np.uint8)
    muts = [r.mut for r in rows] + [gen_mut.layer(rng, v, master, 20)]
    mut_off = np.zeros(len(muts) + 1, np.uint64)
    np.cumsum([m[0].size for m in muts], out=mut_off[1:])
    mu = np.concatenate([m[0] for m in muts])
    mf = np.concatenate([m[1] for m in muts])
    wants = [r.want(orc, after, v) for r in rows] + [luo.list_uids(None, ITERATE, muts[-1][0], muts[-1][1], after, v)]
    need = sum(w.size for w in wants)
    out = np.full(need + 8, 7, np.uint64)
    off = np.zeros(len(muts) + 1, np.uint64)
    with pack_images([r.pack for r in rows] + [None]) as refs:
        empty = _lib.PackView()
        refs[len(rows)].pack = C.pointer(empty)
        _lib.check(lib.dgx_list_uids_rows(refs, _p(mode), mode.size, _p(mu), _p(mf), _p(mut_off), after, _p(v), v.size,
                                          _p(out), _p(off), need))
    for i, g in enumerate(rows_of(out, off)):
        eq(g, wants[i], f"image row {i}")
    assert (out[need:] == 7).all()


def _raw(dgx, rows, mode, mut_off, mu, mf, after, v, out, off, cap):
    from dgraph_b200 import _lib

    refs, keep = dgx.algo._refs_of([r.pack for r in rows])
    return _lib.load().dgx_list_uids_rows(refs, _p(mode), mode.size, _p(mu), _p(mf), _p(mut_off), after, _p(v), v.size,
                                          _p(out), _p(off), cap)


def test_capacity_and_device_checked_errors(dgx, orc):
    rng = np.random.default_rng(93)
    master = gen.zipf_gaps(rng, 200_000, start=10)
    v = gen.thin(rng, master, 0.1)
    lists = [gen.thin(rng, master, p) for p in (0.4, 0.2)]
    rows = [Row(orc, dgx, lists[0], PROBE, gen_mut.layer(rng, lists[0], master, 30)),
            Row(orc, dgx, lists[1], ITERATE, gen_mut.layer(rng, lists[1], master, 30))]
    mode = np.array([r.mode for r in rows], np.uint8)
    mu = np.concatenate([r.mut[0] for r in rows])
    mf = np.concatenate([r.mut[1] for r in rows])
    mut_off = np.array([0, rows[0].mut[0].size, mu.size], np.uint64)
    wants = [r.want(orc, 0, v) for r in rows]
    need = sum(w.size for w in wants)
    out = np.full(need + 4, 7, np.uint64)
    off = np.zeros(3, np.uint64)
    assert _raw(dgx, rows, mode, mut_off, mu, mf, 0, v, out, off, need) == 0  # exact
    for i, g in enumerate(rows_of(out, off)):
        eq(g, wants[i], f"exact cap row {i}")
    out[:] = 7
    assert _raw(dgx, rows, mode, mut_off, mu, mf, 0, v, out, off, need - 1) == ERR_CAP  # one short
    assert (out == 7).all()
    # device-checked: order, uid 0, unknown flag bits, a probe / iterate pack that starts at uid 0
    k = int(mut_off[1]) + 3
    bad_order = mu.copy()
    bad_order[k] = bad_order[k - 1]
    bad_zero = mu.copy()
    bad_zero[0] = 0
    bad_flag = mf.copy()
    bad_flag[k] = 4
    for what, (m2, f2) in {"order": (bad_order, mf), "zero": (bad_zero, mf), "flags": (mu, bad_flag)}.items():
        out[:] = 7
        assert _raw(dgx, rows, mode, mut_off, m2, f2, 0, v, out, off, need) == ERR_ARG, what
        assert (out == 7).all(), what
    for md in (PROBE, ITERATE):
        zrows = [Row(orc, dgx, np.concatenate([[0], lists[0]]).astype(np.uint64), md, rows[0].mut), rows[1]]
        out[:] = 7
        rc = _raw(dgx, zrows, np.array([md, ITERATE], np.uint8), mut_off, mu, mf, 0, v, out, off, need + 1)
        assert rc == ERR_ARG and (out == 7).all(), f"mode {md} pack at uid 0"
    # a compressed row's pack may start at uid 0, as IntersectCompressedWith allows
    zrow = Row(orc, dgx, np.concatenate([[0], lists[0]]).astype(np.uint64), COMPRESSED)
    check(dgx, orc, [zrow, rows[1]], 0, np.concatenate([[0], v]).astype(np.uint64), "compressed pack at 0")


def test_device_form(dgx, orc):
    import torch

    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(94)
    master = gen.zipf_gaps(rng, 1_000_000, start=10)
    v = gen.thin(rng, master, 0.02)
    lists = [gen.thin(rng, master, p) for p in (0.5, 0.001, 0.2, 0.1)]
    rows = [Row(orc, dgx, lists[0], PROBE, gen_mut.layer(rng, lists[0], master, 300)),
            Row(orc, dgx, lists[1], COMPRESSED),
            Row(orc, dgx, lists[2], ITERATE, gen_mut.layer(rng, lists[2], master, 300), bs=7),
            Row(orc, dgx, None, ITERATE, gen_mut.layer(rng, v, master, 100)),
            Row(orc, dgx, lists[3], ITERATE, gen_mut.layer(rng, lists[3], master, 200), delete_all=True)]
    after = int(v[v.size // 2])
    mode = np.array([r.mode for r in rows], np.uint8)
    mut_off = np.zeros(len(rows) + 1, np.uint64)
    np.cumsum([r.mut[0].size for r in rows], out=mut_off[1:])
    mu = np.concatenate([r.mut[0] for r in rows])
    mf = np.concatenate([r.mut[1] for r in rows])
    wants = [r.want(orc, after, v) for r in rows]
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
        d_v = torch.from_numpy(v.view(np.int64)).cuda()
        d_mu = torch.from_numpy(mu.view(np.int64)).cuda()
        d_mf = torch.from_numpy(mf).cuda()
        d_out = torch.full((need + 1,), -7, dtype=torch.int64, device="cuda")
        d_off = torch.zeros(len(rows) + 1, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()

        def run(d_mu_, cap):
            return lib.dgx_dev_list_uids_rows(lane, tab, _p(mode), len(rows), C.c_void_p(d_mu_.data_ptr()),
                                              C.c_void_p(d_mf.data_ptr()), _p(mut_off), after,
                                              C.c_void_p(d_v.data_ptr()), v.size, C.c_void_p(d_out.data_ptr()), cap,
                                              C.c_void_p(d_off.data_ptr()))
        _lib.check(run(d_mu, need))
        _lib.check(lib.dgx_lane_sync(lane))
        out = d_out.cpu().numpy().view(np.uint64)
        off = d_off.cpu().numpy().view(np.uint64)
        for i, g in enumerate(rows_of(out, off)):
            eq(g, wants[i], f"device row {i}")
        assert int(out[need]) == (-7 & MAX)
        # one short: nothing is written and the sync reports DGX_ERR_CAP
        d_out.fill_(-7)
        torch.cuda.synchronize()
        _lib.check(run(d_mu, need - 1))
        assert lib.dgx_lane_sync(lane) == ERR_CAP
        assert bool((d_out == -7).all())
        # entries out of order: reported at the sync, d_out untouched, offsets zeroed
        bad = mu.copy()
        bad[[3, 4]] = bad[[4, 3]]
        d_bad = torch.from_numpy(bad.view(np.int64)).cuda()
        torch.cuda.synchronize()
        _lib.check(run(d_bad, need))
        assert lib.dgx_lane_sync(lane) == ERR_ARG
        assert b"mutable layer" in lib.dgx_last_error()
        assert bool((d_out == -7).all()) and bool((d_off == 0).all())
        _lib.check(lib.dgx_lane_sync(lane))
    finally:
        for h in handles:
            lib.dgx_dev_pack_free(h)
        lib.dgx_lane_destroy(lane)


def test_launch_count_independent_of_rows(dgx, orc):
    from dgraph_b200 import _lib

    rng = np.random.default_rng(95)
    master = gen.zipf_gaps(rng, 2_000_000)
    v = gen.thin(rng, master, 0.05)
    sizes = rng.integers(1, 3000, 10_000)
    starts = rng.integers(0, master.size - 3000, 10_000)
    rows = []
    for i, (s, n) in enumerate(zip(starts, sizes)):
        u = master[s: s + n]
        mode = (COMPRESSED, PROBE, ITERATE)[i % 3]
        rows.append(Row(orc, dgx, u, mode, gen_mut.layer(rng, u, master, int(n) // 50 + 1) if mode else NONE))
    deltas = []
    for n in (10, 10_000):
        k0 = _lib.stats()["kernel_launches"]
        out, off = call(dgx, rows[:n], 0, v)
        deltas.append(_lib.stats()["kernel_launches"] - k0)
        got = rows_of(out, off)
        for i in range(0, n, max(1, n // 200)):
            eq(got[i], rows[i].want(orc, 0, v), f"{n} rows: row {i}")
    assert deltas[0] == deltas[1] == 11, f"launches for 10 rows {deltas[0]}, for 10 000 rows {deltas[1]}"


def test_concurrent_threads(dgx, orc):
    rng = np.random.default_rng(96)
    master = gen.zipf_gaps(rng, 600_000)
    lists = [gen.thin(rng, master, p) for p in (0.5, 0.2, 0.05, 0.3, 0.6, 0.1)]
    rows = [Row(orc, dgx, u, (PROBE, ITERATE, COMPRESSED)[i % 3],
                gen_mut.layer(rng, u, master, 100) if i % 3 != 2 else NONE) for i, u in enumerate(lists)]
    vs = [gen.thin(rng, master, p) for p in (0.01, 0.1, 0.3, 0.002)]
    errs = []

    def work(t):
        try:
            r = np.random.default_rng(200 + t)
            for _ in range(5):
                sel = r.choice(len(rows), 4, replace=False).tolist()  # overlapping named packs across threads
                after = int(master[int(r.integers(0, master.size))]) if r.random() < 0.5 else 0
                check(dgx, orc, [rows[i] for i in sel], after, vs[t], f"thread {t}", [(9500 + i, 1) for i in sel])
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errs, errs[0]
    from dgraph_b200 import _lib

    _lib.load().dgx_cache_clear()


def test_uids_near_2_32_and_2_64(dgx, orc):
    rng = np.random.default_rng(97)
    near32 = np.arange(2**32 - 30_000, 2**32 + 30_000, 3, dtype=np.uint64)
    near64 = np.arange(MAX - 40_000, MAX, 2, dtype=np.uint64)  # below 2^64 - 1
    pool = np.concatenate([near32, near64, np.array([MAX], np.uint64)])
    lists = [gen.thin(rng, near32, 0.5), gen.thin(rng, near64, 0.5), np.concatenate([gen.thin(rng, near32, 0.3),
                                                                                    gen.thin(rng, near64, 0.3)])]
    layered = [Row(orc, dgx, u, md, gen_mut.layer(rng, u, pool, 200)) for u in lists for md in (PROBE, ITERATE)]
    layered.append(Row(orc, dgx, None, ITERATE, (np.array([2**32 - 1, 2**32, MAX], np.uint64),
                                                 np.array([0, MUT_VALUE, 0], np.uint8))))
    compressed = [Row(orc, dgx, u, COMPRESSED) for u in lists]
    v = gen.thin(rng, pool[:-1], 0.4)
    v_max = np.concatenate([v, [MAX]]).astype(np.uint64)
    for after in (0, 2**32 - 1, 2**32, int(near64[near64.size // 2]), MAX - 1, MAX):
        check(dgx, orc, layered + compressed, after, v, "near 2^64 (v below 2^64 - 1)")
        check(dgx, orc, layered, after, v_max, "near 2^64 (v holds 2^64 - 1)")
