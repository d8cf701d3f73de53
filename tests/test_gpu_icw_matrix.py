"""IntersectCompressedWith of one pack against every row of a uid matrix (dgx_intersect_compressed_matrix /
dgx_dev_intersect_compressed_matrix): every row bit-exact against the oracle's IntersectCompressedWith(pack, 0, v_i),
against dgx_intersect_compressed_ref called per row and against dgx_intersect_compressed_rows([pack], 0, v_i).
Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen  # noqa: E402
import gen_sort  # noqa: E402
from test_gpu_parity import eq, generic_bytes, image_bytes, pack_images, to_pack  # noqa: E402

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_CAP = -3, -4
GUARD = np.uint64(0xDEADBEEFCAFEF00D)


@pytest.fixture(scope="module")
def dgx():
    import dgraph_b200
    from dgraph_b200 import _lib

    lib = _lib.load()
    _lib.check(lib.dgx_init(-1))
    return dgraph_b200


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def want_row(orc, op, v):
    if op is None or op.is_nil or v.size == 0:
        return np.zeros(0, np.uint64)
    return orc.intersect_compressed_with(op, 0, v)


def rows_of(out, off):
    return [out[int(off[i]): int(off[i + 1])] for i in range(off.size - 1)]


def csr(rows):
    off = np.zeros(len(rows) + 1, np.uint64)
    np.cumsum([r.size for r in rows], out=off[1:])
    v = np.concatenate(rows) if int(off[-1]) else np.zeros(1, np.uint64)
    return np.ascontiguousarray(v, np.uint64), off


def single_ref(dgx, p, v):
    from dgraph_b200 import _lib

    if p is None:
        return np.zeros(0, np.uint64)
    pn = p.normalized()  # kept alive while the view points at its arrays
    view = dgx.codec.view_of(pn)
    ref = _lib.PackRef(C.pointer(view), 0, 0)
    out = np.empty(max(v.size, 1), np.uint64)
    n = C.c_size_t(0)
    _lib.check(_lib.load().dgx_intersect_compressed_ref(C.byref(ref), 0, _p(v), v.size, _p(out), v.size, C.byref(n)))
    return out[: n.value]


def rows_form(dgx, p, v):
    """The transpose identity: one pack, one v, through the many-packs entry point."""
    out, off = dgx.algo.IntersectCompressedWithRows([p], 0, v)
    return out[int(off[0]): int(off[1])]


def check(dgx, orc, op, p, rows, got_out, got_off, what, every=1):
    """Row i against the oracle; every `every`-th row also against the two other entry points."""
    assert got_off.size == len(rows) + 1 and int(got_off[0]) == 0, what
    got = rows_of(got_out, got_off)
    for i, v in enumerate(rows):
        w = want_row(orc, op, v)
        eq(got[i], w, f"{what} row {i}")
        if i % every == 0:
            eq(got[i], single_ref(dgx, p, v), f"{what} row {i} vs dgx_intersect_compressed_ref")
            eq(got[i], rows_form(dgx, p, v), f"{what} row {i} vs dgx_intersect_compressed_rows")


def row_shapes(rng, u):
    """Rows around the uids u of a pack: empty rows between the others, rows below / above the pack, a row longer than
    the pack, rows inside one block, thinnings, rows straddling the ends."""
    lo, hi = int(u[0]), int(u[-1])
    near = np.unique(np.concatenate([u, u + np.uint64(1), u[u > 0] - np.uint64(1)]))
    e = np.zeros(0, np.uint64)
    rows = [
        e,
        np.arange(max(lo - 500, 0), lo, 3, dtype=np.uint64),                  # below the pack
        gen.thin(rng, near, 0.3),
        e,
        np.arange(hi + 1, hi + 2000, 7, dtype=np.uint64),                      # above the pack
        np.unique(np.concatenate([near, np.arange(lo, lo + 50, dtype=np.uint64)])),  # longer than the pack
        u[:1].copy(),
        u[-1:].copy(),
        near[(near >= u[min(3, u.size - 1)]) & (near <= u[min(40, u.size - 1)])],  # inside one block (or a few)
        gen.thin(rng, u, 0.02),
        np.unique(np.concatenate([np.arange(0, lo + 1, max(lo // 50, 1), dtype=np.uint64), gen.thin(rng, u, 0.1),
                                  np.arange(hi, hi + 100, 9, dtype=np.uint64)])),  # straddles both ends
        e,
    ]
    for _ in range(30):
        a, b = sorted(rng.integers(0, near.size, 2).tolist())
        rows.append(gen.thin(rng, near[a: b + 1], float(rng.random())))
    return [np.ascontiguousarray(r, np.uint64) for r in rows]


PACK_CASES = {
    "bs256": (lambda rng: gen.zipf_gaps(rng, 200_000, start=1000), 256),
    "bs1": (lambda rng: gen.zipf_gaps(rng, 3_000, start=10), 1),
    "bs7": (lambda rng: gen.zipf_gaps(rng, 40_000, start=10), 7),
    "bs5000": (lambda rng: gen.zipf_gaps(rng, 60_000, start=10), 5000),       # blocks of more than 256 uids
    "msb": (lambda rng: np.unique(np.concatenate([
        np.arange(3 * 2**32 - 40_000, 3 * 2**32 + 40_000, 3, dtype=np.uint64),
        np.arange(5 * 2**32 - 1000, 5 * 2**32 + 700, 1, dtype=np.uint64)])), 256),
    "one_uid": (lambda rng: np.array([123_456_789], np.uint64), 256),
}


@pytest.mark.parametrize("case", sorted(PACK_CASES))
def test_matrix_pack_shapes(dgx, orc, case):
    rng = np.random.default_rng(90 + sorted(PACK_CASES).index(case))
    make, bs = PACK_CASES[case]
    u = make(rng)
    op = orc.encode(u, bs)
    p = to_pack(dgx, op)
    rows = row_shapes(rng, u)
    out, off = dgx.algo.IntersectCompressedWithMatrix(p, rows)
    check(dgx, orc, op, p, rows, out, off, case)


def test_matrix_nil_and_empty_pack(dgx):
    """A NULL pack or an empty pack view gives empty rows and runs no kernel; zero rows give [0]."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    rows = [np.array([1, 5, 9], np.uint64), np.zeros(0, np.uint64), np.arange(100, 200, dtype=np.uint64)]
    v, v_off = csr(rows)
    out = np.full(8, GUARD, np.uint64)
    empty = _lib.PackView()
    for pack in (None, C.pointer(empty)):
        ref = _lib.PackRef(pack, 0, 0)
        off = np.full(4, 99, np.uint64)
        k0 = _lib.stats()["kernel_launches"]
        _lib.check(lib.dgx_intersect_compressed_matrix(C.byref(ref), _p(v), _p(v_off), 3, _p(out), _p(off), 8))
        assert _lib.stats()["kernel_launches"] == k0
        assert off.tolist() == [0, 0, 0, 0]
        assert (out == GUARD).all()
    o, oo = dgx.algo.IntersectCompressedWithMatrix(None, rows)
    assert o.size == 0 and oo.tolist() == [0, 0, 0, 0]
    o, oo = dgx.algo.IntersectCompressedWithMatrix(None, [])
    assert o.size == 0 and oo.tolist() == [0]
    off1 = np.full(1, 99, np.uint64)
    ref = _lib.PackRef(None, 0, 0)
    _lib.check(lib.dgx_intersect_compressed_matrix(C.byref(ref), None, None, 0, None, _p(off1), 0))
    assert off1.tolist() == [0]


def test_matrix_chunking_and_row_counts(dgx, orc):
    """50 000 one-uid rows all in block 0 (the block's units spread over many warps), one row of 1e6 uids, and
    100 000 tiny rows, each in one call."""
    rng = np.random.default_rng(81)
    master = gen.zipf_gaps(rng, 3_000_000, start=1000)
    u = gen.thin(rng, master, 0.3)
    op = orc.encode(u, 256)
    p = to_pack(dgx, op)
    first = np.concatenate([u[:256], master[(master > u[0]) & (master < u[255])]])
    rows = [first[int(i): int(i) + 1] for i in rng.integers(0, first.size, 50_000)]
    out, off = dgx.algo.IntersectCompressedWithMatrix(p, rows)
    check(dgx, orc, op, p, rows, out, off, "block 0 x 50 000", every=2_500)
    big = [np.ascontiguousarray(master[: 1_000_000])]
    out, off = dgx.algo.IntersectCompressedWithMatrix(p, big)
    check(dgx, orc, op, p, big, out, off, "one row of 1e6")
    starts = rng.integers(0, master.size - 8, 100_000)
    sizes = rng.integers(0, 5, 100_000)
    tiny = [np.ascontiguousarray(master[s: s + n]) for s, n in zip(starts, sizes)]
    out, off = dgx.algo.IntersectCompressedWithMatrix(p, tiny)
    check(dgx, orc, op, p, tiny, out, off, "100 000 tiny rows", every=5_000)


def test_matrix_launch_count_independent_of_rows(dgx, orc):
    from dgraph_b200 import _lib

    rng = np.random.default_rng(82)
    master = gen.zipf_gaps(rng, 2_000_000)
    u = gen.thin(rng, master, 0.2)
    op = orc.encode(u, 256)
    p = to_pack(dgx, op)
    starts = rng.integers(0, master.size - 40, 100_000)
    allrows = [np.ascontiguousarray(master[s: s + 1 + s % 30]) for s in starts]
    deltas = []
    for n in (3, 100_000):
        k0 = _lib.stats()["kernel_launches"]
        out, off = dgx.algo.IntersectCompressedWithMatrix(p, allrows[:n])
        deltas.append(_lib.stats()["kernel_launches"] - k0)
        got = rows_of(out, off)
        for i in range(0, n, max(1, n // 300)):
            eq(got[i], orc.intersect_compressed_with(op, 0, allrows[i]), f"{n} rows: row {i}")
    assert deltas[0] == deltas[1], f"launches for 3 rows {deltas[0]} != for 100 000 rows {deltas[1]}"


def test_matrix_cache_and_staging_routes(dgx, orc):
    """A named pack misses, then hits; an anonymous pinned flat image and an anonymous generic view take the routes
    h2d_bytes shows: pack bytes + the matrix + its offset table."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(83)
    master = gen.zipf_gaps(rng, 1_000_000)
    u = gen.thin(rng, master, 0.1)
    op = orc.encode(u, 256)
    p = to_pack(dgx, op)
    rows = [gen.thin(rng, master, q) for q in (0.01, 0.001, 0.0, 0.05)] + [u[:7].copy()]
    wants = [want_row(orc, op, r) for r in rows]
    v, v_off = csr(rows)
    m = int(v_off[-1])
    matrix_bytes = 8 * m + 8 * (len(rows) + 3)
    cap = sum(w.size for w in wants)
    out, off = np.empty(cap + 1, np.uint64), np.zeros(len(rows) + 1, np.uint64)

    def call(ref):
        h0 = _lib.stats()["h2d_bytes"]
        _lib.check(lib.dgx_intersect_compressed_matrix(ref, _p(v), _p(v_off), len(rows), _p(out), _p(off), cap))
        for i, g in enumerate(rows_of(out, off)):
            eq(g, wants[i], f"row {i}")
        return _lib.stats()["h2d_bytes"] - h0

    lib.dgx_cache_clear()
    _lib.check(lib.dgx_cache_configure(1 << 30))
    try:
        st = _lib.CacheStats()
        lib.dgx_cache_get_stats(C.byref(st))
        h0, m0 = st.hits, st.misses
        refs, keep = dgx.algo._refs_of([p], [(4242, 7)])
        assert call(refs) == generic_bytes(p) + matrix_bytes
        lib.dgx_cache_get_stats(C.byref(st))
        assert (st.hits - h0, st.misses - m0) == (0, 1)
        assert call(refs) == matrix_bytes
        lib.dgx_cache_get_stats(C.byref(st))
        assert (st.hits - h0, st.misses - m0) == (1, 1)
        o, oo = dgx.algo.IntersectCompressedWithMatrix(p, rows, key=(4242, 7))
        for i, g in enumerate(rows_of(o, oo)):
            eq(g, wants[i], f"mirror named row {i}")
        anon, keep = dgx.algo._refs_of([p])
        assert call(anon) == generic_bytes(p) + matrix_bytes
        with pack_images([p]) as img:
            assert call(img) == image_bytes(p) + matrix_bytes
    finally:
        lib.dgx_cache_clear()
        _lib.check(lib.dgx_cache_configure(16 << 30))


def test_matrix_errors(dgx, orc):
    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(84)
    master = gen.zipf_gaps(rng, 400_000)
    u = gen.thin(rng, master, 0.5)
    op = orc.encode(u, 256)
    p = to_pack(dgx, op)
    rows = [gen.thin(rng, master, 0.2), gen.thin(rng, master, 0.05)]
    wants = [want_row(orc, op, r) for r in rows]
    need = sum(w.size for w in wants)
    v, v_off = csr(rows)
    refs, keep = dgx.algo._refs_of([p])

    def good_call(what):
        o, oo = dgx.algo.IntersectCompressedWithMatrix(p, rows)
        for i, g in enumerate(rows_of(o, oo)):
            eq(g, wants[i], f"after {what}: row {i}")

    # capacity: one short is DGX_ERR_CAP, nothing written past out_cap
    out = np.full(need, GUARD, np.uint64)
    off = np.zeros(3, np.uint64)
    assert lib.dgx_intersect_compressed_matrix(refs, _p(v), _p(v_off), 2, _p(out), _p(off), need - 1) == ERR_CAP
    assert out[need - 1] == GUARD
    _lib.check(lib.dgx_intersect_compressed_matrix(refs, _p(v), _p(v_off), 2, _p(out), _p(off), need))
    assert int(off[2]) == need
    # malformed packs, anonymous and named: refused, no cache entry left referenced, the next call works
    bad = dgx.pb.UidPack(p.block_size, p.base, p.num_uids, p.delta_off.copy(), p.deltas)
    bad.delta_off[3] = bad.delta_off[2] + 2
    for key in (None, (7101, 1)):
        with pytest.raises(_lib.DgxError) as ei:
            dgx.algo.IntersectCompressedWithMatrix(bad, rows, key=key)
        assert ei.value.code == ERR_ARG
        good_call(f"malformed pack key {key}")
    o, oo = dgx.algo.IntersectCompressedWithMatrix(p, rows, key=(7102, 1))  # a good named entry to be released
    lib.dgx_cache_clear()
    st = _lib.CacheStats()
    lib.dgx_cache_get_stats(C.byref(st))
    assert st.entries == 0
    # rows that do not ascend strictly: DGX_ERR_ARG, out untouched, the next call works
    dup = rows[0].copy()
    dup[5] = dup[4]
    desc = rows[1].copy()
    desc[[2, 3]] = desc[[3, 2]]
    for name, bad_rows in (("duplicate", [rows[1], dup]), ("descending", [desc, rows[0]])):
        bv, boff = csr(bad_rows)
        out = np.full(need + 8, GUARD, np.uint64)
        rc = lib.dgx_intersect_compressed_matrix(refs, _p(bv), _p(boff), 2, _p(out), _p(off), need + 8)
        assert rc == ERR_ARG, name
        assert (out == GUARD).all(), name
        good_call(name)
    # bad offsets are refused before anything of v is read (a one-value v buffer)
    tiny_v = np.zeros(1, np.uint64)
    for name, bo in (("first non-zero", [1, 2, 3]), ("decreasing", [0, 5, 4]), ("total >= 2^32", [0, 1, 1 << 32])):
        bo = np.array(bo, np.uint64)
        rc = lib.dgx_intersect_compressed_matrix(refs, _p(tiny_v), _p(bo), 2, _p(out), _p(off), need)
        assert rc == ERR_ARG, name
    good_call("bad offsets")


def test_matrix_device_form(dgx, orc):
    import torch

    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(85)
    master = gen.zipf_gaps(rng, 2_000_000)
    stream = torch.cuda.Stream()
    lane = lib.dgx_lane_create(0, C.c_void_p(stream.cuda_stream))
    assert lane
    handles = []
    try:
        for u, bs in ((gen.thin(rng, master, 0.3), 256), (gen.thin(rng, master, 0.05), 7)):
            op = orc.encode(u, bs)
            pn = to_pack(dgx, op).normalized()
            view = dgx.codec.view_of(pn)
            h = C.c_void_p()
            _lib.check(lib.dgx_dev_pack_upload(lane, C.byref(view), C.byref(h)))
            handles.append((op, h))
        rows = [gen.thin(rng, master, q) for q in (0.01, 0.0, 0.002, 0.1)] + [master[:3].copy()]
        v, v_off = csr(rows)
        d_v = torch.from_numpy(v.view(np.int64)).cuda()

        def run(h, rows_off, cap):
            d_out = torch.full((cap + 1,), -7, dtype=torch.int64, device="cuda")
            d_off = torch.full((len(rows_off),), -9, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            _lib.check(lib.dgx_dev_intersect_compressed_matrix(lane, h, C.c_void_p(d_v.data_ptr()), _p(rows_off),
                                                               len(rows_off) - 1, C.c_void_p(d_out.data_ptr()), cap,
                                                               C.c_void_p(d_off.data_ptr())))
            return d_out, d_off

        for op, h in handles + [(None, None)]:
            wants = [want_row(orc, op, r) for r in rows]
            need = sum(w.size for w in wants)
            d_out, d_off = run(h, v_off, need)
            _lib.check(lib.dgx_lane_sync(lane))
            out = d_out.cpu().numpy().view(np.uint64)
            off = d_off.cpu().numpy().view(np.uint64)
            for i, g in enumerate(rows_of(out, off)):
                eq(g, wants[i], f"device bs {None if op is None else op.block_size} row {i}")
            assert int(out[need]) == np.uint64(-7 & (2**64 - 1))
        # a row out of order surfaces at the sync; nothing reaches d_out; the lane works afterwards
        op, h = handles[0]
        bad = v.copy()
        bad[int(v_off[3]) + 1] = bad[int(v_off[3])]
        d_bad = torch.from_numpy(bad.view(np.int64)).cuda()
        d_v, keep_v = d_bad, d_v
        d_out, d_off = run(h, v_off, int(v_off[-1]))
        assert lib.dgx_lane_sync(lane) == ERR_ARG
        assert bool((d_out == -7).all()) and bool((d_off == 0).all())
        d_v = keep_v
        _lib.check(lib.dgx_lane_sync(lane))
        wants = [want_row(orc, op, r) for r in rows]
        d_out, d_off = run(h, v_off, sum(w.size for w in wants))
        _lib.check(lib.dgx_lane_sync(lane))
        for i, g in enumerate(rows_of(d_out.cpu().numpy().view(np.uint64), d_off.cpu().numpy().view(np.uint64))):
            eq(g, wants[i], f"device after order error row {i}")
        # zero rows: out_off[0] = 0
        d_out, d_off = run(h, np.zeros(1, np.uint64), 0)
        _lib.check(lib.dgx_lane_sync(lane))
        assert d_off.cpu().tolist() == [0]
    finally:
        for _, h in handles:
            lib.dgx_dev_pack_free(h)
        lib.dgx_lane_destroy(lane)


def test_matrix_concurrent_threads(dgx, orc):
    rng = np.random.default_rng(86)
    master = gen.zipf_gaps(rng, 600_000)
    ops = [orc.encode(gen.thin(rng, master, q), bs)
           for q, bs in zip((0.5, 0.2, 0.05, 0.3, 0.6, 0.1, 0.4, 0.01), (256, 256, 7, 256, 256, 1, 256, 256))]
    packs = [to_pack(dgx, op) for op in ops]
    errs = []

    def work(t):
        try:
            r = np.random.default_rng(200 + t)
            for rep in range(4):
                starts = r.integers(0, master.size - 2000, 300)
                rows = [gen.thin(r, master[s: s + int(r.integers(0, 2000))], float(r.random())) for s in starts]
                key = (9000 + t, 1) if rep % 2 else None
                out, off = dgx.algo.IntersectCompressedWithMatrix(packs[t], rows, key=key)
                for i, g in enumerate(rows_of(out, off)):
                    eq(g, want_row(orc, ops[t], rows[i]), f"thread {t} rep {rep} row {i}")
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errs, errs[0]
    from dgraph_b200 import _lib

    _lib.load().dgx_cache_clear()


def test_matrix_scale_c7(dgx, orc):
    """One call at the benchmark's intersectBucket size: the large bucket against all 10 000 rows, in full."""
    master, rows, buckets = gen_sort.c7_inputs()
    op = orc.encode(buckets["large"], 256)
    p = to_pack(dgx, op)
    out, off = dgx.algo.IntersectCompressedWithMatrix(p, rows)
    check(dgx, orc, op, p, rows, out, off, "C7 large", every=500)
