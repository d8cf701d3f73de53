"""Batched IntersectCompressedWith (dgx_intersect_compressed_rows / dgx_dev_intersect_compressed_rows): every row
bit-exact against the oracle's IntersectCompressedWith and against dgx_intersect_compressed_ref called row by row.
Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen  # noqa: E402
import gen_rows  # noqa: E402
from test_gpu_parity import eq, generic_bytes, image_bytes, pack_images, to_pack  # noqa: E402

pytestmark = pytest.mark.gpu

ERR_ARG, ERR_CAP = -3, -4


@pytest.fixture(scope="module")
def dgx():
    import dgraph_b200
    from dgraph_b200 import _lib

    lib = _lib.load()
    _lib.check(lib.dgx_init(-1))
    return dgraph_b200


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def want_row(orc, op, after, v):
    """algo.IntersectCompressedWith(pack, after, v) on the oracle; after past the pack's last uid is the empty row
    (the reference's Bin branch would index past its blocks there, DESIGN section 5)."""
    if op is None or op.is_nil or v.size == 0:
        return np.zeros(0, np.uint64)
    if after > int(orc.decode(op, 0)[-1]):
        return np.zeros(0, np.uint64)
    return orc.intersect_compressed_with(op, after, v)


def rows_of(out, off):
    return [out[int(off[i]): int(off[i + 1])] for i in range(off.size - 1)]


def single_ref(dgx, p, after, v):
    """Today's one-pack-per-call entry point."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    if p is None:
        return np.zeros(0, np.uint64)
    pn = p.normalized()
    view = dgx.codec.view_of(pn)
    ref = _lib.PackRef(C.pointer(view), 0, 0)
    out = np.empty(max(v.size, 1), np.uint64)
    n = C.c_size_t(0)
    _lib.check(lib.dgx_intersect_compressed_ref(C.byref(ref), after, _p(v), v.size, _p(out), v.size, C.byref(n)))
    return out[: n.value]


def mixed_rows(rng):
    """Rows of one uid, one block, thousands of blocks, rows across multiples of 2^32 (MSB block splits), block
    sizes 1 / 7 / 256 / 5000, nil packs between them.  Returns (uid lists or None, block sizes)."""
    master = gen.zipf_gaps(rng, 3_000_000, start=1000)
    hi = np.unique(np.concatenate([np.arange(3 * 2**32 - 40_000, 3 * 2**32 + 40_000, 3, dtype=np.uint64),
                                   np.arange(5 * 2**32 - 1000, 5 * 2**32 + 700, 1, dtype=np.uint64)]))
    rows = [
        (master[500:501], 256),                               # one uid
        (master[1000:1200], 256),                             # one block
        None,
        (gen.thin(rng, master, 0.4), 256),                    # ~4700 blocks
        (gen.thin(rng, hi, 0.6), 256),                        # crosses 3 * 2^32 and 5 * 2^32
        (gen.thin(rng, master[:200_000], 0.5), 1),            # oversize path next to the fast path
        (gen.thin(rng, master[:200_000], 0.5), 7),
        (gen.thin(rng, master[:400_000], 0.2), 5000),
        None,
        (np.concatenate([gen.thin(rng, master, 0.05), gen.thin(rng, hi, 0.3)]), 256),
        (master[-300:], 256),
    ]
    return master, hi, rows


def v_cases(rng, master, hi):
    top = int(hi[-1])
    dense = np.unique(np.concatenate([master[1000:200_000],
                                      np.arange(int(master[1000]), int(master[1000]) + 3_000_000, 3, dtype=np.uint64),
                                      gen.thin(rng, hi, 0.7)]))
    return {
        "sparse": np.unique(np.concatenate([gen.thin(rng, master, 1e-4), gen.thin(rng, hi, 0.002)])),
        "medium": np.unique(np.concatenate([gen.thin(rng, master, 0.02), gen.thin(rng, hi, 0.05)])),
        "dense": dense,
        "empty": np.zeros(0, np.uint64),
        "below": np.arange(0, 1000, 7, dtype=np.uint64),
        "above": np.arange(top + 1, top + 5000, 3, dtype=np.uint64),
    }


def test_rows_mixed_against_oracle_and_single_calls(dgx, orc):
    rng = np.random.default_rng(71)
    master, hi, spec = mixed_rows(rng)
    ops = [None if s is None else orc.encode(s[0], s[1]) for s in spec]
    packs = [to_pack(dgx, op) if op is not None else None for op in ops]
    last = max(int(s[0][-1]) for s in spec if s is not None)
    inside = int(master[master.size // 3])
    regimes = set()
    for name, v in v_cases(rng, master, hi).items():
        for after in (0, inside, inside + 1, last + 1):
            out, off = dgx.algo.IntersectCompressedWithRows(packs, after, v)
            assert off.size == len(packs) + 1 and int(off[0]) == 0
            got = rows_of(out, off)
            for i, (op, p) in enumerate(zip(ops, packs)):
                what = f"v {name} after {after} row {i}"
                eq(got[i], want_row(orc, op, after, v), what)
                eq(got[i], single_ref(dgx, p, after, v), what + " vs single call")
                if p is not None and v.size:
                    regimes.add(p.nblocks > v.size)
    assert regimes == {True, False}, "both range regimes must run"


def test_rows_empty_pack_view_and_no_rows(dgx, orc):
    """An empty pack view (nblocks 0) passed through the ABI is an empty row, like a NULL pack; zero rows: [0]."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(72)
    u = gen.zipf_gaps(rng, 50_000)
    v = gen.thin(rng, u, 0.1)
    op = orc.encode(u, 256)
    p = to_pack(dgx, op).normalized()
    view = dgx.codec.view_of(p)
    empty = _lib.PackView()
    refs = (_lib.PackRef * 4)()
    refs[0].pack, refs[1].pack, refs[2].pack, refs[3].pack = C.pointer(empty), C.pointer(view), None, C.pointer(view)
    cap = 2 * v.size
    out = np.empty(cap, np.uint64)
    off = np.full(5, 99, np.uint64)
    _lib.check(lib.dgx_intersect_compressed_rows(refs, 4, 0, _p(v), v.size, _p(out), _p(off), cap))
    want = orc.intersect_compressed_with(op, 0, v)
    assert off.tolist() == [0, 0, want.size, want.size, 2 * want.size]
    eq(out[: want.size], want, "row 1")
    eq(out[want.size: 2 * want.size], want, "row 3")
    o, oo = dgx.algo.IntersectCompressedWithRows([], 0, v)
    assert o.size == 0 and oo.tolist() == [0]
    off1 = np.full(1, 99, np.uint64)
    _lib.check(lib.dgx_intersect_compressed_rows(refs, 0, 0, _p(v), v.size, _p(out), _p(off1), 0))
    assert off1.tolist() == [0]


def test_rows_named_packs_and_cache(dgx, orc):
    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(73)
    master = gen.zipf_gaps(rng, 1_000_000)
    lists = [gen.thin(rng, master, p) for p in (0.3, 0.1, 0.5, 0.02, 0.2, 0.4)]
    ops = [orc.encode(l, 256) for l in lists]
    packs = [to_pack(dgx, op) for op in ops]
    v = gen.thin(rng, master, 0.05)
    after = int(master[1000])
    want = [want_row(orc, op, after, v) for op in ops]
    # rows 0..5 named, row 6 repeats row 2's (key, version), row 7 anonymous
    batch = packs + [packs[2], packs[4]]
    keys = [(5000 + i, 1) for i in range(6)] + [(5002, 1), (0, 0)]
    wants = want + [want[2], want[4]]
    lib.dgx_cache_clear()
    _lib.check(lib.dgx_cache_configure(1 << 30))
    try:
        st = _lib.CacheStats()
        lib.dgx_cache_get_stats(C.byref(st))
        h0 = st.hits
        for rep in range(2):
            out, off = dgx.algo.IntersectCompressedWithRows(batch, after, v, keys)
            for i, g in enumerate(rows_of(out, off)):
                eq(g, wants[i], f"named rep {rep} row {i}")
        lib.dgx_cache_get_stats(C.byref(st))
        assert st.hits - h0 >= 7 + 1   # the second call hits all 7 named refs (the repeat already hit in the first)
        # a batch larger than a cache that holds about two packs: the rest cross PCIe as one-shot copies
        _lib.check(lib.dgx_cache_configure(int(2.5 * packs[0].deltas.size)))
        for rep in range(2):
            out, off = dgx.algo.IntersectCompressedWithRows(batch, after, v, [(6000 + i, 1) for i in range(len(batch))])
            for i, g in enumerate(rows_of(out, off)):
                eq(g, wants[i], f"small cache rep {rep} row {i}")
        lib.dgx_cache_get_stats(C.byref(st))
        assert st.bytes <= st.max_bytes
    finally:
        lib.dgx_cache_clear()
        _lib.check(lib.dgx_cache_configure(16 << 30))


def test_rows_cap_and_malformed(dgx, orc):
    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(74)
    master = gen.zipf_gaps(rng, 400_000)
    lists = [gen.thin(rng, master, 0.3), gen.thin(rng, master, 0.6)]
    ops = [orc.encode(l, 256) for l in lists]
    packs = [to_pack(dgx, op) for op in ops]
    v = gen.thin(rng, master, 0.2)
    refs, keep = dgx.algo._refs_of(packs)
    need = sum(want_row(orc, op, 0, v).size for op in ops)
    guard = np.uint64(0xDEADBEEFCAFEF00D)
    out = np.full(need, guard, np.uint64)
    off = np.zeros(3, np.uint64)
    rc = lib.dgx_intersect_compressed_rows(refs, 2, 0, _p(v), v.size, _p(out), _p(off), need - 1)
    assert rc == ERR_CAP
    assert out[need - 1] == guard
    _lib.check(lib.dgx_intersect_compressed_rows(refs, 2, 0, _p(v), v.size, _p(out), _p(off), need))
    assert int(off[2]) == need
    # a malformed pack among good ones is refused before any kernel runs
    good = packs[1]
    bad = dgx.pb.UidPack(good.block_size, good.base, good.num_uids, good.delta_off.copy(), good.deltas)
    bad.delta_off[3] = bad.delta_off[2] + 2
    with pytest.raises(_lib.DgxError) as ei:
        dgx.algo.IntersectCompressedWithRows([packs[0], bad, packs[1]], 0, v)
    assert ei.value.code == ERR_ARG
    bad_named = dgx.pb.UidPack(good.block_size, good.base, good.num_uids, good.delta_off.copy(), good.deltas)
    bad_named.delta_off[5] = bad_named.delta_off[4] - 1
    with pytest.raises(_lib.DgxError) as ei:
        dgx.algo.IntersectCompressedWithRows([packs[0], bad_named], 0, v, [(7001, 1), (7002, 1)])
    assert ei.value.code == ERR_ARG
    # the references the failed calls took on good named packs are released: entries still referenced are never
    # evicted, so a leaked one would survive the clear
    with pytest.raises(_lib.DgxError) as ei:
        dgx.algo.IntersectCompressedWithRows([packs[0], packs[1], bad], 0, v, [(7003, 1), (7004, 1), (0, 0)])
    assert ei.value.code == ERR_ARG
    lib.dgx_cache_clear()
    st = _lib.CacheStats()
    lib.dgx_cache_get_stats(C.byref(st))
    assert st.entries == 0
    # v of 2^32 or more uids is refused (the per-block v-ranges are 32-bit); nothing of v is read
    rc = lib.dgx_intersect_compressed_rows(refs, 2, 0, _p(v), 1 << 32, _p(out), _p(off), need)
    assert rc == ERR_ARG
    # the library is usable afterwards
    out2, off2 = dgx.algo.IntersectCompressedWithRows(packs, 0, v)
    for i, g in enumerate(rows_of(out2, off2)):
        eq(g, want_row(orc, ops[i], 0, v), f"after errors row {i}")


def test_rows_pack_images(dgx, orc):
    """Anonymous packs written back to back as flat images into one pinned buffer (what bench.py and the C6 rows of
    tools/bench_ops.py send) cross PCIe as one transfer; a gap between two images sends the call down the route for
    separate arrays; a malformed image among good ones is refused."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(79)
    master = gen.zipf_gaps(rng, 600_000)
    lists = [gen.thin(rng, master, 0.3), gen.thin(rng, master, 0.001), None, gen.thin(rng, master, 0.5), master[:1]]
    ops = [None if l is None else orc.encode(l, bs) for l, bs in zip(lists, (256, 256, 0, 7, 256))]
    packs = [None if op is None else to_pack(dgx, op) for op in ops]
    v = gen.thin(rng, master, 0.05)
    after = int(master[1000])
    wants = [want_row(orc, op, after, v) for op in ops]
    cap = sum(w.size for w in wants)
    out, off = np.empty(cap + 1, np.uint64), np.zeros(len(packs) + 1, np.uint64)

    def call(refs):
        h0 = _lib.stats()["h2d_bytes"]
        _lib.check(lib.dgx_intersect_compressed_rows(refs, len(packs), after, _p(v), v.size, _p(out), _p(off), cap))
        return [r.copy() for r in rows_of(out, off)], _lib.stats()["h2d_bytes"] - h0

    refs, keep = dgx.algo._refs_of(packs)
    separate, h2d_separate = call(refs)
    for i, g in enumerate(separate):
        eq(g, wants[i], f"separate arrays row {i}")
    real = [p for p in packs if p is not None]
    for gaps, extra in (((), sum(image_bytes(p) - generic_bytes(p) for p in real)), ((3,), 0)):
        with pack_images(packs, gaps) as img_refs:
            got, h2d = call(img_refs)
        for i, g in enumerate(got):
            eq(g, wants[i], f"images gaps {gaps} row {i}")
            eq(g, separate[i], f"images gaps {gaps} row {i} vs separate arrays")
        assert h2d == h2d_separate + extra, f"gaps {gaps}: staged through the wrong route"
    bad = dgx.pb.UidPack(packs[3].block_size, packs[3].base, packs[3].num_uids, packs[3].delta_off.copy(), packs[3].deltas)
    bad.delta_off[3] = bad.delta_off[2] + 2
    with pack_images(packs[:3] + [bad] + packs[4:]) as img_refs:
        rc = lib.dgx_intersect_compressed_rows(img_refs, len(packs), after, _p(v), v.size, _p(out), _p(off), cap)
    assert rc == ERR_ARG


def test_rows_device_form(dgx, orc):
    import torch

    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(75)
    master = gen.zipf_gaps(rng, 2_000_000)
    lists = [gen.thin(rng, master, p) for p in (0.5, 0.001, 0.2)] + [master[:1]]
    ops = [orc.encode(l, bs) for l, bs in zip(lists, (256, 256, 7, 256))]
    v = gen.thin(rng, master, 0.01)
    after = int(master[master.size // 2])
    stream = torch.cuda.Stream()
    lane = lib.dgx_lane_create(0, C.c_void_p(stream.cuda_stream))
    assert lane
    handles = []
    try:
        for op in ops:
            p = to_pack(dgx, op).normalized()
            view = dgx.codec.view_of(p)
            h = C.c_void_p()
            _lib.check(lib.dgx_dev_pack_upload(lane, C.byref(view), C.byref(h)))
            handles.append(h)
        order = [0, None, 1, 2, 3, 0]
        tab = (C.c_void_p * len(order))(*[None if i is None else handles[i].value for i in order])
        wants = [np.zeros(0, np.uint64) if i is None else want_row(orc, ops[i], after, v) for i in order]
        need = sum(w.size for w in wants)
        d_v = torch.from_numpy(v.view(np.int64)).cuda()
        d_out = torch.full((need + 1,), -7, dtype=torch.int64, device="cuda")
        d_off = torch.zeros(len(order) + 1, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        _lib.check(lib.dgx_dev_intersect_compressed_rows(lane, tab, len(order), after, C.c_void_p(d_v.data_ptr()), v.size,
                                                         C.c_void_p(d_out.data_ptr()), need, C.c_void_p(d_off.data_ptr())))
        _lib.check(lib.dgx_lane_sync(lane))
        out = d_out.cpu().numpy().view(np.uint64)
        off = d_off.cpu().numpy().view(np.uint64)
        for i, g in enumerate(rows_of(out, off)):
            eq(g, wants[i], f"device row {i}")
        assert int(out[need]) == np.uint64(-7 & (2**64 - 1))
        # one short: nothing is written and the sync reports DGX_ERR_CAP
        d_out.fill_(-7)
        torch.cuda.synchronize()
        _lib.check(lib.dgx_dev_intersect_compressed_rows(lane, tab, len(order), after, C.c_void_p(d_v.data_ptr()), v.size,
                                                         C.c_void_p(d_out.data_ptr()), need - 1, C.c_void_p(d_off.data_ptr())))
        assert lib.dgx_lane_sync(lane) == ERR_CAP
        assert bool((d_out == -7).all())
        _lib.check(lib.dgx_lane_sync(lane))
    finally:
        for h in handles:
            lib.dgx_dev_pack_free(h)
        lib.dgx_lane_destroy(lane)


def test_rows_launch_count_independent_of_rows(dgx, orc):
    from dgraph_b200 import _lib

    rng = np.random.default_rng(76)
    master = gen.zipf_gaps(rng, 2_000_000)
    v = gen.thin(rng, master, 0.05)
    sizes = rng.integers(1, 3000, 10_000)
    starts = rng.integers(0, master.size - 3000, 10_000)
    lists = [master[s: s + n] for s, n in zip(starts, sizes)]
    ops = [orc.encode(l, 256) for l in lists]
    packs = [to_pack(dgx, op) for op in ops]
    deltas = []
    for n in (10, 10_000):
        k0 = _lib.stats()["kernel_launches"]
        out, off = dgx.algo.IntersectCompressedWithRows(packs[:n], 0, v)
        deltas.append(_lib.stats()["kernel_launches"] - k0)
        got = rows_of(out, off)
        for i in range(0, n, max(1, n // 200)):
            eq(got[i], orc.intersect_compressed_with(ops[i], 0, v), f"{n} rows: row {i}")
    assert deltas[0] == deltas[1], f"launches for 10 rows {deltas[0]} != for 10 000 rows {deltas[1]}"


def test_rows_concurrent_threads(dgx, orc):
    rng = np.random.default_rng(77)
    master = gen.zipf_gaps(rng, 600_000)
    lists = [gen.thin(rng, master, p) for p in (0.5, 0.2, 0.05, 0.3, 0.6, 0.1, 0.4, 0.25)]
    ops = [orc.encode(l, 256) for l in lists]
    packs = [to_pack(dgx, op) for op in ops]
    vs = [gen.thin(rng, master, p) for p in (0.01, 0.1, 0.3, 0.002)]
    errs = []

    def work(t):
        try:
            r = np.random.default_rng(100 + t)
            for _ in range(6):
                sel = r.choice(len(packs), 5, replace=False).tolist()   # overlapping named packs across threads
                v = vs[t]
                after = int(master[int(r.integers(0, master.size))]) if r.random() < 0.5 else 0
                out, off = dgx.algo.IntersectCompressedWithRows([packs[i] for i in sel], after, v,
                                                                [(8000 + i, 1) for i in sel])
                for j, g in enumerate(rows_of(out, off)):
                    eq(g, want_row(orc, ops[sel[j]], after, v), f"thread {t} row {j}")
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errs, errs[0]
    from dgraph_b200 import _lib

    _lib.load().dgx_cache_clear()


def test_rows_wire_uid_matrix(dgx, orc):
    """The CSR result framed as pb.Result.uid_matrix and read back row by row."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(78)
    master = gen.zipf_gaps(rng, 300_000)
    lists = [gen.thin(rng, master, 0.3), None, gen.thin(rng, master, 0.05), master[:5]]
    ops = [None if l is None else orc.encode(l, 256) for l in lists]
    packs = [None if op is None else to_pack(dgx, op) for op in ops]
    v = gen.thin(rng, master, 0.2)
    out, off = dgx.algo.IntersectCompressedWithRows(packs, 0, v)
    out = np.ascontiguousarray(out) if out.size else np.zeros(1, np.uint64)
    n = C.c_size_t(0)
    _lib.check(lib.dgx_wire_uid_matrix(_p(out), _p(off), len(packs), None, 0, C.byref(n)))
    buf = np.zeros(max(n.value, 1), np.uint8)
    _lib.check(lib.dgx_wire_uid_matrix(_p(out), _p(off), len(packs), _p(buf), buf.size, C.byref(n)))
    # walk the uid_matrix entries: tag 0x0A, varint length, pb.List bytes
    data, pos, row = buf[: n.value].tobytes(), 0, 0
    while pos < len(data):
        assert data[pos] == 0x0A
        pos += 1
        ln, shift = 0, 0
        while True:
            b = data[pos]
            pos += 1
            ln |= (b & 0x7F) << shift
            shift += 7
            if b < 0x80:
                break
        msg = np.frombuffer(data[pos: pos + ln], np.uint8).copy()
        dec = np.empty(max(ln // 8 + 1, 1), np.uint64)
        cnt = C.c_size_t(0)
        _lib.check(lib.dgx_wire_list_decode(_p(msg), ln, _p(dec), dec.size, C.byref(cnt)))
        eq(dec[: cnt.value], want_row(orc, ops[row], 0, v), f"wire row {row}")
        pos += ln
        row += 1
    assert row == len(packs)


def test_rows_scale_c6(dgx, orc):
    """One call of 10 000 rows at the benchmark's handleUidPostings workload, compared in full with the oracle."""
    master, rows, v = gen_rows.c6_inputs()
    ops = [orc.encode(r, 256) for r in rows]
    packs = [to_pack(dgx, op) for op in ops]
    for after in (0, int(master[master.size // 2])):
        out, off = dgx.algo.IntersectCompressedWithRows(packs, after, v)
        got = rows_of(out, off)
        for i, op in enumerate(ops):
            eq(got[i], want_row(orc, op, after, v), f"C6 after {after} row {i}")
