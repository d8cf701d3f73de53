"""GPU parity, round-2 entry points and BASELINE-size configs: libdgx (through the C ABI) vs the CPU
oracle, bit-exact.  Runs on an H100 only (`pytest -m gpu`).

 - IntersectSorted over packs (dgx_intersect_sorted_packed) with and without the HBM pack cache, as flat images in
   pinned memory and decoded in place (DGX_ZERO_COPY=1)
 - IndexOf batch, shared-list batch
 - malformed packs are refused, not walked
 - BASELINE configs[2] (1e8-UID pack -> decode -> IntersectSorted), configs[3] (10k pairs, power-law sizes),
   configs[4] (MergeSorted k=64 sum 1e8 + Difference) at full size: order-sensitive 64-bit hash + length +
   sampled positions against the oracle (SURVEY 8d: full compare up to 1e7 outputs, hash above).
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen  # noqa: E402
from test_gpu_parity import L, eq, generic_bytes, image_bytes, pack_images, to_pack  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dgx():
    import dgraph_b200
    from dgraph_b200 import _lib

    lib = _lib.load()
    _lib.check(lib.dgx_init(-1))
    return dgraph_b200


def order_hash(a: np.ndarray) -> int:
    """64-bit order-sensitive hash: sum_i (a[i] * M1 + i * M2) ^ rot, wrapping (numpy uint64 arithmetic)."""
    a = np.ascontiguousarray(a, dtype=np.uint64)
    i = np.arange(a.size, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x = a * np.uint64(0x9E3779B97F4A7C15) + i * np.uint64(0xC2B2AE3D27D4EB4F)
        x ^= x >> np.uint64(29)
        x *= np.uint64(0xBF58476D1CE4E5B9)
        return int(x.sum(dtype=np.uint64))


def same(got, want, what):
    """Full compare up to 1e7 values, hash + length + 1e6 sampled positions above."""
    got = np.asarray(got, dtype=np.uint64)
    want = np.asarray(want, dtype=np.uint64)
    assert got.size == want.size, f"{what}: len got {got.size} want {want.size}"
    if got.size <= 10_000_000:
        eq(got, want, what)
        return
    assert order_hash(got) == order_hash(want), f"{what}: order-sensitive hash differs"
    pos = np.random.default_rng(5).integers(0, got.size, 1_000_000)
    assert np.array_equal(got[pos], want[pos]), f"{what}: sampled positions differ"


# ---- IntersectSorted over packs, pack cache -------------------------------------------------------

def test_intersect_sorted_packed(dgx, orc):
    from dgraph_b200 import _lib

    rng = np.random.default_rng(31)
    master = gen.zipf_gaps(rng, 400_000)
    for k, p, bs in ((1, 0.5, 256), (2, 0.5, 256), (3, 0.3, 10), (8, 0.25, 256), (8, 0.9, 256), (12, 0.8, 64)):
        lists = [gen.thin(rng, master, p) for _ in range(k)]
        packs = [to_pack(dgx, orc.encode(l, bs)) for l in lists]
        got = dgx.algo.IntersectSortedPacks(packs)
        eq(got.Uids, orc.intersect_sorted(lists), f"packed k={k} p={p} bs={bs}")
    # nil / empty packs: the empty list; no packs: &pb.List{}
    lists = [gen.thin(rng, master, 0.5) for _ in range(3)]
    packs = [to_pack(dgx, orc.encode(l, 256)) for l in lists]
    assert dgx.algo.IntersectSortedPacks(packs[:2] + [None]).tolist() == []
    assert dgx.algo.IntersectSortedPacks([]).Uids is None
    # values across 32-bit-MSB block splits and at the top of the range
    hi = np.sort(rng.integers(2**63, 2**64 - 1, 50_000, dtype=np.uint64))
    hi = np.unique(hi)
    a, b = hi[rng.random(hi.size) < 0.7], hi[rng.random(hi.size) < 0.7]
    got = dgx.algo.IntersectSortedPacks([to_pack(dgx, orc.encode(a, 256)), to_pack(dgx, orc.encode(b, 256))])
    eq(got.Uids, orc.intersect_sorted([a, b]), "packed full-range")
    # flat images back to back in one pinned buffer cross PCIe as one transfer; a gap between two images sends the
    # call down the route for separate arrays; a malformed image among good ones is refused
    lists = [gen.thin(rng, master, p) for p in (0.5, 0.6, 0.7)]
    packs = [to_pack(dgx, orc.encode(l, bs)) for l, bs in zip(lists, (256, 10, 256))]
    want = orc.intersect_sorted(lists)
    eq(dgx.algo.IntersectSortedPacks(packs).Uids, want, "separate arrays")
    for gaps, staged in (((), sum(image_bytes(p) for p in packs)), ((1,), sum(generic_bytes(p) for p in packs))):
        with pack_images(packs, gaps) as refs:
            got, h2d = sorted_packed(refs, len(packs), want.size)
        eq(got, want, f"images gaps {gaps}")
        assert h2d == staged, f"gaps {gaps}: staged through the wrong route"
    bad = dgx.pb.UidPack(packs[1].block_size, packs[1].base, packs[1].num_uids, packs[1].delta_off.copy(), packs[1].deltas)
    bad.delta_off[3] = bad.delta_off[2] + 2
    with pack_images([packs[0], bad, packs[2]]) as refs:
        with pytest.raises(_lib.DgxError) as ei:
            sorted_packed(refs, 3, want.size)
    assert ei.value.code == -3


def sorted_packed(refs, k, cap):
    """dgx_intersect_sorted_packed over a PackRef array: the result and the h2d_bytes the call counted."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    out = np.empty(max(cap, 1), np.uint64)
    n = C.c_size_t(0)
    h0 = _lib.stats()["h2d_bytes"]
    _lib.check(lib.dgx_intersect_sorted_packed(refs, k, out.ctypes.data_as(C.c_void_p), cap, C.byref(n)))
    return out[: n.value], _lib.stats()["h2d_bytes"] - h0


def test_intersect_sorted_packed_zero_copy(orc):
    """DGX_ZERO_COPY=1, in a subprocess because libdgx reads its knobs once: pinned packs are decoded in place over
    PCIe, a pageable pack in the same call sends every pack through DMA copies, a malformed pinned pack is refused."""
    import subprocess
    code = r'''
import os, sys
import numpy as np
sys.path.insert(0, os.getcwd()); sys.path.insert(0, os.path.join(os.getcwd(), "tests"))
import gen
import dgraph_b200
from dgraph_b200 import _lib
from oracle import pyoracle as orc
from test_gpu_parity import eq, generic_bytes, pack_images, to_pack
from test_gpu_round2 import sorted_packed
rng = np.random.default_rng(37)
master = gen.zipf_gaps(rng, 300_000)
lists = [gen.thin(rng, master, p) for p in (0.5, 0.6, 0.7)]
packs = [to_pack(dgraph_b200, orc.encode(l, bs)) for l, bs in zip(lists, (256, 10, 256))]
want = orc.intersect_sorted(lists)
with pack_images(packs) as refs:
    got, h2d = sorted_packed(refs, 3, want.size)
    eq(got, want, "pinned")
    # only uid_off is copied; the decode kernel's reads over PCIe are counted: base, NumUids, delta_off, deltas
    assert h2d == sum(28 * p.nblocks + 8 + p.deltas.size for p in packs), h2d
    mixed = (_lib.PackRef * 3)()
    pageable, keep = dgraph_b200.algo._refs_of([packs[1]])
    mixed[0], mixed[1], mixed[2] = refs[0], pageable[0], refs[2]
    got, h2d = sorted_packed(mixed, 3, want.size)
    eq(got, want, "pinned and pageable")
    assert h2d == sum(generic_bytes(p) for p in packs), h2d
bad = dgraph_b200.pb.UidPack(packs[1].block_size, packs[1].base, packs[1].num_uids, packs[1].delta_off.copy(), packs[1].deltas)
bad.delta_off[3] = bad.delta_off[2] + 2
with pack_images([packs[0], bad, packs[2]]) as refs:
    try:
        sorted_packed(refs, 3, want.size)
        raise AssertionError("malformed pinned pack accepted")
    except _lib.DgxError as e:
        assert e.code == -3, e.code
print("ZERO_COPY_OK")
'''
    env = dict(os.environ, DGX_ZERO_COPY="1")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, env=env,
                       cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert "ZERO_COPY_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-4000:]


def test_pack_cache(dgx, orc):
    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(32)
    master = gen.zipf_gaps(rng, 300_000)
    lists = [gen.thin(rng, master, 0.5) for _ in range(4)]
    packs = [to_pack(dgx, orc.encode(l, 256)) for l in lists]
    want = orc.intersect_sorted(lists)
    lib.dgx_cache_clear()
    _lib.check(lib.dgx_cache_configure(1 << 30))
    st = _lib.CacheStats()
    lib.dgx_cache_get_stats(C.byref(st))
    h0, m0 = st.hits, st.misses
    keys = [(1000 + i, 7) for i in range(4)]
    h2d0 = _lib.stats()["h2d_bytes"]
    eq(dgx.algo.IntersectSortedPacks(packs, keys).Uids, want, "cache cold")
    h2d1 = _lib.stats()["h2d_bytes"]
    eq(dgx.algo.IntersectSortedPacks(packs, keys).Uids, want, "cache warm")
    h2d2 = _lib.stats()["h2d_bytes"]
    lib.dgx_cache_get_stats(C.byref(st))
    assert st.misses - m0 == 4 and st.hits - h0 == 4 and st.entries >= 4
    assert h2d1 - h2d0 > sum(p.deltas.size for p in packs)      # the cold call copied the packs
    assert h2d2 - h2d1 < 64 * 1024                               # the warm call copied descriptors only
    # a new version of a key names different bytes: it must not hit the old entry
    lists2 = [gen.thin(rng, master, 0.4) for _ in range(4)]
    packs2 = [to_pack(dgx, orc.encode(l, 256)) for l in lists2]
    eq(dgx.algo.IntersectSortedPacks(packs2, [(1000 + i, 8) for i in range(4)]).Uids, orc.intersect_sorted(lists2), "new version")
    # eviction: a cache that holds about two packs still answers correctly and stays within its budget
    one = lib.dgx_cache_get_stats
    _lib.check(lib.dgx_cache_configure(int(2.5 * packs[0].deltas.size)))
    for rep in range(3):
        eq(dgx.algo.IntersectSortedPacks(packs, [(2000 + i, 1) for i in range(4)]).Uids, want, f"evicting rep {rep}")
    one(C.byref(st))
    assert st.bytes <= st.max_bytes and st.evictions > 0
    # disabled cache: named packs still work (one-shot copies)
    _lib.check(lib.dgx_cache_configure(0))
    eq(dgx.algo.IntersectSortedPacks(packs, keys).Uids, want, "cache disabled")
    one(C.byref(st))
    assert st.entries == 0
    _lib.check(lib.dgx_cache_configure(16 << 30))


def test_pack_cache_concurrent(dgx, orc):
    import threading

    rng = np.random.default_rng(33)
    master = gen.zipf_gaps(rng, 200_000)
    lists = [gen.thin(rng, master, 0.5) for _ in range(6)]
    packs = [to_pack(dgx, orc.encode(l, 256)) for l in lists]
    errs = []

    def work(t):
        try:
            r = np.random.default_rng(t)
            for _ in range(8):
                sel = sorted(r.choice(6, 3, replace=False).tolist())
                got = dgx.algo.IntersectSortedPacks([packs[i] for i in sel], [(3000 + i, 1) for i in sel])
                eq(got.Uids, orc.intersect_sorted([lists[i] for i in sel]), f"thread {t} {sel}")
        except Exception as e:  # noqa: BLE001
            errs.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errs, errs[0]


def test_malformed_pack_refused(dgx, orc):
    from dgraph_b200 import _lib

    u = gen.zipf_gaps(np.random.default_rng(34), 5000)
    good = to_pack(dgx, orc.encode(u, 256))
    eq(dgx.codec.Decode(good, 0), u, "well-formed")
    bad = dgx.pb.UidPack(good.block_size, good.base, good.num_uids, good.delta_off.copy(), good.deltas)
    bad.delta_off[3] = bad.delta_off[2] + 2          # block 2 shorter than its groups need
    with pytest.raises(_lib.DgxError) as ei:
        dgx.codec.Decode(bad, 0)
    assert ei.value.code == -3
    bad2 = dgx.pb.UidPack(good.block_size, good.base, good.num_uids, good.delta_off.copy(), good.deltas)
    bad2.delta_off[5] = bad2.delta_off[4] - 1        # offsets go backwards
    with pytest.raises(_lib.DgxError):
        dgx.codec.Decode(bad2, 0)
    # a call refused on a malformed pack, named or not, releases the cache references it took on the good named
    # packs before it: entries still referenced are never evicted, so a leaked one would survive the clear
    lib = _lib.load()
    for keys in ([(9001, 1), (9002, 1), (9003, 1)], [(9001, 1), (9002, 1), (0, 0)]):
        with pytest.raises(_lib.DgxError) as ei:
            dgx.algo.IntersectSortedPacks([good, good, bad], keys)
        assert ei.value.code == -3
    lib.dgx_cache_clear()
    st = _lib.CacheStats()
    lib.dgx_cache_get_stats(C.byref(st))
    assert st.entries == 0
    # tags that claim more bytes than the block holds: memory-safe, library usable afterwards
    evil = dgx.pb.UidPack(good.block_size, good.base, good.num_uids, good.delta_off, np.full_like(good.deltas, 0xFF))
    out = dgx.codec.Decode(evil, 0)
    assert out.size == u.size
    eq(dgx.codec.Decode(good, 0), u, "after corrupt input")
    # deltas summing past 2^32 inside one block follow the reference's 64-bit running sum (codec.go:191-196)
    base = np.array([5], np.uint64)
    num = np.array([9], np.uint32)
    deltas = np.array([0xFF] + [0xFF] * 16 + [0xFF] + [0xFF] * 16, np.uint8)
    p = dgx.pb.UidPack(256, base, num, np.array([0, deltas.size], np.uint64), deltas)
    want = 5 + np.arange(9, dtype=np.uint64) * np.uint64(0xFFFFFFFF)
    eq(dgx.codec.Decode(p, 0), want, "64-bit running sum")


# ---- IndexOf batch, shared-list batch ----------------------------------------------------------------

def test_index_of_batch(dgx, orc):
    rng = np.random.default_rng(35)
    for n, m in ((0, 10), (1, 5), (1000, 0), (1000, 3000), (300_000, 200_000), (5, 100_000)):
        u = gen.uniform_unique(rng, n, max(4 * n, 16))
        q = rng.integers(0, max(4 * n, 16) + 3, m, dtype=np.uint64)       # unsorted probes, ~25 % hits
        if n and m:
            q[:: 7] = u[rng.integers(0, n, q[::7].size)]
        got = dgx.algo.IndexOfBatch(L(dgx, u), q)
        want = np.array([orc.index_of(u, int(x)) for x in q[:2000]], dtype=np.int64)
        assert np.array_equal(got[: want.size], want), f"IndexOf n={n} m={m}"
        if n:
            pos = np.searchsorted(u, q)
            ok = (pos < n) & (u[np.minimum(pos, n - 1)] == q)
            assert np.array_equal(got, np.where(ok, pos, -1)), f"IndexOf n={n} m={m} (all)"
        else:
            assert np.all(got == -1)
    # duplicates in u: sort.Search finds the first copy
    u = np.array([1, 3, 3, 3, 9, 9], np.uint64)
    assert dgx.algo.IndexOfBatch(L(dgx, u), [3, 9, 1, 2]).tolist() == [1, 4, 0, -1]


def test_intersect_batch_shared(dgx, orc):
    rng = np.random.default_rng(36)
    master = gen.zipf_gaps(rng, 500_000)
    dest = gen.thin(rng, master, 0.3)
    rows = [gen.thin(rng, master, float(p)) for p in rng.uniform(0.0005, 0.2, 200)] + [np.zeros(0, np.uint64), dest.copy()]
    a = np.concatenate(rows)
    a_off = np.concatenate([[0], np.cumsum([r.size for r in rows])]).astype(np.uint64)
    out, off = dgx.algo.IntersectBatchShared(a, a_off, dest)
    for i, r in enumerate(rows):
        eq(out[int(off[i]): int(off[i + 1])], orc.intersect_with(r, dest), f"shared row {i}")
    out, off = dgx.algo.IntersectBatchShared(a, a_off, np.zeros(0, np.uint64))
    assert out.size == 0 and np.all(off == 0)


# ---- BASELINE configs at full size --------------------------------------------------------------------

def test_config3_full(dgx, orc):
    """configs[2]: codec.Decode(UidPack blockSize=256) of 1e8 UIDs -> IntersectSorted([decoded, L1, L2])."""
    rng = np.random.default_rng(301)
    master = gen.zipf_gaps(rng, 100_000_000)
    pack = orc.encode(master, 256)
    assert orc.exact_len(pack) == master.size
    p = to_pack(dgx, pack)
    dec = dgx.codec.Decode(p, 0)
    same(dec, master, "C3 decode 1e8")          # round trip == oracle decode (checked below on a seek)
    l1 = gen.thin(np.random.default_rng(302), master, 0.1)
    l2 = gen.thin(np.random.default_rng(303), master, 0.01)
    got = dgx.codec.DecodeIntersectSorted(p, 0, [L(dgx, l1), L(dgx, l2)])
    same(got.Uids, orc.intersect_sorted([master, l1, l2]), "C3 pipeline")
    seek = int(master[60_000_000]) + 1
    same(dgx.codec.Decode(p, seek), orc.decode(pack, seek), "C3 decode from seek")
    o = dgx.pb.List(None)
    dgx.algo.IntersectCompressedWith(p, seek, L(dgx, l2), o)
    same(o.Uids, orc.intersect_compressed_with(pack, seek, l2), "C3 IntersectCompressedWith")


def c4_pairs(npairs, seed=401):
    """configs[3] (SURVEY 8d): sizes i.i.d. truncated power law alpha=2 on [1e4, 1e6]; each pair two
    thinnings (p=0.5) of a Zipf-gap master -- here a random window of one shared 4e6 master (drawing
    10k separate masters would take minutes on the host), re-based per pair."""
    rng = np.random.default_rng(seed)
    lo, hi = 1e4, 1e6
    uu = rng.random(npairs)
    sizes = (1.0 / (1.0 / lo - uu * (1.0 / lo - 1.0 / hi))).astype(np.int64)   # inverse CDF of x^-2 on [lo, hi]
    big = gen.zipf_gaps(np.random.default_rng(seed + 1), 4_000_000)
    a_rows, b_rows = [], []
    for n in sizes:
        w = int(min(2 * n, big.size))
        s0 = int(rng.integers(0, big.size - w + 1))
        win = big[s0: s0 + w]
        bits = np.unpackbits(np.frombuffer(rng.bytes((2 * w + 7) // 8), dtype=np.uint8))   # p = 0.5 coin flips
        a_rows.append(win[bits[:w].view(bool)])
        b_rows.append(win[bits[w: 2 * w].view(bool)])
    return a_rows, b_rows


def test_config4_full(dgx, orc):
    """configs[3]: 10k independent 2-way intersections, 1e4-1e6 UIDs each, one batched call."""
    a_rows, b_rows = c4_pairs(10_000)
    a = np.concatenate(a_rows)
    b = np.concatenate(b_rows)
    a_off = np.concatenate([[0], np.cumsum([r.size for r in a_rows])]).astype(np.uint64)
    b_off = np.concatenate([[0], np.cumsum([r.size for r in b_rows])]).astype(np.uint64)
    out, off = dgx.algo.IntersectBatch(a, a_off, b, b_off)
    want = [orc.intersect_with(x, y) for x, y in zip(a_rows, b_rows)]
    want_off = np.concatenate([[0], np.cumsum([w.size for w in want])]).astype(np.uint64)
    assert np.array_equal(off, want_off), "C4 CSR offsets"
    same(out, np.concatenate(want), "C4 values")


def test_config5_full(dgx, orc):
    """configs[4]: MergeSorted of k=64 lists (lengths ~ 1/rank, sum 1e8, thinnings of a 2e8 master) then
    Difference against a 1e7 thinning."""
    rng = np.random.default_rng(501)
    master = gen.zipf_gaps(rng, 200_000_000)
    w = 1.0 / np.arange(1, 65)
    lens = (w / w.sum() * 1e8).astype(np.int64)
    # a thinning of the master with about n survivors, drawn as sorted distinct random positions (64
    # Bernoulli passes over 2e8 values would take minutes on the host)
    lists = [master[np.unique(rng.integers(0, master.size, int(n)))] for n in lens]
    merged = dgx.algo.MergeSorted([L(dgx, l) for l in lists])
    want = orc.merge_sorted(lists)
    same(merged.Uids, want, "C5 MergeSorted")
    d = gen.thin(np.random.default_rng(502), master, 0.05)
    got = dgx.algo.Difference(merged, L(dgx, d))
    same(got.Uids, orc.difference(want, d), "C5 Difference")


# ---- Decoder seeks on the device (codec_test.go:113-217) ------------------------------------------------

def test_device_seek_tables(dgx, orc):
    from test_oracle_codec import SEEK_TABLE, make_seek_pack

    opack = make_seek_pack(orc)
    dec = dgx.codec.Decoder(to_pack(dgx, opack))
    ref = orc.Decoder(opack)
    # TestSeek :125-151 -- same table the oracle is pinned with, and the oracle's answer call by call
    for uid, out, whence, empty in SEEK_TABLE:
        uids = dec.Seek(uid, whence)
        want = ref.seek(uid, whence)
        eq(uids, want, f"Seek({uid},{whence})")
        assert dec.BlockIdx() == ref.block_idx
        if empty:
            assert uids.size == 0
        else:
            assert int(uids[0]) == out
    # :153-157
    dec.blockIdx = 0
    ref.block_idx = 0
    for i in range(100, 10000, 100):
        got = dec.LinearSeek(i)
        eq(got, ref.linear_seek(i), f"LinearSeek({i})")
        assert i in got.tolist()
    # TestLinearSeek :160-187
    dec = dgx.codec.Decoder(to_pack(dgx, opack))
    ref = orc.Decoder(opack)
    N = 10001
    for i in range(0, 2 * N, 130):
        got = dec.LinearSeek(i)
        eq(got, ref.linear_seek(i), f"LinearSeek({i})")
        assert (i in got.tolist()) == (i < N)
        assert dec.BlockIdx() == ref.block_idx
    for i in range(0, 9990, 370):   # blockIdx now points at the last block
        assert i not in dec.LinearSeek(i).tolist()
    # TestDecoder :190-217
    expected = np.arange(3, N, 3, dtype=np.uint64)
    p3 = orc.encode(expected, 10)
    dec = dgx.codec.Decoder(to_pack(dgx, p3))
    for i in range(3, N, 3 * 97):
        for d in (0, 1, 2):
            assert int(dec.Seek(i - d, dgx.codec.SeekStart)[0]) == i
        assert int(dec.Seek(i, dgx.codec.SeekCurrent)[0]) == i + 3 if i + 3 < N else True
    # SeekToBlock / LinearSeek / Next / UnpackBlock against the oracle, call by call, the block index carried over.
    # (Seek is left out of the walk: it trims the current slice, and the reference's SeekToBlock reuses a trimmed
    # slice when the block does not change, codec.go:262-264 -- state the one-call device form does not carry.)
    dec = dgx.codec.Decoder(to_pack(dgx, opack))
    ref = orc.Decoder(opack)
    dec.UnpackBlock()
    ref.unpack_block()
    rng = np.random.default_rng(40)
    for step in range(300):
        kind = int(rng.integers(0, 4))
        uid = int(rng.integers(0, 10400))
        wh = int(rng.integers(0, 2))
        if not ref.valid():
            dec.blockIdx = ref.block_idx = 0
            dec.UnpackBlock()
            ref.unpack_block()
        if kind == 0:
            got, want = dec.SeekToBlock(uid, wh), ref.seek_to_block(uid, wh)
        elif kind == 1:
            got, want = dec.LinearSeek(uid), ref.linear_seek(uid)
        elif kind == 2:
            got, want = dec.Next(), ref.next()
        else:
            got, want = dec.UnpackBlock(), ref.unpack_block()
        eq(got, want, f"step {step} kind {kind} uid {uid} whence {wh}")
        assert dec.BlockIdx() == ref.block_idx, (step, kind, uid, wh)
    # nil pack
    d0 = dgx.codec.Decoder(None)
    assert d0.Seek(5, 0).size == 0 and d0.LinearSeek(5).size == 0 and not d0.Valid()


def test_intersect_compressed_fused(dgx, orc):
    """The fused block-skipping kernel in both range-search regimes (m < nblocks: bases searched with v;
    m >= nblocks: v searched with the bases), both probe directions, sparse and dense v, afterUID seeks,
    non-reference block sizes (oversize slow path) and the named-pack form."""
    import ctypes as C
    from dgraph_b200 import _lib

    rng = np.random.default_rng(41)
    u = gen.zipf_gaps(rng, 2_000_000)
    pack = orc.encode(u, 256)
    p = to_pack(dgx, pack)
    cases = [gen.thin(rng, u, 1e-4), gen.thin(rng, u, 0.02), gen.thin(rng, u, 0.9),
             np.unique(np.concatenate([gen.thin(rng, u, 0.001), rng.integers(0, int(u[-1]) + 1000, 5000, dtype=np.uint64)])),
             u.copy(), u[:1], u[-1:], np.array([0], np.uint64), np.array([int(u[-1]) + 1], np.uint64)]
    dense = np.unique(np.concatenate([u[1000:200000], np.arange(int(u[1000]), int(u[1000]) + 3_000_000, 3, dtype=np.uint64)]))
    cases.append(dense)   # slices of v far longer than a block: the row probes the slice
    for ci, v in enumerate(cases):
        for after in (0, int(u[u.size // 3]), int(u[u.size // 3]) + 1, int(u[-1])):
            o = dgx.pb.List(None)
            dgx.algo.IntersectCompressedWith(p, after, L(dgx, v), o)
            eq(o.Uids, orc.intersect_compressed_with(pack, after, v), f"case {ci} after {after}")
        # afterUID beyond the last uid: Seek runs off the pack (blockIdx == len(Blocks)) and the reference's Bin branch
        # then indexes Blocks[blockIdx] (algo/uidlist.go:118 -> codec.go:231), a panic in Go; nothing is >= afterUID,
        # so the device answer is the empty list
        o = dgx.pb.List(None)
        dgx.algo.IntersectCompressedWith(p, int(u[-1]) + 1, L(dgx, v), o)
        assert o.Uids is not None and o.Uids.size == 0
    for bs in (1, 7, 100, 1000, 5000):
        w = gen.zipf_gaps(rng, 60_000)
        pk = orc.encode(w, bs)
        for v in (gen.thin(rng, w, 0.3), gen.thin(rng, w, 0.003)):
            o = dgx.pb.List(None)
            dgx.algo.IntersectCompressedWith(to_pack(dgx, pk), int(w[100]), L(dgx, v), o)
            eq(o.Uids, orc.intersect_compressed_with(pk, int(w[100]), v), f"bs {bs}")
    # named pack: second call hits the cache
    lib = _lib.load()
    lib.dgx_cache_clear()
    v = gen.thin(rng, u, 0.01)
    pn = p.normalized()
    view = dgx.codec.view_of(pn)
    ref = _lib.PackRef(C.pointer(view), 777, 3)
    out = np.empty(v.size, np.uint64)
    n = C.c_size_t(0)
    st = _lib.CacheStats()
    for rep in range(2):
        _lib.check(lib.dgx_intersect_compressed_ref(C.byref(ref), 0, v.ctypes.data_as(C.c_void_p), v.size,
                                                    out.ctypes.data_as(C.c_void_p), v.size, C.byref(n)))
        eq(out[: n.value], orc.intersect_compressed_with(pack, 0, v), f"named rep {rep}")
    lib.dgx_cache_get_stats(C.byref(st))
    assert st.hits >= 1
    lib.dgx_cache_clear()


# ---- codec.Encode on the device, packed set operations (algo/packed.go) ------------------------------------

def same_pack(got, want, what):
    """device pack == oracle pack, array by array (bytes included)."""
    if want.is_nil:
        assert got is None, what
        return
    assert got is not None, what
    assert got.block_size == want.block_size, what
    eq(got.base, want.base, what + " base")
    assert np.array_equal(got.num_uids, want.num_uids), what + " num_uids"
    eq(got.delta_off, want.delta_off, what + " delta_off")
    assert np.array_equal(got.deltas, want.deltas), what + " deltas"


def test_encode_matches_oracle_bytes(dgx, orc):
    rng = np.random.default_rng(50)
    same_pack(dgx.codec.Encode(np.zeros(0, np.uint64), 256), orc.encode(np.zeros(0, np.uint64), 256), "empty")
    for bs in (0, 1, 2, 5, 10, 100, 256, 257, 1000):
        for n in (1, 2, 4, 5, 9, 255, 256, 257, 1000, 5003):
            for u in (gen.get_uids(rng, n), gen.zipf_gaps(rng, n)):
                same_pack(dgx.codec.Encode(u, bs), orc.encode(u, bs), f"bs {bs} n {n}")
    for shift in (7, 8, 15, 16, 23, 24, 31):       # every delta width
        g = rng.integers(1, 1 << shift, 4000, dtype=np.uint64) + np.uint64(1 << shift)
        u = np.cumsum(g, dtype=np.uint64)
        same_pack(dgx.codec.Encode(u, 256), orc.encode(u, 256), f"shift {shift}")
    # ~50,000 upper-word changes: with BlockSize 10 the segments overflow the bound's arrays (one retry)
    wide = np.cumsum(rng.integers(1, 1 << 31, 200_000, dtype=np.uint64), dtype=np.uint64)
    same_pack(dgx.codec.Encode(wide, 256), orc.encode(wide, 256), "msb splits")
    same_pack(dgx.codec.Encode(wide, 10), orc.encode(wide, 10), "msb splits bs 10")
    scattered = np.sort(rng.integers(0, 2**64 - 1, 5000, dtype=np.uint64))                  # a new block per uid: > 64 splits
    same_pack(dgx.codec.Encode(scattered, 256), orc.encode(scattered, 256), "every uid its own segment")
    d = gen.with_dups(rng, 3000, 2000)
    same_pack(dgx.codec.Encode(d, 256), orc.encode(d, 256), "duplicates (zero deltas)")
    big = gen.zipf_gaps(rng, 20_000_000)
    p = dgx.codec.Encode(big, 256)
    same_pack(p, orc.encode(big, 256), "2e7")
    eq(dgx.codec.Decode(p, 0), big, "encode -> decode round trip")
    # TestEncoding :306-334 MSB-split shapes
    bigs = [0xF000000000000000, 0xF00F000000000000, 0x00F00F0000000000, 0x000F0F0000000000, 0x0F0F0F0F00000000]
    for n in (0, 1, 2, 3, 5, 13, 18, 100, 99, 98):
        ints = np.zeros(n, dtype=np.uint64)
        for i in range(min(50, n)):
            ints[i] = rng.integers(0, 2**32)
        for i in range(50, n):
            ints[i] = int(rng.integers(0, 2**32)) + bigs[int(rng.integers(0, 5))]
        ints.sort()
        same_pack(dgx.codec.Encode(ints, 256), orc.encode(ints, 256), f"TestEncoding n={n}")


def test_packed_ops_reference_cases(dgx, orc):
    """Every known-answer case of algo/packed_test.go through the device packed operations (BlockSize 5 like
    newUidPack, packed_test.go:18-25), result decoded with the ORACLE's decoder."""
    from test_oracle_packed import DIFF_PACKED, INTERSECT_PACKED, INTERSECT_SORTED_PACKED, MERGE_PACKED

    def mk(data):
        return to_pack(dgx, orc.encode(np.asarray(data, dtype=np.uint64), 5))

    def dec(p):
        return [] if p is None else dgx.codec.Decode(p, 0).tolist()

    for lists, want in MERGE_PACKED:
        assert dec(dgx.algo.MergeSortedPacked([mk(l) for l in lists], 5)) == want, lists
    for u, v, want in INTERSECT_PACKED:
        assert dec(dgx.algo.IntersectWithLinPacked(mk(u), mk(v), 5)) == want, (u, v)
    for lists, want in INTERSECT_SORTED_PACKED:
        assert dec(dgx.algo.IntersectSortedPacked([mk(l) for l in lists], 5)) == want, lists
    for u, v, want in DIFF_PACKED:
        assert dec(dgx.algo.DifferencePacked(mk(u), mk(v), 5)) == want, (u, v)


def test_packed_ops_random(dgx, orc):
    rng = np.random.default_rng(51)
    master = gen.zipf_gaps(rng, 600_000)
    lists = [gen.thin(rng, master, float(p)) for p in (0.5, 0.3, 0.7, 0.05)]
    packs = [to_pack(dgx, orc.encode(l, 256)) for l in lists]
    same_pack(dgx.algo.IntersectWithLinPacked(packs[0], packs[1]), orc.encode(orc.intersect_with(lists[0], lists[1]), 256), "IntersectWithLinPacked")
    same_pack(dgx.algo.DifferencePacked(packs[0], packs[1]), orc.encode(orc.difference(lists[0], lists[1]), 256), "DifferencePacked")
    same_pack(dgx.algo.MergeSortedPacked(packs), orc.encode(orc.merge_sorted(lists), 256), "MergeSortedPacked")
    same_pack(dgx.algo.IntersectSortedPacked(packs), orc.encode(orc.intersect_sorted(lists), 256), "IntersectSortedPacked")
    same_pack(dgx.algo.IntersectWithLinPacked(packs[0], None), orc.encode(np.zeros(0, np.uint64), 256), "nil operand")
    same_pack(dgx.algo.DifferencePacked(packs[0], None), orc.encode(lists[0], 256), "minus nil")
    same_pack(dgx.algo.MergeSortedPacked([None, packs[3], None]), orc.encode(lists[3], 256), "merge with nils")


# ---- filter_pipe 32-bit fast path: geometry stress ------------------------------------------------------------

def test_filter_fast_path_stress(dgx, orc):
    """Many small random queries aimed at the fast path's corners: slice lengths around powers of two and far apart
    (one ladder for several lists needs P <= n <= 3P), empty slices in the middle of a chain, tiles that straddle a
    multiple of 2^32 (must fall back to 64-bit searches), single-row and multi-row warps, Difference, both tile
    geometries (k = 2 -> 1024-value tiles, k >= 3 -> 512)."""
    rng = np.random.default_rng(60)
    bases = [0, (1 << 32) - 40_000, (1 << 32) - 300, (7 << 32) + 123, (1 << 63) + 17, (1 << 64) - 2_000_000]
    for it in range(160):
        base = bases[it % len(bases)]
        k = int(rng.integers(2, 10))
        span = int(rng.choice([3_000, 40_000, 600_000]))
        master = np.unique(rng.integers(0, span, int(rng.integers(50, 9000)), dtype=np.uint64)) + np.uint64(base)
        lists = []
        for j in range(k):
            p = float(rng.choice([0.02, 0.2, 0.5, 0.9, 1.0]))
            l = master[rng.random(master.size) < p]
            if rng.random() < 0.15:        # a list that misses a whole stretch: empty slices for some tiles
                cut = master[master.size // 3], master[2 * master.size // 3]
                l = l[(l < cut[0]) | (l > cut[1])]
            if rng.random() < 0.1:         # a much longer list (different ladder length than its neighbours)
                l = np.unique(np.concatenate([l, rng.integers(0, span, 20_000, dtype=np.uint64) + np.uint64(base)]))
            lists.append(l)
        got = dgx.algo.IntersectSorted([L(dgx, l) for l in lists])
        eq(got.Uids, orc.intersect_sorted(lists), f"stress {it} k={k} base={base:#x}")
        d = dgx.algo.Difference(L(dgx, lists[0]), L(dgx, lists[1]))
        eq(d.Uids, orc.difference(lists[0], lists[1]), f"stress diff {it}")
    # one batch mixing widths (the batch runs the geometry of its widest query)
    rows_a, rows_b = [], []
    for it in range(40):
        m = np.unique(rng.integers(0, 1 << 20, int(rng.integers(0, 5000)), dtype=np.uint64)) + np.uint64(bases[it % 4])
        rows_a.append(m[rng.random(m.size) < 0.6])
        rows_b.append(m[rng.random(m.size) < 0.4])
    a = np.concatenate(rows_a + [np.zeros(0, np.uint64)])
    b = np.concatenate(rows_b + [np.zeros(0, np.uint64)])
    a_off = np.concatenate([[0], np.cumsum([r.size for r in rows_a])]).astype(np.uint64)
    b_off = np.concatenate([[0], np.cumsum([r.size for r in rows_b])]).astype(np.uint64)
    out, off = dgx.algo.IntersectBatch(a, a_off, b, b_off)
    for i in range(40):
        eq(out[int(off[i]): int(off[i + 1])], orc.intersect_with(rows_a[i], rows_b[i]), f"batch row {i}")


def one_list(rng, n, where):
    """n sorted values with runs of equal values across every multiple of 512 (both tile sizes), placed low, straddling
    2^32, or ending at 2^64 - 1."""
    i = np.arange(n)
    gaps = rng.choice(np.array([0, 1, 7, 1000], np.uint64), n, p=[0.2, 0.4, 0.3, 0.1])
    gaps[(i % 512 >= 506) | (i % 512 < 6)] = 0
    span = int(gaps.sum(dtype=np.uint64))
    lo = {"low": 3, "2^32": (1 << 32) - span // 2, "top": (1 << 64) - 1 - span}[where]
    return np.uint64(lo) + np.cumsum(gaps, dtype=np.uint64)


def test_filter_one_list_queries(dgx, orc):
    """Queries of one list (IntersectSorted of one list is a copy) run the pipeline without a plan: alone in a batch
    (tile table + pipeline, two launches), mixed with wider queries, over a capacity one short, and on a resident-inputs
    lane reading the previous batch's output."""
    import torch
    from dgraph_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(90)
    # ---- host form: one list around the 1024-value tile size, and a long one
    for n in (1, 1023, 1024, 1025, 3_000_000):
        for where in ("low", "2^32", "top"):
            l = one_list(rng, n, where)
            before = _lib.stats()["kernel_launches"]
            got = dgx.algo.IntersectSorted([L(dgx, l)])
            assert _lib.stats()["kernel_launches"] - before == 2, f"launches, n={n} {where}"
            eq(got.Uids, orc.intersect_sorted([l]), f"IntersectSorted of one list, n={n} {where}")

    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(stream):
        lane = lib.dgx_lane_create(0, C.c_void_p(stream.cuda_stream))
        assert lane

        def run(queries, cap, op=0, out=None):
            """queries: lists of numpy lists, each copied into its own device buffer.  Returns (out, off, inputs);
            the input tensors must stay alive until the lane is synchronised."""
            flat = [torch.from_numpy(np.concatenate([l, np.zeros(2, np.uint64)]).view(np.int64)).to(dev)
                    for q in queries for l in q]
            lens = [l.size for q in queries for l in q]
            koff = np.concatenate([[0], np.cumsum([len(q) for q in queries])])
            if out is None:
                out = torch.full((cap + 8,), -1, dtype=torch.int64, device=dev)
            off = torch.zeros(len(queries) + 1, dtype=torch.int64, device=dev)
            _lib.check(lib.dgx_dev_filter_batch(lane, op, (C.c_void_p * len(flat))(*[t.data_ptr() for t in flat]),
                                                (C.c_size_t * len(lens))(*lens),
                                                (C.c_size_t * len(koff))(*[int(x) for x in koff]), len(queries),
                                                C.c_void_p(out.data_ptr()), cap, C.c_void_p(off.data_ptr())))
            return out, off, flat

        # ---- device form: ~1000 one-list queries, some empty: one tile-table launch + one pipeline launch
        qs = []
        for q in range(1000):
            n = 0 if q % 9 == 0 else int(rng.integers(1, 3000))
            qs.append([one_list(rng, n, ("low", "2^32", "top")[q % 3])])
        total = sum(q[0].size for q in qs)
        before = lib.dgx_lane_launches(lane)
        out, off, keep = run(qs, total)
        assert lib.dgx_lane_launches(lane) - before == 2
        _lib.check(lib.dgx_lane_sync(lane))
        ho, hoff = out.cpu().numpy().view(np.uint64), off.cpu().numpy().view(np.uint64)
        eq(hoff, np.concatenate([[0], np.cumsum([q[0].size for q in qs])]), "out_off of one-list queries")
        eq(ho[:total], np.concatenate([orc.intersect_sorted(q) for q in qs]), "out of one-list queries")

        # ---- one batch mixing k = 1, 2 and 5 (512-value tiles, with a plan for the wider queries)
        master = gen.zipf_gaps(rng, 200_000, start=(1 << 32) - 600_000)
        mixed = []
        for q in range(60):
            k = (1, 2, 5)[q % 3]
            lists = [gen.thin(rng, master, float(rng.choice([0.3, 0.9]))) for _ in range(k)]
            if q % 7 == 0:
                lists[0] = np.sort(np.concatenate([lists[0], lists[0][::5]]))   # repeated values
            mixed.append(lists)
        cap = sum(min(l.size for l in lists) for lists in mixed)
        out, off, keep = run(mixed, cap)
        _lib.check(lib.dgx_lane_sync(lane))
        ho, hoff = out.cpu().numpy().view(np.uint64), off.cpu().numpy()
        for qi, lists in enumerate(mixed):
            eq(ho[int(hoff[qi]): int(hoff[qi + 1])], orc.intersect_sorted(lists), f"mixed batch query {qi} k={len(lists)}")

        # ---- out_cap one short: the sync reports it and nothing lands past out_cap
        qs = [[one_list(rng, n, "2^32")] for n in (700, 1024, 2500)]
        total = sum(q[0].size for q in qs)
        out, off, keep = run(qs, total - 1)
        assert lib.dgx_lane_sync(lane) == -4  # DGX_ERR_CAP
        assert (out[total - 1:].cpu() == -1).all(), "a value was written past out_cap"

        # ---- resident-inputs lane: a one-list batch whose list is the previous batch's output on the lane
        _lib.check(lib.dgx_lane_set_resident_inputs(lane, 1))
        a, b = gen.thin(rng, master, 0.8), gen.thin(rng, master, 0.7)
        want = orc.intersect_sorted([a, b])
        da = torch.from_numpy(np.concatenate([a, np.zeros(2, np.uint64)]).view(np.int64)).to(dev)
        db = torch.from_numpy(np.concatenate([b, np.zeros(2, np.uint64)]).view(np.int64)).to(dev)
        garbage = torch.arange(a.size + 8, 0, -1, dtype=torch.int64, device=dev) * 977
        mid = garbage.clone()
        mid_off = torch.zeros(2, dtype=torch.int64, device=dev)
        fin = torch.empty(a.size + 8, dtype=torch.int64, device=dev)
        fin_off = torch.zeros(2, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()

        def batch(lists, lens, o, o_off):
            n = len(lists)
            _lib.check(lib.dgx_dev_filter_batch(lane, 0, (C.c_void_p * n)(*[t.data_ptr() for t in lists]),
                                                (C.c_size_t * n)(*lens), (C.c_size_t * 2)(0, n), 1,
                                                C.c_void_p(o.data_ptr()), a.size, C.c_void_p(o_off.data_ptr())))

        for rep in range(3):
            if rep:
                mid.copy_(garbage)
            batch([da, db], [a.size, b.size], mid, mid_off)
            batch([mid], [want.size], fin, fin_off)  # the length is known here only because the test knows the answer
            _lib.check(lib.dgx_lane_sync(lane))
            eq(fin[: int(fin_off[1].item())].cpu().numpy().view(np.uint64), want, f"intersect -> one-list batch, rep {rep}")
        _lib.check(lib.dgx_lane_set_resident_inputs(lane, 0))
        lib.dgx_lane_destroy(lane)


# ---- resident-inputs lanes: the pre-pass of batch i+1 under the pipeline kernel of batch i -------------------------

def test_resident_lane_batches(dgx, orc):
    """dgx_lane_set_resident_inputs: batches queued back to back on one lane (their plan pre-pass runs ahead on a side
    stream, under the previous batch's pipeline kernel; tables alternate between two workspaces).  Every batch is checked against the
    oracle: wide queries, 2-list batches, Difference, duplicates repeated across tile boundaries, empty lists."""
    import torch
    from dgraph_b200 import _lib

    lib = _lib.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(stream):
        lane = lib.dgx_lane_create(0, C.c_void_p(stream.cuda_stream))
        assert lane
        _lib.check(lib.dgx_lane_set_resident_inputs(lane, 1))
        rng = np.random.default_rng(70)
        master = gen.zipf_gaps(rng, 700_000)
        dups = np.sort(rng.integers(0, 3000, 200_000, dtype=np.uint64))          # long runs of equal values
        batches = []
        for b in range(9):
            op = 1 if b % 4 == 3 else 0
            qs = []
            for q in range(int(rng.integers(1, 6))):
                if op == 1:
                    k = 2
                elif b % 3 == 0:
                    k = 2
                else:
                    k = int(rng.integers(3, 9))
                if b == 5:
                    src = dups
                    lists = [src[rng.random(src.size) < float(rng.choice([0.3, 0.7]))] for _ in range(k)]
                else:
                    lists = [gen.thin(rng, master, float(rng.choice([0.02, 0.3, 0.9]))) for _ in range(k)]
                if b == 7 and q == 0:
                    lists[1] = np.zeros(0, np.uint64)
                qs.append(lists)
            batches.append((op, qs))
        # everything resident BEFORE the first call
        dev_lists = [[[torch.from_numpy(l.view(np.int64).copy()).to(dev) for l in lists] for lists in qs] for _, qs in batches]
        outs = []
        for (op, qs), dls in zip(batches, dev_lists):
            cap = sum((lists[0].size if op == 1 else min(l.size for l in lists)) for lists in qs)
            outs.append((torch.empty(cap + 8, dtype=torch.int64, device=dev), torch.zeros(len(qs) + 1, dtype=torch.int64, device=dev), cap))
        torch.cuda.synchronize()
        for rep in range(3):                                                      # back to back, no sync in between
            for (op, qs), dls, (o, off, cap) in zip(batches, dev_lists, outs):
                flat = [t for lists in dls for t in lists]
                koff = np.concatenate([[0], np.cumsum([len(l) for l in dls])])
                ptrs = (C.c_void_p * len(flat))(*[t.data_ptr() for t in flat])
                lens = (C.c_size_t * len(flat))(*[t.numel() for t in flat])
                ck = (C.c_size_t * len(koff))(*[int(x) for x in koff])
                _lib.check(lib.dgx_dev_filter_batch(lane, op, ptrs, lens, ck, len(qs), C.c_void_p(o.data_ptr()), cap,
                                                    C.c_void_p(off.data_ptr())))
        _lib.check(lib.dgx_lane_sync(lane))
        for bi, ((op, qs), (o, off, cap)) in enumerate(zip(batches, outs)):
            ho, hoff = o.cpu().numpy().view(np.uint64), off.cpu().numpy()
            for qi, lists in enumerate(qs):
                want = orc.difference(lists[0], lists[1]) if op == 1 else orc.intersect_sorted(lists)
                eq(ho[int(hoff[qi]): int(hoff[qi + 1])], want, f"resident batch {bi} query {qi} op {op}")
        _lib.check(lib.dgx_lane_set_resident_inputs(lane, 0))
        lib.dgx_lane_destroy(lane)


def test_resident_lane_chains(dgx, orc):
    """A resident-inputs lane whose batches READ what the lane's own queued calls write: Decode -> IntersectSorted and
    intersection -> intersection chains, no synchronisation in between, the intermediate buffers holding descending
    garbage beforehand (a plan taken from it would have r0 > r1).  The lane recognises its own outputs by address and
    plans such a batch behind the producer instead of ahead of it."""
    import torch
    from dgraph_b200 import _lib

    lib = _lib.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(stream):
        lane = lib.dgx_lane_create(0, C.c_void_p(stream.cuda_stream))
        assert lane
        _lib.check(lib.dgx_lane_set_resident_inputs(lane, 1))
        rng = np.random.default_rng(81)
        master = gen.zipf_gaps(rng, 900_000)
        a = gen.thin(rng, master, 0.8)
        others = [gen.thin(rng, master, 0.7) for _ in range(4)]
        pack = to_pack(dgx, orc.encode(a, 256))
        view = dgx.codec.view_of(pack)
        pk = C.c_void_p()
        _lib.check(lib.dgx_dev_pack_upload(lane, C.byref(view), C.byref(pk)))
        d_oth = [torch.from_numpy(l.view(np.int64).copy()).to(dev) for l in others]
        garbage = torch.arange(a.size + 8, 0, -1, dtype=torch.int64, device=dev) * 977
        dec = garbage.clone()
        dec_len = torch.zeros(1, dtype=torch.int64, device=dev)
        mid = garbage.clone()                      # result of the first intersection = first list of the second
        mid_off = torch.zeros(2, dtype=torch.int64, device=dev)
        fin = torch.empty(a.size + 8, dtype=torch.int64, device=dev)
        fin_off = torch.zeros(2, dtype=torch.int64, device=dev)
        want_mid = orc.intersect_sorted([a, others[0], others[1]])
        want_fin = orc.intersect_sorted([want_mid, others[2], others[3]])
        torch.cuda.synchronize()

        def batch(lists, lens, out, off):
            n = len(lists)
            _lib.check(lib.dgx_dev_filter_batch(lane, 0, (C.c_void_p * n)(*[t.data_ptr() for t in lists]), (C.c_size_t * n)(*lens),
                                                (C.c_size_t * 2)(0, n), 1, C.c_void_p(out.data_ptr()), a.size, C.c_void_p(off.data_ptr())))

        for rep in range(4):
            if rep:                                 # garbage again, ordered on the lane's stream
                dec.copy_(garbage)
                mid.copy_(garbage)
            _lib.check(lib.dgx_dev_decode(lane, pk, 0, C.c_void_p(dec.data_ptr()), a.size, C.c_void_p(dec_len.data_ptr())))
            batch([dec, d_oth[0], d_oth[1]], [a.size, others[0].size, others[1].size], mid, mid_off)
            # the second batch reads `mid`; its length is known here only because the test knows the answer
            batch([mid, d_oth[2], d_oth[3]], [want_mid.size, others[2].size, others[3].size], fin, fin_off)
            torch.cuda.current_stream().synchronize()
            eq(mid[: int(mid_off[1].item())].cpu().numpy().view(np.uint64), want_mid, f"decode -> intersect, rep {rep}")
            eq(fin[: int(fin_off[1].item())].cpu().numpy().view(np.uint64), want_fin, f"intersect -> intersect, rep {rep}")
        _lib.check(lib.dgx_lane_sync(lane))
        lib.dgx_dev_pack_free(pk)
        _lib.check(lib.dgx_lane_set_resident_inputs(lane, 0))
        lib.dgx_lane_destroy(lane)
