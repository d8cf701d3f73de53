"""dgx_decode_to_buffer_rows / dgx_encode_from_buffer_rows and their device forms on the H100, checked byte for byte
against the oracle's codec.DecodeToBuffer / codec.EncodeFromBuffer (tests/backup_codec_oracle.c): edge packs and
streams, nil and empty rows, a block with NumUids 0, named and anonymous packs, sizing and capacity, every error found
by the kernels, launch counts that do not depend on the batch, and concurrent callers."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import backup_codec_cases as cases  # noqa: E402
import backup_codec_oracle as bco  # noqa: E402
import gen  # noqa: E402

pytestmark = pytest.mark.gpu
ERR_ARG, ERR_CAP = -3, -4


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _rows(bs, rng):
    """HandPacks (None: nil) covering every edge, and the names of the rows."""
    rows = [cases.pack_of(u, bs) for _, u in cases.edge_lists(rng)]
    rows += [None, cases.wrap_pack(), cases.zero_block_pack(), cases.pack_of(gen.zipf_gaps(rng, 20000), bs), None]
    return rows


def _same_pack(got, rc_want):
    rc, want = rc_want
    assert rc == 0
    if want.is_nil:
        assert got is None
        return
    assert got is not None
    for f in ("base", "num_uids", "delta_off", "deltas"):
        assert np.array_equal(np.asarray(getattr(got, f)), getattr(want, f)), f


@pytest.mark.parametrize("bs", [1, 5, 256, 5000])
def test_roundtrip_rows_against_the_oracle(bs):
    from dgraph_b200 import codec

    rng = np.random.default_rng(100 + bs)
    rows = _rows(bs, rng)
    out, off = codec.DecodeToBufferRows([None if r is None else r.uid_pack() for r in rows])
    streams = []
    for i, r in enumerate(rows):
        got = out[int(off[i]): int(off[i + 1])].tobytes()
        assert got == (bco.decode_to_buffer(r) if r is not None else b""), f"row {i}"
        streams.append(got)
    packs = codec.EncodeFromBufferRows(streams + [b"", bytes.fromhex("8000") * 3], bs)
    for i, s in enumerate(streams + [b"", bytes.fromhex("8000") * 3]):
        _same_pack(packs[i], bco.encode_from_buffer(s, bs))


def test_single_forms_and_zero_block():
    from dgraph_b200 import codec

    assert codec.DecodeToBuffer(None) == b""
    assert codec.DecodeToBuffer(cases.zero_block_pack().uid_pack()) == bytes([10, 3])
    assert codec.DecodeToBuffer(cases.pack_of([0, 5], 256).uid_pack()) == bytes([0, 5])
    assert codec.EncodeFromBuffer(b"", 256) is None
    p = codec.EncodeFromBuffer(bytes([0, 5]), 256)
    assert p.base.tolist() == [0] and p.num_uids.tolist() == [2]


def test_named_packs_hit_the_cache():
    from dgraph_b200 import _lib, codec

    rng = np.random.default_rng(7)
    rows = [cases.pack_of(gen.zipf_gaps(rng, 5000), 256).uid_pack() for _ in range(6)] + [None]
    anon, aoff = codec.DecodeToBufferRows(rows)
    keys = [(9000 + i, 3) for i in range(len(rows))]
    first, _ = codec.DecodeToBufferRows(rows, keys=keys)
    s = _lib.CacheStats()
    _lib.load().dgx_cache_get_stats(C.byref(s))
    hits = s.hits
    again, off = codec.DecodeToBufferRows(rows, keys=keys)
    _lib.load().dgx_cache_get_stats(C.byref(s))
    assert s.hits >= hits + 6
    assert np.array_equal(anon, first) and np.array_equal(anon, again) and np.array_equal(aoff, off)


def test_sizing_and_capacity():
    from dgraph_b200 import _lib, algo

    lib = _lib.load()
    rng = np.random.default_rng(3)
    rows = [cases.pack_of(gen.zipf_gaps(rng, 900), 256).uid_pack(), None, cases.pack_of([7], 256).uid_pack()]
    refs, keep = algo._refs_of(rows)
    off = np.zeros(4, np.uint64)
    assert lib.dgx_decode_to_buffer_rows(refs, 3, None, _p(off), 0) == 0
    total = int(off[-1])
    out = np.full(total + 8, 0xAB, np.uint8)
    off2 = np.zeros(4, np.uint64)
    assert lib.dgx_decode_to_buffer_rows(refs, 3, _p(out), _p(off2), total - 1) == ERR_CAP
    assert np.array_equal(off, off2) and (out == 0xAB).all()
    assert lib.dgx_decode_to_buffer_rows(refs, 3, _p(out), _p(off2), total) == 0
    assert (out[total:] == 0xAB).all()
    # restore side
    bufs = [out[int(off[i]): int(off[i + 1])].tobytes() for i in range(3)]
    buf = np.frombuffer(b"".join(bufs), np.uint8).copy()
    boff = off.copy()
    img_off, nb, db = np.zeros(4, np.uint64), np.zeros(3, np.uint64), np.zeros(3, np.uint64)
    assert lib.dgx_encode_from_buffer_rows(_p(buf), _p(boff), 3, 256, None, 0, _p(img_off), _p(nb), _p(db)) == 0
    itotal = int(img_off[-1])
    raw = np.full(itotal + 64, 0xCD, np.uint8)
    img = raw[(-raw.ctypes.data) % 16:]
    io2, nb2, db2 = np.zeros(4, np.uint64), np.zeros(3, np.uint64), np.zeros(3, np.uint64)
    assert lib.dgx_encode_from_buffer_rows(_p(buf), _p(boff), 3, 256, _p(img), itotal - 1, _p(io2), _p(nb2), _p(db2)) == ERR_CAP
    assert np.array_equal(io2, img_off) and np.array_equal(nb2, nb) and np.array_equal(db2, db) and (img == 0xCD).all()
    assert lib.dgx_encode_from_buffer_rows(_p(buf), _p(boff), 3, 256, _p(img), itotal, _p(io2), _p(nb2), _p(db2)) == 0
    assert (img[itotal:] == 0xCD).all()
    assert nb.tolist()[1] == 0 and int(img_off[2]) == int(img_off[1])  # the nil row has an empty image
    # every row's image is a dgx_pack_view: decode the whole result again as one run of images
    views, refs2 = [], (_lib.PackRef * 3)()
    for i in range(3):
        v = _lib.PackView()
        if nb[i]:
            assert lib.dgx_pack_image_view(C.c_void_p(img.ctypes.data + int(img_off[i])), 256, int(nb[i]), int(db[i]),
                                           C.byref(v)) == 0
            refs2[i].pack = C.pointer(v)
        views.append(v)
    off3 = np.zeros(4, np.uint64)
    out3 = np.zeros(total + 1, np.uint8)
    assert lib.dgx_decode_to_buffer_rows(refs2, 3, _p(out3), _p(off3), total) == 0
    assert np.array_equal(off3, off) and np.array_equal(out3[:total], out[:total])


@pytest.mark.parametrize("stream", ["80" * 9 + "02", "ff" * 11 + "01", "0580", "ff" * 9])
def test_malformed_streams_after_the_kernels(stream):
    from dgraph_b200 import _lib

    lib = _lib.load()
    good = bytes([1, 2, 3])
    buf = np.frombuffer(good + bytes.fromhex(stream) + good, np.uint8).copy()
    boff = np.array([0, 3, 3 + len(bytes.fromhex(stream)), buf.size], np.uint64)
    raw = np.full(4096 + 16, 0xCD, np.uint8)
    img = raw[(-raw.ctypes.data) % 16:][:4096]
    io, nb, db = np.full(4, 5, np.uint64), np.full(3, 5, np.uint64), np.full(3, 5, np.uint64)
    assert lib.dgx_encode_from_buffer_rows(_p(buf), _p(boff), 3, 256, _p(img), 4096, _p(io), _p(nb), _p(db)) == ERR_ARG
    assert not io.any() and not nb.any() and not db.any() and (img == 0xCD).all()
    assert lib.dgx_encode_from_buffer_rows(_p(buf), _p(boff), 3, 256, None, 0, _p(io), _p(nb), _p(db)) == ERR_ARG


def test_value_split_across_rows_is_refused():
    from dgraph_b200 import codec

    with pytest.raises(Exception):
        codec.EncodeFromBufferRows([bytes([0x81]), bytes([0x01])], 256)
    # each half alone is malformed, together they are one value: rows never join
    assert codec.EncodeFromBuffer(bytes([0x81, 0x01]), 256).base.tolist() == [129]


def _launches():
    from dgraph_b200 import _lib

    return _lib.stats()["kernel_launches"]


def test_launch_counts_do_not_depend_on_the_batch():
    from dgraph_b200 import codec

    rng = np.random.default_rng(11)
    counts = []
    for n in (10, 10000):
        packs = [cases.pack_of(gen.zipf_gaps(rng, int(rng.integers(1, 400))), 256).uid_pack() for _ in range(n)]
        a = _launches()
        out, off = codec.DecodeToBufferRows(packs)
        b = _launches()
        codec.EncodeFromBufferRows([out[int(off[i]): int(off[i + 1])].tobytes() for i in range(n)], 256)
        counts.append((b - a, _launches() - b))
    # packs -> bytes: 4 launches to size, the write again into the exact buffer; bytes -> packs: 9, then the write
    assert counts[0] == counts[1] == (5, 10), counts


def test_device_forms():
    import torch

    from dgraph_b200 import _lib, codec

    lib = _lib.load()
    rng = np.random.default_rng(5)
    hps = [cases.pack_of(gen.zipf_gaps(rng, 3000), 256), None, cases.wrap_pack(), cases.zero_block_pack()]
    lane = lib.dgx_lane_create(0, None)
    assert lane
    dev = []
    keep = []
    for hp in hps:
        if hp is None:
            dev.append(None)
            continue
        up = hp.uid_pack().normalized()
        v = codec.view_of(up)
        keep.append((up, v))
        h = C.c_void_p()
        _lib.check(lib.dgx_dev_pack_upload(lane, C.byref(v), C.byref(h)))
        dev.append(h.value)
    packs = (C.c_void_p * len(dev))(*dev)
    want = [bco.decode_to_buffer(hp) if hp is not None else b"" for hp in hps]
    total = sum(len(w) for w in want)
    d_out = torch.full((total + 16,), 0xAB, dtype=torch.uint8, device="cuda")
    d_off = torch.zeros(len(dev) + 1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    _lib.check(lib.dgx_dev_decode_to_buffer_rows(lane, packs, len(dev), C.c_void_p(d_out.data_ptr()), total,
                                                 C.c_void_p(d_off.data_ptr())))
    _lib.check(lib.dgx_lane_sync(lane))
    out, off = d_out.cpu().numpy(), d_off.cpu().numpy().astype(np.uint64)
    assert out[:total].tobytes() == b"".join(want) and int(off[-1]) == total
    # one short: CAP at the sync, nothing written
    d_out.fill_(0xAB)
    torch.cuda.synchronize()
    _lib.check(lib.dgx_dev_decode_to_buffer_rows(lane, packs, len(dev), C.c_void_p(d_out.data_ptr()), total - 1,
                                                 C.c_void_p(d_off.data_ptr())))
    assert lib.dgx_lane_sync(lane) == ERR_CAP
    assert (d_out.cpu().numpy() == 0xAB).all() and int(d_off[-1].item()) == total
    # restore on the device
    boff = np.array([0] + list(np.cumsum([len(w) for w in want])), np.uint64)
    d_buf = torch.from_numpy(np.frombuffer(b"".join(want) + b"\0", np.uint8).copy()).cuda()
    n = len(dev)
    d_img = torch.full((1 << 16,), 0xCD, dtype=torch.uint8, device="cuda")
    d_io = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
    d_nb = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_db = torch.zeros(n, dtype=torch.int64, device="cuda")
    ptr = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    torch.cuda.synchronize()
    _lib.check(lib.dgx_dev_encode_from_buffer_rows(lane, ptr(d_buf), _p(boff), n, 256, ptr(d_img), 1 << 16, ptr(d_io),
                                                   ptr(d_nb), ptr(d_db)))
    _lib.check(lib.dgx_lane_sync(lane))
    back = [bco.encode_from_buffer(w, 256) for w in want]
    assert all(rc == 0 for rc, _ in back)
    w_img, w_io, w_nb, w_db = cases.pack_images([None if q.is_nil else q for _, q in back])
    itotal = int(w_io[-1])
    img = d_img.cpu().numpy()
    assert np.array_equal(d_io.cpu().numpy().view(np.uint64), w_io)
    assert np.array_equal(d_nb.cpu().numpy().view(np.uint64), w_nb)
    assert np.array_equal(d_db.cpu().numpy().view(np.uint64), w_db)
    assert np.array_equal(img[:itotal], w_img[:itotal]) and (img[itotal:] == 0xCD).all()
    # one short: CAP at the sync, the image untouched, the exact offsets and sizes left behind
    d_img.fill_(0xCD)
    d_io.zero_()
    torch.cuda.synchronize()
    _lib.check(lib.dgx_dev_encode_from_buffer_rows(lane, ptr(d_buf), _p(boff), n, 256, ptr(d_img), itotal - 1,
                                                   ptr(d_io), ptr(d_nb), ptr(d_db)))
    assert lib.dgx_lane_sync(lane) == ERR_CAP
    assert (d_img.cpu().numpy() == 0xCD).all() and np.array_equal(d_io.cpu().numpy().view(np.uint64), w_io)
    # a malformed row: ARG at the sync, arrays zeroed, image untouched
    bad = np.frombuffer(bytes([1, 0x80]), np.uint8).copy()
    d_bad = torch.from_numpy(np.concatenate([bad, np.zeros(14, np.uint8)])).cuda()
    d_img.fill_(0xCD)
    torch.cuda.synchronize()
    _lib.check(lib.dgx_dev_encode_from_buffer_rows(lane, ptr(d_bad), _p(np.array([0, 2], np.uint64)), 1, 256, ptr(d_img),
                                                   1 << 16, ptr(d_io), ptr(d_nb), ptr(d_db)))
    assert lib.dgx_lane_sync(lane) == ERR_ARG
    assert int(d_io[:2].abs().sum().item()) == 0 and int(d_nb[0].item()) == 0 and (d_img.cpu().numpy() == 0xCD).all()
    for h in dev:
        if h:
            lib.dgx_dev_pack_free(C.c_void_p(h))
    lib.dgx_lane_destroy(lane)


def test_four_host_threads():
    from dgraph_b200 import codec

    rng = np.random.default_rng(21)
    lists = [[cases.pack_of(gen.zipf_gaps(rng, int(rng.integers(1, 3000))), 256) for _ in range(50)] for _ in range(4)]
    errors = []

    def work(t):
        try:
            for _ in range(3):
                hps = lists[t]
                out, off = codec.DecodeToBufferRows([h.uid_pack() for h in hps])
                streams = [out[int(off[i]): int(off[i + 1])].tobytes() for i in range(len(hps))]
                assert streams == [bco.decode_to_buffer(h) for h in hps]
                for s, p in zip(streams, codec.EncodeFromBufferRows(streams, 256)):
                    _same_pack(p, bco.encode_from_buffer(s, 256))
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    th = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    for x in th:
        x.start()
    for x in th:
        x.join()
    assert not errors, errors
