"""The backup codec on the device at the edges of its restore and backup plans (fixtures and host model:
tests/backup_codec_geometry.py): values of every length ending at every offset of a thread's range, terminators on a
tile's first byte, 10-byte and non-minimal values, overflows and truncated rows on tile edges, rows on tile and thread
edges and runs of empty rows, upper-word and row changes on value tiles' and threads' first values, 33 and more tiles
of look-back, wrapping sums, more than 2048 segments and blocks, blocks of 129 to 258 values, BlockSize 0 to
2^32 - 1, 2048 and 2049 rows, every image padding; on the backup side boundary varints of every length, NumUids 0
blocks, 255 to 73 800 blocks, nil and empty packs between packs, and a total of 0 bytes.

Every restore fixture runs through dgx_encode_from_buffer_rows and dgx_dev_encode_from_buffer_rows, every backup
fixture through dgx_decode_to_buffer_rows and dgx_dev_decode_to_buffer_rows, at every capacity the fixture names:
the return code (and dgx_lane_sync's on the device forms), the launches, the offsets and sizes, and the bytes equal
the model's and the oracle's, and nothing is written past a capacity or, on an error, into the output at all.  Every
restored image decodes back to the oracle's DecodeToBuffer of its pack: the input stream itself, up to non-minimal
varints, wherever the uids do not decrease inside a block.  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import functools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import backup_codec_geometry as bg  # noqa: E402
import backup_codec_oracle as bco  # noqa: E402

pytestmark = pytest.mark.gpu

RESTORE = {f.name: f for f in bg.all_restore_fixtures()}
BACKUP = {f.name: f for f in bg.all_backup_fixtures()}
RESTORE_CASES = [(n, c) for n, f in RESTORE.items() for c in f.caps]
BACKUP_CASES = [(n, c) for n, f in BACKUP.items() for c in f.caps]
GUARD = 64          # bytes past each capacity that must stay untouched
FILL8 = 0xCD
FILL64 = 5


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def lib():
    from dgraph_b200 import _lib

    L = _lib.load()
    _lib.check(L.dgx_init(-1))
    return L


@pytest.fixture(scope="module")
def lane(lib):
    ln = lib.dgx_lane_create(0, None)
    assert ln
    yield ln
    lib.dgx_lane_destroy(ln)


@functools.lru_cache(maxsize=None)
def restore_plan(name):
    f = RESTORE[name]
    return bg.simulate_restore(f.rows, f.bsz, f.caps)


@functools.lru_cache(maxsize=None)
def restore_image(name):
    return restore_plan(name)[0].image()[0]


@functools.lru_cache(maxsize=None)
def backup_plan(name):
    f = BACKUP[name]
    return bg.simulate_backup(f.packs, f.caps)


def _launched(fn):
    from dgraph_b200 import _lib

    k0 = _lib.stats()["kernel_launches"]
    res = fn()
    return res, _lib.stats()["kernel_launches"] - k0


def _aligned(n, fill):
    raw = np.full(n + 16, fill, np.uint8)
    return raw[(-raw.ctypes.data) % 16:][:n]


def _buf(f):
    buf = np.frombuffer(b"".join(f.rows) + b"\0" * 16, np.uint8).copy()
    boff = np.concatenate([[0], np.cumsum([len(r) for r in f.rows])]).astype(np.uint64)
    return buf, boff


def _check_restore(name, ch, want, img_off, nblocks, delta_bytes, img, cap):
    p = restore_plan(name)[0]
    assert np.array_equal(img_off, want.img_off), f"{name} {ch}: img_off"
    assert np.array_equal(nblocks, want.nblocks.astype(np.uint64)), f"{name} {ch}: nblocks"
    assert np.array_equal(delta_bytes, want.delta_bytes.astype(np.uint64)), f"{name} {ch}: delta_bytes"
    if img is None:
        return
    if want.written:
        total = p.total
        w = restore_image(name)
        bad = np.nonzero(img[:total] != w[:total])[0]
        assert bad.size == 0, f"{name} {ch}: {bad.size} image bytes differ, first at {bad[:8]}"
        assert (img[total:] == FILL8).all(), f"{name} {ch}: written past the image"
    else:
        assert (img == FILL8).all(), f"{name} {ch}: image written on rc {want.rc} / {want.sync}"


@pytest.mark.parametrize("name, ch", RESTORE_CASES)
def test_restore_host_form(lib, name, ch):
    """dgx_encode_from_buffer_rows: return code, launches, offsets, sizes and image bytes equal the model's (and the
    oracle's, which the model equals on the CPU); ARG zeroes the arrays and writes no image; CAP writes no image."""
    f = RESTORE[name]
    p, calls = restore_plan(name)
    want = calls[ch][0]
    cap = p.cap_of(ch, set())
    buf, boff = _buf(f)
    nr = len(f.rows)
    io, nb, db = (np.full(nr + 1, FILL64, np.uint64), np.full(nr, FILL64, np.uint64), np.full(nr, FILL64, np.uint64))
    img = None if cap is None else _aligned(cap + GUARD, FILL8)
    rc, launches = _launched(lambda: lib.dgx_encode_from_buffer_rows(_p(buf), _p(boff), nr, f.bsz, _p(img),
                                                                     0 if cap is None else cap, _p(io), _p(nb), _p(db)))
    assert (rc, launches) == (want.rc, want.launches), f"{name} {ch}: device {(rc, launches)}, model {want}"
    _check_restore(name, ch, want, io, nb, db, img, cap)


@pytest.mark.parametrize("name, ch", RESTORE_CASES)
def test_restore_device_form(lib, lane, name, ch):
    """dgx_dev_encode_from_buffer_rows: DGX_OK from the call, the model's verdict from dgx_lane_sync, nine launches,
    and the same arrays and image as the host form."""
    import torch

    f = RESTORE[name]
    p, calls = restore_plan(name)
    want = calls[ch][1]
    cap = p.cap_of(ch, set())
    buf, boff = _buf(f)
    nr = len(f.rows)
    d_buf = torch.from_numpy(buf).cuda()
    d_io = torch.full((nr + 1,), FILL64, dtype=torch.int64, device="cuda")
    d_nb = torch.full((nr,), FILL64, dtype=torch.int64, device="cuda")
    d_db = torch.full((nr,), FILL64, dtype=torch.int64, device="cuda")
    d_img = None if cap is None else torch.full((cap + GUARD,), FILL8, dtype=torch.uint8, device="cuda")
    ptr = lambda t: None if t is None else C.c_void_p(t.data_ptr())  # noqa: E731
    torch.cuda.synchronize()
    rc, launches = _launched(lambda: lib.dgx_dev_encode_from_buffer_rows(
        lane, ptr(d_buf), _p(boff), nr, f.bsz, ptr(d_img), 0 if cap is None else cap, ptr(d_io), ptr(d_nb), ptr(d_db)))
    sync = lib.dgx_lane_sync(lane)
    assert (rc, sync, launches) == (want.rc, want.sync, want.launches), f"{name} {ch}: device {(rc, sync, launches)}, model {want}"
    u = lambda t: t.cpu().numpy().view(np.uint64)  # noqa: E731
    _check_restore(name, ch, want, u(d_io), u(d_nb), u(d_db), None if d_img is None else d_img.cpu().numpy(), cap)


@pytest.mark.parametrize("name", [n for n, f in RESTORE.items() if "exact" in f.caps])
def test_restored_images_decode_back(lib, name):
    """Every row's restored image, viewed with dgx_pack_image_view and read by dgx_decode_to_buffer_rows, gives back
    the row's stream as the model decodes it (which the CPU suite checks against the oracle's round trip)."""
    from dgraph_b200 import _lib

    f = RESTORE[name]
    p = restore_plan(name)[0]
    buf, boff = _buf(f)
    nr = len(f.rows)
    io, nb, db = np.zeros(nr + 1, np.uint64), np.zeros(nr, np.uint64), np.zeros(nr, np.uint64)
    img = _aligned(p.total + GUARD, FILL8)
    assert lib.dgx_encode_from_buffer_rows(_p(buf), _p(boff), nr, f.bsz, _p(img), p.total, _p(io), _p(nb), _p(db)) == 0
    views, refs = [], (_lib.PackRef * nr)()
    for i in range(nr):
        v = _lib.PackView()
        if nb[i]:
            assert lib.dgx_pack_image_view(C.c_void_p(img.ctypes.data + int(io[i])), f.bsz & 0xFFFFFFFF, int(nb[i]),
                                           int(db[i]), C.byref(v)) == 0
            refs[i].pack = C.pointer(v)
        views.append(v)
    want = [p.decoded_stream(i) for i in range(nr)]
    total = sum(len(w) for w in want)
    out, off = np.full(total + GUARD, FILL8, np.uint8), np.zeros(nr + 1, np.uint64)
    assert lib.dgx_decode_to_buffer_rows(refs, nr, _p(out), _p(off), total) == 0
    got = [out[int(off[i]): int(off[i + 1])].tobytes() for i in range(nr)]
    for i in range(nr):
        assert got[i] == want[i], f"{name}: row {i} does not decode back"


def _refs(packs):
    from dgraph_b200 import algo

    hands = {}
    ups = [None if pk is None or not pk.blocks else hands.setdefault(id(pk), pk.hand()).uid_pack() for pk in packs]
    refs, keep = algo._refs_of(ups)
    return refs, (keep, hands, ups)


def _check_backup(name, ch, want, off, out, cap):
    p = backup_plan(name)[0]
    assert np.array_equal(off, want.out_off), f"{name} {ch}: out_off"
    if out is None:
        return
    if want.written:
        w = b"".join(p.streams)
        assert out[: p.total].tobytes() == w, f"{name} {ch}: bytes"
        assert (out[p.total:] == FILL8).all(), f"{name} {ch}: written past the bytes"
    else:
        assert (out == FILL8).all(), f"{name} {ch}: bytes written on rc {want.rc} / {want.sync}"


@pytest.mark.parametrize("name, ch", BACKUP_CASES)
def test_backup_host_form(lib, name, ch):
    """dgx_decode_to_buffer_rows: return code, launches (four, and the write pass unless nothing is written), offsets
    and bytes equal the model's, and the model's bytes the oracle's row by row."""
    f = BACKUP[name]
    p, calls = backup_plan(name)
    want = calls[ch][0]
    cap = p.cap_of(ch, set())
    hands = {}
    for r, pk in enumerate(f.packs):
        if pk is not None:
            assert p.streams[r] == bco.decode_to_buffer(hands.setdefault(id(pk), pk.hand())), f"{name}: row {r}"
    refs, keep = _refs(f.packs)
    nr = len(f.packs)
    off = np.full(nr + 1, FILL64, np.uint64)
    out = None if cap is None else np.full(cap + GUARD, FILL8, np.uint8)
    rc, launches = _launched(lambda: lib.dgx_decode_to_buffer_rows(refs, nr, _p(out), _p(off), 0 if cap is None else cap))
    assert (rc, launches) == (want.rc, want.launches), f"{name} {ch}: device {(rc, launches)}, model {want}"
    _check_backup(name, ch, want, off, out, cap)


@pytest.mark.parametrize("name, ch", BACKUP_CASES)
def test_backup_device_form(lib, lane, name, ch):
    """dgx_dev_decode_to_buffer_rows over uploaded packs: DGX_OK from the call, CAP from dgx_lane_sync when the bytes do
    not fit, four launches, the model's offsets and bytes."""
    import torch

    from dgraph_b200 import _lib, codec

    f = BACKUP[name]
    p, calls = backup_plan(name)
    want = calls[ch][1]
    cap = p.cap_of(ch, set())
    handles, keep = {}, []
    dev = []
    for pk in f.packs:
        if pk is None or not pk.blocks:
            dev.append(None)
            continue
        if id(pk) not in handles:
            up = pk.hand().uid_pack().normalized()
            v = codec.view_of(up)
            keep.append((up, v))
            h = C.c_void_p()
            _lib.check(lib.dgx_dev_pack_upload(lane, C.byref(v), C.byref(h)))
            handles[id(pk)] = h.value
        dev.append(handles[id(pk)])
    nr = len(dev)
    packs = (C.c_void_p * nr)(*dev)
    d_out = None if cap is None else torch.full((cap + GUARD,), FILL8, dtype=torch.uint8, device="cuda")
    d_off = torch.full((nr + 1,), FILL64, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    try:
        rc, launches = _launched(lambda: lib.dgx_dev_decode_to_buffer_rows(
            lane, packs, nr, None if d_out is None else C.c_void_p(d_out.data_ptr()), 0 if cap is None else cap,
            C.c_void_p(d_off.data_ptr())))
        sync = lib.dgx_lane_sync(lane)
    finally:
        for h in handles.values():
            lib.dgx_dev_pack_free(C.c_void_p(h))
    assert (rc, sync, launches) == (want.rc, want.sync, want.launches), f"{name} {ch}: device {(rc, sync, launches)}, model {want}"
    _check_backup(name, ch, want, d_off.cpu().numpy().view(np.uint64), None if d_out is None else d_out.cpu().numpy(),
                  cap)
