"""codec.Encode on the device at the edges of its segment, block and capacity plan (fixtures and host model:
tests/encode_geometry.py), array by array against the oracle: upper-word changes at a tile's first index, a thread's
first index and the last uid, n around multiples of 2048, 41 tiles of look-back, 1024, 1025 and 2049 segments,
segments that fill seg_cap exactly and overflow it by one, the list that needed three calls before the overflow report
was fixed, segments of bsz * k and bsz * k +- 1 uids, blocks of 129 to 260 uids, block counts at the bound and one
past it, every delta width at every position of a group, duplicates across block and tile edges, uid 0 and 2^64 - 1,
BlockSize 0 to 2^32 - 1, and caller capacities of 0, one block short, one delta byte short and exact.

Every fixture runs through codec.Encode (the launches of every call checked against the model) and through the raw
dgx_encode from each capacity the fixture names: each call's return code and returned sizes equal the model's, a
DGX_ERR_CAP call leaves the guard-filled caller arrays untouched, a DGX_OK call writes nothing past the pack, and
one call again with the returned sizes succeeds.  The packed fixtures run through the four packed entry points and
are compared with the oracle's pack and decoded back.  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import functools
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import encode_geometry as eg  # noqa: E402
from test_gpu_parity import eq, to_pack  # noqa: E402
from test_gpu_round2 import same_pack  # noqa: E402

pytestmark = pytest.mark.gpu

FIXTURES = {f.name: f for f in eg.all_fixtures()}
PACKED = {f.name: f for f in eg.all_packed_fixtures()}
RAW = [(n, c) for n, f in FIXTURES.items() for c in f.caps]
GUARD = 8          # elements past each capacity that must stay untouched
FILL64 = 0xDEADBEEFCAFEB00D
FILL32 = 0xCAFEB00D
FILL8 = 0xA5


@pytest.fixture(scope="module")
def dgx():
    import dgraph_b200
    from dgraph_b200 import _lib

    _lib.check(_lib.load().dgx_init(-1))
    return dgraph_b200


@functools.lru_cache(maxsize=None)
def plan(name):
    return eg.simulate(FIXTURES[name])[0]


def want_pack(u, bsz):
    """The oracle's pack; above the oracle's int BlockSize, gen.encode_pack_np's (checked against the oracle on the CPU
    at every BlockSize it takes)."""
    if bsz <= (1 << 31) - 1:
        from oracle import pyoracle

        return pyoracle.encode(np.asarray(u, np.uint64), bsz)
    _, base, num, doff, deltas = eg.pack_of(u, bsz)
    return SimpleNamespace(is_nil=False, block_size=bsz, base=base, num_uids=num, delta_off=doff, deltas=deltas,
                           nblocks=base.size)


def _launched(fn):
    from dgraph_b200 import _lib

    k0 = _lib.stats()["kernel_launches"]
    res = fn()
    return res, _lib.stats()["kernel_launches"] - k0


@pytest.mark.parametrize("name", list(FIXTURES))
def test_encode(dgx, name):
    """codec.Encode: the pack equals the oracle's array by array; five launches per call the model makes."""
    f = FIXTURES[name]
    got, launches = _launched(lambda: dgx.codec.Encode(f.uids, f.bsz))
    same_pack(got, want_pack(f.uids, f.bsz), name)
    model = eg.calls(f.uids, f.bsz, eg.bound(f.uids.size, f.bsz))
    assert launches == sum(c.launches for c in model), (launches, model)


def raw_call(u, bsz, nb_cap, db_cap):
    """dgx_encode into guard-filled arrays of the given capacities: (rc, nblocks, delta_bytes, arrays, launches)."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    base = np.full(nb_cap + GUARD, FILL64, np.uint64)
    num = np.full(nb_cap + GUARD, FILL32, np.uint32)
    doff = np.full(nb_cap + 1 + GUARD, FILL64, np.uint64)
    deltas = np.full(db_cap + GUARD, FILL8, np.uint8)
    nb, db, view = C.c_size_t(nb_cap), C.c_size_t(db_cap), _lib.PackView()
    p = [a.ctypes.data_as(C.c_void_p) for a in (u, base, num, doff, deltas)]
    rc, launches = _launched(lambda: lib.dgx_encode(p[0], u.size, bsz, p[1], p[2], p[3], p[4], C.byref(nb),
                                                    C.byref(db), C.byref(view)))
    return rc, nb.value, db.value, (base, num, doff, deltas), launches


def _untouched(arrs, nb, db, what):
    base, num, doff, deltas = arrs
    assert (base[nb:] == FILL64).all() and (num[nb:] == FILL32).all(), what + ": base / num written past the pack"
    assert (doff[nb + 1:] == FILL64).all(), what + ": delta_off written past the pack"
    assert (deltas[db:] == FILL8).all(), what + ": deltas written past the pack"


@pytest.mark.parametrize("name, caps", RAW)
def test_raw_calls(dgx, name, caps):
    """dgx_encode from the capacities the fixture names, called again with the sizes it returns: one retry
    succeeds, every call answers as the model does, DGX_ERR_CAP leaves the caller's arrays as they were, DGX_OK
    writes the oracle's pack and nothing past it."""
    f = FIXTURES[name]
    model = plan(name)[caps]
    u = np.ascontiguousarray(f.uids, np.uint64)
    cap = model[0].caps
    got = []
    for _ in range(2):
        rc, nb, db, arrs, launches = raw_call(u, f.bsz, *cap)
        got.append((rc, nb, db, cap, launches))
        if rc == eg.ERR_CAP:
            _untouched(arrs, 0, 0, f"{name} {caps}: call {len(got)}")
            assert arrs[2][0] == FILL64, f"{name} {caps}: delta_off[0] written on DGX_ERR_CAP"
            cap = (nb, db)
            continue
        assert rc == eg.OK, (name, caps, rc)
        w = want_pack(u, f.bsz)
        assert (nb, db) == (w.base.size, w.deltas.size)
        eq(arrs[0][:nb], w.base, name + " base")
        assert np.array_equal(arrs[1][:nb], w.num_uids) and np.array_equal(arrs[2][:nb + 1], w.delta_off), name
        assert np.array_equal(arrs[3][:db], w.deltas), name + " deltas"
        _untouched(arrs, nb, db, f"{name} {caps}")
        break
    assert got[-1][0] == eg.OK, f"{name} {caps}: DGX_ERR_CAP again after the sizes the first call returned: {got}"
    want = [(c.rc, c.nblocks, c.delta_bytes, c.caps, c.launches) for c in model]
    assert got == want, f"{name} {caps}: device {got}, model {want}"


def test_empty_list(dgx):
    """No uids: the nil pack, no launch, delta_off[0] = 0."""
    rc, nb, db, arrs, launches = raw_call(np.zeros(0, np.uint64), 256, 4, 64)
    assert (rc, nb, db, launches) == (eg.OK, 0, 0, 0) and arrs[2][0] == 0
    assert dgx.codec.Encode(np.zeros(0, np.uint64), 256) is None


@pytest.mark.parametrize("name", list(PACKED))
def test_packed_ops(dgx, orc, name):
    """The four packed entry points, whose result length is read on the device: the pack equals the oracle's encoding
    of the set the model computes, and decodes back to it."""
    f = PACKED[name]
    packs = [to_pack(dgx, orc.encode(np.asarray(l, np.uint64), f.bsz)) for l in f.lists]
    entry = {"intersect": lambda: dgx.algo.IntersectWithLinPacked(packs[0], packs[1], f.bsz),
             "difference": lambda: dgx.algo.DifferencePacked(packs[0], packs[1], f.bsz),
             "merge": lambda: dgx.algo.MergeSortedPacked(packs, f.bsz),
             "intersect_sorted": lambda: dgx.algo.IntersectSortedPacked(packs, f.bsz)}
    for op in eg.PACKED_OPS:
        res, _ = eg.packed_result(op, f.lists)
        got = entry[op]()
        same_pack(got, orc.encode(res, f.bsz), f"{name} {op}")
        if res.size:
            eq(dgx.codec.Decode(got, 0), res, f"{name} {op}: decode round trip")
