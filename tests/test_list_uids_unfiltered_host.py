"""dgx_list_uids_unfiltered_rows, dgx_list_count_rows and their device forms on a box without a GPU: every argument the
host checks is refused before a device is needed, nrows == 0 needs none, and anything else fails loudly (no CPU
fallback)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen  # noqa: E402

ERR_ARG, ERR_NODEV = -3, -5


def _pack(uids):
    from dgraph_b200 import pb

    bs, base, num, doff, deltas = gen.encode_pack_np(np.asarray(uids, np.uint64), 256)
    return pb.UidPack(bs, base, num, doff, deltas)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _call(count, packs, mut_uids, mut_flags, mut_off, after=0, first=0, null=()):
    """The raw host entry point (rows, or counts when `count`); names in `null` are passed as NULL."""
    from dgraph_b200 import _lib, algo

    lib = _lib.load()
    refs, keep = algo._refs_of(packs)
    mut_uids, mut_flags = np.asarray(mut_uids, np.uint64), np.asarray(mut_flags, np.uint8)
    mut_off = np.asarray(mut_off, np.uint64)
    out = np.zeros(64, np.uint64)
    out_off = np.zeros(len(packs) + 1, np.uint64)
    counts = np.zeros(len(packs), np.uint32)
    arg = {"refs": refs, "mu": _p(mut_uids), "mf": _p(mut_flags), "off": _p(mut_off), "out_off": _p(out_off),
           "counts": _p(counts)}
    for k in null:
        arg[k] = None
    if count:
        return lib.dgx_list_count_rows(arg["refs"], len(packs), arg["mu"], arg["mf"], arg["off"], after, arg["counts"])
    return lib.dgx_list_uids_unfiltered_rows(arg["refs"], len(packs), arg["mu"], arg["mf"], arg["off"], after, first,
                                             _p(out), arg["out_off"], out.size)


def test_zero_rows_need_no_device():
    from dgraph_b200 import _lib, algo

    out, off = algo.ListUidsUnfilteredRows([], [], 5, 10)
    assert out.size == 0 and off.tolist() == [0]
    assert algo.ListCountRows([], [], 5).size == 0
    lib = _lib.load()
    off = np.full(1, 7, np.uint64)
    assert lib.dgx_list_uids_unfiltered_rows(None, 0, None, None, None, 0, 0, None, _p(off), 0) == 0
    assert off.tolist() == [0]
    assert lib.dgx_list_count_rows(None, 0, None, None, None, 0, None) == 0


@pytest.mark.parametrize("count", [False, True], ids=["rows", "counts"])
def test_host_checks_fire_without_a_device(count):
    p = _pack(np.arange(10, 2000, 3))
    ok = dict(packs=[p, None], mut_uids=[13, 20], mut_flags=[1, 0], mut_off=[0, 1, 2])
    cases = {
        "mut_off[0] != 0": dict(ok, mut_off=[1, 1, 2]),
        "decreasing offsets": dict(ok, mut_off=[0, 2, 1]),
        # each row passes its own bound; the total alone is refused, before any entry is read
        "2^31 entries in all": dict(ok, mut_off=[0, 2**30, 2**31]),
    }
    for what, kw in cases.items():
        assert _call(count, **kw) == ERR_ARG, what
    for name in ("refs", "off", "mu", "mf", "counts" if count else "out_off"):
        assert _call(count, **ok, null=(name,)) == ERR_ARG, f"null {name}"


def test_device_forms_check_before_queueing():
    """The device forms refuse a null lane before anything is read."""
    from dgraph_b200 import _lib

    lib = _lib.load()
    off = np.array([0, 2, 1], np.uint64)
    tab = (C.c_void_p * 2)()
    d = C.c_void_p(16)  # never dereferenced: the checks fire first
    assert lib.dgx_dev_list_uids_unfiltered_rows(None, tab, 2, d, d, _p(off), 0, 0, d, 8, d) == ERR_ARG
    assert lib.dgx_dev_list_count_rows(None, tab, 2, d, d, _p(off), 0, d) == ERR_ARG


def test_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from dgraph_b200 import _lib, algo

    packs = [_pack([3, 9, 27]), None, _pack(np.arange(1000, 5000, 3))]
    muts = [None, (np.array([9], np.uint64), np.array([0], np.uint8)), (np.array([1003], np.uint64), np.array([1], np.uint8))]
    for fn in (lambda: algo.ListUidsUnfilteredRows(packs, muts, 0, 10), lambda: algo.ListCountRows(packs, muts, 0)):
        with pytest.raises(_lib.DgxError) as ei:
            fn()
        assert ei.value.code == ERR_NODEV
    # no mutable entry at all still needs the device
    assert _call(False, [packs[0]], [], [], [0, 0]) == ERR_NODEV
    assert _call(True, [packs[0]], [], [], [0, 0]) == ERR_NODEV
