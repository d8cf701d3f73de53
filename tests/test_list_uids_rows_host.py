"""dgx_list_uids_rows on a box without a GPU: every argument the host checks is refused before a device is needed,
nrows == 0 needs none, and anything else fails loudly (no CPU fallback)."""
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


def _call(packs, mode, mut_uids, mut_flags, mut_off, after, v, null=()):
    """The raw entry point; names in `null` are passed as NULL."""
    from dgraph_b200 import _lib, algo

    lib = _lib.load()
    refs, keep = algo._refs_of(packs)
    mode = np.asarray(mode, np.uint8)
    mut_uids, mut_flags = np.asarray(mut_uids, np.uint64), np.asarray(mut_flags, np.uint8)
    mut_off, v = np.asarray(mut_off, np.uint64), np.asarray(v, np.uint64)
    out = np.zeros(64, np.uint64)
    out_off = np.zeros(len(packs) + 1, np.uint64)
    arg = {"refs": refs, "mode": _p(mode), "mu": _p(mut_uids), "mf": _p(mut_flags), "off": _p(mut_off), "v": _p(v),
           "out_off": _p(out_off)}
    for k in null:
        arg[k] = None
    return lib.dgx_list_uids_rows(arg["refs"], arg["mode"], len(packs), arg["mu"], arg["mf"], arg["off"], after,
                                  arg["v"], v.size, _p(out), arg["out_off"], out.size)


def test_zero_rows_need_no_device():
    from dgraph_b200 import algo

    out, off = algo.ListUidsRows([], [], [], 5, np.array([1, 2], np.uint64))
    assert out.size == 0 and off.tolist() == [0]
    from dgraph_b200 import _lib

    off = np.full(1, 7, np.uint64)
    assert _lib.load().dgx_list_uids_rows(None, None, 0, None, None, None, 0, None, 0, None, _p(off), 0) == 0
    assert off.tolist() == [0]


def test_host_checks_fire_without_a_device():
    p = _pack(np.arange(10, 2000, 3))
    v = [10, 13, 16, 500]
    ok = dict(packs=[p, None], mode=[1, 2], mut_uids=[13, 20], mut_flags=[1, 0], mut_off=[0, 1, 2], after=0, v=v)
    cases = {
        "unknown mode": dict(ok, mode=[1, 3]),
        "compressed row with entries": dict(ok, mode=[0, 2]),
        "mut_off[0] != 0": dict(ok, mut_off=[1, 1, 2]),
        "decreasing offsets": dict(ok, mut_off=[0, 2, 1]),
        # each row passes its own bounds; the total alone is refused, before any entry is read
        "2^31 entries in all": dict(ok, mut_off=[0, 2**30, 2**31]),
        "empty v": dict(ok, v=[]),
    }
    for what, kw in cases.items():
        assert _call(**kw) == ERR_ARG, what
    for name in ("refs", "mode", "off", "v", "mu", "mf", "out_off"):
        assert _call(**ok, null=(name,)) == ERR_ARG, f"null {name}"


def test_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from dgraph_b200 import _lib, algo

    packs = [_pack([3, 9, 27]), None, _pack(np.arange(1000, 5000, 3))]
    muts = [None, (np.array([9], np.uint64), np.array([0], np.uint8)), (np.array([1003], np.uint64), np.array([1], np.uint8))]
    with pytest.raises(_lib.DgxError) as ei:
        algo.ListUidsRows(packs, [0, 2, 1], muts, 0, np.array([3, 9, 27, 1003], np.uint64))
    assert ei.value.code == ERR_NODEV
    # no mutable entry at all still needs the device
    assert _call([packs[0]], [0], [], [], [0, 0], 0, [3, 9]) == ERR_NODEV
