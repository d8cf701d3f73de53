"""algo.IntersectCompressedWithMatrix on a box without a GPU: shapes the library produces without a device, and a
loud failure (no CPU fallback) for anything that needs one."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen  # noqa: E402


def _pack(uids):
    from dgraph_b200 import pb

    bs, base, num, doff, deltas = gen.encode_pack_np(np.asarray(uids, np.uint64), 256)
    return pb.UidPack(bs, base, num, doff, deltas)


def test_zero_rows_and_nil_pack_need_no_device():
    from dgraph_b200 import _lib, algo, pb

    out, off = algo.IntersectCompressedWithMatrix(_pack([3, 9, 27]), [])
    assert out.size == 0 and off.dtype == np.uint64 and off.tolist() == [0]
    out, off = algo.IntersectCompressedWithMatrix(None, [pb.List([1, 2, 3]), np.zeros(0, np.uint64), [4, 5]])
    assert out.size == 0 and off.tolist() == [0, 0, 0, 0]
    lib = _lib.load()
    off1 = np.full(1, 7, np.uint64)
    ref = _lib.PackRef(None, 0, 0)
    _lib.check(lib.dgx_intersect_compressed_matrix(C.byref(ref), None, None, 0, None, off1.ctypes.data_as(C.c_void_p), 0))
    assert off1.tolist() == [0]


def test_bad_offsets_refused_on_the_host():
    from dgraph_b200 import _lib, algo

    lib = _lib.load()
    refs, keep = algo._refs_of([_pack([3, 9, 27])])
    v = np.zeros(1, np.uint64)
    off = np.zeros(3, np.uint64)
    for bo in ([1, 2, 3], [0, 5, 4], [0, 1, 1 << 32]):
        bo = np.array(bo, np.uint64)
        rc = lib.dgx_intersect_compressed_matrix(refs, v.ctypes.data_as(C.c_void_p), bo.ctypes.data_as(C.c_void_p), 2,
                                                 v.ctypes.data_as(C.c_void_p), off.ctypes.data_as(C.c_void_p), 1)
        assert rc == -3, bo  # DGX_ERR_ARG


def test_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from dgraph_b200 import _lib, algo

    rows = [np.array([3, 27, 1003], np.uint64), np.zeros(0, np.uint64), np.arange(1000, 1100, dtype=np.uint64)]
    with pytest.raises(_lib.DgxError) as ei:
        algo.IntersectCompressedWithMatrix(_pack(np.arange(1000, 5000, 3)), rows)
    assert ei.value.code == -5  # DGX_ERR_NODEV
    with pytest.raises(_lib.DgxError) as ei:
        algo.IntersectCompressedWithMatrix(_pack([3, 9, 27]), rows, key=(1, 1))
    assert ei.value.code == -5
