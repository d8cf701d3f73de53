"""algo.MergeSortedMatrix on a box without a GPU: the shapes the library answers without a device, the offsets it
refuses before copying anything, and a loud failure (no CPU fallback) for anything that needs a device."""
import ctypes as C

import numpy as np
import pytest


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def test_no_rows_and_empty_rows_need_no_device():
    from dgraph_b200 import _lib, algo, pb

    assert algo.MergeSortedMatrix([]).Uids.size == 0
    got = algo.MergeSortedMatrix([pb.List(None), np.zeros(0, np.uint64), pb.List([])])
    assert got.Uids.size == 0 and got.Uids.dtype == np.uint64
    lib = _lib.load()
    n = C.c_size_t(7)
    _lib.check(lib.dgx_merge_sorted_matrix(None, None, 0, None, 0, C.byref(n)))
    assert n.value == 0
    off = np.zeros(4, np.uint64)
    n = C.c_size_t(7)
    _lib.check(lib.dgx_merge_sorted_matrix(None, _p(off), 3, None, 0, C.byref(n)))
    assert n.value == 0


@pytest.mark.parametrize("bad", [[1, 2, 3], [0, 5, 4], [0, 1, 1 << 32]], ids=["first-not-zero", "decreasing", "too-many"])
def test_bad_offsets_refused_on_the_host(bad):
    from dgraph_b200 import _lib

    lib = _lib.load()
    v = np.zeros(8, np.uint64)
    out = np.full(8, 0xABCD, np.uint64)
    off = np.array(bad, np.uint64)
    n = C.c_size_t(7)
    rc = lib.dgx_merge_sorted_matrix(_p(v), _p(off), 2, _p(out), out.size, C.byref(n))
    assert rc == -3, bad  # DGX_ERR_ARG
    assert n.value == 7 and (out == 0xABCD).all()


def test_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from dgraph_b200 import _lib, algo

    rows = [np.array([3, 27, 1003], np.uint64), np.zeros(0, np.uint64), np.arange(1000, 1100, dtype=np.uint64)]
    with pytest.raises(_lib.DgxError) as ei:
        algo.MergeSortedMatrix(rows)
    assert ei.value.code == -5  # DGX_ERR_NODEV
