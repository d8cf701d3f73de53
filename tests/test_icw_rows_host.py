"""algo.IntersectCompressedWithRows on a box without a GPU: shapes the host mirror produces itself, and a loud
failure (no CPU fallback) for anything that needs the device."""
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


def test_zero_rows_need_no_call():
    from dgraph_b200 import algo, pb

    out, off = algo.IntersectCompressedWithRows([], 5, pb.List([1, 2, 3]))
    assert out.size == 0 and off.dtype == np.uint64 and off.tolist() == [0]
    out, off = algo.IntersectCompressedWithRows([], 0, np.zeros(0, np.uint64))
    assert off.tolist() == [0]


def test_fails_loudly_without_gpu():
    import torch

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from dgraph_b200 import _lib, algo

    packs = [_pack([3, 9, 27]), None, _pack(np.arange(1000, 5000, 3))]
    with pytest.raises(_lib.DgxError) as ei:
        algo.IntersectCompressedWithRows(packs, 0, np.array([3, 27, 1003], np.uint64))
    assert ei.value.code == -5  # DGX_ERR_NODEV
    with pytest.raises(_lib.DgxError):
        algo.IntersectCompressedWithRows(packs, 0, np.array([3], np.uint64), keys=[(1, 1), (0, 0), (2, 1)])
