"""The set formula of an unfiltered List.Uids row and of its count, in numpy: a second opinion on the line-by-line
restatement of list_uids_unfiltered_oracle.c (tests/test_list_uids_unfiltered_oracle.py), and the result bound of
tools/bench_ops.py C10.  The mutable layers themselves come from gen_mut.layer."""
from __future__ import annotations

import numpy as np


def most_kept(first: int) -> int:
    """The most values an unfiltered List.Uids row keeps for opts.First (an int32): 0 is MaxInt32, and a negative First
    stops the callback after one value (posting/list.go:1759-1761, 1841-1843, 1864-1872)."""
    return 0x7FFFFFFF if first == 0 else (1 if first < 0 else first)


def want_unfiltered(pack_uids, mut_uids, mut_flags, after: int, first: int = 0) -> np.ndarray:
    """S = {x > after : mut(x) exists ? mut(x) has no flag : x in pack}, cut to most_kept(first) values; its size is the
    count.  pack_uids None: a delete-all marker (or an empty immutable layer)."""
    pk = np.zeros(0, np.uint64) if pack_uids is None else np.asarray(pack_uids, np.uint64)
    mu = np.asarray(mut_uids, np.uint64)
    mf = np.asarray(mut_flags, np.uint8)
    s = np.union1d(pk[~np.isin(pk, mu)], mu[mf == 0]).astype(np.uint64)
    return s[s > np.uint64(after)][: most_kept(first)]
