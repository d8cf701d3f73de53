"""Seeded inputs of the intersectBucket workload (tools/bench_ops.py C7, tests/test_gpu_icw_matrix.py): one uid matrix,
each row a sorted sample of one master list, intersected with the index buckets of a sort, each bucket a UidPack
(worker/sort.go:605-700 -> algo.IntersectCompressedWith)."""
from __future__ import annotations

import numpy as np

import gen


def c7_inputs(n_rows: int = 10_000, n_master: int = 20_000_000, lo: float = 10, hi: float = 1e4):
    """Seeded inputs of the intersectBucket workload (tools/bench_ops.py C7): one uid matrix of n_rows rows walked
    against the index buckets of a sort (worker/sort.go:605-700 -> algo.IntersectCompressedWith).
    master: Zipf-gap list (seed 701).  Row sizes i.i.d. truncated power law alpha = 2 on [lo, hi], each row a sorted
    sample of the master without replacement (seed 702).  Buckets (seed 703), each a sorted sample of the master:
    "large" 1e6 uids, "medium" 1e4 uids, "tiny" 100 uids below 2^32 (one block at BlockSize 256).
    Returns (master, rows, {name: bucket uids})."""
    master = gen.zipf_gaps(np.random.default_rng(701), n_master)
    r = np.random.default_rng(702)
    u = r.random(n_rows)
    sizes = np.minimum((1.0 / (1.0 / lo - u * (1.0 / lo - 1.0 / hi))).astype(np.int64), int(hi))
    rows = [master[np.sort(r.choice(n_master, int(s), replace=False))] for s in sizes]
    rb = np.random.default_rng(703)
    low = int(np.searchsorted(master, np.uint64(1 << 32)))
    buckets = {
        "large": master[np.sort(rb.choice(n_master, 1_000_000, replace=False))],
        "medium": master[np.sort(rb.choice(n_master, 10_000, replace=False))],
        "tiny": master[np.sort(rb.choice(low, 100, replace=False))],
    }
    return master, rows, buckets


def matrix_algorithmic_bytes(base, delta_off, rows, out_len: int) -> int:
    """Bytes one pack against a whole uid matrix must move at least: every touched block's header and deltas once
    (12 + len(Deltas)), every uid of the matrix once, and the result: sum_touched (12 + len(Deltas)) + 8 * M + 8 * |out|."""
    m = sum(r.size for r in rows)
    touched = np.zeros(base.size, bool)
    for r in rows:
        b = np.searchsorted(base, r, side="right") - 1
        touched[b[b >= 0]] = True
    return int((12 + (delta_off[1:] - delta_off[:-1])[touched].astype(np.int64)).sum()) + 8 * m + 8 * out_len
