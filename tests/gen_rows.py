"""Seeded inputs of the handleUidPostings workload (tools/bench_ops.py C6, tests/test_gpu_icw_rows.py): a task's N
posting lists, each a sorted sample of one master list, all intersected with the same v
(worker/task.go:783-987 -> algo.IntersectCompressedWith)."""
from __future__ import annotations

import numpy as np

import gen


def c6_inputs(n_rows: int = 10_000, n_master: int = 20_000_000, lo: float = 1e3, hi: float = 1e6, p_v: float = 0.05):
    """master: Zipf-gap list (seed 601); row sizes i.i.d. truncated power law alpha = 2 on [lo, hi] (seed 600); each row a
    sorted sample of the master without replacement (seed 602); v a thinning p_v of the master (seed 603)."""
    master = gen.zipf_gaps(np.random.default_rng(601), n_master)
    u = np.random.default_rng(600).random(n_rows)
    sizes = np.minimum((1.0 / (1.0 / lo - u * (1.0 / lo - 1.0 / hi))).astype(np.int64), int(hi))
    r = np.random.default_rng(602)
    rows = [master[np.sort(r.choice(n_master, int(s), replace=False))] for s in sizes]
    v = gen.thin(np.random.default_rng(603), master, p_v)
    return master, rows, v


def algorithmic_bytes(packs, after: int, v: np.ndarray, out_len: int) -> int:
    """Bytes the batched IntersectCompressedWith must move at least: every touched block's header and deltas
    (12 + len(Deltas)), every v element inside a touched block's range once per row, and the result:
    sum_touched (12 + len(Deltas)) + 8 * sum_rows (touched v elements) + 8 * |out|.
    packs: (base, delta_off) array pairs, None for a nil pack."""
    total = 8 * out_len
    for p in packs:
        if p is None or p[0].size == 0:
            continue
        base, doff = p
        first = np.maximum(base, np.uint64(after))
        lo = np.searchsorted(v, first, side="left")
        hi = np.append(np.searchsorted(v, base[1:], side="left"), v.size)
        t = hi > lo
        total += int((12 + (doff[1:] - doff[:-1])[t].astype(np.int64)).sum()) + 8 * int((hi - lo)[t].sum())
    return total
