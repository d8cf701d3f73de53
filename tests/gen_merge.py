"""Seeded inputs of the DestUIDs workload (tools/bench_ops.py C8, tests/test_gpu_merge_matrix.py): a task's uid matrix
unioned into the next level's DestUIDs, sg.DestUIDs = algo.MergeSorted(result.UidMatrix) (query/query.go:2290).
Every input is a CSR matrix (v, v_off): row i is v[v_off[i] .. v_off[i+1])."""
from __future__ import annotations

import numpy as np

import gen
import gen_rows
import gen_sort


def csr(rows):
    v_off = np.zeros(len(rows) + 1, np.uint64)
    if rows:
        np.cumsum([r.size for r in rows], out=v_off[1:])
    v = np.concatenate(rows).astype(np.uint64) if int(v_off[-1]) else np.zeros(0, np.uint64)
    return np.ascontiguousarray(v), v_off


def rows_of(v, v_off):
    return [v[int(v_off[i]): int(v_off[i + 1])] for i in range(v_off.size - 1)]


def c8a():
    """The C7 matrix: gen_sort.c7_inputs rows (10 000 rows, 6.49e5 uids)."""
    return csr(gen_sort.c7_inputs()[1])


def c8b():
    """The C6 rows: gen_rows.c6_inputs (10 000 rows, about 6.9e7 uids, heavy overlap from one 2e7-uid master)."""
    return csr(gen_rows.c6_inputs()[1])


def c8c(n_rows: int = 200_000, n_master: int = 10_000_000, lo: int = 1, hi: int = 32):
    """n_rows rows of lo..hi uids (uniform, seed 802) drawn with replacement from a Zipf-gap master (seed 801), plus one
    hub uid, the master's middle uid, in every row (the same `country` node for every `person`).  Rows are sorted and
    de-duplicated."""
    master = gen.zipf_gaps(np.random.default_rng(801), n_master)
    r = np.random.default_rng(802)
    sizes = r.integers(lo, hi + 1, n_rows)
    row = np.repeat(np.arange(n_rows), sizes)
    vals = master[r.integers(0, n_master, int(sizes.sum()))]
    hub = master[n_master // 2]
    row = np.concatenate([row, np.arange(n_rows)])
    vals = np.concatenate([vals, np.full(n_rows, hub, np.uint64)])
    o = np.lexsort((vals, row))
    row, vals = row[o], vals[o]
    keep = np.ones(row.size, bool)
    keep[1:] = (row[1:] != row[:-1]) | (vals[1:] != vals[:-1])
    row, vals = row[keep], vals[keep]
    v_off = np.zeros(n_rows + 1, np.uint64)
    np.cumsum(np.bincount(row, minlength=n_rows), out=v_off[1:])
    return np.ascontiguousarray(vals, np.uint64), v_off


C8 = {"C8a": c8a, "C8b": c8b, "C8c": c8c}


def algorithmic_bytes(m: int, out_len: int) -> int:
    """Bytes the union of a matrix must move at least: every uid of the matrix read once and the result written once,
    8 * (M + |Out|)."""
    return 8 * (m + out_len)
