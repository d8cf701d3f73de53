"""Seeded mutable layers for List.Uids rows (tests/test_list_uids_oracle.py, tests/test_gpu_list_uids_rows.py,
tools/bench_ops.py C9): a posting list's pending postings, resolved to one (uid, flags) entry per uid as List.Uids sees
them -- deletes of uids in the pack and of uids not in it, re-SETs of uids already in the pack, new uids, and value
postings (flag MUT_VALUE) on both sides."""
from __future__ import annotations

import numpy as np

COMPRESSED, PROBE, ITERATE = 0, 1, 2
MUT_DEL, MUT_VALUE = 1, 2


def layer(rng, row: np.ndarray, pool: np.ndarray, n: int, p_flags=(0.45, 0.35, 0.15, 0.05)):
    """About n entries: half drawn from the pack's uids `row`, half from `pool` (new uids, or deletes of uids the pack
    does not hold).  Flags drawn from (SET, DEL, VALUE, DEL | VALUE) with probabilities p_flags.  uid 0 never occurs."""
    if n <= 0:
        return np.zeros(0, np.uint64), np.zeros(0, np.uint8)
    k_row = min(row.size, (n + 1) // 2)
    # indices drawn with replacement (a permutation of a large pool per call would dominate); repeats merge below
    a = row[rng.integers(0, row.size, k_row)] if k_row else np.zeros(0, np.uint64)
    b = pool[rng.integers(0, pool.size, n - k_row)] if pool.size else np.zeros(0, np.uint64)
    uids = np.unique(np.concatenate([a, b]).astype(np.uint64))
    uids = uids[uids != 0]
    flags = rng.choice(np.array([0, MUT_DEL, MUT_VALUE, MUT_DEL | MUT_VALUE], np.uint8), uids.size, p=p_flags)
    return uids, flags.astype(np.uint8)


def mode_of(approx_len: int, m: int, has_layer: bool) -> int:
    """The branch List.Uids takes (posting/list.go:1795-1822): compressed without a mutable layer, probe when
    len(v) < ApproxLen, iterate otherwise."""
    if not has_layer:
        return COMPRESSED
    return PROBE if m < approx_len else ITERATE


def want_row(mode: int, pack_uids, mut_uids, mut_flags, after: int, v: np.ndarray) -> np.ndarray:
    """The set formula of each branch, in numpy (a second opinion on the oracle's line-by-line restatement).
    pack_uids None: a delete-all marker (or an empty immutable layer)."""
    v = np.asarray(v, np.uint64)
    pk = np.zeros(0, np.uint64) if pack_uids is None else np.asarray(pack_uids, np.uint64)
    in_pack = np.isin(v, pk)
    if mode == COMPRESSED:
        return v[in_pack & (v >= np.uint64(after))]
    mu = np.asarray(mut_uids, np.uint64)
    mf = np.asarray(mut_flags, np.uint8)
    j = np.searchsorted(mu, v)
    jc = np.minimum(j, max(mu.size - 1, 0))
    has = (j < mu.size) & (mu[jc] == v) if mu.size else np.zeros(v.size, bool)
    f = mf[jc] if mu.size else np.zeros(v.size, np.uint8)
    if mode == PROBE:
        keep = np.where(has, (f & MUT_DEL) == 0, in_pack)
        return v[keep]
    keep = np.where(has, f == 0, in_pack) & (v > np.uint64(after))
    return v[keep]
