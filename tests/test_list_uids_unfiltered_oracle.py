"""The line-by-line restatement of an unfiltered List.Uids and of the count (list_uids_unfiltered_oracle.c: iterate with the REF
filter and the First cut, posting/list.go:1758-1874; List.Postings, :1878-1890): the reference's own expectations of
TestAfterUIDCount, TestAfterUIDCount2, TestAddMutation / TestAddAndDelMutation (checkUids) and TestMillion
(posting/list_test.go) restated as resolved layers, the First values the worker may pass, and the set formula in numpy
on a few thousand random rows."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(__file__))
import gen  # noqa: E402
import gen_mut  # noqa: E402
import gen_mut_unfiltered as gmu  # noqa: E402
import list_uids_unfiltered_oracle as luo  # noqa: E402
from gen_mut import MUT_DEL, MUT_VALUE  # noqa: E402

MAXI32 = 2**31 - 1


def _counts(uids, flags, p=None):
    """List.Length(readTs, after) of REF-only postings at after 0 / 199 / 300, read as the count and as the row."""
    u, f = np.asarray(uids, np.uint64), np.asarray(flags, np.uint8)
    c = [luo.list_count(p, u, f, a) for a in (0, 199, 300)]
    assert c == [luo.list_uids_unfiltered(p, u, f, a).size for a in (0, 199, 300)]
    return c


def test_after_uid_count(orc):
    """TestAfterUIDCount (:812-881): one transaction's latest op per uid is the resolved entry."""
    op = {i: 0 for i in range(100, 300)}
    assert _counts(list(op), list(op.values())) == [200, 100, 0]
    for i in range(100, 300, 2):
        op[i] = MUT_DEL
    assert _counts(list(op), list(op.values())) == [100, 50, 0]
    for i in range(100, 300, 2):  # redundant deletes
        op[i] = MUT_DEL
    assert _counts(list(op), list(op.values())) == [100, 50, 0]
    for i in range(100, 300):
        op[i] = MUT_DEL
    assert _counts(list(op), list(op.values())) == [0, 0, 0]
    for _ in range(2):  # the second pass changes nothing
        for i in range(100, 300, 4):
            op[i] = 0
        assert _counts(list(op), list(op.values())) == [50, 25, 0]
    for i in range(103, 300, 4):
        op[i] = 0
    assert _counts(list(op), list(op.values())) == [100, 50, 0]


def test_after_uid_count2(orc):
    """TestAfterUIDCount2 (:883-908): re-SETs of a quarter of the uids leave the counts alone, whether the first SETs
    are pending or rolled up into the pack."""
    op = {i: 0 for i in range(100, 300)}
    assert _counts(list(op), list(op.values())) == [200, 100, 0]
    for i in range(100, 300, 4):
        op[i] = 0
    assert _counts(list(op), list(op.values())) == [200, 100, 0]
    p = orc.encode(np.arange(100, 300, dtype=np.uint64), 256)
    assert _counts(list(range(100, 300, 4)), [0] * 50, p) == [200, 100, 0]


def _check_uids(p, mu, mf, uids):
    """checkUids (:66-74): the list from after 0, and with three or more uids from after 10, 80 and 82."""
    assert luo.list_uids_unfiltered(p, mu, mf, 0).tolist() == uids
    if len(uids) >= 3:
        assert luo.list_uids_unfiltered(p, mu, mf, 10).tolist() == uids[1:]
        assert luo.list_uids_unfiltered(p, mu, mf, 80).tolist() == [81]
        assert luo.list_uids_unfiltered(p, mu, mf, 82).tolist() == []


def test_check_uids(orc):
    """TestAddMutation (:160-215) and TestAddAndDelMutation (:782-810) through checkUids."""
    _check_uids(None, [9, 49, 81], [0, 0, 0], [9, 49, 81])
    _check_uids(None, [9, 49, 69, 81], [0, MUT_DEL, 0, 0], [9, 69, 81])
    rolled = orc.encode(np.array([9, 49, 81], np.uint64), 256)
    _check_uids(rolled, [9, 49, 69], [0, MUT_DEL, 0], [9, 69, 81])
    _check_uids(None, [2], [MUT_DEL], [])
    _check_uids(orc.encode(np.array([2], np.uint64), 256), [2], [MUT_DEL], [])


def test_million_reduced(orc):
    """TestMillion (:586-624) at 1e5: SETs of the even uids, rolled up every 10 000; the final Uids is every SET.  The
    last batch is left pending, so that both layers take part."""
    n = 100_000
    evens = np.arange(2, n + 1, 2, dtype=np.uint64)
    rolled = evens[evens <= n - 10_000]
    pending = evens[evens > rolled[-1]]
    p = orc.encode(rolled, 256)
    got = luo.list_uids_unfiltered(p, pending, np.zeros(pending.size, np.uint8), 0)
    assert np.array_equal(got, evens)
    assert luo.list_count(p, pending, np.zeros(pending.size, np.uint8), 0) == evens.size


def test_first_values(orc):
    """first > 0 keeps the smallest values; 0 keeps all; a negative First keeps one (the callback stops after the first
    value, and the negative cut keeps what there is), including MinInt32."""
    p = orc.encode(np.arange(10, 1000, 3, dtype=np.uint64), 256)
    mu, mf = [11, 13, 16, 19], [0, 0, MUT_DEL, MUT_VALUE]
    full = luo.list_uids_unfiltered(p, mu, mf, 12)
    assert full[0] == 13 and 16 not in full and 19 not in full and full.size == luo.list_count(p, mu, mf, 12)
    for first, want in ((0, full), (MAXI32, full), (1, full[:1]), (5, full[:5]), (-1, full[:1]), (-5, full[:1]),
                        (-(2**31), full[:1])):
        assert np.array_equal(luo.list_uids_unfiltered(p, mu, mf, 12, first), want), first
    assert luo.list_uids_unfiltered(p, mu, mf, 2**64 - 1, -3).size == 0


def test_oracle_matches_set_formula(orc):
    """3 000 random rows: after inside and outside the pack, delete-all rows, value postings, re-SETs of pack uids and
    deletes of uids outside it, every First the worker may pass."""
    rng = np.random.default_rng(1001)
    master = gen.zipf_gaps(rng, 200_000, start=1)
    firsts = (0, MAXI32, 1, 10, 255, 256, 257, -1, -5)
    for t in range(3000):
        n = int(rng.integers(0, 3000))
        row = np.sort(rng.choice(master, n, replace=False)) if n else np.zeros(0, np.uint64)
        delete_all = t % 7 == 0
        mu, mf = gen_mut.layer(rng, row, master, int(rng.integers(0, 60)))
        after = [0, int(row[row.size // 2]) if row.size else 5, int(master[master.size // 3]), int(master[-1]),
                 2**64 - 1][int(rng.integers(0, 5))]
        first = firsts[t % len(firsts)]
        op = None if delete_all or row.size == 0 else orc.encode(row, int(rng.choice([4, 10, 256])))
        pk = None if op is None else row
        got = luo.list_uids_unfiltered(op, mu, mf, after, first)
        assert np.array_equal(got, gmu.want_unfiltered(pk, mu, mf, after, first)), f"row {t} after {after}"
        assert luo.list_count(op, mu, mf, after) == gmu.want_unfiltered(pk, mu, mf, after).size, f"count {t}"
