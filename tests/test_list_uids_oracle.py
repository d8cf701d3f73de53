"""The line-by-line List.Uids restatement (list_uids_oracle.c, posting/list.go:1758-1874) for one row of each branch:
the reference's own expectations of TestAddAndDelMutation, TestAfterUIDCount and TestAfterUIDCount2
(posting/list_test.go:782-909) restated as resolved layers, and the set formula of every branch in numpy on a few
thousand random rows."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(__file__))
import gen  # noqa: E402
import gen_mut  # noqa: E402
import list_uids_oracle as luo  # noqa: E402
from gen_mut import COMPRESSED, ITERATE, MUT_DEL, PROBE  # noqa: E402

V_ALL = np.arange(1, 400, dtype=np.uint64)  # every uid the tests touch


def _lengths(orc, uids, flags):
    """List.Length(readTs, after) at after 0 / 199 / 300 of an empty immutable layer plus the resolved layer."""
    u, f = np.asarray(uids, np.uint64), np.asarray(flags, np.uint8)
    return [luo.list_uids(None, ITERATE, u, f, a, V_ALL).size for a in (0, 199, 300)]


def test_after_uid_count(orc):
    """TestAfterUIDCount (:812-881): one transaction's latest op per uid is the resolved entry."""
    op = {i: 0 for i in range(100, 300)}
    assert _lengths(orc, list(op), list(op.values())) == [200, 100, 0]
    for i in range(100, 300, 2):
        op[i] = MUT_DEL
    assert _lengths(orc, list(op), list(op.values())) == [100, 50, 0]
    for i in range(100, 300, 2):  # redundant deletes
        op[i] = MUT_DEL
    assert _lengths(orc, list(op), list(op.values())) == [100, 50, 0]
    for i in range(100, 300):
        op[i] = MUT_DEL
    assert _lengths(orc, list(op), list(op.values())) == [0, 0, 0]
    for _ in range(2):  # the second pass changes nothing
        for i in range(100, 300, 4):
            op[i] = 0
        assert _lengths(orc, list(op), list(op.values())) == [50, 25, 0]
    for i in range(103, 300, 4):
        op[i] = 0
    assert _lengths(orc, list(op), list(op.values())) == [100, 50, 0]


def test_after_uid_count2(orc):
    """TestAfterUIDCount2 (:883-908): re-SETs of a quarter of the uids leave the counts alone."""
    op = {i: 0 for i in range(100, 300)}
    assert _lengths(orc, list(op), list(op.values())) == [200, 100, 0]
    for i in range(100, 300, 4):
        op[i] = 0
    assert _lengths(orc, list(op), list(op.values())) == [200, 100, 0]


def test_add_and_del_mutation(orc):
    """TestAddAndDelMutation (:782-810): SET 0x02 committed, then DEL 0x02 twice: checkUids sees nothing, whether the
    SET is still pending or already rolled up into the pack, in either branch that reads a mutable layer."""
    for mode in (ITERATE, PROBE):
        assert luo.list_uids(None, mode, [2], [MUT_DEL], 0, V_ALL).size == 0
        assert luo.list_uids(orc.encode(np.array([2], np.uint64), 256), mode, [2], [MUT_DEL], 0, V_ALL).size == 0


def test_branches_by_hand(orc):
    p = orc.encode(np.array([2, 3, 4, 5, 6], np.uint64), 256)
    v = np.arange(1, 20, dtype=np.uint64)
    mu, mf = [3, 5, 7], [MUT_DEL, 0, 2]
    assert luo.list_uids(p, COMPRESSED, [], [], 3, v).tolist() == [3, 4, 5, 6]
    assert luo.list_uids(p, PROBE, mu, mf, 3, v).tolist() == [2, 4, 5, 6, 7]      # after ignored, a value is found
    assert luo.list_uids(p, ITERATE, mu, mf, 3, v).tolist() == [4, 5, 6]          # strictly above after, REF only
    assert luo.list_uids(p, ITERATE, mu, mf, 4, v).tolist() == [5, 6]
    assert luo.list_uids(None, ITERATE, mu, [0, 0, 0], 0, v).tolist() == [3, 5, 7]  # delete-all hides the pack
    assert luo.list_uids(None, PROBE, mu, mf, 0, v).tolist() == [5, 7]


def test_oracle_matches_set_formulas(orc):
    """A few thousand random rows in all three modes: after inside v and inside the pack, delete-all rows, value
    postings, re-SETs of uids in the pack and deletes of uids outside it."""
    rng = np.random.default_rng(901)
    master = gen.zipf_gaps(rng, 200_000, start=1)
    checked = {COMPRESSED: 0, PROBE: 0, ITERATE: 0}
    for t in range(3000):
        n = int(rng.integers(0, 3000))
        row = np.sort(rng.choice(master, n, replace=False)) if n else np.zeros(0, np.uint64)
        v = gen.thin(rng, master[: int(rng.integers(1, master.size))], float(rng.choice([0.001, 0.01, 0.1])))
        if v.size == 0:
            v = master[:1].copy()
        mode = t % 3
        delete_all = mode != COMPRESSED and t % 7 == 0
        mu, mf = (np.zeros(0, np.uint64), np.zeros(0, np.uint8)) if mode == COMPRESSED else \
            gen_mut.layer(rng, row, master, int(rng.integers(0, 60)))
        pick = int(rng.integers(0, 4))
        after = [0, int(v[v.size // 2]), int(row[row.size // 2]) if row.size else 5, int(master[-1])][pick]
        op = None if delete_all or row.size == 0 else orc.encode(row, int(rng.choice([4, 256])))
        got = luo.list_uids(op, mode, mu, mf, after, v)
        if mode == COMPRESSED and op is not None and after > int(row[-1]):
            continue  # past the pack's last uid the reference's Bin branch indexes past its blocks (DESIGN section 5)
        want = gen_mut.want_row(mode, None if op is None else row, mu, mf, after, v)
        assert np.array_equal(got, want), f"row {t} mode {mode} after {after}"
        checked[mode] += 1
    assert min(checked.values()) > 500
