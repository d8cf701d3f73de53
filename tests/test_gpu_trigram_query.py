"""uidsForRegex on the device (dgx_trigram_query and dgx_dev_trigram_query): every result compared in full with the
line-by-line restatement (trigram_oracle.c), launches with the plan model (trigram_plan.py).  Runs on an H100 only
(`pytest -m gpu`)."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen_trigram as gt  # noqa: E402
import trigram_oracle as tgo  # noqa: E402
import trigram_plan as tp  # noqa: E402
from trigram_cases import ERR_ARG, ERR_CAP, OK, SENTINEL, Raw, error_cases  # noqa: E402

pytestmark = pytest.mark.gpu

QAND, QOR = gt.QAND, gt.QOR


@pytest.fixture(scope="module")
def lib():
    from dgraph_b200 import _lib

    L = _lib.load()
    _lib.check(L.dgx_init(-1))
    return L


@pytest.fixture(scope="module")
def lane(lib):
    import torch

    stream = torch.cuda.Stream()
    ln = lib.dgx_lane_create(0, C.c_void_p(stream.cuda_stream))
    assert ln
    yield ln
    lib.dgx_lane_destroy(ln)


def raw_of(tree, leaves, keys=None):
    """Raw ABI arguments of raw leaves (gen_trigram form): pack leaves first, the tree renumbered."""
    pids = [j for j, lf in enumerate(leaves) if lf[0] == "pack"]
    lids = [j for j, lf in enumerate(leaves) if lf[0] == "list"]
    order = {j: k for k, j in enumerate(pids + lids)}
    al = gt.to_algo(leaves)
    tr = [(op, [order[j] for j in ls], list(subs)) for op, ls, subs in tree]
    return Raw(tr, packs=[al[j][0] for j in pids], muts=[al[j][1] for j in pids], lists=[al[j] for j in lids],
               keys=[keys[j] for j in pids] if keys else None)


def bound_of(tree, leaves):
    return tp.plan(tree, [gt.leaf_bound(lf) for lf in leaves]).root_bound


class Dev:
    """The device form's arguments: packs uploaded once, layers and lists in device memory."""

    def __init__(self, lib, lane, raw: Raw):
        import torch

        from dgraph_b200 import codec

        self.lib, self.lane, self.raw = lib, lane, raw
        self.tab = (C.c_void_p * max(raw.npacks, 1))()
        self.handles = []
        for i, p in enumerate(raw.packs):
            if p is None or p.nblocks == 0:
                continue
            view = codec.view_of(p.normalized())
            h = C.c_void_p()
            assert lib.dgx_dev_pack_upload(lane, C.byref(view), C.byref(h)) == OK
            self.handles.append(h)
            self.tab[i] = h.value
        self.d_mu = torch.from_numpy(raw.mu.view(np.int64)).cuda()
        self.d_mf = torch.from_numpy(raw.mf).cuda()
        self.d_lists = torch.from_numpy(raw.lists.view(np.int64)).cuda()
        self.d_len = torch.full((1,), -7, dtype=torch.int64, device="cuda")

    def run(self, after, cap):
        """(rc of the call, rc of the sync, result, launches of the call); d_out holds SENTINEL past the result."""
        import torch

        d_out = torch.full((max(cap, 1) + 4,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        l0 = self.lib.dgx_lane_launches(self.lane)
        r = self.raw
        rc = self.lib.dgx_dev_trigram_query(
            self.lane, C.byref(r.qt), self.tab, r.npacks, C.c_void_p(self.d_mu.data_ptr()),
            C.c_void_p(self.d_mf.data_ptr()), r.mut_off.ctypes.data, C.c_void_p(self.d_lists.data_ptr()),
            r.list_off.ctypes.data, r.nlists, after, C.c_void_p(d_out.data_ptr()), cap, C.c_void_p(self.d_len.data_ptr()))
        launches = self.lib.dgx_lane_launches(self.lane) - l0
        rs = self.lib.dgx_lane_sync(self.lane) if rc == OK else None
        out = d_out.cpu().numpy().view(np.uint64)
        n = int(self.d_len.cpu().numpy().view(np.uint64)[0])
        return rc, rs, out, n, launches

    def free(self):
        for h in self.handles:
            self.lib.dgx_dev_pack_free(h)


def check_both(lib, lane, tree, leaves, after, what, keys=None, launches=True):
    want = tgo.uids_for_regex(tree, gt.to_oracle(leaves), after)
    assert np.array_equal(want, gt.want(tree, leaves, after)), what
    raw = raw_of(tree, leaves, keys)
    cap = bound_of(tree, leaves)
    rc, out, n = raw.host(after, cap)
    assert rc == OK, what
    assert np.array_equal(out[:n], want), what
    assert np.all(out[n:] == np.uint64(SENTINEL)), what
    dev = Dev(lib, lane, raw)
    try:
        rc, rs, out, n, nl = dev.run(after, cap)
        assert (rc, rs) == (OK, OK), what
        assert np.array_equal(out[:n], want), what
        assert np.all(out[n:] == np.uint64(SENTINEL)), what
        if launches:
            p = tp.plan(raw.tree, [gt.leaf_bound(leaves[j]) for j in
                                   [j for j, lf in enumerate(leaves) if lf[0] == "pack"] +
                                   [j for j, lf in enumerate(leaves) if lf[0] == "list"]])
            assert nl == tp.launches(p, raw.npacks), what
    finally:
        dev.free()
    return want


def test_random_trees(lib, lane):
    for seed in range(240):
        rng = np.random.default_rng(50_000 + seed)
        universe = int(rng.choice([300, 5000, 200_000]))
        after = [0, universe // 2, gt.U64][seed % 3]
        nleaves = int(rng.integers(1, 12))
        leaves = gt.random_leaves(rng, nleaves, universe, str(rng.choice(["mixed", "probe", "iterate"])), after=after)
        tree = gt.random_tree(rng, nleaves, int(rng.integers(1, 10)), max_depth=int(rng.choice([2, 6, 32])))
        check_both(lib, lane, tree, leaves, after, f"seed {seed}")


def _index_leaves(idx, tris, rng, kinds):
    out = []
    for k, t in enumerate(tris):
        u = idx.posting(t)
        kind = kinds[k % len(kinds)]
        if kind == "list":
            out.append(("list", u))
        elif kind == "pack":
            out.append(("pack", u if u.size else None, None, 0))
        else:  # a layer of REF postings on top of the pack
            pool = np.arange(1, idx.n_nodes + 1, dtype=np.uint64)
            from gen_mut import layer
            out.append(("pack", u if u.size else None, layer(rng, u if u.size else pool, pool, 64,
                                                             p_flags=(0.5, 0.5, 0.0, 0.0)), 1 << 40))
    return out


def test_patterns_named_anonymous_lists_and_mixed(lib, lane):
    from dgraph_b200 import _lib, algo

    idx = gt.TrigramIndex(seed=11, n_nodes=300_000, n_words=3000)
    rng = np.random.default_rng(12)
    for kinds in (["pack"], ["list"], ["pack", "list", "layer"]):
        for pat, nodes in gt.PATTERNS.items():
            tree, tris = gt.tree_of_pattern(nodes)
            leaves = _index_leaves(idx, tris, rng, kinds)
            keys = [(hash((pat, t)) & 0xFFFFFFFF | 1, 7) for t in tris]
            want = check_both(lib, lane, tree, leaves, 0, f"{pat} {kinds}")
            # the product's Python call, named packs: the second call hits the cache
            st0 = _lib.CacheStats()
            lib.dgx_cache_get_stats(C.byref(st0))
            for _ in range(2):
                got = algo.UidsForRegex(tree, gt.to_algo(leaves), 0, keys=keys)
                assert np.array_equal(got.Uids, want), pat
            st1 = _lib.CacheStats()
            lib.dgx_cache_get_stats(C.byref(st1))
            npk = sum(1 for lf in leaves if lf[0] == "pack" and lf[1] is not None)
            assert st1.hits - st0.hits >= npk, pat
            after = int(want[want.size // 2]) if want.size else 0
            check_both(lib, lane, tree, leaves if "list" not in kinds else
                       [("list", lf[1][lf[1] > np.uint64(after)]) if lf[0] == "list" else lf for lf in leaves],
                       after, f"{pat} {kinds} after")


def test_shapes(lib, lane):
    rng = np.random.default_rng(77)
    universe = 100_000
    lv = gt.random_leaves(rng, 40, universe, "mixed")
    lv[3] = ("pack", None, None, 0)                        # empty list
    lv[4] = ("list", np.zeros(0, np.uint64))               # missing trigram: an empty list
    lv[5] = ("pack", None, (np.array([7, 9], np.uint64), np.array([0, 0], np.uint8)), 0)  # delete-all marker + SETs
    cases = {
        "one leaf OR": [(QOR, [0], [])],
        "one leaf AND": [(QAND, [1], [])],
        "shared leaves": [(QAND, [2, 2], [1, 2]), (QOR, [2, 6], []), (QOR, [2, 7], [3]), (QAND, [2], [])],
        "empty and missing": [(QOR, [3, 4, 5], [1]), (QAND, [0, 4], [])],
        "empty OR sub": [(QAND, [0], [1]), (QOR, [], [])],
        "AND of ORs": [(QAND, [], [1, 2]), (QOR, list(range(6, 20)), []), (QOR, list(range(15, 30)), [])],
    }
    # a chain at the depth limit: 32 nodes, alternating AND / OR, shared leaves on every level
    cases["depth 32"] = [(QAND if i % 2 == 0 else QOR, [i % 7, 8 + i % 5], [i + 1] if i < 31 else [])
                         for i in range(32)]
    for name, tree in cases.items():
        for after in (0, universe // 3, gt.U64):
            leaves = [("list", lf[1][lf[1] > np.uint64(after)]) if lf[0] == "list" else lf for lf in lv]
            check_both(lib, lane, tree, leaves, after, f"{name} after {after}")


def test_or_of_1000_leaves(lib, lane):
    rng = np.random.default_rng(1000)
    leaves = gt.random_leaves(rng, 1000, 100_000, "mixed", p_list=0.3)
    check_both(lib, lane, [(QOR, list(range(1000)), [])], leaves, 0, "OR of 1000")
    check_both(lib, lane, [(QAND, [0], [1]), (QOR, list(range(1, 1000)), [])], leaves, 0, "AND over an OR of 999")


def test_out_cap_exact_and_one_short(lib, lane):
    rng = np.random.default_rng(5)
    leaves = gt.random_leaves(rng, 6, 50_000, "mixed", p_list=0.0)
    for tree in ([(QOR, [0, 1, 2], [])], [(QAND, [0], [1]), (QOR, [2, 3, 4, 5], [])]):
        raw = raw_of(tree, leaves)
        cap = bound_of(tree, leaves)
        want = tgo.uids_for_regex(tree, gt.to_oracle(leaves), 0)
        rc, out, n = raw.host(0, cap)
        assert rc == OK and np.array_equal(out[:n], want)
        rc, out, n = raw.host(0, cap - 1)
        assert rc == ERR_CAP and np.all(out == np.uint64(SENTINEL)) and n == SENTINEL
        dev = Dev(lib, lane, raw)
        try:
            rc, rs, out, n, _ = dev.run(0, cap)
            assert (rc, rs) == (OK, OK) and np.array_equal(out[:n], want)
            rc, rs, out, n, nl = dev.run(0, cap - 1)
            assert rc == ERR_CAP and nl == 0 and np.all(out == np.uint64(SENTINEL))
        finally:
            dev.free()


@pytest.mark.parametrize("name,kw,want_rc", error_cases(), ids=[c[0] for c in error_cases()])
def test_argument_errors(lib, lane, name, kw, want_rc):
    r = Raw(**kw)
    rc, out, n = r.host(0, 64)
    assert rc == want_rc and np.all(out == np.uint64(SENTINEL)) and n == SENTINEL, name
    dev = Dev(lib, lane, r)
    try:
        rc, rs, out, n, nl = dev.run(0, 64)
        if name == "DGX_MUT_VALUE":  # found on the device: reported at the sync, out untouched, length 0
            assert (rc, rs, n) == (OK, ERR_ARG, 0)
            assert b"mutable layer" in lib.dgx_last_error()
        else:
            assert rc == want_rc and nl == 0 and n == (-7 & gt.U64), name
        assert np.all(out == np.uint64(SENTINEL)), name
    finally:
        dev.free()


def test_four_threads(lib):
    from dgraph_b200 import algo

    cases = []
    for t in range(4):
        rng = np.random.default_rng(400 + t)
        leaves = gt.random_leaves(rng, 10, 300_000, "mixed")
        tree = gt.random_tree(rng, 10, 6)
        cases.append((tree, leaves, tgo.uids_for_regex(tree, gt.to_oracle(leaves), 0), gt.to_algo(leaves)))
    errs = []

    def work(t):
        tree, leaves, want, al = cases[t]
        try:
            for _ in range(20):
                got = algo.UidsForRegex(tree, al, 0, keys=[(1000 * t + j + 1, 3) for j in range(len(al))])
                assert np.array_equal(got.Uids, want)
        except Exception as e:  # noqa: BLE001
            errs.append((t, e))

    ts = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    for th in ts:
        th.start()
    for th in ts:
        th.join()
    assert not errs, errs
