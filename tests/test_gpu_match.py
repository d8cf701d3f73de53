"""match() on the device (dgx_match and dgx_dev_match): every result compared in full with the line-by-line
restatement (match_oracle.c), with guard words after every output, and launches with the plan.  Runs on an H100 only
(`pytest -m gpu`)."""
import ctypes as C
import threading

import numpy as np
import pytest

import gen_match as gm
import gen_trigram as gt
import match_cases as mc
import match_oracle as mo

pytestmark = pytest.mark.gpu
SIZE = 256  # a value size in bytes; the tiers are chosen by the query's runes alone


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


def _dev(a, dtype=np.int64):
    import torch

    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(dtype) if a.dtype != np.uint8 else a).cuda()


class Dev:
    """The device form's arguments: the column resident, packs uploaded, layers, lists and UidList in device memory."""

    def __init__(self, lib, lane, raw: mc.Raw):
        from dgraph_b200 import _lib, codec

        self.lib, self.lane, self.raw = lib, lane, raw
        c = raw.col
        self.t = [_dev(c.uid), _dev(c.val_off), _dev(c.byte_off), _dev(c.bytes)]
        self.dcol = _lib.StrColumn(self.t[0].data_ptr(), self.t[1].data_ptr(), self.t[2].data_ptr(),
                                   self.t[3].data_ptr(), raw.cs.n, raw.cs.nvals, raw.cs.nbytes)
        self.tab = (C.c_void_p * max(raw.npacks, 1))()
        self.handles = []
        for i, p in enumerate(raw.packs):
            if p is None or p.nblocks == 0:
                continue
            view = codec.view_of(p.normalized())
            h = C.c_void_p()
            assert lib.dgx_dev_pack_upload(lane, C.byref(view), C.byref(h)) == mc.OK
            self.handles.append(h)
            self.tab[i] = h.value
        self.d_mu, self.d_mf, self.d_lists = _dev(raw.mu), _dev(raw.mf), _dev(raw.lists)
        self.d_uids = _dev(raw.uids if raw.uids.size else np.zeros(1, np.uint64))
        self.d_len = _dev(np.array([-7], np.int64))

    def run(self, after, cap, use_uids=None, nuids=None, d_nuids=None, d_uids=None):
        """(rc of the call, rc of the sync, out with its guard words, length, launches)."""
        import torch

        r = self.raw
        use = (r.uids.size > 0) if use_uids is None else use_uids
        d_out = torch.full((max(cap, 1) + 4,), mc.SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
        self.d_len.fill_(-7)
        torch.cuda.synchronize()
        l0 = self.lib.dgx_lane_launches(self.lane)
        rc = self.lib.dgx_dev_match(
            self.lane, self.tab, r.npacks, C.c_void_p(self.d_mu.data_ptr()), C.c_void_p(self.d_mf.data_ptr()),
            r.mut_off.ctypes.data, C.c_void_p(self.d_lists.data_ptr()), r.list_off.ctypes.data, r.nlists, after,
            int(use), C.c_void_p(d_uids if d_uids is not None else self.d_uids.data_ptr()),
            r.uids.size if nuids is None else nuids, C.c_void_p(d_nuids) if d_nuids else None, C.byref(self.dcol),
            r.qa.ctypes.data, len(r.q), r.max, C.c_void_p(d_out.data_ptr()), cap, C.c_void_p(self.d_len.data_ptr()))
        launches = self.lib.dgx_lane_launches(self.lane) - l0
        rs = self.lib.dgx_lane_sync(self.lane) if rc == mc.OK else None
        out = d_out.cpu().numpy().view(np.uint64)
        n = int(self.d_len.cpu().numpy().view(np.uint64)[0])
        return rc, rs, out, n, launches

    def free(self):
        for h in self.handles:
            self.lib.dgx_dev_pack_free(h)


def check_both(lib, lane, col, query, mx, uids=(), leaves=(), after=0, what="", launches=True):
    want = mo.match(col, query, mx, uids=np.asarray(uids, np.uint64) if len(uids) else None,
                    leaves=gt.to_oracle(leaves), after=after)
    raw = mc.Raw(col, query, mx, uids=uids, leaves=leaves)
    cap = raw.bound
    rc, out, n = raw.host(after, cap)
    assert rc == mc.OK, (what, lib.dgx_last_error())
    assert np.array_equal(out[:n], want), what
    assert np.all(out[n:] == np.uint64(mc.SENTINEL)), what
    dev = Dev(lib, lane, raw)
    try:
        rc, rs, out, n, nl = dev.run(after, cap)
        assert (rc, rs) == (mc.OK, mc.OK), (what, lib.dgx_last_error())
        assert np.array_equal(out[:n], want), what
        assert np.all(out[n:] == np.uint64(mc.SENTINEL)), what
        if launches:
            assert nl == mc.launches(leaves, len(uids)), what
    finally:
        dev.free()
    return want


def test_random_cases(lib, lane):
    for seed in range(300):
        rng = np.random.default_rng(910_000 + seed)
        uids, values, q, mx, cands = gm.random_case(rng, nuids=int(rng.choice([10, 60, 300])), universe=400)
        col = mc.column(uids, values)
        if not len(cands):
            continue
        check_both(lib, lane, col, q, mx, uids=cands, what=f"seed {seed}")


def test_golden(lib, lane):
    g, cols = mc.golden()
    from dgraph_b200 import algo

    for case in g["cases"]:
        uids, vals = cols[case["pred"]]
        col = mc.column(uids, vals)
        q = case["query"].encode()
        after = case["after"]
        idx = mc.trigram_index(uids, vals)
        for kinds in (("list",), ("pack",)):
            leaves = [("list", lf[1][lf[1] > np.uint64(after)]) if lf[0] == "list" else lf
                      for lf in mc.trigram_leaves(idx, q, kinds)]
            got = check_both(lib, lane, col, q, case["max"], leaves=leaves, after=after, what=case["test"])
            first = case["first"] or len(got)
            assert got[:first].tolist() == case["want"], case["test"]
            res = algo.MatchFuzzy(col, case["query"], case["max"], leaves=gt.to_algo(leaves), afterUID=after)
            assert res.Uids[:first].tolist() == case["want"], case["test"]


def _ascii(rng, n):
    return bytes(rng.integers(97, 101, n).astype(np.uint8))


def test_tier_boundaries(lib, lane):
    rng = np.random.default_rng(5)
    for qrunes in (1, 63, 64, 65, 128, 129, 4096):
        for qkind in ("ascii", "mixed"):
            q = _ascii(rng, qrunes) if qkind == "ascii" else gm.rand_bytes(rng, qrunes)
            while len(gm.runes(q)) > qrunes:  # a piece may decode to several runes
                q = q[:-1]
            uids, values = [], []
            for k, vlen in enumerate((SIZE - 1, SIZE, SIZE + 1, 40, 3000)):
                for e in range(4):
                    base = (q * (vlen // max(len(q), 1) + 1))[:vlen]
                    values.append([gm.mutate(rng, base, e)])
                    uids.append(10 * k + e + 1)
            col = mc.column(uids, values)
            for mx in (0, 1, 3, 40, 200):
                check_both(lib, lane, col, q, mx, uids=uids, what=f"q {qrunes} {qkind} max {mx}")


def test_multibyte_values_around_256_bytes(lib, lane):
    # values of 255 to 257 bytes of 2-byte runes, a multi-byte rune cut at the end, on both sides of every max
    rng = np.random.default_rng(6)
    q = "é" * 30 + "abc"
    uids, values = [], []
    for k, vlen in enumerate((SIZE - 1, SIZE, SIZE + 1)):
        for e in range(6):
            v = bytearray(("é" * 200).encode()[:vlen])
            v = gm.mutate(rng, bytes(v), e)[:vlen].ljust(vlen, b"a")
            values.append([v])
            uids.append(100 * k + e + 1)
    col = mc.column(uids, values)
    for mx in (0, 5, 100, 127, 128, 129, 200, 256):
        check_both(lib, lane, col, q.encode(), mx, uids=uids, what=f"max {mx}")


def test_long_tier_dp_past_32_words(lib, lane):
    # queries of 2 048, 2 049 and 4 096 runes (32, 33 and 64 words: the second word per lane, the lane 31 -> lane 0
    # carry and the score owner of W > 32) against values of about the same rune count, so that no shortcut decides
    # and the distance itself is tested with max on both sides of it
    rng = np.random.default_rng(17)
    for qrunes in (2048, 2049, 4096):
        for kind in ("ascii", "mixed"):
            if kind == "ascii":
                q = _ascii(rng, qrunes)
            else:
                q = b"".join([b"a", "é".encode(), "€".encode(), "😀".encode(), b"\xff", b"b"][int(i)]
                             for i in rng.integers(0, 6, qrunes))
            assert len(gm.runes(q)) == qrunes
            uids, values, dists, dp_both = [], [], [], 0
            for k, edits in enumerate((0, 1, 7, 40, 150)):
                v = gm.mutate(rng, q, edits)
                d = mo.levenshtein(v, q)
                n = len(gm.runes(v))
                uids.append(k + 1)
                values.append([v])
                dists.append(d)
                assert d < max(n, qrunes)  # max = d is decided by the DP
                dp_both += abs(n - qrunes) < d  # and so is max = d - 1
            assert dp_both >= 3, (qrunes, kind)
            col = mc.column(uids, values)
            for mx in sorted({0} | {d - 1 for d in dists if d} | set(dists)):
                got = check_both(lib, lane, col, q, mx, uids=uids, what=f"q {qrunes} {kind} max {mx}")
                assert got.tolist() == [u for u, d in zip(uids, dists) if d <= mx]


def test_shortcuts_and_utf8(lib, lane):
    T = gm.TRICKY
    uids = list(range(1, len(T) + 1))
    col = mc.column(uids + [100, 101], [[t] for t in T] + [[b""], [b"", b"x"]])
    for q in T + [b"", b"abc", "é€😀".encode()]:
        for mx in (0, 1, 2, 3, 4, gm.MAX_I32):
            check_both(lib, lane, col, q, mx, uids=uids + [100, 101, 102], what=f"{q!r} {mx}")


def test_hub_with_many_list_values(lib, lane):
    rng = np.random.default_rng(8)
    q = b"alice"
    hub = [gm.rand_bytes(rng, int(rng.integers(1, 12))) for _ in range(20_000)]
    hub[-1] = b"alicf"  # the only passing value is the last
    uids = [7, 9, 11]
    col = mc.column(uids, [[b"zzzzzz"], hub, [b"bob", b"alice" * 100]])
    for mx in (0, 1, 2):
        check_both(lib, lane, col, q, mx, uids=uids, what=f"hub max {mx}")


def test_trigram_branch_layers_and_after(lib, lane):
    for seed in range(60):
        rng = np.random.default_rng(920_000 + seed)
        uids, values, q, mx, _ = gm.random_case(rng, nuids=300, universe=600)
        after = int(rng.choice([0, 200, 599]))
        leaves = gt.random_leaves(rng, int(rng.integers(1, 7)), 600, "mixed", after=after)
        col = mc.column(uids, values)
        check_both(lib, lane, col, q, mx, leaves=leaves, after=after, what=f"seed {seed}")


@pytest.mark.parametrize("name,kw,want_rc,on_device", mc.error_cases(), ids=[c[0] for c in mc.error_cases()])
def test_argument_errors(lib, lane, name, kw, want_rc, on_device):
    r = mc.Raw(**kw)
    rc, out, n = r.host(0, 64)
    if on_device and name != "DGX_MUT_VALUE":  # the host form checks the layer's flags on the host
        assert rc == mc.ERR_ARG and n == 0, name
    else:
        assert rc == want_rc and n == mc.SENTINEL, name
    assert np.all(out == np.uint64(mc.SENTINEL)), name
    if name in ("val_off decreasing", "val_off[0] != 0", "byte_off decreasing", "nvals != val_off[n]",
                "nbytes != byte_off[nvals]"):
        on_device = True  # the device form checks the column's offsets on the device
    dev = Dev(lib, lane, r)
    try:
        rc, rs, out, n, nl = dev.run(0, 64)
        if on_device:
            assert (rc, rs, n) == (mc.OK, mc.ERR_ARG, 0), name
            assert b"match() input" in lib.dgx_last_error() or b"mutable layer" in lib.dgx_last_error(), name
        else:
            assert rc == want_rc and nl == 0 and n == (-7 & gt.U64), name
        assert np.all(out == np.uint64(mc.SENTINEL)), name
    finally:
        dev.free()


def test_count_word_and_empty_uidlist(lib, lane):
    import torch

    col = mc.column([3, 5, 9], [[b"abc"], [b"abd"], [b"abe"]])
    raw = mc.Raw(col, "abc", 1, uids=[3, 5, 9])
    dev = Dev(lib, lane, raw)
    try:
        for k in (0, 1, 2, 3):
            w = torch.tensor([k | (0xABC << 32)], dtype=torch.int64, device="cuda")  # the low 32 bits count
            rc, rs, out, n, _ = dev.run(0, 3, d_nuids=w.data_ptr())
            assert (rc, rs) == (mc.OK, mc.OK) and out[:n].tolist() == [3, 5, 9][:k] and n == k
            assert np.all(out[n:] == np.uint64(mc.SENTINEL))
        w = torch.tensor([4], dtype=torch.int64, device="cuda")  # past the room
        rc, rs, out, n, _ = dev.run(0, 3, d_nuids=w.data_ptr())
        assert (rc, rs, n) == (mc.OK, mc.ERR_ARG, 0) and np.all(out == np.uint64(mc.SENTINEL))
        rc, rs, out, n, nl = dev.run(0, 0, nuids=0)  # an empty UidList: an empty result, no launch
        assert (rc, rs, n, nl) == (mc.OK, mc.OK, 0, 0)
        rc, rs, out, n, nl = dev.run(0, 2)  # out_cap below the room
        assert rc == mc.ERR_CAP and nl == 0
    finally:
        dev.free()


def test_launches_constant_as_candidates_grow(lib, lane):
    counts = set()
    for scale in (1, 10, 100):
        rng = np.random.default_rng(11)
        n = 2000 * scale
        uids = np.arange(1, n + 1, dtype=np.uint64)
        values = [[gm.rand_bytes(rng, int(rng.integers(1, 9)))] + ([b"x" * 400] if i % 97 == 0 else [])
                  for i in range(n)]
        col = mc.column(uids, values)
        raw = mc.Raw(col, "abcé", 2, uids=uids)
        want = mo.match(col, "abcé", 2, uids=uids)
        dev = Dev(lib, lane, raw)
        try:
            rc, rs, out, k, nl = dev.run(0, n)
            assert (rc, rs) == (mc.OK, mc.OK) and np.array_equal(out[:k], want)
            counts.add(nl)
        finally:
            dev.free()
    assert counts == {mc.FZ_LAUNCHES}


def test_device_chain_trigram_match_match_var_order(lib, lane):
    # dgx_dev_trigram_query's result and length word feed dgx_dev_match's UidList branch with no host read, whose
    # output and length word feed a second dgx_dev_match, whose output and length word are dgx_dev_var_order's dest
    import torch

    from dgraph_b200 import algo

    rng = np.random.default_rng(12)
    uids, values, q, _, _ = gm.random_case(rng, nuids=3000, universe=5000, qmax=10)
    q = q or b"abcd"
    col = mc.column(uids, values)
    leaves = gt.random_leaves(rng, 5, 5000, "mixed", p_list=0.5)
    tree = [(gt.QOR, list(range(5)), [])]
    cand = algo.UidsForRegex(tree, gt.to_algo(leaves), 0).Uids
    want1 = mo.match(col, q, 3, uids=cand)
    want2 = mo.match(col, q, 1, uids=want1) if want1.size else want1
    raw = mc.Raw(col, q, 3, leaves=leaves)
    dev = Dev(lib, lane, raw)
    try:
        from trigram_cases import Raw as TRaw
        tr = TRaw(tree, packs=raw.packs, muts=raw.muts, lists=[gt.to_algo([lf])[0] for lf in leaves if lf[0] == "list"])
        cap = raw.bound
        d_c = torch.zeros(cap + 1, dtype=torch.int64, device="cuda")
        d_cl = torch.zeros(1, dtype=torch.int64, device="cuda")
        rc = lib.dgx_dev_trigram_query(lane, C.byref(tr.qt), dev.tab, raw.npacks, C.c_void_p(dev.d_mu.data_ptr()),
                                       C.c_void_p(dev.d_mf.data_ptr()), raw.mut_off.ctypes.data,
                                       C.c_void_p(dev.d_lists.data_ptr()), raw.list_off.ctypes.data, raw.nlists, 0,
                                       C.c_void_p(d_c.data_ptr()), cap, C.c_void_p(d_cl.data_ptr()))
        assert rc == mc.OK
        d_m = torch.full((cap + 4,), mc.SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
        d_ml = torch.zeros(1, dtype=torch.int64, device="cuda")
        d_m2 = torch.full((cap + 4,), mc.SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
        d_ml2 = torch.zeros(1, dtype=torch.int64, device="cuda")
        algo.dev_match(lane, dev.dcol, q, 3, d_m.data_ptr(), cap, d_ml.data_ptr(), d_uids=d_c.data_ptr(), nuids=cap,
                       d_nuids=d_cl.data_ptr())
        algo.dev_match(lane, dev.dcol, q, 1, d_m2.data_ptr(), cap, d_ml2.data_ptr(), d_uids=d_m.data_ptr(),
                       nuids=cap, d_nuids=d_ml.data_ptr())
        # the second match's output and length word are the dest of an orderdesc by an int variable over one row
        import var_order_oracle as vo
        from dgraph_b200 import _lib

        row = np.asarray(uids, np.uint64)
        ivals = rng.integers(0, 50, row.size).astype(np.int64)
        d_key, d_word, d_row = _dev(row), _dev(ivals.view(np.uint64)), _dev(row)
        d_roff = _dev(np.array([0, row.size], np.uint64))
        leaf = _lib.MathLeaf(d_key.data_ptr(), d_word.data_ptr(), None, None, row.size, 1, 0)
        d_vo = torch.full((row.size + 4,), mc.SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
        d_voff = torch.zeros(2, dtype=torch.int64, device="cuda")
        d_vdest = torch.full((cap + 4,), mc.SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
        d_vlen = torch.zeros(1, dtype=torch.int64, device="cuda")
        assert lib.dgx_dev_var_order(lane, C.byref(leaf), 1, C.c_void_p(d_m2.data_ptr()), cap,
                                     C.c_void_p(d_ml2.data_ptr()), C.c_void_p(d_row.data_ptr()),
                                     C.c_void_p(d_roff.data_ptr()), 1, row.size, 0, 0, C.c_void_p(d_vo.data_ptr()),
                                     C.c_void_p(d_voff.data_ptr()), row.size, C.c_void_p(d_vdest.data_ptr()), cap,
                                     C.c_void_p(d_vlen.data_ptr())) == mc.OK
        assert lib.dgx_lane_sync(lane) == mc.OK
        wrows, wdest = vo.var_order((row, ivals), True, want2, [row], 0, 0)
        k = int(d_voff[1].item())
        o3 = d_vo.cpu().numpy().view(np.uint64)
        assert np.array_equal(o3[:k], wrows[0]) and np.all(o3[k:] == np.uint64(mc.SENTINEL))
        assert np.array_equal(d_vdest[:int(d_vlen.item())].cpu().numpy().view(np.uint64), wdest)
        assert wrows[0].size == want2.size
        n1, n2 = int(d_ml.item()), int(d_ml2.item())
        o1, o2 = d_m.cpu().numpy().view(np.uint64), d_m2.cpu().numpy().view(np.uint64)
        assert np.array_equal(o1[:n1], want1) and np.all(o1[n1:] == np.uint64(mc.SENTINEL))
        assert np.array_equal(o2[:n2], want2) and np.all(o2[n2:] == np.uint64(mc.SENTINEL))
        assert want1.size > want2.size > 0 or want1.size == 0
    finally:
        dev.free()


def test_four_threads(lib):
    from dgraph_b200 import algo

    cases = []
    for t in range(4):
        rng = np.random.default_rng(400 + t)
        uids, values, q, mx, cands = gm.random_case(rng, nuids=2000, universe=4000)
        col = mc.column(uids, values)
        cases.append((col, q, mx, cands, mo.match(col, q, mx, uids=cands)))
    errs = []

    def work(t):
        col, q, mx, cands, want = cases[t]
        try:
            for _ in range(20):
                got = algo.MatchFuzzy(col, q, mx, uids=cands)
                assert np.array_equal(got.Uids, want)
        except Exception as e:  # noqa: BLE001
            errs.append((t, e))

    ts = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    for th in ts:
        th.start()
    for th in ts:
        th.join()
    assert not errs, errs


def test_c21a_sized_call(lib):
    from dgraph_b200 import algo

    rng = np.random.default_rng(21)
    col = gm.name_column(rng, 10_000_000)
    cands = np.sort(rng.choice(col.uid, 3_000_000, replace=False))
    got = algo.MatchFuzzy(col, "alice", 2, uids=cands)
    want = mo.match(col, "alice", 2, uids=cands)
    assert np.array_equal(got.Uids, want) and want.size > 1000
