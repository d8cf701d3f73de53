"""regexp()'s value test on the device (dgx_regex_match and dgx_dev_regex_match): every result compared in full with
the restatement (regex_oracle.py), or on the large call with the formula (gen_regex.py's rules over Python's re),
with guard words after every output, and launches counted.  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import re
import threading

import numpy as np
import pytest

import gen_regex as gr
import gen_trigram as gt
import regex_oracle as ro

pytestmark = pytest.mark.gpu
OK, ERR_ARG, ERR_CAP = 0, -3, -4
SENTINEL = 0xDEADBEEFCAFEF00D
LONG = 4096  # RX_LONG_BYTES: longer values of a DFA of at most 64 states take the warp tier
WARP_STATES = 64


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


def _dev(a):
    import torch

    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.int64) if a.dtype != np.uint8 else a).cuda()


class DevCol:
    """A resident column: its arrays in device memory and the dgx_str_column over them."""

    def __init__(self, col):
        from dgraph_b200 import _lib

        self.t = [_dev(col.uid if col.uid.size else np.zeros(1, np.uint64)), _dev(col.val_off), _dev(col.byte_off),
                  _dev(col.bytes)]
        nv = col.byte_off.size - 1
        self.s = _lib.StrColumn(self.t[0].data_ptr(), self.t[1].data_ptr(), self.t[2].data_ptr(), self.t[3].data_ptr(),
                                col.uid.size, nv, int(col.byte_off[-1]))


def dev_run(lib, lane, dcol, prog, cands, cap=None, d_nuids=None):
    """(rc, rc of the sync, out with its guard words, length, launches) of the device form over a UidList."""
    import torch

    from dgraph_b200 import algo

    cands = np.asarray(cands, np.uint64)
    cap = cands.size if cap is None else cap
    d_u = _dev(cands if cands.size else np.zeros(1, np.uint64))
    d_out = torch.full((max(cap, 1) + 4,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
    d_len = torch.full((1,), -7, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    l0 = lib.dgx_lane_launches(lane)
    try:
        algo.dev_match_regex(lane, dcol.s, prog, d_out.data_ptr(), cap, d_len.data_ptr(), d_uids=d_u.data_ptr(),
                             nuids=cands.size, d_nuids=d_nuids)
        rc = OK
    except Exception as e:  # noqa: BLE001
        rc = e.code
    nl = lib.dgx_lane_launches(lane) - l0
    rs = lib.dgx_lane_sync(lane) if rc == OK else None
    return rc, rs, d_out.cpu().numpy().view(np.uint64), int(d_len.cpu().numpy().view(np.uint64)[0]), nl


def check_both(lib, lane, col, pat, cands, fold=False, want=None, what=""):
    from dgraph_b200 import algo

    prog = algo.RegexProg(pat, fold)
    cands = np.asarray(cands, np.uint64)
    if want is None:
        want = ro.regex_match(col, ro.Prog(pat, fold), cands)
    got = algo.MatchRegex(col, prog, uids=cands)
    assert np.array_equal(got.Uids, want), what
    rc, rs, out, n, nl = dev_run(lib, lane, DevCol(col), prog, cands)
    assert (rc, rs) == (OK, OK), (what, lib.dgx_last_error())
    assert np.array_equal(out[:n], want) and np.all(out[n:] == np.uint64(SENTINEL)), what
    assert nl == (5 if cands.size else 0), what
    return want


def want_by_re(col, pat: str, cands):
    """matchRegex by the formula's rules over Python's re in bytes mode, for patterns whose items are ASCII bytes (so
    multi-byte runes and invalid bytes cannot change the answer): the large values' checker."""
    rx = re.compile(pat.encode(), re.MULTILINE)
    pos = {int(u): i for i, u in enumerate(col.uid)}
    data, bo, vo = col.bytes.tobytes(), col.byte_off, col.val_off
    out = []
    for u in np.asarray(cands, np.uint64):
        i = pos.get(int(u))
        if i is None:
            continue
        for j in range(int(vo[i]), int(vo[i + 1])):
            v = data[int(bo[j]):int(bo[j + 1])]
            lines = v.split(b"\n") if v else []
            hit = next((k for k, ln in enumerate(lines) if rx.search(ln)), None)
            if hit is not None and not (hit == 0 and lines[0] == b""):
                out.append(int(u))
                break
    return np.array(out, np.uint64)


def test_random_cases(lib, lane):
    from dgraph_b200 import algo

    for seed in range(200):
        rng = np.random.default_rng(1_500_000 + seed)
        pat, fold_arg, _, _, _ = gr.random_case(rng)
        uids, vals = gr.column_case(rng, int(rng.choice([5, 50, 300])))
        col = algo.StrColumn(uids, vals)
        extra = rng.integers(1, uids.max() + 5, 20).astype(np.uint64)  # candidates without a value
        cands = np.unique(np.concatenate([uids[rng.random(uids.size) < 0.7], extra]))
        check_both(lib, lane, col, pat, cands, fold_arg, what=f"seed {seed} {pat!r}")


def _long_values(rng, n):
    """Values around the tier boundary and the warp's chunk edges: a needle at the start, end or a chunk edge, '\\n'
    and multi-byte runes straddling 16-byte segments."""
    out = []
    for k in range(n):
        ln = [LONG - 1, LONG, LONG + 1, LONG + 16, 32 * 16 * 9 + 7, 100_000, 1 << 20][k % 7]
        b = bytearray(rng.choice(np.frombuffer(b"abcdxyz \n", np.uint8), ln).tobytes())
        for at in rng.integers(0, ln - 1, 8):  # two-byte runes, some across a 16-byte segment edge
            b[int(at):int(at) + 2] = "é".encode()
        where = int(rng.choice([0, ln - 6, (ln // 32) // 16 * 16 - 3, (ln // 32) // 16 * 16 * 5 - 1, -1]))
        if where >= 0 and rng.random() < 0.7:
            b[where:where + 6] = rng.choice([b"needle", "nééd".encode()[:6], b"\nneedl"])
        out.append(bytes(b[:ln]))
    return out


def test_tier_boundary_and_chunk_edges(lib, lane):
    from dgraph_b200 import algo

    rng = np.random.default_rng(7)
    vals = _long_values(rng, 70)
    uids = np.arange(1, len(vals) + 1, dtype=np.uint64) * 3
    col = algo.StrColumn(uids, [[v] for v in vals])
    for pat in ["needle", "^needle", "needle$", "y\\nz", "(?i)NEEDLE|zzzzzz", "^[a-d]x", "d[a-d]{2,3}x"]:
        check_both(lib, lane, col, pat, uids, want=want_by_re(col, pat.replace("\\n", "\\x00"), uids), what=pat)


def _literal_with_states(n):
    from dgraph_b200 import algo

    c = algo.RegexProg("ab" * 5).tables()[1].shape[0] - 10
    pat = "ab" * ((n - c) // 2) + "a" * ((n - c) % 2)
    assert algo.RegexProg(pat).tables()[1].shape[0] == n
    return pat


def test_warp_tier_state_bound(lib, lane):
    from dgraph_b200 import algo

    rng = np.random.default_rng(8)
    for ns in (WARP_STATES - 1, WARP_STATES, WARP_STATES + 1):
        pat = _literal_with_states(ns)
        vals = []
        for k in range(12):
            b = bytearray(rng.choice(np.frombuffer(b"ab\n", np.uint8), LONG + 1 + 997 * k).tobytes())
            if k % 3:
                at = [0, len(b) // 2 - len(pat) // 2, len(b) - len(pat)][k % 3]
                b[at:at + len(pat)] = pat.encode()
            vals.append(bytes(b))
        uids = np.arange(1, len(vals) + 1, dtype=np.uint64)
        col = algo.StrColumn(uids, [[v] for v in vals])
        check_both(lib, lane, col, pat, uids, want=want_by_re(col, pat, uids), what=f"{ns} states")


def test_hub_with_many_list_values(lib, lane):
    from dgraph_b200 import algo

    rng = np.random.default_rng(9)
    hub = [rng.choice(np.frombuffer(b"abcde", np.uint8), 12).tobytes() for _ in range(20_000)]
    hub[17_311] = b"xx" + b"needle" + b"yy"
    col = algo.StrColumn([5, 6, 7], [[b"a"], hub, [b"needle"]])
    check_both(lib, lane, col, "needle", [5, 6, 7], what="hub")
    check_both(lib, lane, col, "e{3}d", [5, 6, 7], what="hub counted")


def dev_leaves_run(lib, lane, raw, prog, after, cap):
    """The lane form's trigram branch over match_cases.Raw's leaves, uploaded as test_gpu_match.Dev uploads them:
    (rc, rc of the sync, out with its guard words, length, launches)."""
    import torch

    from test_gpu_match import Dev

    dev = Dev(lib, lane, raw)
    try:
        dcol = DevCol(raw.col)
        d_out = torch.full((max(cap, 1) + 4,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
        d_len = torch.full((1,), -7, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        l0 = lib.dgx_lane_launches(lane)
        rc = lib.dgx_dev_regex_match(lane, dev.tab, raw.npacks, C.c_void_p(dev.d_mu.data_ptr()),
                                     C.c_void_p(dev.d_mf.data_ptr()), raw.mut_off.ctypes.data,
                                     C.c_void_p(dev.d_lists.data_ptr()), raw.list_off.ctypes.data, raw.nlists, after,
                                     0, None, 0, None, C.byref(dcol.s), prog.handle, C.c_void_p(d_out.data_ptr()), cap,
                                     C.c_void_p(d_len.data_ptr()))
        nl = lib.dgx_lane_launches(lane) - l0
        rs = lib.dgx_lane_sync(lane) if rc == OK else None
        return rc, rs, d_out.cpu().numpy().view(np.uint64), int(d_len.cpu().numpy().view(np.uint64)[0]), nl
    finally:
        dev.free()


def test_trigram_branch_layers_and_after(lib, lane):
    import match_cases as mc

    from dgraph_b200 import algo

    for seed in range(30):
        rng = np.random.default_rng(1_600_000 + seed)
        pat, fold_arg, _, _, _ = gr.random_case(rng)
        uids, vals = gr.column_case(rng, 300)
        uids = np.unique(rng.integers(1, 600, uids.size)).astype(np.uint64)
        vals = vals[:uids.size]
        col = algo.StrColumn(uids, vals)
        after = int(rng.choice([0, 200, 599]))
        leaves = gt.random_leaves(rng, int(rng.integers(1, 7)), 600, "mixed", after=after)
        al = gt.to_algo(leaves)
        cand = algo.UidsForRegex([(gt.QOR, list(range(len(leaves))), [])], al, after).Uids
        prog = algo.RegexProg(pat, fold_arg)
        want = ro.regex_match(col, ro.Prog(pat, fold_arg), cand)
        got = algo.MatchRegex(col, prog, leaves=al, afterUID=after)
        assert np.array_equal(got.Uids, want), (seed, pat)
        raw = mc.Raw(col, "", 0, leaves=leaves)
        rc, rs, out, n, _ = dev_leaves_run(lib, lane, raw, prog, after, raw.bound)
        assert (rc, rs) == (OK, OK), (seed, lib.dgx_last_error())
        assert np.array_equal(out[:n], want) and np.all(out[n:] == np.uint64(SENTINEL)), (seed, pat)


def test_golden(lib, lane):
    # TestFilterRegex6-13's published answers, both forms
    import json
    import os

    from dgraph_b200 import algo

    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "regex_common.json")) as f:
        g = json.load(f)
    col = algo.StrColumn([u for u, _ in g["value"]], [[v] for _, v in g["value"]])
    for c in g["cases"]:
        check_both(lib, lane, col, c["pattern"], col.uid, c["fold"], want=np.array(c["want"], np.uint64),
                   what=c["test"])


def test_device_refusals(lib, lane):
    import torch

    from dgraph_b200 import algo

    prog = algo.RegexProg("a")
    col = algo.StrColumn([3, 5, 9], [[b"a"], [b"ba"], [b"c"]])
    dcol = DevCol(col)
    # unordered candidates
    rc, rs, out, n, _ = dev_run(lib, lane, dcol, prog, [5, 3, 9])
    assert (rc, rs, n) == (OK, ERR_ARG, 0) and np.all(out == np.uint64(SENTINEL))
    from dgraph_b200 import _lib

    with pytest.raises(_lib.DgxError) as e:
        algo.MatchRegex(col, prog, uids=[5, 3, 9])
    assert e.value.code == ERR_ARG
    # column uids not ascending
    bad = algo.StrColumn.from_csr([5, 3, 9], col.val_off, col.byte_off, col.bytes)
    rc, rs, out, n, _ = dev_run(lib, lane, DevCol(bad), prog, [3, 5, 9])
    assert (rc, rs, n) == (OK, ERR_ARG, 0) and np.all(out == np.uint64(SENTINEL))
    # column offsets (checked on the device by the lane form)
    bad = algo.StrColumn.from_csr(col.uid, np.array([0, 2, 1, 3], np.uint64), col.byte_off, col.bytes)
    rc, rs, out, n, _ = dev_run(lib, lane, DevCol(bad), prog, [3, 5, 9])
    assert (rc, rs, n) == (OK, ERR_ARG, 0) and np.all(out == np.uint64(SENTINEL))
    assert b"regexp()" in lib.dgx_last_error()
    # a count word past its room, then within it
    w = torch.tensor([4], dtype=torch.int64, device="cuda")
    rc, rs, out, n, _ = dev_run(lib, lane, dcol, prog, [3, 5, 9], d_nuids=w.data_ptr())
    assert (rc, rs, n) == (OK, ERR_ARG, 0) and np.all(out == np.uint64(SENTINEL))
    w = torch.tensor([2 | (0xABC << 32)], dtype=torch.int64, device="cuda")
    rc, rs, out, n, _ = dev_run(lib, lane, dcol, prog, [3, 5, 9], d_nuids=w.data_ptr())
    assert (rc, rs, n) == (OK, OK, 2) and out[:2].tolist() == [3, 5] and np.all(out[2:] == np.uint64(SENTINEL))
    # out_cap below the room: refused at the call
    rc, rs, out, n, nl = dev_run(lib, lane, dcol, prog, [3, 5, 9], cap=2)
    assert rc == ERR_CAP and nl == 0
    # a DGX_MUT_VALUE layer entry: the host form refuses it at the call, the lane form on the device
    import match_cases as mc

    from dgraph_b200 import _lib

    kw = next(c[1] for c in mc.error_cases() if c[0] == "DGX_MUT_VALUE")
    raw = mc.Raw(**kw)
    with pytest.raises(_lib.DgxError) as e:
        algo.MatchRegex(raw.col, prog, leaves=gt.to_algo(kw["leaves"]))
    assert e.value.code == ERR_ARG
    rc, rs, out, n, _ = dev_leaves_run(lib, lane, raw, prog, 0, 64)
    assert (rc, rs, n) == (OK, ERR_ARG, 0) and np.all(out == np.uint64(SENTINEL))


def test_launches_constant_as_sizes_grow(lib, lane):
    from dgraph_b200 import algo

    counts = set()
    for scale in (1, 30, 1000):
        rng = np.random.default_rng(11)
        n = 100 * scale
        uids = np.arange(1, n + 1, dtype=np.uint64)
        vals = [[b"ab" * int(rng.integers(1, 5 * scale))] for _ in range(n)]
        if scale == 1000:
            vals[7] = [b"x" * 200_000 + b"abc"]
        prog = algo.RegexProg("b.?c")
        l0 = lib.dgx_lane_launches(lane)
        rc, rs, out, k, nl = dev_run(lib, lane, DevCol(algo.StrColumn(uids, vals)), prog, uids)
        assert (rc, rs) == (OK, OK)
        counts.add(nl)
    assert counts == {5}


def test_device_chain_trigram_regex_regex_match(lib, lane):
    # dgx_dev_trigram_query's result and length word feed dgx_dev_regex_match, whose output and length word feed a
    # second dgx_dev_regex_match and then dgx_dev_match, with no host read between them
    import torch

    from dgraph_b200 import algo
    from trigram_cases import Raw as TRaw

    rng = np.random.default_rng(12)
    uids = np.arange(1, 3001, dtype=np.uint64)
    vals = [[rng.choice(np.frombuffer(b"abcdef\n", np.uint8), int(rng.integers(1, 30))).tobytes()] for _ in uids]
    col = algo.StrColumn(uids, vals)
    dcol = DevCol(col)
    leaves = [("list", np.sort(rng.choice(uids, 1500, replace=False)))]
    al = gt.to_algo(leaves)
    tree = [(gt.QOR, [0], [])]
    cand = algo.UidsForRegex(tree, al, 0).Uids
    p1, p2 = algo.RegexProg("a[b-d]"), algo.RegexProg("^[a-c]")
    want1 = ro.regex_match(col, ro.Prog("a[b-d]"), cand)
    want2 = ro.regex_match(col, ro.Prog("^[a-c]"), want1)
    import match_oracle as mo

    want3 = mo.match(col, b"abc", 2, uids=want2)
    tr = TRaw(tree, lists=[al[0]])
    cap = cand.size
    d_lists = _dev(np.asarray(leaves[0][1], np.uint64))
    lo = np.array([0, cap], np.uint64)
    d_c = torch.zeros(cap + 1, dtype=torch.int64, device="cuda")
    d_cl = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.dgx_dev_trigram_query(lane, C.byref(tr.qt), (C.c_void_p * 1)(), 0, None, None,
                                     np.zeros(1, np.uint64).ctypes.data, C.c_void_p(d_lists.data_ptr()), lo.ctypes.data,
                                     1, 0, C.c_void_p(d_c.data_ptr()), cap, C.c_void_p(d_cl.data_ptr())) == OK
    outs = [torch.full((cap + 4,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda") for _ in range(3)]
    lens = [torch.zeros(1, dtype=torch.int64, device="cuda") for _ in range(3)]
    algo.dev_match_regex(lane, dcol.s, p1, outs[0].data_ptr(), cap, lens[0].data_ptr(), d_uids=d_c.data_ptr(),
                         nuids=cap, d_nuids=d_cl.data_ptr())
    algo.dev_match_regex(lane, dcol.s, p2, outs[1].data_ptr(), cap, lens[1].data_ptr(), d_uids=outs[0].data_ptr(),
                         nuids=cap, d_nuids=lens[0].data_ptr())
    algo.dev_match(lane, dcol.s, b"abc", 2, outs[2].data_ptr(), cap, lens[2].data_ptr(), d_uids=outs[1].data_ptr(),
                   nuids=cap, d_nuids=lens[1].data_ptr())
    assert lib.dgx_lane_sync(lane) == OK
    for o, ln, w in zip(outs, lens, (want1, want2, want3)):
        k = int(ln.item())
        a = o.cpu().numpy().view(np.uint64)
        assert np.array_equal(a[:k], w) and np.all(a[k:] == np.uint64(SENTINEL))
    assert want1.size > want2.size > 0


def test_four_threads(lib):
    from dgraph_b200 import algo

    cases = []
    for t in range(4):
        rng = np.random.default_rng(400 + t)
        uids, vals = gr.column_case(rng, 2000)
        col = algo.StrColumn(uids, vals)
        pat = ["a.b", "^k", "(?i)s$", "[^a]{2}"][t]
        cases.append((col, algo.RegexProg(pat), uids, ro.regex_match(col, ro.Prog(pat), uids)))
    errs = []

    def work(t):
        col, prog, cands, want = cases[t]
        try:
            for _ in range(20):
                assert np.array_equal(algo.MatchRegex(col, prog, uids=cands).Uids, want)
        except Exception as e:  # noqa: BLE001
            errs.append((t, e))

    ts = [threading.Thread(target=work, args=(t,)) for t in range(4)]
    for th in ts:
        th.start()
    for th in ts:
        th.join()
    assert not errs, errs


def test_large_call(lib):
    # 3e6 candidates over a 1e7-uid name column; the answer by the formula's rules (valid UTF-8, one line per value)
    import gen_match as gm

    from dgraph_b200 import algo

    rng = np.random.default_rng(22)
    col = gm.name_column(rng, 10_000_000)
    cands = np.sort(rng.choice(col.uid, 3_000_000, replace=False))
    pat = "al[a-z]ce[^x]"
    got = algo.MatchRegex(col, algo.RegexProg(pat), uids=cands)
    idx = np.searchsorted(col.uid, cands)
    rx = re.compile(pat.encode())
    data = col.bytes.tobytes()
    bo = col.byte_off
    keep = [int(cands[k]) for k, i in enumerate(idx) if rx.search(data[int(bo[i]):int(bo[i + 1])])]
    assert np.array_equal(got.Uids, np.array(keep, np.uint64)) and len(keep) > 1000
