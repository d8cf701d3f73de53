"""@groupby over a uid predicate on the device (dgx_groupby_uid and dgx_dev_groupby_uid): every result compared in full
with the line-by-line restatement (groupby_oracle.c), guard words past every capacity, launches with the plan model
(groupby_plan.py).  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import os
import sys
import threading

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import gen_groupby as gg  # noqa: E402
import groupby_oracle as gbo  # noqa: E402
import groupby_plan as gp  # noqa: E402

pytestmark = pytest.mark.gpu

OK, ERR_ARG, ERR_CAP = 0, -3, -4
SENT = 0xDEADBEEFCAFEF00D
GUARD = 4
FRIEND_SRC = [1, 23, 31]
FRIEND_ROWS = [[23, 24, 25, 31, 101], [1], [24]]


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


class Args:
    """One call's inputs as flat arrays (each with room for at least one value)."""

    def __init__(self, parents, src, rows, dest, flat=None):
        if flat is not None:
            self.src, self.v, self.v_off, self.par, self.par_off = flat
        else:
            self.src = np.asarray(src, np.uint64)
            self.v, self.v_off = gbo.csr(rows)
            self.par, self.par_off = gbo.csr(parents)
        self.dest = np.asarray(dest, np.uint64)
        self.nrows, self.npar, self.ndest = self.v_off.size - 1, self.par_off.size - 1, self.dest.size
        self.src_b = self.src if self.src.size else np.zeros(1, np.uint64)
        self.dest_b = self.dest if self.dest.size else np.zeros(1, np.uint64)

    def want(self):
        L = gbo.lib()
        lens = np.diff(self.v_off.astype(np.int64))
        cap = 1
        for p in range(self.npar):
            ul = self.par[int(self.par_off[p]):int(self.par_off[p + 1])]
            cap += int(lens[np.isin(self.src[:self.nrows], ul)].sum())
        keys, agg, mem = (np.empty(cap, np.uint64) for _ in range(3))
        grp_off, mem_off = np.empty(self.npar + 1, np.uint64), np.empty(cap + 1, np.uint64)
        n = L.orc_groupby_uid(self.src_b.ctypes.data, self.nrows, self.v.ctypes.data, self.v_off.ctypes.data,
                              self.par.ctypes.data, self.par_off.ctypes.data, self.npar, keys.ctypes.data,
                              agg.ctypes.data, grp_off.ctypes.data, mem_off.ctypes.data, mem.ctypes.data)
        grp_off[self.npar] = n
        assert np.array_equal(np.diff(mem_off[:n + 1]), agg[:n])
        return keys[:n], grp_off, mem_off[:n + 1], mem[:int(mem_off[n])]


def _p(a):
    return C.c_void_p(a.ctypes.data)


def host(lib, a: Args, gcap, mcap, members=True):
    keys = np.full(gcap + GUARD, SENT, np.uint64)
    grp_off = np.full(a.npar + 1 + GUARD, SENT, np.uint64)
    mem_off = np.full(gcap + 1 + GUARD, SENT, np.uint64)
    mem = np.full(mcap + GUARD, SENT, np.uint64)
    ng, nm = C.c_size_t(7), C.c_size_t(7)
    rc = lib.dgx_groupby_uid(_p(a.src_b), a.nrows, _p(a.v), _p(a.v_off), _p(a.dest_b), a.ndest, _p(a.par),
                             _p(a.par_off), a.npar, _p(keys), _p(grp_off), _p(mem_off), gcap,
                             _p(mem) if members else None, mcap, C.byref(ng), C.byref(nm))
    return rc, ng.value, nm.value, keys, grp_off, mem_off, mem


def dev(lib, lane, a: Args, gcap, mcap, members=True, e_cap=None):
    """(rc of the call, rc of the sync, sizes, keys, grp_off, mem_off, members, launches)."""
    import torch

    def up(x):
        return torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).cuda()

    def sent(n):
        return torch.full((n,), SENT - (1 << 64), dtype=torch.int64, device="cuda")

    d_src, d_v, d_v_off, d_dest, d_par, d_par_off = (up(x) for x in (a.src_b, a.v, a.v_off, a.dest_b, a.par, a.par_off))
    d_keys, d_grp, d_moff, d_mem, d_sizes = sent(gcap + GUARD), sent(a.npar + 1 + GUARD), sent(gcap + 1 + GUARD), \
        sent(mcap + GUARD), sent(2)
    want_e = a.want()[2][-1] if e_cap is None else e_cap
    e_cap = int(want_e) if e_cap is None else e_cap
    torch.cuda.synchronize()
    l0 = lib.dgx_lane_launches(lane)
    rc = lib.dgx_dev_groupby_uid(lane, d_src.data_ptr(), a.nrows, d_v.data_ptr(), d_v_off.data_ptr(),
                                 int(a.v_off[-1]), d_dest.data_ptr(), a.ndest, d_par.data_ptr(), d_par_off.data_ptr(),
                                 a.npar, int(a.par_off[-1]), e_cap, d_keys.data_ptr(), d_grp.data_ptr(),
                                 d_moff.data_ptr(), gcap, d_mem.data_ptr() if members else None, mcap,
                                 d_sizes.data_ptr())
    src = lib.dgx_lane_sync(lane)
    h = [t.cpu().numpy().view(np.uint64) for t in (d_sizes, d_keys, d_grp, d_moff, d_mem)]
    return rc, src, h[0], h[1], h[2], h[3], h[4], lib.dgx_lane_launches(lane) - l0


def _check_out(a, keys, grp_off, mem_off, mem, members, gcap, mcap):
    wk, wg, wm, wmem = a.want()
    G, E = wk.size, wmem.size
    assert np.array_equal(keys[:G], wk), "keys"
    assert np.all(keys[gcap:] == SENT), "keys guard"
    assert np.array_equal(grp_off[:a.npar + 1], wg), "grp_off"
    assert np.all(grp_off[a.npar + 1:] == SENT), "grp_off guard"
    assert np.array_equal(mem_off[:G + 1], wm), "mem_off"
    assert np.all(mem_off[gcap + 1:] == SENT), "mem_off guard"
    if members:
        assert np.array_equal(mem[:E], wmem), "members"
    assert np.all(mem[E if members else 0:] == SENT), "members guard"


def run_both(lib, lane, a: Args, members=True, slack=0):
    wk, _, _, wmem = a.want()
    G, E = wk.size, wmem.size
    gcap, mcap = G + slack, E + slack
    rc, ng, nm, keys, grp_off, mem_off, mem = host(lib, a, gcap, mcap, members)
    assert rc == OK, lib.dgx_last_error()
    assert (ng, nm) == (G, E)
    _check_out(a, keys, grp_off, mem_off, mem, members, gcap, mcap)
    rc, src, sizes, keys, grp_off, mem_off, mem, launches = dev(lib, lane, a, gcap, mcap, members)
    assert rc == OK and src == OK, lib.dgx_last_error()
    if a.npar and a.nrows and int(a.v_off[-1]) and int(a.par_off[-1]):
        assert tuple(sizes) == (G, E)
        assert launches == gp.launches(a.nrows, a.ndest, a.npar, int(a.v_off[-1]), int(a.par_off[-1]), E, True)
    _check_out(a, keys, grp_off, mem_off, mem, members, gcap, mcap)


def test_reference_known_answers(lib, lane):
    a = Args([[23, 24, 25, 31, 101], [1], [24]], FRIEND_SRC, FRIEND_ROWS, [1, 23, 24, 25, 31, 101])
    run_both(lib, lane, a)
    keys, grp_off, mem_off, mem = a.want()
    assert keys.tolist() == [1, 24, 23, 24, 25, 31, 101] and grp_off.tolist() == [0, 2, 7, 7]
    v = Args([FRIEND_SRC], FRIEND_SRC, FRIEND_ROWS, [1, 23, 24, 25, 31, 101])
    run_both(lib, lane, v, members=False)
    run_both(lib, lane, v)
    k, _, mo, m = v.want()
    assert k[-1] == 24 and m[mo[-2]:mo[-1]].tolist() == [1, 31]


@pytest.mark.parametrize("kind", ["small", "high", "mixed", "hub"])
def test_random_cases(lib, lane, kind):
    rng = np.random.default_rng(100 + ["small", "high", "mixed", "hub"].index(kind))
    for i in range(40):
        parents, src, rows, dest = gg.case(rng, kind)
        a = Args(parents, src, rows, dest)
        k, g, mo, m = a.want()
        fk, _, fg, fmo, fm = gg.groupby_uid(parents, src, rows)
        assert all(np.array_equal(x, y) for x, y in zip((k, g, mo, m), (fk, fg, fmo, fm)))
        run_both(lib, lane, a, members=i % 3 != 0, slack=i % 2)


def test_hub_in_every_row(lib, lane):
    rng = np.random.default_rng(7)
    nrows = 5000
    src = np.unique(rng.integers(1, 1 << 40, 3 * nrows, dtype=np.uint64))[:nrows]
    dest = np.unique(rng.integers(1, 1 << 40, 3000, dtype=np.uint64))
    hub = dest[1234]
    rows = [np.unique(np.r_[rng.choice(dest, int(rng.integers(0, 8))), hub]).astype(np.uint64) for _ in range(nrows)]
    a = Args([src, src[::3], src[:1]], src, rows, dest)
    run_both(lib, lane, a)
    keys, grp_off, mem_off, mem = a.want()
    assert keys[grp_off[1] - 1] == hub and mem_off[grp_off[1]] - mem_off[grp_off[1] - 1] == nrows


def test_overlapping_and_repeated_parents(lib, lane):
    rng = np.random.default_rng(8)
    parents, src, rows, dest = gg.case(rng, "small", nrows=300, npar=0, nd=80)
    ps = [src[:200], src[100:], src[:200], src, np.r_[src[::2], np.array([99999], np.uint64)]]
    run_both(lib, lane, Args([np.unique(p) for p in ps], src, rows, dest))


def test_empty_inputs(lib, lane):
    run_both(lib, lane, Args([], [1, 2], [[3], [4]], [3, 4]))
    run_both(lib, lane, Args([[1, 2], []], [1, 2], [[], []], []))
    run_both(lib, lane, Args([[], []], [1, 2], [[3], [4]], [3, 4]))
    run_both(lib, lane, Args([[5, 6]], [1, 2], [[3], [4]], [3, 4]))  # parents reach no source: front only
    assert host(lib, Args([[5, 6]], [1, 2], [[3], [4]], [3, 4]), 0, 0)[0] == OK


def test_capacities(lib, lane):
    rng = np.random.default_rng(9)
    parents, src, rows, dest = gg.case(rng, "mixed", nrows=60, npar=4, nd=30)
    a = Args(parents, src, rows, dest)
    wk, _, _, wmem = a.want()
    G, E = wk.size, wmem.size
    assert G > 1 and E > 1
    for gcap, mcap, members in ((0, E, True), (G - 1, E, True), (G, 0, True), (G, E - 1, True), (G - 1, 0, False)):
        rc, ng, nm, keys, grp_off, mem_off, mem = host(lib, a, gcap, mcap, members)
        assert rc == ERR_CAP and (ng, nm) == (G, E)
        assert np.all(keys == SENT) and np.all(grp_off == SENT) and np.all(mem_off == SENT) and np.all(mem == SENT)
        rc, src_rc, sizes, keys, grp_off, mem_off, mem, _ = dev(lib, lane, a, gcap, mcap, members)
        assert rc == OK and src_rc == ERR_CAP and tuple(sizes) == (G, E)
        assert np.all(keys == SENT) and np.all(grp_off == SENT) and np.all(mem_off == SENT) and np.all(mem == SENT)
    # counts only: mem_cap is not read
    rc, ng, nm, *_ = host(lib, a, G, 0, False)
    assert rc == OK and (ng, nm) == (G, E)
    # room for edges in the device form: one short is DGX_ERR_CAP with the edge count, exact runs
    rc, src_rc, sizes, keys, *_ = dev(lib, lane, a, G, E, True, e_cap=E - 1)
    assert rc == OK and src_rc == ERR_CAP and tuple(sizes) == (0, E) and np.all(keys == SENT)
    rc, src_rc, sizes, *_ = dev(lib, lane, a, G, E, True, e_cap=E)
    assert rc == OK and src_rc == OK and tuple(sizes) == (G, E)


def _bad_cases():
    src, rows, dest, par = [1, 2, 3], [[10, 20], [20], [30]], [10, 20, 30], [[1, 2, 3], [2]]
    yield "src not ascending", ([[1, 2, 3]], [2, 1, 3], rows, dest)
    yield "src repeats", ([[1, 2]], [1, 1, 3], rows, dest)
    yield "row not ascending", (par, src, [[20, 10], [20], [30]], dest)
    yield "row repeats", (par, src, [[10, 10], [20], [30]], dest)
    yield "parent row not ascending", ([[1, 2, 3], [3, 2]], src, rows, dest)
    yield "dest not ascending", (par, src, rows, [10, 30, 20])
    yield "value missing from dest", (par, src, rows, [10, 20])
    yield "no dest", (par, src, rows, [])


@pytest.mark.parametrize("name,case", list(_bad_cases()), ids=[n for n, _ in _bad_cases()])
def test_device_detected_errors(lib, lane, name, case):
    a = Args(*case)
    rc, ng, nm, keys, grp_off, mem_off, mem = host(lib, a, 10, 10)
    assert rc == ERR_ARG, name
    assert np.all(keys == SENT) and np.all(grp_off == SENT) and np.all(mem_off == SENT) and np.all(mem == SENT)
    rc, src_rc, sizes, keys, grp_off, mem_off, mem, _ = dev(lib, lane, a, 10, 10, e_cap=10)
    assert rc == OK and src_rc == ERR_ARG and tuple(sizes) == (0, 0), name
    assert np.all(keys == SENT) and np.all(grp_off == SENT) and np.all(mem_off == SENT) and np.all(mem == SENT)


def test_offsets_refused(lib, lane):
    import torch

    a = Args([[1, 2]], [1, 2], [[10], [20]], [10, 20])
    for name, fix in (("v_off decreasing", lambda: a.v_off.__setitem__(1, 3)),
                      ("v_off[0] not 0", lambda: a.v_off.__setitem__(0, 1)),
                      ("par_off decreasing", lambda: a.par_off.__setitem__(0, 3))):
        v_off, par_off = a.v_off.copy(), a.par_off.copy()
        fix()
        rc, *_ , keys, grp_off, mem_off, mem = host(lib, a, 4, 4)
        assert rc == ERR_ARG and np.all(grp_off == SENT), name
        d_v_off = torch.from_numpy(a.v_off.view(np.int64)).cuda()
        d = [torch.from_numpy(x.view(np.int64)).cuda() for x in (a.src_b, a.v, a.dest_b, a.par, a.par_off)]
        outs = [torch.full((8,), -1, dtype=torch.int64, device="cuda") for _ in range(5)]
        rc = lib.dgx_dev_groupby_uid(lane, d[0].data_ptr(), 2, d[1].data_ptr(), d_v_off.data_ptr(), 2, d[2].data_ptr(),
                                     2, d[3].data_ptr(), d[4].data_ptr(), 1, 2, 4, outs[0].data_ptr(),
                                     outs[1].data_ptr(), outs[2].data_ptr(), 4, outs[3].data_ptr(), 4, outs[4].data_ptr())
        assert rc == OK and lib.dgx_lane_sync(lane) == ERR_ARG, name
        assert all(bool((o[:4] == -1).all()) for o in outs[:4]), name
        a.v_off[:], a.par_off[:] = v_off, par_off
    # host-detected: null arrays, 32-bit sizes
    ng, nm = C.c_size_t(), C.c_size_t()
    z = np.zeros(8, np.uint64)
    assert lib.dgx_groupby_uid(_p(a.src), 2, _p(a.v), _p(a.v_off), _p(a.dest), 2, _p(a.par), _p(a.par_off), 1, _p(z),
                               None, _p(z), 4, _p(z), 4, C.byref(ng), C.byref(nm)) == ERR_ARG
    assert lib.dgx_groupby_uid(None, 2, _p(a.v), _p(a.v_off), _p(a.dest), 2, _p(a.par), _p(a.par_off), 1, _p(z),
                               _p(z), _p(z), 4, _p(z), 4, C.byref(ng), C.byref(nm)) == ERR_ARG
    assert lib.dgx_groupby_uid(_p(a.src), 1 << 32, _p(a.v), _p(a.v_off), _p(a.dest), 2, _p(a.par), _p(a.par_off), 1,
                               _p(z), _p(z), _p(z), 4, _p(z), 4, C.byref(ng), C.byref(nm)) == ERR_ARG
    assert lib.dgx_dev_groupby_uid(lane, None, 2, None, None, 2, None, 2, None, None, 1, 2, 1 << 32, None, None, None,
                                   0, None, 0, None) == ERR_ARG
    assert np.all(z == 0)


def test_device_offsets_far_from_zero(lib, lane):
    """d_v_off = {5, 6, 7}: refused on the device with no output written, and no row search below d_v_off."""
    import torch

    d = [torch.from_numpy(np.array(x, np.uint64).view(np.int64)).cuda()
         for x in ([1, 2], [10, 20, 30, 40, 50, 60, 70, 80], [5, 6, 7], [10, 20, 30, 40, 50, 60, 70], [1, 2], [0, 2])]
    outs = [torch.full((8,), -1, dtype=torch.int64, device="cuda") for _ in range(5)]
    rc = lib.dgx_dev_groupby_uid(lane, d[0].data_ptr(), 2, d[1].data_ptr(), d[2].data_ptr(), 8, d[3].data_ptr(), 7,
                                 d[4].data_ptr(), d[5].data_ptr(), 1, 2, 4, outs[0].data_ptr(), outs[1].data_ptr(),
                                 outs[2].data_ptr(), 4, outs[3].data_ptr(), 4, outs[4].data_ptr())
    assert rc == OK and lib.dgx_lane_sync(lane) == ERR_ARG
    assert all(bool((o == -1).all()) for o in outs[:4])
    assert outs[4][:2].tolist() == [0, 0]


def _launch_case(n, seed):
    rng = np.random.default_rng(seed)
    src = np.arange(1, n + 1, dtype=np.uint64) * 3
    dest = np.arange(1, 201, dtype=np.uint64) * 7
    rows = [np.unique(rng.choice(dest, 3)) for _ in range(n)]
    return Args([src[i:i + 2] for i in range(n)], src, rows, dest)


@pytest.mark.parametrize("n", [1, 10, 10000])
def test_launches_match_the_plan(lib, lane, n):
    """1, 10 and 10 000 parents and rows: the device form's count is the plan model's (run_both checks it)."""
    run_both(lib, lane, _launch_case(n, n))


def test_launches_do_not_grow_with_parents_or_rows(lib, lane):
    """129 and 255 parents and rows need the same key widths (8 bits each): the launch count is the same, whatever the
    edge and group counts are."""
    counts = []
    for n in (129, 255):
        a = _launch_case(n, n)
        wk, _, _, wmem = a.want()
        rc, src_rc, sizes, *_, launches = dev(lib, lane, a, wk.size, wmem.size)
        assert rc == OK and src_rc == OK and tuple(sizes) == (wk.size, wmem.size)
        counts.append(launches)
    assert counts[0] == counts[1] == gp.launches(129, 200, 129, 1, 1, 1, True)


@pytest.mark.parametrize("n", [255, 256, 257, 512])
def test_every_edge_its_own_group(lib, lane, n):
    """G == E: every row has one value of its own, so the last member offset mem_off[G] falls on a thread past every
    edge, also when E is a multiple of the CTA size."""
    src = np.arange(1, n + 1, dtype=np.uint64)
    dest = src * 5
    a = Args([src], src, [[int(d)] for d in dest], dest)
    wk, _, wm, _ = a.want()
    assert wk.size == n and int(wm[-1]) == n
    run_both(lib, lane, a)
    run_both(lib, lane, a, members=False)
    run_both(lib, lane, Args([src, src[:1]], src, [[int(d)] for d in dest], dest))


def test_device_form_fed_by_unfiltered_rows(lib, lane):
    """The rows of dgx_dev_list_uids_unfiltered_rows and their dgx_dev_merge_sorted_matrix as dest, with no host
    round trip in between."""
    import torch

    from dgraph_b200 import codec, pb
    from oracle import pyoracle as orc

    rng = np.random.default_rng(11)
    nrows = 50
    src = np.unique(rng.integers(1, 10 ** 6, 200, dtype=np.uint64))[:nrows]
    lists = [np.unique(rng.integers(1, 5000, int(rng.integers(0, 300)), dtype=np.uint64)) for _ in range(nrows)]
    tab = (C.c_void_p * nrows)()
    handles, keep = [], []
    for i, l in enumerate(lists):
        if l.size == 0:
            continue
        op = orc.encode(l, 256)
        pk = pb.UidPack(op.block_size, op.base, op.num_uids, op.delta_off, op.deltas).normalized()
        view = codec.view_of(pk)
        keep.append((pk, view))
        h = C.c_void_p()
        assert lib.dgx_dev_pack_upload(lane, C.byref(view), C.byref(h)) == OK
        handles.append(h)
        tab[i] = h.value
    m = int(sum(l.size for l in lists))
    mut_off = np.zeros(nrows + 1, np.uint64)
    d_rows = torch.zeros(m + 1, dtype=torch.int64, device="cuda")
    d_off = torch.zeros(nrows + 1, dtype=torch.int64, device="cuda")
    d_dest = torch.zeros(m + 1, dtype=torch.int64, device="cuda")
    d_dlen = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.dgx_dev_list_uids_unfiltered_rows(lane, tab, nrows, None, None, _p(mut_off), 0, 0, d_rows.data_ptr(), m,
                                                 d_off.data_ptr()) == OK
    assert lib.dgx_dev_merge_sorted_matrix(lane, d_rows.data_ptr(), d_off.data_ptr(), nrows, m, d_dest.data_ptr(), m,
                                           d_dlen.data_ptr()) == OK
    ndest = int(np.unique(np.concatenate(lists)).size)
    parents = [src[::2], src, src[5:9]]
    par, par_off = gbo.csr(parents)
    d_src, d_par, d_par_off = (torch.from_numpy(x.view(np.int64)).cuda() for x in (src, par, par_off))
    a = Args(parents, src, lists, np.unique(np.concatenate(lists)))
    wk, wg, wm, wmem = a.want()
    G, E = wk.size, wmem.size
    outs = [torch.full((n,), -1, dtype=torch.int64, device="cuda") for n in (G, 4, G + 1, E, 2)]
    rc = lib.dgx_dev_groupby_uid(lane, d_src.data_ptr(), nrows, d_rows.data_ptr(), d_off.data_ptr(), m,
                                 d_dest.data_ptr(), ndest, d_par.data_ptr(), d_par_off.data_ptr(), 3, par.size, E,
                                 outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), G, outs[3].data_ptr(), E,
                                 outs[4].data_ptr())
    assert rc == OK and lib.dgx_lane_sync(lane) == OK, lib.dgx_last_error()
    h = [o.cpu().numpy().view(np.uint64) for o in outs]
    assert np.array_equal(h[0], wk) and np.array_equal(h[1], wg) and np.array_equal(h[2], wm)
    assert np.array_equal(h[3], wmem) and tuple(h[4]) == (G, E)
    for h_ in handles:
        lib.dgx_dev_pack_free(h_)


def test_concurrent_callers(lib):
    rng = np.random.default_rng(12)
    cases = [Args(*gg.case(rng, "mixed", nrows=200, npar=8, nd=60)) for _ in range(8)]
    errors = []

    def worker(k):
        try:
            for a in cases[k::4]:
                wk, _, _, wmem = a.want()
                rc, ng, nm, keys, grp_off, mem_off, mem = host(lib, a, wk.size, wmem.size)
                assert rc == OK
                _check_out(a, keys, grp_off, mem_off, mem, True, wk.size, wmem.size)
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    ts = [threading.Thread(target=worker, args=(k,)) for k in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


def test_c13_sized_call(lib, lane):
    rng = np.random.default_rng(13)
    src, v, v_off, dest = gg.c13_rows(rng)
    par, par_off = src.copy(), np.array([0, src.size], np.uint64)
    a = Args(None, None, None, dest, flat=(src, v, v_off, par, par_off))
    run_both(lib, lane, a, members=True)
