"""@cascade's level kernels and @filter's evaluator at their node, level, CTA and tile edges (fixtures and host model:
tests/cascade_geometry.py): levels of 2 047 to 4 097 value slots with a NEW row cut on both sides of a tile edge,
dest slots across a tile edge in a node that is not its level's first, rows, nodes and empty rows on CTA edges,
zero-slot nodes first, between and last, levels without work and a depth-63 chain, forests of 1 023 to 65 535 nodes,
the prune edges, device value rooms far above the rows, descents across node and row edges and every device-side
refusal on a CTA and a tile edge; |D0| of 255 to 4 097 with slack that holds under the tree, values far below v_cap,
D1 of 0, 2 048 and 2 049 with and without paging, the leaf slot space, counts of 2^32 and more, the walk at its node,
leaf and depth limits and a truth table over small trees.

Every cascade case runs through dgx_cascade and dgx_dev_cascade, every @filter case through dgx_sg_filter and
dgx_dev_sg_filter with and without length words and in counts-only mode, as the fixture names it.  Return codes, the
lane's sync code, sizes and length words equal the model's, and the device form's launches equal the plan models'; the
outputs equal the restatements' (cascade_oracle.c, sg_filter_oracle.c) bit for bit; nothing is written past an output,
and a refused call writes only what include/dgx.h documents.  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import functools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import cascade_geometry as cg  # noqa: E402
import cascade_plan as cp  # noqa: E402
import gen_cascade as gc  # noqa: E402
import sg_filter_plan as sp  # noqa: E402

pytestmark = pytest.mark.gpu

SENT = 0xDEADBEEFCAFEF00D
CSENT = 0xA5A5A5A5
GUARD = 4
FIXTURES = {f.name: f for f in cg.all_fixtures()}
CC = [(n, k) for n, f in FIXTURES.items() if isinstance(f, cg.CcFix) for k in range(len(f.cases))]
SF = [n for n, f in FIXTURES.items() if isinstance(f, cg.SfFix)]


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


@functools.lru_cache(maxsize=None)
def model(name):
    return cg.outcomes(FIXTURES[name])[0]


def _t(a, dtype=np.uint64):
    import torch

    a = np.ascontiguousarray(np.asarray(a, dtype))
    if a.size == 0:
        a = np.zeros(1, dtype)
    view = {np.dtype(np.uint64): np.int64, np.dtype(np.uint32): np.int32}.get(a.dtype, a.dtype)
    return torch.from_numpy(a.view(view)).cuda()


def sent(n, counts=False):
    import torch

    if counts:
        return torch.full((n,), CSENT - (1 << 32), dtype=torch.int32, device="cuda")
    return torch.full((n,), SENT - (1 << 64), dtype=torch.int64, device="cuda")


def u64(t):
    return t.cpu().numpy().view(np.uint64)


# ---- @cascade ---------------------------------------------------------------------------------------------------------

def cc_host(lib, nodes):
    """dgx_cascade with guard words: (rc, (sizes, out, out_off, dest_out, dest_off), guards intact)."""
    from dgraph_b200.algo import cascade_arrays, cascade_tree

    a = cascade_arrays(nodes)
    m, nd, rows, n = int(a["v_off"][-1]), int(a["dest_off"][-1]), int(a["row_off"][-1]), a["nnodes"]
    out, dout = np.full(m + GUARD, SENT, np.uint64), np.full(nd + GUARD, SENT, np.uint64)
    oo, do = np.full(rows + 1 + GUARD, SENT, np.uint64), np.full(n + 1 + GUARD, SENT, np.uint64)
    tree = cascade_tree(a)
    p = lambda x: x.ctypes.data  # noqa: E731
    rc = lib.dgx_cascade(C.byref(tree), p(a["v"]), p(a["v_off"]), p(a["row_off"]), p(a["dest"]), p(a["dest_off"]),
                         p(a["has_val"]), p(a["hv_off"]), p(out), p(oo), m, p(dout), p(do), nd)
    if rc != cg.OK:
        return rc, None, all(np.all(x == SENT) for x in (out, dout, oo, do))
    K, D = int(oo[rows]), int(do[n])
    guards = np.all(out[K:] == SENT) and np.all(dout[D:] == SENT) and np.all(oo[rows + 1:] == SENT) and \
        np.all(do[n + 1:] == SENT)
    return rc, (np.array([K, D], np.int64), out[:K], oo[:rows + 1].astype(np.int64), dout[:D],
                do[:n + 1].astype(np.int64)), guards


def cc_dev(lib, lane, case):
    """dgx_dev_cascade over per-node device arrays as cascade_geometry.cc_inputs gives them: (rc, sync rc, sizes,
    (sizes, out, out_off, dest_out, dest_off) or None, launches, guards intact)."""
    import torch

    from dgraph_b200 import _lib
    from dgraph_b200.algo import cascade_arrays, cascade_tree

    keep, descs = [], []
    for v, off, nrows, cap, dest, hv in cg.cc_inputs(case, "dev"):
        d = [_t(v), _t(off), _t(dest), _t(hv, np.uint8)]
        keep += d
        descs.append(_lib.CascadeNode(d[0].data_ptr(), d[1].data_ptr(), nrows, cap, d[2].data_ptr(), dest.size,
                                      d[3].data_ptr(), hv.size))
    a = cascade_arrays(case.nodes)
    tab = (_lib.CascadeNode * max(len(descs), 1))(*descs)
    out_cap, dest_cap = sum(d.v_cap for d in descs), sum(d.ndest for d in descs)
    rows, n = int(a["row_off"][-1]), len(case.nodes)
    d_out, d_oo, d_dout, d_do, d_sz = (sent(out_cap + GUARD), sent(rows + 1 + GUARD), sent(dest_cap + GUARD),
                                       sent(n + 1 + GUARD), sent(2 + GUARD))
    torch.cuda.synchronize()
    tree = cascade_tree(a)
    l0 = lib.dgx_lane_launches(lane)
    rc = lib.dgx_dev_cascade(lane, C.byref(tree), tab, d_out.data_ptr(), d_oo.data_ptr(), out_cap, d_dout.data_ptr(),
                             d_do.data_ptr(), dest_cap, d_sz.data_ptr())
    src = lib.dgx_lane_sync(lane)
    launches = lib.dgx_lane_launches(lane) - l0
    out, oo, dout, do, sz = (u64(t) for t in (d_out, d_oo, d_dout, d_do, d_sz))
    guards = np.all(out[out_cap:] == SENT) and np.all(oo[rows + 1:] == SENT) and np.all(dout[dest_cap:] == SENT) and \
        np.all(do[n + 1:] == SENT) and np.all(sz[2:] == SENT)
    if rc != cg.OK or src != cg.OK:  # a refused call writes d_sizes = {0, 0} and nothing else
        guards = guards and all(np.all(x == SENT) for x in (out, oo, dout, do))
        return rc, src, sz[:2].astype(np.int64), None, launches, guards
    K, D = int(sz[0]), int(sz[1])
    guards = guards and np.all(out[K:out_cap] == SENT) and np.all(dout[D:dest_cap] == SENT)
    return rc, src, sz[:2].astype(np.int64), (sz[:2].astype(np.int64), out[:K], oo[:rows + 1].astype(np.int64),
                                              dout[:D], do[:n + 1].astype(np.int64)), launches, guards


def _same(got, want):
    return len(got) == len(want) and all(np.array_equal(g, w) for g, w in zip(got, want))


@pytest.mark.parametrize("name, k", CC, ids=[f"{n}-{k}" for n, k in CC])
def test_cascade_edges(lib, lane, name, k):
    case, outs = FIXTURES[name].cases[k], model(name)[k]
    for form, o in zip(case.forms, outs):
        what = (name, k, form)
        want = cg.cc_expected(case, form)
        assert cg.cc_agrees(o, want, form), what
        if form == "host":
            rc, got, guards = cc_host(lib, case.nodes)
            assert rc == o.rc and guards, (what, lib.dgx_last_error())
            if want is not None:
                assert _same(got, want), what
            continue
        rc, src, sizes, got, launches, guards = cc_dev(lib, lane, case)
        assert (rc, src) == (o.rc, o.sync) and guards, (what, lib.dgx_last_error())
        assert np.array_equal(sizes, o.sizes), what
        caps = [s[3] for s in cg.cc_inputs(case, "dev")]
        assert launches == o.launches == cp.launches(gc.levels_with_work(case.nodes, caps)), what
        if want is not None:
            assert _same(got, want), what


# ---- @filter ----------------------------------------------------------------------------------------------------------

def sf_host(lib, case, call):
    """dgx_sg_filter with guard words: (rc, (rows, counts, dest), guards intact)."""
    from dgraph_b200.algo import sg_filter_flat, sg_filter_leaf_arrays, sg_filter_tree

    I = cg.sf_inputs(case, call)
    leaves = [("list", lf["p"]) if lf["kind"] == "list" else (lf["kind"], lf["cmp"], lf["thr"], lf["a"])
              for lf in I["leaves"]]
    d0, v, v_off, nrows = I["d0"], I["v"], I["v_off"], I["nrows"]
    n0, m = d0.size, int(v_off[-1])
    keep, tab = sg_filter_leaf_arrays(leaves, n0)
    f = sg_filter_flat(case.tree)
    dest = np.full(n0 + GUARD, SENT, np.uint64)
    out = np.full(m + GUARD, SENT, np.uint64)
    oo = np.full(nrows + 1 + GUARD, SENT, np.uint64)
    cnt = np.full(nrows + GUARD, CSENT, np.uint32)
    n = C.c_size_t(SENT)
    t = sg_filter_tree(f)
    d0p = d0 if n0 else np.zeros(1, np.uint64)
    vp = v if v.size else np.zeros(1, np.uint64)
    rc = lib.dgx_sg_filter(C.byref(t), tab, len(leaves), d0p.ctypes.data, n0, vp.ctypes.data, v_off.ctypes.data, nrows,
                           case.count, case.offset, dest.ctypes.data, n0, C.byref(n),
                           None if call.counts_only else out.ctypes.data, oo.ctypes.data, m, cnt.ctypes.data)
    del keep
    guards = np.all(dest[n0:] == SENT) and np.all(oo[nrows + 1:] == SENT) and np.all(cnt[nrows:] == CSENT) and \
        (np.all(out == SENT) if call.counts_only else np.all(out[m:] == SENT))
    if rc != cg.OK:
        return rc, None, guards and n.value == SENT and np.all(dest == SENT) and np.all(oo == SENT)
    K = int(oo[nrows])
    guards = guards and np.all(dest[n.value:] == SENT) and (call.counts_only or np.all(out[K:] == SENT))
    rows = [out[int(oo[i]):int(oo[i + 1])].copy() for i in range(nrows)]
    return rc, (rows, cnt[:nrows].copy(), dest[:n.value].copy(), oo[:nrows + 1].astype(np.int64)), guards


def sf_dev(lib, lane, case, call):
    """dgx_dev_sg_filter over the arrays of cascade_geometry.sf_inputs: (rc, sync rc, length word, (rows, counts,
    dest, out_off) or None, launches, guards intact)."""
    import torch

    from dgraph_b200 import _lib
    from dgraph_b200.algo import SGF_CMP, sg_filter_flat, sg_filter_tree

    I = cg.sf_inputs(case, call)
    keep, descs = [], []
    for lf in I["leaves"]:
        if lf["kind"] == "list":
            d = _t(lf["p"])
            dl = _t([lf["word"]]) if lf["word"] is not None else None
            keep += [d, dl]
            descs.append(_lib.SgFilterLeaf(0, 0, 0, d.data_ptr(), lf["room"], dl.data_ptr() if dl is not None else None,
                                           None, None))
        else:
            d = _t(lf["a"], np.uint32 if lf["kind"] == "count" else np.uint64)
            keep.append(d)
            descs.append(_lib.SgFilterLeaf(1, SGF_CMP[lf["cmp"]], lf["thr"], None, 0, None,
                                           d.data_ptr() if lf["kind"] == "count" else None,
                                           d.data_ptr() if lf["kind"] == "len" else None))
    tab = (_lib.SgFilterLeaf * max(len(descs), 1))(*descs)
    d0_cap, v_cap, nrows = I["d0_cap"], I["v_cap"], I["nrows"]
    d_d0, d_v, d_off = _t(I["d0"]), _t(I["v"]), _t(I["v_off"])
    d_len = _t([I["d0_word"]]) if I["d0_word"] is not None else None
    d_dest, d_dl = sent(d0_cap + GUARD), sent(1 + GUARD)
    d_out = None if call.counts_only else sent(v_cap + GUARD)
    d_oo, d_cnt = sent(nrows + 1 + GUARD), sent(nrows + GUARD, counts=True)
    torch.cuda.synchronize()
    f = sg_filter_flat(case.tree)   # the tree's arrays must outlive the call
    t = sg_filter_tree(f)
    l0 = lib.dgx_lane_launches(lane)
    rc = lib.dgx_dev_sg_filter(lane, C.byref(t), tab, len(descs), d_d0.data_ptr(), d0_cap,
                               d_len.data_ptr() if d_len is not None else None, d_v.data_ptr(), d_off.data_ptr(),
                               nrows, v_cap, case.count, case.offset, d_dest.data_ptr(), d0_cap, d_dl.data_ptr(),
                               d_out.data_ptr() if d_out is not None else None, d_oo.data_ptr(), v_cap,
                               d_cnt.data_ptr())
    src = lib.dgx_lane_sync(lane)
    launches = lib.dgx_lane_launches(lane) - l0
    dest, dl, oo = u64(d_dest), u64(d_dl), u64(d_oo)
    out = u64(d_out) if d_out is not None else None
    cnt = d_cnt.cpu().numpy().view(np.uint32)
    guards = np.all(dest[d0_cap:] == SENT) and np.all(dl[1:] == SENT) and np.all(oo[nrows + 1:] == SENT) and \
        np.all(cnt[nrows:] == CSENT) and (out is None or np.all(out[v_cap:] == SENT))
    if rc != cg.OK or src != cg.OK:  # a refused call writes the length word 0 and nothing else
        guards = guards and np.all(dest == SENT) and np.all(oo == SENT) and np.all(cnt == CSENT) and \
            (out is None or np.all(out == SENT))
        return rc, src, int(dl[0]), None, launches, guards
    D, K = int(dl[0]), int(oo[nrows])
    guards = guards and np.all(dest[D:] == SENT) and (out is None or np.all(out[K:] == SENT))
    rows = None if out is None else [out[int(oo[i]):int(oo[i + 1])].copy() for i in range(nrows)]
    return rc, src, D, (rows, cnt[:nrows].copy(), dest[:D].copy(), oo[:nrows + 1].astype(np.int64)), launches, guards


def _sf_same(got, want, counts_only):
    rows, counts, dest, oo = got
    wrows, wcounts, wdest = want
    off = np.zeros(len(wrows) + 1, np.int64)
    np.cumsum([r.size for r in wrows], out=off[1:])
    return (np.array_equal(counts, wcounts) and np.array_equal(dest, wdest) and np.array_equal(oo, off) and
            (counts_only or (len(rows) == len(wrows) and all(np.array_equal(a, b) for a, b in zip(rows, wrows)))))


@pytest.mark.parametrize("name", SF)
def test_sg_filter_edges(lib, lane, name):
    f = FIXTURES[name]
    for k, (case, outs) in enumerate(zip(f.cases, model(name))):
        for call, o in zip(f.calls, outs):
            what = (name, k, call)
            want = cg.sf_expected(case, call)
            assert cg.sf_agrees(o, want, case, call), what
            if call.form == "host":
                rc, got, guards = sf_host(lib, case, call)
                assert rc == o.rc and guards, (what, lib.dgx_last_error())
            else:
                rc, src, dl, got, launches, guards = sf_dev(lib, lane, case, call)
                assert (rc, src, dl) == (o.rc, o.sync, o.dest_len) and guards, (what, lib.dgx_last_error())
                assert launches == o.launches == sp.launches(cg.sf_inputs(case, call)["d0_cap"]), what
            if want is not None:
                assert _sf_same(got, want, call.counts_only), what
