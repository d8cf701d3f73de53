"""The radix sort's edges through @groupby and value variables (fixtures and host model: tests/radix_geometry.py): sorts
of 2048k - 1, 2048k and 2048k + 1 items, last tiles ending mid-warp, mid-round and on a round, trailing empty tiles
and n = 0, hist scans of 8 and 9 tiles, warps of one digit and of 32 digits, a tile of all 256 digits, digits over
three tiles, key widths of 8k with the all-ones key and 8k + 1, groupby P1 = 0-6 and P2 = 1-5, value-variable levels of
1-4 passes, ties of equal-size groups over a tile edge, Go's ranges at every residue of nrows mod 4, float segments of
1-17 items and over tiles, int segments at warp and CTA edges, sparse maps, a three-level path, and la_fold's row
lengths, present masks and NaNs.

Every call runs as the fixture names it: dgx_groupby_uid (members and counts only), dgx_dev_groupby_uid at the
fixture's e_cap, dgx_var_propagate / dgx_dev_var_propagate for each of its int64 and float64 maps (device v_cap as
named), and dgx_var_level_agg / dgx_dev_var_level_agg for every function.  The return codes, the lane's sync code, the
sizes and the launches equal the model's; the outputs equal the oracle's bit for bit (floats as u64 words); nothing is
written past an output, and an over-capacity call writes only the sizes.  Runs on an H100 only (`pytest -m gpu`)."""
import ctypes as C
import functools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import radix_geometry as rg  # noqa: E402

pytestmark = pytest.mark.gpu

SENT = 0xDEADBEEFCAFEF00D
GUARD = 4
FIXTURES = {f.name: f for f in rg.all_fixtures()}
GB = [(n, i) for n, f in FIXTURES.items() if isinstance(f, rg.GbFix) for i in range(len(f.calls))]
VV = [(n, i, x) for n, f in FIXTURES.items() if isinstance(f, rg.VvFix) for i in range(len(f.calls))
      for x in range(len(f.vals))]
LA = [(n, i, x) for n, f in FIXTURES.items() if isinstance(f, rg.LaFix) for i in range(len(f.calls))
      for x in range(len(f.vals))]


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
    return rg.outcomes(FIXTURES[name])[0]


@functools.lru_cache(maxsize=None)
def oracle(name, x=0, fn=None):
    f = FIXTURES[name]
    if isinstance(f, rg.GbFix):
        return rg.gb_oracle(f)
    if isinstance(f, rg.VvFix):
        return rg.vv_oracle(f, f.vals[x])
    return rg.la_oracle(f, f.vals[x], fn)


def _b(x):
    x = np.ascontiguousarray(x, np.uint64)
    return x if x.size else np.zeros(1, np.uint64)


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _up(x):
    import torch

    return torch.from_numpy(_b(x).view(np.int64).copy()).cuda()


def _sent(n):
    import torch

    return torch.full((n,), SENT - (1 << 64), dtype=torch.int64, device="cuda")


def _h(t):
    return t.cpu().numpy().view(np.uint64)


def _launches(lib, lane=None):
    from dgraph_b200 import _lib

    return lib.dgx_lane_launches(lane) if lane else _lib.stats()["kernel_launches"]


def _eq(got, want, n, what):
    assert np.array_equal(got[:n], want), what
    assert np.all(got[n:] == np.uint64(SENT)), f"{what}: written past {n}"


@pytest.mark.parametrize("name, i", GB)
def test_groupby(lib, lane, name, i):
    import torch

    f, c = FIXTURES[name], FIXTURES[name].calls[i]
    o = model(name)[i]
    keys, grp_off, mem_off, mem = oracle(name)
    G, E = keys.size, mem.size
    npar, nrows = f.par_off.size - 1, f.v_off.size - 1
    gcap, mcap = max(G, 1), max(E, 1)
    if c.form == "host":
        out = [np.full(n + GUARD, SENT, np.uint64) for n in (gcap, npar + 1, gcap + 1, mcap)]
        ng, nm = C.c_size_t(7), C.c_size_t(7)
        l0 = _launches(lib)
        rc = lib.dgx_groupby_uid(_p(_b(f.src)), nrows, _p(_b(f.v)), _p(f.v_off), _p(_b(f.dest)), f.dest.size,
                                 _p(_b(f.par)), _p(f.par_off), npar, _p(out[0]), _p(out[1]), _p(out[2]), gcap,
                                 _p(out[3]) if c.members else None, mcap, C.byref(ng), C.byref(nm))
        assert rc == o.rc == rg.OK, lib.dgx_last_error()
        assert _launches(lib) - l0 == o.launches
        assert (ng.value, nm.value) == (o.G, o.E) == (G, E)
        got = out
    else:
        d = [_up(x) for x in (f.src, f.v, f.v_off, f.dest, f.par, f.par_off)]
        out = [_sent(n + GUARD) for n in (gcap, npar + 1, gcap + 1, mcap)]
        sizes = _sent(2 + GUARD)
        e_cap = E if c.e_cap is None else c.e_cap
        torch.cuda.synchronize()
        l0 = _launches(lib, lane)
        rc = lib.dgx_dev_groupby_uid(lane, d[0].data_ptr(), nrows, d[1].data_ptr(), d[2].data_ptr(), int(f.v_off[-1]),
                                     d[3].data_ptr(), f.dest.size, d[4].data_ptr(), d[5].data_ptr(), npar,
                                     int(f.par_off[-1]), e_cap, out[0].data_ptr(), out[1].data_ptr(),
                                     out[2].data_ptr(), gcap, out[3].data_ptr() if c.members else None, mcap,
                                     sizes.data_ptr())
        assert rc == o.rc == rg.OK, lib.dgx_last_error()
        assert lib.dgx_lane_sync(lane) == o.sync, lib.dgx_last_error()
        assert _launches(lib, lane) - l0 == o.launches
        s = _h(sizes)
        assert (int(s[0]), int(s[1])) == (o.G, o.E) and np.all(s[2:] == np.uint64(SENT))
        got = [_h(t) for t in out]
        if o.sync != rg.OK:  # over capacity: the sizes alone
            assert all(np.all(g == np.uint64(SENT)) for g in got), name
            return
    _eq(got[0], keys, G, f"{name}: keys")
    _eq(got[1], grp_off, npar + 1, f"{name}: grp_off")
    _eq(got[2], mem_off, G + 1, f"{name}: mem_off")
    _eq(got[3], mem if c.members else mem[:0], E if c.members else 0, f"{name}: members")


def _levels(f):
    from dgraph_b200 import _lib

    keep = [(_b(L.src), _b(L.v), L.v_off, _b(L.dest)) for L in f.levels]
    lv = (_lib.VarLevel * len(keep))()
    for k, (s, v, o, d) in enumerate(keep):
        lv[k] = _lib.VarLevel(s.ctypes.data, o.ctypes.data, v.ctypes.data, d.ctypes.data, o.size - 1, 0,
                              f.levels[k].dest.size)
    return keep, lv


@pytest.mark.parametrize("name, i, x", VV)
def test_propagate(lib, lane, name, i, x):
    import torch

    from dgraph_b200 import _lib

    f, c = FIXTURES[name], FIXTURES[name].calls[i]
    o = model(name)[i][x]
    vals = f.vals[x]
    typ = 2 if vals.dtype == np.float64 else 1
    wk, wv = oracle(name, x)
    cap = wk.size if c.out_cap is None else c.out_cap
    if c.form == "host":
        keep, lv = _levels(f)
        ok, ov = np.full(cap + GUARD, SENT, np.uint64), np.full(cap + GUARD, SENT, np.uint64)
        n = C.c_size_t(7)
        l0 = _launches(lib)
        rc = lib.dgx_var_propagate(typ, _p(_b(f.keys)), _p(_b(vals.view(np.uint64))), f.keys.size, lv, len(keep),
                                   _p(ok), _p(ov), cap, C.byref(n))
        assert rc == o.rc, lib.dgx_last_error()
        assert _launches(lib) - l0 == o.launches
        assert n.value == o.n == wk.size
    else:
        dl = [(_up(L.src), _up(L.v), _up(L.v_off), _up(L.dest)) for L in f.levels]
        lv = (_lib.VarLevel * len(dl))()
        for k, (s, v, off, d) in enumerate(dl):
            L = f.levels[k]
            vc = int(L.v_off[-1]) if c.v_caps is None else c.v_caps[k]
            lv[k] = _lib.VarLevel(s.data_ptr(), off.data_ptr(), v.data_ptr(), d.data_ptr(), L.v_off.size - 1, vc,
                                  L.dest.size)
        dk, dv = _up(f.keys), _up(vals.view(np.uint64))
        tk, tv, dn = _sent(cap + GUARD), _sent(cap + GUARD), _sent(1 + GUARD)
        torch.cuda.synchronize()
        l0 = _launches(lib, lane)
        rc = lib.dgx_dev_var_propagate(lane, typ, dk.data_ptr(), dv.data_ptr(), f.keys.size, lv, len(dl),
                                       tk.data_ptr(), tv.data_ptr(), cap, dn.data_ptr())
        assert rc == o.rc, lib.dgx_last_error()
        assert lib.dgx_lane_sync(lane) == o.sync, lib.dgx_last_error()
        assert _launches(lib, lane) - l0 == o.launches
        nn = _h(dn)
        assert int(nn[0]) == o.n == wk.size and np.all(nn[1:] == np.uint64(SENT))
        ok, ov = _h(tk), _h(tv)
    if o.sync != rg.OK:
        assert np.all(ok == np.uint64(SENT)) and np.all(ov == np.uint64(SENT)), name
        return
    _eq(ok, wk, wk.size, f"{name}: keys")
    _eq(ov, wv, wk.size, f"{name}: values")


@pytest.mark.parametrize("name, i, x", LA)
def test_level_agg(lib, lane, name, i, x):
    import torch

    f, c = FIXTURES[name], FIXTURES[name].calls[i]
    vals = f.vals[x]
    typ = 2 if vals.dtype == np.float64 else 1
    nrows = f.v_off.size - 1
    for k, fn in enumerate(f.fns):
        o = model(name)[i][x][k]
        wk, wv = oracle(name, x, fn)
        cap = wk.size if c.out_cap is None else c.out_cap
        if c.form == "host":
            ok, ov = np.full(cap + GUARD, SENT, np.uint64), np.full(cap + GUARD, SENT, np.uint64)
            n = C.c_size_t(7)
            l0 = _launches(lib)
            rc = lib.dgx_var_level_agg(typ, rg.FNS[fn], _p(_b(f.keys)), _p(_b(vals.view(np.uint64))), f.keys.size,
                                       _p(_b(f.src)), nrows, _p(f.v_off), _p(_b(f.v)), _p(ok), _p(ov), cap,
                                       C.byref(n))
            assert rc == o.rc, lib.dgx_last_error()
            assert _launches(lib) - l0 == o.launches
            assert n.value == o.n == wk.size
        else:
            t = [_up(a) for a in (f.keys, vals.view(np.uint64), f.src, f.v_off, f.v)]
            tk, tv, dn = _sent(cap + GUARD), _sent(cap + GUARD), _sent(1 + GUARD)
            v_cap = int(f.v_off[-1]) if c.v_cap is None else c.v_cap
            torch.cuda.synchronize()
            l0 = _launches(lib, lane)
            rc = lib.dgx_dev_var_level_agg(lane, typ, rg.FNS[fn], t[0].data_ptr(), t[1].data_ptr(), f.keys.size,
                                           t[2].data_ptr(), nrows, t[3].data_ptr(), t[4].data_ptr(), v_cap,
                                           tk.data_ptr(), tv.data_ptr(), cap, dn.data_ptr())
            assert rc == o.rc, lib.dgx_last_error()
            assert lib.dgx_lane_sync(lane) == o.sync, lib.dgx_last_error()
            assert _launches(lib, lane) - l0 == o.launches
            nn = _h(dn)
            assert int(nn[0]) == o.n == wk.size and np.all(nn[1:] == np.uint64(SENT))
            ok, ov = _h(tk), _h(tv)
        if o.sync != rg.OK:
            assert np.all(ok == np.uint64(SENT)) and np.all(ov == np.uint64(SENT)), (name, fn)
            continue
        _eq(ok, wk, wk.size, f"{name} {fn}: keys")
        _eq(ov, wv, wk.size, f"{name} {fn}: values")
