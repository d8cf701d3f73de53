"""The host model of the UidPack readers' block walk (tests/pack_geometry.py), on the CPU: the constants and the
matched statements parse, every fixture of tests/test_gpu_pack_edges.py reaches the events it names, the fixtures
together reach every branch the model names, both range searches agree, and the model's results equal the oracle's.
A fixture that drifts off its edge (a constant changed, a builder edited) fails here, before any GPU run."""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import pack_geometry as pg  # noqa: E402
from list_uids_unfiltered_oracle import list_count, list_uids_unfiltered  # noqa: E402

FIXTURES = {f.name: f for f in pg.all_fixtures()}
_RUNS = {}


def run(name):
    if name not in _RUNS:
        _RUNS[name] = pg.simulate(FIXTURES[name])
    return _RUNS[name]


def test_constants_and_matched_statements():
    assert (pg.D_BPW, pg.D_WB, pg.SLOW_NUM, pg.MX_SERIAL, pg.CP_TILE) == (64, 4096, 256, 8, 2048)
    assert (pg.K["D_WARPS"], pg.K["D_MAXG"], pg.K["D_STAGE"], pg.K["PROBE_RATIO"]) == (4, 64, 260, 4)


@pytest.mark.parametrize("fn, what, to, err", [
    ("decode_kernel.cuh", "(num > 256u && lane < nb)", "(num > 255u && lane < nb)", "slow-path"),
    ("list_uids_unfiltered_kernel.cuh", "(num > 256u && lane < run)", "(num >= 256u && lane < run)", "slow-path"),
    ("compressed_kernel.cuh", "num <= 256u && (dnext", "num < 257u && (dnext", "slow-path"),
    ("compressed_kernel.cuh", "if (hi - lo <= 4u * n) {", "if (hi - lo < 4u * n) {", "probe-direction"),
    ("dgx_api.cu", "if (m < nb) icw_ranges_by_v_kernel", "if (m <= nb) icw_ranges_by_v_kernel", "m < nb"),
    ("dgx_api.cu", "J.by_v = pnb > m;", "J.by_v = pnb >= m;", "pnb > m"),
    ("decode_kernel.cuh", "D_WB = 4096;", "D_WINDOW = 4096;", "D_WB"),
    ("compressed_kernel.cuh", "MX_SERIAL = 8;", "MX_SERIAL = kSerial;", "MX_SERIAL"),
    ("compressed_kernel.cuh", "CP_NT = 256, CP_VT = 8", "CP_NT = 256, CP_VT = 4", "CP_NT"),
])
def test_a_rewritten_statement_fails(monkeypatch, fn, what, to, err):
    """A rewritten slow-path, probe-direction or range-side test, or a renamed constant, is an error, not a silently
    different model."""
    real = pg._src
    assert what in real(fn)
    monkeypatch.setattr(pg, "_src", lambda f: real(f).replace(what, to) if f == fn else real(f))
    if err == "CP_NT":  # a retuned tile moves the model with it
        assert pg.read_constants()["CP_VT"] == 4
        return
    with pytest.raises((KeyError, ValueError), match=re.escape(err)):
        pg.read_constants()


@pytest.mark.parametrize("name", list(FIXTURES))
def test_fixture_reaches_its_events(name):
    f, r = FIXTURES[name], run(name)
    missing = f.events - r.events
    assert not missing, f"{name}: does not reach {sorted(missing)}"


def test_every_event_is_reached():
    reached = set().union(*(run(n).events for n in FIXTURES))
    missing = pg.EVENTS - reached
    assert not missing, f"no fixture reaches {sorted(missing)}"


def test_every_event_name_in_the_model_is_registered():
    """Every name the model's source can record is in EVENTS (literal, or an f-string whose every expansion the table
    must list at least once), so a new branch name without a fixture fails test_every_event_is_reached."""
    src = open(pg.__file__).read()
    assert len(re.findall(r"\b(?:events|ev)\.add\(", src)) == 1, "events are recorded through _add only"
    calls = re.findall(r"_add\(\w+, (f?)\"([^\"]*)\"\)", src)
    assert len(calls) == src.count("_add(") - 1, "an _add call with a computed name"  # minus the definition
    for is_f, text in calls:
        if not is_f:
            assert text in pg.EVENTS, f"{text!r} is recorded but not registered"
            continue
        pat = "".join(".+" if i % 2 else re.escape(part) for i, part in enumerate(re.split(r"[{}]", text)))
        assert any(re.fullmatch(pat, e) for e in pg.EVENTS), f"f-string {text!r} matches no registered event"


def _icw_inputs():
    for f in FIXTURES.values():
        if f.kind == "icw":
            yield f.name, f.args[0], f.args[1], f.args[2]
        elif f.kind == "rows":
            for p in f.args[0]:
                if p is not None and p.nb:
                    yield f.name, p, f.args[1], f.args[2]


def test_range_searches_agree():
    """icw_range_by_v and icw_range_by_block give every block the same v-range on every fixture, whichever side the
    host picks; so does the by-v search with `after` dropped from its predecessor test only where no block holds v
    elements on both sides of after."""
    n = 0
    for name, pk, after, v in _icw_inputs():
        v = [int(x) for x in v]
        assert pg.icw_ranges_by_v(pk, v, after) == pg.icw_ranges_by_block(pk, v, after), name
        n += 1
    assert n > 20


def test_compaction_has_one_writer():
    """Exactly one compact_kernel tile writes out_len, m a multiple of the tile included."""
    for name, f in FIXTURES.items():
        if f.kind == "icw" and len(f.args[2]) and f.args[0].nb:
            assert run(name).writers == 1, name


def icw_oracle(orc, pk, after, v):
    """IntersectCompressedWith on the oracle.  With after past the pack's last uid the Go reference's SeekToBlock
    indexes Blocks[len(Blocks)] and panics (or, on the LinearSeek path, returns nothing); the oracle clamps the index
    and reads the last block.  The answer the readers define there is v ∩ pack[>= after], which is empty."""
    if pk.flat and after > pk.flat[-1]:
        return np.zeros(0, np.uint64)
    return orc.intersect_compressed_with(pg.oracle_pack(pk), after, np.asarray(v, np.uint64))


def oracle_result(orc, f):
    if f.kind == "decode":
        pk, seek, _ = f.args
        return orc.decode(pg.oracle_pack(pk), seek)
    if f.kind == "batch":
        return [orc.decode(pg.oracle_pack(p), 0) if p is not None and p.nb else np.zeros(0, np.uint64)
                for p in f.args[0]]
    if f.kind == "icw":
        pk, after, v = f.args
        return icw_oracle(orc, pk, after, v)
    if f.kind == "rows":
        packs, after, v = f.args
        return [icw_oracle(orc, p, after, v) if p is not None and p.nb else np.zeros(0, np.uint64) for p in packs]
    if f.kind == "mx":
        pk, rows = f.args
        op = pg.oracle_pack(pk)
        return [orc.intersect_compressed_with(op, 0, np.asarray(r, np.uint64)) if len(r) else np.zeros(0, np.uint64)
                for r in rows]
    rows, after, first = f.args
    return [(list_uids_unfiltered(pg.oracle_pack(p) if p is not None and p.nb else None, mu, mf, after, first),
             list_count(pg.oracle_pack(p) if p is not None and p.nb else None, mu, mf, after)) for p, mu, mf in rows]


def check_against_oracle(orc, f, r, what):
    want = oracle_result(orc, f)
    if f.kind in ("decode", "icw"):
        assert np.array_equal(r.result, want), f"{what}: model {r.result.size} values, oracle {want.size}"
    elif f.kind == "luu":
        for i, ((w, c), got) in enumerate(zip(want, r.results)):
            assert np.array_equal(got, w), f"{what}: row {i}: model {got.size} values, oracle {w.size}"
            assert r.counts[i] == c, f"{what}: row {i}: count {r.counts[i]}, oracle {c}"
    else:
        for i, (w, got) in enumerate(zip(want, r.results)):
            assert np.array_equal(got, w), f"{what}: row {i}: model {got.size} values, oracle {w.size}"


@pytest.mark.parametrize("name", list(FIXTURES))
def test_model_equals_oracle(orc, name):
    check_against_oracle(orc, FIXTURES[name], run(name), name)


def _random_pack(rng):
    import gen

    n = int(rng.integers(1, 3000))
    u = gen.zipf_gaps(rng, n, start=int(rng.choice([1, (1 << 32) - 500, 1 << 40])))
    if rng.random() < 0.3:
        u = u * np.uint64(rng.integers(1, 1 << 20))
    bs = int(rng.choice([4, 9, 64, 256, 300]))
    enc = gen.encode_pack_np(np.unique(u), bs)
    return pg.Pack(enc[1], enc[2], enc[3], enc[4], bs)


def test_model_random_packs(orc):
    """The model against the oracle on seeded random packs: BlockSize 4 to 300, uids around 2^32, every reader."""
    rng = np.random.default_rng(23)
    for it in range(25):
        pk = _random_pack(rng)
        flat = np.asarray(pk.flat, np.uint64)
        pool = np.unique(np.concatenate([flat, flat + np.uint64(1), [1, int(flat[-1]) + 2]]))
        v = [int(x) for x in np.sort(rng.choice(pool, int(rng.integers(1, min(pool.size, 400) + 1)), replace=False))]
        after = int(rng.choice([0, int(flat[flat.size // 3]), int(flat[flat.size // 2]) + 1]))
        seek = int(rng.choice([0, int(flat[flat.size // 2]), int(flat[-1]) + 1]))
        rows = [sorted(set(int(x) for x in rng.choice(pool, int(rng.integers(0, 50))))) for _ in range(4)]
        mu = np.unique(rng.choice(pool, 30)).astype(np.uint64)
        mf = rng.integers(0, 2, mu.size).astype(np.uint8)
        first = int(rng.choice([0, 1, 50, 1000]))
        for f in (pg.Fixture("r", "decode", (pk, seek, 0), set()), pg.Fixture("r", "icw", (pk, after, v), set()),
                  pg.Fixture("r", "rows", ([pk, None, pk], after, v), set()), pg.Fixture("r", "mx", (pk, rows), set()),
                  pg.Fixture("r", "luu", ([(pk, mu, mf), (None, mu, mf)], after, first), set())):
            check_against_oracle(orc, f, pg.simulate(f), f"random {it} {f.kind}")
