"""The host model of codec.Encode on the device (tests/encode_geometry.py), on the CPU: the constants and the matched
statements parse, every fixture of tests/test_gpu_encode_edges.py reaches the events it names, the fixtures together
reach every branch the model names, the model's block plan matches the packs, the packs equal the oracle's byte for
byte, and every call sequence succeeds by its second call.  A fixture that drifts off its edge (a constant changed, a
builder edited) fails here, before any GPU run."""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import encode_geometry as eg  # noqa: E402

FIXTURES = {f.name: f for f in eg.all_fixtures()}
PACKED = {f.name: f for f in eg.all_packed_fixtures()}
_RUNS = {}


def run(name):
    if name not in _RUNS:
        _RUNS[name] = eg.simulate(FIXTURES[name]) if name in FIXTURES else eg.simulate_packed(PACKED[name])
    return _RUNS[name]


def test_constants_and_matched_statements():
    assert (eg.K["EN_NT"], eg.EN_VT, eg.EN_TILE, eg.SEGSCAN) == (256, 8, 2048, 1024)
    assert (eg.SEG_SPARE, eg.SPARE, eg.GROUP_MAX, eg.LAUNCHES) == (2, 64, 17, 5)
    assert eg.K["GV"] == (1 << 8, 1 << 16, 1 << 24)


@pytest.mark.parametrize("fn, what, to, err", [
    ("encode_kernel.cuh", "return v < (1u << 8) ? 1u", "return v <= (1u << 8) ? 1u", "gv_len"),
    ("encode_kernel.cuh", "if (e0 > 0 && e0 <= n) { prev_hi", "if (e0 > 0 && e0 < n) { prev_hi", "have_prev"),
    ("encode_kernel.cuh", "dst + carry + inc - bytes", "dst + inc - bytes", "group offset"),
    ("encode_kernel.cuh", "P.counts[1] = nb < n ? nb : n;", "P.counts[1] = nseg;", "overflow report"),
    ("encode_kernel.cuh", "start < nseg; start += 1024)", "start < nseg; start += 512)", "segscan CTA width"),
    ("dgx_api.cu", "std::min<size_t>(n, nblocks_cap) + 2;", "std::min<size_t>(n, nblocks_cap) + 2 + n / 8;", "seg_cap"),
    ("dgx_api.cu", "(n + B - 1) / B + 64 : 0;", "(n + B - 1) / B + kSpare : 0;", "spare blocks"),
    ("dgx_api.cu", "*delta_cap = 17 * (n / 4", "*delta_cap = 18 * (n / 4", "17-byte group bound"),
    ("dgx_api.cu", "l->launches += 5;\n    g_stats.launches += 5;\n    out->base",
     "l->launches += n_launch;\n    g_stats.launches += n_launch;\n    out->base", "launch count"),
])
def test_a_rewritten_statement_fails(monkeypatch, fn, what, to, err):
    """A rewritten threshold, load, offset, report, capacity or launch count is an error, not a silently different
    model."""
    real = eg._src
    assert what in real(fn)
    monkeypatch.setattr(eg, "_src", lambda f: real(f).replace(what, to) if f == fn else real(f))
    with pytest.raises(ValueError, match=re.escape(err)):
        eg.read_constants()


@pytest.mark.parametrize("name", list(FIXTURES) + list(PACKED))
def test_fixture_reaches_its_events(name):
    f = FIXTURES.get(name) or PACKED[name]
    missing = f.events - run(name)[1]
    assert not missing, f"{name}: does not reach {sorted(missing)}"


def test_every_event_is_reached():
    reached = set().union(*(run(n)[1] for n in list(FIXTURES) + list(PACKED)))
    missing = eg.EVENTS - reached
    assert not missing, f"no fixture reaches {sorted(missing)}"


def test_every_event_name_in_the_model_is_registered():
    """Every name the model's source can record is in EVENTS (literal, or an f-string whose every expansion the table
    must list at least once), so a new branch name without a fixture fails test_every_event_is_reached."""
    src = open(eg.__file__).read()
    assert len(re.findall(r"\bev\.add\(", src)) == 1, "events are recorded through _add only"
    literal = re.findall(r"_add\(ev, (f?)\"([^\"]*)\"", src)
    for is_f, text in literal:
        if not is_f:
            assert text in eg.EVENTS, f"{text!r} is recorded but not registered"
            continue
        pat = "".join(".+" if i % 2 else re.escape(part) for i, part in enumerate(re.split(r"[{}]", text)))
        assert any(re.fullmatch(pat, e) for e in eg.EVENTS), f"f-string {text!r} matches no registered event"
    # names picked from a conditional or a table are quoted literals as well
    for text in re.findall(r"\"((?:seg|scan|blk|write|host|calls|caps|packed|bytes scan): [^\"]*)\"", src):
        if "{" not in text:
            assert text in eg.EVENTS, f"{text!r} is named in the model but not registered"


def _oracle_comparable(bsz):
    return bsz <= (1 << 31) - 1      # the oracle takes BlockSize as an int


def check_pack(orc, u, bsz, what):
    """The model's plan against gen.encode_pack_np's arrays, and those against the oracle byte for byte."""
    pk = eg.pack_of(u, bsz)
    if len(u) == 0:
        assert pk is None
        return
    eg.Plan(u, bsz, *eg.bound(len(u), bsz)).check_pack(pk)
    if not _oracle_comparable(bsz):
        return
    want = orc.encode(np.asarray(u, np.uint64), bsz)
    assert np.array_equal(pk[1], want.base), what
    assert np.array_equal(pk[2], want.num_uids), what
    assert np.array_equal(pk[3], want.delta_off), what
    assert np.array_equal(pk[4], want.deltas), what


@pytest.mark.parametrize("name", list(FIXTURES))
def test_model_equals_oracle(orc, name):
    f = FIXTURES[name]
    check_pack(orc, f.uids, f.bsz, name)


def test_packed_fixtures_equal_oracle(orc):
    for name, f in PACKED.items():
        seqs, _ = run(name)
        for op, (res, _) in seqs.items():
            if res.size:
                check_pack(orc, res, f.bsz, f"{name} {op}")


def test_model_random_lists(orc):
    """Seeded random lists: BlockSize 0 to 1000, uids around several upper words, duplicates, and every capacity
    choice; the plan matches the pack, the pack the oracle, and every call sequence ends by its second call."""
    rng = np.random.default_rng(4102)
    for it in range(40):
        n = int(rng.integers(1, 6000))
        u = np.cumsum(rng.integers(0, int(rng.choice([2, 40, 1 << 12, 1 << 30])), n, dtype=np.uint64))
        u += np.uint64(int(rng.integers(0, 1 << 34)))
        for a in rng.choice(np.arange(n), min(n, int(rng.choice([0, 3, 70, 400]))), replace=False):
            u[a:] += np.uint64(1 << 32)
        bsz = int(rng.choice([0, 1, 2, 5, 10, 64, 256, 1000]))
        check_pack(orc, u, bsz, f"random {it}")
        for choice in ("bound", "zero", "nb-1", "db-1", "exact"):
            if choice == "nb-1" and eg.pack_of(u, bsz)[1].size == 0:
                continue
            seq = eg.calls(u, bsz, eg.resolve_caps(u, bsz, choice))
            assert len(seq) <= 2 and seq[-1].rc == eg.OK
            assert seq[-1].nblocks == eg.pack_of(u, bsz)[1].size


def test_call_sequences():
    """The capacities each call gets and what it answers: exact sizes come back whenever the segments fit the arrays,
    sizes that suffice otherwise, and the second call always succeeds."""
    for name, f in FIXTURES.items():
        seqs, _ = run(name)
        pk = eg.pack_of(f.uids, f.bsz)
        nb, db = pk[1].size, pk[4].size
        for choice, seq in seqs.items():
            assert 1 <= len(seq) <= 2 and seq[-1].rc == eg.OK, (name, choice)
            assert all(c.launches == eg.LAUNCHES for c in seq)
            assert (seq[-1].nblocks, seq[-1].delta_bytes) == (nb, db), (name, choice)
            if choice == "exact":
                assert len(seq) == 1
            if choice == "db-1":
                assert seq[0].rc == eg.ERR_CAP and (seq[0].nblocks, seq[0].delta_bytes) == (nb, db)
            if choice == "nb-1":
                assert seq[0].rc == eg.ERR_CAP and seq[0].nblocks == nb
    three = FIXTURES["three calls before the fix"]
    seq = run(three.name)[0]["bound"]
    assert [(c.rc, c.caps[0], c.nblocks) for c in seq] == [(eg.ERR_CAP, 564, 1000), (eg.OK, 1000, 900)]


def test_the_old_overflow_report_needed_a_third_call():
    """The report the segment pass gave before: the segment count.  On the three-call list the second call's segments
    then fit, its exact count (900) exceeds its capacity (801), and it fails again."""
    u = eg.three_call_list()
    first = eg.Plan(u, 2, *eg.bound(u.size, 2))
    assert first.overflow and first.nseg == 801 and first.exact_nblocks == 900
    old = eg.Plan(u, 2, first.nseg, eg.GROUP_MAX * (u.size // 4 + first.nseg + 1))
    assert not old.overflow and old.rc == eg.ERR_CAP and old.nb_out == 900
