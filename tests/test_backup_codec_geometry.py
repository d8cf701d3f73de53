"""The host model of the backup codec on the device (tests/backup_codec_geometry.py), on the CPU: the constants and the
matched statements parse, every fixture of tests/test_gpu_backup_codec_edges.py reaches the events it names, the
fixtures together reach every branch the model names, and on every fixture the model's bytes, packs, images and
verdicts equal the oracle's.  A fixture that drifts off its edge (a constant changed, a builder edited) fails here,
before any GPU run."""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(__file__))
import backup_codec_geometry as bg  # noqa: E402
import backup_codec_oracle as bco  # noqa: E402
import gen_uvarint as guv  # noqa: E402

RESTORE = {f.name: f for f in bg.all_restore_fixtures()}
BACKUP = {f.name: f for f in bg.all_backup_fixtures()}
_RUNS = {}


def run(name):
    if name not in _RUNS:
        if name in RESTORE:
            f = RESTORE[name]
            _RUNS[name] = bg.simulate_restore(f.rows, f.bsz, f.caps)
        else:
            f = BACKUP[name]
            _RUNS[name] = bg.simulate_backup(f.packs, f.caps)
    return _RUNS[name]


def test_constants_and_matched_statements():
    assert (bg.K["EN_NT"], bg.EN_VT, bg.EN_TILE, bg.K["TB_NT"]) == (256, 8, 2048, 256)
    assert (bg.SCAN, bg.K["OVF"]) == (10, (10, 9, 1))
    assert (bg.TB_LAUNCHES, bg.BF_LAUNCHES) == (4, 9)
    assert [bg.meta_bytes(nb) - (20 * nb + 8) for nb in (1, 2, 3, 4)] == [4, 0, 12, 8]


@pytest.mark.parametrize("fn, what, to, err", [
    ("encode_kernel.cuh", "EN_TILE = EN_NT * EN_VT;", "EN_TILE = 4096;", "EN_TILE"),
    ("backup_codec_kernel.cuh", "__launch_bounds__(256) tb_sizes_kernel", "__launch_bounds__(128) tb_sizes_kernel",
     "grid width"),
    ("dgx_api.cu", "tb_blocks_kernel<<<g_blk, 256, 0", "tb_blocks_kernel<<<g_blk, 512, 0", "grid width"),
    ("backup_codec_kernel.cuh", "while (c < 10 && k > c", "while (c < 9 && k > c", "backward scan"),
    ("backup_codec_kernel.cuh", "(c == 9 && P.buf[k] > 1)", "(c == 9 && P.buf[k] > 0)", "overflow rule"),
    ("backup_codec_kernel.cuh", "if (c >= 10 ||", "if (c > 10 ||", "overflow rule"),
    ("backup_codec_kernel.cuh", "if (P.row_off[row] == start[i])", "if (P.row_off[row] == k)", "rowbase"),
    ("backup_codec_kernel.cuh", "if (j == 0 || row != prow || ", "if (j == 0 || ", "segment-start"),
    ("backup_codec_kernel.cuh", "if (e0 > 0 && e0 <= m) { prow", "if (e0 > 0 && e0 < m) { prow", "previous-value"),
    ("backup_codec_kernel.cuh", "+ P.bsz - 1) / P.bsz;", ") / P.bsz;", "ceiling"),
    ("backup_codec_kernel.cuh", "if (o1 > o0 && P.buf[o1 - 1] >= 0x80)", "if (o1 > o0 + 1 && P.buf[o1 - 1] >= 0x80)",
     "truncated-row"),
    ("backup_codec_kernel.cuh", "{ P.bytes[g] = 0; return; }", "return;", "stop skip"),
    ("backup_codec_kernel.cuh", "const u64 prev = b ? P.last[g - 1] : 0;", "const u64 prev = g ? P.last[g - 1] : 0;",
     "b ? P.last[g - 1] : 0"),
    ("backup_codec_kernel.cuh", "atomicMin(P.stop + P.jobs[j].row, b);", "P.stop[P.jobs[j].row] = b;", "atomicMin"),
    ("backup_codec_kernel.cuh", "lane > __ffs(pm) - 1", "lane >= __ffs(pm) - 1", "nearest prefix"),
    ("backup_codec_kernel.cuh", "z < meta; ++z) im[z] = 0;", "z < meta; ++z) {}", "zero fill"),
    ("common.cuh", "nb * 4 + 15) & ~15ull;", "nb * 4 + 7) & ~7ull;", "pack_image_meta_bytes"),
    ("dgx_api.cu", "P.bsz = block_size ? block_size : 1;", "P.bsz = block_size;", "BlockSize"),
    ("dgx_api.cu", "launches = 4;", "launches = kTbLaunches;", "tb_launch's launches"),
    ("dgx_api.cu", "launches = 9;", "launches = kBfLaunches;", "bf_launch's launches"),
    ("dgx_api.cu", "if ((rc = tb_launch(l, R, true))) return rc;", "", "write pass"),
    ("dgx_api.cu", "if (!img || total == 0) return DGX_OK;", "if (!img) return DGX_OK;", "write pass"),
])
def test_a_rewritten_statement_fails(monkeypatch, fn, what, to, err):
    """A rewritten constant, scan, rule, condition, load, check, cut, fill or launch count is an error, not a silently
    different model."""
    real = bg._src
    assert what in real(fn)
    monkeypatch.setattr(bg, "_src", lambda f: real(f).replace(what, to) if f == fn else real(f))
    with pytest.raises(ValueError, match=re.escape(err)):
        bg.read_constants()


@pytest.mark.parametrize("name", list(RESTORE) + list(BACKUP))
def test_fixture_reaches_its_events(name):
    f = RESTORE.get(name) or BACKUP[name]
    missing = f.events - run(name)[0].events
    assert not missing, f"{name}: does not reach {sorted(missing)}"


def test_every_event_is_reached():
    reached = set().union(*(run(n)[0].events for n in list(RESTORE) + list(BACKUP)))
    missing = bg.EVENTS - reached
    assert not missing, f"no fixture reaches {sorted(missing)}"


def test_every_event_name_in_the_model_is_registered():
    """Every name the model's source can record is in EVENTS (literal, or an f-string whose every expansion the table
    must list at least once), so a new branch name without a fixture fails test_every_event_is_reached."""
    src = open(bg.__file__).read()
    assert len(re.findall(r"\bev\.add\(", src)) == 1, "events are recorded through _add only"
    for is_f, text in re.findall(r"_add\(ev, (f?)\"([^\"]*)\"", src):
        if not is_f:
            assert text in bg.EVENTS, f"{text!r} is recorded but not registered"
            continue
        pat = "".join(".+" if i % 2 else re.escape(part) for i, part in enumerate(re.split(r"[{}]", text)))
        assert any(re.fullmatch(pat, e) for e in bg.EVENTS), f"f-string {text!r} matches no registered event"
    for text in re.findall(r"\"((?:val|bad|row|seg|blk|img|restore|bk|backup|cap): [^\"]*)\"", src):
        if "{" not in text:
            assert text in bg.EVENTS, f"{text!r} is named in the model but not registered"


def _oracle_comparable(bsz):
    return bsz <= (1 << 31) - 1      # the oracle takes BlockSize as an int


@pytest.mark.parametrize("name", list(RESTORE))
def test_restore_model_equals_oracle(name):
    """Row by row: the model's verdict is the oracle's OVERFLOW / TRUNCATED; its values are gen_uvarint's reading; its
    packs (gen.encode_pack_np's, checked against the plan's blocks and group bytes) are the oracle's byte for byte;
    its image offsets and sizes are pack_images'."""
    f = RESTORE[name]
    p, calls = run(name)
    want_rc = {None: 0, "overflow": bco.OVERFLOW, "truncated": bco.TRUNCATED}
    for r, row in enumerate(f.rows):
        vals = guv.read_uvarints_np(row)
        assert (vals is None) == (p.verdicts[r] is not None), (name, r)
        if _oracle_comparable(f.bsz):
            rc, _ = bco.encode_from_buffer(row, f.bsz)
            assert rc == want_rc[p.verdicts[r]], (name, r, rc, p.verdicts[r])
        if p.bad or vals is None or not len(row):
            continue
        assert np.array_equal(p.x[p.vrow == r], vals), (name, r)
        assert np.array_equal(p.row_uids(r), np.cumsum(vals, dtype=np.uint64)), (name, r)
    if p.bad:
        assert not p.img_off.any() and not p.nblocks.any() and not p.delta_bytes.any()
        for host, dev in calls.values():
            assert host.rc == bg.ERR_ARG and dev.sync == bg.ERR_ARG and not host.written
        return
    packs = p.packs()
    for r, row in enumerate(f.rows):
        if not _oracle_comparable(f.bsz):
            break
        rc, want = bco.encode_from_buffer(row, f.bsz)
        assert rc == 0
        if want.is_nil:
            assert packs[r] is None, (name, r)
            continue
        for fld in ("base", "num_uids", "delta_off", "deltas"):
            assert np.array_equal(getattr(packs[r], fld), getattr(want, fld)), (name, r, fld)
        back = p.decoded_stream(r)
        assert back == bco.decode_to_buffer(want), (name, r)
        u = p.row_uids(r)
        if u.size < 2 or (u[1:] >= u[:-1]).all():
            assert back == guv.put_uvarints_np(guv.read_uvarints_np(row)).tobytes(), (name, r)
    if p.n:
        p.image()


@pytest.mark.parametrize("name", list(BACKUP))
def test_backup_model_equals_oracle(name):
    """Row by row: the model's bytes are the oracle's DecodeToBuffer of the pack, and its offsets their lengths."""
    f = BACKUP[name]
    p, calls = run(name)
    hands = {}
    for r, pk in enumerate(f.packs):
        if pk is None:
            assert p.streams[r] == b""
            continue
        h = hands.setdefault(id(pk), pk.hand())
        assert p.streams[r] == bco.decode_to_buffer(h), (name, r)
    assert int(p.out_off[-1]) == sum(len(s) for s in p.streams)
    for ch, (host, dev) in calls.items():
        assert host.launches == bg.TB_LAUNCHES + (1 if host.written else 0)
        if ch == "short":
            assert host.rc == bg.ERR_CAP and dev.sync == bg.ERR_CAP


def test_restore_after_backup_in_the_model():
    """Every backup fixture's streams, restored by the model at the packs' BlockSize, give back the packs' uids."""
    for f in BACKUP.values():
        p, _ = run(f.name)
        bs = next((pk.block_size for pk in f.packs if pk is not None), 256)
        rp = bg.RestorePlan(p.streams, bs)
        assert not rp.bad
        for r, pk in enumerate(f.packs):
            if pk is None:
                continue
            stop = p.stop[r] if p.stop[r] is not None else len(pk.blocks)
            want = [u for i in range(stop) for u in pk.block_uids(i)]
            assert rp.row_uids(r).tolist() == want, (f.name, r)


def test_row_verdicts():
    """The oracle's verdict on short rows at every edge of the rule: 10 and 11 bytes, 10th byte 0, 1 and 2, a row that
    ends after 1, 10 and 11 continuation bytes."""
    for row, want in ((b"\x80" * 9 + b"\x01", None), (b"\x80" * 9 + b"\x00", None), (b"\x80" * 9 + b"\x02", "overflow"),
                      (b"\xff" * 10 + b"\x01", "overflow"), (b"\x05\x80", "truncated"), (b"\x80" * 10, "truncated"),
                      (b"\x80" * 11, "overflow"), (b"\x80\x00", None), (b"", None)):
        assert bg.row_verdict(row) == want, row
        rc, _ = bco.encode_from_buffer(row, 256)
        assert rc == {None: 0, "overflow": bco.OVERFLOW, "truncated": bco.TRUNCATED}[want], row
