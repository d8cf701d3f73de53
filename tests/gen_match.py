"""Seeded cases for match() (tests/test_match_host.py, tests/test_gpu_match.py, tools/bench_ops.py C21) and an
independent formula: Go's UTF-8 decoding written here from its acceptance table, and the textbook full-matrix edit
distance over the runes -- a second opinion on the line-by-line restatement (match_oracle.c).

Python's bytes.decode("utf-8", "replace") is NOT Go's []rune: it replaces a maximal invalid subpart with one U+FFFD,
where Go gives one U+FFFD per byte (e2 82 is one rune to Python and two to Go), so the decoder below is written out.
"""
from __future__ import annotations

import numpy as np

FFFD = 0xFFFD
MAX_I32 = (1 << 31) - 1

# lead byte -> (width, accepted range of the second byte); every other lead byte is (U+FFFD, width 1)
_LEAD = {}
for b in range(0xC2, 0xE0):
    _LEAD[b] = (2, 0x80, 0xBF)
for b in range(0xE0, 0xF0):
    _LEAD[b] = (3, 0xA0 if b == 0xE0 else 0x80, 0x9F if b == 0xED else 0xBF)
for b in range(0xF0, 0xF5):
    _LEAD[b] = (4, 0x90 if b == 0xF0 else 0x80, 0x8F if b == 0xF4 else 0xBF)


def runes(s: bytes) -> list[int]:
    """Go's []rune(s)."""
    out, i = [], 0
    while i < len(s):
        b = s[i]
        if b < 0x80:
            out.append(b)
            i += 1
            continue
        lead = _LEAD.get(b)
        ok = lead is not None and i + lead[0] <= len(s) and lead[1] <= s[i + 1] <= lead[2] and all(
            0x80 <= s[i + k] <= 0xBF for k in range(2, lead[0]))
        if not ok:
            out.append(FFFD)
            i += 1
            continue
        w = lead[0]
        v = b & (0x1F, 0x0F, 0x07)[w - 2]
        for k in range(1, w):
            v = (v << 6) | (s[i + k] & 0x3F)
        out.append(v)
        i += w
    return out


def distance(a: bytes, b: bytes) -> int:
    """The unit-cost edit distance between the rune sequences, full matrix."""
    x, y = runes(a), runes(b)
    D = np.zeros((len(x) + 1, len(y) + 1), np.int64)
    D[:, 0] = np.arange(len(x) + 1)
    D[0, :] = np.arange(len(y) + 1)
    for i in range(1, len(x) + 1):
        for j in range(1, len(y) + 1):
            D[i, j] = min(D[i - 1, j] + 1, D[i, j - 1] + 1, D[i - 1, j - 1] + (x[i - 1] != y[j - 1]))
    return int(D[len(x), len(y)])


def formula(values_of: dict, query: bytes, max: int, cands) -> list[int]:
    """The candidates (ascending) with a non-empty value within max edits of the query; values_of[uid] is the list of
    the uid's values, absent for ErrNoValue."""
    return [int(u) for u in cands if any(v and distance(v, query) <= max for v in values_of.get(int(u), ()))]


# ---- seeded values -----------------------------------------------------------------------------------------------

TRICKY = [b"", b"\xef\xbf\xbd", b"\xe2\x82", b"\xf0\x9f", b"\xf0\x9f\x98", b"\xf0\x9f\x98\x80", b"\xc0\x80", b"\xc1",
          b"\xed\xa0\x80", b"\xf4\x90\x80\x80", b"\xf5", b"\xff", b"\x80", b"\xbf", b"\xe0\x80\x80", b"\xe0\xa0\x80",
          b"\xc3\xa9", b"\xe2\x82\xac", b"\xf4\x8f\xbf\xbf", b"a\xe2\x82b", b"\xe2\x82\xe2\x82\xac"]
ALPHA = [b"a", b"b", b"c", b"e", b"\xc3\xa9", b"\xe2\x82\xac", b"\xf0\x9f\x98\x80", b"\xef\xbf\xbd", b"\xe2", b"\x82",
         b"\xf0\x9f", b"\xff", b"\xed\xa0\x80"]


def rand_bytes(rng, n: int, alpha=ALPHA) -> bytes:
    """n pieces drawn from alpha: ASCII, 2-, 3- and 4-byte runes, U+FFFD, stray, truncated and surrogate bytes."""
    return b"".join(alpha[int(i)] for i in rng.integers(0, len(alpha), n))


def mutate(rng, s: bytes, k: int) -> bytes:
    """s with k random byte-level edits (a piece inserted, a byte deleted or replaced)."""
    b = bytearray(s)
    for _ in range(k):
        op = int(rng.integers(0, 3))
        pos = int(rng.integers(0, len(b) + 1))
        if op == 0 or not b:
            b[pos:pos] = ALPHA[int(rng.integers(0, len(ALPHA)))]
        elif op == 1:
            del b[min(pos, len(b) - 1)]
        else:
            b[min(pos, len(b) - 1)] = int(rng.integers(0, 256))
    return bytes(b)


def random_case(rng, nuids: int = 40, universe: int = 200, qmax: int = 12, vmax: int = 16):
    """(uids, values, query, max, cands): a column over some of 1 .. universe (some uids with a list of values, the
    first one often failing and a later one passing), a query, a max drawn among 0, the length difference, 2^31 - 1
    and small values, and ascending candidates some of which have no value."""
    q = rand_bytes(rng, int(rng.integers(0, qmax + 1)))
    allu = np.sort(rng.choice(np.arange(1, universe + 1), size=min(nuids, universe), replace=False)).astype(np.uint64)
    col_u = allu[rng.random(allu.size) < 0.8]
    values = []
    for _ in range(col_u.size):
        k = int(rng.choice([1, 1, 1, 2, 3]))
        vs = []
        for _ in range(k):
            r = rng.random()
            if r < 0.1:
                vs.append(b"")
            elif r < 0.25:
                vs.append(TRICKY[int(rng.integers(0, len(TRICKY)))])
            elif r < 0.6:
                vs.append(mutate(rng, q, int(rng.integers(0, 4))))
            else:
                vs.append(rand_bytes(rng, int(rng.integers(0, vmax + 1))))
        values.append(vs)
    r = rng.random()
    if r < 0.2:
        mx = 0
    elif r < 0.3:
        mx = MAX_I32
    elif r < 0.5 and values:
        vs = values[int(rng.integers(0, len(values)))]
        mx = abs(len(runes(vs[0])) - len(runes(q)))
    else:
        mx = int(rng.integers(0, 5))
    cands = allu[rng.random(allu.size) < 0.7]
    return col_u, values, q, mx, cands


# ---- benchmark-sized columns (tools/bench_ops.py C21, tests/test_gpu_match.py) -------------------------------------

def name_column(rng, n: int, step: int = 3):
    """A name-like StrColumn: uids step, 2 step, ..., one value of 5-20 bytes each from a small alphabet, about 5 % with
    an "é" and 2 % starting with "alice"."""
    from dgraph_b200 import algo

    alpha = np.frombuffer(b"abcdeilnorst", np.uint8)
    lens = rng.integers(5, 21, n)
    off = np.zeros(n + 1, np.uint64)
    np.cumsum(lens, out=off[1:])
    data = alpha[rng.integers(0, alpha.size, int(off[-1]))]
    pos = off[np.flatnonzero(rng.random(n) < 0.05)].astype(np.int64)
    data[pos], data[pos + 1] = 0xC3, 0xA9
    starts = off[np.flatnonzero(rng.random(n) < 0.02)].astype(np.int64)
    for k, c in enumerate(b"alice"):
        data[starts + k] = c
    return algo.StrColumn.from_csr(np.arange(1, n + 1, dtype=np.uint64) * step, np.arange(n + 1, dtype=np.uint64), off,
                                   data)


def text_column(rng, n: int, lo: int, hi: int, base: bytes = b"", edits: int = 0):
    """A StrColumn of n uids (1 .. n), one value each of lo .. hi bytes: words of a small vocabulary with some
    multi-byte runes, or, when base is given, base with about `edits` random edits."""
    from dgraph_b200 import algo

    words = [b"the", b"graph", b"query", b"node", "caf\u00e9".encode(), b"edge", "\u20ac".encode(), b"index", b"a"]
    vals = []
    for _ in range(n):
        if base:
            vals.append(mutate(rng, base, int(rng.integers(0, edits + 1))))
            continue
        want = int(rng.integers(lo, hi + 1))
        b = b" ".join(words[int(i)] for i in rng.integers(0, len(words), want // 4 + 1))
        vals.append(b[:want])
    return algo.StrColumn(np.arange(1, n + 1, dtype=np.uint64), [[v] for v in vals])
