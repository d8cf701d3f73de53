"""regexp()'s per-value test as an independent formula, and the seeded random cases that hold it against the
restatement (regex_oracle.py) and the library.

The formula: Python's re, line by line, with re.ASCII (so \\d \\w and (?i) are ASCII only) and the matchRegex rules
stated directly -- an empty value fails, some line must hold a match, \\A only on the first line and \\z only on the
last, and an empty first line that matches reports offset 0, so it fails.  It answers only for valid UTF-8 values and
for patterns whose folds stay ASCII; elsewhere (invalid bytes, K / long s under (?i)) only the restatement answers.

A pattern is generated as a small tree and rendered twice: in Go's syntax, and in Python's for a given line position
(\\A and \\z become an impossible match on the lines where they cannot hold).
"""
from __future__ import annotations

import re

import numpy as np

ALPHA = ["a", "b", "c", "k", "s", "K", "x", "é", "€", "😀", " ", "."]
VALUE_PIECES = [b"a", b"b", b"c", b"k", b"s", b"K", b"x", b" ", b".", b"\n", "é".encode(), "€".encode(),
                "😀".encode(), "K".encode(), "ſ".encode(), b"\xff", b"\xe2\x82", b"\xc0\x80", b"\xed\xa0\x80"]
CLASSES = [("[a-c]", "[a-c]"), ("[^a]", "[^a]"), ("[^\\n]", "[^\\n]"), ("\\d", "\\d"), ("\\w", "\\w"),
           ("\\s", "[\\t\\n\\f\\r ]"), ("\\W", "\\W"), ("[[:alpha:]]", "[A-Za-z]"), ("[[:^alpha:]]", "[^A-Za-z]"),
           ("[é-€]", "[é-€]"), (".", "."), ("[kx]", "[kx]"), ("[^ks]", "[^ks]"), ("\\x{20AC}", "\\u20ac")]


def _lit(c: str) -> str:
    return re.escape(c) if c in ".^$|()[]{}*+?\\" else c


def gen_tree(rng, depth=0):
    r = rng.random()
    if depth > 2 or r < 0.35:
        if rng.random() < 0.6:
            return ("lit", ALPHA[rng.integers(len(ALPHA))])
        return ("cls", CLASSES[rng.integers(len(CLASSES))])
    if r < 0.55:
        return ("cat", [gen_tree(rng, depth + 1) for _ in range(int(rng.integers(2, 4)))])
    if r < 0.65:
        return ("alt", [gen_tree(rng, depth + 1) for _ in range(2)])
    if r < 0.8:
        q = ["*", "+", "?", "*?", "+?", "??"][rng.integers(6)]
        return ("rep", q, gen_tree(rng, depth + 1))
    if r < 0.86:
        mn = int(rng.integers(0, 4))
        form = rng.integers(3)
        q = "{%d}" % mn if form == 0 else "{%d,}" % mn if form == 1 else "{%d,%d}" % (mn, mn + int(rng.integers(0, 3)))
        return ("rep", q, gen_tree(rng, depth + 1))
    if r < 0.92:  # (?-m:...): Go's OneLine again inside, so ^ / $ are \\A / \\z there
        return ("oneline", gen_tree(rng, depth + 1))
    return ("anchor", ["^", "$", "\\A", "\\z"][rng.integers(4)])


def render(t, py: bool, first: bool = True, last: bool = True, oneline: bool = False) -> str:
    k = t[0]
    if k == "oneline":
        inner = render(t[1], py, first, last, True)
        return "(?:" + inner + ")" if py else "(?-m:" + inner + ")"
    if k == "lit":
        return _lit(t[1])
    if k == "cls":
        return t[1][1] if py else t[1][0]
    if k == "cat":
        return "".join(render(s, py, first, last, oneline) for s in t[1])
    if k == "alt":
        return "(?:" + "|".join(render(s, py, first, last, oneline) for s in t[1]) + ")"
    if k == "rep":
        return "(?:" + render(t[2], py, first, last, oneline) + ")" + t[1]
    a = t[1]
    if oneline:
        a = {"^": "\\A", "$": "\\z"}.get(a, a)
    if not py:
        return a
    if a == "\\A":
        return "\\A" if first else "(?!)"
    if a == "\\z":
        return "\\Z" if last else "(?!)"
    return a


def formula(tree, fold: bool, value: bytes):
    """matchRegex by Python's re, or None where the formula has no answer."""
    try:
        text = value.decode("utf-8")
    except UnicodeDecodeError:
        return None
    if fold and any(c in text for c in "Kſ"):
        return None
    if "\ud800" <= max(text, default="a") and any("\ud800" <= c <= "\udfff" for c in text):
        return None
    if not text:
        return False
    lines = text.split("\n")
    flags = re.ASCII | re.MULTILINE | (re.IGNORECASE if fold else 0)
    for k, ln in enumerate(lines):
        pat = render(tree, True, k == 0, k == len(lines) - 1)
        if re.search(pat, ln, flags):
            return not (k == 0 and ln == "")
    return False


def _has_nonascii_fold(t) -> bool:
    if t[0] == "lit":
        return ord(t[1]) >= 128 and t[1].isalpha() or t[1] in "é€😀"
    if t[0] == "cls":
        return t[1][0] in ("[é-€]", "\\x{20AC}", "[^a]", "[^\\n]", "\\W", "[[:^alpha:]]", ".", "[^ks]")
    if t[0] in ("cat", "alt"):
        return any(_has_nonascii_fold(s) for s in t[1])
    if t[0] == "rep":
        return _has_nonascii_fold(t[2])
    if t[0] == "oneline":
        return _has_nonascii_fold(t[1])
    return False


def random_value(rng, weight_lines: bool = True) -> bytes:
    n = int(rng.integers(0, 10))
    parts = []
    for _ in range(n):
        if weight_lines and rng.random() < 0.15:
            parts.append(b"\n")
        else:
            parts.append(VALUE_PIECES[rng.integers(len(VALUE_PIECES))])
    return b"".join(parts)


def random_case(rng):
    """(go_pattern, fold, tree, value).  A folded pattern holds only items whose folds stay ASCII-decidable."""
    while True:
        tree = gen_tree(rng)
        fold = bool(rng.random() < 0.25)
        if fold and _has_nonascii_fold(tree):
            continue
        pat = render(tree, False)
        if fold and rng.random() < 0.5:
            pat = "(?i)" + pat
            fold_arg = False
        else:
            fold_arg = fold
        return pat, fold_arg, fold, tree, random_value(rng)


def column_case(rng, n: int):
    """n uids with 0-3 values each, for the library checks."""
    uids = np.unique(rng.integers(1, 10 * n + 10, n).astype(np.uint64))
    vals = [[random_value(rng) for _ in range(int(rng.integers(0, 4)))] for _ in uids]
    return uids, vals
