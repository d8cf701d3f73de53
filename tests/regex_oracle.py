"""regexp()'s per-value test restated: matchRegex (worker/task.go:1809-1811) over codesearch's line-oriented matcher,
with the pattern "(?m)" + pattern parsed as Go's regexp/syntax parses it with Perl flags.  TEST INFRASTRUCTURE ONLY:
the checker of dgx_regex_match / dgx_dev_regex_match, written apart from the library's compiler (regex_compile.hpp).

It shares no construction with the library: the pattern is parsed here into a rune-level program, and each line of the
value is run through a backtracking-free simulation of that program over its runes (a Pike VM: a set of threads per
position), not through a DFA.  The rules it restates:
  - an empty value never matches;
  - the value matches when some line holds a match (lines split at '\\n', which no match crosses); ^ / $ hold at a
    line's ends, \\A only at the value's start, \\z only at its end;
  - codesearch reports a match at the end of its line and matchRegex needs an offset > 0, so when the first line that
    matches is an empty first line the answer is no match;
  - runes decode as Go's utf8.DecodeRune; an invalid byte is a rune no pattern item matches, '.' and negated classes
    included (codesearch compiles rune ranges to UTF-8 byte sequences, so an invalid byte has no path);
  - under (?-m) Go's OneLine is set again, so ^ is \\A and $ is \\z;
  - (?i) folds ASCII letters, with K (U+212A) in k's orbit and long s (U+017F) in s's.
Patterns outside the library's subset raise Unsupported.  Not checked against codesearch itself: no Go toolchain is
available to run tests/go_regex_pin/main.go, so the empty-first-line offset, invalid UTF-8 and the non-ASCII folds
are this restatement's reading of codesearch's design.
"""
from __future__ import annotations


class Unsupported(ValueError):
    pass


MAXR = 0x10FFFF
PERL = {"d": [(48, 57)], "s": [(9, 10), (12, 13), (32, 32)], "w": [(48, 57), (65, 90), (95, 95), (97, 122)]}
POSIX = {"alnum": [(48, 57), (65, 90), (97, 122)], "alpha": [(65, 90), (97, 122)], "ascii": [(0, 127)],
         "blank": [(9, 9), (32, 32)], "cntrl": [(0, 31), (127, 127)], "digit": [(48, 57)], "graph": [(33, 126)],
         "lower": [(97, 122)], "print": [(32, 126)], "punct": [(33, 47), (58, 64), (91, 96), (123, 126)],
         "space": [(9, 13), (32, 32)], "upper": [(65, 90)], "word": [(48, 57), (65, 90), (95, 95), (97, 122)],
         "xdigit": [(48, 57), (65, 70), (97, 102)]}
ESC = {"a": 7, "f": 12, "t": 9, "n": 10, "r": 13, "v": 11}
ORBITS = [(ord("k"), ord("K"), 0x212A), (ord("s"), ord("S"), 0x17F)]


def decode(b: bytes, i: int):
    """utf8.DecodeRune at i: (rune, width), rune -1 for an invalid byte."""
    b0 = b[i]
    if b0 < 0x80:
        return b0, 1
    if b0 < 0xC2 or b0 > 0xF4:
        return -1, 1
    need = 1 if b0 < 0xE0 else 2 if b0 < 0xF0 else 3
    if i + need >= len(b):
        return -1, 1
    lo, hi = {0xE0: (0xA0, 0xBF), 0xED: (0x80, 0x9F), 0xF0: (0x90, 0xBF), 0xF4: (0x80, 0x8F)}.get(b0, (0x80, 0xBF))
    if not lo <= b[i + 1] <= hi or any(not 0x80 <= b[i + k] <= 0xBF for k in range(2, need + 1)):
        return -1, 1
    v = b0 & (0x1F if need == 1 else 0x0F if need == 2 else 0x07)
    for k in range(1, need + 1):
        v = (v << 6) | (b[i + k] & 0x3F)
    return v, need + 1


def runes(b: bytes):
    out, i = [], 0
    while i < len(b):
        r, w = decode(b, i)
        out.append(r)
        i += w
    return out


def _norm(rs):
    rs = sorted(rs)
    out = []
    for lo, hi in rs:
        if out and lo <= out[-1][1] + 1:
            out[-1] = (out[-1][0], max(out[-1][1], hi))
        else:
            out.append((lo, hi))
    return out


def _neg(rs):
    out, nxt = [], 0
    for lo, hi in _norm(rs):
        if lo > nxt:
            out.append((nxt, lo - 1))
        nxt = hi + 1
    if nxt <= MAXR:
        out.append((nxt, MAXR))
    return out


def _fold(rs):
    out = list(rs)
    for lo, hi in rs:
        if hi >= 0x80 and not (lo == hi and lo in (0x212A, 0x17F)):
            raise Unsupported("(?i) over a non-ASCII rune outside k / s's orbits")
        for x in range(lo, min(hi, 127) + 1):
            if chr(x).isalpha() and x < 128:
                out.append((x ^ 0x20, x ^ 0x20))
        for orb in ORBITS:
            if any(lo <= x <= hi for x in orb):
                out += [(x, x) for x in orb]
    return _norm(out)


class _P:
    """Recursive-descent parser to an AST: ('cls', ranges) ('cat', [..]) ('alt', [..]) ('rep', min, max, sub)
    ('empty',) ('bol',) ('eol',) ('bot',) ('eot',)."""

    def __init__(self, pat: str, fold: bool):
        self.s, self.i, self.fold, self.dotnl, self.oneline = pat, 0, fold, False, False

    def peek(self, k=0):
        return self.s[self.i + k] if self.i + k < len(self.s) else None

    def parse(self):
        t = self.alt()
        if self.i != len(self.s):
            raise Unsupported("unmatched )")
        return t

    def alt(self):
        subs = [self.cat()]
        while self.peek() == "|":
            self.i += 1
            subs.append(self.cat())
        return subs[0] if len(subs) == 1 else ("alt", subs)

    def esc_rune(self):
        c = self.peek()
        if c is None:
            raise Unsupported("trailing backslash")
        self.i += 1
        if ord(c) < 128 and not c.isalnum():
            return ord(c)
        if c in ESC:
            return ESC[c]
        if c == "x":
            if self.peek() == "{":
                j = self.s.index("}", self.i)
                v = int(self.s[self.i + 1:j], 16)
                if v > MAXR or j - self.i - 1 > 8 or j == self.i + 1:
                    raise Unsupported("bad \\x{}")
                self.i = j + 1
                return v
            h = self.s[self.i:self.i + 2]
            if len(h) != 2 or any(ch not in "0123456789abcdefABCDEF" for ch in h):
                raise Unsupported("bad \\x")
            self.i += 2
            return int(h, 16)
        raise Unsupported("escape \\" + c)

    def cls(self, rs, neg):
        rs = _norm(rs)
        if self.fold:
            rs = _fold(rs)
        return ("cls", _neg(rs) if neg else rs)

    def bracket(self):
        neg = self.peek() == "^"
        if neg:
            self.i += 1
        rs, first = [], True
        while True:
            c = self.peek()
            if c is None:
                raise Unsupported("missing ]")
            if c == "]" and not first:
                self.i += 1
                break
            first = False
            if self.s.startswith("[:", self.i):
                j = self.s.find(":]", self.i + 2)
                if j < 0:
                    raise Unsupported("[: without :]")
                name = self.s[self.i + 2:j]
                pn = name.startswith("^")
                if name.lstrip("^") not in POSIX:
                    raise Unsupported("unknown class")
                sub = POSIX[name.lstrip("^")]
                rs += _neg(sub) if pn else sub
                self.i = j + 2
                continue
            if c == "\\" and self.peek(1) is not None and self.peek(1) in "dDsSwW":
                k = self.peek(1)
                self.i += 2
                rs += _neg(PERL[k.lower()]) if k.isupper() else PERL[k]
                continue
            lo = self.one()
            hi = lo
            if self.peek() == "-" and self.peek(1) not in (None, "]"):
                self.i += 1
                hi = self.one()
                if hi < lo:
                    raise Unsupported("bad range")
            rs.append((lo, hi))
        return self.cls(rs, neg)

    def one(self):
        c = self.s[self.i]
        self.i += 1
        return self.esc_rune() if c == "\\" else ord(c)

    def counts(self):
        j = self.s.find("}", self.i)
        if j < 0:
            raise Unsupported("literal {")
        body = self.s[self.i + 1:j]
        parts = body.split(",")
        if len(parts) > 2 or not parts[0].isdigit() or (len(parts) == 2 and parts[1] and not parts[1].isdigit()):
            raise Unsupported("literal {")
        if any(len(p) > 1 and p[0] == "0" for p in parts) or any(len(p) > 8 for p in parts):
            raise Unsupported("literal {")
        mn = int(parts[0])
        mx = mn if len(parts) == 1 else (-1 if parts[1] == "" else int(parts[1]))
        if mn > 1000 or mx > 1000 or (mx >= 0 and mn > mx):
            raise Unsupported("bad repeat count")
        self.i = j + 1
        return mn, mx

    def cat(self):
        items, after_flags = [], False
        while self.peek() not in (None, "|", ")"):
            c = self.peek()
            if c in "*+?{":
                if not items or after_flags:
                    raise Unsupported("missing argument to repetition operator")
                if c == "{":
                    mn, mx = self.counts()
                else:
                    self.i += 1
                    mn, mx = (1 if c == "+" else 0), (1 if c == "?" else -1)
                if self.peek() == "?":
                    self.i += 1
                if self.peek() is not None and self.peek() in "*+?{":
                    raise Unsupported("invalid nested repetition operator")
                items[-1] = ("rep", mn, mx, items[-1])
                continue
            after_flags = False
            self.i += 1
            if c == "(":
                saved = (self.fold, self.dotnl, self.oneline)
                if self.peek() == "?":
                    self.i += 1
                    sign, saw, f = 1, False, [self.fold, self.dotnl, self.oneline]
                    while True:
                        k = self.peek()
                        if k is None:
                            raise Unsupported("missing )")
                        self.i += 1
                        if k in "imsU":
                            if k == "i":
                                f[0] = sign > 0
                            if k == "s":
                                f[1] = sign > 0
                            if k == "m":  # the "(?m)" prefix cleared Perl's OneLine; (?-m) sets it again
                                f[2] = sign < 0
                            saw = True
                        elif k == "-":
                            if sign < 0:
                                raise Unsupported("double -")
                            sign, saw = -1, False
                        elif k in ":)":
                            if sign < 0 and not saw:
                                raise Unsupported("missing flag after -")
                            self.fold, self.dotnl, self.oneline = f
                            if k == ")":
                                after_flags = True
                                break
                            items.append(self.alt())
                            self.fold, self.dotnl, self.oneline = saved
                            if self.peek() != ")":
                                raise Unsupported("missing )")
                            self.i += 1
                            break
                        else:
                            raise Unsupported("group syntax")
                    continue
                items.append(self.alt())
                self.fold, self.dotnl, self.oneline = saved
                if self.peek() != ")":
                    raise Unsupported("missing )")
                self.i += 1
            elif c == "[":
                items.append(self.bracket())
            elif c == ".":
                items.append(("cls", [(0, MAXR)] if self.dotnl else [(0, 9), (11, MAXR)]))
            elif c == "^":
                items.append(("bot",) if self.oneline else ("bol",))
            elif c == "$":
                items.append(("eot",) if self.oneline else ("eol",))
            elif c == "\\":
                k = self.peek()
                if k == "A":
                    self.i += 1
                    items.append(("bot",))
                elif k == "z":
                    self.i += 1
                    items.append(("eot",))
                elif k is not None and k in "dDsSwW":
                    self.i += 1
                    items.append(self.cls(PERL[k.lower()], k.isupper()))
                else:
                    r = self.esc_rune()
                    items.append(self.cls([(r, r)], False))
            else:
                items.append(self.cls([(ord(c), ord(c))], False))
        if not items:
            return ("empty",)
        return items[0] if len(items) == 1 else ("cat", items)


def _repeat_ok(t, n):
    if t[0] == "rep":
        m = t[2]
        if m == 0:
            return True
        if m < 0:
            m = t[1]
        if m > n:
            return False
        if m > 0:
            n //= m
        return _repeat_ok(t[3], n)
    if t[0] in ("cat", "alt"):
        return all(_repeat_ok(s, n) for s in t[1])
    return True


def _check_repeats(t):
    if t[0] == "rep":
        if (t[1] >= 2 or t[2] >= 2) and not _repeat_ok(t, 1000):
            raise Unsupported("invalid repeat size")
        _check_repeats(t[3])
    elif t[0] in ("cat", "alt"):
        for s in t[1]:
            _check_repeats(s)


class Prog:
    """A rune-level program: insts[k] = (op, arg, next, next2)."""

    def __init__(self, pattern, fold: bool = False):
        p = pattern.decode("utf-8") if isinstance(pattern, bytes) else pattern  # invalid UTF-8: Go rejects it too
        tree = _P(p, fold).parse()
        _check_repeats(tree)
        self.insts = [("match", None, -1, -1)]
        self.start = self._comp(tree, 0)

    def _add(self, inst):
        self.insts.append(inst)
        return len(self.insts) - 1

    def _comp(self, t, nxt):
        op = t[0]
        if op == "empty":
            return nxt
        if op in ("bol", "eol", "bot", "eot"):
            return self._add(("assert", op, nxt, -1))
        if op == "cls":
            return self._add(("cls", t[1], nxt, -1))
        if op == "cat":
            for s in reversed(t[1]):
                nxt = self._comp(s, nxt)
            return nxt
        if op == "alt":
            e = self._comp(t[1][-1], nxt)
            for s in reversed(t[1][:-1]):
                e = self._add(("split", None, self._comp(s, nxt), e))
            return e
        _, mn, mx, sub = t
        e = nxt
        if mx < 0:
            sp = self._add(("split", None, -1, nxt))
            body = self._comp(sub, sp)
            self.insts[sp] = ("split", None, body, nxt)
            e = sp
        else:
            for _ in range(mx - mn):
                e = self._add(("split", None, self._comp(sub, e), nxt))
        for _ in range(mn):
            e = self._comp(sub, e)
        return e

    def _closure(self, seeds, held):
        seen, stack, out = set(), list(seeds), []
        while stack:
            k = stack.pop()
            if k in seen:
                continue
            seen.add(k)
            op, arg, a, b = self.insts[k]
            if op == "split":
                stack += [b, a]
            elif op == "assert":
                if arg in held:
                    stack.append(a)
            else:
                out.append(k)
        return out

    def line_matches(self, rs, first: bool, last: bool) -> bool:
        """Some position of the line's runes starts a match (Pike VM over the line)."""
        threads = []
        for pos in range(len(rs) + 1):
            held = set()
            if pos == 0:
                held.add("bol")
                if first:
                    held.add("bot")
            if pos == len(rs):
                held.add("eol")
                if last:
                    held.add("eot")
            cur = self._closure(threads + [self.start], held)
            if any(self.insts[k][0] == "match" for k in cur):
                return True
            if pos == len(rs):
                break
            r = rs[pos]
            threads = [self.insts[k][2] for k in cur if self.insts[k][0] == "cls" and r >= 0
                       and any(lo <= r <= hi for lo, hi in self.insts[k][1])]
        return False

    def match(self, value: bytes) -> bool:
        """matchRegex(value): len(value) > 0 and MatchString(value, true, true) > 0."""
        if not value:
            return False
        lines = value.split(b"\n")
        for k, ln in enumerate(lines):
            if self.line_matches(runes(ln), k == 0, k == len(lines) - 1):
                return not (k == 0 and ln == b"")  # a match in an empty first line reports offset 0
        return False


def regex_match(col, prog: Prog, uids):
    """handleRegexFunction's value loop: the candidates in uids (ascending) one of whose values prog matches."""
    import numpy as np

    out = []
    pos = {int(u): i for i, u in enumerate(col.uid)}
    for u in uids:
        i = pos.get(int(u))
        if i is None:
            continue
        for j in range(int(col.val_off[i]), int(col.val_off[i + 1])):
            if prog.match(col.bytes[int(col.byte_off[j]):int(col.byte_off[j + 1])].tobytes()):
                out.append(int(u))
                break
    return np.array(out, np.uint64)
