"""regexp()'s value test on the CPU: the restatement (regex_oracle.py) against the independent formula (gen_regex.py),
the library's compiled DFA (walked here on the host) against the restatement, the compiler's refusals and its state
cap.  None of these needs a device."""
import numpy as np
import pytest

import gen_regex as gr
import regex_oracle as ro
from dgraph_b200 import _lib, algo


def dfa_match(tables, value: bytes) -> bool:
    """Walk the library's tables as the kernels do: state 2, stop at an absorbing state, accept by term bit 4."""
    cls, trans, term = tables
    if not value:
        return False
    s = 2
    for b in value:
        s = int(trans[s, cls[b]])
        if term[s] & 2:
            break
    return bool(term[s] & 4)


def test_restatement_equals_formula_random():
    seen = {"answered": 0, "unanswered": 0, "true": 0, "multiline": 0, "empty first": 0, "counted": 0, "anchor": 0,
            "oneline": 0}
    for seed in range(4000):
        rng = np.random.default_rng(1_300_000 + seed)
        pat, fold_arg, fold, tree, value = gr.random_case(rng)
        got = ro.Prog(pat, fold_arg).match(value)
        want = gr.formula(tree, fold, value)
        if want is None:
            seen["unanswered"] += 1
            continue
        assert got == want, (seed, pat, fold, value)
        seen["answered"] += 1
        seen["true"] += want
        seen["multiline"] += b"\n" in value
        seen["empty first"] += value.startswith(b"\n")
        seen["counted"] += "{" in pat
        seen["anchor"] += any(a in pat for a in ("^", "$", "\\A", "\\z"))
        seen["oneline"] += "(?-m:" in pat and b"\n" in value
    assert all(v > 50 for v in seen.values()), seen


def test_library_dfa_equals_restatement_random():
    # every case, invalid UTF-8 and the non-ASCII folds included: the formula has no say here
    n = 0
    for seed in range(3000):
        rng = np.random.default_rng(1_400_000 + seed)
        pat, fold_arg, _, _, value = gr.random_case(rng)
        prog = algo.RegexProg(pat, fold_arg)
        tables = prog.tables()
        want = ro.Prog(pat, fold_arg).match(value)
        assert dfa_match(tables, value) == want, (seed, pat, fold_arg, value)
        n += want
    assert n > 300


# (pattern, fold, value, answer): the corners the restatement pins (see regex_oracle.py for which are not checked
# against codesearch itself)
CORNERS = [
    ("^$", False, b"\nabc", False),         # the first matching line is an empty first line: offset 0
    ("^$", False, b"abc\n", True),          # an empty last line
    ("^$", False, b"abc\n\nx", True),
    ("x*", False, b"\n", False),            # matches the empty first line first
    ("x*", False, b"a\n", True),
    ("b$", False, b"ab\ncd", True),
    ("^c", False, b"ab\ncd", True),
    ("\\Ac", False, b"ab\ncd", False),
    ("b\\z", False, b"ab\ncd", False),
    ("d\\z", False, b"ab\ncd", True),
    ("a.b", False, b"a\nb", False),         # no match crosses a line
    ("a\\nb", False, b"a\nb", False),
    ("a[^x]b", False, b"a\nb", False),
    ("a.b", False, b"a\xffb", False),       # an invalid byte matches nothing, not even '.'
    ("a[^x]b", False, b"a\xffb", False),
    ("a.b", False, "aéb".encode(), True),
    ("a..b", False, b"a\xe2\x82b", False),
    ("a.b", False, b"a\xed\xa0\x80b", False),  # a surrogate's bytes are invalid
    ("k", True, "\u212a".encode(), True),    # K (Kelvin sign) folds to k
    ("(?i)s", False, "\u017f".encode(), True),  # long s folds to s
    ("K", False, "\u212a".encode(), False),
    ("(?i)\\w", False, "\u212a".encode(), True),
    ("(?i)\\W", False, "\u212a".encode(), False),
    ("[^k]", True, "\u212a".encode(), False),
    ("\\x{20AC}", False, "€".encode(), True),
    ("(?-m)^a", False, b"x\na", False),        # (?-m) sets Go's OneLine again: ^ is \A
    ("(?-m)^x", False, b"x\na", True),
    ("(?-m)a$", False, b"a\nb", False),        # and $ is \z
    ("(?-m)b$", False, b"a\nb", True),
    ("(?m-m:^a)", False, b"x\na", False),
    ("(?-m:^a)|^b", False, b"x\nb", True),     # the group ends OneLine
    ("(?-m)(?m)^a", False, b"x\na", True),
    ("", False, b"", False),                 # an empty value never matches
    ("", False, b"x", True),
]


@pytest.mark.parametrize("pat,fold,value,want", CORNERS)
def test_corners(pat, fold, value, want):
    assert ro.Prog(pat, fold).match(value) == want
    assert dfa_match(algo.RegexProg(pat, fold).tables(), value) == want


# outside the subset (the caller keeps its own matcher)
OUTSIDE = ["\\b", "\\B", "\\pL", "\\p{Greek}", "\\PL", "\\Qa\\E", "\\1", "\\0", "(?P<n>a)", "(?<n>a)", "a{", "a{,3}",
           "x{01}", "\\C", "(?i)é", "(?i)[à-ÿ]", "(?i)[^\\W]"]
# rejected by Go's regexp/syntax itself
GO_REJECTS = ["a**", "a*+", "a+?*", "a{2}{3}", "*a", "(*a)", "a|*", "(", ")", "a)", "(a", "[a", "[z-a]", "\\",
              "a{1001}", "a{2,1}", "(a{100}){11}", "((a{10}){10}){11}", "\\q", "\\Z", "[[:foo:]]", "(?z)", "(?-)",
              "(?i-)", "\\x{110000}", "\\x{}", "\\xZ", "(?i"]


@pytest.mark.parametrize("pat", OUTSIDE + GO_REJECTS)
def test_refused(pat):
    with pytest.raises(_lib.DgxError) as e:
        algo.RegexProg(pat)
    assert e.value.code == _lib.DGX_ERR_ARG


def test_invalid_utf8_pattern_refused():
    with pytest.raises(_lib.DgxError) as e:
        algo.RegexProg(b"a\xffb")
    assert e.value.code == _lib.DGX_ERR_ARG


def test_go_limits_accepted():
    for pat in ["a{1000}", "(a{10}){100}", "a{0,1000}", "(?:)", "()", "a|", "^*", "(?)", "\\_", "[]a]", "[^]a]",
                "[a-b-c]", "(?i:k)s", "(?-i)a", "(?im-sU)a", "a*?", "a{2}?", "\\x41\\x{263a}"]:
        algo.RegexProg(pat)


def test_state_cap_at_n_and_n_plus_1():
    # a line-anchored literal of length L gives L + c states (its NFA sets stay small, so the work bound is far off);
    # c from two small literals, then the cap on both sides
    def states(n):
        return algo.RegexProg("^" + "a" * n).tables()[1].shape[0]

    c = states(10) - 10
    assert states(11) - 11 == c
    cap = 4096  # DGX_REGEX_MAX_STATES
    n = cap - c
    assert states(n) == cap
    with pytest.raises(_lib.DgxError) as e:
        states(n + 1)
    assert e.value.code == _lib.DGX_ERR_CAP


def test_unknown_flags_refused():
    import ctypes as C

    h = C.c_void_p()
    assert _lib.load().dgx_regex_compile(b"a", 1, 2, C.byref(h)) == _lib.DGX_ERR_ARG


def test_null_prog_refused():
    col = algo.StrColumn([1], [[b"a"]])
    cs = col.struct()
    import ctypes as C

    u = np.array([1], np.uint64)
    out = np.zeros(1, np.uint64)
    n = C.c_size_t(0)
    rc = _lib.load().dgx_regex_match(None, 0, None, None, None, None, None, 0, 0, u.ctypes.data, 1, C.byref(cs), None,
                                     out.ctypes.data, 1, C.byref(n))
    assert rc == _lib.DGX_ERR_ARG


def golden():
    import json
    import os

    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "regex_common.json")) as f:
        g = json.load(f)
    col = algo.StrColumn([u for u, _ in g["value"]], [[v] for _, v in g["value"]])
    return g, col


def test_golden_restatement_and_library_tables():
    # TestFilterRegex6-13's published answers over the 24 `value` strings
    g, col = golden()
    for c in g["cases"]:
        want = c["want"]
        assert ro.regex_match(col, ro.Prog(c["pattern"], c["fold"]), col.uid).tolist() == want, c["test"]
        tables = algo.RegexProg(c["pattern"], c["fold"]).tables()
        assert [int(u) for u, (_, v) in zip(col.uid, g["value"]) if dfa_match(tables, v.encode())] == want, c["test"]


def test_work_bound_refuses_fast():
    # patterns whose subset construction would visit too many NFA nodes are DGX_ERR_CAP, the caller's fallback, within
    # a bounded host time rather than after building thousands of states
    import time

    for pat in ["(?:" + "|".join("abcdefghijklmnop") + "){1,300}q", ".{200}\\n?x", ".{0,1000}x", "[^a]{1000}",
                "a" * 4000]:
        t = time.perf_counter()
        with pytest.raises(_lib.DgxError) as e:
            algo.RegexProg(pat)
        assert e.value.code == _lib.DGX_ERR_CAP, pat
        assert time.perf_counter() - t < 2.0, pat
