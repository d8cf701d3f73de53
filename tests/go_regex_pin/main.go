// Command go_regex_pin prints codesearch's answer for the corner cases tests/test_regex_host.py pins to the
// restatement (tests/regex_oracle.py): one line "i matchRegex end" per (pattern, fold, value), where end is
// MatchString's offset and matchRegex is handleRegexFunction's test, len(s) > 0 && end > 0 (worker/task.go:1809-1811).
// The pattern is compiled as handleRegexFunction compiles it: "(?m)" + pattern, "(?i)" in front for the i modifier
// (task.go:2144-2161).  There is no Go toolchain where the library is tested, so these corners -- a match in an empty
// first line, invalid UTF-8 against '.' and negated classes, (?i) over K (U+212A) and long s (U+017F), ^ / $ under
// (?-m), \A / \z on later lines, and \b, which the library refuses -- are checked against the restatement's reading
// of codesearch's design, not against codesearch.  Run this with a Go toolchain and codesearch in the module path
// (go run ./tests/go_regex_pin) and compare its lines with
//
//	python -c "import sys; sys.path.insert(0, 'tests'); import test_regex_host as t, regex_oracle as r; [print(i, int(r.Prog(p, f).match(v))) for i, (p, f, v, _) in enumerate(t.CORNERS)]"
//
// Any difference in the matchRegex column is a slip in the restatement and so in the library.  Not run by pytest.
package main

import (
	"fmt"

	cregexp "github.com/google/codesearch/regexp"
)

type corner struct {
	pat   string
	fold  bool
	value string
}

// the order of tests/test_regex_host.py's CORNERS
var corners = []corner{
	{"^$", false, "\nabc"}, {"^$", false, "abc\n"}, {"^$", false, "abc\n\nx"}, {"x*", false, "\n"}, {"x*", false, "a\n"},
	{"b$", false, "ab\ncd"}, {"^c", false, "ab\ncd"}, {"\\Ac", false, "ab\ncd"}, {"b\\z", false, "ab\ncd"},
	{"d\\z", false, "ab\ncd"}, {"a.b", false, "a\nb"}, {"a\\nb", false, "a\nb"}, {"a[^x]b", false, "a\nb"},
	{"a.b", false, "a\xffb"}, {"a[^x]b", false, "a\xffb"}, {"a.b", false, "a\xc3\xa9b"}, {"a..b", false, "a\xe2\x82b"},
	{"a.b", false, "a\xed\xa0\x80b"}, {"k", true, "\u212a"}, {"(?i)s", false, "\u017f"}, {"K", false, "\u212a"},
	{"(?i)\\w", false, "\u212a"}, {"(?i)\\W", false, "\u212a"}, {"[^k]", true, "\u212a"},
	{"\\x{20AC}", false, "\u20ac"}, {"(?-m)^a", false, "x\na"}, {"(?-m)^x", false, "x\na"},
	{"(?-m)a$", false, "a\nb"}, {"(?-m)b$", false, "a\nb"}, {"(?m-m:^a)", false, "x\na"},
	{"(?-m:^a)|^b", false, "x\nb"}, {"(?-m)(?m)^a", false, "x\na"}, {"", false, ""}, {"", false, "x"},
}

// \b is outside the library's subset; these show what codesearch does with it
var wordBoundary = []corner{{"\\bab", false, "xab"}, {"\\bab", false, "x ab"}, {"ab\\b", false, "ab\u00e9"}}

func run(i int, c corner) {
	mod := "(?m)"
	if c.fold {
		mod = "(?mi)"
	}
	re, err := cregexp.Compile(mod + c.pat)
	if err != nil {
		fmt.Println(i, "error", err)
		return
	}
	end := re.MatchString(c.value, true, true)
	ok := len(c.value) > 0 && end > 0
	v := 0
	if ok {
		v = 1
	}
	fmt.Println(i, v, end)
}

func main() {
	for i, c := range corners {
		run(i, c)
	}
	for i, c := range wordBoundary {
		run(100+i, c)
	}
}
