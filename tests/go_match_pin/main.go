// Command go_match_pin prints the edit distance between Go's []rune conversions of the byte strings of
// tests/gen_match.py's TRICKY list, every pair, one line "i j distance": levenshteinDistance's answer (worker/match.go)
// computed with Go's own decoding.  There is no Go toolchain where
// the device code is tested, so the decoding of invalid UTF-8 is checked against the C restatement
// (tests/match_oracle.c) and Go's published decoding table, not against Go.  Run this with a Go toolchain
// (go run ./tests/go_match_pin) and compare its lines with
//
//	python -c "import sys; sys.path.insert(0, 'tests'); import gen_match as g, match_oracle as m; [print(i, j, m.levenshtein(a, b)) for i, a in enumerate(g.TRICKY) for j, b in enumerate(g.TRICKY)]"
//
// Any difference is a slip in the restatement.  Not run by pytest.
package main

import "fmt"

var tricky = []string{"", "\xef\xbf\xbd", "\xe2\x82", "\xf0\x9f", "\xf0\x9f\x98", "\xf0\x9f\x98\x80", "\xc0\x80", "\xc1",
	"\xed\xa0\x80", "\xf4\x90\x80\x80", "\xf5", "\xff", "\x80", "\xbf", "\xe0\x80\x80", "\xe0\xa0\x80", "\xc3\xa9",
	"\xe2\x82\xac", "\xf4\x8f\xbf\xbf", "a\xe2\x82b", "\xe2\x82\xe2\x82\xac"}

// distance is the textbook full-matrix edit distance over []rune(a) and []rune(b): the conversion is what this pins.
func distance(a, b string) int {
	x, y := []rune(a), []rune(b)
	d := make([][]int, len(x)+1)
	for i := range d {
		d[i] = make([]int, len(y)+1)
		d[i][0] = i
	}
	for j := range d[0] {
		d[0][j] = j
	}
	for i := 1; i <= len(x); i++ {
		for j := 1; j <= len(y); j++ {
			sub := d[i-1][j-1]
			if x[i-1] != y[j-1] {
				sub++
			}
			d[i][j] = min(d[i-1][j]+1, d[i][j-1]+1, sub)
		}
	}
	return d[len(x)][len(y)]
}

func main() {
	for i, a := range tricky {
		for j, b := range tricky {
			fmt.Println(i, j, distance(a, b))
		}
	}
}
