// Command go_sort_pin prints the permutation Go's sort.Sort gives the fixed tied inputs of
// tests/var_order_oracle.py's pin_inputs(), under the comparator of dgraph's types/sort.go byValue.Less with one value
// per uid.  There is no Go toolchain where the device code is tested, so for tied rows longer than 12 entries the
// device is checked against the C restatement of Go's pdqsort (tests/var_order_oracle.c), not against Go.  Run this
// with a Go toolchain (go run ./tests/go_sort_pin) and compare its lines with
//
//	python -c "import sys; sys.path.insert(0, 'tests'); import var_order_oracle as v; v.print_pins()"
//
// Any difference is a slip in the restatement.  Not run by pytest.
package main

import (
	"fmt"
	"math"
	"sort"
	"strings"
)

const (
	tInt   = 1
	tFloat = 2
	tBool  = 3
	tNil   = 4
)

type val struct {
	tag int
	i   int64
	f   float64
	b   bool
}

// Go's TypeIDs: INT 2, FLOAT 3, BOOL 4
func tid(t int) int { return map[int]int{tInt: 2, tFloat: 3, tBool: 4, tNil: 0}[t] }

func less(a, b val) bool {
	if a.tag != b.tag {
		if (a.tag != tInt && a.tag != tFloat) || (b.tag != tInt && b.tag != tFloat) {
			return tid(a.tag) < tid(b.tag)
		}
		if a.tag == tFloat {
			return a.f < float64(b.i)
		}
		return float64(a.i) < b.f
	}
	switch a.tag {
	case tInt:
		return a.i < b.i
	case tFloat:
		return a.f < b.f
	}
	return false
}

func equal(a, b val) bool {
	if a.tag != b.tag {
		return false
	}
	switch a.tag {
	case tInt:
		return a.i == b.i
	case tFloat:
		return a.f == b.f
	case tBool:
		return a.b == b.b
	}
	return false
}

type byValue struct {
	v    []val
	u    []uint64
	desc bool
}

func (s byValue) Len() int { return len(s.v) }
func (s byValue) Swap(i, j int) {
	s.v[i], s.v[j] = s.v[j], s.v[i]
	s.u[i], s.u[j] = s.u[j], s.u[i]
}
func (s byValue) Less(i, j int) bool {
	a, b := s.v[i], s.v[j]
	if a.tag == tNil && b.tag == tNil {
		return s.desc
	}
	if a.tag == tNil {
		return false
	}
	if b.tag == tNil {
		return true
	}
	if equal(a, b) {
		return false
	}
	l := less(a, b)
	if s.desc {
		return !l
	}
	return l
}

// gen mirrors pin_inputs() in tests/var_order_oracle.py.
func gen(kind string, n int) []val {
	v := make([]val, n)
	for i := 0; i < n; i++ {
		switch kind {
		case "mod13":
			v[i] = val{tag: tInt, i: int64((i * 7919) % 13)}
		case "nil":
			v[i] = val{tag: tNil}
		case "nanmix":
			if i%5 == 0 {
				v[i] = val{tag: tFloat, f: math.NaN()}
			} else {
				v[i] = val{tag: tFloat, f: float64((i * 31) % 17)}
			}
		case "mixed":
			switch i % 3 {
			case 0:
				v[i] = val{tag: tFloat, f: float64(i % 7)}
			case 1:
				v[i] = val{tag: tInt, i: int64(i % 7)}
			default:
				v[i] = val{tag: tNil}
			}
		}
	}
	return v
}

func main() {
	for _, kind := range []string{"mod13", "nil", "nanmix", "mixed"} {
		for _, n := range []int{13, 50, 100, 1000, 5000} {
			for _, desc := range []bool{false, true} {
				s := byValue{gen(kind, n), make([]uint64, n), desc}
				for i := range s.u {
					s.u[i] = uint64(i + 1)
				}
				sort.Sort(s)
				parts := make([]string, n)
				for i, x := range s.u {
					parts[i] = fmt.Sprint(x)
				}
				fmt.Printf("%s %d %v: %s\n", kind, n, desc, strings.Join(parts, " "))
			}
		}
	}
}
