//go:build dgx

// Package algo -- cgo shim that routes dgraph's posting-list set operations to
// libdgx (H100, sm_90a).  Drop this file next to algo/uidlist.go and build alpha
// with `-tags dgx`; uidlist.go's bodies are renamed to *Go (intersectWithGo, ...) by
// the companion patch in INTEGRATION.md and stay as the fallback.
//
// NOT COMPILED IN THIS REPOSITORY: the build image has no Go toolchain.  The C side
// of every call below is exercised by tests/ through the same C ABI (ctypes and the
// C++ mirror include/dgx_algo.hpp), with the same borrowing rules.
package algo

/*
#cgo CFLAGS: -I${SRCDIR}/../include
#cgo LDFLAGS: -ldgx
#include <stdint.h>
#include <stdlib.h>
#include "dgx.h"
*/
import "C"

import (
	"runtime"
	"sort"
	"unsafe"

	"github.com/dgraph-io/dgraph/v25/protos/pb"
)

// Below this many input UIDs a PCIe round trip costs more than the Go loop.
const dgxMinUids = 1 << 16

func u64ptr(s []uint64) *C.uint64_t {
	if len(s) == 0 {
		return nil
	}
	return (*C.uint64_t)(unsafe.Pointer(&s[0]))
}

// IntersectWith keeps algo/uidlist.go:142's signature and aliasing rules:
// o may be u; v is never written; o.Uids reuses its capacity like dst := o.Uids[:0].
func IntersectWith(u, v, o *pb.List) {
	n, m := len(u.Uids), len(v.Uids)
	if n+m < dgxMinUids {
		intersectWithGo(u, v, o)
		return
	}
	capN := n
	if m < n {
		capN = m
	}
	dst := o.Uids
	if cap(dst) < capN {
		dst = make([]uint64, capN) // make([]uint64, 0, n) in the reference
	}
	dst = dst[:capN]
	var outLen C.size_t
	rc := C.dgx_intersect2(u64ptr(u.Uids), C.size_t(n), u64ptr(v.Uids), C.size_t(m),
		u64ptr(dst), C.size_t(capN), &outLen)
	runtime.KeepAlive(u)
	runtime.KeepAlive(v)
	if rc != C.DGX_OK {
		intersectWithGo(u, v, o) // the reference cannot fail: stay total
		return
	}
	o.Uids = dst[:int(outLen)]
}

func totalUids(lists []*pb.List) int {
	t := 0
	for _, l := range lists {
		if l != nil {
			t += len(l.Uids)
		}
	}
	return t
}

// pinLists builds the C pointer/length tables for a []*pb.List.  cgo forbids passing
// Go memory that itself holds Go pointers, so the table lives in C memory and the
// list backing arrays are pinned for the duration of the call (Go >= 1.21).
func pinLists(lists []*pb.List) (ptrs **C.uint64_t, lens *C.size_t, total, minLen int, pin *runtime.Pinner, free func()) {
	k := len(lists)
	p := (*[1 << 28]*C.uint64_t)(C.malloc(C.size_t(k) * C.size_t(unsafe.Sizeof(uintptr(0)))))
	l := (*[1 << 28]C.size_t)(C.malloc(C.size_t(k) * C.size_t(unsafe.Sizeof(C.size_t(0)))))
	pin = &runtime.Pinner{}
	minLen = int(^uint(0) >> 1)
	for i, li := range lists {
		var s []uint64
		if li != nil {
			s = li.Uids
		}
		if len(s) > 0 {
			pin.Pin(&s[0])
		}
		p[i] = u64ptr(s)
		l[i] = C.size_t(len(s))
		total += len(s)
		if len(s) < minLen {
			minLen = len(s)
		}
	}
	return (**C.uint64_t)(unsafe.Pointer(p)), (*C.size_t)(unsafe.Pointer(l)), total, minLen, pin,
		func() { pin.Unpin(); C.free(unsafe.Pointer(p)); C.free(unsafe.Pointer(l)) }
}

// IntersectSorted: algo/uidlist.go:297.  No lists -> &pb.List{} (nil Uids).
func IntersectSorted(lists []*pb.List) *pb.List {
	if len(lists) == 0 {
		return &pb.List{}
	}
	if totalUids(lists) < dgxMinUids { // decided before anything is pinned or malloc'ed
		return intersectSortedGo(lists)
	}
	ptrs, lens, _, minLen, _, free := pinLists(lists)
	defer free()
	out := make([]uint64, minLen)
	var outLen C.size_t
	if rc := C.dgx_intersect_sorted(ptrs, lens, C.size_t(len(lists)), u64ptr(out), C.size_t(minLen), &outLen); rc != C.DGX_OK {
		return intersectSortedGo(lists)
	}
	return &pb.List{Uids: out[:int(outLen)]}
}

// MergeSorted: algo/uidlist.go:448.
func MergeSorted(lists []*pb.List) *pb.List {
	if totalUids(lists) < dgxMinUids {
		return mergeSortedGo(lists)
	}
	ptrs, lens, total, _, _, free := pinLists(lists)
	defer free()
	out := make([]uint64, total)
	var outLen C.size_t
	if rc := C.dgx_merge_sorted(ptrs, lens, C.size_t(len(lists)), u64ptr(out), C.size_t(total), &outLen); rc != C.DGX_OK {
		return mergeSortedGo(lists)
	}
	return &pb.List{Uids: out[:int(outLen)]}
}

// dgxMinMergeMatrix: below this many uids MergeSortedMatrix stays on the Go path.  Set from the C8 record
// (profiles/h100_c8_merge_matrix.json, H100 80GB HBM3, 700 W): the host form took 1.1-1.4 ms for the C8a matrix
// (6.49e5 uids in 10 000 rows) and the reference's 10-thread MergeSorted spent 78 ns per uid on it, so about 16 000
// uids cost the Go merge what one library call costs.
const dgxMinMergeMatrix = 1 << 14

// MergeSortedMatrix is algo.MergeSorted(matrix) in ONE library call for the rows of a uid matrix:
// sg.DestUIDs = algo.MergeSorted(result.UidMatrix) (query/query.go:2290, 2505; query/recurse.go:134;
// worker/task.go:1629, 1706; worker/match.go:100).  The rows travel as one CSR allocation in C memory, written in one
// pass; the library's launch count does not depend on the number of rows.  Rows must ascend (a uid matrix row does);
// on any error, or when the call is too small to pay off, the result is mergeSortedGo's.
func MergeSortedMatrix(matrix []*pb.List) *pb.List {
	n, m := len(matrix), totalUids(matrix)
	if m < dgxMinMergeMatrix || uint64(m) >= 1<<32 {
		return mergeSortedGo(matrix)
	}
	// [v_off: n + 1 values | v: m values]
	csr := (*[1 << 30]C.uint64_t)(C.malloc(C.size_t(n+1+m) * 8))
	defer C.free(unsafe.Pointer(csr))
	voff, o := csr[:n+1:n+1], 0
	v := csr[n+1 : n+1+m : n+1+m]
	for i, r := range matrix {
		voff[i] = C.uint64_t(o)
		if r != nil && len(r.Uids) > 0 {
			C.memcpy(unsafe.Pointer(&v[o]), unsafe.Pointer(&r.Uids[0]), C.size_t(len(r.Uids)*8))
			o += len(r.Uids)
		}
	}
	voff[n] = C.uint64_t(o)
	out := make([]uint64, m)
	var outLen C.size_t
	if rc := C.dgx_merge_sorted_matrix(&v[0], &voff[0], C.size_t(n), u64ptr(out), C.size_t(m), &outLen); rc != C.DGX_OK {
		return mergeSortedGo(matrix)
	}
	return &pb.List{Uids: out[:int(outLen)]}
}

// Difference: algo/uidlist.go:332.  nil u or v -> non-nil empty list.
func Difference(u, v *pb.List) *pb.List {
	if u == nil || v == nil {
		return &pb.List{Uids: make([]uint64, 0)}
	}
	n, m := len(u.Uids), len(v.Uids)
	if n+m < dgxMinUids {
		return differenceGo(u, v)
	}
	out := make([]uint64, n)
	var outLen C.size_t
	rc := C.dgx_difference(u64ptr(u.Uids), C.size_t(n), u64ptr(v.Uids), C.size_t(m), u64ptr(out), C.size_t(n), &outLen)
	runtime.KeepAlive(u)
	runtime.KeepAlive(v)
	if rc != C.DGX_OK {
		return differenceGo(u, v)
	}
	return &pb.List{Uids: out[:int(outLen)]}
}

// IndexOfBatch answers algo.IndexOf(u, uid) (algo/uidlist.go:546-552) for every uid in one call: the
// shape of updateDestUids / updateFacetMatrix (query/query.go:1396-1416, 2594-2608), which probe
// sg.DestUIDs once per uid of the uid matrix.  idx[i] = -1 when uids[i] is absent.
func IndexOfBatch(u *pb.List, uids []uint64) []int64 {
	idx := make([]int64, len(uids))
	if len(uids) == 0 {
		return idx
	}
	if len(u.Uids)+len(uids) >= dgxMinUids {
		rc := C.dgx_index_of_batch(u64ptr(u.Uids), C.size_t(len(u.Uids)), u64ptr(uids), C.size_t(len(uids)),
			(*C.int64_t)(unsafe.Pointer(&idx[0])))
		runtime.KeepAlive(u)
		if rc == C.DGX_OK {
			return idx
		}
	}
	for i, x := range uids {
		idx[i] = int64(IndexOf(u, x))
	}
	return idx
}

// IntersectRowsWith replaces the loop `for _, l := range matrix { algo.IntersectWith(l, dest, l) }`
// (query/query.go:1425-1438 updateUidMatrix; worker/task.go:1351, 1616, 1691, 1777) with one batched call:
// the rows are flattened to CSR, `dest` crosses PCIe once, every row is filtered in place.
func IntersectRowsWith(matrix []*pb.List, dest *pb.List) {
	total := len(dest.Uids)
	for _, l := range matrix {
		total += len(l.Uids)
	}
	if total < dgxMinUids || len(matrix) == 0 {
		for _, l := range matrix {
			IntersectWith(l, dest, l)
		}
		return
	}
	flat := make([]uint64, 0, total-len(dest.Uids))
	off := make([]uint64, len(matrix)+1)
	for i, l := range matrix {
		flat = append(flat, l.Uids...)
		off[i+1] = uint64(len(flat))
	}
	out := make([]uint64, len(flat))
	outOff := make([]uint64, len(matrix)+1)
	rc := C.dgx_intersect_batch_shared(u64ptr(flat), u64ptr(off), C.size_t(len(matrix)), u64ptr(dest.Uids),
		C.size_t(len(dest.Uids)), u64ptr(out), u64ptr(outOff), C.size_t(len(out)))
	runtime.KeepAlive(dest)
	if rc != C.DGX_OK {
		for _, l := range matrix {
			IntersectWith(l, dest, l)
		}
		return
	}
	for i, l := range matrix {
		l.Uids = append(l.Uids[:0], out[outOff[i]:outOff[i+1]]...)
	}
}

// dgxMinGroupBy: below this many row values GroupByUid stays on the Go path (formResult's per-edge map).  The C13
// record (profiles/h100_c13_groupby.json) times the library against a C restatement of that path, not against Go, so
// this is the same bound as dgxMinMergeMatrix until a Go comparison sets it.
const dgxMinGroupBy = 1 << 14

// UidGroup is one group of a parent row of a @groupby over a uid predicate: its key (a uid of child.DestUIDs), its
// count(uid), and its ascending source uids when GroupByUid was asked for members.
type UidGroup struct {
	Key   uint64
	Count int
	Uids  []uint64
}

// GroupByUid is formResult's UID-node branch (query/groupby.go:208-221) for every parent row at once, and
// fillGroupedVars with parents = [{SrcUIDs}]: row i of matrix belongs to srcUIDs[i]; for each parent, the rows whose
// source is in it are grouped by destination, and the groups come back ordered by (count, key).  That is
// sort.Slice(groupLess)'s order when every aggregate child is count(uid); with value aggregates the caller sorts
// again.  dest is child.DestUIDs.  It returns false, and the caller keeps the Go path, below dgxMinGroupBy row values,
// when a parent row does not strictly ascend (orderasc / orderdesc on sg), and on any library error.
func GroupByUid(parents []*pb.List, srcUIDs []uint64, matrix []*pb.List, dest []uint64,
	withMembers bool) ([][]UidGroup, bool) {
	n, m, np := len(matrix), totalUids(matrix), len(parents)
	if n != len(srcUIDs) || m < dgxMinGroupBy || uint64(m) >= 1<<32 || np == 0 || uint64(np) >= 1<<32 {
		return nil, false
	}
	// every slice handed to C is its own Go allocation holding no Go pointers
	vOff, v := make([]uint64, n+1), make([]uint64, 0, m)
	for i, r := range matrix {
		vOff[i] = uint64(len(v))
		if r != nil {
			v = append(v, r.Uids...)
		}
	}
	vOff[n] = uint64(len(v))
	parOff, par := make([]uint64, np+1), make([]uint64, 0, totalUids(parents))
	for i, p := range parents {
		parOff[i] = uint64(len(par))
		if p != nil {
			for k, u := range p.Uids {
				if k > 0 && p.Uids[k-1] >= u {
					return nil, false // ordered parents: IndexOf bisects an unsorted list, keep Go's answer
				}
			}
			par = append(par, p.Uids...)
		}
	}
	parOff[np] = uint64(len(par))
	src := append([]uint64(nil), srcUIDs...)
	dst := append([]uint64(nil), dest...)
	grpOff := make([]uint64, np+1)
	gcap, mcap := m, m // one parent never has more; a larger call is sized again from the exact counts
	var keys, memOff, mem []uint64
	var ng, nm C.size_t
	rc := C.int(C.DGX_ERR_CAP)
	for attempt := 0; attempt < 2 && rc == C.DGX_ERR_CAP; attempt++ {
		keys, memOff = make([]uint64, gcap+1), make([]uint64, gcap+1)
		var memPtr *C.uint64_t
		if withMembers {
			mem = make([]uint64, mcap+1)
			memPtr = u64ptr(mem)
		}
		rc = C.dgx_groupby_uid(u64ptr(src), C.size_t(n), u64ptr(v), u64ptr(vOff), u64ptr(dst), C.size_t(len(dst)),
			u64ptr(par), u64ptr(parOff), C.size_t(np), u64ptr(keys), u64ptr(grpOff), u64ptr(memOff), C.size_t(gcap),
			memPtr, C.size_t(mcap), &ng, &nm)
		gcap, mcap = int(ng), int(nm)
	}
	if rc != C.DGX_OK {
		return nil, false
	}
	out := make([][]UidGroup, np)
	for p := 0; p < np; p++ {
		g0, g1 := int(grpOff[p]), int(grpOff[p+1])
		gs := make([]UidGroup, g1-g0)
		for g := g0; g < g1; g++ {
			lo, hi := memOff[g], memOff[g+1]
			gs[g-g0] = UidGroup{Key: keys[g], Count: int(hi - lo)}
			if withMembers {
				gs[g-g0].Uids = mem[lo:hi:hi]
			}
		}
		out[p] = gs
	}
	return out, true
}

// dgxMinRecurse: an expandRecurse attr moves its taken edges to the device once one sg's matrix of that attr reaches
// this many values; below it the Go map stays.  From the C14 record (profiles/h100_c14_recurse.json, H100 80GB HBM3,
// 700 W): a device-form step costs about 0.46 ms at C14b's sizes, and the C restatement of the Go loop spends 0.09-0.11
// us per value, so the two meet near 5 000 values.  The restatement is C with a hash set, not Go with Sprintf keys,
// which is slower, so the bound errs towards the Go path.
const dgxMinRecurse = 1 << 13

// Edge is one key of expandRecurse's reachMap for one attr: (fromUID, toUID).
type Edge struct{ From, To uint64 }

// ReachSet holds the edges one sg.Attr has taken during one @recurse (query/recurse.go expandRecurse, loop: false) in
// device memory.  Keep one per distinct Attr for the life of one expandRecurse; Close it when the recursion ends.
type ReachSet struct{ s *C.dgx_reach_set }

// NewReachSet creates a set from the edges Go has taken so far (any order; they are sorted here).  It returns false
// when the library refuses them (2^32 edges or more, no device); the caller keeps its map.
func NewReachSet(edges []Edge) (*ReachSet, bool) {
	sorted := append([]Edge(nil), edges...)
	sortEdges(sorted)
	from, to := make([]uint64, len(sorted)), make([]uint64, len(sorted))
	for i, e := range sorted {
		from[i], to[i] = e.From, e.To
	}
	var s *C.dgx_reach_set
	if C.dgx_reach_create(u64ptr(from), u64ptr(to), C.size_t(len(from)), &s) != C.DGX_OK {
		return nil, false
	}
	return &ReachSet{s: s}, true
}

func sortEdges(e []Edge) {
	sort.Slice(e, func(i, j int) bool { return e[i].From < e[j].From || (e[i].From == e[j].From && e[i].To < e[j].To) })
}

// Filter is :106-134 for one sg: with dest != nil (the sg has filters) every row is first intersected with dest
// (updateUidMatrix), then every edge already in the set is dropped and the rest are added.  It returns the kept rows
// (the new sg.uidMatrix), sg.DestUIDs and the step's contribution to numEdges.  ok == false, on any library error,
// means nothing was written and the set is unchanged: the caller exports it and finishes the attr in Go.
func (r *ReachSet) Filter(src *pb.List, matrix []*pb.List, dest *pb.List) (rows []*pb.List, destUIDs *pb.List,
	kept uint64, ok bool) {
	n, m := len(matrix), totalUids(matrix)
	if n != len(src.Uids) {
		return nil, nil, 0, false
	}
	// every slice handed to C is its own Go allocation holding no Go pointers
	vOff, v := make([]uint64, n+1), make([]uint64, 0, m)
	for i, l := range matrix {
		vOff[i] = uint64(len(v))
		if l != nil {
			v = append(v, l.Uids...)
		}
	}
	vOff[n] = uint64(len(v))
	srcs := append([]uint64(nil), src.Uids...)
	var dst []uint64
	var dstPtr *C.uint64_t
	var nd int
	if dest != nil {
		dst = append(make([]uint64, 0, len(dest.Uids)+1), dest.Uids...)
		dstPtr, nd = (*C.uint64_t)(unsafe.Pointer(&dst[:1][0])), len(dest.Uids)
	}
	out, outOff, dOut := make([]uint64, m+1), make([]uint64, n+1), make([]uint64, m+1)
	var dLen C.size_t
	rc := C.dgx_recurse_filter(r.s, u64ptr(srcs), C.size_t(n), u64ptr(v), u64ptr(vOff), dstPtr, C.size_t(nd),
		u64ptr(out), u64ptr(outOff), C.size_t(m), u64ptr(dOut), C.size_t(m), &dLen)
	if rc != C.DGX_OK {
		return nil, nil, 0, false
	}
	rows = make([]*pb.List, n)
	for i := range rows {
		lo, hi := outOff[i], outOff[i+1]
		rows[i] = &pb.List{Uids: out[lo:hi:hi]}
	}
	return rows, &pb.List{Uids: dOut[:dLen:dLen]}, outOff[n], true
}

// Export returns the set's edges, ascending by (From, To): how a recursion hands back to the Go map.
func (r *ReachSet) Export() ([]Edge, bool) {
	var n C.size_t
	if C.dgx_reach_size(r.s, &n) != C.DGX_OK {
		return nil, false
	}
	from, to := make([]uint64, int(n)+1), make([]uint64, int(n)+1)
	var got C.size_t
	if C.dgx_reach_export(r.s, u64ptr(from), u64ptr(to), n, &got) != C.DGX_OK {
		return nil, false
	}
	e := make([]Edge, int(got))
	for i := range e {
		e[i] = Edge{From: from[i], To: to[i]}
	}
	return e, true
}

// Close frees the set's device memory.
func (r *ReachSet) Close() {
	if r.s != nil {
		C.dgx_reach_destroy(r.s)
		r.s = nil
	}
}

// dgxMinCascade: below this many row values in a forest Cascade stays on the Go path (populateVarMap's per-row loops).
// The C15 record (profiles/h100_c15_cascade.json) times the library against a C restatement of that path, not against
// Go, so this is the same bound as dgxMinMergeMatrix until a Go comparison sets it.
const dgxMinCascade = 1 << 14

// Cascade flags, resolved by the caller from each SubGraph (INTEGRATION.md, @cascade).
const (
	CascadeOn       = uint8(C.DGX_CASCADE_CASCADE)  // len(Params.Cascade.Fields) > 0
	CascadeChecked  = uint8(C.DGX_CASCADE_CHECKED)  // the parent's cascade consults it: listed or __all__, not uid, not internal
	CascadeFiltered = uint8(C.DGX_CASCADE_FILTERED) // len(Filters) > 0
	CascadeOrdered  = uint8(C.DGX_CASCADE_ORDERED)  // Order or FacetsOrder
	CascadeSkip     = uint8(C.DGX_CASCADE_SKIP)     // IsGroupBy() or the shortest alias; such a node has no children here
)

// CascadeNode is one SubGraph of a @cascade forest, in pre-order: Parent is -1 for a query root and a smaller index
// otherwise; Rows is sg.uidMatrix, HasVal[i] is len(sg.valueMatrix[i].Values) > 0, CountsLen is len(sg.counts).
type CascadeNode struct {
	Parent        int
	Flags         uint8
	First, Offset int
	CountsLen     int
	Dest          []uint64
	Rows          []*pb.List
	HasVal        []byte
}

// Cascade runs populateVarMap's cascade path (query/query.go:1445-1527, updateUidMatrix without facets) for the whole
// forest and ProcessQuery's root pagination (:3004-3011) in one call.  It returns every node's rows and DestUIDs after
// the cascade, in node order.  It returns false, and the caller keeps the Go path, below dgxMinCascade row values,
// when a First / Offset does not fit int32, and on any library error (a malformed forest, rows that do not ascend).
func Cascade(nodes []CascadeNode) ([][][]uint64, [][]uint64, bool) {
	n := len(nodes)
	parent, flags := make([]uint32, n+1), make([]uint8, n+1)
	first, offset := make([]int32, n+1), make([]int32, n+1)
	counts := make([]uint64, n+1)
	rowOff, destOff, hvOff := make([]uint64, n+1), make([]uint64, n+1), make([]uint64, n+1)
	m, nd, nh, nr := 0, 0, 0, 0
	for _, c := range nodes {
		m += totalUids(c.Rows)
		nd += len(c.Dest)
		nh += len(c.HasVal)
		nr += len(c.Rows)
	}
	if m < dgxMinCascade || n == 0 {
		return nil, nil, false
	}
	// every slice handed to C directly is its own Go allocation holding no Go pointers
	v, vOff := make([]uint64, 0, m), make([]uint64, 1, nr+1)
	dest, hv := make([]uint64, 0, nd+1), make([]uint8, 0, nh+1)
	for k, c := range nodes {
		if c.First != int(int32(c.First)) || c.Offset != int(int32(c.Offset)) {
			return nil, nil, false
		}
		parent[k] = ^uint32(0)
		if c.Parent >= 0 {
			parent[k] = uint32(c.Parent)
		}
		flags[k], first[k], offset[k], counts[k] = c.Flags, int32(c.First), int32(c.Offset), uint64(c.CountsLen)
		for _, r := range c.Rows {
			if r != nil {
				v = append(v, r.Uids...)
			}
			vOff = append(vOff, uint64(len(v)))
		}
		rowOff[k+1] = uint64(len(vOff) - 1)
		dest = append(dest, c.Dest...)
		destOff[k+1] = uint64(len(dest))
		hv = append(hv, c.HasVal...)
		hvOff[k+1] = uint64(len(hv))
	}
	out, outOff := make([]uint64, m+1), make([]uint64, nr+1)
	dout, doutOff := make([]uint64, nd+1), make([]uint64, n+1)
	// the tree struct points at its arrays, so it and they live in C memory: Go memory handed to C must not hold Go
	// pointers
	frees := []func(){}
	defer func() {
		for _, f := range frees {
			f()
		}
	}()
	carr := func(p unsafe.Pointer, free func()) unsafe.Pointer {
		frees = append(frees, free)
		return p
	}
	tree := (*C.dgx_cascade_tree)(carr(cArray([]C.dgx_cascade_tree{{nnodes: C.size_t(n)}})))
	tree.parent = (*C.uint32_t)(carr(cArray(parent)))
	tree.flags = (*C.uint8_t)(carr(cArray(flags)))
	tree.first = (*C.int32_t)(carr(cArray(first)))
	tree.offset = (*C.int32_t)(carr(cArray(offset)))
	tree.counts_len = (*C.uint64_t)(carr(cArray(counts)))
	var hvPtr *C.uint8_t
	if len(hv) > 0 {
		hvPtr = (*C.uint8_t)(unsafe.Pointer(&hv[0]))
	}
	rc := C.dgx_cascade(tree, u64ptr(v), u64ptr(vOff), u64ptr(rowOff), u64ptr(dest), u64ptr(destOff), hvPtr,
		u64ptr(hvOff), u64ptr(out), u64ptr(outOff), C.size_t(m), u64ptr(dout), u64ptr(doutOff), C.size_t(nd))
	if rc != C.DGX_OK {
		return nil, nil, false
	}
	rows, dests := make([][][]uint64, n), make([][]uint64, n)
	for k := range nodes {
		rows[k] = make([][]uint64, rowOff[k+1]-rowOff[k])
		for i := range rows[k] {
			r := rowOff[k] + uint64(i)
			rows[k][i] = out[outOff[r]:outOff[r+1]:outOff[r+1]]
		}
		dests[k] = dout[doutOff[k]:doutOff[k+1]:doutOff[k+1]]
	}
	return rows, dests, true
}

// cArray copies v into a C allocation of max(len(v), 1) elements (an empty array still has an address) and returns it
// with the function that frees it.
func cArray[T any](v []T) (unsafe.Pointer, func()) {
	var zero T
	p := C.malloc(C.size_t(int(unsafe.Sizeof(zero)) * max(len(v), 1)))
	copy(unsafe.Slice((*T)(p), len(v)), v)
	return p, func() { C.free(p) }
}

// dgxMinShortest: a shortest() block goes to the device when the rows of its first level (From's edges over every
// child) hold at least this many values; below it Go's shortestPath runs.  From the C16 record
// (profiles/h100_c16_shortest.json, H100 80GB HBM3, 700 W): C16c, TestShortestPath4's 3 levels of 20 values, takes
// 0.70 ms through the host form, about 0.23 ms a level, and the C restatement spends about 2.4 us per row value at
// C16a's sizes, so the two meet near 100 values a level.  The restatement is C, not Go, and a first level is the
// smallest of a search, so the bound errs towards the Go path.
const dgxMinShortest = 1 << 10

// PathSearch is shortest() with numpaths <= 1 and no facets (query/shortest.go expandOut + shortestPath at unit
// cost) as a breadth-first search held in device memory.  Create one per query with NewPathSearch, call Expand once
// per level with that level's exec sgs in exec order, read the answer with Path, and Close it.
type PathSearch struct{ ps *C.dgx_path_search }

// PathSg is one exec sg of a level: the index of its child in sg.Children, SrcUIDs, the uidMatrix after
// updateUidMatrix (one row per source) and DestUIDs.
type PathSg struct {
	Attr   uint32
	Src    []uint64
	Matrix []*pb.List
	Dest   []uint64
}

// PathStats is one level's result: its numEdges, the nodes it discovered, and To's level (0 while unreached).
type PathStats struct{ Edges, Discovered, ToLevel uint64 }

// NewPathSearch starts a search from `from` to `to`.  It returns false when the library refuses them (a uid of 0,
// from == to, no device); the caller runs Go's shortestPath.
func NewPathSearch(from, to uint64) (*PathSearch, bool) {
	var ps *C.dgx_path_search
	if C.dgx_path_create(C.uint64_t(from), C.uint64_t(to), &ps) != C.DGX_OK {
		return nil, false
	}
	return &PathSearch{ps: ps}, true
}

// Expand runs one level over the exec sgs and returns each sg's next SrcUIDs.  ok == false, on any library error,
// means nothing was written: the caller closes the search and runs Go's shortestPath from the start.
func (p *PathSearch) Expand(sgs []PathSg) (next [][]uint64, st PathStats, ok bool) {
	n := len(sgs)
	if n == 0 {
		return nil, st, false
	}
	attr := make([]uint32, n)
	srcOff, destOff := make([]uint64, n+1), make([]uint64, n+1)
	var src, vOff, v, dest []uint64
	vOff = append(vOff, 0)
	for i, sg := range sgs {
		if len(sg.Matrix) != len(sg.Src) {
			return nil, st, false
		}
		attr[i] = sg.Attr
		src = append(src, sg.Src...)
		srcOff[i+1] = uint64(len(src))
		for _, l := range sg.Matrix {
			if l != nil {
				v = append(v, l.Uids...)
			}
			vOff = append(vOff, uint64(len(v)))
		}
		dest = append(dest, sg.Dest...)
		destOff[i+1] = uint64(len(dest))
	}
	// the level struct points at its arrays, so it and they live in C memory: Go memory handed to C must not hold Go
	// pointers
	frees := []func(){}
	defer func() {
		for _, f := range frees {
			f()
		}
	}()
	carr := func(q unsafe.Pointer, free func()) unsafe.Pointer {
		frees = append(frees, free)
		return q
	}
	lv := (*C.dgx_path_level)(carr(cArray([]C.dgx_path_level{{nsg: C.size_t(n)}})))
	lv.attr = (*C.uint32_t)(carr(cArray(attr)))
	lv.src_off = (*C.uint64_t)(carr(cArray(srcOff)))
	lv.src = (*C.uint64_t)(carr(cArray(src)))
	lv.v_off = (*C.uint64_t)(carr(cArray(vOff)))
	lv.v = (*C.uint64_t)(carr(cArray(v)))
	lv.dest_off = (*C.uint64_t)(carr(cArray(destOff)))
	lv.dest = (*C.uint64_t)(carr(cArray(dest)))
	out, outOff := make([]uint64, len(dest)+1), make([]uint64, n+1)
	var cst C.dgx_path_stats
	if C.dgx_path_expand(p.ps, lv, u64ptr(out), u64ptr(outOff), C.size_t(len(dest)), &cst) != C.DGX_OK {
		return nil, st, false
	}
	next = make([][]uint64, n)
	for i := range next {
		lo, hi := outOff[i], outOff[i+1]
		next[i] = out[lo:hi:hi]
	}
	return next, PathStats{Edges: uint64(cst.edges), Discovered: uint64(cst.discovered),
		ToLevel: uint64(cst.to_level)}, true
}

// Path returns the path From .. To and the child index of each hop (attrs[i] is the hop into uids[i+1]), both empty
// when To was not reached.
func (p *PathSearch) Path() (uids []uint64, attrs []uint32, ok bool) {
	var n C.size_t
	if rc := C.dgx_path_result(p.ps, nil, nil, 0, &n); rc != C.DGX_OK && rc != C.DGX_ERR_CAP {
		return nil, nil, false
	}
	if n == 0 {
		return nil, nil, true
	}
	uids, attrs = make([]uint64, int(n)), make([]uint32, int(n))
	if C.dgx_path_result(p.ps, u64ptr(uids), (*C.uint32_t)(unsafe.Pointer(&attrs[0])), n, &n) != C.DGX_OK {
		return nil, nil, false
	}
	return uids, attrs[:int(n)-1], true
}

// Close frees the search's device memory.
func (p *PathSearch) Close() {
	if p.ps != nil {
		C.dgx_path_destroy(p.ps)
		p.ps = nil
	}
}

// dgxMinVarProp / dgxMinLevelAgg: below this many row values (summed over a path's levels, or in relSG's matrix) a
// value variable stays on the Go path (transformTo, evalLevelAgg).  The C17 record (profiles/h100_c17_value_vars.json)
// times the library against a C restatement, not against Go, and every call also pays the ShardedMap <-> sorted-array
// conversion on the host, so both are the dgxMinMergeMatrix bound until a Go comparison sets them.
const (
	dgxMinVarProp  = dgxMinMergeMatrix
	dgxMinLevelAgg = dgxMinMergeMatrix
)

// VarLevel is one node of a value variable's path: SrcUIDs, uidMatrix (one row per source) and DestUIDs.
type VarLevel struct {
	Src    []uint64
	Matrix []*pb.List
	Dest   []uint64
}

// Value-map types (DGX_VAL_*) and level aggregations (DGX_AGG_*).
const (
	ValInt64   = C.DGX_VAL_INT64
	ValFloat64 = C.DGX_VAL_FLOAT64
	AggMin     = C.DGX_AGG_MIN
	AggMax     = C.DGX_AGG_MAX
	AggSum     = C.DGX_AGG_SUM
	AggAvg     = C.DGX_AGG_AVG
)

// varValues counts a uid matrix's values, for the gates, before anything is copied.
func varValues(rows []*pb.List) int {
	m := 0
	for _, l := range rows {
		if l != nil {
			m += len(l.Uids)
		}
	}
	return m
}

// varFlat flattens a uid matrix into C memory: (values, offsets, count, free).
func varFlat(rows []*pb.List) (unsafe.Pointer, unsafe.Pointer, int, func()) {
	off := make([]uint64, 1, len(rows)+1)
	var v []uint64
	for _, l := range rows {
		if l != nil {
			v = append(v, l.Uids...)
		}
		off = append(off, uint64(len(v)))
	}
	pv, fv := cArray(v)
	po, fo := cArray(off)
	return pv, po, len(v), func() { fv(); fo() }
}

// PropagateVar runs transformTo (query/query.go:1143-1236) over levels, the path from len(fromNode.path) on with
// index 0 skipped, for a map given as strictly ascending keys and 64-bit words of type typ (ValInt64 or
// ValFloat64).  It returns the map at the last level, ascending.  ok == false, below dgxMinVarProp values or on any
// library error, means the caller keeps transformTo.
func PropagateVar(typ int, keys, words []uint64, levels []VarLevel) (outKeys, outWords []uint64, ok bool) {
	if len(levels) == 0 || len(keys) != len(words) {
		return nil, nil, false
	}
	total := 0
	for _, l := range levels {
		if len(l.Matrix) != len(l.Src) {
			return nil, nil, false
		}
		total += varValues(l.Matrix)
	}
	if total < dgxMinVarProp {
		return nil, nil, false
	}
	frees := []func(){}
	defer func() {
		for _, f := range frees {
			f()
		}
	}()
	lv := make([]C.dgx_var_level, len(levels))
	for i, l := range levels {
		pv, po, _, free := varFlat(l.Matrix)
		ps, fs := cArray(l.Src)
		pd, fd := cArray(l.Dest)
		frees = append(frees, free, fs, fd)
		lv[i] = C.dgx_var_level{src: (*C.uint64_t)(ps), v_off: (*C.uint64_t)(po), v: (*C.uint64_t)(pv),
			dest: (*C.uint64_t)(pd), nrows: C.size_t(len(l.Src)), ndest: C.size_t(len(l.Dest))}
	}
	plv, flv := cArray(lv)
	frees = append(frees, flv)
	d := len(levels[len(levels)-1].Dest)
	outKeys, outWords = make([]uint64, d+1), make([]uint64, d+1)
	var n C.size_t
	if C.dgx_var_propagate(C.int(typ), u64ptr(keys), u64ptr(words), C.size_t(len(keys)),
		(*C.dgx_var_level)(plv), C.size_t(len(levels)), u64ptr(outKeys), u64ptr(outWords), C.size_t(d),
		&n) != C.DGX_OK {
		return nil, nil, false
	}
	return outKeys[:int(n)], outWords[:int(n)], true
}

// LevelAgg runs evalLevelAgg's per-row branch (query/query.go:1088-1123): fn (AggMin .. AggAvg) of the map's values
// over each row of relSG's uidMatrix.  It returns the keys (src[i] of every row with a present value) and the words,
// of type ValFloat64 for AggAvg and typ otherwise.  ok == false, below dgxMinLevelAgg values or on any library error,
// means the caller keeps evalLevelAgg.
func LevelAgg(typ, fn int, keys, words, src []uint64, matrix []*pb.List) (outKeys, outWords []uint64, ok bool) {
	if len(matrix) != len(src) || len(keys) != len(words) || varValues(matrix) < dgxMinLevelAgg {
		return nil, nil, false
	}
	pv, po, _, free := varFlat(matrix)
	defer free()
	outKeys, outWords = make([]uint64, len(src)+1), make([]uint64, len(src)+1)
	var n C.size_t
	if C.dgx_var_level_agg(C.int(typ), C.int(fn), u64ptr(keys), u64ptr(words), C.size_t(len(keys)), u64ptr(src),
		C.size_t(len(src)), (*C.uint64_t)(po), (*C.uint64_t)(pv), u64ptr(outKeys), u64ptr(outWords),
		C.size_t(len(src)), &n) != C.DGX_OK {
		return nil, nil, false
	}
	return outKeys[:int(n)], outWords[:int(n)], true
}

// dgxMinMath: below this many leaf entries (summed over a math() tree's variables) evalMathTree stays in Go.  No Go
// comparison exists yet (the C18 record, profiles/h100_c18_math.json, times the library against a C restatement), and
// every call pays the ShardedMap <-> sorted-array conversion on the host, so it is the dgxMinMergeMatrix bound.
const dgxMinMath = dgxMinMergeMatrix

// Math ops (DGX_MATH_*) and the extra entry tags of a math() map (DGX_VAL_*).
const (
	ValBool       = C.DGX_VAL_BOOL
	ValNil        = C.DGX_VAL_NIL
	MathKindNone  = C.DGX_MATH_KIND_NONE
	MathKindMap   = C.DGX_MATH_KIND_MAP
	MathKindConst = C.DGX_MATH_KIND_CONST
)

// MathNode is one node of a math() program in post-order (dgx_math_node): Op a DGX_MATH_* op, Child the indices of
// its children (earlier nodes), Leaf the Leaves index of a DGX_MATH_VAR node, ConstTag / ConstWord a constant's
// ValInt64 / ValFloat64 tag and bits.
type MathNode struct {
	Op, ConstTag uint8
	Child        [3]uint16
	Leaf         uint32
	ConstWord    uint64
}

// MathLeaf is one variable's map after transformTo: ascending keys, one word and one DGX_VAL_* tag per key; Nil for
// a variable with no map (a nil ShardedMap).
type MathLeaf struct {
	Keys, Words []uint64
	Tags        []uint8
	Nil         bool
}

// EvalMath runs evalMathTree (query/math.go) and valueVarAggregation's math branch (query/query.go:1290-1361) in one
// call.  rangeOver is SrcUIDs (DestUIDs at the root), nil when Go's rangeOver is nil.  It returns the kind
// (MathKindMap, MathKindConst, MathKindNone) and the entries, ascending.  ok == false, for a program outside the
// library's bounds, below dgxMinMath entries, or on any library error (including a refusal where Go's answer is an
// error or depends on map iteration order), means the caller keeps evalMathTree.
func EvalMath(prog []MathNode, leaves []MathLeaf, rangeOver []uint64, hasRange bool) (kind int, keys, words []uint64,
	tags []uint8, ok bool) {
	if len(prog) == 0 || len(prog) > C.DGX_MATH_MAX_NODES || len(leaves) > C.DGX_MATH_MAX_LEAVES {
		return 0, nil, nil, nil, false
	}
	total := 0
	for _, l := range leaves {
		if len(l.Keys) != len(l.Words) || len(l.Keys) != len(l.Tags) {
			return 0, nil, nil, nil, false
		}
		total += len(l.Keys)
	}
	if total < dgxMinMath {
		return 0, nil, nil, nil, false
	}
	cl := make([]C.dgx_math_leaf, max(len(leaves), 1))
	var frees []func()
	defer func() {
		for _, f := range frees {
			f()
		}
	}()
	for j, l := range leaves {
		pk, fk := cArray(l.Keys)
		pw, fw := cArray(l.Words)
		pt, ft := cArray(l.Tags)
		frees = append(frees, fk, fw, ft)
		n, isNil := len(l.Keys), C.int(0)
		if l.Nil {
			n, isNil = 0, 1
		}
		cl[j] = C.dgx_math_leaf{key: (*C.uint64_t)(pk), word: (*C.uint64_t)(pw), tag: (*C.uint8_t)(pt),
			n: C.size_t(n), _type: C.DGX_VAL_INT64, nil: isNil}
	}
	cp := make([]C.dgx_math_node, len(prog))
	for i, p := range prog {
		cp[i] = C.dgx_math_node{op: C.uint8_t(p.Op), const_tag: C.uint8_t(p.ConstTag), leaf: C.uint32_t(p.Leaf),
			const_word: C.uint64_t(p.ConstWord)}
		for c := 0; c < 3; c++ {
			cp[i].child[c] = C.uint16_t(p.Child[c])
		}
	}
	pl, fl := cArray(cl)
	pp, fp := cArray(cp)
	frees = append(frees, fl, fp)
	var pr *C.uint64_t
	if hasRange {
		r, fr := cArray(rangeOver)
		frees = append(frees, fr)
		pr = (*C.uint64_t)(r)
	}
	cap := max(total+1, len(rangeOver))
	keys, words, tags = make([]uint64, cap), make([]uint64, cap), make([]uint8, cap)
	var info C.uint64_t
	if C.dgx_math_eval((*C.dgx_math_node)(pp), C.size_t(len(prog)), (*C.dgx_math_leaf)(pl), C.size_t(len(leaves)), pr,
		C.size_t(len(rangeOver)), u64ptr(keys), u64ptr(words), (*C.uint8_t)(unsafe.Pointer(&tags[0])),
		C.size_t(cap), &info) != C.DGX_OK {
		return 0, nil, nil, nil, false
	}
	n := int(uint64(info) & 0xffffffff)
	return int((uint64(info) >> 32) & 0xff), keys[:n], words[:n], tags[:n], true
}

// dgxMinSgFilter: below this many D0 values plus row values a node's @filter and pagination stay in Go (ProcessGraph's
// filter block, applyPagination).  The C19 record (profiles/h100_c19_sg_filter.json) times the library against a C
// restatement of that path, not against Go, so this is the same bound as dgxMinMergeMatrix until a Go comparison sets
// it.
const dgxMinSgFilter = dgxMinMergeMatrix

// SgFilter tree ops and leaf kinds (include/dgx.h).
const (
	SgfLeaf = uint8(C.DGX_SGF_LEAF)
	SgfAnd  = uint8(C.DGX_SGF_AND)
	SgfOr   = uint8(C.DGX_SGF_OR)
	SgfNot  = uint8(C.DGX_SGF_NOT)
)

// SgFilterLeaf is one resolved filter leaf: a LIST (Uids strictly ascending: a function's DestUIDs, uid(var), literal
// uids, D0 or nil for gt(len(x), n)), or a COUNT (Cmp one of "le" "ge" "lt" "gt" "eq", Threshold, and either Counts,
// one per D0 value, or Off, D0's row offsets).
type SgFilterLeaf struct {
	IsCount   bool
	Uids      []uint64
	Cmp       string
	Threshold int64
	Counts    []uint32
	Off       []uint64
}

// SgFilter runs ProcessGraph's filter block, applyPagination (updateUidMatrix, x.PageRange) and the DoCount block
// (query/query.go:2310-2413) for one node in one call: op / parent / leaf are filterCopy's tree flattened (node 0 the
// root, parents below their children), d0 the node's DestUIDs from processTask, rows its uid matrix.  It returns the
// rows (nil when countsOnly), their lengths and the new DestUIDs.  It returns false, and the caller keeps the Go path,
// below dgxMinSgFilter values, when the node has facets, an Order or FacetsOrder without DoCount, a count or offset
// outside int32, a literal uid(...) leaf that does not strictly ascend (the parser keeps duplicates, and Go's answer
// then depends on which IntersectWith variant runs), a COUNT leaf without exactly one of Counts (len(d0) entries) and
// Off (len(d0) + 1 entries), and on any library error.
func SgFilter(op []uint8, parent, leaf []uint32, leaves []SgFilterLeaf, d0 []uint64, rows []*pb.List, count, offset int,
	ordered, doCount, facets, countsOnly bool) ([][]uint64, []uint32, []uint64, bool) {
	if facets || (ordered && !doCount) || count != int(int32(count)) || offset != int(int32(offset)) {
		return nil, nil, nil, false
	}
	if ordered { // DoCount with an order skips pagination (:2375-2394)
		count, offset = 0, 0
	}
	m, nrows := totalUids(rows), len(rows)
	if len(d0)+m < dgxMinSgFilter || len(op) == 0 {
		return nil, nil, nil, false
	}
	cmps := map[string]C.int{"le": C.DGX_SGF_CMP_LE, "ge": C.DGX_SGF_CMP_GE, "lt": C.DGX_SGF_CMP_LT,
		"gt": C.DGX_SGF_CMP_GT, "eq": C.DGX_SGF_CMP_EQ}
	frees := []func(){}
	defer func() {
		for _, f := range frees {
			f()
		}
	}()
	carr := func(p unsafe.Pointer, free func()) unsafe.Pointer {
		frees = append(frees, free)
		return p
	}
	cl := make([]C.dgx_sg_filter_leaf, len(leaves)+1)
	for j, l := range leaves {
		if !l.IsCount {
			for i := 1; i < len(l.Uids); i++ {
				if l.Uids[i-1] >= l.Uids[i] {
					return nil, nil, nil, false
				}
			}
			cl[j].kind, cl[j].n = C.DGX_SGF_LIST, C.size_t(len(l.Uids))
			cl[j].uids = (*C.uint64_t)(carr(cArray(l.Uids)))
			continue
		}
		c, ok := cmps[l.Cmp]
		// the library copies exactly len(d0) counts or len(d0) + 1 offsets: anything else stays in Go
		if !ok || (l.Counts != nil) == (l.Off != nil) || (l.Counts != nil && len(l.Counts) != len(d0)) ||
			(l.Off != nil && len(l.Off) != len(d0)+1) {
			return nil, nil, nil, false
		}
		cl[j].kind, cl[j].cmp, cl[j].threshold = C.DGX_SGF_COUNT, c, C.int64_t(l.Threshold)
		if l.Counts != nil {
			cl[j].counts = (*C.uint32_t)(carr(cArray(l.Counts)))
		} else {
			cl[j].off = (*C.uint64_t)(carr(cArray(l.Off)))
		}
	}
	tree := (*C.dgx_sg_filter_tree)(carr(cArray([]C.dgx_sg_filter_tree{{nnodes: C.size_t(len(op))}})))
	tree.op = (*C.uint8_t)(carr(cArray(op)))
	tree.parent = (*C.uint32_t)(carr(cArray(parent)))
	tree.leaf = (*C.uint32_t)(carr(cArray(leaf)))
	ctab := (*C.dgx_sg_filter_leaf)(carr(cArray(cl)))
	v, vOff := make([]uint64, 0, m+1), make([]uint64, 1, nrows+1)
	for _, r := range rows {
		if r != nil {
			v = append(v, r.Uids...)
		}
		vOff = append(vOff, uint64(len(v)))
	}
	dest, out, outOff := make([]uint64, len(d0)+1), make([]uint64, m+1), make([]uint64, nrows+1)
	counts := make([]uint32, nrows+1)
	var n C.size_t
	outPtr := u64ptr(out)
	if countsOnly {
		outPtr = nil
	}
	d0c := append(make([]uint64, 0, len(d0)+1), d0...)
	rc := C.dgx_sg_filter(tree, ctab, C.size_t(len(leaves)), u64ptr(d0c), C.size_t(len(d0)), u64ptr(v), u64ptr(vOff),
		C.size_t(nrows), C.int32_t(count), C.int32_t(offset), u64ptr(dest), C.size_t(len(d0)), &n, outPtr,
		u64ptr(outOff), C.size_t(m), (*C.uint32_t)(unsafe.Pointer(&counts[0])))
	if rc != C.DGX_OK {
		return nil, nil, nil, false
	}
	var res [][]uint64
	if !countsOnly {
		res = make([][]uint64, nrows)
		for i := range res {
			res[i] = out[outOff[i]:outOff[i+1]:outOff[i+1]]
		}
	}
	return res, counts[:nrows], dest[:n], true
}

// dgxMinVarOrder: below this many dest values plus row values a node's order by a value variable stays in Go
// (applyOrderAndPagination's value-variable branch).  The C20 record (profiles/h100_c20_var_order.json) times the
// library against a C restatement of that path, not against Go, so this is the dgxMinMergeMatrix bound until a Go
// comparison sets it.
const dgxMinVarOrder = dgxMinMergeMatrix

// OrderByVar runs applyOrderAndPagination's value-variable branch (query/query.go:2511-2530: updateUidMatrix's order
// branch, sortAndPaginateUsingVar with types.Sort and x.PageRange, updateDestUids) in one call, in Go's exact order,
// ties included.  m is Params.UidToVal as a MathLeaf: int64 and float64 values as ValInt64 / ValFloat64 words, a
// math() map's bools and nils as ValBool / ValNil; a map holding any other type (string, DateTime, ...) is not passed
// here.  dest is sg.DestUIDs after the filter block, rows the uid matrix, count / offset Params.Count / Offset.  It
// returns the new rows and DestUIDs.  ok == false -- FacetsOrder set (sortAndPaginateUsingFacet), DoCount, a nil map
// (Go's "used before definition" error, which Go then returns), sizes outside the library's bounds, below
// dgxMinVarOrder values, or any library error (including a row whose first mapped value is a bool, Go's "isn't
// sortable") -- means the caller keeps Go's path.
func OrderByVar(m MathLeaf, desc bool, dest []uint64, rows []*pb.List, count, offset int, facetsOrder,
	doCount bool) ([][]uint64, []uint64, bool) {
	if facetsOrder || doCount || m.Nil || count != int(int32(count)) || offset != int(int32(offset)) ||
		len(m.Keys) != len(m.Words) || len(m.Keys) != len(m.Tags) {
		return nil, nil, false
	}
	mv, nrows := totalUids(rows), len(rows)
	if len(dest)+mv < dgxMinVarOrder {
		return nil, nil, false
	}
	var frees []func()
	defer func() {
		for _, f := range frees {
			f()
		}
	}()
	pk, fk := cArray(m.Keys)
	pw, fw := cArray(m.Words)
	pt, ft := cArray(m.Tags)
	frees = append(frees, fk, fw, ft)
	leaf := []C.dgx_math_leaf{{key: (*C.uint64_t)(pk), word: (*C.uint64_t)(pw), tag: (*C.uint8_t)(pt),
		n: C.size_t(len(m.Keys)), _type: C.DGX_VAL_INT64}}
	pl, fl := cArray(leaf)
	frees = append(frees, fl)
	v, vOff := make([]uint64, 0, mv+1), make([]uint64, 1, nrows+1)
	for _, r := range rows {
		if r != nil {
			v = append(v, r.Uids...)
		}
		vOff = append(vOff, uint64(len(v)))
	}
	d := append(make([]uint64, 0, len(dest)+1), dest...)
	destOut, out, outOff := make([]uint64, len(dest)+1), make([]uint64, mv+1), make([]uint64, nrows+1)
	var n C.size_t
	isDesc := C.int(0)
	if desc {
		isDesc = 1
	}
	if C.dgx_var_order((*C.dgx_math_leaf)(pl), isDesc, u64ptr(d), C.size_t(len(dest)), u64ptr(v), u64ptr(vOff),
		C.size_t(nrows), C.int32_t(count), C.int32_t(offset), u64ptr(out), u64ptr(outOff), C.size_t(mv),
		u64ptr(destOut), C.size_t(len(dest)), &n) != C.DGX_OK {
		return nil, nil, false
	}
	res := make([][]uint64, nrows)
	for i := range res {
		res[i] = out[outOff[i]:outOff[i+1]:outOff[i+1]]
	}
	return res, destOut[:n], true
}

// dgxMinPredOrder: below this many dest values plus row values a node's order by a predicate stays in Go
// (applyOrderAndPagination's predicate branch).  No measurement of the call exists yet, so this is the
// dgxMinMergeMatrix bound until one sets it.
const dgxMinPredOrder = dgxMinMergeMatrix

// OrderByPred runs applyOrderAndPagination's predicate branch for a predicate whose sortWithIndex fails before it
// reads (no index, or no sortable tokenizer: worker/sort.go:210-240), so that processSort's answer is always
// sortWithoutIndex's (worker/sort.go:139-187, sortByValue, paginate), in one dgx_pred_order call.  col holds the
// predicate's values as fetchValue reads them (ValueFor at ReadTs, types.Convert to the schema type, a failed
// conversion marked Bad, an absent value left out); order is sg.Params.Order; sortable reports whether sortWithIndex
// could run; isList the schema's list flag; dest is sg.DestUIDs, rows the matrix updateUidMatrix left, count (already
// 1000 for 0) / offset the SortMessage's.  It returns the new rows and DestUIDs.  ok == false -- a sortable index (the
// answer is then a race with the indexed sort), more than one order key (multiSort), Langs, FacetsOrder, a list
// predicate, a type other than int64, float64, datetime and string (bool keeps Go's error and its all-null case),
// sizes outside the library's bounds, below dgxMinPredOrder values, or any library error -- means the caller keeps
// SortOverNetwork.  The facets reorder after the sort stays in Go.
func OrderByPred(col *ValColumn, order []*pb.Order, sortable, isList, facetsOrder bool, dest []uint64,
	rows []*pb.List, count, offset int) ([][]uint64, []uint64, bool) {
	if sortable || len(order) != 1 || len(order[0].Langs) > 0 || facetsOrder || isList || count < 0 ||
		count != int(int32(count)) || offset != int(int32(offset)) {
		return nil, nil, false
	}
	switch col.Type {
	case ValInt64, ValFloat64, ValDateTime, ValString:
	default:
		return nil, nil, false
	}
	mv, nrows := totalUids(rows), len(rows)
	if len(dest)+mv < dgxMinPredOrder {
		return nil, nil, false
	}
	pc, _, free := cValCall(col, &ValArgs{})
	defer free()
	v, vOff := make([]uint64, 0, mv+1), make([]uint64, 1, nrows+1)
	for _, r := range rows {
		if r != nil {
			v = append(v, r.Uids...)
		}
		vOff = append(vOff, uint64(len(v)))
	}
	d := append(make([]uint64, 0, len(dest)+1), dest...)
	destOut, out, outOff := make([]uint64, len(dest)+1), make([]uint64, mv+1), make([]uint64, nrows+1)
	var n C.size_t
	isDesc := C.int(0)
	if order[0].Desc {
		isDesc = 1
	}
	if C.dgx_pred_order((*C.dgx_val_column)(pc), isDesc, u64ptr(d), C.size_t(len(dest)), u64ptr(v), u64ptr(vOff),
		C.size_t(nrows), C.int32_t(count), C.int32_t(offset), u64ptr(out), u64ptr(outOff), C.size_t(mv),
		u64ptr(destOut), C.size_t(len(dest)), &n) != C.DGX_OK {
		return nil, nil, false
	}
	res := make([][]uint64, nrows)
	for i := range res {
		res[i] = out[outOff[i]:outOff[i+1]:outOff[i+1]]
	}
	return res, destOut[:n], true
}

// dgxMinMatch: below this many candidates a match() stays in Go (handleMatchFunction).  The C21 record
// (profiles/h100_c21_match.json) times the library against a C restatement of that loop, not against Go, so this is
// the dgxMinMergeMatrix bound until a Go comparison sets it.
const dgxMinMatch = dgxMinMergeMatrix

// StrColumn is a predicate's string values as handleMatchFunction reads them at ReadTs: Uids strictly ascending,
// Vals[i] the values of Uids[i] from the same choice Go's loop makes (pl.ValueForTag(lang) with a lang,
// pl.AllUntaggedValues for a list predicate, pl.Value otherwise); a uid whose read is ErrNoValue is left out.
type StrColumn struct {
	Uids []uint64
	Vals [][][]byte
}

// MatchFuzzy runs handleMatchFunction's candidate loop (worker/task.go:1526-1620) in one call: the candidates are
// uids when it is not empty (the filter's UidList), otherwise the union of rows, uidsForMatch's pl.Uids reads of the
// query's trigram tokens (worker/match.go:72-100), and a candidate is kept when one of its values passes
// matchFuzzy(query, val, max).  It returns the kept uids, the task's one UidMatrix row.  ok == false -- max outside
// int32 or negative, a query above DGX_MATCH_MAX_RUNES runes, fewer than dgxMinMatch candidates, sizes outside the
// library's bounds (DGX_ERR_ARG / DGX_ERR_CAP) or any other library error -- means the caller keeps Go's loop.
func MatchFuzzy(col *StrColumn, query string, max int64, uids []uint64, rows [][]uint64) ([]uint64, bool) {
	bound := len(uids)
	if bound == 0 {
		for _, r := range rows {
			bound += len(r)
		}
	}
	if bound < dgxMinMatch || len(col.Uids) != len(col.Vals) {
		return nil, false
	}
	pc, free := cStrColumn(col)
	defer free()
	pq, fq := cArray([]byte(query))
	defer fq()
	lists, listOff := candidateRows(uids, rows, bound)
	out := make([]uint64, bound+1)
	var n C.size_t
	if C.dgx_match(nil, 0, nil, nil, nil, u64ptr(lists), u64ptr(listOff), C.size_t(len(listOff)-1), 0,
		u64ptr(uids), C.size_t(len(uids)), (*C.dgx_str_column)(pc), (*C.uint8_t)(pq), C.size_t(len(query)), C.int64_t(max),
		u64ptr(out), C.size_t(bound), &n) != C.DGX_OK {
		return nil, false
	}
	return out[:n:n], true
}

// cStrColumn copies col into C memory as a dgx_str_column: the struct holds pointers, so it and every array it names
// live in C memory (cgo's pointer rules).  The caller calls free when the library is done with it.
func cStrColumn(col *StrColumn) (unsafe.Pointer, func()) {
	valOff, byteOff := make([]uint64, 1, len(col.Uids)+1), make([]uint64, 1, len(col.Uids)+1)
	var data []byte
	for _, vs := range col.Vals {
		for _, v := range vs {
			data = append(data, v...)
			byteOff = append(byteOff, uint64(len(data)))
		}
		valOff = append(valOff, uint64(len(byteOff)-1))
	}
	pu, fu := cArray(col.Uids)
	pv, fv := cArray(valOff)
	pbo, fbo := cArray(byteOff)
	pd, fd := cArray(data)
	pc, fc := cArray([]C.dgx_str_column{{uid: (*C.uint64_t)(pu), val_off: (*C.uint64_t)(pv),
		byte_off: (*C.uint64_t)(pbo), bytes: (*C.uint8_t)(pd), n: C.size_t(len(col.Uids)),
		nvals: C.size_t(len(byteOff) - 1), nbytes: C.size_t(len(data))}})
	return pc, func() { fc(); fd(); fbo(); fv(); fu() }
}

// candidateRows lays rows out as list leaves when uids is empty (the trigram branch), as dgx_match and
// dgx_regex_match take them.
func candidateRows(uids []uint64, rows [][]uint64, bound int) ([]uint64, []uint64) {
	lists, listOff := make([]uint64, 0, bound+1), make([]uint64, 1, len(rows)+1)
	if len(uids) == 0 {
		for _, r := range rows {
			lists = append(lists, r...)
			listOff = append(listOff, uint64(len(lists)))
		}
	}
	return lists, listOff
}

// dgxMinRegex: below this many candidates a regexp() stays in Go (handleRegexFunction).  No C22 record times the
// library against Go's loop yet, so this is the dgxMinMatch bound until one sets it.
const dgxMinRegex = dgxMinMatch

// MatchRegex is handleRegexFunction's value loop (worker/task.go:1240-1356, matchRegex :1809-1811) in one
// dgx_regex_match call: pattern is the regexp's pattern as cregexp.Compile takes it before the "(?m)" prefix, fold the
// i modifier.  The candidates are uids when not empty (the @filter branch's UidList), otherwise the union of rows,
// uidsForRegex's result.  Returns the kept candidates and true; false -- a pattern outside the compiled subset
// (DGX_ERR_ARG), a DFA past DGX_REGEX_MAX_STATES (DGX_ERR_CAP), fewer than dgxMinRegex candidates, or any other
// library error -- means the caller keeps cregexp and Go's loop.  The caller then intersects every UidMatrix row with
// the result as before.
func MatchRegex(col *StrColumn, pattern string, fold bool, uids []uint64, rows [][]uint64) ([]uint64, bool) {
	bound := len(uids)
	if bound == 0 {
		for _, r := range rows {
			bound += len(r)
		}
	}
	if bound < dgxMinRegex || len(col.Uids) != len(col.Vals) {
		return nil, false
	}
	pp, fp := cArray([]byte(pattern))
	defer fp()
	flags := C.int(0)
	if fold {
		flags = C.DGX_REGEX_FOLD
	}
	var prog *C.dgx_regex_prog
	if C.dgx_regex_compile((*C.char)(pp), C.size_t(len(pattern)), flags, &prog) != C.DGX_OK {
		return nil, false
	}
	defer C.dgx_regex_free(prog)
	pc, free := cStrColumn(col)
	defer free()
	lists, listOff := candidateRows(uids, rows, bound)
	out := make([]uint64, bound+1)
	var n C.size_t
	if C.dgx_regex_match(nil, 0, nil, nil, nil, u64ptr(lists), u64ptr(listOff), C.size_t(len(listOff)-1), 0,
		u64ptr(uids), C.size_t(len(uids)), (*C.dgx_str_column)(pc), prog, u64ptr(out), C.size_t(bound), &n) != C.DGX_OK {
		return nil, false
	}
	return out[:n:n], true
}

// dgxMinCompare: below this many candidates (or index-row values) a compare function stays in Go.  No C23 record times
// the library against Go's loops yet, so this is the dgxMinMergeMatrix bound, as dgxMinMatch is, until one sets it.
const dgxMinCompare = dgxMinMergeMatrix

// The types of a ValColumn beyond ValInt64 / ValFloat64 / ValBool, and the compare ops (DGX_SGF_CMP_*).
const (
	ValDateTime = C.DGX_VAL_DATETIME
	ValString   = C.DGX_VAL_STRING
	CmpLE       = C.DGX_SGF_CMP_LE
	CmpGE       = C.DGX_SGF_CMP_GE
	CmpLT       = C.DGX_SGF_CMP_LT
	CmpGT       = C.DGX_SGF_CMP_GT
	CmpEQ       = C.DGX_SGF_CMP_EQ
	CmpBetween  = C.DGX_SGF_CMP_BETWEEN
)

// ValColumn is a predicate's values converted to its schema type as Go's compare loops read them (types.Convert of
// each stored value): Uids strictly ascending; for Type ValString the values of Uids[i] are Str.Vals[i] (Str.Uids is
// Uids), otherwise Words[i] (int64, float64 bits, bool 0 / 1, or a datetime's Unix seconds with Nsec[i] its
// nanoseconds).  Bad[i][j], when Bad is set, marks a value whose conversion failed or gave nil.
type ValColumn struct {
	Type  int
	Uids  []uint64
	Words [][]uint64
	Nsec  [][]uint32
	Str   *StrColumn
	Bad   [][]bool
}

// ValArgs are a compare function's arguments (srcFn.eqTokens) of the column's type: Words (and Nsec) or Strs.
type ValArgs struct {
	Words []uint64
	Nsec  []uint32
	Strs  [][]byte
}

// cValCall copies col and args into C memory as a dgx_val_column and a dgx_val_args (cgo's pointer rules), the
// string values through cStrColumn, the helper MatchFuzzy uses.  The caller calls free when the library is done.
func cValCall(col *ValColumn, args *ValArgs) (unsafe.Pointer, unsafe.Pointer, func()) {
	var frees []func()
	keep := func(p unsafe.Pointer, f func()) unsafe.Pointer { frees = append(frees, f); return p }
	valOff := []uint64{0}
	var words []uint64
	var nsec []uint32
	var bad []uint8
	var str unsafe.Pointer
	for i := range col.Uids {
		k := 0
		if col.Type == ValString {
			k = len(col.Str.Vals[i])
		} else {
			k = len(col.Words[i])
			words = append(words, col.Words[i]...)
			if col.Type == ValDateTime {
				nsec = append(nsec, col.Nsec[i]...)
			}
		}
		if col.Bad != nil {
			for _, b := range col.Bad[i] {
				if b {
					bad = append(bad, 1)
				} else {
					bad = append(bad, 0)
				}
			}
		}
		valOff = append(valOff, valOff[len(valOff)-1]+uint64(k))
	}
	if col.Type == ValString {
		str = keep(cStrColumn(col.Str))
	}
	var pbad unsafe.Pointer
	if col.Bad != nil {
		pbad = keep(cArray(bad))
	}
	pc := keep(cArray([]C.dgx_val_column{{_type: C.int(col.Type), uid: (*C.uint64_t)(keep(cArray(col.Uids))),
		val_off: (*C.uint64_t)(keep(cArray(valOff))), word: (*C.uint64_t)(keep(cArray(words))),
		nsec: (*C.uint32_t)(keep(cArray(nsec))), bad: (*C.uint8_t)(pbad), str: (*C.dgx_str_column)(str),
		n: C.size_t(len(col.Uids)), nvals: C.size_t(valOff[len(valOff)-1])}}))
	argOff := []uint64{0}
	var argBytes []byte
	for _, s := range args.Strs {
		argBytes = append(argBytes, s...)
		argOff = append(argOff, uint64(len(argBytes)))
	}
	n := len(args.Words)
	if col.Type == ValString {
		n = len(args.Strs)
	}
	pa := keep(cArray([]C.dgx_val_args{{word: (*C.uint64_t)(keep(cArray(args.Words))),
		nsec: (*C.uint32_t)(keep(cArray(args.Nsec))), bytes: (*C.uint8_t)(keep(cArray(argBytes))),
		byte_off: (*C.uint64_t)(keep(cArray(argOff))), n: C.size_t(n)}}))
	return pc, pa, func() {
		for i := len(frees) - 1; i >= 0; i-- {
			frees[i]()
		}
	}
}

// CompareUids is handleValuePostings' compareAttrFn branch (worker/task.go:540-575) in one dgx_compare_uids call:
// op is CmpLE .. CmpEQ or CmpBetween, uids the task's UidList.  It returns the kept uids (the merged DestUIDs) and,
// per candidate, Go's row length (UidList[i] appended once per matching value).  ok == false -- fewer than
// dgxMinCompare candidates, sizes or types outside the library's bounds, a candidate's bad value (Go returns the
// conversion error; the caller's loop then reports it) or any other library error -- means the caller keeps Go's loop.
func CompareUids(col *ValColumn, op int, args *ValArgs, uids []uint64) ([]uint64, []uint32, bool) {
	if len(uids) < dgxMinCompare {
		return nil, nil, false
	}
	pc, pa, free := cValCall(col, args)
	defer free()
	out := make([]uint64, len(uids)+1)
	counts := make([]uint32, len(uids)+1)
	var n C.size_t
	if C.dgx_compare_uids(C.int(op), (*C.dgx_val_args)(pa), (*C.dgx_val_column)(pc), u64ptr(uids), C.size_t(len(uids)),
		u64ptr(out), C.size_t(len(uids)), &n, (*C.uint32_t)(unsafe.Pointer(&counts[0]))) != C.DGX_OK {
		return nil, nil, false
	}
	return out[:n:n], counts[:len(uids):len(uids)], true
}

// CompareRowArgs builds row_arg from handleCompareFunction's three cases (worker/task.go:1487-1520): eq pairs row r
// with eqTokens[r] (ok == false where Go would index past eqTokens), between filters rows 0 and nrows - 1, another op
// row 0 when tokens[0] == ineqValueToken[0].
func CompareRowArgs(op, nrows, nEqTokens int, firstIsIneq bool) ([]uint32, bool) {
	ra := make([]uint32, nrows)
	for r := range ra {
		ra[r] = ^uint32(0)
	}
	switch {
	case op == CmpEQ:
		if nrows > nEqTokens {
			return nil, false
		}
		for r := range ra {
			ra[r] = uint32(r)
		}
	case op == CmpBetween:
		if nrows > 0 {
			ra[0], ra[nrows-1] = 0, 0
		}
	case firstIsIneq && nrows > 0:
		ra[0] = 0
	}
	return ra, true
}

// CompareRows is handleCompareFunction's filterRow calls (worker/task.go:1395-1520) in one dgx_compare_rows call over
// the index uid matrix rows, row_arg from CompareRowArgs.  It returns the filtered rows; ok == false -- fewer than
// dgxMinCompare values or any library error -- means the caller keeps Go's filterRow loop.
func CompareRows(col *ValColumn, op int, args *ValArgs, rows []*pb.List, rowArg []uint32) ([][]uint64, bool) {
	m := varValues(rows)
	if m < dgxMinCompare || len(rowArg) != len(rows) || len(rows) == 0 {
		return nil, false
	}
	pc, pa, free := cValCall(col, args)
	defer free()
	pv, pvo, _, fv := varFlat(rows)
	defer fv()
	pr, fr := cArray(rowArg)
	defer fr()
	out := make([]uint64, m+1)
	outOff := make([]uint64, len(rows)+1)
	if C.dgx_compare_rows(C.int(op), (*C.dgx_val_args)(pa), (*C.dgx_val_column)(pc), (*C.uint64_t)(pv),
		(*C.uint64_t)(pvo), C.size_t(len(rows)), (*C.uint32_t)(pr), u64ptr(out), u64ptr(outOff), C.size_t(m)) != C.DGX_OK {
		return nil, false
	}
	res := make([][]uint64, len(rows))
	for r := range rows {
		res[r] = out[outOff[r]:outOff[r+1]:outOff[r+1]]
	}
	return res, true
}
