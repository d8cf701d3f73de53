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
