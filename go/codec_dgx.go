//go:build dgx

// Package codec -- cgo shim for codec.Decode (codec/codec.go:444) over libdgx.
// NOT COMPILED IN THIS REPOSITORY (no Go toolchain in the build image); see
// go/algo_dgx.go and INTEGRATION.md.
package codec

/*
#cgo CFLAGS: -I${SRCDIR}/../include
#cgo LDFLAGS: -ldgx
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "dgx.h"
*/
import "C"

import (
	"math"
	"unsafe"

	"github.com/dgraph-io/dgraph/v25/protos/pb"
)

const dgxMinDecode = 1 << 16

// flatten copies pb.UidPack (Blocks []*UidBlock: pointers to structs, each with its
// own Deltas slice) into the struct-of-arrays dgx_pack_view, in C memory: cgo cannot
// pass Go memory that contains Go pointers.
func flatten(pack *pb.UidPack) (C.dgx_pack_view, func()) {
	nb := len(pack.Blocks)
	total := 0
	for _, b := range pack.Blocks {
		total += len(b.Deltas)
	}
	base := (*[1 << 28]C.uint64_t)(C.malloc(C.size_t(nb*8 + 8)))
	num := (*[1 << 28]C.uint32_t)(C.malloc(C.size_t(nb*4 + 4)))
	off := (*[1 << 28]C.uint64_t)(C.malloc(C.size_t(nb*8 + 8)))
	del := C.malloc(C.size_t(total + 16))
	o := 0
	for i, b := range pack.Blocks {
		base[i] = C.uint64_t(b.Base)
		num[i] = C.uint32_t(b.NumUids)
		off[i] = C.uint64_t(o)
		if len(b.Deltas) > 0 {
			C.memcpy(unsafe.Add(del, o), unsafe.Pointer(&b.Deltas[0]), C.size_t(len(b.Deltas)))
		}
		o += len(b.Deltas)
	}
	off[nb] = C.uint64_t(o)
	var v C.dgx_pack_view
	v.block_size = C.uint32_t(pack.BlockSize)
	v.nblocks = C.size_t(nb)
	v.base = (*C.uint64_t)(unsafe.Pointer(base))
	v.num_uids = (*C.uint32_t)(unsafe.Pointer(num))
	v.delta_off = (*C.uint64_t)(unsafe.Pointer(off))
	v.deltas = (*C.uint8_t)(del)
	return v, func() { C.free(unsafe.Pointer(base)); C.free(unsafe.Pointer(num)); C.free(unsafe.Pointer(off)); C.free(del) }
}

// Decode keeps codec/codec.go:444's contract: uids from Seek(seek, SeekStart) onward,
// a non-nil (possibly empty) slice, sized with ExactLen (ApproxLen is 0 for
// BlockSize-0 packs and only an estimate otherwise).
func Decode(pack *pb.UidPack, seek uint64) []uint64 {
	n := ExactLen(pack)
	if pack == nil || n < dgxMinDecode {
		return decodeGo(pack, seek)
	}
	view, free := flatten(pack)
	defer free()
	out := make([]uint64, n)
	var outLen C.size_t
	if rc := C.dgx_decode(&view, C.uint64_t(seek), (*C.uint64_t)(unsafe.Pointer(&out[0])), C.size_t(n), &outLen); rc != C.DGX_OK {
		return decodeGo(pack, seek)
	}
	return out[:int(outLen)]
}

// DecodeStored decodes the uids of a posting list straight from its stored bytes (the
// value proto.Unmarshal receives at posting/list.go:1045): the pb.UidPack inside the
// serialized pb.PostingList is parsed into the struct-of-arrays view by libdgx itself
// (dgx_wire_*), so no []*pb.UidBlock is ever built.  New entry point (not in the
// reference); nil for a posting list without a pack.
func DecodeStored(value []byte, seek uint64) ([]uint64, bool) {
	if len(value) == 0 {
		return []uint64{}, true
	}
	buf := (*C.uint8_t)(unsafe.Pointer(&value[0]))
	var sub *C.uint8_t
	var subLen C.size_t
	if C.dgx_wire_posting_list_pack(buf, C.size_t(len(value)), &sub, &subLen) != C.DGX_OK {
		return nil, false
	}
	if sub == nil {
		return []uint64{}, true
	}
	var nb, db C.size_t
	if C.dgx_wire_pack_measure(sub, subLen, &nb, &db) != C.DGX_OK {
		return nil, false
	}
	base := C.malloc(nb*8 + 8)
	num := C.malloc(nb*4 + 4)
	off := C.malloc(nb*8 + 16)
	del := C.malloc(db + 16)
	defer func() { C.free(base); C.free(num); C.free(off); C.free(del) }()
	var view C.dgx_pack_view
	if C.dgx_wire_pack_parse(sub, subLen, (*C.uint64_t)(base), (*C.uint32_t)(num), (*C.uint64_t)(off),
		(*C.uint8_t)(del), nb, db, &view) != C.DGX_OK {
		return nil, false
	}
	n := 0
	nums := (*[1 << 28]C.uint32_t)(num)[:int(nb):int(nb)]
	for _, c := range nums {
		n += int(c) // codec.ExactLen
	}
	out := make([]uint64, n)
	var outLen C.size_t
	var outPtr *C.uint64_t
	if n > 0 {
		outPtr = (*C.uint64_t)(unsafe.Pointer(&out[0]))
	}
	if C.dgx_decode(&view, C.uint64_t(seek), outPtr, C.size_t(n), &outLen) != C.DGX_OK {
		return nil, false
	}
	return out[:int(outLen)], true
}

// packRef names a pack for the HBM-resident cache of libdgx: key = hash of the posting list's Badger key,
// version = commit timestamp of the immutable layer the pack was rolled up at (posting.List.minTs).
// key 0 = anonymous (copied for this call only).
type PackRef struct {
	Pack    *pb.UidPack
	Key     uint64
	Version uint64
}

// IntersectCompressedWithRef is algo.IntersectCompressedWith (algo/uidlist.go:33-61), the entry point of
// posting.List.Uids for filtered reads (posting/list.go:1795-1800): o.Uids = v ∩ pack[>= afterUID].  The pack
// crosses PCIe compressed (or not at all when (Key, Version) is already resident); only blocks whose range
// holds an element of v are decoded.  Returns false when the caller must run the Go path.
func IntersectCompressedWithRef(ref PackRef, afterUID uint64, v, o *pb.List) bool {
	if ref.Pack == nil {
		return true // `if pack == nil { return }`: o untouched
	}
	if ApproxLen(ref.Pack)+len(v.Uids) < dgxMinDecode {
		return false
	}
	view, free := flatten(ref.Pack)
	defer free()
	cref := C.dgx_pack_ref{pack: &view, key: C.uint64_t(ref.Key), version: C.uint64_t(ref.Version)}
	out := make([]uint64, len(v.Uids))
	var outLen C.size_t
	var vp, op *C.uint64_t
	if len(v.Uids) > 0 {
		vp = (*C.uint64_t)(unsafe.Pointer(&v.Uids[0]))
		op = (*C.uint64_t)(unsafe.Pointer(&out[0]))
	}
	if C.dgx_intersect_compressed_ref(&cref, C.uint64_t(afterUID), vp, C.size_t(len(v.Uids)), op, C.size_t(len(out)), &outLen) != C.DGX_OK {
		return false
	}
	o.Uids = out[:int(outLen)]
	return true
}

// IntersectCompressedWithRows is algo.IntersectCompressedWith(refs[i].Pack, afterUID, v, o_i) for every i in ONE
// library call: the loop handleUidPostings (worker/task.go:783-987) runs over a task's keys with one ListOptions
// (posting/list.go:1795-1800).  Row i of the result is o_i; a nil pack leaves its row as &pb.List{} (the reference
// leaves o untouched).  Anonymous packs (Key 0) are flattened back to back into one C staging buffer in the
// library's flat-image layout, so they cross PCIe as one transfer; named packs use the HBM cache.  The rows are
// slices of one result buffer.  The size threshold applies to the batch total, not to each row: a task of many
// small lists is what pays off.  Returns false when the caller must run the Go path.
func IntersectCompressedWithRows(refs []PackRef, afterUID uint64, v *pb.List) ([]*pb.List, bool) {
	n := len(refs)
	if n == 0 {
		return []*pb.List{}, true
	}
	total, capOut, img := len(v.Uids), 0, 0
	for _, r := range refs {
		if r.Pack == nil || len(r.Pack.Blocks) == 0 {
			continue
		}
		total += ApproxLen(r.Pack)
		if e := ExactLen(r.Pack); e < len(v.Uids) {
			capOut += e
		} else {
			capOut += len(v.Uids)
		}
		if r.Key == 0 {
			img += int(C.dgx_pack_image_size(C.size_t(len(r.Pack.Blocks)), C.size_t(deltaBytes(r.Pack))))
		}
	}
	if total < dgxMinDecode || uint64(len(v.Uids)) >= 1<<32 {
		return nil, false
	}
	crefs := (*[1 << 28]C.dgx_pack_ref)(C.malloc(C.size_t(n) * C.size_t(unsafe.Sizeof(C.dgx_pack_ref{}))))
	views := (*[1 << 28]C.dgx_pack_view)(C.malloc(C.size_t(n) * C.size_t(unsafe.Sizeof(C.dgx_pack_view{}))))
	stage := C.malloc(C.size_t(img + 64))
	frees := []func(){}
	defer func() {
		for _, f := range frees {
			f()
		}
		C.free(unsafe.Pointer(crefs))
		C.free(unsafe.Pointer(views))
		C.free(stage)
	}()
	o := 0
	for i, r := range refs {
		crefs[i] = C.dgx_pack_ref{key: C.uint64_t(r.Key), version: C.uint64_t(r.Version)}
		if r.Pack == nil || len(r.Pack.Blocks) == 0 {
			continue // empty row
		}
		if r.Key != 0 {
			view, free := flatten(r.Pack)
			frees = append(frees, free)
			views[i] = view
		} else {
			nb, db := len(r.Pack.Blocks), deltaBytes(r.Pack)
			if C.dgx_pack_image_view(unsafe.Add(stage, o), C.uint32_t(r.Pack.BlockSize), C.size_t(nb), C.size_t(db), &views[i]) != C.DGX_OK {
				return nil, false
			}
			fillImage(&views[i], r.Pack)
			o += int(C.dgx_pack_image_size(C.size_t(nb), C.size_t(db)))
		}
		crefs[i].pack = &views[i]
	}
	out := make([]uint64, capOut+1)
	off := make([]uint64, n+1)
	var vp *C.uint64_t
	if len(v.Uids) > 0 {
		vp = (*C.uint64_t)(unsafe.Pointer(&v.Uids[0]))
	}
	if C.dgx_intersect_compressed_rows(&crefs[0], C.size_t(n), C.uint64_t(afterUID), vp, C.size_t(len(v.Uids)),
		(*C.uint64_t)(unsafe.Pointer(&out[0])), (*C.uint64_t)(unsafe.Pointer(&off[0])), C.size_t(capOut)) != C.DGX_OK {
		return nil, false
	}
	rows := make([]*pb.List, n)
	for i, r := range refs {
		if r.Pack == nil {
			rows[i] = &pb.List{}
			continue
		}
		rows[i] = &pb.List{Uids: out[off[i]:off[i+1]:off[i+1]]}
	}
	return rows, true
}

// dgxMinMatrix: below this many uids (ApproxLen of the bucket + all rows) IntersectCompressedWithMatrix stays on the
// Go path.  Set from the C7 record (profiles/h100_c7_sort_buckets.json, H100 80GB HBM3, 400 W): the host form took
// 0.62 ms for the whole tiny-bucket call, and the row loop on one CPU thread spent 0.64 us per matrix uid there, so
// a matrix of about 1 000 uids costs the Go loop what one library call costs.
const dgxMinMatrix = 1 << 10

// IntersectCompressedWithMatrix is algo.IntersectCompressedWith(ref.Pack, 0, rows[i], o_i) for every row of a uid
// matrix in ONE library call: the loop intersectBucket (worker/sort.go:605-700) runs for each index bucket of a sort,
// reaching algo.IntersectCompressedWith through posting/list.go:1795-1800.  Every row must be strictly ascending (a
// uid matrix row is).  The rows travel as one CSR allocation in C memory; the result rows are slices of one buffer.
// A nil / empty pack gives empty rows.  Returns false when the caller must keep pl.Uids: on any error, when the call
// is too small to pay off (dgxMinMatrix), or when the matrix holds 2^32 uids or more.
func IntersectCompressedWithMatrix(ref PackRef, rows []*pb.List) ([]*pb.List, bool) {
	n := len(rows)
	if n == 0 {
		return []*pb.List{}, true
	}
	m, capOut := 0, 0
	exact := ExactLen(ref.Pack)
	for _, r := range rows {
		m += len(r.Uids)
		if len(r.Uids) < exact {
			capOut += len(r.Uids)
		} else {
			capOut += exact
		}
	}
	if ApproxLen(ref.Pack)+m < dgxMinMatrix || uint64(m) >= 1<<32 {
		return nil, false
	}
	// [v_off: n + 1 values | v: m values]
	csr := (*[1 << 30]C.uint64_t)(C.malloc(C.size_t(n+1+m) * 8))
	defer C.free(unsafe.Pointer(csr))
	voff, o := csr[:n+1:n+1], 0
	v := csr[n+1 : n+1+m : n+1+m]
	for i, r := range rows {
		voff[i] = C.uint64_t(o)
		if len(r.Uids) > 0 {
			C.memcpy(unsafe.Pointer(&v[o]), unsafe.Pointer(&r.Uids[0]), C.size_t(len(r.Uids)*8))
		}
		o += len(r.Uids)
	}
	voff[n] = C.uint64_t(o)
	cref := C.dgx_pack_ref{key: C.uint64_t(ref.Key), version: C.uint64_t(ref.Version)}
	if ref.Pack != nil && len(ref.Pack.Blocks) > 0 {
		view, free := flatten(ref.Pack)
		defer free()
		cref.pack = &view
	}
	out := make([]uint64, capOut+1)
	off := make([]uint64, n+1)
	var vp *C.uint64_t
	if m > 0 {
		vp = &v[0]
	}
	if C.dgx_intersect_compressed_matrix(&cref, vp, &voff[0], C.size_t(n), (*C.uint64_t)(unsafe.Pointer(&out[0])),
		(*C.uint64_t)(unsafe.Pointer(&off[0])), C.size_t(capOut)) != C.DGX_OK {
		return nil, false
	}
	res := make([]*pb.List, n)
	for i := range rows {
		res[i] = &pb.List{Uids: out[off[i]:off[i+1]:off[i+1]]}
	}
	return res, true
}

func deltaBytes(pack *pb.UidPack) int {
	t := 0
	for _, b := range pack.Blocks {
		t += len(b.Deltas)
	}
	return t
}

// fillImage writes pack's blocks into the arrays dgx_pack_image_view pointed v at.
func fillImage(v *C.dgx_pack_view, pack *pb.UidPack) {
	nb := len(pack.Blocks)
	base := (*[1 << 28]C.uint64_t)(unsafe.Pointer(v.base))[:nb:nb]
	num := (*[1 << 28]C.uint32_t)(unsafe.Pointer(v.num_uids))[:nb:nb]
	off := (*[1 << 28]C.uint64_t)(unsafe.Pointer(v.delta_off))[: nb+1 : nb+1]
	o := 0
	for i, b := range pack.Blocks {
		base[i] = C.uint64_t(b.Base)
		num[i] = C.uint32_t(b.NumUids)
		off[i] = C.uint64_t(o)
		if len(b.Deltas) > 0 {
			C.memcpy(unsafe.Add(unsafe.Pointer(v.deltas), o), unsafe.Pointer(&b.Deltas[0]), C.size_t(len(b.Deltas)))
		}
		o += len(b.Deltas)
	}
	off[nb] = C.uint64_t(o)
}

// IntersectSortedPacks is algo.IntersectSorted over lists still held as packs: every pack is decoded on the
// device (codec.Decode(p, 0)) and the k-way intersection runs there; ~1.5 B/UID cross PCIe instead of 8.
func IntersectSortedPacks(refs []PackRef) (*pb.List, bool) {
	if len(refs) == 0 {
		return &pb.List{}, true
	}
	crefs := (*[1 << 20]C.dgx_pack_ref)(C.malloc(C.size_t(len(refs)) * C.size_t(unsafe.Sizeof(C.dgx_pack_ref{}))))
	views := (*[1 << 20]C.dgx_pack_view)(C.malloc(C.size_t(len(refs)) * C.size_t(unsafe.Sizeof(C.dgx_pack_view{}))))
	frees := make([]func(), 0, len(refs))
	defer func() {
		for _, f := range frees {
			f()
		}
		C.free(unsafe.Pointer(crefs))
		C.free(unsafe.Pointer(views))
	}()
	minLen := int(^uint(0) >> 1)
	for i, r := range refs {
		crefs[i] = C.dgx_pack_ref{key: C.uint64_t(r.Key), version: C.uint64_t(r.Version)}
		if r.Pack == nil || len(r.Pack.Blocks) == 0 {
			return &pb.List{Uids: []uint64{}}, true // an empty operand empties the intersection
		}
		v, free := flatten(r.Pack)
		frees = append(frees, free)
		views[i] = v
		crefs[i].pack = &views[i]
		if n := ExactLen(r.Pack); n < minLen {
			minLen = n
		}
	}
	out := make([]uint64, minLen+1)
	var outLen C.size_t
	if C.dgx_intersect_sorted_packed(&crefs[0], C.size_t(len(refs)), (*C.uint64_t)(unsafe.Pointer(&out[0])), C.size_t(minLen), &outLen) != C.DGX_OK {
		return nil, false
	}
	return &pb.List{Uids: out[:int(outLen)]}, true
}

// EncodeDevice is codec.Encode (codec/codec.go:393-399) with the block split and the group-varint bytes produced
// on the device; the result is rebuilt as a pb.UidPack whose blocks share one Deltas backing array.
func EncodeDevice(uids []uint64, blockSize int) (*pb.UidPack, bool) {
	if len(uids) == 0 {
		return nil, true
	}
	var nbCap, dbCap C.size_t
	C.dgx_encode_bound(C.size_t(len(uids)), C.uint32_t(blockSize), &nbCap, &dbCap)
	for attempt := 0; attempt < 2; attempt++ {
		base := make([]uint64, int(nbCap)+1)
		num := make([]uint32, int(nbCap)+1)
		off := make([]uint64, int(nbCap)+2)
		del := make([]byte, int(dbCap)+1)
		nb, db := nbCap, dbCap
		rc := C.dgx_encode((*C.uint64_t)(unsafe.Pointer(&uids[0])), C.size_t(len(uids)), C.uint32_t(blockSize),
			(*C.uint64_t)(unsafe.Pointer(&base[0])), (*C.uint32_t)(unsafe.Pointer(&num[0])),
			(*C.uint64_t)(unsafe.Pointer(&off[0])), (*C.uint8_t)(unsafe.Pointer(&del[0])), &nb, &db, nil)
		if rc == C.DGX_ERR_CAP && (nb > nbCap || db > dbCap) {
			nbCap, dbCap = nb, db // the exact sizes came back: one more try
			continue
		}
		if rc != C.DGX_OK {
			return nil, false
		}
		pack := &pb.UidPack{BlockSize: uint32(blockSize), Blocks: make([]*pb.UidBlock, int(nb))}
		blocks := make([]pb.UidBlock, int(nb))
		for i := range blocks {
			blocks[i] = pb.UidBlock{Base: base[i], NumUids: num[i], Deltas: del[off[i]:off[i+1]:off[i+1]]}
			pack.Blocks[i] = &blocks[i]
		}
		return pack, true
	}
	return nil, false
}

// MutRow is a key's mutable layer as List.Uids sees it, resolved by the caller under l.RLock (INTEGRATION §2): one
// entry per uid, strictly ascending, Flags[i] = DGX_MUT_DEL (Op == Del) | DGX_MUT_VALUE (PostingType != REF).
type MutRow struct {
	Uids  []uint64
	Flags []uint8
}

// ListUidsRows is posting.List.Uids(opts) (posting/list.go:1758-1874) for every key of a task in ONE library call:
// the handleUidPostings loop (worker/task.go:783-987) of a filtered read (opts.Intersect = v, non-empty) of unsplit
// lists, mutable layers included.  modes[i] is the branch List.Uids takes for key i (DGX_UIDS_COMPRESSED without a
// mutable layer, DGX_UIDS_PROBE when len(v) < ApproxLen, DGX_UIDS_ITERATE otherwise); refs[i].Pack is nil for a key
// whose delete-all marker hides the immutable layer.  Packs are staged as in IntersectCompressedWithRows; the mutable
// layers cross as one C allocation (offsets, uids, flags, modes).  The size threshold applies to the batch total.
// Returns false when the caller must keep pl.Uids.
func ListUidsRows(refs []PackRef, modes []uint8, muts []MutRow, afterUID uint64, v *pb.List) ([]*pb.List, bool) {
	n, m := len(refs), len(v.Uids)
	if n == 0 {
		return []*pb.List{}, true
	}
	if m == 0 || uint64(m) >= 1<<31 || len(modes) != n || len(muts) != n {
		return nil, false
	}
	total, capOut, img, nmut := m, 0, 0, 0
	for i, r := range refs {
		nm, e := len(muts[i].Uids), 0
		nmut += nm
		if r.Pack != nil && len(r.Pack.Blocks) > 0 {
			total += ApproxLen(r.Pack)
			e = ExactLen(r.Pack)
			if r.Key == 0 {
				img += int(C.dgx_pack_image_size(C.size_t(len(r.Pack.Blocks)), C.size_t(deltaBytes(r.Pack))))
			}
		}
		if e+nm < m {
			capOut += e + nm
		} else {
			capOut += m
		}
	}
	if total+nmut < dgxMinDecode {
		return nil, false
	}
	// [mut_off (n + 1) | mut_uids (nmut, plus one spare word so &words[n+1] exists) | mut_flags (nmut bytes) | modes]
	csr := C.malloc(C.size_t((n+2+nmut)*8 + nmut + n + 16))
	crefs := (*[1 << 28]C.dgx_pack_ref)(C.malloc(C.size_t(n) * C.size_t(unsafe.Sizeof(C.dgx_pack_ref{}))))
	views := (*[1 << 28]C.dgx_pack_view)(C.malloc(C.size_t(n) * C.size_t(unsafe.Sizeof(C.dgx_pack_view{}))))
	stage := C.malloc(C.size_t(img + 64))
	frees := []func(){}
	defer func() {
		for _, f := range frees {
			f()
		}
		C.free(csr)
		C.free(unsafe.Pointer(crefs))
		C.free(unsafe.Pointer(views))
		C.free(stage)
	}()
	words := unsafe.Slice((*uint64)(csr), n+2+nmut)
	small := unsafe.Slice((*uint8)(unsafe.Add(csr, (n+2+nmut)*8)), nmut+n)
	w := 0
	for i, mr := range muts {
		if len(mr.Flags) != len(mr.Uids) {
			return nil, false
		}
		words[i] = uint64(w)
		copy(words[n+1+w:], mr.Uids)
		copy(small[w:], mr.Flags)
		w += len(mr.Uids)
	}
	words[n] = uint64(w)
	copy(small[nmut:], modes)
	o := 0
	for i, r := range refs {
		crefs[i] = C.dgx_pack_ref{key: C.uint64_t(r.Key), version: C.uint64_t(r.Version)}
		if r.Pack == nil || len(r.Pack.Blocks) == 0 {
			continue // delete-all marker or empty immutable layer
		}
		if r.Key != 0 {
			view, free := flatten(r.Pack)
			frees = append(frees, free)
			views[i] = view
		} else {
			nb, db := len(r.Pack.Blocks), deltaBytes(r.Pack)
			if C.dgx_pack_image_view(unsafe.Add(stage, o), C.uint32_t(r.Pack.BlockSize), C.size_t(nb), C.size_t(db), &views[i]) != C.DGX_OK {
				return nil, false
			}
			fillImage(&views[i], r.Pack)
			o += int(C.dgx_pack_image_size(C.size_t(nb), C.size_t(db)))
		}
		crefs[i].pack = &views[i]
	}
	out := make([]uint64, capOut+1)
	off := make([]uint64, n+1)
	if C.dgx_list_uids_rows(&crefs[0], (*C.uint8_t)(unsafe.Pointer(&small[nmut])), C.size_t(n),
		(*C.uint64_t)(unsafe.Pointer(&words[n+1])), (*C.uint8_t)(unsafe.Pointer(&small[0])), (*C.uint64_t)(unsafe.Pointer(&words[0])),
		C.uint64_t(afterUID), (*C.uint64_t)(unsafe.Pointer(&v.Uids[0])), C.size_t(m),
		(*C.uint64_t)(unsafe.Pointer(&out[0])), (*C.uint64_t)(unsafe.Pointer(&off[0])), C.size_t(capOut)) != C.DGX_OK {
		return nil, false
	}
	rows := make([]*pb.List, n)
	for i := range refs {
		rows[i] = &pb.List{}
		if off[i+1] > off[i] {
			rows[i].Uids = out[off[i]:off[i+1]:off[i+1]]
		}
	}
	return rows, true
}

// unfilteredStage holds what the unfiltered and count calls pass: the packs staged as in ListUidsRows and the mutable
// layers as one C allocation [mut_off (n + 1) | mut_uids (nmut, plus one spare word) | mut_flags (nmut bytes)].
type unfilteredStage struct {
	crefs *C.dgx_pack_ref
	off   *C.uint64_t
	uids  *C.uint64_t
	flags *C.uint8_t
	exact []int // ExactLen + |mut| per key
	free  func()
}

// stageUnfiltered stages a task's keys for dgx_list_uids_unfiltered_rows / dgx_list_count_rows.  It returns false
// when the batch is too small to pay for a call or the input is malformed.
func stageUnfiltered(refs []PackRef, muts []MutRow) (*unfilteredStage, bool) {
	n := len(refs)
	if len(muts) != n {
		return nil, false
	}
	total, img, nmut := 0, 0, 0
	exact := make([]int, n)
	for i, r := range refs {
		if len(muts[i].Flags) != len(muts[i].Uids) {
			return nil, false
		}
		nmut += len(muts[i].Uids)
		exact[i] = len(muts[i].Uids)
		if r.Pack != nil && len(r.Pack.Blocks) > 0 {
			total += ApproxLen(r.Pack)
			exact[i] += ExactLen(r.Pack)
			if r.Key == 0 {
				img += int(C.dgx_pack_image_size(C.size_t(len(r.Pack.Blocks)), C.size_t(deltaBytes(r.Pack))))
			}
		}
	}
	if total+nmut < dgxMinDecode || nmut >= 1<<31 {
		return nil, false
	}
	csr := C.malloc(C.size_t((n+2+nmut)*8 + nmut + 16))
	crefs := (*[1 << 28]C.dgx_pack_ref)(C.malloc(C.size_t(n) * C.size_t(unsafe.Sizeof(C.dgx_pack_ref{}))))
	views := (*[1 << 28]C.dgx_pack_view)(C.malloc(C.size_t(n) * C.size_t(unsafe.Sizeof(C.dgx_pack_view{}))))
	stage := C.malloc(C.size_t(img + 64))
	frees := []func(){}
	s := &unfilteredStage{exact: exact, free: func() {
		for _, f := range frees {
			f()
		}
		C.free(csr)
		C.free(unsafe.Pointer(crefs))
		C.free(unsafe.Pointer(views))
		C.free(stage)
	}}
	words := unsafe.Slice((*uint64)(csr), n+2+nmut)
	flags := unsafe.Slice((*uint8)(unsafe.Add(csr, (n+2+nmut)*8)), nmut+1)
	w := 0
	for i, mr := range muts {
		words[i] = uint64(w)
		copy(words[n+1+w:], mr.Uids)
		copy(flags[w:], mr.Flags)
		w += len(mr.Uids)
	}
	words[n] = uint64(w)
	o := 0
	for i, r := range refs {
		crefs[i] = C.dgx_pack_ref{key: C.uint64_t(r.Key), version: C.uint64_t(r.Version)}
		if r.Pack == nil || len(r.Pack.Blocks) == 0 {
			continue // delete-all marker or empty immutable layer
		}
		if r.Key != 0 {
			view, free := flatten(r.Pack)
			frees = append(frees, free)
			views[i] = view
		} else {
			nb, db := len(r.Pack.Blocks), deltaBytes(r.Pack)
			if C.dgx_pack_image_view(unsafe.Add(stage, o), C.uint32_t(r.Pack.BlockSize), C.size_t(nb), C.size_t(db), &views[i]) != C.DGX_OK {
				s.free()
				return nil, false
			}
			fillImage(&views[i], r.Pack)
			o += int(C.dgx_pack_image_size(C.size_t(nb), C.size_t(db)))
		}
		crefs[i].pack = &views[i]
	}
	s.crefs = &crefs[0]
	s.off = (*C.uint64_t)(unsafe.Pointer(&words[0]))
	s.uids = (*C.uint64_t)(unsafe.Pointer(&words[n+1]))
	s.flags = (*C.uint8_t)(unsafe.Pointer(&flags[0]))
	return s, true
}

// ListUidsUnfilteredRows is posting.List.Uids(opts) with opts.Intersect == nil (posting/list.go:1758-1874) for every
// key of a task in ONE library call: the default branch of handleUidPostings without facets (worker/task.go:960-967)
// over unsplit lists, mutable layers included (INTEGRATION §2 lists the keys that qualify).  refs[i].Pack is nil for a
// key whose delete-all marker hides the immutable layer; first is opts.First.  Returns false when the caller must keep
// pl.Uids.
func ListUidsUnfilteredRows(refs []PackRef, muts []MutRow, afterUID uint64, first int32) ([]*pb.List, bool) {
	n := len(refs)
	if n == 0 {
		return []*pb.List{}, true
	}
	s, ok := stageUnfiltered(refs, muts)
	if !ok {
		return nil, false
	}
	defer s.free()
	keep := int(first)
	if first == 0 {
		keep = math.MaxInt32
	} else if first < 0 {
		keep = 1
	}
	capOut := 0
	for _, e := range s.exact {
		if e < keep {
			capOut += e
		} else {
			capOut += keep
		}
	}
	out := make([]uint64, capOut+1)
	off := make([]uint64, n+1)
	if C.dgx_list_uids_unfiltered_rows(s.crefs, C.size_t(n), s.uids, s.flags, s.off, C.uint64_t(afterUID), C.int32_t(first),
		(*C.uint64_t)(unsafe.Pointer(&out[0])), (*C.uint64_t)(unsafe.Pointer(&off[0])), C.size_t(capOut)) != C.DGX_OK {
		return nil, false
	}
	rows := make([]*pb.List, n)
	for i := range refs {
		rows[i] = &pb.List{}
		if off[i+1] > off[i] {
			rows[i].Uids = out[off[i]:off[i+1]:off[i+1]]
		}
	}
	return rows, true
}

// ListCountRows is countForUidPostings with a nil facets tree (worker/task.go:743-755) for every key of a task in ONE
// library call: the DoCount branch of handleUidPostings (:866-876), the REF postings List.Postings yields above
// afterUID.  Arguments as in ListUidsUnfilteredRows.  Returns false when the caller must keep the count loop.
func ListCountRows(refs []PackRef, muts []MutRow, afterUID uint64) ([]uint32, bool) {
	n := len(refs)
	if n == 0 {
		return []uint32{}, true
	}
	s, ok := stageUnfiltered(refs, muts)
	if !ok {
		return nil, false
	}
	defer s.free()
	counts := make([]uint32, n)
	if C.dgx_list_count_rows(s.crefs, C.size_t(n), s.uids, s.flags, s.off, C.uint64_t(afterUID),
		(*C.uint32_t)(unsafe.Pointer(&counts[0]))) != C.DGX_OK {
		return nil, false
	}
	return counts, true
}
