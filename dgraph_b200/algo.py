"""Host-side mirror of dgraph's `algo` package over libdgx (sm_90a CUDA).

Same function names, argument meaning and result shapes as
/root/reference/algo/uidlist.go; every body is one C-ABI call into libdgx.so
(include/dgx.h), exactly what the cgo shim in INTEGRATION.md does.  No set
arithmetic happens in Python and there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import numpy as np

from . import _lib
from .pb import List, _u64


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def _ptr_table(arrs: Sequence[np.ndarray]):
    k = len(arrs)
    ptrs = (C.c_void_p * max(k, 1))(*[a.ctypes.data if a.size else None for a in arrs])
    lens = (C.c_size_t * max(k, 1))(*[a.size for a in arrs])
    return ptrs, lens


def IntersectWith(u: List, v: List, o: List) -> None:
    """algo.IntersectWith(u, v, o) (algo/uidlist.go:142-167): o.Uids = u ∩ v.

    `o` may be `u` (in place).  When o.Uids has room the result is written into
    it (the reference reuses o.Uids[:0]); v is never modified.
    """
    lib = _lib.load()
    uu = np.zeros(0, np.uint64) if u.Uids is None else u.Uids
    vv = np.zeros(0, np.uint64) if v.Uids is None else v.Uids
    cap = min(uu.size, vv.size)
    if o.Uids is not None and o.Uids.size >= cap and o.Uids.flags.writeable:
        out = o.Uids  # dst := o.Uids[:0]
    else:
        out = np.empty(max(cap, 1), dtype=np.uint64)  # make([]uint64, 0, n)
    n = C.c_size_t(0)
    _lib.check(lib.dgx_intersect2(_p(uu), uu.size, _p(vv), vv.size, _p(out), cap, C.byref(n)))
    o.Uids = out[: n.value]


def IntersectSorted(lists: Sequence[List]) -> List:
    """algo.IntersectSorted (algo/uidlist.go:297-329).  No lists -> &pb.List{} (nil Uids)."""
    if len(lists) == 0:
        return List(None)
    lib = _lib.load()
    arrs = [np.zeros(0, np.uint64) if l.Uids is None else l.Uids for l in lists]
    ptrs, lens = _ptr_table(arrs)
    cap = min(a.size for a in arrs)
    out = np.empty(max(cap, 1), dtype=np.uint64)
    n = C.c_size_t(0)
    _lib.check(lib.dgx_intersect_sorted(ptrs, lens, len(arrs), _p(out), cap, C.byref(n)))
    return List(out[: n.value])


def MergeSorted(lists: Sequence[List]) -> List:
    """algo.MergeSorted (algo/uidlist.go:448-542): sorted union, globally de-duplicated."""
    lib = _lib.load()
    arrs = [np.zeros(0, np.uint64) if (l is None or l.Uids is None) else l.Uids for l in lists]
    ptrs, lens = _ptr_table(arrs)
    cap = sum(a.size for a in arrs)
    out = np.empty(max(cap, 1), dtype=np.uint64)
    n = C.c_size_t(0)
    _lib.check(lib.dgx_merge_sorted(ptrs, lens, len(arrs), _p(out), cap, C.byref(n)))
    return List(out[: n.value])


def Difference(u: List, v: List) -> List:
    """algo.Difference (algo/uidlist.go:332-362): u \\ v; nil u or v -> empty non-nil list."""
    if u is None or v is None:
        return List(np.zeros(0, np.uint64))
    lib = _lib.load()
    uu = np.zeros(0, np.uint64) if u.Uids is None else u.Uids
    vv = np.zeros(0, np.uint64) if v.Uids is None else v.Uids
    out = np.empty(max(uu.size, 1), dtype=np.uint64)
    n = C.c_size_t(0)
    _lib.check(lib.dgx_difference(_p(uu), uu.size, _p(vv), vv.size, _p(out), uu.size, C.byref(n)))
    return List(out[: n.value])


def IntersectCompressedWith(pack, afterUID: int, v: List, o: List) -> None:
    """algo.IntersectCompressedWith(pack, afterUID, v, o) (algo/uidlist.go:33-61): o.Uids = v ∩ pack[>= afterUID].

    A nil pack leaves `o` untouched, like the reference (:34-36)."""
    if pack is None:
        return
    from .codec import view_of

    lib = _lib.load()
    vv = np.zeros(0, np.uint64) if v.Uids is None else v.Uids
    out = np.empty(max(vv.size, 1), dtype=np.uint64)
    n = C.c_size_t(0)
    pack = pack.normalized()
    view = view_of(pack)
    _lib.check(lib.dgx_intersect_compressed(C.byref(view), afterUID, _p(vv), vv.size, _p(out), vv.size, C.byref(n)))
    o.Uids = out[: n.value]


def IntersectBatch(a: np.ndarray, a_off: np.ndarray, b: np.ndarray, b_off: np.ndarray):
    """Batched independent IntersectWith in CSR form (dgx_intersect_batch).

    Returns (out, out_off): pair i's result is out[out_off[i]:out_off[i+1]].
    """
    lib = _lib.load()
    a, b = _u64(a), _u64(b)
    a_off, b_off = _u64(a_off), _u64(b_off)
    npairs = a_off.size - 1
    cap = int(np.minimum(np.diff(a_off.astype(np.int64)), np.diff(b_off.astype(np.int64))).sum()) if npairs > 0 else 0
    out = np.empty(max(cap, 1), dtype=np.uint64)
    out_off = np.zeros(npairs + 1, dtype=np.uint64)
    _lib.check(lib.dgx_intersect_batch(_p(a), _p(a_off), _p(b), _p(b_off), npairs, _p(out), _p(out_off), cap))
    return out[: int(out_off[-1])], out_off


def IntersectSortedPacks(packs, keys=None) -> List:
    """algo.IntersectSorted over lists held as UidPacks (dgx_intersect_sorted_packed): the packs cross
    PCIe compressed and are decoded on the device (codec.Decode(p, 0) for each, codec/codec.go:444).

    keys: optional [(key, version)] naming each pack for the HBM-resident cache (0 = anonymous)."""
    if len(packs) == 0:
        return List(None)
    lib = _lib.load()
    refs, keep = _refs_of(packs, keys)
    cap = min(_exact(p) for p in packs)
    out = np.empty(max(cap, 1), dtype=np.uint64)
    n = C.c_size_t(0)
    _lib.check(lib.dgx_intersect_sorted_packed(refs, len(packs), _p(out), cap, C.byref(n)))
    return List(out[: n.value])


def IndexOfBatch(u: List, uids) -> np.ndarray:
    """algo.IndexOf(u, uid) for every uid (algo/uidlist.go:546-552): int64 positions, -1 when absent."""
    lib = _lib.load()
    uu = np.zeros(0, np.uint64) if u.Uids is None else u.Uids
    q = _u64(uids)
    idx = np.empty(max(q.size, 1), dtype=np.int64)
    _lib.check(lib.dgx_index_of_batch(_p(uu), uu.size, _p(q), q.size, idx.ctypes.data_as(C.c_void_p)))
    return idx[: q.size]


def IntersectBatchShared(a: np.ndarray, a_off: np.ndarray, b: np.ndarray):
    """Rows a[a_off[i]:a_off[i+1]] each intersected with the one list b (dgx_intersect_batch_shared):
    the `algo.IntersectWith(l, sg.DestUIDs, l)` loop of query/query.go:1425-1438."""
    lib = _lib.load()
    a, b, a_off = _u64(a), _u64(b), _u64(a_off)
    npairs = a_off.size - 1
    cap = int(np.minimum(np.diff(a_off.astype(np.int64)), b.size).sum()) if npairs > 0 else 0
    out = np.empty(max(cap, 1), dtype=np.uint64)
    out_off = np.zeros(npairs + 1, dtype=np.uint64)
    _lib.check(lib.dgx_intersect_batch_shared(_p(a), _p(a_off), npairs, _p(b), b.size, _p(out), _p(out_off), cap))
    return out[: int(out_off[-1])], out_off


def _refs_of(packs, keys=None):
    from .codec import view_of

    k = len(packs)
    refs = (_lib.PackRef * max(k, 1))()
    keep = []
    for i, p in enumerate(packs):
        if p is None or p.nblocks == 0:
            refs[i].pack = None
        else:
            p = p.normalized()
            v = view_of(p)
            keep.append((p, v))
            refs[i].pack = C.pointer(v)
        refs[i].key, refs[i].version = (keys[i] if keys is not None else (0, 0))
    return refs, keep


def IntersectCompressedWithRows(packs, afterUID: int, v, keys=None):
    """algo.IntersectCompressedWith(packs[i], afterUID, v, o_i) for every i in ONE call
    (dgx_intersect_compressed_rows): the handleUidPostings loop (worker/task.go:783-987) over a task's keys.

    v: ascending, duplicate-free uids (a pb.List or an array).  keys: optional [(key, version)] naming each pack for
    the HBM-resident cache (0 = anonymous).  A nil / empty pack gives an empty row.  Returns (out, out_off):
    row i is out[out_off[i]:out_off[i+1]]."""
    vv = v.Uids if isinstance(v, List) else v
    vv = np.zeros(0, np.uint64) if vv is None else _u64(vv)
    nrows = len(packs)
    if nrows == 0:
        return np.zeros(0, np.uint64), np.zeros(1, np.uint64)
    lib = _lib.load()
    refs, keep = _refs_of(packs, keys)
    cap = sum(min(vv.size, _exact(p)) for p in packs if p is not None)
    out = np.empty(max(cap, 1), dtype=np.uint64)
    out_off = np.zeros(nrows + 1, dtype=np.uint64)
    _lib.check(lib.dgx_intersect_compressed_rows(refs, nrows, afterUID, _p(vv), vv.size, _p(out), _p(out_off), cap))
    return out[: int(out_off[-1])], out_off


UIDS_COMPRESSED, UIDS_PROBE, UIDS_ITERATE = 0, 1, 2  # List.Uids branch of a row (include/dgx.h DGX_UIDS_*)
MUT_DEL, MUT_VALUE = 1, 2                             # flags of a resolved mutable entry (DGX_MUT_*)


def _mut_csr(muts):
    """The resolved mutable layers of a task's rows as one CSR: (uids, flags, off), never empty arrays."""
    mu = [np.zeros(0, np.uint64) if t is None else _u64(t[0]) for t in muts]
    mf = [np.zeros(0, np.uint8) if t is None else np.ascontiguousarray(np.asarray(t[1], np.uint8)) for t in muts]
    off = np.zeros(len(muts) + 1, dtype=np.uint64)
    np.cumsum([a.size for a in mu], out=off[1:])
    n = int(off[-1])
    return (np.concatenate(mu) if n else np.zeros(1, np.uint64)), (np.concatenate(mf) if n else np.zeros(1, np.uint8)), off


def ListUidsRows(packs, modes, muts, afterUID: int, v, keys=None):
    """posting.List.Uids(opts) for every key of a task in ONE call (dgx_list_uids_rows), mutable layers included: the
    handleUidPostings loop (worker/task.go:783-987) of a filtered read of unsplit lists.

    packs[i]: the immutable layer (None for an empty one, or for a delete-all marker).  modes[i]: the branch of List.Uids
    row i takes (UIDS_COMPRESSED / UIDS_PROBE / UIDS_ITERATE).  muts[i]: None or (uids, flags), the resolved mutable
    entries of row i, strictly ascending, flags MUT_DEL / MUT_VALUE.  v: opts.Intersect, ascending and non-empty.
    keys: optional [(key, version)] naming each pack for the HBM-resident cache.  Returns (out, out_off): row i is
    out[out_off[i]:out_off[i+1]]."""
    vv = v.Uids if isinstance(v, List) else v
    vv = np.zeros(0, np.uint64) if vv is None else _u64(vv)
    nrows = len(packs)
    if nrows == 0:
        return np.zeros(0, np.uint64), np.zeros(1, np.uint64)
    mode = np.ascontiguousarray(np.asarray(modes, dtype=np.uint8))
    mut_uids, mut_flags, mut_off = _mut_csr(muts)
    lib = _lib.load()
    refs, keep = _refs_of(packs, keys)
    cap = sum(min(vv.size, (_exact(p) if p is not None else 0) + int(mut_off[i + 1] - mut_off[i]))
              for i, p in enumerate(packs))
    out = np.empty(max(cap, 1), dtype=np.uint64)
    out_off = np.zeros(nrows + 1, dtype=np.uint64)
    _lib.check(lib.dgx_list_uids_rows(refs, _p(mode), nrows, _p(mut_uids), _p(mut_flags), _p(mut_off), afterUID,
                                      _p(vv), vv.size, _p(out), _p(out_off), cap))
    return out[: int(out_off[-1])], out_off


def ListUidsUnfilteredRows(packs, muts, afterUID: int, first: int = 0, keys=None):
    """posting.List.Uids(opts) with opts.Intersect == nil for every key of a task in ONE call
    (dgx_list_uids_unfiltered_rows): the handleUidPostings loop (worker/task.go:783-987) of a plain edge traversal over
    unsplit lists, mutable layers included.

    packs[i]: the immutable layer (None for an empty one, or for a delete-all marker).  muts[i]: None or (uids, flags),
    the resolved mutable entries of row i, strictly ascending, flags MUT_DEL / MUT_VALUE.  first: opts.First as an
    int32 (0 is MaxInt32; a negative value keeps at most one uid).  keys: optional [(key, version)] naming each pack for
    the HBM-resident cache.  Returns (out, out_off): row i is out[out_off[i]:out_off[i+1]]."""
    nrows = len(packs)
    if nrows == 0:
        return np.zeros(0, np.uint64), np.zeros(1, np.uint64)
    mut_uids, mut_flags, mut_off = _mut_csr(muts)
    lib = _lib.load()
    refs, keep = _refs_of(packs, keys)
    most = 0x7FFFFFFF if first == 0 else (1 if first < 0 else first)
    cap = sum(min(most, (_exact(p) if p is not None else 0) + int(mut_off[i + 1] - mut_off[i]))
              for i, p in enumerate(packs))
    out = np.empty(max(cap, 1), dtype=np.uint64)
    out_off = np.zeros(nrows + 1, dtype=np.uint64)
    _lib.check(lib.dgx_list_uids_unfiltered_rows(refs, nrows, _p(mut_uids), _p(mut_flags), _p(mut_off), afterUID, first,
                                                 _p(out), _p(out_off), cap))
    return out[: int(out_off[-1])], out_off


def ListCountRows(packs, muts, afterUID: int, keys=None):
    """countForUidPostings with a nil facets tree (worker/task.go:743-755, 866-876) for every key of a task in ONE call
    (dgx_list_count_rows): the REF postings List.Postings yields above afterUID, mutable layers included.  Arguments as
    in ListUidsUnfilteredRows.  Returns a uint32 array of counts."""
    nrows = len(packs)
    counts = np.zeros(nrows, dtype=np.uint32)
    if nrows == 0:
        return counts
    mut_uids, mut_flags, mut_off = _mut_csr(muts)
    refs, keep = _refs_of(packs, keys)
    _lib.check(_lib.load().dgx_list_count_rows(refs, nrows, _p(mut_uids), _p(mut_flags), _p(mut_off), afterUID,
                                               _p(counts)))
    return counts


def IntersectCompressedWithMatrix(pack, rows, key=None):
    """algo.IntersectCompressedWith(pack, 0, rows[i], o_i) for every row i in ONE call
    (dgx_intersect_compressed_matrix): the intersectBucket loop (worker/sort.go:605-700) of one index bucket over a
    uid matrix.

    rows: strictly ascending uid lists (pb.List values or arrays).  key: optional (key, version) naming the pack for the
    HBM-resident cache.  A nil / empty pack gives empty rows.  Returns (out, out_off): row i is
    out[out_off[i]:out_off[i+1]]."""
    arrs = []
    for r in rows:
        u = r.Uids if isinstance(r, List) else r
        arrs.append(np.zeros(0, np.uint64) if u is None else _u64(u))
    nrows = len(arrs)
    out_off = np.zeros(nrows + 1, dtype=np.uint64)
    if nrows == 0:
        return np.zeros(0, np.uint64), out_off
    v_off = np.zeros(nrows + 1, dtype=np.uint64)
    np.cumsum([a.size for a in arrs], out=v_off[1:])
    v = np.concatenate(arrs) if int(v_off[-1]) else np.zeros(1, np.uint64)
    lib = _lib.load()
    refs, keep = _refs_of([pack], [key] if key is not None else None)
    exact = _exact(pack)
    cap = sum(min(a.size, exact) for a in arrs)
    out = np.empty(max(cap, 1), dtype=np.uint64)
    _lib.check(lib.dgx_intersect_compressed_matrix(refs, _p(v), _p(v_off), nrows, _p(out), _p(out_off), cap))
    return out[: int(out_off[-1])], out_off


def MergeSortedMatrix(rows) -> List:
    """algo.MergeSorted(rows) over the rows of a uid matrix in ONE call (dgx_merge_sorted_matrix):
    sg.DestUIDs = algo.MergeSorted(result.UidMatrix) (query/query.go:2290).

    rows: ascending uid lists (pb.List values or arrays); duplicates inside and across rows are removed.  The rows
    cross PCIe as one CSR copy, and the launch count does not depend on the number of rows."""
    arrs = []
    for r in rows:
        u = r.Uids if isinstance(r, List) else r
        arrs.append(np.zeros(0, np.uint64) if u is None else _u64(u))
    nrows = len(arrs)
    v_off = np.zeros(nrows + 1, dtype=np.uint64)
    if nrows:
        np.cumsum([a.size for a in arrs], out=v_off[1:])
    m = int(v_off[-1])
    v = np.concatenate(arrs) if m else np.zeros(1, np.uint64)
    out = np.empty(max(m, 1), dtype=np.uint64)
    n = C.c_size_t(0)
    _lib.check(_lib.load().dgx_merge_sorted_matrix(_p(v), _p(v_off), nrows, _p(out), m, C.byref(n)))
    return List(out[: n.value])


def _exact(p) -> int:
    from .codec import ExactLen

    return ExactLen(p)


def IntersectWithLinPacked(u, v, blockSize: int = 256):
    """algo.IntersectWithLinPacked(u, v *pb.UidPack) *pb.UidPack (algo/packed.go:35-101): result as a pack."""
    from .codec import _call_pack_out

    lib = _lib.load()
    refs, keep = _refs_of([u, v])
    return _call_pack_out(lambda b, n, d, dl, pnb, pdb, pv: lib.dgx_intersect_packed(
        C.byref(refs[0]), C.byref(refs[1]), blockSize, b, n, d, dl, pnb, pdb, pv), min(_exact(u), _exact(v)), blockSize)


def DifferencePacked(u, v, blockSize: int = 256):
    """algo.DifferencePacked(u, v) (algo/packed.go:141-226): u \\ v as a pack."""
    from .codec import _call_pack_out

    lib = _lib.load()
    refs, keep = _refs_of([u, v])
    return _call_pack_out(lambda b, n, d, dl, pnb, pdb, pv: lib.dgx_difference_packed(
        C.byref(refs[0]), C.byref(refs[1]), blockSize, b, n, d, dl, pnb, pdb, pv), _exact(u), blockSize)


def MergeSortedPacked(lists, blockSize: int = 256):
    """algo.MergeSortedPacked(lists) (algo/packed.go:228-297): sorted de-duplicated union as a pack."""
    from .codec import _call_pack_out

    lib = _lib.load()
    refs, keep = _refs_of(lists)
    return _call_pack_out(lambda b, n, d, dl, pnb, pdb, pv: lib.dgx_merge_sorted_packed(
        refs, len(lists), blockSize, b, n, d, dl, pnb, pdb, pv), sum(_exact(p) for p in lists), blockSize)


def IntersectSortedPacked(lists, blockSize: int = 256):
    """algo.IntersectSortedPacked(lists) (algo/packed.go:103-139) over ALL lists (the reference's loop keeps only
    ls[0] ∩ ls[1], see DESIGN section 5); no lists -> nil pack."""
    from .codec import _call_pack_out

    if len(lists) == 0:
        return None
    lib = _lib.load()
    refs, keep = _refs_of(lists)
    return _call_pack_out(lambda b, n, d, dl, pnb, pdb, pv: lib.dgx_intersect_sorted_packed_out(
        refs, len(lists), blockSize, b, n, d, dl, pnb, pdb, pv), min(_exact(p) for p in lists), blockSize)
