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


QAND, QOR = 2, 3  # cindex.Query ops of a trigram query node (include/dgx.h DGX_QAND / DGX_QOR)


def query_tree(tree):
    """A cindex.Query tree as the CSR arrays of dgx_query_tree: (tree struct, the arrays it points at).  tree[i] is
    (op, leaf indices, sub-node indices); node 0 is the root."""
    n = len(tree)
    op = np.array([t[0] for t in tree] or [0], dtype=np.uint8)
    leaf_off, sub_off = np.zeros(n + 1, np.uint32), np.zeros(n + 1, np.uint32)
    np.cumsum([len(t[1]) for t in tree], out=leaf_off[1:])
    np.cumsum([len(t[2]) for t in tree], out=sub_off[1:])
    leaf_idx = np.array([i for t in tree for i in t[1]] or [0], dtype=np.uint32)
    sub_idx = np.array([i for t in tree for i in t[2]] or [0], dtype=np.uint32)
    arrays = (op, leaf_off, leaf_idx, sub_off, sub_idx)
    return _lib.QueryTree(n, *[a.ctypes.data for a in arrays]), arrays


def query_bound(tree, leaf_bounds) -> int:
    """The root's bound of a trigram query (the out_cap dgx_trigram_query needs): a leaf's is ExactLen + |mut| or its
    length, an AND's the minimum of its children's, an OR's their sum."""
    b = [0] * len(tree)
    for i in reversed(range(len(tree))):
        op, leaves, subs = tree[i]
        ch = [leaf_bounds[j] for j in leaves] + [b[s] for s in subs]
        b[i] = min(ch) if op == QAND and ch else sum(ch)
    return b[0] if tree else 0


def UidsForRegex(tree, leaves, afterUID: int, keys=None) -> List:
    """uidsForRegex(attr, arg, query, &pb.List{}) (worker/trigram.go:24-102) over a regexp()'s trigram query tree in ONE
    call (dgx_trigram_query): every trigram's List.Uids read, the ANDs and ORs, on the device.

    tree[i]: (op, leaf indices, sub-node indices) with op QAND / QOR; node 0 is the root, every other node has one
    parent and a larger index.  leaves[j]: a pack leaf (pack, mut) -- pack None for an empty list or a delete-all
    marker, mut None or (uids, flags), the resolved layer of REF postings as in ListUidsUnfilteredRows -- or a list leaf,
    an ascending duplicate-free array (or pb.List) the caller decoded itself.  keys: optional [(key, version)] per leaf
    naming the pack leaves for the HBM-resident cache.  Returns the root's uids."""
    pack_ids = [j for j, lf in enumerate(leaves) if isinstance(lf, tuple)]
    list_ids = [j for j, lf in enumerate(leaves) if not isinstance(lf, tuple)]
    order = {j: k for k, j in enumerate(pack_ids + list_ids)}  # the ABI numbers pack leaves first
    tr = [(op, [order[j] for j in ls], list(subs)) for op, ls, subs in tree]
    packs = [leaves[j][0] for j in pack_ids]
    mut_uids, mut_flags, mut_off = _mut_csr([leaves[j][1] for j in pack_ids])
    arrs = []
    for j in list_ids:
        u = leaves[j].Uids if isinstance(leaves[j], List) else leaves[j]
        arrs.append(np.zeros(0, np.uint64) if u is None else _u64(u))
    list_off = np.zeros(len(arrs) + 1, dtype=np.uint64)
    np.cumsum([a.size for a in arrs], out=list_off[1:])
    lists = np.concatenate(arrs) if int(list_off[-1]) else np.zeros(1, np.uint64)
    bounds = [(_exact(p) if p is not None else 0) + int(mut_off[k + 1] - mut_off[k]) for k, p in enumerate(packs)]
    cap = query_bound(tr, bounds + [a.size for a in arrs])
    refs, keep = _refs_of(packs, [keys[j] for j in pack_ids] if keys is not None else None)
    qt, qa = query_tree(tr)
    out = np.empty(max(cap, 1), dtype=np.uint64)
    n = C.c_size_t(0)
    _lib.check(_lib.load().dgx_trigram_query(C.byref(qt), refs, len(packs), _p(mut_uids), _p(mut_flags), _p(mut_off),
                                             _p(lists), _p(list_off), len(arrs), afterUID, _p(out), cap, C.byref(n)))
    return List(out[: n.value])


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


def _csr_u64(rows):
    arrs = []
    for r in rows:
        u = r.Uids if isinstance(r, List) else r
        arrs.append(np.zeros(0, np.uint64) if u is None else _u64(u))
    off = np.zeros(len(arrs) + 1, dtype=np.uint64)
    np.cumsum([a.size for a in arrs], out=off[1:])
    flat = np.concatenate(arrs) if int(off[-1]) else np.zeros(1, np.uint64)
    return flat, off


def GroupByUid(parents, src, rows, dest, members: bool = True):
    """@groupby over one uid predicate (query/groupby.go formResult / formGroups / groupLess) for every parent row in
    ONE call (dgx_groupby_uid).

    parents: sg.uidMatrix, strictly ascending rows; src: child.SrcUIDs, strictly ascending; rows: child.uidMatrix,
    row i the values of src[i], strictly ascending; dest: child.DestUIDs, holding every value of every row.  A parent
    with one row equal to src gives fillGroupedVars' grouping.  Returns per parent (keys, counts, members): its groups
    ordered by (count, key), each group's key and count(uid), and members = (values, offsets) with each group's
    ascending source uids, or None when members is False (counts only: the members stay on the device)."""
    par, par_off = _csr_u64(parents)
    v, v_off = _csr_u64(rows)
    src_a = _u64(src.Uids if isinstance(src, List) else src)
    dest_a = _u64(dest.Uids if isinstance(dest, List) else dest)
    if src_a.size != len(rows):
        raise ValueError(f"{src_a.size} sources for {len(rows)} rows")
    lib = _lib.load()
    npar = len(parents)
    grp_off = np.zeros(npar + 1, dtype=np.uint64)
    ng, nm = C.c_size_t(0), C.c_size_t(0)
    gcap = mcap = int(v_off[-1])  # a single parent never has more; a larger call is sized again from the exact counts
    for _ in range(2):
        keys = np.empty(max(gcap, 1), dtype=np.uint64)
        mem_off = np.empty(gcap + 1, dtype=np.uint64)
        mem = np.empty(max(mcap, 1), dtype=np.uint64) if members else None
        rc = lib.dgx_groupby_uid(_p(src_a), src_a.size, _p(v), _p(v_off), _p(dest_a), dest_a.size, _p(par),
                                 _p(par_off), npar, _p(keys), _p(grp_off), _p(mem_off), gcap,
                                 _p(mem) if members else None, mcap, C.byref(ng), C.byref(nm))
        if rc != _lib.DGX_ERR_CAP:
            break
        gcap, mcap = ng.value, nm.value
    _lib.check(rc)
    out = []
    for p in range(npar):
        g0, g1 = int(grp_off[p]), int(grp_off[p + 1])
        off = mem_off[g0:g1 + 1] if g1 > g0 else np.zeros(1, np.uint64)
        counts = np.diff(off)
        m = (mem[int(off[0]):int(off[-1])].copy(), off - off[0]) if members else None
        out.append((keys[g0:g1].copy(), counts, m))
    return out


CC_CASCADE, CC_CHECKED, CC_FILTERED, CC_ORDERED, CC_SKIP = 1, 2, 4, 8, 16  # DGX_CASCADE_* (include/dgx.h)


class CascadeNode:
    """One subgraph node of a @cascade forest, in pre-order (dgx_cascade): parent index (-1 for a query root), CC_* flags
    resolved from the SubGraph, Params.Cascade.First / Offset, len(counts), DestUIDs (strictly ascending), uidMatrix
    rows (row i belongs to parent.DestUIDs[i]) and has_val (one byte per row: valueMatrix[i] has values)."""

    __slots__ = ("parent", "flags", "first", "offset", "counts_len", "dest", "rows", "has_val")

    def __init__(self, parent=-1, flags=0, first=0, offset=0, counts_len=0, dest=(), rows=(), has_val=()):
        self.parent, self.flags, self.first, self.offset, self.counts_len = parent, flags, first, offset, counts_len
        self.dest = _u64(dest.Uids if isinstance(dest, List) else dest)
        self.rows = [_u64(r.Uids if isinstance(r, List) else r) for r in rows]
        self.has_val = np.ascontiguousarray(np.asarray(has_val, np.uint8))


def cascade_arrays(nodes) -> dict:
    """The flat CSR form of dgx_cascade: tree arrays, values with per-row offsets and per-node row offsets, dest and
    has_val with per-node offsets.  Every array has at least one element."""
    n = len(nodes)

    def off(sizes):
        o = np.zeros(len(sizes) + 1, np.uint64)
        np.cumsum(sizes, out=o[1:])
        return o

    def cat(arrs, dt):
        arrs = [a for a in arrs if a.size]
        return np.ascontiguousarray(np.concatenate(arrs).astype(dt)) if arrs else np.zeros(1, dt)

    rows = [r for nd in nodes for r in nd.rows]
    a = {"parent": np.array([0xFFFFFFFF if nd.parent < 0 else nd.parent for nd in nodes] or [0], np.uint32),
         "flags": np.array([nd.flags for nd in nodes] or [0], np.uint8),
         "first": np.array([nd.first for nd in nodes] or [0], np.int32),
         "offset": np.array([nd.offset for nd in nodes] or [0], np.int32),
         "counts_len": np.array([nd.counts_len for nd in nodes] or [0], np.uint64),
         "v": cat(rows, np.uint64), "v_off": off([r.size for r in rows]),
         "row_off": off([len(nd.rows) for nd in nodes]),
         "dest": cat([nd.dest for nd in nodes], np.uint64), "dest_off": off([nd.dest.size for nd in nodes]),
         "has_val": cat([nd.has_val for nd in nodes], np.uint8), "hv_off": off([nd.has_val.size for nd in nodes])}
    a["nnodes"] = n
    return a


def cascade_split(a, out, out_off, dest_out, dest_out_off):
    """Per-node results of a flat call: ([rows of each node], [dest of each node])."""
    ro = a["row_off"]
    rows = [[out[int(out_off[r]):int(out_off[r + 1])].copy() for r in range(int(ro[k]), int(ro[k + 1]))]
            for k in range(a["nnodes"])]
    dests = [dest_out[int(dest_out_off[k]):int(dest_out_off[k + 1])].copy() for k in range(a["nnodes"])]
    return rows, dests


def cascade_tree(a) -> _lib.CascadeTree:
    """The dgx_cascade_tree over the tree arrays of cascade_arrays (which must outlive it)."""
    return _lib.CascadeTree(a["nnodes"], *[a[k].ctypes.data for k in ("parent", "flags", "first", "offset",
                                                                        "counts_len")])


def Cascade(nodes):
    """@cascade over a forest (query/query.go populateVarMap :1445-1527 and ProcessQuery's root pagination :3004-3011)
    in one call (dgx_cascade).  Returns ([rows of each node], [DestUIDs of each node as List]) after the cascade."""
    a = cascade_arrays(nodes)
    m, nd = int(a["v_off"][-1]), int(a["dest_off"][-1])
    out, dest_out = np.empty(max(m, 1), np.uint64), np.empty(max(nd, 1), np.uint64)
    out_off, dest_off = np.zeros(int(a["row_off"][-1]) + 1, np.uint64), np.zeros(len(nodes) + 1, np.uint64)
    tree = cascade_tree(a)
    _lib.check(_lib.load().dgx_cascade(C.byref(tree), _p(a["v"]), _p(a["v_off"]), _p(a["row_off"]), _p(a["dest"]),
                                       _p(a["dest_off"]), _p(a["has_val"]), _p(a["hv_off"]), _p(out), _p(out_off), m,
                                       _p(dest_out), _p(dest_off), nd))
    rows, dests = cascade_split(a, out, out_off, dest_out, dest_off)
    return rows, [List(d) for d in dests]


SGF_OPS = {"and": 1, "or": 2, "not": 3}   # DGX_SGF_AND / _OR / _NOT; DGX_SGF_LEAF is 0
SGF_CMP = {"le": 0, "ge": 1, "lt": 2, "gt": 3, "eq": 4}  # DGX_SGF_CMP_*


def sg_filter_flat(tree) -> dict:
    """The flat dgx_sg_filter_tree arrays of a nested filter tree: an int is a leaf index, ("and" | "or", [children])
    an op and ("not", child) a negation.  Nodes are numbered in pre-order, so node 0 is the root and every parent lies
    below its children."""
    op, parent, leaf = [], [], []

    def walk(t, p):
        k = len(op)
        parent.append(p)
        if isinstance(t, (int, np.integer)):
            op.append(0)
            leaf.append(int(t))
            return
        op.append(SGF_OPS[t[0]])
        leaf.append(0)
        for c in ([t[1]] if t[0] == "not" else t[1]):
            walk(c, k)

    walk(tree, 0xFFFFFFFF)
    return {"nnodes": len(op), "op": np.array(op, np.uint8), "parent": np.array(parent, np.uint32),
            "leaf": np.array(leaf, np.uint32)}


def sg_filter_tree(f) -> "_lib.SgFilterTree":
    """The dgx_sg_filter_tree over the arrays of sg_filter_flat (which must outlive it)."""
    return _lib.SgFilterTree(f["nnodes"], f["op"].ctypes.data, f["parent"].ctypes.data, f["leaf"].ctypes.data)


def sg_filter_leaf_arrays(leaves, n0: int):
    """Host arrays of the leaves: ("list", uids), ("count", cmp, threshold, counts) with one uint32 count per D0 value,
    or ("len", cmp, threshold, off) with D0's n0 + 1 row offsets.  Returns (kept arrays, dgx_sg_filter_leaf table).
    Raises ValueError when a COUNT leaf's array does not match n0: the library copies exactly that many entries."""
    keep, descs = [], []
    for lf in leaves:
        if lf[0] == "list":
            u = _u64(lf[1].Uids if isinstance(lf[1], List) else lf[1])
            keep.append(u)
            descs.append(_lib.SgFilterLeaf(0, 0, 0, u.ctypes.data if u.size else None, u.size, None, None, None))
        else:
            a = np.ascontiguousarray(np.asarray(lf[3], np.uint32 if lf[0] == "count" else np.uint64))
            want = n0 if lf[0] == "count" else n0 + 1
            if a.size != want:
                raise ValueError(f"a {lf[0]!r} leaf holds {a.size} entries for {n0} D0 values: {want} expected")
            if a.size == 0:
                a = np.zeros(1, a.dtype)
            keep.append(a)
            descs.append(_lib.SgFilterLeaf(1, SGF_CMP[lf[1]], int(lf[2]), None, 0, None,
                                           a.ctypes.data if lf[0] == "count" else None,
                                           a.ctypes.data if lf[0] == "len" else None))
    return keep, (_lib.SgFilterLeaf * max(len(descs), 1))(*descs)


def SubgraphFilter(tree, leaves, d0, rows, count: int = 0, offset: int = 0, counts_only: bool = False):
    """A subgraph's @filter and first / offset (query/query.go ProcessGraph's filter block, applyPagination and the
    DoCount block) in ONE call (dgx_sg_filter).

    tree: the filter tree as sg_filter_flat takes it; leaves: as sg_filter_leaf_arrays takes them; d0: DestUIDs from
    processTask; rows: the uid matrix (strictly ascending rows).  Returns (rows, counts, dest): the filtered and paged
    rows (None in counts-only mode), counts[i] = len(row i) and the new DestUIDs as a List."""
    f = sg_filter_flat(tree)
    d0a = _u64(d0.Uids if isinstance(d0, List) else d0)
    keep, tab = sg_filter_leaf_arrays(leaves, d0a.size)
    v, v_off = _csr_u64(rows)
    nrows, m = len(rows), int(v_off[-1])
    dest = np.empty(max(d0a.size, 1), np.uint64)
    out = None if counts_only else np.empty(max(m, 1), np.uint64)
    out_off = np.zeros(nrows + 1, np.uint64)
    counts = np.zeros(max(nrows, 1), np.uint32)
    n = C.c_size_t(0)
    t = sg_filter_tree(f)
    _lib.check(_lib.load().dgx_sg_filter(C.byref(t), tab, len(leaves), _p(d0a), d0a.size, _p(v), _p(v_off), nrows,
                                         count, offset, _p(dest), d0a.size, C.byref(n),
                                         None if counts_only else _p(out), _p(out_off), m, _p(counts)))
    res = None if counts_only else [out[int(out_off[i]):int(out_off[i + 1])].copy() for i in range(nrows)]
    return res, counts[:nrows].copy(), List(dest[: n.value].copy())


class ReachSet:
    """The edges one sg.Attr has taken during one @recurse (query/recurse.go expandRecurse's reachMap, loop: false),
    kept in device memory (dgx_reach_set).  One set per distinct Attr, for the life of one recursion."""

    def __init__(self):
        self._set = None
        self._open(np.zeros(1, np.uint64), np.zeros(1, np.uint64), 0)

    def _open(self, f, t, n):
        h = C.c_void_p()
        _lib.check(_lib.load().dgx_reach_create(_p(f), _p(t), n, C.byref(h)))
        self._set = h

    @classmethod
    def from_edges(cls, frm, to) -> "ReachSet":
        """A set holding the edges (frm[k], to[k]), strictly ascending by (from, to): how a recursion started on the
        host continues on the device."""
        f, t = _u64(frm), _u64(to)
        if f.size != t.size:
            raise ValueError(f"{f.size} from values for {t.size} to values")
        s = cls.__new__(cls)
        s._set = None
        s._open(f if f.size else np.zeros(1, np.uint64), t if t.size else np.zeros(1, np.uint64), f.size)
        return s

    @property
    def handle(self):
        """The dgx_reach_set pointer, for dgx_dev_recurse_filter."""
        if self._set is None:
            raise ValueError("ReachSet is closed")
        return self._set

    def filter(self, src, rows, dest=None):
        """One sg of one level (:105-134): rows[i] (strictly ascending) belongs to src[i] (strictly ascending).  dest
        (sg.DestUIDs after its filters) or None when the sg has no filters.  Returns (kept rows, DestUIDs, kept), and
        the kept edges join the set."""
        v, v_off = _csr_u64(rows)
        src_a = _u64(src.Uids if isinstance(src, List) else src)
        if src_a.size != len(rows):
            raise ValueError(f"{src_a.size} sources for {len(rows)} rows")
        d = None if dest is None else _u64(dest.Uids if isinstance(dest, List) else dest)
        m = int(v_off[-1])
        out, dest_out = np.empty(max(m, 1), np.uint64), np.empty(max(m, 1), np.uint64)
        out_off = np.zeros(len(rows) + 1, np.uint64)
        n = C.c_size_t(0)
        if src_a.size == 0:
            src_a = np.zeros(1, np.uint64)
        if d is not None and d.size == 0:
            d = np.zeros(1, np.uint64)
        nd = 0 if dest is None else int(np.size(dest.Uids if isinstance(dest, List) else dest))
        _lib.check(_lib.load().dgx_recurse_filter(self.handle, _p(src_a), len(rows), _p(v), _p(v_off),
                                                  None if d is None else _p(d), nd, _p(out), _p(out_off), m,
                                                  _p(dest_out), m, C.byref(n)))
        kept = [out[int(out_off[i]):int(out_off[i + 1])].copy() for i in range(len(rows))]
        return kept, List(dest_out[: n.value].copy()), int(out_off[-1])

    def size(self) -> int:
        n = C.c_size_t(0)
        _lib.check(_lib.load().dgx_reach_size(self.handle, C.byref(n)))
        return n.value

    def export(self):
        """(from, to) of every edge, ascending: how a recursion hands back to the host."""
        n = self.size()
        f, t = np.empty(max(n, 1), np.uint64), np.empty(max(n, 1), np.uint64)
        got = C.c_size_t(0)
        _lib.check(_lib.load().dgx_reach_export(self.handle, _p(f), _p(t), n, C.byref(got)))
        return f[: got.value].copy(), t[: got.value].copy()

    def close(self) -> None:
        if self._set is not None:
            _lib.load().dgx_reach_destroy(self._set)
            self._set = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def path_level_arrays(sgs):
    """One shortest-path level as the CSR arrays of dgx_path_level: sgs is a list of (attr, src, rows, dest) in exec
    order, rows[i] the values of src[i].  Returns (attr u32, src_off, src, v_off, v, dest_off, dest); empty arrays hold
    one element so that every pointer is valid."""
    attr = np.asarray([int(a) for a, _, _, _ in sgs], np.uint32)
    srcs = [_u64(s.Uids if isinstance(s, List) else s) for _, s, _, _ in sgs]
    rows = [r for _, _, rs, _ in sgs for r in rs]
    for (_, _, rs, _), s in zip(sgs, srcs):
        if len(rs) != s.size:
            raise ValueError(f"{s.size} sources for {len(rs)} rows")
    src, src_off = _csr_u64(srcs)
    v, v_off = _csr_u64(rows)
    dest, dest_off = _csr_u64([d.Uids if isinstance(d, List) else d for _, _, _, d in sgs])
    return (attr if attr.size else np.zeros(1, np.uint32)), src_off, src, v_off, v, dest_off, dest


def path_level(arrays, nsg: int) -> "_lib.PathLevel":
    """The dgx_path_level over path_level_arrays' arrays (host) or over device tensors of the same layout."""
    ptr = [a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr() for a in arrays]
    return _lib.PathLevel(nsg, *ptr)


class PathSearch:
    """shortest() with numpaths <= 1 and no facets (query/shortest.go expandOut + shortestPath at unit cost): a
    breadth-first search from `frm` to `to` held in device memory (dgx_path_search), one expand() per level."""

    def __init__(self, frm: int, to: int):
        self._ps = None
        h = C.c_void_p()
        _lib.check(_lib.load().dgx_path_create(int(frm), int(to), C.byref(h)))
        self._ps = h

    @property
    def handle(self):
        """The dgx_path_search pointer, for dgx_dev_path_expand."""
        if self._ps is None:
            raise ValueError("PathSearch is closed")
        return self._ps

    def expand(self, sgs):
        """One level: sgs is a list of (attr, src, rows, dest) in exec order (attr the child index, rows[i] the values
        of src[i], dest the sg's DestUIDs).  Returns (next SrcUIDs per sg, (edges, discovered, to_level))."""
        if not sgs:
            raise ValueError("a level has at least one sg")
        arrs = path_level_arrays(sgs)
        lv = path_level(arrs, len(sgs))
        d = int(arrs[5][-1])
        nxt, nxt_off = np.empty(max(d, 1), np.uint64), np.zeros(len(sgs) + 1, np.uint64)
        st = _lib.PathStats()
        _lib.check(_lib.load().dgx_path_expand(self.handle, C.byref(lv), _p(nxt), _p(nxt_off), d, C.byref(st)))
        nexts = [nxt[int(nxt_off[i]):int(nxt_off[i + 1])].copy() for i in range(len(sgs))]
        return nexts, (st.edges, st.discovered, st.to_level)

    def path(self):
        """(uids From .. To, attr index of each hop), both empty when To was not reached."""
        n = C.c_size_t(0)
        lib = _lib.load()
        rc = lib.dgx_path_result(self.handle, None, None, 0, C.byref(n))
        if rc != _lib.DGX_OK and n.value == 0:
            _lib.check(rc)
        uids, attrs = np.empty(max(n.value, 1), np.uint64), np.empty(max(n.value, 1), np.uint32)
        _lib.check(lib.dgx_path_result(self.handle, _p(uids), _p(attrs), n.value, C.byref(n)))
        return uids[: n.value].copy(), attrs[: max(n.value - 1, 0)].copy()

    def close(self) -> None:
        if self._ps is not None:
            _lib.load().dgx_path_destroy(self._ps)
            self._ps = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


VAL_INT64, VAL_FLOAT64 = 1, 2  # DGX_VAL_* (include/dgx.h)
AGG = {"min": 0, "max": 1, "sum": 2, "avg": 3}  # DGX_AGG_*


def _val_map(keys, vals):
    """(type, keys u64, values as u64 words) of a value map: int64 values are DGX_VAL_INT64, float64 DGX_VAL_FLOAT64."""
    v = np.asarray(vals)
    if v.dtype == np.int64:
        typ = VAL_INT64
    elif v.dtype == np.float64:
        typ = VAL_FLOAT64
    else:
        raise TypeError(f"a value map holds int64 or float64 values, not {v.dtype}")
    k = _u64(keys.Uids if isinstance(keys, List) else keys)
    if k.size != v.size:
        raise ValueError(f"{k.size} keys for {v.size} values")
    w = np.ascontiguousarray(v).view(np.uint64)
    return typ, (k if k.size else np.zeros(1, np.uint64)), (w if w.size else np.zeros(1, np.uint64)), k.size


def _val_out(typ, key, val, n):
    return key[:n].copy(), val[:n].view(np.float64 if typ == VAL_FLOAT64 else np.int64).copy()


def var_level_arrays(src, rows, dest):
    """One level of a value variable's path as host arrays (src, v_off, v, dest), each holding at least one value,
    and its ndest."""
    s = _u64(src.Uids if isinstance(src, List) else src)
    if s.size != len(rows):
        raise ValueError(f"{s.size} sources for {len(rows)} rows")
    v, v_off = _csr_u64(rows)
    d = _u64(dest.Uids if isinstance(dest, List) else dest)
    return (s if s.size else np.zeros(1, np.uint64)), v_off, v, (d if d.size else np.zeros(1, np.uint64)), d.size


def PropagateVar(keys, vals, levels):
    """transformTo (query/query.go :1143-1236) over a whole path in ONE call (dgx_var_propagate).

    keys: the map's uids, strictly ascending; vals: int64 or float64 values (the map's type).  levels: the path's nodes
    from len(fromNode.path) on, index 0 skipped, each (SrcUIDs, uidMatrix rows, DestUIDs).  Returns the map at the last
    level as (keys, values of the same dtype)."""
    if not levels:
        raise ValueError("a path has at least one level")
    typ, k, w, n = _val_map(keys, vals)
    arrs = [var_level_arrays(*lv) for lv in levels]
    lv = (_lib.VarLevel * len(arrs))()
    for i, (s, o, v, d, nd) in enumerate(arrs):
        lv[i] = _lib.VarLevel(s.ctypes.data, o.ctypes.data, v.ctypes.data, d.ctypes.data, o.size - 1, int(o[-1]), nd)
    cap = arrs[-1][4]
    ok, ov = np.empty(max(cap, 1), np.uint64), np.empty(max(cap, 1), np.uint64)
    m = C.c_size_t(0)
    _lib.check(_lib.load().dgx_var_propagate(typ, _p(k), _p(w), n, lv, len(arrs), _p(ok), _p(ov), cap, C.byref(m)))
    return _val_out(typ, ok, ov, m.value)


def LevelAgg(fn: str, keys, vals, src, rows):
    """evalLevelAgg's per-row branch (query/query.go :1088-1123) in ONE call (dgx_var_level_agg): fn one of min, max,
    sum, avg over the map (keys, int64 or float64 vals) for every row of relSG's uid matrix (rows[i] the values of
    src[i]).  Returns (keys, values): float64 for avg, the map's dtype otherwise."""
    if fn not in AGG:
        raise ValueError(f"unknown aggregation {fn!r}")
    typ, k, w, n = _val_map(keys, vals)
    s, v_off, v, _, _ = var_level_arrays(src, rows, ())
    nrows = v_off.size - 1
    ok, ov = np.empty(max(nrows, 1), np.uint64), np.empty(max(nrows, 1), np.uint64)
    m = C.c_size_t(0)
    _lib.check(_lib.load().dgx_var_level_agg(typ, AGG[fn], _p(k), _p(w), n, _p(s), nrows, _p(v_off), _p(v), _p(ok),
                                             _p(ov), nrows, C.byref(m)))
    return _val_out(VAL_FLOAT64 if fn == "avg" else typ, ok, ov, m.value)


VAL_BOOL, VAL_NIL = 3, 4  # DGX_VAL_* of math() entries
MATH_OPS = {"const": 0, "var": 1, "+": 2, "-": 3, "*": 4, "/": 5, "%": 6, "min": 7, "max": 8, "u-": 9, "sqrt": 10,
            "floor": 11, "ceil": 12, "<": 13, ">": 14, "<=": 15, ">=": 16, "==": 17, "!=": 18, "cond": 19}
MATH_KIND = {0: "none", 1: "map", 2: "const"}  # DGX_MATH_KIND_*


def math_program(tree, names):
    """A math() tree as a post-order list of _lib.MathNode.  tree: ("var", name), ("const", int or float) or
    (op, child, ...) with op a key of MATH_OPS; names: leaf index of each variable name, filled in first-use order."""
    nodes = []

    def walk(t):
        op = t[0]
        if op not in MATH_OPS:
            raise ValueError(f"unknown math op {op!r}")
        kids = [walk(c) for c in t[1:]] if op not in ("var", "const") else []
        n = _lib.MathNode()
        n.op = MATH_OPS[op]
        for i, c in enumerate(kids):
            n.child[i] = c
        if op == "var":
            n.leaf = names.setdefault(t[1], len(names))
        elif op == "const":
            v = t[1]
            if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, float, np.integer, np.floating)):
                raise TypeError(f"a math constant is an int or a float, not {v!r}")
            is_f = isinstance(v, (float, np.floating))
            n.const_tag = VAL_FLOAT64 if is_f else VAL_INT64
            n.const_word = int(np.array([v], np.float64 if is_f else np.int64).view(np.uint64)[0])
        nodes.append(n)
        return len(nodes) - 1

    walk(tree)
    return nodes


def math_leaf_arrays(m):
    """(keys u64, words u64, tags u8 or None, type, nil) of one variable's map: None (no map), (keys, int64 or
    float64 values) or (keys, u64 words, u8 tags)."""
    if m is None:
        return np.zeros(1, np.uint64), np.zeros(1, np.uint64), None, VAL_INT64, 1
    if len(m) == 3:
        k, w, t = _u64(m[0]), np.ascontiguousarray(m[1], np.uint64), np.ascontiguousarray(m[2], np.uint8)
        if not (k.size == w.size == t.size):
            raise ValueError("keys, words and tags of one size")
        return k, w, t, VAL_INT64, 0
    typ, k, w, n = _val_map(m[0], m[1])
    return k[:n], w[:n], None, typ, 0  # an empty map has no entries (not the one zero key _val_map pads it with)


def EvalMath(tree, maps, range_uids=None):
    """evalMathTree (query/math.go) and valueVarAggregation's math branch (query/query.go :1290-1361) in ONE call
    (dgx_math_eval).  tree: see math_program; maps: variable name -> its map after transformTo (see
    math_leaf_arrays); range_uids: SrcUIDs (DestUIDs at the root), or None.  Returns (kind, keys, words, tags): kind
    "map", "const" or "none", words the 64-bit patterns of the values and tags their DGX_VAL_* types."""
    names = {}
    nodes = math_program(tree, names)
    arrs = [None] * len(names)
    for name, j in names.items():
        arrs[j] = math_leaf_arrays(maps.get(name))
    lv = (_lib.MathLeaf * max(len(arrs), 1))()
    cap = 1
    for j, (k, w, t, typ, nil) in enumerate(arrs):
        n = 0 if nil else k.size
        lv[j] = _lib.MathLeaf(k.ctypes.data, w.ctypes.data, t.ctypes.data if t is not None else None, None, n, typ,
                              nil)
        cap += n
    r = None if range_uids is None else _u64(range_uids.Uids if isinstance(range_uids, List) else range_uids)
    nr = 0 if r is None else r.size
    cap = max(cap, nr, 1)
    ok, ow, ot = np.empty(cap, np.uint64), np.empty(cap, np.uint64), np.empty(cap, np.uint8)
    info = C.c_uint64(0)
    rbuf = None if r is None else (r if r.size else np.zeros(1, np.uint64))
    rp = None if rbuf is None else rbuf.ctypes.data
    prog = (_lib.MathNode * len(nodes))(*nodes)
    _lib.check(_lib.load().dgx_math_eval(prog, len(nodes), lv, len(arrs), rp, nr, _p(ok), _p(ow), _p(ot), cap,
                                         C.byref(info)))
    n = info.value & 0xFFFFFFFF
    return MATH_KIND[(info.value >> 32) & 0xFF], ok[:n].copy(), ow[:n].copy(), ot[:n].copy()


def var_order_leaf(m):
    """(kept arrays, dgx_math_leaf) of the map an order reads: None (Go's nil map, which the call refuses), (keys,
    int64 or float64 values) as PropagateVar / LevelAgg return it, or (keys, u64 words, u8 tags) as EvalMath returns a
    "map" result."""
    k, w, t, typ, nil = math_leaf_arrays(m)
    n = 0 if nil else k.size
    keep = [np.ascontiguousarray(a) if a.size else np.zeros(1, a.dtype) for a in (k, w)]
    if t is not None:
        keep.append(t if t.size else np.zeros(1, np.uint8))
    leaf = _lib.MathLeaf(keep[0].ctypes.data, keep[1].ctypes.data, keep[2].ctypes.data if t is not None else None,
                         None, n, typ, nil)
    return keep, leaf


def OrderByVar(m, desc: bool, dest, rows, count: int = 0, offset: int = 0):
    """orderasc / orderdesc by a value variable (query/query.go applyOrderAndPagination's value-variable branch:
    updateUidMatrix, sortAndPaginateUsingVar with types.Sort and x.PageRange, updateDestUids) in ONE call
    (dgx_var_order), in Go's exact order, ties included.

    m: the variable's map (see var_order_leaf); desc: orderdesc; dest: the node's DestUIDs after its filters; rows:
    its uid matrix (strictly ascending rows); count / offset: Params.Count / Offset.  Returns (rows, dest): the ordered
    and paged rows and the new DestUIDs as a List.  A nil map and a row whose first mapped value is a bool raise
    DgxError (DGX_ERR_ARG), where Go returns an error."""
    keep, leaf = var_order_leaf(m)
    d = _u64(dest.Uids if isinstance(dest, List) else dest)
    v, v_off = _csr_u64(rows)
    nrows, M = len(rows), int(v_off[-1])
    out = np.empty(max(M, 1), np.uint64)
    out_off = np.zeros(nrows + 1, np.uint64)
    dout = np.empty(max(d.size, 1), np.uint64)
    n = C.c_size_t(0)
    _lib.check(_lib.load().dgx_var_order(C.byref(leaf), int(bool(desc)), _p(d), d.size, _p(v), _p(v_off), nrows,
                                         count, offset, _p(out), _p(out_off), M, _p(dout), d.size, C.byref(n)))
    del keep
    return [out[int(out_off[i]):int(out_off[i + 1])].copy() for i in range(nrows)], List(dout[:n.value].copy())


class StrColumn:
    """A string value column (dgx_str_column): the values Go's match loop reads for one predicate.  uids: strictly
    ascending, the uids that have a value; values[i]: the values of uids[i], each bytes (any bytes, valid UTF-8 or
    not) or a str (taken as UTF-8).  One value per uid is a scalar predicate, several a list predicate's."""

    def __init__(self, uids, values):
        self.uid = np.ascontiguousarray(np.asarray(uids, np.uint64).reshape(-1))
        if len(values) != self.uid.size:
            raise ValueError("one list of values per uid")
        vals = [[v.encode() if isinstance(v, str) else bytes(v) for v in vs] for vs in values]
        self.val_off = np.zeros(self.uid.size + 1, np.uint64)
        np.cumsum([len(vs) for vs in vals], out=self.val_off[1:])
        flat = [v for vs in vals for v in vs]
        self.byte_off = np.zeros(len(flat) + 1, np.uint64)
        np.cumsum([len(v) for v in flat], out=self.byte_off[1:])
        self.bytes = np.frombuffer(b"".join(flat) or b"\0", np.uint8).copy()

    @classmethod
    def from_csr(cls, uid, val_off, byte_off, data) -> "StrColumn":
        c = cls.__new__(cls)
        c.uid, c.val_off, c.byte_off = (np.ascontiguousarray(np.asarray(a, np.uint64)) for a in (uid, val_off, byte_off))
        d = np.ascontiguousarray(np.asarray(data, np.uint8))
        c.bytes = d if d.size else np.zeros(1, np.uint8)
        return c

    def struct(self) -> "_lib.StrColumn":
        n = self.uid.size
        nv = self.byte_off.size - 1
        return _lib.StrColumn(self.uid.ctypes.data if n else None, self.val_off.ctypes.data, self.byte_off.ctypes.data,
                              self.bytes.ctypes.data, n, nv, int(self.byte_off[-1]))


def _query_bytes(query) -> np.ndarray:
    q = query.encode() if isinstance(query, str) else bytes(query)
    return np.frombuffer(q + b"\0", np.uint8)[: len(q)].copy() if q else np.zeros(1, np.uint8)


def MatchFuzzy(col: StrColumn, query, threshold: int, uids=None, leaves=(), afterUID: int = 0, keys=None) -> List:
    """match(attr, query, threshold) (worker/task.go handleMatchFunction, worker/match.go uidsForMatch / matchFuzzy) in ONE
    call (dgx_match): the candidates' values tested on the device with Go's []rune Levenshtein distance.

    col: the predicate's StrColumn, holding the values Go reads (Value, ValueForTag or AllUntaggedValues).  query: str
    or bytes.  uids: the filter's UidList (ascending); when it is empty or None the candidates are the union of the
    query's trigram rows, leaves as algo.UidsForRegex takes them (pack leaves (pack, mut) or lists) read from afterUID.
    keys: optional [(key, version)] per leaf naming the pack leaves for the HBM-resident cache.  Returns the kept
    candidates."""
    u = np.zeros(0, np.uint64) if uids is None else _u64(uids.Uids if isinstance(uids, List) else uids)
    pack_ids = [j for j, lf in enumerate(leaves) if isinstance(lf, tuple)]
    list_ids = [j for j, lf in enumerate(leaves) if not isinstance(lf, tuple)]
    packs = [leaves[j][0] for j in pack_ids]
    mut_uids, mut_flags, mut_off = _mut_csr([leaves[j][1] for j in pack_ids])
    arrs = [_u64(leaves[j].Uids if isinstance(leaves[j], List) else leaves[j]) for j in list_ids]
    list_off = np.zeros(len(arrs) + 1, dtype=np.uint64)
    np.cumsum([a.size for a in arrs], out=list_off[1:])
    lists = np.concatenate(arrs) if int(list_off[-1]) else np.zeros(1, np.uint64)
    refs, keep = _refs_of(packs, [keys[j] for j in pack_ids] if keys is not None else None)
    cap = u.size if u.size else sum((_exact(p) if p is not None else 0) + int(mut_off[k + 1] - mut_off[k])
                                    for k, p in enumerate(packs)) + int(list_off[-1])
    q = _query_bytes(query)
    qlen = len(query.encode() if isinstance(query, str) else bytes(query))
    cs = col.struct()
    out = np.empty(max(cap, 1), dtype=np.uint64)
    n = C.c_size_t(0)
    _lib.check(_lib.load().dgx_match(refs, len(packs), _p(mut_uids), _p(mut_flags), _p(mut_off), _p(lists),
                                     _p(list_off), len(arrs), afterUID, _p(u) if u.size else None, u.size,
                                     C.byref(cs), _p(q), qlen, threshold, _p(out), cap, C.byref(n)))
    return List(out[: n.value].copy())


def dev_match(lane, dcol: "_lib.StrColumn", query, threshold: int, d_out: int, out_cap: int, d_out_len: int,
              d_uids: int | None = None, nuids: int = 0, d_nuids: int | None = None, packs=(), d_mut_uids=None,
              d_mut_flags=None, mut_off=None, d_lists=None, list_off=None, afterUID: int = 0) -> None:
    """The lane form of MatchFuzzy (dgx_dev_match), asynchronous: every pointer argument is a device address.

    dcol: a StrColumn struct whose arrays are device memory (a resident column).  d_uids given: the UidList branch,
    its count nuids or the low 32 bits of the device word d_nuids (at most nuids); an empty list is an empty result.
    Otherwise the trigram branch: packs are dgx_dev_pack_upload handles, the layers and lists device arrays with host
    offsets mut_off / list_off.  Writes the kept uids to d_out and their count to the device word d_out_len; a
    malformed input surfaces at the next dgx_lane_sync."""
    tab = (C.c_void_p * max(len(packs), 1))(*packs)
    mo = np.zeros(1, np.uint64) if mut_off is None else np.ascontiguousarray(np.asarray(mut_off, np.uint64))
    lo = np.zeros(1, np.uint64) if list_off is None else np.ascontiguousarray(np.asarray(list_off, np.uint64))
    q = _query_bytes(query)
    qlen = len(query.encode() if isinstance(query, str) else bytes(query))
    _lib.check(_lib.load().dgx_dev_match(lane, tab, len(packs), d_mut_uids, d_mut_flags, _p(mo), d_lists, _p(lo),
                                         lo.size - 1, afterUID, int(d_uids is not None), d_uids, nuids, d_nuids,
                                         C.byref(dcol), _p(q), qlen, threshold, d_out, out_cap, d_out_len))


class RegexProg:
    """regexp()'s pattern compiled for MatchRegex (dgx_regex_compile): Go's "(?m)" + pattern as codesearch matches it,
    one line at a time, as a byte DFA.  fold: the /i modifier.  Raises DgxError (DGX_ERR_ARG) for a pattern outside the
    compiled subset or one Go rejects, and (DGX_ERR_CAP) for a DFA past DGX_REGEX_MAX_STATES states; a caller then
    keeps its own matcher."""

    def __init__(self, pattern, fold: bool = False):
        p = pattern.encode() if isinstance(pattern, str) else bytes(pattern)
        buf = np.frombuffer(p + b"\0", np.uint8)
        h = C.c_void_p()
        _lib.check(_lib.load().dgx_regex_compile(_p(buf), len(p), 1 if fold else 0, C.byref(h)))
        self.handle = h.value

    def __del__(self):
        if getattr(self, "handle", None):
            _lib.load().dgx_regex_free(self.handle)
            self.handle = None

    def tables(self):
        """(cls[256], trans[nstates, nclasses], term[nstates]) copies of the compiled tables."""
        ns, nc = C.c_size_t(), C.c_size_t()
        cp, tp, mp = C.c_void_p(), C.c_void_p(), C.c_void_p()
        _lib.check(_lib.load().dgx_regex_tables(self.handle, C.byref(ns), C.byref(nc), C.byref(cp), C.byref(tp),
                                                C.byref(mp)))
        n, k = ns.value, nc.value
        cls = np.ctypeslib.as_array(C.cast(cp, C.POINTER(C.c_uint8)), (256,)).copy()
        trans = np.ctypeslib.as_array(C.cast(tp, C.POINTER(C.c_uint16)), (n * k,)).reshape(n, k).copy()
        term = np.ctypeslib.as_array(C.cast(mp, C.POINTER(C.c_uint8)), (n,)).copy()
        return cls, trans, term


def MatchRegex(col: StrColumn, prog: RegexProg, uids=None, leaves=(), afterUID: int = 0, keys=None) -> List:
    """regexp(attr, /pattern/) (worker/task.go handleRegexFunction, matchRegex) in ONE call (dgx_regex_match): the
    candidates' values tested on the device with the compiled program.  Candidates as MatchFuzzy takes them: uids (the
    filter's UidList) when not empty, otherwise the union of leaves read from afterUID.  Returns the kept candidates."""
    u = np.zeros(0, np.uint64) if uids is None else _u64(uids.Uids if isinstance(uids, List) else uids)
    pack_ids = [j for j, lf in enumerate(leaves) if isinstance(lf, tuple)]
    list_ids = [j for j, lf in enumerate(leaves) if not isinstance(lf, tuple)]
    packs = [leaves[j][0] for j in pack_ids]
    mut_uids, mut_flags, mut_off = _mut_csr([leaves[j][1] for j in pack_ids])
    arrs = [_u64(leaves[j].Uids if isinstance(leaves[j], List) else leaves[j]) for j in list_ids]
    list_off = np.zeros(len(arrs) + 1, dtype=np.uint64)
    np.cumsum([a.size for a in arrs], out=list_off[1:])
    lists = np.concatenate(arrs) if int(list_off[-1]) else np.zeros(1, np.uint64)
    refs, keep = _refs_of(packs, [keys[j] for j in pack_ids] if keys is not None else None)
    cap = u.size if u.size else sum((_exact(p) if p is not None else 0) + int(mut_off[k + 1] - mut_off[k])
                                    for k, p in enumerate(packs)) + int(list_off[-1])
    cs = col.struct()
    out = np.empty(max(cap, 1), dtype=np.uint64)
    n = C.c_size_t(0)
    _lib.check(_lib.load().dgx_regex_match(refs, len(packs), _p(mut_uids), _p(mut_flags), _p(mut_off), _p(lists),
                                           _p(list_off), len(arrs), afterUID, _p(u) if u.size else None, u.size,
                                           C.byref(cs), prog.handle, _p(out), cap, C.byref(n)))
    return List(out[: n.value].copy())


def dev_match_regex(lane, dcol: "_lib.StrColumn", prog: RegexProg, d_out: int, out_cap: int, d_out_len: int,
                    d_uids: int | None = None, nuids: int = 0, d_nuids: int | None = None, packs=(), d_mut_uids=None,
                    d_mut_flags=None, mut_off=None, d_lists=None, list_off=None, afterUID: int = 0) -> None:
    """The lane form of MatchRegex (dgx_dev_regex_match), asynchronous, with dev_match's arguments and prog in place of
    the query and threshold."""
    tab = (C.c_void_p * max(len(packs), 1))(*packs)
    mo = np.zeros(1, np.uint64) if mut_off is None else np.ascontiguousarray(np.asarray(mut_off, np.uint64))
    lo = np.zeros(1, np.uint64) if list_off is None else np.ascontiguousarray(np.asarray(list_off, np.uint64))
    _lib.check(_lib.load().dgx_dev_regex_match(lane, tab, len(packs), d_mut_uids, d_mut_flags, _p(mo), d_lists,
                                               _p(lo), lo.size - 1, afterUID, int(d_uids is not None), d_uids, nuids,
                                               d_nuids, C.byref(dcol), prog.handle, d_out, out_cap, d_out_len))


VAL_DATETIME, VAL_STRING = 5, 6  # DGX_VAL_* of a typed value column
CMP_OPS = {"le": 0, "ge": 1, "lt": 2, "gt": 3, "eq": 4, "between": 5}  # DGX_SGF_CMP_*
CMP_NO_ARG = 0xFFFFFFFF  # compare_rows' row_arg: the row passes unchanged


def _addr(a):
    return None if a is None else a.ctypes.data


def _val_words(typ: int, vals) -> tuple:
    """(words, nsec) of values of one type: int, float, bool or (unix seconds, nanoseconds)."""
    if typ == VAL_INT64:
        return np.asarray([int(v) for v in vals], np.int64).view(np.uint64), None
    if typ == VAL_FLOAT64:
        return np.asarray([float(v) for v in vals], np.float64).view(np.uint64), None
    if typ == VAL_BOOL:
        return np.asarray([1 if v else 0 for v in vals], np.uint64), None
    if typ == VAL_DATETIME:
        return (np.asarray([int(v[0]) for v in vals], np.int64).view(np.uint64),
                np.asarray([int(v[1]) for v in vals], np.uint32))
    raise ValueError(f"type {typ} has no words")


class ValColumn:
    """A typed value column (dgx_val_column): a predicate's values converted to its schema type, as Go's compare loops
    read them.  typ: VAL_INT64, VAL_FLOAT64, VAL_BOOL, VAL_DATETIME or VAL_STRING.  uids: strictly ascending;
    values[i]: the values of uids[i], each an int, a float, a bool, a (unix seconds, nanoseconds) pair or bytes / str
    by type.  bad: optional, per uid the list of flags of its values whose conversion failed or gave nil."""

    def __init__(self, typ: int, uids, values, bad=None):
        self.type = typ
        flat = [v for vs in values for v in vs]
        if typ == VAL_STRING:
            self.str = StrColumn(uids, values)
            self.uid, self.val_off = self.str.uid, self.str.val_off
            self.word = self.nsec = None
        else:
            self.str = None
            self.uid = np.ascontiguousarray(np.asarray(uids, np.uint64).reshape(-1))
            if len(values) != self.uid.size:
                raise ValueError("one list of values per uid")
            self.val_off = np.zeros(self.uid.size + 1, np.uint64)
            np.cumsum([len(vs) for vs in values], out=self.val_off[1:])
            w, ns = _val_words(typ, flat)
            self.word = w if w.size else np.zeros(1, np.uint64)
            self.nsec = None if ns is None else (ns if ns.size else np.zeros(1, np.uint32))
        self.bad = None if bad is None else np.asarray([1 if b else 0 for bs in bad for b in bs] or [0], np.uint8)

    @classmethod
    def from_arrays(cls, typ: int, uid=None, val_off=None, word=None, nsec=None, bad=None, str_col=None):
        c = cls.__new__(cls)
        c.type, c.str = typ, str_col
        if typ == VAL_STRING:
            c.uid, c.val_off = str_col.uid, str_col.val_off
        else:
            c.uid, c.val_off = (np.ascontiguousarray(np.asarray(a, np.uint64)) for a in (uid, val_off))
        c.word = None if word is None else np.ascontiguousarray(np.asarray(word).view(np.uint64))
        c.nsec = None if nsec is None else np.ascontiguousarray(np.asarray(nsec, np.uint32))
        c.bad = None if bad is None else np.ascontiguousarray(np.asarray(bad, np.uint8))
        return c

    def struct(self) -> "_lib.ValColumn":
        n, nv = self.uid.size, int(self.val_off[-1])
        if self.type == VAL_STRING:
            self._s = self.str.struct()
            return _lib.ValColumn(self.type, None, None, None, None, _addr(self.bad), C.pointer(self._s), 0, 0)
        return _lib.ValColumn(self.type, self.uid.ctypes.data if n else None, self.val_off.ctypes.data,
                              _addr(self.word), _addr(self.nsec), _addr(self.bad), None, n, nv)


class ValArgs:
    """A compare function's arguments (dgx_val_args) of one type, as ValColumn takes values."""

    def __init__(self, typ: int, args):
        args = list(args)
        self.n = len(args)
        if typ == VAL_STRING:
            bs = [a.encode() if isinstance(a, str) else bytes(a) for a in args]
            self.off = np.zeros(len(bs) + 1, np.uint64)
            np.cumsum([len(b) for b in bs], out=self.off[1:])
            self.bytes = np.frombuffer(b"".join(bs) + b"\0", np.uint8).copy()
            self.word = self.nsec = None
        else:
            w, ns = _val_words(typ, args)
            self.word = w if w.size else np.zeros(1, np.uint64)
            self.nsec = ns
            self.bytes = self.off = None

    def struct(self) -> "_lib.ValArgs":
        return _lib.ValArgs(_addr(self.word), _addr(self.nsec), _addr(self.bytes), _addr(self.off), self.n)


def _cmp_op(op) -> int:
    return CMP_OPS[op] if isinstance(op, str) else int(op)


def CompareUids(col: ValColumn, op, args, uids, counts: bool = False):
    """eq / le / lt / ge / gt / between over a UidList (worker/task.go handleValuePostings, compareAttrFn branch) in ONE
    call (dgx_compare_uids): candidate uids[i] is kept when one of its values in col passes types.CompareVals(op, v,
    arg) (CompareBetween for between; eq: any argument).  args: a ValArgs or values of col's type.  Returns the kept
    candidates as a List, and with counts=True also Go's row lengths (matching values per candidate, np.uint32).  A
    candidate with a bad value raises DgxError (DGX_ERR_ARG), where Go returns the conversion error."""
    a = args if isinstance(args, ValArgs) else ValArgs(col.type, args)
    u = _u64(uids.Uids if isinstance(uids, List) else uids)
    cs, ast = col.struct(), a.struct()
    out = np.empty(max(u.size, 1), np.uint64)
    cnt = np.zeros(max(u.size, 1), np.uint32)
    n = C.c_size_t(0)
    _lib.check(_lib.load().dgx_compare_uids(_cmp_op(op), C.byref(ast), C.byref(cs), _p(u) if u.size else None, u.size,
                                            _p(out), u.size, C.byref(n), _p(cnt) if counts else None))
    res = List(out[: n.value].copy())
    return (res, cnt[: u.size].copy()) if counts else res


def CompareRowArgs(op, nrows: int, neq: int = 1, first_is_ineq: bool = False) -> np.ndarray:
    """row_arg for CompareRows from handleCompareFunction's three cases (worker/task.go :1491-1520): eq pairs row r
    with eqTokens[r] (neq of them; Go indexes past them otherwise, which raises ValueError here), between filters
    rows 0 and nrows - 1 against the pair, any other op row 0 when tokens[0] == ineqValueToken[0]."""
    ra = np.full(nrows, CMP_NO_ARG, np.uint32)
    name = op if isinstance(op, str) else {v: k for k, v in CMP_OPS.items()}[int(op)]
    if name == "eq":
        if nrows > neq:
            raise ValueError(f"eq over {nrows} index rows and {neq} eqTokens: Go indexes past eqTokens")
        ra[:] = np.arange(nrows, dtype=np.uint32)
    elif name == "between":
        if nrows:
            ra[0] = ra[nrows - 1] = 0
    elif first_is_ineq and nrows:
        ra[0] = 0
    return ra


def CompareRows(col: ValColumn, op, args, rows, row_arg) -> list:
    """handleCompareFunction's filterRow over the index rows (worker/task.go :1395-1520) in ONE call
    (dgx_compare_rows): row r stays as it is when row_arg[r] is CMP_NO_ARG, otherwise keeps the uids with a value in
    col passing op against argument row_arg[r] (between: row_arg[r] and the next); a bad value never passes.  Rows
    need not ascend.  Returns the filtered rows."""
    a = args if isinstance(args, ValArgs) else ValArgs(col.type, args)
    v, v_off = _csr_u64(rows)
    ra = np.ascontiguousarray(np.asarray(row_arg, np.uint32))
    nrows, M = len(rows), int(v_off[-1])
    cs, ast = col.struct(), a.struct()
    out = np.empty(max(M, 1), np.uint64)
    out_off = np.zeros(nrows + 1, np.uint64)
    _lib.check(_lib.load().dgx_compare_rows(_cmp_op(op), C.byref(ast), C.byref(cs), _p(v), _p(v_off), nrows,
                                            _p(ra) if nrows else None, _p(out), _p(out_off), M))
    return [out[int(out_off[i]):int(out_off[i + 1])].copy() for i in range(nrows)]


def dev_compare_uids(lane, dcol: "_lib.ValColumn", op, args: ValArgs, d_uids: int, nuids: int, d_out: int,
                     out_cap: int, d_out_len: int, d_nuids: int | None = None, d_counts: int | None = None) -> None:
    """The lane form of CompareUids (dgx_dev_compare_uids), asynchronous: dcol is a ValColumn struct whose arrays are
    device memory (a resident column), args stay on the host, the other pointers are device addresses; the count is
    nuids or the low 32 bits of the device word d_nuids.  Refusals found on the device surface at dgx_lane_sync."""
    ast = args.struct()
    _lib.check(_lib.load().dgx_dev_compare_uids(lane, _cmp_op(op), C.byref(ast), C.byref(dcol), d_uids, nuids,
                                                d_nuids, d_out, out_cap, d_out_len, d_counts))


def dev_compare_rows(lane, dcol: "_lib.ValColumn", op, args: ValArgs, d_v: int, d_v_off: int, nrows: int, v_cap: int,
                     row_arg, d_out: int, d_out_off: int, out_cap: int) -> None:
    """The lane form of CompareRows (dgx_dev_compare_rows), asynchronous: the rows calls' (d_out, d_out_off) as they
    are, v_cap their room; row_arg on the host."""
    ast = args.struct()
    ra = np.ascontiguousarray(np.asarray(row_arg, np.uint32))
    _lib.check(_lib.load().dgx_dev_compare_rows(lane, _cmp_op(op), C.byref(ast), C.byref(dcol), d_v, d_v_off, nrows,
                                                v_cap, _p(ra) if nrows else None, d_out, d_out_off, out_cap))


def OrderByPred(col: ValColumn, desc: bool, dest, rows, count: int = 0, offset: int = 0):
    """orderasc / orderdesc by a predicate without its index (query/query.go applyOrderAndPagination's predicate
    branch with worker/sort.go sortWithoutIndex: sortByValue, paginate) in ONE call (dgx_pred_order), in Go's exact
    order, ties included.

    col: the predicate's ValColumn (VAL_INT64, VAL_FLOAT64, VAL_DATETIME or VAL_STRING, one value per uid; a bad value
    counts as none); desc: orderdesc; dest: the node's DestUIDs; rows: its uid matrix (strictly ascending rows);
    count / offset: the SortMessage's Count (already 1000 for 0, as the query layer sets it) and Offset.  Each row is
    its dest uids with a value sorted by value, then those without one in row order, cut by x.PageRange.  Returns
    (rows, dest): the ordered and paged rows and the new DestUIDs as a List.  A bool column, a negative count and a
    list predicate's column raise DgxError (DGX_ERR_ARG), where Go returns an error."""
    d = _u64(dest.Uids if isinstance(dest, List) else dest)
    v, v_off = _csr_u64(rows)
    nrows, M = len(rows), int(v_off[-1])
    cs = col.struct()
    out = np.empty(max(M, 1), np.uint64)
    out_off = np.zeros(nrows + 1, np.uint64)
    dout = np.empty(max(d.size, 1), np.uint64)
    n = C.c_size_t(0)
    _lib.check(_lib.load().dgx_pred_order(C.byref(cs), int(bool(desc)), _p(d), d.size, _p(v), _p(v_off), nrows,
                                          count, offset, _p(out), _p(out_off), M, _p(dout), d.size, C.byref(n)))
    return [out[int(out_off[i]):int(out_off[i + 1])].copy() for i in range(nrows)], List(dout[:n.value].copy())


def dev_order_by_pred(lane, dcol: "_lib.ValColumn", desc: bool, d_dest: int, ndest: int, d_v: int, d_v_off: int,
                      nrows: int, v_cap: int, d_out: int, d_out_off: int, out_cap: int, d_dest_out: int,
                      dest_cap: int, d_dest_len: int, count: int = 0, offset: int = 0,
                      d_ndest: int | None = None) -> None:
    """The lane form of OrderByPred (dgx_dev_pred_order), asynchronous: dcol is a ValColumn struct whose arrays are
    device memory (a resident column), every other pointer a device address; |dest| is ndest or the low 32 bits of
    the device word d_ndest.  Refusals found on the device surface at dgx_lane_sync."""
    _lib.check(_lib.load().dgx_dev_pred_order(lane, C.byref(dcol), int(bool(desc)), d_dest, ndest, d_ndest, d_v,
                                              d_v_off, nrows, v_cap, count, offset, d_out, d_out_off, out_cap,
                                              d_dest_out, dest_cap, d_dest_len))


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
