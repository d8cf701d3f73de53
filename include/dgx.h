/*
 * dgx.h -- C ABI of libdgx.so: H100-native (sm_90a) sorted-uint64 posting-list
 * set operations and UidPack decode, the drop-in for dgraph's algo/ + codec/
 * hot path.
 *
 * The reference has no plugin interface for this path: callers invoke
 * package-level Go functions.  The boundary is therefore the Go signatures
 * themselves; a cgo shim (go/algo_dgx.go, see INTEGRATION.md) keeps each
 * signature and forwards to the entry point listed beside it here.  All
 * citations are relative to /root/reference.
 *
 * Conventions
 *  - Plain pointers and sizes only.  Inputs are BORROWED for the duration of
 *    the call (Go memory may move afterwards): every entry point has finished
 *    reading its inputs when it returns.  Outputs are CALLER-ALLOCATED; the
 *    library writes at most out_cap values and reports the length.
 *  - Return value: DGX_OK (0) or a negative dgx_status.  The reference
 *    functions cannot fail; the shim falls back to the Go code on non-zero.
 *  - Thread safety: every entry point may be called concurrently from many
 *    threads (goroutines pinned to OS threads by cgo); each call borrows an
 *    execution lane (CUDA stream + workspace) from a pool.
 *  - Lists are sorted ascending uint64 (pb.List.Uids, protos/pb.proto:22-24).
 *    Duplicates follow the reference: multiset-min for intersections,
 *    multiset difference, global dedup for MergeSorted.
 */
#ifndef DGX_H
#define DGX_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum dgx_status {
    DGX_OK = 0,
    DGX_ERR_CUDA = -1,   /* a CUDA runtime call failed (dgx_last_error has the text) */
    DGX_ERR_OOM = -2,    /* device or pinned-host allocation failed */
    DGX_ERR_ARG = -3,    /* invalid argument */
    DGX_ERR_CAP = -4,    /* out_cap too small for the result */
    DGX_ERR_NODEV = -5   /* no CUDA device / library not initialised */
} dgx_status;

/* ---- lifecycle ---------------------------------------------------------- */

/* Bind the library to CUDA device `device` (-1: current device).  Idempotent;
 * called implicitly by the first host-pointer entry point. */
int dgx_init(int device);
void dgx_shutdown(void);
/* Text of the last error on the calling thread ("" when none). */
const char* dgx_last_error(void);
/* Library / device description for logs: writes a NUL-terminated string. */
int dgx_describe(char* buf, size_t buf_len);

/* Pinned host memory: lists allocated here cross PCIe at full DMA speed. */
void* dgx_host_alloc(size_t bytes);
void dgx_host_free(void* p);

/* Counters (SURVEY.md section 5: metrics). */
typedef struct dgx_stats {
    uint64_t calls;
    uint64_t uids_in;
    uint64_t uids_out;
    uint64_t h2d_bytes;
    uint64_t d2h_bytes;
    uint64_t kernel_launches;
} dgx_stats;
void dgx_get_stats(dgx_stats* out);

/* ---- host-pointer entry points (what the cgo shim binds) ---------------- */

/* algo.IntersectWith(u, v, o *pb.List)            algo/uidlist.go:142-167
 * o.Uids = u ∩ v.  `out` may alias `u` (the in-place form every caller uses);
 * `v` is never written.  out_cap >= min(n, m). */
int dgx_intersect2(const uint64_t* u, size_t n, const uint64_t* v, size_t m,
                   uint64_t* out, size_t out_cap, size_t* out_len);

/* algo.IntersectSorted(lists []*pb.List) *pb.List  algo/uidlist.go:297-329
 * k == 0 -> length 0; k == 1 -> copy.  out_cap >= min_i lens[i]. */
int dgx_intersect_sorted(const uint64_t* const* lists, const size_t* lens, size_t k,
                         uint64_t* out, size_t out_cap, size_t* out_len);

/* algo.MergeSorted(lists []*pb.List) *pb.List      algo/uidlist.go:448-542
 * Sorted union with global de-duplication.  NULL / empty lists are skipped.
 * out_cap >= sum(lens). */
int dgx_merge_sorted(const uint64_t* const* lists, const size_t* lens, size_t k,
                     uint64_t* out, size_t out_cap, size_t* out_len);

/* algo.Difference(u, v *pb.List) *pb.List          algo/uidlist.go:332-362
 * u \ v (multiset: one v consumes one equal u).  out_cap >= n. */
int dgx_difference(const uint64_t* u, size_t n, const uint64_t* v, size_t m,
                   uint64_t* out, size_t out_cap, size_t* out_len);

/* Batched independent 2-way intersections in CSR form: pair i intersects
 * a[a_off[i]..a_off[i+1]) with b[b_off[i]..b_off[i+1]); results are written
 * back to back into `out` with out_off[i]..out_off[i+1] (npairs+1 offsets).
 * This is the handleUidPostings / updateUidMatrix shape
 * (worker/task.go:783-987, query/query.go:1425-1438): N rows each filtered by
 * algo.IntersectWith. */
int dgx_intersect_batch(const uint64_t* a, const uint64_t* a_off,
                        const uint64_t* b, const uint64_t* b_off, size_t npairs,
                        uint64_t* out, uint64_t* out_off, size_t out_cap);

/* pb.UidPack (protos/pb.proto:379-400) flattened to a struct of arrays.
 * Block i: Base = base[i], NumUids = num_uids[i],
 * Deltas = deltas[delta_off[i] .. delta_off[i+1]).  `deltas` need not be padded. */
typedef struct dgx_pack_view {
    uint32_t block_size;
    size_t nblocks;
    const uint64_t* base;
    const uint32_t* num_uids;
    const uint64_t* delta_off; /* nblocks + 1 entries, delta_off[0] == 0 */
    const uint8_t* deltas;
} dgx_pack_view;

/* codec.Decode(pack *pb.UidPack, seek uint64) []uint64   codec/codec.go:444-452
 * Decoder.Seek(seek, SeekStart) (:279-337) then every following block.
 * out_cap >= ExactLen(pack) (codec/codec.go:427-440).  p == NULL is the nil pack. */
int dgx_decode(const dgx_pack_view* p, uint64_t seek,
               uint64_t* out, size_t out_cap, size_t* out_len);

/* codec.Decode followed by algo.IntersectSorted([decoded, lists...]) without
 * the decoded list leaving the device (BASELINE config 3 pipeline). */
int dgx_decode_intersect_sorted(const dgx_pack_view* p, uint64_t seek,
                                const uint64_t* const* lists, const size_t* lens, size_t k,
                                uint64_t* out, size_t out_cap, size_t* out_len);

/* algo.IntersectCompressedWith(pack *pb.UidPack, afterUID uint64, v, o *pb.List)
 *                                                        algo/uidlist.go:33-61
 * o.Uids = v ∩ (uids of pack from Decoder.Seek(afterUID, SeekStart) onward) -- the entry
 * point posting.List.Uids uses for filtered reads (posting/list.go:1795-1800).  The pack
 * crosses PCIe compressed and is decoded on the device; the reference's LinJump / Bin
 * split (:49-59) only changes how the same set is computed.  out_cap >= m.
 * Defined, like the reference's own tests, for duplicate-free inputs. */
int dgx_intersect_compressed(const dgx_pack_view* p, uint64_t after_uid, const uint64_t* v, size_t m,
                             uint64_t* out, size_t out_cap, size_t* out_len);

/* ---- posting lists as production holds them: UidPacks, optionally HBM-resident ----------- */
/* posting.List keeps its uids as a pb.UidPack (posting/list.go:1795-1800, 1861) and every query
 * decodes what it needs.  A pack crosses PCIe at ~1.5 B/UID where the decoded list costs 8, so the
 * entry points below take packs, expand them on the device and run the set operation there.
 * A pack the caller can NAME stays resident in HBM (compressed) between calls:
 *   key     != 0: identity of the posting list, e.g. a 64-bit hash of its Badger key; 0 = anonymous
 *   version     : commit timestamp of the immutable layer the pack was built from (List.minTs);
 *                 (key, version) must name immutable bytes -- a rollup produces a new version.
 * On a hit nothing is copied; on a miss the pack is uploaded and kept, least-recently-used packs
 * making room (capacity: DGX_CACHE_BYTES, default 16 GiB, or dgx_cache_configure). */
typedef struct dgx_pack_ref {
    const dgx_pack_view* pack;
    uint64_t key;
    uint64_t version;
} dgx_pack_ref;

/* Flat image of a pack: [base u64 x n | delta_off u64 x (n+1) | num_uids u32 x n | pad to 16 | deltas | pad to 16],
 * 16-byte aligned.  A shim that flattens pb.UidPack.Blocks ([]*UidBlock, each with its own Deltas slice) into
 * pinned staging memory can write this layout directly: dgx_pack_image_view points a dgx_pack_view at the arrays of
 * an image buffer (the caller fills them), and the views of images placed back to back in one buffer cross PCIe
 * as ONE transfer when passed to the same call (a DMA of every small array costs microseconds of set-up each). */
size_t dgx_pack_image_size(size_t nblocks, size_t delta_bytes);
int dgx_pack_image_view(void* image, uint32_t block_size, size_t nblocks, size_t delta_bytes, dgx_pack_view* view);

/* algo.IntersectSorted over lists held as packs: codec.Decode(pack_i, 0) for every i
 * (codec/codec.go:444-452) then algo.IntersectSorted (algo/uidlist.go:297-329), the decoded lists
 * never leaving the device.  A NULL / empty pack is the empty list.  out_cap >= min_i ExactLen. */
int dgx_intersect_sorted_packed(const dgx_pack_ref* refs, size_t k,
                                uint64_t* out, size_t out_cap, size_t* out_len);

/* codec.Encode(uids, blockSize) (codec/codec.go:57-136, 393-399) on the device: block split at a change of the
 * upper 32 bits or after BlockSize uids, group-varint deltas.  The caller allocates base[*nblocks],
 * num_uids[*nblocks], delta_off[*nblocks + 1], deltas[*delta_bytes] (dgx_encode_bound gives sizes that hold any
 * list with at most 64 upper-word changes); on return *nblocks / *delta_bytes are the pack's sizes and `view`
 * points at the arrays.  DGX_ERR_CAP: the arrays are too small, sizes that suffice were returned (the exact ones
 * when the list's segments fit the arrays given), and one call again with them succeeds.
 * n == 0 is the nil pack (nblocks 0). */
void dgx_encode_bound(size_t n, uint32_t block_size, size_t* nblocks_cap, size_t* delta_cap);
int dgx_encode(const uint64_t* uids, size_t n, uint32_t block_size,
               uint64_t* base, uint32_t* num_uids, uint64_t* delta_off, uint8_t* deltas,
               size_t* nblocks, size_t* delta_bytes, dgx_pack_view* view);

/* Packed set operations (algo/packed.go:35-297): operands and result are UidPacks; decode, the plain-list
 * kernel and Encode run back to back on the device, so both directions cross PCIe compressed.
 *   dgx_intersect_packed             IntersectWithLinPacked(u, v)      :35-101
 *   dgx_intersect_sorted_packed_out  IntersectSortedPacked(lists)      :103-139 (all k lists, see DESIGN section 5)
 *   dgx_difference_packed            DifferencePacked(u, v)            :141-226
 *   dgx_merge_sorted_packed          MergeSortedPacked(lists)          :228-297
 * Output arrays and capacities as in dgx_encode (bound: the result is at most min / |u| / sum of the operands'
 * ExactLen uids).  NULL / empty packs are empty lists. */
int dgx_intersect_packed(const dgx_pack_ref* u, const dgx_pack_ref* v, uint32_t block_size,
                         uint64_t* base, uint32_t* num_uids, uint64_t* delta_off, uint8_t* deltas,
                         size_t* nblocks, size_t* delta_bytes, dgx_pack_view* view);
int dgx_intersect_sorted_packed_out(const dgx_pack_ref* refs, size_t k, uint32_t block_size,
                                    uint64_t* base, uint32_t* num_uids, uint64_t* delta_off, uint8_t* deltas,
                                    size_t* nblocks, size_t* delta_bytes, dgx_pack_view* view);
int dgx_difference_packed(const dgx_pack_ref* u, const dgx_pack_ref* v, uint32_t block_size,
                          uint64_t* base, uint32_t* num_uids, uint64_t* delta_off, uint8_t* deltas,
                          size_t* nblocks, size_t* delta_bytes, dgx_pack_view* view);
int dgx_merge_sorted_packed(const dgx_pack_ref* refs, size_t k, uint32_t block_size,
                            uint64_t* base, uint32_t* num_uids, uint64_t* delta_off, uint8_t* deltas,
                            size_t* nblocks, size_t* delta_bytes, dgx_pack_view* view);

/* algo.IntersectCompressedWith with a named (cacheable) pack; dgx_intersect_compressed is the anonymous form. */
int dgx_intersect_compressed_ref(const dgx_pack_ref* ref, uint64_t after_uid, const uint64_t* v, size_t m,
                                 uint64_t* out, size_t out_cap, size_t* out_len);

/* algo.IntersectCompressedWith(pack_i, afterUID, v, o_i) for every row i, one call: the handleUidPostings loop
 * (worker/task.go:783-987 -> posting/list.go:1795-1800) with its one ListOptions.  Row i of the CSR result is
 * out[out_off[i] .. out_off[i+1]) (nrows + 1 offsets).  refs[i] as in dgx_intersect_sorted_packed (named packs use the
 * HBM cache, anonymous ones cross PCIe together); a NULL / empty pack is an empty row.  v is ascending and
 * duplicate-free, m < 2^32 (DGX_ERR_ARG otherwise).  out_cap >= sum_i min(m, ExactLen(pack_i)).  The batch runs a fixed
 * number of kernel launches whatever nrows is. */
int dgx_intersect_compressed_rows(const dgx_pack_ref* refs, size_t nrows, uint64_t after_uid,
                                  const uint64_t* v, size_t m,
                                  uint64_t* out, uint64_t* out_off, size_t out_cap);

/* algo.IntersectCompressedWith(pack, 0, v_i, o_i) for every row i of a uid matrix, one call: the intersectBucket loop
 * (worker/sort.go:605-700 -> posting/list.go:1795-1800).  Row i of the input is v[v_off[i] .. v_off[i+1]) (host
 * offsets, nrows + 1 values, v_off[0] == 0); row i of the result is out[out_off[i] .. out_off[i+1]).  ref as in
 * dgx_intersect_compressed_ref (named packs use the HBM cache).  out_cap >= sum_i min(|v_i|, ExactLen(pack)).
 * Every row must ascend strictly; a row that does not is DGX_ERR_ARG and nothing is written to out.  v_off[0] != 0,
 * decreasing offsets, v_off[nrows] >= 2^32 and malformed packs are DGX_ERR_ARG before anything is copied.  A NULL /
 * empty pack gives empty rows and nrows == 0 gives out_off[0] = 0; neither needs a device.  The call runs a fixed
 * number of kernel launches whatever nrows, the number of uids and the pack's size are. */
int dgx_intersect_compressed_matrix(const dgx_pack_ref* ref, const uint64_t* v, const uint64_t* v_off, size_t nrows,
                                    uint64_t* out, uint64_t* out_off, size_t out_cap);

/* posting.List.Uids(opts) for every key of a task, mutable layers included, one call: the handleUidPostings loop
 * (worker/task.go:783-987 -> posting/list.go:1758-1870) of a filtered read of unsplit lists.  v = opts.Intersect.Uids
 * (ascending, duplicate-free, 0 < m < 2^31), after_uid = opts.AfterUid.  Row i takes the branch mode[i] of List.Uids:
 *   DGX_UIDS_COMPRESSED  no mutable layer (:1795-1800): {x in v : x in pack, x >= after}, exactly
 *                        dgx_intersect_compressed_rows; such a row has no mutable entries
 *   DGX_UIDS_PROBE       len(v) < ApproxLen (:1805-1820), findPostingWithItr per x of v, after ignored:
 *                        {x in v : mut(x) exists ? mut(x) is not DGX_MUT_DEL : x in pack}
 *   DGX_UIDS_ITERATE     otherwise (:1822-1862), iterate with the REF filter then IntersectWith; the pack side is
 *                        Seek(after, SeekCurrent): {x in v : x > after, mut(x) exists ? mut(x) has no flag : x in pack}
 * mut(x) is row i's resolved mutable entry of uid x -- the posting List.Uids would see (first of pickPostings per uid
 * for iterate rows, MutableLayer.findPosting for probe rows): the caller does the MVCC work.  Row i's entries are
 * mut_uids / mut_flags[mut_off[i] .. mut_off[i+1]) (host offsets, mut_off[0] == 0), strictly ascending, nonzero, with
 * flags DGX_MUT_DEL (Op == Del) and DGX_MUT_VALUE (PostingType != REF).  A row with a delete-all marker is passed with a
 * NULL pack.  refs[i] as in dgx_intersect_compressed_rows.  Row i of the CSR result is out[out_off[i] .. out_off[i+1]);
 * out_cap >= sum_i min(m, ExactLen(pack_i) + |mut_i|) always suffices; a longer result than out_cap is DGX_ERR_CAP and
 * nothing is written past out_cap.  nrows == 0 gives out_off[0] = 0 and needs no device.
 * DGX_ERR_ARG before anything is copied: a mode not listed, a compressed row with mutable entries, mut_off[0] != 0 or
 * decreasing offsets, m == 0 or m >= 2^31, 2^31 or more mutable entries in all, an iterate row with
 * ExactLen + |mut| >= 2^31 (the MaxInt32 cut of :1864-1870 must not bite), a null array that is needed.
 * DGX_ERR_ARG after the kernels, with out untouched: a mutable entry that does not ascend strictly, is 0 or has other
 * flag bits, or a probe / iterate row whose pack starts at uid 0.  The call runs a fixed number of kernel launches
 * whatever nrows, the number of mutable entries and the pack sizes are. */
enum { DGX_UIDS_COMPRESSED = 0, DGX_UIDS_PROBE = 1, DGX_UIDS_ITERATE = 2 };
enum { DGX_MUT_DEL = 1, DGX_MUT_VALUE = 2 };
int dgx_list_uids_rows(const dgx_pack_ref* refs, const uint8_t* mode, size_t nrows,
                       const uint64_t* mut_uids, const uint8_t* mut_flags, const uint64_t* mut_off,
                       uint64_t after_uid, const uint64_t* v, size_t m,
                       uint64_t* out, uint64_t* out_off, size_t out_cap);

/* posting.List.Uids(opts) with opts.Intersect == nil for every key of a task, mutable layers included, one call: the
 * handleUidPostings loop (worker/task.go:783-987, the default branch without facets) of a plain edge traversal over
 * unsplit lists.  Every row runs iterate(readTs, after_uid) with the REF filter (posting/list.go:1116-1232, 1830-1845)
 * and the First cut (:1864-1872).  With refs / mut_* / mut_off as in dgx_list_uids_rows (NULL pack: delete-all marker
 * or empty immutable layer; mut(x) the first posting of pickPostings for uid x):
 *   S_i = {x > after_uid : mut_i(x) exists ? mut_i(x) has no flag : x in pack_i}
 * The pack side is Decoder.Seek(after_uid, SeekCurrent), the mutable side starts at the first entry above after_uid.
 * first = opts.First as the worker passes it (q.First + q.Offset): 0 means MaxInt32; first > 0 keeps the first
 * smallest values of S_i; first < 0 keeps min(|S_i|, 1) values, as the callback stops after one value and the
 * negative cut keeps it.  Row i of the CSR result is out[out_off[i] .. out_off[i+1]); out_cap >=
 * sum_i min(first_eff, ExactLen(pack_i) + |mut_i|) always suffices (first_eff: the values a row keeps); a longer
 * result than out_cap is DGX_ERR_CAP and nothing is written past out_cap.  nrows == 0 gives out_off[0] = 0 and needs
 * no device.
 * DGX_ERR_ARG before anything is copied: mut_off[0] != 0 or decreasing offsets, 2^31 or more mutable entries in all, a
 * row with ExactLen + |mut| >= 2^31, a null array that is needed.
 * DGX_ERR_ARG after the kernels, with out untouched and out_off zeroed: a mutable entry that does not ascend strictly,
 * is 0 or has other flag bits, or a non-NULL pack that starts at uid 0.  The call runs a fixed number of kernel
 * launches whatever nrows, the number of mutable entries and the pack sizes are; a block of a pack is read only when
 * it holds a value of the row above after_uid and within the first cut. */
int dgx_list_uids_unfiltered_rows(const dgx_pack_ref* refs, size_t nrows,
                                  const uint64_t* mut_uids, const uint8_t* mut_flags, const uint64_t* mut_off,
                                  uint64_t after_uid, int32_t first,
                                  uint64_t* out, uint64_t* out_off, size_t out_cap);
/* countForUidPostings with a nil facets tree (worker/task.go:743-755, 866-876) for every key of a task:
 * counts[i] = |S_i| as above, which List.Postings (posting/list.go:1878-1890) yields; First plays no part.  Arguments
 * and errors as in dgx_list_uids_unfiltered_rows; a device-detected error zeroes counts.  Only the block each row's
 * seek lands in and the block each entry lands in are read. */
int dgx_list_count_rows(const dgx_pack_ref* refs, size_t nrows,
                        const uint64_t* mut_uids, const uint8_t* mut_flags, const uint64_t* mut_off,
                        uint64_t after_uid, uint32_t* counts);

/* algo.MergeSorted(rows) over the rows of a uid matrix, one call: sg.DestUIDs = algo.MergeSorted(result.UidMatrix)
 * (query/query.go:2290, 2505; query/recurse.go:134; worker/task.go:1629, 1706; worker/match.go:100).
 * Row i is v[v_off[i] .. v_off[i+1]) (host offsets, nrows + 1 values, v_off[0] == 0).  Rows ascend; duplicates
 * inside a row and across rows are allowed and removed, as MergeSorted does (TestMergeSorted9 {1,1,1} -> {1}).
 * out_cap >= the result length (v_off[nrows] always suffices), else DGX_ERR_CAP.  v_off[0] != 0, decreasing offsets
 * and v_off[nrows] >= 2^32 are DGX_ERR_ARG before anything is copied; a row that descends is DGX_ERR_ARG and nothing is
 * written to out.  nrows == 0 or all rows empty gives *out_len = 0 and needs no device.  v and v_off cross PCIe as one
 * copy each; the number of kernel launches does not depend on nrows. */
int dgx_merge_sorted_matrix(const uint64_t* v, const uint64_t* v_off, size_t nrows,
                            uint64_t* out, size_t out_cap, size_t* out_len);

/* codec.Decoder positioned calls (codec/codec.go:154-384), one call each, computed on the device:
 *   kind 0 Decoder.Seek(uid, whence)          :279-337   whence 0 = SeekStart (>= uid), 1 = SeekCurrent (> uid)
 *   kind 1 Decoder.SeekToBlock(uid, whence)   :219-271   resumes the base search at block_idx
 *   kind 2 Decoder.LinearSeek(uid)            :349-359   advances from block_idx while uid >= next base
 *   kind 3 Decoder.Next()                     :370-376
 *   kind 4 Decoder.UnpackBlock()              :154-200   (block_idx itself)
 * `block_idx` is the decoder's blockIdx before the call (its current block counts as fully unpacked); the
 * returned slice is what the Go call returns, *block_idx_after the decoder's blockIdx afterwards.
 * out_cap >= the pack's largest NumUids (BlockSize for packs built by codec.Encode). */
int dgx_pack_seek(const dgx_pack_view* p, int kind, uint64_t uid, int whence, size_t block_idx,
                  uint64_t* out, size_t out_cap, size_t* out_len, size_t* block_idx_after);

typedef struct dgx_cache_stats {
    uint64_t hits, misses, evictions;
    uint64_t bytes, entries, max_bytes;
} dgx_cache_stats;
int dgx_cache_configure(size_t max_bytes); /* 0 disables caching (and empties the cache) */
void dgx_cache_clear(void);
void dgx_cache_get_stats(dgx_cache_stats* out);

/* algo.IndexOf(u, uid) for a batch of uids (algo/uidlist.go:546-552): idx[i] = position of uids[i]
 * in the ascending list u, -1 when absent.  `uids` need not be sorted.  Callers: updateDestUids,
 * updateFacetMatrix, updateUidMatrix (query/query.go:1396-1438, 2594-2608) probe sg.DestUIDs with
 * every uid of the uid matrix. */
int dgx_index_of_batch(const uint64_t* u, size_t n, const uint64_t* uids, size_t m, int64_t* idx);

/* dgx_intersect_batch with ONE list `b` shared by every row: out row i = a[a_off[i]..a_off[i+1]) ∩ b.
 * The `algo.IntersectWith(l, sg.DestUIDs, l)` loop over a uid matrix (query/query.go:1425-1438) and
 * the per-row filters of worker/task.go:1351, 1616, 1691, 1777; `b` crosses PCIe once. */
int dgx_intersect_batch_shared(const uint64_t* a, const uint64_t* a_off, size_t npairs,
                               const uint64_t* b, size_t m,
                               uint64_t* out, uint64_t* out_off, size_t out_cap);

/* ---- protobuf wire-format adjacency (host only, no device needed) ----------- */
/* Posting lists reach the path as serialized pb.PostingList values read from Badger
 * (proto.Unmarshal, posting/list.go:1045, posting/mvcc.go:634) and leave it as pb.List
 * inside pb.Result.uid_matrix (protos/pb.proto:22-24, 76-78).  These entry points read
 * and write exactly those bytes, so a caller can go from a stored value to dgx_pack_view
 * and from a result buffer to a pb.List message without building Go structs in between.
 * Standard proto3 wire format; unknown fields are skipped; malformed or truncated input
 * is DGX_ERR_ARG. */

/* pb.PostingList{pack = 1} (protos/pb.proto:402-408): locate the serialized pb.UidPack
 * inside a stored value.  *pack == NULL, *pack_len == 0 when the field is absent (nil pack). */
int dgx_wire_posting_list_pack(const uint8_t* buf, size_t len, const uint8_t** pack, size_t* pack_len);

/* pb.UidPack{block_size = 1, blocks = 2, alloc_ref = 23} / pb.UidBlock{base = 1,
 * deltas = 2, num_uids = 3} (protos/pb.proto:378-400): count blocks and delta bytes so
 * the caller can allocate the struct of arrays. */
int dgx_wire_pack_measure(const uint8_t* buf, size_t len, size_t* nblocks, size_t* delta_bytes);

/* Parse the same message into caller-allocated arrays (base[nblocks], num_uids[nblocks],
 * delta_off[nblocks + 1], deltas[delta_bytes]) and point `view` at them: the result feeds
 * dgx_decode / dgx_intersect_compressed / dgx_dev_pack_upload directly.  DGX_ERR_CAP when
 * the arrays are too small. */
int dgx_wire_pack_parse(const uint8_t* buf, size_t len,
                        uint64_t* base, uint32_t* num_uids, uint64_t* delta_off, uint8_t* deltas,
                        size_t nblocks_cap, size_t delta_cap, dgx_pack_view* view);

/* pb.List{repeated fixed64 uids = 1} (protos/pb.proto:22-24) is packed: tag 0x0A, varint
 * byte length, then the little-endian values -- a result buffer IS the payload.  Writes the
 * header for n values into hdr (at most 11 bytes) and returns its length; 0 for n == 0
 * (proto3 omits an empty repeated field).  The message is hdr || values. */
size_t dgx_wire_list_header(size_t n, uint8_t* hdr);

/* pb.Result{repeated List uid_matrix = 1} (protos/pb.proto:76-78): frame a CSR result -- the
 * (out, out_off) pair dgx_intersect_batch / dgx_dev_filter_batch produce, nrows + 1 offsets -- as
 * the uid_matrix rows of a serialized pb.Result: per row tag 0x0A, the row's byte length, then the
 * pb.List message (empty rows are `0A 00`).  buf == NULL only sizes.  Other pb.Result fields can be
 * appended by the caller; DGX_ERR_CAP when buf_cap is too small. */
int dgx_wire_uid_matrix(const uint64_t* out, const uint64_t* out_off, size_t nrows,
                        uint8_t* buf, size_t buf_cap, size_t* len);

/* Inverse: the uids of a serialized pb.List, packed chunks and unpacked entries in order.
 * out == NULL only counts.  DGX_ERR_CAP when out_cap is too small. */
int dgx_wire_list_decode(const uint8_t* buf, size_t len, uint64_t* out, size_t out_cap, size_t* out_len);

/* ---- device-resident API ------------------------------------------------- */
/* For callers that keep posting lists in HBM (a pack / list cache) and for
 * roofline measurement.  All pointers named d_* are device pointers on the
 * lane's device; they must be 16-byte aligned.  Calls are asynchronous on the
 * lane's stream unless stated; dgx_lane_sync waits. */

typedef struct dgx_lane dgx_lane; /* one CUDA stream + its workspace */

/* stream: an existing cudaStream_t to run on (e.g. torch's current stream) or
 * NULL to create a private non-blocking stream. */
dgx_lane* dgx_lane_create(int device, void* stream);
void dgx_lane_destroy(dgx_lane* lane);
int dgx_lane_sync(dgx_lane* lane);
void* dgx_lane_stream(dgx_lane* lane);
/* Declare that the device lists passed to dgx_dev_filter_batch on this lane are RESIDENT: complete before the call
 * and not written by anything queued on the lane's stream (the contract of a pack / list cache: posting lists are
 * immutable once rolled up).  The plan pre-pass of a batch then runs on a side stream while the pipeline kernel of the
 * previous batch is still busy (its tables alternate between two workspaces).  Results (d_out, d_out_off) stay ordered
 * on the lane's stream as before.  A batch that reads a buffer this lane's own queued calls write (the output of an
 * earlier dgx_dev_decode / dgx_dev_merge_sorted / dgx_dev_filter_batch since the last dgx_lane_sync) is recognised by
 * its address and planned behind them instead of ahead, so chains on one lane stay correct; lists written by OTHER
 * streams must be complete before the call.  Off by default; the host-pointer entry points never use it. */
int dgx_lane_set_resident_inputs(dgx_lane* lane, int on);
/* Number of kernels this lane has launched so far. */
uint64_t dgx_lane_launches(const dgx_lane* lane);

void* dgx_dev_alloc(size_t bytes);
void dgx_dev_free(void* d_ptr);
int dgx_memcpy_h2d(dgx_lane* lane, void* d_dst, const void* h_src, size_t bytes);
int dgx_memcpy_d2h(dgx_lane* lane, void* h_dst, const void* d_src, size_t bytes);

typedef enum dgx_setop { DGX_OP_INTERSECT = 0, DGX_OP_DIFFERENCE = 1 } dgx_setop;

/* Batched filter: query q keeps the values of its first list that are
 * (INTERSECT) present in every other list of the query / (DIFFERENCE, exactly
 * two lists) absent from the second.  Query q owns lists
 * [k_off[q], k_off[q+1]) of d_lists/lens.  For INTERSECT the library drives
 * from the shortest list, like IntersectSorted's length sort
 * (algo/uidlist.go:309-311).  Results are concatenated in query order into
 * d_out; d_out_off (nq + 1 device uint64) receives the CSR offsets.  If the
 * total exceeds out_cap nothing beyond it is written and the following
 * dgx_lane_sync returns DGX_ERR_CAP. */
int dgx_dev_filter_batch(dgx_lane* lane, int op,
                         const uint64_t* const* d_lists, const size_t* lens,
                         const size_t* k_off, size_t nq,
                         uint64_t* d_out, size_t out_cap, uint64_t* d_out_off);

/* MergeSorted on device lists.  d_out_len: one device uint64. */
int dgx_dev_merge_sorted(dgx_lane* lane, const uint64_t* const* d_lists, const size_t* lens, size_t k,
                         uint64_t* d_out, size_t out_cap, uint64_t* d_out_len);

/* A UidPack resident in HBM (deltas padded for 16-byte bulk copies, per-block
 * output offsets precomputed). */
typedef struct dgx_dev_pack dgx_dev_pack;
int dgx_dev_pack_upload(dgx_lane* lane, const dgx_pack_view* p, dgx_dev_pack** out);
void dgx_dev_pack_free(dgx_dev_pack* pk);
size_t dgx_dev_pack_exact_len(const dgx_dev_pack* pk);  /* codec.ExactLen */
size_t dgx_dev_pack_bytes(const dgx_dev_pack* pk);      /* bytes of the pack in HBM */
/* Decode(pack, seek) into d_out; d_out_len: one device uint64. */
int dgx_dev_decode(dgx_lane* lane, const dgx_dev_pack* pk, uint64_t seek,
                   uint64_t* d_out, size_t out_cap, uint64_t* d_out_len);
/* Device-resident form of dgx_intersect_compressed_rows: packs already in HBM (dgx_dev_pack_upload; NULL = empty
 * row), d_v / d_out / d_out_off (nrows + 1 values) device pointers.  Asynchronous on the lane; past out_cap nothing is
 * written and the next dgx_lane_sync returns DGX_ERR_CAP. */
int dgx_dev_intersect_compressed_rows(dgx_lane* lane, const dgx_dev_pack* const* packs, size_t nrows,
                                      uint64_t after_uid, const uint64_t* d_v, size_t m,
                                      uint64_t* d_out, size_t out_cap, uint64_t* d_out_off);
/* Device form of dgx_intersect_compressed_matrix: pack resident (dgx_dev_pack_upload; NULL = empty rows), d_v / d_out
 * / d_out_off (nrows + 1 values) device pointers, v_off in HOST memory (checked and staged by the call).  Asynchronous
 * on the lane: past out_cap nothing is written and the next dgx_lane_sync returns DGX_ERR_CAP; a row that does not
 * ascend strictly leaves d_out untouched, zeroes d_out_off and makes the next dgx_lane_sync return DGX_ERR_ARG. */
int dgx_dev_intersect_compressed_matrix(dgx_lane* lane, const dgx_dev_pack* pk, const uint64_t* d_v,
                                        const uint64_t* v_off, size_t nrows,
                                        uint64_t* d_out, size_t out_cap, uint64_t* d_out_off);
/* Device form of dgx_list_uids_rows: packs resident (dgx_dev_pack_upload; NULL = empty pack or delete-all marker),
 * d_mut_uids / d_mut_flags / d_v / d_out / d_out_off (nrows + 1 values) device pointers; mode and mut_off in HOST
 * memory, checked as in the host form before anything is queued.  Asynchronous on the lane: past out_cap nothing is
 * written and the next dgx_lane_sync returns DGX_ERR_CAP; a malformed mutable entry or a probe / iterate pack that
 * starts at uid 0 leaves d_out untouched, zeroes d_out_off and makes the next dgx_lane_sync return DGX_ERR_ARG. */
int dgx_dev_list_uids_rows(dgx_lane* lane, const dgx_dev_pack* const* packs, const uint8_t* mode, size_t nrows,
                           const uint64_t* d_mut_uids, const uint8_t* d_mut_flags, const uint64_t* mut_off,
                           uint64_t after_uid, const uint64_t* d_v, size_t m,
                           uint64_t* d_out, size_t out_cap, uint64_t* d_out_off);
/* Device forms of dgx_list_uids_unfiltered_rows and dgx_list_count_rows: packs resident (dgx_dev_pack_upload; NULL =
 * empty pack or delete-all marker), d_mut_uids / d_mut_flags / d_out / d_out_off (nrows + 1 values) / d_counts (nrows
 * values) device pointers; mut_off in HOST memory, checked as in the host forms before anything is queued.
 * Asynchronous on the lane: past out_cap nothing is written and the next dgx_lane_sync returns DGX_ERR_CAP; a malformed
 * mutable entry or a pack that starts at uid 0 leaves d_out untouched, zeroes d_out_off / d_counts and makes the next
 * dgx_lane_sync return DGX_ERR_ARG. */
int dgx_dev_list_uids_unfiltered_rows(dgx_lane* lane, const dgx_dev_pack* const* packs, size_t nrows,
                                      const uint64_t* d_mut_uids, const uint8_t* d_mut_flags, const uint64_t* mut_off,
                                      uint64_t after_uid, int32_t first,
                                      uint64_t* d_out, size_t out_cap, uint64_t* d_out_off);
int dgx_dev_list_count_rows(dgx_lane* lane, const dgx_dev_pack* const* packs, size_t nrows,
                            const uint64_t* d_mut_uids, const uint8_t* d_mut_flags, const uint64_t* mut_off,
                            uint64_t after_uid, uint32_t* d_counts);
/* Device form of dgx_merge_sorted_matrix: d_v and d_v_off (nrows + 1 values) are DEVICE pointers, so the
 * (d_out, d_out_off) of dgx_dev_intersect_compressed_rows / dgx_dev_filter_batch feed it directly.  v_cap >=
 * d_v_off[nrows] sizes the workspace (v_cap >= 2^32 is DGX_ERR_ARG).  d_out_len: one device uint64, the result length.
 * Asynchronous on the lane: past out_cap nothing is written and the next dgx_lane_sync returns DGX_ERR_CAP, as it does
 * when d_v_off[nrows] > v_cap; a row that descends makes the next dgx_lane_sync return DGX_ERR_ARG. */
int dgx_dev_merge_sorted_matrix(dgx_lane* lane, const uint64_t* d_v, const uint64_t* d_v_off, size_t nrows,
                                size_t v_cap, uint64_t* d_out, size_t out_cap, uint64_t* d_out_len);
/* Buckets of the matrix merges that were too large for shared memory and took the slower global-memory sort: of this
 * lane as of its last dgx_lane_sync, or of the whole process for lane == NULL.  Results do not depend on it. */
uint64_t dgx_merge_matrix_overflows(const dgx_lane* lane);
/* Intersection queries of 3+ lists whose sparse tail of lists was searched after the streaming pass (on a lane with
 * resident inputs, a sample of a driving list of at least 65536 values found few candidates reaching those lists): of
 * this lane as of its last dgx_lane_sync, or of the whole process for lane == NULL.  Results do not depend on it. */
uint64_t dgx_filter_tail_queries(const dgx_lane* lane);

#ifdef __cplusplus
}
#endif
#endif /* DGX_H */
