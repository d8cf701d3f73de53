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

/* The uid path of backup and restore over a task's keys, one call each: List.ToBackupPostingList writes
 * BackupPostingList.uid_bytes with codec.DecodeToBuffer (posting/list.go:1461-1482, codec/codec.go:456-467) and
 * FromBackupPostingList rebuilds the pack with codec.EncodeFromBuffer(uid_bytes, 256) (posting/list.go:2427-2441,
 * codec/codec.go:402-414).  uid_bytes is binary.PutUvarint(u - last) for every uid u of Decode(pack, 0), the subtraction
 * on uint64 (it wraps: a pack need not ascend), last starting at 0.  Decoding stops at the first block with NumUids 0, as
 * the reference's `for len(uids) > 0` loop does; dgx_decode is not changed by this.
 *
 * codec.DecodeToBuffer(pack_i) for every row: row i's bytes are out[out_off[i] .. out_off[i+1]).  refs[i] as in
 * dgx_intersect_compressed_rows (named packs use the HBM cache, anonymous ones cross PCIe together); a NULL / empty pack
 * gives no bytes.  out == NULL only sizes (out_off is filled; a device is still needed).  A result longer than out_cap
 * is DGX_ERR_CAP: nothing is written to out and out_off holds the exact offsets, so out_off[nrows] is the capacity that
 * makes one more call succeed.  DGX_ERR_ARG before anything is copied: a null array that is needed, a sum of ExactLen of
 * 2^32 or more, a malformed pack.  nrows == 0 gives out_off[0] = 0 and needs no device.  The call runs a fixed number of
 * kernel launches whatever nrows, the number of uids and the pack sizes are. */
int dgx_decode_to_buffer_rows(const dgx_pack_ref* refs, size_t nrows,
                              uint8_t* out, uint64_t* out_off, size_t out_cap);
/* codec.EncodeFromBuffer(buf_i, block_size) for every row: row i's input is buf[buf_off[i] .. buf_off[i+1]) (host
 * offsets, nrows + 1 values, buf_off[0] == 0), a value never continues into the next row.  Row i's pack is a flat image
 * (dgx_pack_image_view layout) at img + img_off[i] with nblocks[i] blocks and delta_bytes[i] delta bytes; an empty row
 * is the nil pack (nblocks 0, empty image).  The images are 16-byte aligned and back to back, so the result passed to
 * any pack entry point crosses PCIe as one transfer.  binary.Uvarint rules: a byte < 0x80 ends a value, non-minimal
 * encodings are accepted, a value has at most 10 bytes and its 10th is <= 1.  img == NULL only sizes (img_off, nblocks
 * and delta_bytes are filled; a device is still needed).  Images longer than img_cap are DGX_ERR_CAP: nothing is written
 * to img and the offset and size arrays hold the exact values.  DGX_ERR_ARG before anything is copied: buf_off[0] != 0,
 * decreasing offsets, buf_off[nrows] >= 2^32, a null array that is needed, img not 16-byte aligned.  DGX_ERR_ARG after
 * the kernels, with img untouched and img_off / nblocks / delta_bytes zeroed: a row that is not a sequence of valid
 * uvarints (a value of more than 10 bytes, a 10th byte > 1, a row that ends inside a value -- where the reference
 * panics or loops).  nrows == 0 gives img_off[0] = 0 and needs no device.  The call runs a fixed number of kernel
 * launches whatever nrows, the number of bytes and block_size are.  Workspace: the value, segment and block counts are
 * only known on the device, so the call reserves room for one of each per input byte, about 52 bytes of HBM per input
 * byte (5.2 GB for 100 MB of uid_bytes); a batch larger than the free HBM allows is DGX_ERR_OOM, and the caller splits
 * it by keys.  A lane of the host form whose workspace grew past 4 GiB gives it back when the call returns. */
int dgx_encode_from_buffer_rows(const uint8_t* buf, const uint64_t* buf_off, size_t nrows, uint32_t block_size,
                                void* img, size_t img_cap, uint64_t* img_off, uint64_t* nblocks, uint64_t* delta_bytes);

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

/* uidsForRegex(attr, arg, query, &pb.List{}) (worker/trigram.go:24-102): the cindex.Query tree of a regexp() over a
 * trigram index, every trigram's posting list read with List.Uids, evaluated in one call.  Node 0 is the root; node i
 * has op[i] (DGX_QAND or DGX_QOR, cindex's values), the leaves leaf_idx[leaf_off[i] .. leaf_off[i+1]) (its trigrams) and
 * the sub-nodes sub_idx[sub_off[i] .. sub_off[i+1]).  Every node but the root has exactly one parent and a larger index
 * than it; two nodes may name the same leaf. */
enum { DGX_QAND = 2, DGX_QOR = 3 };
typedef struct dgx_query_tree {
    size_t nnodes;
    const uint8_t* op;         /* nnodes */
    const uint32_t* leaf_off;  /* nnodes + 1, leaf_off[0] == 0 */
    const uint32_t* leaf_idx;  /* leaf_off[nnodes] */
    const uint32_t* sub_off;   /* nnodes + 1, sub_off[0] == 0 */
    const uint32_t* sub_idx;   /* sub_off[nnodes] */
} dgx_query_tree;
/* Leaves 0 .. npacks-1 are PACK leaves: refs[i] (NULL pack: empty list or delete-all marker) with its resolved layer
 * mut_uids / mut_flags[mut_off[i] .. mut_off[i+1]), exactly as row i of dgx_list_uids_unfiltered_rows; the layers hold
 * REF postings only (no DGX_MUT_VALUE).  Leaves npacks .. npacks+nlists-1 are LIST leaves: list j is
 * lists[list_off[j] .. list_off[j+1]) (host offsets, list_off[0] == 0), ascending and duplicate-free, a list the caller
 * decoded itself (a split list's pl.Uids, calculatedUids), which is above after_uid as such a read is.  With S_i the
 * unfiltered List.Uids row of pack leaf i from after_uid (First = MaxInt32) and the list itself for a list leaf, the
 * result is f(root) with f(leaf) = S_leaf, f(AND) = the intersection of its leaves and subs, f(OR) = their union: what
 * uidsForRegex returns whichever List.Uids branch each filtered read takes (DESIGN section 5).  *out_len values are
 * written, ascending.
 * Bounds: a pack leaf's is ExactLen + |mut|, a list leaf's its length; an AND's the minimum of its children's, an OR's
 * their sum.  out_cap < the root's bound is DGX_ERR_CAP before anything is copied; a root bound of 0 gives *out_len = 0
 * and needs no device.  DGX_ERR_ARG before anything is copied: nnodes == 0 or >= 2^16, npacks + nlists >= 2^16,
 * leaf_off[nnodes] >= 2^20, an op that is not DGX_QAND / DGX_QOR, an AND with no leaf and no sub (codesearch makes that
 * QAll), a node with a second parent, a sub index not above its parent's or past nnodes, a node deeper than 32 (the root
 * is depth 1), a leaf index past the leaves, a sum of leaf bounds of 2^32 or more, list_off not starting at 0 or
 * decreasing, a DGX_MUT_VALUE flag, the layer errors of dgx_list_uids_unfiltered_rows, a null array that is needed.
 * The kernel launches depend only on the plan's case: see DESIGN section 3.8. */
int dgx_trigram_query(const dgx_query_tree* tree, const dgx_pack_ref* refs, size_t npacks, const uint64_t* mut_uids,
                      const uint8_t* mut_flags, const uint64_t* mut_off, const uint64_t* lists, const uint64_t* list_off,
                      size_t nlists, uint64_t after_uid, uint64_t* out, size_t out_cap, size_t* out_len);

/* @groupby over one uid predicate (query/groupby.go formResult :208-221, formGroups, groupLess, fillGroupedVars): the
 * child's uid matrix inverted into groups `dest uid -> ascending source uids`, restricted to every parent row, in one
 * call.  Row i (v[v_off[i] .. v_off[i+1]), strictly ascending) belongs to source src[i] (src strictly ascending); parent
 * p is par[par_off[p] .. par_off[p+1]) (strictly ascending).  Row i takes part in parent p iff src[i] is in parent p, and
 * each of its values d then adds src[i] to parent p's group d.  dest (strictly ascending, child.DestUIDs) holds every
 * value of every row.
 * Output: parent p owns the groups grp_off[p] .. grp_off[p+1] (npar + 1 values), ordered by (size, key) ascending, which
 * is groupLess's order when every group has the same number of aggregates; group g has key keys[g] and its members
 * members[mem_off[g] .. mem_off[g+1]), ascending (mem_off has room for grp_cap + 1 values).  members == NULL: counts
 * only, nothing is written to members and mem_cap is not read.  *ngroups / *nmembers get the exact sizes (nmembers is
 * the number of restricted edges).  npar == 0, or no row value or parent value at all: zero groups, no device.
 * DGX_ERR_CAP, with the exact sizes and nothing else written: *ngroups > grp_cap, or *nmembers > mem_cap with members.
 * DGX_ERR_ARG with nothing written: nrows, npar or ndest of 2^32 or more, offsets not starting at 0, decreasing or
 * totalling 2^32 or more, a null array that is needed (checked on the host); src, a row, a parent row or dest not
 * strictly ascending, a row value not in dest, 2^32 restricted edges or more (checked on the device).
 * Launches: 11 + 3 (P1 + P2) with P1 = ceil((b_p + b_d) / 8), P2 = ceil((b_p + b_s) / 8), b_p, b_d and b_s the bit
 * widths of npar - 1, ndest - 1 and nrows (DESIGN section 3.9). */
int dgx_groupby_uid(const uint64_t* src, size_t nrows, const uint64_t* v, const uint64_t* v_off, const uint64_t* dest,
                    size_t ndest, const uint64_t* par, const uint64_t* par_off, size_t npar, uint64_t* keys,
                    uint64_t* grp_off, uint64_t* mem_off, size_t grp_cap, uint64_t* members, size_t mem_cap,
                    size_t* ngroups, size_t* nmembers);

/* @recurse with loop: false (query/recurse.go expandRecurse :96-135): the edges one sg.Attr has taken so far, kept in
 * device memory for the life of one recursion.  An edge is (from, to) with from = sg.SrcUIDs[i] and to a value of row
 * i.  Calls on one set are serialised by the library; different sets may be used concurrently.  A set that a
 * device-form step bound to a lane must be waited for (dgx_reach_size / dgx_reach_export) or destroyed before that
 * lane is destroyed: the set refers to the lane's stream until then. */
typedef struct dgx_reach_set dgx_reach_set;
/* A set holding the n edges (from[k], to[k]), which strictly ascend by (from, to); n == 0 makes an empty set.
 * DGX_ERR_ARG: n of 2^32 or more, a null array with n > 0, edges that do not strictly ascend. */
int dgx_reach_create(const uint64_t* from, const uint64_t* to, size_t n, dgx_reach_set** set);
void dgx_reach_destroy(dgx_reach_set* set);
/* The exact edge count; waits for the device-form steps queued on the set. */
int dgx_reach_size(dgx_reach_set* set, size_t* n);
/* The edges, ascending by (from, to), into from / to (room for cap each); *n gets the count.  Waits like
 * dgx_reach_size.  DGX_ERR_CAP with *n set and nothing written when the count exceeds cap. */
int dgx_reach_export(dgx_reach_set* set, uint64_t* from, uint64_t* to, size_t cap, size_t* n);
/* One sg of one level: row i (v[v_off[i] .. v_off[i+1]), strictly ascending) belongs to src[i] (strictly ascending).
 * dest == NULL: the sg has no filters; otherwise (strictly ascending, ndest values) updateUidMatrix first drops every
 * value not in dest.  Then every edge already in the set is dropped and the rest are added to it.  out / out_off get
 * the kept rows (out_off has nrows + 1 values; the kept count is out_off[nrows]) and dest_out / *dest_len their sorted
 * union (sg.DestUIDs).  nrows == 0 or no value at all keeps nothing and launches nothing.
 * DGX_ERR_ARG before anything is copied: a null array that is needed, v_off not starting at 0 or decreasing, nrows or
 * v_off[nrows] of 2^32 or more, or a set that could reach 2^32 edges; the set is bound to a lane with queued
 * device-form steps.  DGX_ERR_CAP before anything is copied: out_cap or dest_cap below v_off[nrows].  DGX_ERR_ARG
 * after the kernels: src, a row or dest not strictly ascending.  A refused step writes nothing to the outputs and
 * leaves the set unchanged.  Launches: 7 plus the matrix merge's 7 + max(1, ceil(log2 ceil(v_off[nrows] / 2048)))
 * (DESIGN section 3.10). */
int dgx_recurse_filter(dgx_reach_set* set, const uint64_t* src, size_t nrows, const uint64_t* v, const uint64_t* v_off,
                       const uint64_t* dest, size_t ndest, uint64_t* out, uint64_t* out_off, size_t out_cap,
                       uint64_t* dest_out, size_t dest_cap, size_t* dest_len);

/* shortest() with numpaths <= 1 and no facets, so every edge costs 1 (query/shortest.go expandOut :141-273 and
 * shortestPath :457-618): a breadth-first search held in device memory for the life of one query.  It keeps
 *   seen      the discovered nodes, each with its parent, the attr index of the hop into it and its level (From: 0);
 *   expanded  the sources that have had a kept edge (adjacencyMap's keys).
 * Level k's rules, which Go's Dijkstra loop reduces to at unit cost (DESIGN section 5):
 *   - a row value is kept iff it is in its sg's dest (updateUidMatrix); stats.edges counts the kept values of every sg
 *     (the level's numEdges: an edge held by two sgs counts twice);
 *   - a kept value not yet in seen is discovered at level k; its parent is the smallest source with a kept edge to it
 *     at this level, and its attr index is attr[s] of the largest sg index s holding (parent, node);
 *   - every source with a kept edge joins expanded, and sg s's next SrcUIDs are its dest minus expanded;
 *   - a source with a kept edge must be a node discovered at the previous level (at level 1: From), as every such
 *     source of Go's exec lists is; any other is refused, which also refuses a source already expanded.
 * Calls on one search are serialised by the library; different searches may be used concurrently.  A search that a
 * device-form level bound to a lane must be waited for (dgx_path_result) or destroyed before that lane is. */
typedef struct dgx_path_search dgx_path_search;
/* One level: nsg sgs in exec order.  Sg s has the child index attr[s], the sources src[src_off[s] .. src_off[s+1])
 * (strictly ascending), one row per source (row r = v[v_off[r] .. v_off[r+1]), strictly ascending) and its DestUIDs
 * dest[dest_off[s] .. dest_off[s+1]) (strictly ascending).  Host memory for dgx_path_expand, device memory for
 * dgx_dev_path_expand. */
typedef struct {
    size_t nsg;
    const uint32_t* attr;      /* nsg */
    const uint64_t* src_off;   /* nsg + 1 */
    const uint64_t* src;       /* src_off[nsg] */
    const uint64_t* v_off;     /* src_off[nsg] + 1 */
    const uint64_t* v;         /* v_off[src_off[nsg]] */
    const uint64_t* dest_off;  /* nsg + 1 */
    const uint64_t* dest;      /* dest_off[nsg] */
} dgx_path_level;
/* edges: the level's numEdges; discovered: the nodes it reached first; to_level: To's level, 0 while unreached. */
typedef struct {
    uint64_t edges, discovered, to_level;
} dgx_path_stats;
/* A search from `from` to `to`: seen = {from at level 0}, expanded empty.  DGX_ERR_ARG: a uid of 0, or from == to. */
int dgx_path_create(uint64_t from, uint64_t to, dgx_path_search** ps);
void dgx_path_destroy(dgx_path_search* ps);
/* Expands one level (the rules above) and returns each sg's next SrcUIDs as CSR over the sgs: next_off has nsg + 1
 * values, next[next_off[s] .. next_off[s+1]).  Each input array is copied to the device once.
 * DGX_ERR_ARG before anything is copied: a null array that is needed, nsg of 0, offsets not starting at 0 or
 * decreasing, nsg, rows, values or dests of 2^32 or more, a search that could reach 2^32 nodes.  DGX_ERR_CAP before
 * anything is copied: next_cap below dest_off[nsg].  DGX_ERR_ARG after the kernels: src, a row or a dest not strictly
 * ascending, or a source with a kept edge not discovered at the previous level.  A refused level writes nothing to the outputs and
 * leaves the search unchanged.  Launches: 11 plus two matrix merges of 7 + max(1, ceil(log2 ceil(n / 2048))) each,
 * with n = max(1, values) and max(1, rows) (DESIGN section 3.12), whatever the sg count and the set sizes. */
int dgx_path_expand(dgx_path_search* ps, const dgx_path_level* level, uint64_t* next, uint64_t* next_off,
                    size_t next_cap, dgx_path_stats* stats);
/* Waits for the search's queued levels and returns the path From .. To: uids[0 .. len) and attrs[0 .. len - 1) (attrs[i]
 * is the attr index of the hop into uids[i + 1]), both with room for cap.  len is To's level + 1, or 0 when To was not
 * reached.  DGX_ERR_CAP with *len set and nothing written when len exceeds cap.  One launch. */
int dgx_path_result(dgx_path_search* ps, uint64_t* uids, uint32_t* attrs, size_t cap, size_t* len);

/* Value variables (query/query.go): a value map is key[n] (strictly ascending uids) with val[n], 64-bit words that are
 * int64 two's-complement patterns (DGX_VAL_INT64) or IEEE binary64 patterns (DGX_VAL_FLOAT64); one type per map.
 * clamp is aggregator.Value's: +Inf -> MaxFloat64, -Inf -> -MaxFloat64, NaN -> +0.0. */
#define DGX_VAL_INT64 1
#define DGX_VAL_FLOAT64 2
#define DGX_AGG_MIN 0
#define DGX_AGG_MAX 1
#define DGX_AGG_SUM 2
#define DGX_AGG_AVG 3
/* One level of a path, a node curNode: row i (v[v_off[i] .. v_off[i+1]), in stored order, not necessarily ascending)
 * belongs to src[i] (curNode.SrcUIDs, strictly ascending); dest (curNode.DestUIDs, strictly ascending) holds every row
 * value.  Host memory for dgx_var_propagate, device memory for dgx_dev_var_propagate.  v_cap is the room of v, read by
 * the device form only (the host form reads v_off[nrows]). */
typedef struct {
    const uint64_t* src;    /* nrows */
    const uint64_t* v_off;  /* nrows + 1 */
    const uint64_t* v;
    const uint64_t* dest;   /* ndest */
    size_t nrows, v_cap, ndest;
} dgx_var_level;
/* transformTo (query/query.go :1143-1236) over the levels in path order (len(fromNode.path) to the end, index 0
 * skipped): the map at the last level into out_key / out_val (ascending keys, the input's type) and *out_len.  Each
 * level: row i contributes iff src[i] is a key of the current map, and then each of its values dst receives
 * curVal = map[src[i]].  int64: a wrapping sum.  float64: the rows split into Go's 4 ranges (width = nrows / 4, the
 * last to nrows); within a range dst's contributions in row-major order fold as v = clamp(curVal), then
 * v = clamp(curVal + v); the ranges then combine in ascending order, acc = clamp(acc + part) (the chunks finishing in
 * index order).  Intermediate maps stay on the device.  n == 0 gives *out_len = 0 and needs no device.
 * out_cap >= the last level's ndest always suffices; a longer result is DGX_ERR_CAP with *out_len set and nothing
 * written.  DGX_ERR_ARG before anything is copied: an unknown type, nlevels of 0, n, nlevels, nrows, v_off[nrows] or
 * ndest of 2^32 or more, v_off not starting at 0 or decreasing, a null array that is needed.  DGX_ERR_ARG after the
 * kernels, with nothing written: map keys, src or dest not strictly ascending, a row value not in its level's dest.
 * Launches: 9 + 3 ceil((b_d + 2) / 8) per level, b_d the bit width of the level's ndest - 1 (DESIGN section 3.13). */
int dgx_var_propagate(int type, const uint64_t* key, const uint64_t* val, size_t n, const dgx_var_level* levels,
                      size_t nlevels, uint64_t* out_key, uint64_t* out_val, size_t out_cap, size_t* out_len);
/* evalLevelAgg's per-row branch (query/query.go :1088-1123): for every row i with at least one value present in the
 * map, key src[i] and the fold of its present values in row order, as aggregator.Apply does: MIN acc = acc < x ? acc : x
 * and MAX acc = acc < x ? x : acc (the later of equal values wins), SUM a wrapping int64 add or sequential IEEE adds,
 * AVG the sum over the count in float64 (an int64 sum through float64(int64)); clamp once on float results.  Output
 * type: DGX_VAL_FLOAT64 for AVG, the input type otherwise.  Row i is v[v_off[i] .. v_off[i+1]); src strictly ascends,
 * so the keys come out ascending.  out_cap >= nrows always suffices; a longer result is DGX_ERR_CAP with *out_len set
 * and nothing written.  n == 0 or no row value gives *out_len = 0 and needs no device.  DGX_ERR_ARG before anything is
 * copied: an unknown type or fn, n, nrows or v_off[nrows] of 2^32 or more, v_off not starting at 0 or decreasing, a
 * null array that is needed.  DGX_ERR_ARG after the kernels, with nothing written: map keys or src not strictly
 * ascending.  4 launches. */
int dgx_var_level_agg(int type, int fn, const uint64_t* key, const uint64_t* val, size_t n, const uint64_t* src,
                      size_t nrows, const uint64_t* v_off, const uint64_t* v, uint64_t* out_key, uint64_t* out_val,
                      size_t out_cap, size_t* out_len);

/* math() over value variables (query/math.go evalMathTree, with transformVars' leaf rule and valueVarAggregation's
 * math branch, query/query.go :1239-1361).  Entries of a math() map carry a tag each: DGX_VAL_INT64, DGX_VAL_FLOAT64,
 * DGX_VAL_BOOL (word 0 or 1, from comparisons) or DGX_VAL_NIL (Go's Val{}, from cond; word 0). */
#define DGX_VAL_BOOL 3
#define DGX_VAL_NIL 4
/* Ops of a dgx_math_node: a leaf (CONST, VAR), binary (ADD .. MAX), unary (NEG .. CEIL), comparison (LT .. NE) and
 * the ternary COND.  ln, exp, pow, logbase, since and dot are not offered: their Go results are not fixed by IEEE 754
 * or depend on the clock or on vector types. */
#define DGX_MATH_CONST 0
#define DGX_MATH_VAR 1
#define DGX_MATH_ADD 2
#define DGX_MATH_SUB 3
#define DGX_MATH_MUL 4
#define DGX_MATH_DIV 5
#define DGX_MATH_MOD 6
#define DGX_MATH_MIN 7
#define DGX_MATH_MAX 8
#define DGX_MATH_NEG 9
#define DGX_MATH_SQRT 10
#define DGX_MATH_FLOOR 11
#define DGX_MATH_CEIL 12
#define DGX_MATH_LT 13
#define DGX_MATH_GT 14
#define DGX_MATH_LE 15
#define DGX_MATH_GE 16
#define DGX_MATH_EQ 17
#define DGX_MATH_NE 18
#define DGX_MATH_COND 19
/* A program holds at most DGX_MATH_MAX_NODES nodes and DGX_MATH_MAX_LEAVES leaves: the evaluation keeps one tag and
 * one word per node for every key in thread-local storage and the node table in shared memory, and the leaves are the
 * rows of one key-union merge.  math() expressions in queries have a handful of nodes; a larger one stays in Go. */
#define DGX_MATH_MAX_NODES 64
#define DGX_MATH_MAX_LEAVES 16
/* One node; nodes are in post-order (children before parents, the root last).  child[0 .. arity) index earlier nodes
 * (arity 2 for binary and comparison ops, 1 for unary, 3 for COND, 0 for leaves).  VAR reads leaves[leaf]; several VAR
 * nodes may share a leaf.  CONST is the literal (const_tag DGX_VAL_INT64 or DGX_VAL_FLOAT64, const_word its word). */
typedef struct {
    uint8_t op;
    uint8_t const_tag;
    uint16_t child[3];
    uint32_t leaf;
    uint64_t const_word;
} dgx_math_node;
/* One variable's map after transformTo: key[0 .. n) strictly ascending, word[n], and either tag[n] (one DGX_VAL_* per
 * entry, a previous math() output) or tag NULL and every entry of type `type` (DGX_VAL_INT64 or DGX_VAL_FLOAT64, a
 * dgx_var_propagate output).  nil = 1 is a variable with no map at all (Go's nil ShardedMap), which cond tells apart
 * from an empty one; a nil leaf has no entries.  Host form: n is the entry count.  Device form: n is the room of the
 * arrays and d_len, when not NULL, one device uint64 whose low 32 bits hold the entry count (at most n), so the
 * d_out_len of dgx_dev_var_propagate or dgx_dev_var_level_agg, or the info word of a previous dgx_dev_math_eval, feeds
 * a leaf without a host read. */
typedef struct {
    const uint64_t* key;
    const uint64_t* word;
    const uint8_t* tag;
    const uint64_t* d_len;
    size_t n;
    int type;
    int nil;
} dgx_math_leaf;
/* The info word of a result: its length (low 32 bits), its kind (bits 32-39) and the set of tags in it (bits 40-47,
 * bit 1 << t for DGX_VAL_ t).  MAP: a non-empty map, Go's UidToVal.  CONST: a constant set for every uid of the range
 * (or on uid 0 when there is no range).  NONE: no map and no constant; Go assigns nothing. */
#define DGX_MATH_KIND_NONE 0
#define DGX_MATH_KIND_MAP 1
#define DGX_MATH_KIND_CONST 2
#define DGX_MATH_INFO_LEN(w) ((uint64_t)(w) & 0xffffffffull)
#define DGX_MATH_INFO_KIND(w) ((int)(((uint64_t)(w) >> 32) & 0xff))
#define DGX_MATH_INFO_TAGS(w) ((unsigned)(((uint64_t)(w) >> 40) & 0xff))
/* evalMathTree over prog[0 .. nnodes) and valueVarAggregation's math branch: the result map into out_key / out_word /
 * out_tag (ascending keys) and *info.  Go's rules, bit for bit: a leaf {MaxUint64: v} is the constant v; at a binary
 * node a child {0: v} becomes a constant (the left child first, the right only when the left did not); a binary node
 * over maps ranges over the union of their keys, a missing entry or a nil value being int64 0, and drops a key whose
 * operation fails; int op float converts the int; int + - * / overflow and division by zero fail; / and % by zero
 * fail; MinInt64 / -1 is MinInt64 and MinInt64 % -1 is 0; float % is math.Mod; min / max take the left operand unless
 * it is less (a NaN makes min take the right, max the left); u- MinInt64, sqrt of a negative value fail; sqrt of an int
 * is a float, floor / ceil of an int the int; Value()'s clamp (+Inf -> MaxFloat64, -Inf -> -MaxFloat64, NaN -> +0.0)
 * follows every binary and unary result.  A comparison ranges over its left child's keys, a missing right entry being
 * nil; ints meet floats as floats, nil compared with nil is neither ordered nor equal.  cond ranges over its first
 * child's keys, and a missing branch entry is stored as a nil value.  At the top a map holding both ints and floats
 * has its ints converted to float; a constant is set on every uid of range (range NULL: on uid 0, nrange ignored).
 * out_cap >= the sum of the leaves' n plus 1, and >= nrange, always suffices; a longer result is DGX_ERR_CAP with
 * *info set and nothing written.
 * DGX_ERR_ARG before anything is copied: a malformed program (an unknown op or constant tag, a child not earlier in
 * post-order, a leaf index out of range, more than DGX_MATH_MAX_NODES nodes or DGX_MATH_MAX_LEAVES leaves), a leaf's
 * unknown type, a nil leaf with entries, sizes of 2^32 or more, a null array that is needed.
 * DGX_ERR_ARG after the kernels, with nothing written, where Go's answer is an error or depends on map iteration order:
 * evalMathTree failing (an operation on two constants or a unary one on a constant failing, cond over a constant or a
 * nil map), a unary, comparison or cond node failing on some but not all of more than one key, a leaf holding key 0
 * with other keys, leaf keys or range not strictly ascending, an unknown entry tag.
 * Launches: 7 plus the key-union merge's (DESIGN section 3.14), whatever the tree and map sizes. */
int dgx_math_eval(const dgx_math_node* prog, size_t nnodes, const dgx_math_leaf* leaves, size_t nleaves,
                  const uint64_t* range, size_t nrange, uint64_t* out_key, uint64_t* out_word, uint8_t* out_tag,
                  size_t out_cap, uint64_t* info);

/* @cascade over a forest of subgraph nodes (query/query.go populateVarMap :1445-1527, updateUidMatrix :1425-1439
 * without facets, and ProcessQuery's root pagination :3004-3011), in pre-order: parent[n] is UINT32_MAX for a query root
 * and below n otherwise.  flags[n] is a set of DGX_CASCADE_* bits resolved on the host; first[n] / offset[n] are
 * Params.Cascade.First / Offset; counts_len[n] is len(n.counts). */
#define DGX_CASCADE_CASCADE 1u  /* len(Params.Cascade.Fields) > 0 */
#define DGX_CASCADE_CHECKED 2u  /* the parent's cascade consults it: listed or __all__, Attr != "uid", not internal */
#define DGX_CASCADE_FILTERED 4u /* len(Filters) > 0 */
#define DGX_CASCADE_ORDERED 8u  /* Order or FacetsOrder: rows not uid-sorted */
#define DGX_CASCADE_SKIP 16u    /* IsGroupBy() or the shortest alias: populateVarMap does nothing; it has no children */
typedef struct dgx_cascade_tree {
    size_t nnodes;
    const uint32_t* parent;       /* nnodes */
    const uint8_t* flags;         /* nnodes */
    const int32_t* first;         /* nnodes */
    const int32_t* offset;        /* nnodes */
    const uint64_t* counts_len;   /* nnodes */
} dgx_cascade_tree;
/* Node n has dest[dest_off[n] .. dest_off[n+1]) (n.DestUIDs, strictly ascending), the rows row_off[n] .. row_off[n+1]
 * of the forest's uid matrix (row r is v[v_off[r] .. v_off[r+1]); its i-th row belongs to parent.dest[i], and rows past
 * the last count as empty) and has_val[hv_off[n] .. hv_off[n+1]) (nonzero iff valueMatrix[i] has values; missing bytes
 * count as zero).  Rows of a node without DGX_CASCADE_ORDERED strictly ascend.  Post-order, every node:
 *   FILTERED and not SKIP: its rows are filtered by its dest;
 *   every CASCADE child: its rows are filtered by its dest as it stands after its own step, then cut by
 *     x.PageRange(first, offset, len);
 *   CASCADE and not SKIP: dest keeps dest[i] unless a CHECKED child has an empty or missing row i, a zero or missing
 *     has_val byte i and i >= counts_len;
 * and a CASCADE root with first or offset has its rows filtered by its new dest and paged.  The filters keep row order.
 * out / out_off get every node's new rows (out_off has row_off[nnodes] + 1 values, node n's rows are rows row_off[n]
 * .. row_off[n+1]), dest_out / dest_out_off (nnodes + 1 values) every node's new dest.  out_cap >= v_off[row_off[nnodes]]
 * and dest_cap >= dest_off[nnodes] (the bounds) are required: DGX_ERR_CAP before anything is copied otherwise.
 * DGX_ERR_ARG before anything is copied: nnodes >= 2^16, a parent not below its child, an unknown flag bit, a SKIP node
 * with a child, a node deeper than 63 (64 levels), offsets not starting at 0 or decreasing, 2^32 or more rows, values or
 * dest values in all, a null array that is needed.  DGX_ERR_ARG after the kernels, with nothing written to the outputs:
 * a dest, or a row of a node without ORDERED, that does not strictly ascend.  nnodes == 0, or a forest without a dest
 * value and a row value, writes zero offsets and needs no device.  Launches: 4 + 7 * D, D the levels holding a dest or
 * a row value (DESIGN section 3.11). */
int dgx_cascade(const dgx_cascade_tree* tree, const uint64_t* v, const uint64_t* v_off, const uint64_t* row_off,
                const uint64_t* dest, const uint64_t* dest_off, const uint8_t* has_val, const uint64_t* hv_off,
                uint64_t* out, uint64_t* out_off, size_t out_cap, uint64_t* dest_out, uint64_t* dest_out_off,
                size_t dest_cap);

/* A subgraph's @filter tree and first / offset (query/query.go ProcessGraph :2310-2413: filterCopy's tree, the filter
 * block, applyPagination :2492-2507 with updateUidMatrix :1425-1439 and x.PageRange, and the DoCount block), without
 * order or facets.  d0 is the node's DestUIDs from processTask (strictly ascending) and row i of its uid matrix is
 * v[v_off[i] .. v_off[i+1]) (strictly ascending, v_off[0] == 0).  The tree is flat: node 0 is the root and parent[k] <
 * k for every other node (parent[0] is ignored); op[k] is DGX_SGF_AND, _OR or _NOT (exactly one child; AND and OR have
 * at least one) or DGX_SGF_LEAF, which reads leaves[leaf[k]] (several nodes may share a leaf).  Children keep index
 * order.  At most DGX_SGF_MAX_NODES nodes and DGX_SGF_MAX_LEAVES leaves, and a node at most DGX_SGF_MAX_DEPTH below
 * the root: filter trees in queries have a handful of nodes, a larger one stays in Go. */
#define DGX_SGF_LEAF 0
#define DGX_SGF_AND 1
#define DGX_SGF_OR 2
#define DGX_SGF_NOT 3
#define DGX_SGF_MAX_NODES 1024
#define DGX_SGF_MAX_LEAVES 1024
#define DGX_SGF_MAX_DEPTH 64
typedef struct dgx_sg_filter_tree {
    size_t nnodes;
    const uint8_t* op;        /* nnodes */
    const uint32_t* parent;   /* nnodes */
    const uint32_t* leaf;     /* nnodes: the leaf of a DGX_SGF_LEAF node */
} dgx_sg_filter_tree;
/* A leaf, resolved on the host to one of two kinds:
 *   DGX_SGF_LIST: uids[0 .. n), strictly ascending (a function leaf's DestUIDs, uid(var), a literal uid(...) list, or
 *     d0 / nothing for gt(len(x), n)).  Device form: d_len, when set, is a device word whose low 32 bits hold the length
 *     (at most n, then the room), so the d_out_len of dgx_dev_merge_sorted_matrix or dgx_dev_trigram_query feeds it.
 *   DGX_SGF_COUNT: d0[i] is in the set iff evalCompare(cmp, c_i, threshold) (worker/compare.go, int64), with c_i =
 *     counts[i] (a count per d0 value, as dgx_list_count_rows writes) or off[i + 1] - off[i] (row lengths, as the
 *     d_out_off of dgx_list_uids_rows over d0's keys): exactly one of counts / off is set.  cmp is DGX_SGF_CMP_*. */
#define DGX_SGF_LIST 0
#define DGX_SGF_COUNT 1
#define DGX_SGF_CMP_LE 0
#define DGX_SGF_CMP_GE 1
#define DGX_SGF_CMP_LT 2
#define DGX_SGF_CMP_GT 3
#define DGX_SGF_CMP_EQ 4
typedef struct dgx_sg_filter_leaf {
    int kind;
    int cmp;
    int64_t threshold;
    const uint64_t* uids;
    size_t n;
    const uint64_t* d_len;
    const uint32_t* counts;
    const uint64_t* off;
} dgx_sg_filter_leaf;
/* With f(LIST) its uids, f(COUNT) the d0 values it holds, f(AND) / f(OR) the intersection / union of the children and
 * f(NOT) = d0 minus its child: D1 = f(root) ∩ d0.  Then each row becomes row ∩ D1 and, when count or offset is not 0,
 * is cut to x.PageRange(count, offset, len); the new dest is D1 without pagination and MergeSorted(rows) with it.
 * Writes the new dest to dest_out (*dest_len values), the rows to out / out_off (nrows + 1 offsets) and counts[i] =
 * len(row i) (the DoCount block; pass count = offset = 0 for DoCount with an order).  out == NULL is counts-only mode:
 * no row value is written.  dest_cap >= n0 and, unless out is NULL, out_cap >= v_off[nrows] are required:
 * DGX_ERR_CAP before anything is copied otherwise.  DGX_ERR_ARG before anything is copied: a malformed tree (an
 * unknown op, a parent not below its child or a leaf node as parent, NOT without exactly one child, AND / OR without
 * one, a leaf index past nleaves, the limits above), a leaf's unknown kind or cmp, a COUNT leaf without exactly one of
 * counts / off, n0, nrows, v_off[nrows] or a list length of 2^32 or more, v_off not starting at 0 or decreasing, a null
 * array that is needed.  DGX_ERR_ARG after the kernels, with nothing written: d0, a row or a LIST leaf that does not
 * strictly ascend, or a COUNT leaf's off that decreases.  n0 == 0 writes zero lengths and needs no device.
 * Launches: 11 (DESIGN section 3.15), whatever the rows, values, n0, leaves and tree. */
int dgx_sg_filter(const dgx_sg_filter_tree* tree, const dgx_sg_filter_leaf* leaves, size_t nleaves, const uint64_t* d0,
                  size_t n0, const uint64_t* v, const uint64_t* v_off, size_t nrows, int32_t count, int32_t offset,
                  uint64_t* dest_out, size_t dest_cap, size_t* dest_len, uint64_t* out, uint64_t* out_off,
                  size_t out_cap, uint32_t* counts);

/* orderasc / orderdesc by a value variable (query/query.go applyOrderAndPagination :2511-2530, value-variable branch:
 * updateUidMatrix's order branch :1425-1439, sortAndPaginateUsingVar :2697-2738 and updateDestUids :2594-2609), in
 * Go's exact order.  dest is the node's DestUIDs after its filters (strictly ascending, e.g. dgx_sg_filter's new dest)
 * and row i of its uid matrix is v[v_off[i] .. v_off[i+1]) (strictly ascending, v_off[0] == 0).  var is the variable's
 * map as dgx_math_eval takes a leaf: a dgx_var_propagate / dgx_var_level_agg output (tag NULL, type DGX_VAL_INT64 or
 * DGX_VAL_FLOAT64) or a dgx_math_eval output (one DGX_VAL_* tag per entry); var->nil is Go's nil map.
 * Each row keeps, in row order, its uids in dest (U); W is U's uids with a map entry, in row order.  A row with an
 * empty W stays U.  Otherwise it becomes W sorted by types.Sort(values, &uids, []bool{desc}, ""): sort.Sort(byValue),
 * Go's pdqsort with its tie order, under byValue.Less (both nil: desc; one nil sorts last; equal values are not less,
 * -0.0 equals +0.0 and a NaN is neither less nor equal; otherwise types.less, mismatchedLess between int and float or
 * by Go's type id, negated for desc).  When count or offset is not 0 every row is then cut to x.PageRange(count,
 * offset, len), a negative count taking items from the back.  The new dest is the dest values some row still holds.
 * Writes the rows to out / out_off (nrows + 1 offsets) and the new dest to dest_out (*dest_len values).
 * DGX_ERR_ARG before anything is copied: a nil map (Go's "used before definition"), a tagless map of another type,
 * d_len set in the host form, var->n, ndest, nrows or v_off[nrows] of 2^32 or more, v_off not starting at 0 or
 * decreasing, a null array that is needed.  DGX_ERR_CAP before anything is copied: out_cap below v_off[nrows] or
 * dest_cap below ndest.  DGX_ERR_ARG after the kernels, with nothing written but *dest_len = 0: map keys, dest or a row
 * not strictly ascending, an unknown entry tag, or a row whose first W entry is a bool (Go's "isn't sortable").
 * ndest == 0 or nrows == 0 writes zero offsets and *dest_len = 0 and needs no device.
 * Launches: 37 + 3 ceil(b_r / 8), b_r the bit width of nrows - 1 (DESIGN section 3.16), whatever the values, ties, map
 * size and the rows' tiers. */
int dgx_var_order(const dgx_math_leaf* var, int desc, const uint64_t* dest, size_t ndest, const uint64_t* v,
                  const uint64_t* v_off, size_t nrows, int32_t count, int32_t offset, uint64_t* out, uint64_t* out_off,
                  size_t out_cap, uint64_t* dest_out, size_t dest_cap, size_t* dest_len);

/* A string value column: the values Go's loop reads at ReadTs for one predicate, built by the caller.  uid[0 .. n) are
 * strictly ascending, the uids that have a value; uid i owns values val_off[i] .. val_off[i+1) (n + 1 offsets,
 * val_off[0] == 0, val_off[n] == nvals); value j is bytes[byte_off[j] .. byte_off[j+1]) (nvals + 1 offsets,
 * byte_off[0] == 0, byte_off[nvals] == nbytes), any bytes, valid UTF-8 or not.  A uid that is absent has no value
 * (posting.ErrNoValue); a uid with several values is a list predicate's.  The column may hold more uids than a call's
 * candidates: one column per predicate can stay resident across calls until the predicate changes. */
typedef struct dgx_str_column {
    const uint64_t* uid;
    const uint64_t* val_off;
    const uint64_t* byte_off;
    const uint8_t* bytes;
    size_t n;
    size_t nvals;
    size_t nbytes;
} dgx_str_column;

/* The longest query dgx_match takes, in runes. */
#define DGX_MATCH_MAX_RUNES 4096

/* match(attr, query, max) (worker/task.go handleMatchFunction :1526-1620, uidsForMatch and matchFuzzy /
 * levenshteinDistance in worker/match.go :24-100).  The candidates are uids[0 .. nuids) when nuids > 0 (the filter's
 * UidList, strictly ascending); otherwise the union of every trigram row, the leaves taken exactly as
 * dgx_trigram_query takes them (refs / npacks with their layers, list leaves, after_uid) under one OR: uidsForMatch's
 * List.Uids reads with First = MaxInt32 and algo.MergeSorted.  No leaf (a query shorter than 3 bytes) is no candidate.
 * A candidate is kept when one of its values in col is not empty and lies within max edits of the query, the
 * unit-cost edit distance between Go's []rune conversions of both (an invalid UTF-8 byte is one U+FFFD, equal to a
 * genuine U+FFFD).  Writes the kept candidates in ascending order to out (*out_len values).
 * DGX_ERR_ARG before anything is copied: max < 0 or above 2^31 - 1; a query of more than DGX_MATCH_MAX_RUNES runes;
 * nuids, col->n, col->nvals, col->nbytes or the leaves' bounds of 2^32 or more; column offsets not starting at 0,
 * decreasing or not ending at nvals / nbytes; a null array that is needed; the layer errors of
 * dgx_list_uids_unfiltered_rows, a DGX_MUT_VALUE entry included.  DGX_ERR_CAP before anything is copied: out_cap
 * below the candidates' bound (nuids, or the sum of the leaves' bounds).  DGX_ERR_ARG after the kernels, with
 * nothing written but *out_len = 0: candidates or column uids not strictly ascending.
 * Launches: 5, after the trigram stages of dgx_trigram_query for one OR node in the trigram branch, whatever the
 * candidates, the column, the value lengths and max (DESIGN section 3.17). */
int dgx_match(const dgx_pack_ref* refs, size_t npacks, const uint64_t* mut_uids, const uint8_t* mut_flags,
              const uint64_t* mut_off, const uint64_t* lists, const uint64_t* list_off, size_t nlists,
              uint64_t after_uid, const uint64_t* uids, size_t nuids, const dgx_str_column* col, const uint8_t* query,
              size_t query_len, int64_t max, uint64_t* out, size_t out_cap, size_t* out_len);

/* regexp()'s pattern compiled for dgx_regex_match: a line-oriented byte DFA (DESIGN section 3.18).  It restates
 * codesearch's matcher over "(?m)" + pattern as Go's regexp/syntax parses it with Perl flags, for this subset:
 * literals and escapes (punctuation, \a \f \t \n \r \v, \xHH, \x{H..}), '.', bracket classes with ranges, negation,
 * \d \s \w \D \S \W and [:name:] / [:^name:] inside, the same Perl classes outside, groups ( ), (?: ), flag groups
 * (?flags) and (?flags: ) over i m s U with '-', alternation, * + ? and their lazy forms, {n} {n,} {n,m} up to 1000
 * (nested counts multiplying to at most 1000, as Go requires), ^ $ \A \z; under (?-m) ^ and $ are \A and \z, as
 * Go's OneLine makes them.  Under (?i) (or DGX_REGEX_FOLD, the /i
 * modifier) ASCII letters fold, with K U+212A and long s U+017F in the orbits of k and s; a folded literal or class item
 * holding any other non-ASCII rune is outside the subset.  A rune matches only its own well-formed UTF-8 bytes: an
 * invalid byte matches nothing, not even '.' or a negated class.  Everything else -- \p{..}, \b, \B, \Q..\E, octal
 * escapes, named groups, a '{' that is not a repeat count, stacked repetition operators, invalid UTF-8 in the pattern,
 * and every pattern Go rejects -- is DGX_ERR_ARG, so a caller can keep its own matcher for it.  A DFA of more than
 * DGX_REGEX_MAX_STATES states, a byte NFA past its own bound, or a construction past its work bound (which keeps the
 * host's compile time to tens of milliseconds before a caller falls back) is DGX_ERR_CAP.  The program is host memory,
 * immutable and shareable between threads and calls; dgx_regex_free releases it. */
#define DGX_REGEX_FOLD 1
#define DGX_REGEX_MAX_STATES 4096
typedef struct dgx_regex_prog dgx_regex_prog;
int dgx_regex_compile(const char* pattern, size_t len, int flags, dgx_regex_prog** prog);
void dgx_regex_free(dgx_regex_prog* prog);
/* The compiled tables, read-only and owned by prog: cls[256] maps a byte to its class, trans[s * nclasses + c] is the
 * next state, term[s] has bit 1 when s absorbs (0 dead, 1 accept) and bit 2 when a value ending in s matches.  A value
 * starts in state 2; '\n' leads every live state to 3, a later line's start, or to 0 / 1. */
int dgx_regex_tables(const dgx_regex_prog* prog, size_t* nstates, size_t* nclasses, const uint8_t** cls,
                     const uint16_t** trans, const uint8_t** term);

/* regexp(attr, /pattern/) (worker/task.go handleRegexFunction :1240-1356, matchRegex :1809-1811) over a string value
 * column.  The candidates are uids[0 .. nuids) when nuids > 0 (the filter's UidList, strictly ascending); otherwise
 * the union of the leaves, taken exactly as dgx_match takes them (uidsForRegex's trigram rows: the caller passes the
 * query's leaves; dgx_trigram_query evaluates a whole AND/OR tree, whose result is a UidList for this call).  A
 * candidate is kept when one of its values in col is not empty and prog matches it: some line of the value holds a
 * match, the first line only when it is not empty (codesearch reports that match at offset 0, which matchRegex counts
 * as none).  Writes the kept candidates in ascending order to out (*out_len values).  Refusals as dgx_match's, with
 * prog in place of the query: a null prog is DGX_ERR_ARG.  Launches: 5, after the trigram stages in the trigram
 * branch, whatever the candidates, the column, the value lengths and the program (DESIGN section 3.18). */
int dgx_regex_match(const dgx_pack_ref* refs, size_t npacks, const uint64_t* mut_uids, const uint8_t* mut_flags,
                    const uint64_t* mut_off, const uint64_t* lists, const uint64_t* list_off, size_t nlists,
                    uint64_t after_uid, const uint64_t* uids, size_t nuids, const dgx_str_column* col,
                    const dgx_regex_prog* prog, uint64_t* out, size_t out_cap, size_t* out_len);

/* A typed value column: the values of one predicate converted to its schema type, as Go's compare loops read them
 * (types.Convert of each stored value).  The layout is dgx_str_column's: uid[0 .. n) strictly ascending, uid i owning
 * values val_off[i] .. val_off[i+1) (n + 1 offsets, val_off[0] == 0, val_off[n] == nvals), several values per uid for a
 * list predicate, every count below 2^32.  type picks the value's form:
 *   DGX_VAL_INT64     word[j] is the int64
 *   DGX_VAL_FLOAT64   word[j] is the IEEE binary64 pattern
 *   DGX_VAL_BOOL      word[j] != 0 is true
 *   DGX_VAL_DATETIME  word[j] is the instant's Unix seconds (int64, negative before 1970), nsec[j] its nanoseconds
 *                     (below 10^9); the location is not part of the value, as time.Time.Before / Equal ignore it
 *   DGX_VAL_STRING    str is the column (a dgx_str_column, shared with match() and regexp()): uid, val_off, word,
 *                     nsec, n and nvals are unused and str's are taken
 * bad, when set, holds one byte per value: nonzero when the value's conversion to the schema type failed or gave nil. */
#define DGX_VAL_DATETIME 5
#define DGX_VAL_STRING 6
typedef struct dgx_val_column {
    int type;
    const uint64_t* uid;
    const uint64_t* val_off;
    const uint64_t* word;
    const uint32_t* nsec;
    const uint8_t* bad;
    const dgx_str_column* str;
    size_t n;
    size_t nvals;
} dgx_val_column;
/* A compare function's arguments, converted to the column's type (convertValue): n values given as a column's values
 * are (word[k], nsec[k] for DATETIME), or for DGX_VAL_STRING the bytes bytes[byte_off[k] .. byte_off[k+1)).  Host
 * memory in both forms. */
typedef struct dgx_val_args {
    const uint64_t* word;
    const uint32_t* nsec;
    const uint8_t* bytes;
    const uint64_t* byte_off;
    size_t n;
} dgx_val_args;
/* between(v, a, b): the compare op code past DGX_SGF_CMP_EQ.  dgx_sg_filter does not take it. */
#define DGX_SGF_CMP_BETWEEN 5

/* The compare functions eq / le / lt / ge / gt / between on the value path (worker/task.go handleValuePostings,
 * compareAttrFn branch :540-575, with types.CompareVals / CompareBetween, types/compare.go): candidate uids[i] (the
 * filter's UidList, strictly ascending) is tested against each of its values in col.  op is DGX_SGF_CMP_LE .. EQ or
 * DGX_SGF_CMP_BETWEEN; args holds 1 argument (le, lt, ge, gt), at least 1 (eq: a value equal to any one matches) or
 * exactly 2 (between a and b).  Go's rules: ge is !Less(v, a), le !Less(a, v), gt Less(a, v), lt Less(v, a), eq
 * Equal(v, a), between ge(v, a) && le(v, b), each false where Less / Equal returns an error.  So for float64 a NaN value
 * passes ge, le and between but not gt, lt or eq, a NaN argument makes ge / le true and gt / lt / eq false, and -0
 * equals +0; a bool passes eq only; strings compare bytewise, unsigned, a proper prefix less.  Writes the candidates
 * with at least one matching value in ascending order to out (*out_len values) and, when counts is set, counts[i] the
 * number of uids[i]'s matching values (the length of Go's result row i: a list value matching appends the uid once).
 * DGX_ERR_ARG before anything is copied: an unknown op or type, a wrong argument count, a DATETIME argument's
 * nanoseconds of 10^9 or more, nuids or the column's sizes of 2^32 or more, column offsets not starting at 0,
 * decreasing or not ending at nvals / nbytes, a null array that is needed.  DGX_ERR_CAP before anything is copied:
 * out_cap below nuids.  DGX_ERR_ARG after the kernels, with nothing written but *out_len = 0: candidates or column
 * uids not strictly ascending, or a candidate owning a bad value or a DATETIME value's nanoseconds of 10^9 or more (Go
 * returns the conversion error); such values of uids that are not candidates are not read.  nuids == 0 writes
 * *out_len = 0 and needs no device.  Launches: 5, whatever the candidates, the column, the values and the arguments
 * (DESIGN section 3.19). */
int dgx_compare_uids(int op, const dgx_val_args* args, const dgx_val_column* col, const uint64_t* uids, size_t nuids,
                     uint64_t* out, size_t out_cap, size_t* out_len, uint32_t* counts);
/* The compare functions on the index path (worker/task.go handleCompareFunction :1358-1524): the uid matrix
 * v[v_off[r] .. v_off[r+1]) of the index rows, rows in any order, filtered row by row.  row_arg[r] == UINT32_MAX
 * keeps row r as it is; otherwise a value of row r is kept when one of its values in col passes op against argument
 * row_arg[r] (between: arguments row_arg[r] and row_arg[r] + 1), a bad value (or an absent uid) never passing.  Go's
 * three cases are: eq, row r against eqTokens[r]; between, rows 0 and nrows - 1 against the pair; any other op, row 0
 * when tokens[0] == ineqValueToken[0].  Writes the kept values in row order to out and nrows + 1 offsets to out_off.
 * DGX_ERR_ARG before anything is copied: op, type and argument rules as dgx_compare_uids's (any argument count for eq,
 * 2 for between), a row_arg past the arguments, nrows, v_off[nrows] or the column's sizes of 2^32 or more, v_off not
 * starting at 0 or decreasing, the column's offsets, a null array that is needed.  DGX_ERR_CAP: out_cap below
 * v_off[nrows].  DGX_ERR_ARG after the kernels, with every offset 0 and no value written: column uids not strictly
 * ascending.  nrows == 0 writes out_off[0] = 0 and needs no device.  Launches: 4, whatever the rows, the column and the
 * arguments (DESIGN section 3.19). */
int dgx_compare_rows(int op, const dgx_val_args* args, const dgx_val_column* col, const uint64_t* v,
                     const uint64_t* v_off, size_t nrows, const uint32_t* row_arg, uint64_t* out, uint64_t* out_off,
                     size_t out_cap);

/* orderasc / orderdesc by a predicate whose values have no sortable index (query/query.go applyOrderAndPagination
 * :2511-2592, predicate branch, with worker/sort.go sortWithoutIndex :139-187: sortByValue :775-822, fetchValue and
 * paginate :740-773), in Go's exact order.  processSort returns sortWithoutIndex's answer whenever sortWithIndex
 * fails before reading, that is for a predicate with no index or no sortable tokenizer; for an indexed predicate its
 * answer is a race with the indexed sort, which this call does not restate.  dest, v and v_off are dgx_var_order's:
 * the node's DestUIDs (strictly ascending) and its uid matrix (strictly ascending rows, v_off[0] == 0).  col is the
 * predicate's typed value column (dgx_val_column) of type DGX_VAL_INT64, DGX_VAL_FLOAT64, DGX_VAL_DATETIME or
 * DGX_VAL_STRING, one value per uid (Go refuses to sort by a list predicate).
 * Each row keeps, in row order, its uids in dest (U).  W is U's uids with a value, N the rest: a uid absent from the
 * column, owning no value, or whose value is marked bad (fetchValue's error: no value, or a failed conversion).  The
 * row becomes W sorted by types.Sort(values, &uids, []bool{desc}, ""): sort.Sort(byValue), Go's pdqsort with its tie
 * order, under byValue.Less (equal values are not less; otherwise types.less, negated for desc: int64 <, float64 < with
 * -0 equal to +0 and a NaN neither less nor equal, datetime the instant, strings bytewise and unsigned with a proper
 * prefix less), followed by N in row order, unsorted; then it is cut to x.PageRange(count, offset, |U|).  The query
 * layer replaces a count of 0 with 1000 before processSort; this call applies the count it is given.  The new dest is
 * the dest values some row still holds.  Writes the rows to out / out_off (nrows + 1 offsets) and the new dest to
 * dest_out (*dest_len values).
 * DGX_ERR_ARG before anything is copied: a null column, DGX_VAL_BOOL (SortWithFacet refuses a bool as not sortable)
 * or an unknown type, count < 0 (processSort refuses it), ndest, nrows, v_off[nrows] or the column's sizes of 2^32 or
 * more, v_off or the column's offsets not starting at 0 or decreasing (and not ending at nvals / nbytes), a null
 * array that is needed.  DGX_ERR_CAP before anything is copied: out_cap below v_off[nrows] or dest_cap below ndest.
 * DGX_ERR_ARG after the kernels, with nothing written but *dest_len = 0: dest, a row or the column's uids not strictly
 * ascending, a U uid owning more than one value, or a U uid's datetime value with nanoseconds of 10^9 or more.  Bad
 * values, and the values of uids outside U, are not otherwise read.  ndest == 0 or nrows == 0 writes zero offsets and
 * *dest_len = 0 and needs no device.
 * Launches: 38 + 3 ceil(b_r / 8) for int64, float64 and string columns and 51 + 3 ceil(b_r / 8) for datetime, b_r the
 * bit width of nrows - 1 (DESIGN section 3.20), whatever the values, ties, column size and the rows' tiers. */
int dgx_pred_order(const dgx_val_column* col, int desc, const uint64_t* dest, size_t ndest, const uint64_t* v,
                   const uint64_t* v_off, size_t nrows, int32_t count, int32_t offset, uint64_t* out, uint64_t* out_off,
                   size_t out_cap, uint64_t* dest_out, size_t dest_cap, size_t* dest_len);

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
/* Device forms of dgx_decode_to_buffer_rows and dgx_encode_from_buffer_rows: packs resident (dgx_dev_pack_upload; NULL
 * = nil pack), d_out / d_out_off (nrows + 1 values) and d_buf / d_img / d_img_off (nrows + 1 values) / d_nblocks /
 * d_delta_bytes (nrows values) device pointers, buf_off in HOST memory, checked as in the host forms before anything is
 * queued.  d_out == NULL / d_img == NULL only size.  Asynchronous on the lane: past out_cap / img_cap nothing is written
 * to d_out / d_img, the offsets are exact and the next dgx_lane_sync returns DGX_ERR_CAP; a malformed uid_bytes row
 * leaves d_img untouched, zeroes d_img_off / d_nblocks / d_delta_bytes and makes the next dgx_lane_sync return
 * DGX_ERR_ARG. */
int dgx_dev_decode_to_buffer_rows(dgx_lane* lane, const dgx_dev_pack* const* packs, size_t nrows,
                                  uint8_t* d_out, size_t out_cap, uint64_t* d_out_off);
int dgx_dev_encode_from_buffer_rows(dgx_lane* lane, const uint8_t* d_buf, const uint64_t* buf_off, size_t nrows,
                                    uint32_t block_size, void* d_img, size_t img_cap, uint64_t* d_img_off,
                                    uint64_t* d_nblocks, uint64_t* d_delta_bytes);
/* Device form of dgx_merge_sorted_matrix: d_v and d_v_off (nrows + 1 values) are DEVICE pointers, so the
 * (d_out, d_out_off) of dgx_dev_intersect_compressed_rows / dgx_dev_filter_batch feed it directly.  v_cap >=
 * d_v_off[nrows] sizes the workspace (v_cap >= 2^32 is DGX_ERR_ARG).  d_out_len: one device uint64, the result length.
 * Asynchronous on the lane: past out_cap nothing is written and the next dgx_lane_sync returns DGX_ERR_CAP, as it does
 * when d_v_off[nrows] > v_cap; a row that descends makes the next dgx_lane_sync return DGX_ERR_ARG. */
int dgx_dev_merge_sorted_matrix(dgx_lane* lane, const uint64_t* d_v, const uint64_t* d_v_off, size_t nrows,
                                size_t v_cap, uint64_t* d_out, size_t out_cap, uint64_t* d_out_len);
/* Device form of dgx_trigram_query: packs resident (dgx_dev_pack_upload; NULL = empty pack or delete-all marker),
 * d_mut_uids / d_mut_flags / d_lists / d_out device pointers, d_out_len one device uint64; tree, mut_off and list_off in
 * HOST memory, checked as in the host form before anything is queued (the DGX_MUT_VALUE check runs on the device: such
 * a flag leaves d_out untouched, writes d_out_len = 0 and makes the next dgx_lane_sync return DGX_ERR_ARG, as a malformed
 * layer does).  Asynchronous on the lane; nothing waits on the host between the stages. */
int dgx_dev_trigram_query(dgx_lane* lane, const dgx_query_tree* tree, const dgx_dev_pack* const* packs, size_t npacks,
                          const uint64_t* d_mut_uids, const uint8_t* d_mut_flags, const uint64_t* mut_off,
                          const uint64_t* d_lists, const uint64_t* list_off, size_t nlists, uint64_t after_uid,
                          uint64_t* d_out, size_t out_cap, uint64_t* d_out_len);
/* Device form of dgx_groupby_uid: every array in device memory, offsets included, so the rows of
 * dgx_dev_list_uids_unfiltered_rows (and their dgx_dev_merge_sorted_matrix as d_dest) feed it directly.  v_cap and
 * par_cap are the room of d_v and d_par (d_v_off[nrows] and d_par_off[npar] must not pass them); e_cap is the room for
 * restricted edges the workspace holds (94 bytes each).  d_sizes is two device uint64: [ngroups, nmembers].  Sizes of
 * 2^32 or more and missing pointers are DGX_ERR_ARG at the call; npar, nrows, v_cap or par_cap of 0 writes zero groups
 * without a launch.  Every other check runs on the device and surfaces at the next dgx_lane_sync: a refused input
 * writes d_sizes = {0, 0} and nothing else (DGX_ERR_ARG); an output that does not fit writes the exact d_sizes and
 * nothing else (DGX_ERR_CAP); more than e_cap edges writes d_sizes = {0, edges} and nothing else (DGX_ERR_CAP).
 * Asynchronous on the lane. */
int dgx_dev_groupby_uid(dgx_lane* lane, const uint64_t* d_src, size_t nrows, const uint64_t* d_v,
                        const uint64_t* d_v_off, size_t v_cap, const uint64_t* d_dest, size_t ndest,
                        const uint64_t* d_par, const uint64_t* d_par_off, size_t npar, size_t par_cap, size_t e_cap,
                        uint64_t* d_keys, uint64_t* d_grp_off, uint64_t* d_mem_off, size_t grp_cap,
                        uint64_t* d_members, size_t mem_cap, uint64_t* d_sizes);
/* Device form of dgx_recurse_filter: every array in device memory, offsets included, so the rows of
 * dgx_dev_list_uids_unfiltered_rows feed it directly.  v_cap is the room of d_v (d_v_off[nrows] must not pass it) and
 * stands for v_off[nrows] in the host form's limits: out_cap and dest_cap below v_cap are DGX_ERR_CAP.  d_sizes is two
 * device uint64: {kept, dest_len}.  Sizes, missing pointers and a set bound to another lane (one whose queued steps no
 * dgx_reach_size or dgx_reach_export has waited for yet) are DGX_ERR_ARG at the call; nrows or v_cap of 0 writes
 * zero offsets and sizes without a launch.  Every other check (offsets, ascending src, rows and dest) runs on the
 * device: a refused step writes d_sizes = {0, 0}, nothing else, leaves the set unchanged and surfaces as DGX_ERR_ARG at
 * the next dgx_lane_sync.  Asynchronous on the lane: the set is bound to it until waited for.  Growing the set past its
 * capacity allocates device memory; DGX_ERR_OOM leaves the set unchanged. */
int dgx_dev_recurse_filter(dgx_lane* lane, dgx_reach_set* set, const uint64_t* d_src, size_t nrows, const uint64_t* d_v,
                           const uint64_t* d_v_off, size_t v_cap, const uint64_t* d_dest, size_t ndest,
                           uint64_t* d_out, uint64_t* d_out_off, size_t out_cap, uint64_t* d_dest_out,
                           size_t dest_cap, uint64_t* d_sizes);
/* Device form of dgx_path_expand: every array of *level in device memory, offsets and attr included, so the rows of
 * dgx_dev_list_uids_unfiltered_rows and the dest of dgx_dev_merge_sorted_matrix feed it directly.  src_cap, v_cap and
 * dest_cap are the room of src, v and dest (the offsets must end inside them) and stand for the host form's counts in
 * its limits: next_cap below dest_cap is DGX_ERR_CAP.  d_stats is three device uint64 {edges, discovered, to_level}.
 * Sizes, missing pointers and a search bound to another lane are DGX_ERR_ARG at the call.  Every other check
 * (offsets, ascending src, rows and dests, the level of sources with an edge) runs on the device: a refused level writes nothing, leaves
 * the search unchanged and surfaces as DGX_ERR_ARG at the next dgx_lane_sync.  Asynchronous on the lane: the search is
 * bound to it until waited for.  Growing the search past its capacity allocates device memory (24 bytes per node in
 * each of two buffers, reserved for min(v_cap, dest_cap) new nodes per queued level; 8 bytes per source in each of
 * two buffers, for src_cap per level); DGX_ERR_OOM leaves it unchanged.  Launches as the host form's with values = v_cap and rows = src_cap. */
int dgx_dev_path_expand(dgx_lane* lane, dgx_path_search* ps, const dgx_path_level* level, size_t src_cap,
                        size_t v_cap, size_t dest_cap, uint64_t* d_next, uint64_t* d_next_off, size_t next_cap,
                        uint64_t* d_stats);
/* Device form of dgx_var_propagate: the map, the outputs and every array of *levels (host array, nlevels entries) in
 * device memory, so the rows of dgx_dev_list_uids_unfiltered_rows and the dest of dgx_dev_merge_sorted_matrix feed it
 * directly.  v_cap is the room of a level's v (its v_off[nrows] must not pass it).  nrows and ndest are exact sizes
 * the host must know: a dest made by dgx_dev_merge_sorted_matrix has its length in a device word, which the caller
 * reads (one sync) before this call, since a dest padded to a cap does not strictly ascend and is refused.  d_out_len
 * is one device uint64.
 * Argument errors are DGX_ERR_ARG at the call, as in the host form (sizes, type, null pointers with a nonzero size);
 * n == 0 writes *d_out_len = 0 without a launch.  Offsets and the order and membership checks run on the device: a
 * refused call writes nothing and surfaces as DGX_ERR_ARG at the next dgx_lane_sync; a result longer than out_cap
 * writes only *d_out_len and surfaces as DGX_ERR_CAP.  Asynchronous on the lane; launches as the host form's. */
int dgx_dev_var_propagate(dgx_lane* lane, int type, const uint64_t* d_key, const uint64_t* d_val, size_t n,
                          const dgx_var_level* levels, size_t nlevels, uint64_t* d_out_key, uint64_t* d_out_val,
                          size_t out_cap, uint64_t* d_out_len);
/* Device form of dgx_var_level_agg: every array in device memory, offsets included; v_cap is the room of d_v.
 * Argument errors at the call as in the host form; n, nrows or v_cap of 0 writes *d_out_len = 0 without a launch.
 * Offsets, map keys and src are checked on the device: a refused call writes nothing (DGX_ERR_ARG at the next
 * dgx_lane_sync); a result longer than out_cap writes only *d_out_len (DGX_ERR_CAP).  Asynchronous on the lane. */
int dgx_dev_var_level_agg(dgx_lane* lane, int type, int fn, const uint64_t* d_key, const uint64_t* d_val, size_t n,
                          const uint64_t* d_src, size_t nrows, const uint64_t* d_v_off, const uint64_t* d_v,
                          size_t v_cap, uint64_t* d_out_key, uint64_t* d_out_val, size_t out_cap,
                          uint64_t* d_out_len);
/* Device form of dgx_math_eval: prog and leaves are host arrays, every array a leaf points to, d_range and the outputs
 * are device memory.  A leaf's entry count is *d_len when d_len is set (n its room), n otherwise; nrange is an exact
 * host size.  d_info is one device uint64.  Argument errors are DGX_ERR_ARG at the call, as in the host form; order,
 * tags, the count words and Go's errors are checked on the device: a refused call writes nothing (DGX_ERR_ARG at the
 * next dgx_lane_sync), a result longer than out_cap writes only *d_info (DGX_ERR_CAP).  Asynchronous on the lane. */
int dgx_dev_math_eval(dgx_lane* lane, const dgx_math_node* prog, size_t nnodes, const dgx_math_leaf* leaves,
                      size_t nleaves, const uint64_t* d_range, size_t nrange, uint64_t* d_out_key,
                      uint64_t* d_out_word, uint8_t* d_out_tag, size_t out_cap, uint64_t* d_info);
/* One node of dgx_dev_cascade, every pointer in device memory: its rows v[v_off[i] .. v_off[i+1]) (v_off has nrows + 1
 * values, v_off[0] == 0, v_off[nrows] <= v_cap, the room of v), its dest (ndest values) and its has_val (nhas bytes). */
typedef struct dgx_cascade_node {
    const uint64_t* v;
    const uint64_t* v_off;
    size_t nrows;
    size_t v_cap;
    const uint64_t* dest;
    size_t ndest;
    const uint8_t* has_val;
    size_t nhas;
} dgx_cascade_node;
/* Device form of dgx_cascade: tree and nodes in host memory, the arrays they point at in device memory, so the rows of
 * dgx_dev_list_uids_unfiltered_rows and the dest of dgx_dev_merge_sorted_matrix feed it directly.  d_out_off gets
 * sum(nrows) + 1 offsets, d_dest_out_off nnodes + 1, d_sizes two device uint64 {values, dest values}.  The bounds are
 * sum(v_cap) and sum(ndest): out_cap or dest_cap below them is DGX_ERR_CAP at the call, as every argument error of the
 * host form is DGX_ERR_ARG there (a null pointer with a nonzero size).  Offsets, and dest and rows that do not strictly
 * ascend, are checked on the device: a refused call writes d_sizes = {0, 0} and nothing else, and surfaces as
 * DGX_ERR_ARG at the next dgx_lane_sync.  A forest with no dest value and every v_cap 0 writes the zero offsets and
 * sizes without a launch and without reading the nodes' v_off, which then go unchecked (every row is empty whatever
 * they hold).  Asynchronous on the lane. */
int dgx_dev_cascade(dgx_lane* lane, const dgx_cascade_tree* tree, const dgx_cascade_node* nodes, uint64_t* d_out,
                    uint64_t* d_out_off, size_t out_cap, uint64_t* d_dest_out, uint64_t* d_dest_out_off,
                    size_t dest_cap, uint64_t* d_sizes);
/* Device form of dgx_sg_filter: tree and leaves in host memory, d_d0, the rows, the arrays the leaves point at and the
 * outputs in device memory, so the rows calls' (d_out, d_out_off), dgx_dev_list_count_rows' d_counts and
 * dgx_dev_merge_sorted_matrix's dest feed it directly.  |D0| is d0_cap, or the low 32 bits of the device word d_d0_len
 * when it is set (at most d0_cap); COUNT arrays hold at least |D0| counts or |D0| + 1 offsets.  v_cap is the room of d_v
 * (d_v_off[nrows] must not pass it).  The bounds are d0_cap and v_cap: dest_cap or out_cap below them is DGX_ERR_CAP at
 * the call, as every argument error of the host form is DGX_ERR_ARG there.  d_dest_len is one device uint64.  The order
 * and offset checks, and a length word past its room, run on the device: a refused call writes *d_dest_len = 0 and
 * nothing else, and surfaces as DGX_ERR_ARG at the next dgx_lane_sync.  Asynchronous on the lane; 11 launches. */
int dgx_dev_sg_filter(dgx_lane* lane, const dgx_sg_filter_tree* tree, const dgx_sg_filter_leaf* leaves, size_t nleaves,
                      const uint64_t* d_d0, size_t d0_cap, const uint64_t* d_d0_len, const uint64_t* d_v,
                      const uint64_t* d_v_off, size_t nrows, size_t v_cap, int32_t count, int32_t offset,
                      uint64_t* d_dest_out, size_t dest_cap, uint64_t* d_dest_len, uint64_t* d_out,
                      uint64_t* d_out_off, size_t out_cap, uint32_t* d_counts);
/* Device form of dgx_var_order: var is a host struct whose arrays are device memory (its d_len, when set, a device word
 * whose low 32 bits hold the entry count, at most var->n), d_dest, the rows and the outputs are device memory, so
 * dgx_dev_sg_filter's new dest and rows and a dgx_dev_var_propagate / dgx_dev_math_eval map feed it without a host read.
 * |dest| is ndest, or the low 32 bits of the device word d_ndest when it is set (at most ndest).  v_cap is the room of
 * d_v (d_v_off[nrows] must not pass it).  The bounds are v_cap and ndest: out_cap or dest_cap below them is DGX_ERR_CAP
 * at the call, as every argument error of the host form is DGX_ERR_ARG there.  d_dest_len is one device uint64.  The
 * order, offset and tag checks, a length word past its room and the bool refusal run on the device: a refused call
 * writes *d_dest_len = 0 and nothing else, and surfaces as DGX_ERR_ARG at the next dgx_lane_sync.  ndest == 0 or
 * nrows == 0 writes zero offsets and length without a launch.  Asynchronous on the lane; launches as the host form's. */
int dgx_dev_var_order(dgx_lane* lane, const dgx_math_leaf* var, int desc, const uint64_t* d_dest, size_t ndest,
                      const uint64_t* d_ndest, const uint64_t* d_v, const uint64_t* d_v_off, size_t nrows,
                      size_t v_cap, int32_t count, int32_t offset, uint64_t* d_out, uint64_t* d_out_off,
                      size_t out_cap, uint64_t* d_dest_out, size_t dest_cap, uint64_t* d_dest_len);
/* Device form of dgx_match: packs from dgx_dev_pack_upload; the layers, list leaves, d_uids, col's arrays and the
 * outputs are device memory; mut_off, list_off and the query stay in host memory, as in dgx_dev_trigram_query.  The
 * caller picks the branch: use_uids != 0 takes d_uids, whose count is the low 32 bits of the device word d_nuids (at
 * most nuids, the room; d_nuids NULL: exactly nuids), so dgx_dev_sg_filter's D1, dgx_dev_merge_sorted_matrix,
 * dgx_dev_trigram_query or a previous dgx_dev_match feed it without a host read.  Go's query layer never sends an
 * empty UidList to a filter, so here an empty list is an empty result.  use_uids == 0 takes the trigram leaves.  The
 * bound is nuids or the sum of the leaves' bounds: out_cap below it is DGX_ERR_CAP at the call, as every argument
 * error of the host form is DGX_ERR_ARG there, except the column's offsets, which are checked on the device.
 * d_out_len is one device uint64.  The order and offset checks, a count word past its room and a DGX_MUT_VALUE entry
 * are found on the device: a refused call writes *d_out_len = 0 and nothing else, and surfaces as DGX_ERR_ARG at the
 * next dgx_lane_sync.  A bound of 0 writes a zero length without a launch.  Asynchronous on the lane; launches as the
 * host form's. */
int dgx_dev_match(dgx_lane* lane, const dgx_dev_pack* const* packs, size_t npacks, const uint64_t* d_mut_uids,
                  const uint8_t* d_mut_flags, const uint64_t* mut_off, const uint64_t* d_lists,
                  const uint64_t* list_off, size_t nlists, uint64_t after_uid, int use_uids, const uint64_t* d_uids,
                  size_t nuids, const uint64_t* d_nuids, const dgx_str_column* col, const uint8_t* query,
                  size_t query_len, int64_t max, uint64_t* d_out, size_t out_cap, uint64_t* d_out_len);
/* Device form of dgx_regex_match, with dgx_dev_match's arguments and rules (use_uids, d_nuids, the device-side
 * refusals surfacing at dgx_lane_sync), prog in place of the query.  The program's tables are copied with the call's
 * workspace, so a device chain of dgx_dev_trigram_query, dgx_dev_sg_filter, dgx_dev_match or dgx_dev_regex_match
 * outputs feeds it with no host read.  col's arrays need no padding or alignment: no byte outside
 * [bytes, bytes + nbytes) is read. */
int dgx_dev_regex_match(dgx_lane* lane, const dgx_dev_pack* const* packs, size_t npacks, const uint64_t* d_mut_uids,
                        const uint8_t* d_mut_flags, const uint64_t* mut_off, const uint64_t* d_lists,
                        const uint64_t* list_off, size_t nlists, uint64_t after_uid, int use_uids,
                        const uint64_t* d_uids, size_t nuids, const uint64_t* d_nuids, const dgx_str_column* col,
                        const dgx_regex_prog* prog, uint64_t* d_out, size_t out_cap, uint64_t* d_out_len);
/* Device form of dgx_compare_uids: col is a host struct whose arrays (its str's included) are device memory, args stay
 * in host memory, d_uids and the outputs are device memory.  The candidate count is the low 32 bits of the device word
 * d_nuids (at most nuids, the room; d_nuids NULL: exactly nuids), so the outputs of dgx_dev_sg_filter,
 * dgx_dev_merge_sorted_matrix, dgx_dev_match or a previous dgx_dev_compare_uids feed it without a host read.  The bound
 * is nuids: out_cap below it is DGX_ERR_CAP at the call, as every argument error of the host form is DGX_ERR_ARG there,
 * except the column's offsets, which are checked on the device.  d_out_len is one device uint64; d_counts, when set,
 * room for nuids uint32.  The order and offset checks, a count word past its room and a candidate's bad value are found
 * on the device: a refused call writes *d_out_len = 0 and nothing else, and surfaces as DGX_ERR_ARG at the next
 * dgx_lane_sync.  nuids == 0 writes a zero length without a launch.  Asynchronous on the lane; 5 launches. */
int dgx_dev_compare_uids(dgx_lane* lane, int op, const dgx_val_args* args, const dgx_val_column* col,
                         const uint64_t* d_uids, size_t nuids, const uint64_t* d_nuids, uint64_t* d_out,
                         size_t out_cap, uint64_t* d_out_len, uint32_t* d_counts);
/* Device form of dgx_compare_rows: col as in dgx_dev_compare_uids, args and row_arg in host memory, d_v, d_v_off and
 * the outputs device memory, so the rows calls' (d_out, d_out_off) feed it as they are.  v_cap is the room of d_v
 * (d_v_off[nrows] must not pass it); out_cap below v_cap is DGX_ERR_CAP at the call.  v_off and the column are checked
 * on the device: a refused call writes nrows + 1 zero offsets and no value, and surfaces as DGX_ERR_ARG at the next
 * dgx_lane_sync.  nrows == 0 writes a zero offset without a launch.  Asynchronous on the lane; 4 launches. */
int dgx_dev_compare_rows(dgx_lane* lane, int op, const dgx_val_args* args, const dgx_val_column* col,
                         const uint64_t* d_v, const uint64_t* d_v_off, size_t nrows, size_t v_cap,
                         const uint32_t* row_arg, uint64_t* d_out, uint64_t* d_out_off, size_t out_cap);
/* Device form of dgx_pred_order, with dgx_dev_var_order's rules: col is a host struct whose arrays (its str's
 * included) are device memory, d_dest, the rows and the outputs are device memory, so dgx_dev_sg_filter's new dest
 * and rows and a resident column feed it without a host read.  |dest| is ndest, or the low 32 bits of the device word
 * d_ndest when it is set (at most ndest).  v_cap is the room of d_v (d_v_off[nrows] must not pass it).  The bounds are
 * v_cap and ndest: out_cap or dest_cap below them is DGX_ERR_CAP at the call, as every argument error of the host form
 * is DGX_ERR_ARG there, except the offsets of v_off and the column, which are checked on the device.  d_dest_len is
 * one device uint64.  The order and offset checks, a length word past its room, a list value and a datetime's
 * nanoseconds run on the device: a refused call writes *d_dest_len = 0 and nothing else, and surfaces as DGX_ERR_ARG
 * at the next dgx_lane_sync.  ndest == 0 or nrows == 0 writes zero offsets and length without a launch.  Asynchronous
 * on the lane; launches as the host form's. */
int dgx_dev_pred_order(dgx_lane* lane, const dgx_val_column* col, int desc, const uint64_t* d_dest, size_t ndest,
                       const uint64_t* d_ndest, const uint64_t* d_v, const uint64_t* d_v_off, size_t nrows,
                       size_t v_cap, int32_t count, int32_t offset, uint64_t* d_out, uint64_t* d_out_off,
                       size_t out_cap, uint64_t* d_dest_out, size_t dest_cap, uint64_t* d_dest_len);
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
