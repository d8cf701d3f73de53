// list_uids_kernel.cuh -- posting.List.Uids for a task's rows, the mutable layer included.
//
// handleUidPostings (worker/task.go:783-987) reads every key of a task with List.Uids (posting/list.go:1758-1870)
// under one ListOptions whose Intersect v is non-empty.  Three branches of it are reachable for an unsplit list; row i
// takes mode[i]:
//   0 compressed  no mutable layer (:1795-1800): {x in v : x in pack, x >= after}
//   1 probe       len(v) < ApproxLen (:1805-1820), findPostingWithItr per x of v, after ignored:
//                 {x in v : mut(x) exists ? mut(x) is not a delete : x in pack}
//   2 iterate     otherwise (:1822-1862), iterate + the REF filter + IntersectWith, pack side Seek(after, SeekCurrent):
//                 {x in v : x > after, mut(x) exists ? mut(x) is a SET of a REF posting : x in pack}
// mut(x) is the caller's resolved mutable entry of x (one per uid, ascending): the MVCC choice is made by the caller.
// Every row is a subset of v, so a row is (pack ∩ v above the row's bound) corrected by its mutable entries:
//   icw_rows_* (compressed_kernel.cuh)  pack ∩ v of every row, after = 0 (the bound differs per mode, applied below)
//   lu_classify_kernel   thread per mutable entry: its row (search of mut_off), the order / zero / flag checks against
//                        its predecessor, then whether it INSERTS a uid (emits, in v above the bound, not in the row's
//                        pack ∩ v) or DROPS one (does not emit, in the row's pack ∩ v above the bound)
//   scan_u64_kernel      drop | insert << 31 per entry -> counts of drops and inserts before every entry
//   lu_rows_kernel       thread per row: first element above the bound, row length, the pack-starts-at-0 check
//   scan_u64_kernel      row lengths -> out_off
//   lu_write_kernel      thread per pack ∩ v element and per inserting entry: position = row start + rank among the
//                        kept elements - drops below it + inserts below it
// Workspace is linear in sum_i min(m, ExactLen_i), the number of mutable entries and the number of blocks.
#pragma once

#include "compressed_kernel.cuh"

namespace dgx {

constexpr int kLaneErrMut = 4;  // lane error flag bit: a mutable entry (or a mode-1/2 pack) is malformed (DGX_ERR_ARG)
constexpr unsigned LU_COMPRESSED = 0, LU_PROBE = 1, LU_ITERATE = 2;  // a row's mode (DGX_UIDS_*)
constexpr unsigned LU_DEL = 1, LU_VALUE = 2;                          // an entry's flags (DGX_MUT_*)

// An entry's class word: drops in bits 0..30, inserts in bits 31..61.  scan_u64_kernel sums the words; the host keeps
// a call's entries below 2^31, so no sum carries from one field into the other.
constexpr u64 kLuDrop = 1, kLuInsert = 1ull << 31;
constexpr u64 kLuMask = kLuInsert - 1;

// n with the drops of the summed class word d taken out and its inserts added.
__device__ __forceinline__ u64 lu_apply(u64 n, u64 d) { return n - (d & kLuMask) + (d >> 31); }
__device__ __forceinline__ bool lu_drops(u64 c) { return c & kLuMask; }
__device__ __forceinline__ bool lu_inserts(u64 c) { return c >> 31; }

struct LuParams {
    const unsigned char* mode;  // nrows
    const u64* mut_off;         // nrows + 1
    const u64* const* first;    // nrows: the base array of a mode-1/2 row's non-empty pack (its first uid), else null
    u64 nrows;
    const u64* mut;             // nmut resolved entries, rows concatenated
    const unsigned char* flags; // nmut
    u64 nmut;
    u64 after;
    const u64* v;
    u64 m;
    const u64* a;               // pack ∩ v of every row (after = 0) ...
    const u64* a_off;           // ... as CSR, nrows + 1
    u64 a_cap;                  // values allocated behind a: threads of the write launch for elements
    u64* cls;                   // nmut: drop | insert << 31
    u64* cls_ex;                // nmut + 1: exclusive scan of cls
    u64* lo;                    // nrows: first element of the row's slice of a above the bound
    u64* cnt;                   // nrows: row length
    u64* out;
    u64 out_cap;
    u64* out_off;               // nrows + 1: exclusive scan of cnt
    int* bad;                   // workspace word, zero-initialised: some entry or pack is malformed
    int* err;
};

// Row of element k of a CSR with offsets off[0 .. nrows]: the last r with off[r] <= k.
__device__ __forceinline__ u64 lu_row_of(const u64* off, u64 nrows, u64 k) {
    u64 lo = 1, hi = nrows;
    while (lo < hi) {
        const u64 mid = lo + ((hi - lo) >> 1);
        if (ld_probe(off + mid) <= k) lo = mid + 1; else hi = mid;
    }
    return lo - 1;
}

// First index in [0, n) with a[i] > x (n if none).
__device__ __forceinline__ u64 upper_bound_g(const u64* __restrict__ a, u64 n, u64 x) {
    u64 lo = 0, hi = n;
    while (lo < hi) {
        const u64 mid = lo + ((hi - lo) >> 1);
        if (ld_probe(a + mid) <= x) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// The row's lower bound: >= after (mode 0, Seek SeekStart), > after (mode 2, Seek SeekCurrent), none (mode 1).
__device__ __forceinline__ bool lu_passes(unsigned mode, u64 x, u64 after) {
    return mode == LU_PROBE || (mode == LU_ITERATE ? x > after : x >= after);
}

// Entry k of row r (uid x, flags f) of LuParams or LuuParams P: uid 0, an unknown flag, or a uid not above the row's
// previous entry marks the call malformed.
template <class Params>
__device__ __forceinline__ void lu_check_entry(const Params& P, u64 r, u64 k, u64 x, unsigned f) {
    if (x == 0 || (f & ~(LU_DEL | LU_VALUE)) || (k > ld_probe(P.mut_off + r) && P.mut[k - 1] >= x)) {
        *P.bad = 1;
        atomicOr(P.err, kLaneErrMut);
    }
}

__global__ void __launch_bounds__(256) lu_classify_kernel(const LuParams P) {
    const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P.nmut) return;
    const u64 r = lu_row_of(P.mut_off, P.nrows, k);
    const u64 x = P.mut[k];
    const unsigned f = P.flags[k];
    lu_check_entry(P, r, k, x, f);
    const unsigned mode = P.mode[r];
    u64 c = 0;
    if (lu_passes(mode, x, P.after)) {
        // probe: findPosting finds any non-deleted posting, value postings included; iterate: only a SET of a REF
        const bool emits = mode == LU_PROBE ? !(f & LU_DEL) : f == 0;
        const u64 s = ld_probe(P.a_off + r), e = ld_probe(P.a_off + r + 1);
        const u64 p = s + lower_bound_g(P.a + s, e - s, x);
        const bool in_a = p < e && ld_probe(P.a + p) == x;
        if (in_a && !emits) c = kLuDrop;
        if (!in_a && emits) {
            const u64 j = lower_bound_g(P.v, P.m, x);
            if (j < P.m && ld_probe(P.v + j) == x) c = kLuInsert;
        }
    }
    P.cls[k] = c;
}

__global__ void __launch_bounds__(256) lu_rows_kernel(const LuParams P) {
    const u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= P.nrows) return;
    const unsigned mode = P.mode[r];
    const u64 s = P.a_off[r], e = P.a_off[r + 1];
    u64 lo = s;
    if (mode == LU_COMPRESSED) lo = s + lower_bound_g(P.a + s, e - s, P.after);
    else if (mode == LU_ITERATE) lo = s + upper_bound_g(P.a + s, e - s, P.after);
    const u64 d = P.cls_ex[P.mut_off[r + 1]] - P.cls_ex[P.mut_off[r]];
    P.lo[r] = lo;
    P.cnt[r] = lu_apply(e - lo, d);
    const u64* first = P.first[r];
    if (first && *first == 0) {  // iterate reads uid 0 as the end of the list (:1178-1196)
        *P.bad = 1;
        atomicOr(P.err, kLaneErrMut);
    }
}

// Thread t < a_cap places element t of a (when above its row's bound and not dropped); thread a_cap + k places entry k
// when it inserts.  A malformed entry or pack empties the result (out untouched, every offset 0); past out_cap nothing
// of out is written.
__global__ void __launch_bounds__(256) lu_write_kernel(const LuParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) {
        if (t <= P.nrows) P.out_off[t] = 0;
        return;
    }
    if (P.out_off[P.nrows] > P.out_cap) {
        if (t == 0) atomicExch(P.err, 1);
        return;
    }
    u64 r, x, rank, below;
    if (t < P.a_cap) {
        if (t >= P.a_off[P.nrows]) return;
        r = lu_row_of(P.a_off, P.nrows, t);
        const u64 lo = P.lo[r];
        if (t < lo) return;
        x = P.a[t];
        const u64 ms = ld_probe(P.mut_off + r), me = ld_probe(P.mut_off + r + 1);
        const u64 j = ms + lower_bound_g(P.mut + ms, me - ms, x);
        if (j < me && ld_probe(P.mut + j) == x && lu_drops(P.cls[j])) return;
        rank = t - lo;
        below = P.cls_ex[j] - P.cls_ex[ms];
    } else {
        const u64 k = t - P.a_cap;
        if (k >= P.nmut || !lu_inserts(P.cls[k])) return;
        r = lu_row_of(P.mut_off, P.nrows, k);
        x = P.mut[k];
        const u64 lo = P.lo[r], e = P.a_off[r + 1];
        rank = lower_bound_g(P.a + lo, e - lo, x);
        below = P.cls_ex[k] - P.cls_ex[ld_probe(P.mut_off + r)];
    }
    P.out[lu_apply(P.out_off[r] + rank, below)] = x;
}

}  // namespace dgx
