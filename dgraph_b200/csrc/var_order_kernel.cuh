// var_order_kernel.cuh -- a uid matrix ordered by a value variable (query/query.go applyOrderAndPagination :2511-2530,
// value-variable branch: updateUidMatrix's order branch :1425-1439, sortAndPaginateUsingVar :2697-2738 and
// updateDestUids :2594-2609) in one call, in Go's exact order.
//
// Row i keeps, in row order, the uids found in dest (U).  W is U's uids with a map entry, in row order.  A row with an
// empty W stays U; otherwise it becomes W ordered by types.Sort: sort.Sort(byValue), Go's pdqsort, whose result on ties
// is one defined permutation.  Both are then cut by x.PageRange(count, offset, len) when either is set, and the new
// dest is the dest values some output row holds.  byValue.Less (types/sort.go :49-82): two nils compare as `desc`, one
// nil sorts last, equal values are not less, otherwise less / mismatchedLess, negated for desc.
//
// Tier 1: a row where any correct sort is Go's answer -- every entry of one numeric tag, no NaN, and either at most 12
// entries (pdqsort runs insertionSort, stable under a strict weak order) or no two equal order keys (the order is
// unique).  Its order comes from a stable LSD radix sort of W by (row, order key): first the 64-bit order key, then
// the row, both through groupby_kernel.cuh's gb_hist_kernel / scan_u64_kernel / gb_scatter_kernel.
// Tier 2: every other row runs Go's pdqsort restated over W in its pre-sort order.  Rows of at most VO_CTA_MIN entries
// run it on one thread; longer rows on one CTA of a persistent grid, where partition and partitionEqual are computed
// cooperatively (the Hoare loop swaps the k-th misplaced entry from the left of the left part with the k-th from the
// right of the right part) and every other step -- choosePivot, breakPatterns, reverseRange, partialInsertionSort,
// insertionSort of short ranges, heapSort -- runs on thread 0 in Go's order.  The ranges stay in Go's order because
// partialInsertionSort's left shift runs down to index 1, not to its range's start, and so can reach an earlier range
// when the comparator is not a strict weak order (NaN, bool, mixed tags).
//
//   vo_check_kernel     thread per slot: dest, map keys and rows strictly ascend, tags are known, offsets start at 0,
//                       do not decrease and end inside v_cap, length words inside their rooms; the size words
//   vo_gather_kernel    thread per value: in dest (IndexOf) and its map entry (Get)
//   scan_u64_kernel x2  U and W positions (look-back)
//   vo_compact_kernel   U and W compacted in row order, W's tags, words, rows and order keys; row offsets of both
//   3 x 8 launches      radix sort of W by order key (64 bits)
//   vo_rowkey_kernel    the sorted entries' rows as the next key
//   3 x P_r launches    radix sort by row, P_r = ceil(bits(nrows - 1) / 8)
//   vo_tier_kernel      ties between adjacent sorted keys and rows unfit for tier 1; a bool first in W is refused
//   vo_rows_kernel      thread per row: its tier, the short tier-2 rows' pdqsort, the long ones listed, page range
//   vo_cta_kernel       fixed grid: the long tier-2 rows, pulled from a counter
//   scan_u64_kernel     page lengths -> output row offsets
//   vo_write_kernel     thread per output slot: the rows; dest positions marked
//   scan_u64_kernel     marks -> new dest positions
//   vo_dest_kernel      the new dest and its length; a refused call writes the length word 0 and nothing else
// Launches: 37 + 3 P_r, set by nrows alone.
#pragma once

#include "cascade_kernel.cuh"  // cc_page_range
#include "groupby_kernel.cuh"  // gb_hist_kernel, gb_scatter_kernel, lanemask_lt, scan_u64_kernel

namespace dgx {

constexpr int kLaneErrVarOrder = 2048;  // lane error flag bit: an order-by-variable input is refused (DGX_ERR_ARG)
constexpr u32 VO_INT = 1, VO_FLOAT = 2, VO_BOOL = 3, VO_NIL = 4;  // DGX_VAL_*
constexpr long VO_MAX_INSERTION = 12;   // pdqsort's maxInsertion
constexpr u64 VO_CTA_MIN = 4096;        // tier-2 rows longer than this run on a CTA
constexpr int VO_NT = 256;
constexpr int VO_STACK_THREAD = 13;     // pdqsort's recursion depth is at most floor(log2 n): 12 for VO_CTA_MIN
constexpr int VO_STACK_CTA = 32;        // and 31 for 32-bit n
constexpr int VO_KEY_PASSES = 8;        // the 64-bit order key
constexpr u32 VO_TIE = 1, VO_MIXED = 2, VO_TIER2 = 4;  // row flags
// words: values, W entries, radix hist length, |dest|, |map|, rows, long tier-2 rows
constexpr int VO_W_M = 0, VO_W_W = 1, VO_W_H = 2, VO_W_ND = 3, VO_W_NM = 4, VO_W_R = 5, VO_W_L = 6, VO_WORDS = 8;
static_assert((u64)1 << (VO_STACK_THREAD - 1) >= VO_CTA_MIN, "a thread's pdqsort stack covers its rows");

struct VoParams {
    const u64* key;         // the map: keys, words, tags (null: every entry of mtype)
    const u64* word;
    const unsigned char* tag;
    const u64* mlen;        // null: mcap entries; else a device word whose low 32 bits are the count
    u64 mcap;
    u32 mtype;
    int desc;
    const u64* dest;
    const u64* dlen;        // null: dcap values; else a device word whose low 32 bits are |dest|
    u64 dcap;
    const u64* v;
    const u64* v_off;       // nrows + 1
    u64 nrows, v_cap;
    int count, offset;
    u64 tiles;              // radix tiles over v_cap
    u64* words;             // VO_WORDS, zeroed
    int* bad;
    int* err;
    u32* ticket;            // the CTA grid's row counter, zeroed
    u64 *uf, *ux, *wf, *wx; // v_cap flags and their scans (v_cap + 1)
    u32* mj;                // v_cap: map index of a W value
    u64* U;                 // v_cap
    u64 *uoff, *woff;       // nrows + 1
    u64 *wuid, *wword;      // v_cap: W in row order; tier 2 sorts it in place
    unsigned char* wtag;
    u32* wrow;
    u64* okey;              // v_cap: order keys
    u64* ek;                // v_cap: the radix sort's first keys (the order keys) ...
    u32* ep;                // ... and payloads (W indices)
    const u32* S;           // the radix sort's payload: W indices in (row, key) order
    u32* rflag;             // nrows, zeroed
    u32* longrows;          // nrows
    u32* pairs;             // v_cap: the cooperative partitions' left positions
    u32* pstart;            // nrows: page starts
    u64* plen;              // nrows: page lengths ...
    u64* po;                // ... scanned (nrows + 1)
    u64* mark;              // dcap, zeroed
    u64* mx;                // dcap + 1
    u64* out;
    u64* out_off;
    u64* dest_out;
    u64* dest_len;
};

__device__ __forceinline__ void vo_refuse(const VoParams& P) {
    atomicOr(P.bad, 1);
    atomicOr(P.err, kLaneErrVarOrder);
}

__device__ __forceinline__ u64 vo_word_len(const u64* w, u64 room, bool& over) {
    if (!w) return room;
    const u64 n = *w & 0xffffffffull;
    over = n > room;
    return over ? 0 : n;
}

// ---- byValue.Less -------------------------------------------------------------------------------------------------

struct VoVal {
    u32 tag;
    u64 w;
};

__device__ __forceinline__ double vo_f64(u64 w) { return __longlong_as_double((long long)w); }
__device__ __forceinline__ int vo_go_tid(u32 t) { return t == VO_INT ? 2 : t == VO_FLOAT ? 3 : t == VO_BOOL ? 4 : 0; }

// types.less with mismatchedLess (types/sort.go :188-232); a bool pair has no case and is not less
__device__ __forceinline__ bool vo_less(VoVal a, VoVal b) {
    const bool an = a.tag == VO_INT || a.tag == VO_FLOAT, bn = b.tag == VO_INT || b.tag == VO_FLOAT;
    if (a.tag != b.tag) {
        if (!an || !bn) return vo_go_tid(a.tag) < vo_go_tid(b.tag);
        if (a.tag == VO_FLOAT) return vo_f64(a.w) < (double)(long long)b.w;
        return (double)(long long)a.w < vo_f64(b.w);
    }
    if (a.tag == VO_INT) return (long long)a.w < (long long)b.w;
    if (a.tag == VO_FLOAT) return vo_f64(a.w) < vo_f64(b.w);
    return false;
}

// types.equal: one tag; -0.0 == +0.0, a NaN equals nothing
__device__ __forceinline__ bool vo_equal(VoVal a, VoVal b) {
    if (a.tag != b.tag) return false;
    if (a.tag == VO_FLOAT) return vo_f64(a.w) == vo_f64(b.w);
    return a.w == b.w;  // int, bool (nil never gets here)
}

__device__ __forceinline__ bool vo_Less(VoVal a, VoVal b, bool desc) {
    const bool an = a.tag == VO_NIL, bn = b.tag == VO_NIL;
    if (an && bn) return desc;
    if (an) return false;
    if (bn) return true;
    if (vo_equal(a, b)) return false;
    const bool l = vo_less(a, b);
    return desc ? !l : l;
}

// The order key of tier 1: int64 with its sign bit flipped; float64's order-preserving bits with -0.0 on +0.0;
// complemented for desc.
__device__ __forceinline__ u64 vo_order_key(u32 tag, u64 w, bool desc) {
    constexpr u64 kSign = 0x8000000000000000ull;
    u64 k = 0;
    if (tag == VO_INT) {
        k = w ^ kSign;
    } else if (tag == VO_FLOAT) {
        if (w == kSign) w = 0;
        k = (w & kSign) ? ~w : (w | kSign);
    }
    return desc ? ~k : k;
}

__device__ __forceinline__ bool vo_is_nan(u32 tag, u64 w) {
    return tag == VO_FLOAT && (w & 0x7ff0000000000000ull) == 0x7ff0000000000000ull && (w & 0x000fffffffffffffull);
}

// One row of W, indexed from its start (Go's data[0 .. n)).
struct VoRow {
    unsigned char* tag;
    u64* w;
    u64* uid;
    bool desc;
    __device__ __forceinline__ VoVal at(long i) const { return VoVal{tag[i], w[i]}; }
    __device__ __forceinline__ bool less(long i, long j) const { return vo_Less(at(i), at(j), desc); }
    __device__ __forceinline__ void swap(long i, long j) const {
        const unsigned char t = tag[i];
        tag[i] = tag[j];
        tag[j] = t;
        const u64 x = w[i];
        w[i] = w[j];
        w[j] = x;
        const u64 u = uid[i];
        uid[i] = uid[j];
        uid[j] = u;
    }
};

// W of row-start b0 as the sort reads it
__device__ __forceinline__ VoRow vo_row(const VoParams& P, u64 b0) {
    return VoRow{P.wtag + b0, P.wword + b0, P.wuid + b0, P.desc != 0};
}

// ---- Go's pdqsort (sort/zsortinterface.go), one thread -------------------------------------------------------------

__device__ __forceinline__ int vo_bits_len(u64 x) { return x ? 64 - __clzll((long long)x) : 0; }

template <class Row>
__device__ __forceinline__ void vo_insertion_sort(const Row& d, long a, long b) {
    for (long i = a + 1; i < b; i++)
        for (long j = i; j > a && d.less(j, j - 1); j--) d.swap(j, j - 1);
}

template <class Row>
__device__ __forceinline__ void vo_sift_down(const Row& d, long lo, long hi, long first) {
    long root = lo;
    for (;;) {
        long child = 2 * root + 1;
        if (child >= hi) return;
        if (child + 1 < hi && d.less(first + child, first + child + 1)) child++;
        if (!d.less(first + root, first + child)) return;
        d.swap(first + root, first + child);
        root = child;
    }
}

template <class Row>
__device__ __forceinline__ void vo_heap_sort(const Row& d, long a, long b) {
    const long first = a, lo = 0, hi = b - a;
    for (long i = (hi - 1) / 2; i >= 0; i--) vo_sift_down(d, i, hi, first);
    for (long i = hi - 1; i >= 0; i--) {
        d.swap(first, first + i);
        vo_sift_down(d, lo, i, first);
    }
}

// partition with the pivot already swapped to a: returns mid, sets *already
template <class Row>
__device__ __forceinline__ long vo_partition(const Row& d, long a, long b, bool* already) {
    long i = a + 1, j = b - 1;
    while (i <= j && d.less(i, a)) i++;
    while (i <= j && !d.less(j, a)) j--;
    if (i > j) {
        *already = true;
        return j;
    }
    d.swap(i, j);
    i++;
    j--;
    for (;;) {
        while (i <= j && d.less(i, a)) i++;
        while (i <= j && !d.less(j, a)) j--;
        if (i > j) break;
        d.swap(i, j);
        i++;
        j--;
    }
    *already = false;
    return j;
}

// partitionEqual with the pivot already swapped to a
template <class Row>
__device__ __forceinline__ long vo_partition_equal(const Row& d, long a, long b) {
    long i = a + 1, j = b - 1;
    for (;;) {
        while (i <= j && !d.less(a, i)) i++;
        while (i <= j && d.less(a, j)) j--;
        if (i > j) break;
        d.swap(i, j);
        i++;
        j--;
    }
    return i;
}

template <class Row>
__device__ __forceinline__ bool vo_partial_insertion_sort(const Row& d, long a, long b) {
    constexpr int kMaxSteps = 5;
    constexpr long kShortestShifting = 50;
    long i = a + 1;
    for (int j = 0; j < kMaxSteps; j++) {
        while (i < b && !d.less(i, i - 1)) i++;
        if (i == b) return true;
        if (b - a < kShortestShifting) return false;
        d.swap(i, i - 1);
        if (i - a >= 2) {
            for (long k = i - 1; k >= 1; k--) {  // Go's bound: down to 1, not to a
                if (!d.less(k, k - 1)) break;
                d.swap(k, k - 1);
            }
        }
        if (b - i >= 2) {
            for (long k = i + 1; k < b; k++) {
                if (!d.less(k, k - 1)) break;
                d.swap(k, k - 1);
            }
        }
    }
    return false;
}

template <class Row>
__device__ __forceinline__ void vo_break_patterns(const Row& d, long a, long b) {
    const long length = b - a;
    if (length >= 8) {
        u64 random = (u64)length;  // xorshift seeded by the length
        const u64 modulus = 1ull << vo_bits_len((u64)length);  // nextPowerOfTwo
        const long idx = a + (length / 4) * 2 - 1;
        for (int i = 0; i < 3; i++) {
            random ^= random << 13;
            random ^= random >> 7;
            random ^= random << 17;
            long other = (long)(random & (modulus - 1));
            if (other >= length) other -= length;
            d.swap(idx - 1 + i, a + other);
        }
    }
}

template <class Row>
__device__ __forceinline__ void vo_order2(const Row& d, long& a, long& b, int& swaps) {
    if (d.less(b, a)) {
        swaps++;
        const long t = a;
        a = b;
        b = t;
    }
}

template <class Row>
__device__ __forceinline__ long vo_median(const Row& d, long a, long b, long c, int& swaps) {
    vo_order2(d, a, b, swaps);
    vo_order2(d, b, c, swaps);
    vo_order2(d, a, b, swaps);
    return b;
}

constexpr int VO_HINT_UNKNOWN = 0, VO_HINT_INC = 1, VO_HINT_DEC = 2;

template <class Row>
__device__ __forceinline__ long vo_choose_pivot(const Row& d, long a, long b, int& hint) {
    constexpr long kShortestNinther = 50;
    constexpr int kMaxSwaps = 4 * 3;
    const long l = b - a;
    int swaps = 0;
    long i = a + l / 4 * 1, j = a + l / 4 * 2, k = a + l / 4 * 3;
    if (l >= 8) {
        if (l >= kShortestNinther) {
            i = vo_median(d, i - 1, i, i + 1, swaps);
            j = vo_median(d, j - 1, j, j + 1, swaps);
            k = vo_median(d, k - 1, k, k + 1, swaps);
        }
        j = vo_median(d, i, j, k, swaps);
    }
    hint = swaps == 0 ? VO_HINT_INC : swaps == kMaxSwaps ? VO_HINT_DEC : VO_HINT_UNKNOWN;
    return j;
}

template <class Row>
__device__ __forceinline__ void vo_reverse_range(const Row& d, long a, long b) {
    long i = a, j = b - 1;
    while (i < j) {
        d.swap(i, j);
        i++;
        j--;
    }
}

// pdqsort's loop state: one call's (a, b, limit, wasBalanced, wasPartitioned).  Go recurses into the smaller side and
// loops on the larger; here the larger side's continuation is pushed and the smaller runs next, in the same order.
struct VoFrame {
    u32 a, b;
    int limit;
    int wb, wp;
};

constexpr int VO_DONE = 0, VO_PART = 1, VO_PART_EQUAL = 2;

// Runs the loop until it needs a partition of [f.a, f.b) (the pivot already swapped to f.a): VO_PART or
// VO_PART_EQUAL; VO_DONE when the sort has finished.
template <class Row>
__device__ __forceinline__ int vo_advance(const Row& d, VoFrame& f, VoFrame* st, int& top) {
    for (;;) {
        const long a = f.a, b = f.b, length = b - a;
        bool ret = false;
        if (length <= VO_MAX_INSERTION) {
            vo_insertion_sort(d, a, b);
            ret = true;
        } else if (f.limit == 0) {
            vo_heap_sort(d, a, b);
            ret = true;
        } else {
            if (!f.wb) {
                vo_break_patterns(d, a, b);
                f.limit--;
            }
            int hint;
            long pivot = vo_choose_pivot(d, a, b, hint);
            if (hint == VO_HINT_DEC) {
                vo_reverse_range(d, a, b);
                pivot = (b - 1) - (pivot - a);
                hint = VO_HINT_INC;
            }
            if (f.wb && f.wp && hint == VO_HINT_INC && vo_partial_insertion_sort(d, a, b)) {
                ret = true;
            } else {
                const int kind = a > 0 && !d.less(a - 1, pivot) ? VO_PART_EQUAL : VO_PART;
                d.swap(a, pivot);
                return kind;
            }
        }
        if (ret) {
            if (top == 0) return VO_DONE;
            f = st[--top];
        }
    }
}

// After the partition: mid and alreadyPartitioned (VO_PART, the pivot already swapped to mid) or mid (VO_PART_EQUAL).
__device__ __forceinline__ void vo_after(VoFrame& f, VoFrame* st, int& top, int kind, long mid, bool already) {
    if (kind == VO_PART_EQUAL) {
        f.a = (u32)mid;
        return;
    }
    const long a = f.a, b = f.b, length = b - a;
    f.wp = already;
    const long left = mid - a, right = b - mid, thr = length / 8;
    if (left < right) {
        f.wb = left >= thr;
        st[top++] = VoFrame{(u32)(mid + 1), (u32)b, f.limit, f.wb, f.wp};
        f = VoFrame{(u32)a, (u32)mid, f.limit, 1, 1};
    } else {
        f.wb = right >= thr;
        st[top++] = VoFrame{(u32)a, (u32)mid, f.limit, f.wb, f.wp};
        f = VoFrame{(u32)(mid + 1), (u32)b, f.limit, 1, 1};
    }
}

// sort.Sort on one thread
template <class Row>
__device__ __forceinline__ void vo_sort_thread(const Row& d, long n) {
    if (n <= 1) return;
    VoFrame st[VO_STACK_THREAD];
    int top = 0;
    VoFrame f{0, (u32)n, vo_bits_len((u64)n), 1, 1};
    for (int kind; (kind = vo_advance(d, f, st, top)) != VO_DONE;) {
        bool already = false;
        const long mid = kind == VO_PART ? vo_partition(d, f.a, f.b, &already) : vo_partition_equal(d, f.a, f.b);
        if (kind == VO_PART) d.swap(mid, f.a);
        vo_after(f, st, top, kind, mid, already);
    }
}

// ---- kernels -------------------------------------------------------------------------------------------------------

__device__ __forceinline__ u64 vo_row_of(const VoParams& P, u64 t) { return lower_bound_g(P.v_off, P.nrows + 1, t + 1) - 1; }

// Grid over max(dcap, mcap, nrows + 1, v_cap) threads.
__global__ void __launch_bounds__(256) vo_check_kernel(const VoParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    bool dover = false, mover = false;
    const u64 nd = vo_word_len(P.dlen, P.dcap, dover), nm = vo_word_len(P.mlen, P.mcap, mover);
    const u64 m = P.v_off[P.nrows];
    if (t == 0) {
        if (dover || mover || m > P.v_cap) vo_refuse(P);
        P.words[VO_W_M] = m > P.v_cap ? 0 : m;
        P.words[VO_W_H] = (u64)GB_RADIX * P.tiles;
        P.words[VO_W_ND] = nd;
        P.words[VO_W_NM] = nm;
        P.words[VO_W_R] = P.nrows;
    }
    if (t > 0 && t < nd && P.dest[t - 1] >= P.dest[t]) vo_refuse(P);
    if (t < nm) {
        if (t > 0 && P.key[t - 1] >= P.key[t]) vo_refuse(P);
        if (P.tag && (P.tag[t] < VO_INT || P.tag[t] > VO_NIL)) vo_refuse(P);
    }
    if (t <= P.nrows) {
        const u64 x = P.v_off[t];
        if (t == 0 ? x != 0 : x < P.v_off[t - 1]) vo_refuse(P);
    }
    // only a row start may descend; with v_off[0] != 0 (refused above) the row search could land before the array
    if (t > 0 && t < m && m <= P.v_cap && P.v_off[0] == 0 && P.v[t - 1] >= P.v[t]) {
        if (P.v_off[vo_row_of(P, t)] != t) vo_refuse(P);
    }
}

// Thread per value slot (grid over v_cap): in dest, and its map entry.
__global__ void __launch_bounds__(256) vo_gather_kernel(const VoParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.words[VO_W_M]) return;
    u64 u = 0, w = 0;
    if (!*P.bad) {
        const u64 x = P.v[t], nd = P.words[VO_W_ND], nm = P.words[VO_W_NM];
        const u64 i = lower_bound_g(P.dest, nd, x);
        if (i < nd && P.dest[i] == x) {
            u = 1;
            const u64 j = lower_bound_g(P.key, nm, x);
            if (j < nm && P.key[j] == x) {
                w = 1;
                P.mj[t] = (u32)j;
            }
        }
    }
    P.uf[t] = u;
    P.wf[t] = w;
}

// Grid over max(v_cap, nrows + 1) threads.
__global__ void __launch_bounds__(256) vo_compact_kernel(const VoParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) return;
    if (t < P.words[VO_W_M]) {
        const u64 x = P.v[t];
        if (P.uf[t]) P.U[P.ux[t]] = x;
        if (P.wf[t]) {
            const u64 p = P.wx[t];
            const u32 j = P.mj[t];
            const u32 tag = P.tag ? P.tag[j] : P.mtype;
            const u64 w = P.word[j];
            P.wuid[p] = x;
            P.wword[p] = w;
            P.wtag[p] = (unsigned char)tag;
            P.wrow[p] = (u32)vo_row_of(P, t);
            P.okey[p] = P.ek[p] = vo_order_key(tag, w, P.desc);
            P.ep[p] = (u32)p;
        }
    }
    if (t <= P.nrows) {
        const u64 o = P.v_off[t];
        P.uoff[t] = P.ux[o];
        P.woff[t] = P.wx[o];
    }
}

// Thread per W entry (grid over v_cap): the order-sorted entries' rows and payloads into the row sort's buffers.
__global__ void __launch_bounds__(256) vo_rowkey_kernel(const VoParams P, const u32* ep, u64* rk, u32* rp) {
    const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || k >= P.words[VO_W_W]) return;
    const u32 p = ep[k];
    rk[k] = P.wrow[p];
    rp[k] = p;
}

// Grid over max(v_cap, nrows) threads: thread k < |W| flags its row when it ties with the entry before it in sorted
// order or is unfit for tier 1; thread r < nrows refuses a row whose first W entry is a bool.
__global__ void __launch_bounds__(256) vo_tier_kernel(const VoParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) return;
    if (t < P.words[VO_W_W]) {
        const u32 p = P.S[t];
        const u32 r = P.wrow[p];
        const u64 first = P.woff[r];
        const u32 tag = P.wtag[p], ft = P.wtag[first];
        u32 f = 0;
        if ((tag != VO_INT && tag != VO_FLOAT) || tag != ft || vo_is_nan(tag, P.wword[p])) f |= VO_MIXED;
        if (t > first && P.okey[P.S[t - 1]] == P.okey[p]) f |= VO_TIE;
        if (f) atomicOr(P.rflag + r, f);
    }
    if (t < P.nrows && P.woff[t + 1] > P.woff[t] && P.wtag[P.woff[t]] == VO_BOOL) vo_refuse(P);
}

// Thread per row (grid over nrows): its tier; a short tier-2 row sorted here, a long one listed for the CTAs; the
// page range of its final length.
__global__ void __launch_bounds__(256, 1) vo_rows_kernel(const VoParams P) {
    const u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || r >= P.nrows) return;
    const u64 b = P.woff[r], n = P.woff[r + 1] - b;
    const u32 f = P.rflag[r];
    if (n > 1 && ((f & VO_MIXED) || ((f & VO_TIE) && n > (u64)VO_MAX_INSERTION))) {
        P.rflag[r] = f | VO_TIER2;
        if (n > VO_CTA_MIN) {
            P.longrows[atomicAdd((unsigned long long*)(P.words + VO_W_L), 1ull)] = (u32)r;
        } else {
            vo_sort_thread(VoRow{P.wtag + b, P.wword + b, P.wuid + b, P.desc != 0}, (long)n);
        }
    }
    const u64 len = n ? n : P.uoff[r + 1] - P.uoff[r];
    long long s = 0, e = (long long)len;
    if (P.count != 0 || P.offset != 0) cc_page_range(P.count, P.offset, (long long)len, s, e);
    P.pstart[r] = (u32)s;
    P.plen[r] = (u64)(e - s);
}

// Block-wide helpers of the cooperative partition (every thread of the CTA calls them).
__device__ __forceinline__ u64 vo_block_sum(u64 x) {
    __shared__ u64 s_sum[VO_NT / 32];
    for (int d = 16; d; d >>= 1) x += __shfl_down_sync(0xffffffffu, x, d);
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = x;
    __syncthreads();
    u64 tot = 0;
#pragma unroll
    for (int w = 0; w < VO_NT / 32; ++w) tot += s_sum[w];
    __syncthreads();
    return tot;
}

// Exclusive rank of a set flag among the CTA's set flags, in thread order; *total the count.
__device__ __forceinline__ u32 vo_block_rank(bool g, u32* total) {
    __shared__ u32 s_cnt[VO_NT / 32];
    const int wid = threadIdx.x >> 5;
    const u32 bal = __ballot_sync(0xffffffffu, g);
    if ((threadIdx.x & 31) == 0) s_cnt[wid] = __popc(bal);
    __syncthreads();
    u32 off = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < VO_NT / 32; ++w) {
        const u32 c = s_cnt[w];
        off += w < wid ? c : 0;
        tot += c;
    }
    __syncthreads();
    *total = tot;
    return off + __popc(bal & lanemask_lt());
}

// partition (eq false) or partitionEqual (eq true) of [a, b) with the pivot at a, by the whole CTA.  An entry goes left
// when Less(i, a) (partition) or !Less(a, i) (partitionEqual); with m of them, the left part is [a + 1, a + m].  Go's
// Hoare loop swaps the k-th entry of the left part that goes right, counted from the left, with the k-th entry of the
// right part that goes left, counted from the right.  Returns mid (before partition's final swap) and the pair count.
template <class Row>
__device__ __forceinline__ void vo_coop_partition(const Row& d, long a, long b, bool eq, u32* pairs, long* mid, u64* npairs) {
    const auto pv = d.at(a);
    auto left = [&](long i) { return eq ? !vo_Less(pv, d.at(i), d.desc) : vo_Less(d.at(i), pv, d.desc); };
    u64 c = 0;
    for (long i = a + 1 + threadIdx.x; i < b; i += VO_NT) c += left(i);
    const long m = (long)vo_block_sum(c), l1 = a + m;
    u64 s = 0;
    for (long c0 = a + 1; c0 <= l1; c0 += VO_NT) {
        const long i = c0 + threadIdx.x;
        const bool g = i <= l1 && !left(i);
        u32 tot;
        const u32 rk = vo_block_rank(g, &tot);
        if (g) pairs[s + rk] = (u32)i;
        s += tot;
    }
    __syncthreads();
    u64 seen = 0;
    for (long c0 = l1 + 1; c0 < b; c0 += VO_NT) {
        const long j = c0 + threadIdx.x;
        const bool g = j < b && left(j);
        u32 tot;
        const u32 rk = vo_block_rank(g, &tot);
        if (g) d.swap(pairs[s - 1 - (seen + rk)], j);
        seen += tot;
    }
    __syncthreads();
    *mid = eq ? l1 + 1 : l1;
    *npairs = s;
}

// Fixed grid of VO_NT-thread CTAs: each pulls long tier-2 rows from the counter and runs Go's pdqsort over it, thread 0
// driving the loop and the whole CTA computing each partition.  Like vo_rows_kernel it declares one CTA per SM as its
// minimum: with the default occupancy target ptxas spills the inlined pdqsort at 40 registers.
template <class Params>
__global__ void __launch_bounds__(VO_NT, 1) vo_cta_kernel(const Params P) {
    __shared__ VoFrame s_f;
    __shared__ VoFrame s_st[VO_STACK_CTA];
    __shared__ int s_top, s_kind;
    __shared__ u32 s_i;
    if (*P.bad) return;
    const u64 nlong = P.words[VO_W_L];
    for (;;) {
        if (threadIdx.x == 0) s_i = atomicAdd(P.ticket, 1u);
        __syncthreads();
        const u32 i = s_i;
        if (i >= nlong) return;
        const u32 r = P.longrows[i];
        const u64 b0 = P.woff[r], n = P.woff[r + 1] - b0;
        const auto d = vo_row(P, b0);
        if (threadIdx.x == 0) {
            s_f = VoFrame{0, (u32)n, vo_bits_len(n), 1, 1};
            s_top = 0;
            s_kind = vo_advance(d, s_f, s_st, s_top);
        }
        __syncthreads();
        while (s_kind != VO_DONE) {
            const int kind = s_kind;
            const long a = s_f.a, b = s_f.b;
            long mid;
            u64 np;
            vo_coop_partition(d, a, b, kind == VO_PART_EQUAL, P.pairs + b0, &mid, &np);
            if (threadIdx.x == 0) {
                if (kind == VO_PART) d.swap(mid, a);
                vo_after(s_f, s_st, s_top, kind, mid, np == 0);
                s_kind = vo_advance(d, s_f, s_st, s_top);
            }
            __syncthreads();
        }
    }
}

// Grid over max(v_cap, nrows + 1) threads: output slot t of row r is the (pstart + rank)-th entry of its final row:
// U for an empty W, the sorted W in place for tier 2, through the radix payload for tier 1.
__global__ void __launch_bounds__(256) vo_write_kernel(const VoParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) return;
    if (t <= P.nrows) P.out_off[t] = P.po[t];
    if (t >= P.po[P.nrows]) return;
    const u64 r = lower_bound_g(P.po, P.nrows + 1, t + 1) - 1;
    const u64 i = P.pstart[r] + (t - P.po[r]), wb = P.woff[r];
    u64 x;
    if (P.woff[r + 1] == wb) x = P.U[P.uoff[r] + i];
    else if (P.rflag[r] & VO_TIER2) x = P.wuid[wb + i];
    else x = P.wuid[P.S[wb + i]];
    P.out[t] = x;
    P.mark[lower_bound_g(P.dest, P.words[VO_W_ND], x)] = 1;
}

// Grid over dcap threads.
template <class Params>
__global__ void __launch_bounds__(256) vo_dest_kernel(const Params P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) {
        if (t == 0) *P.dest_len = 0;
        return;
    }
    const u64 nd = P.words[VO_W_ND];
    if (t < nd && P.mark[t]) P.dest_out[P.mx[t]] = P.dest[t];
    if (t == 0) *P.dest_len = P.mx[nd];
}

}  // namespace dgx
