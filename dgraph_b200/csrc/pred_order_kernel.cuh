// pred_order_kernel.cuh -- a uid matrix ordered by a predicate's values without its index (query/query.go
// applyOrderAndPagination :2511-2592, predicate branch: updateUidMatrix's order branch :1425-1439, worker/sort.go
// sortWithoutIndex :139-187 with sortByValue :775-822, fetchValue and paginate :740-773, and updateDestUids
// :2594-2609) in one call, in Go's exact order.
//
// Row i keeps, in row order, the uids found in dest (U).  W is U's uids with a value in the column, in row order; N is
// the rest of U (no value, or a value whose conversion failed: the column's bad byte), also in row order.  The row
// becomes W sorted by types.Sort -- sort.Sort(byValue), Go's pdqsort, under byValue.Less: equal values are not less,
// otherwise types.less, negated for desc -- followed by N unsorted, then cut by x.PageRange(count, offset, |U|).  The
// new dest is the dest values some output row holds.  Every W value has the column's type: int64 (<), float64 (<, ==:
// -0 equals +0, a NaN is neither less nor equal, so under desc a NaN pair is less both ways), datetime (the instant,
// seconds then nanoseconds) or string (bytes, unsigned, a proper prefix less).
//
// The tiers are var_order_kernel.cuh's.  Tier 1: rows whose order any correct sort gives -- no NaN, and either no two
// equal sort keys or (int64, float64, datetime, whose keys are the whole value) at most 12 entries, where pdqsort runs
// a stable insertionSort.  A string's key is its first 8 bytes, big-endian and zero-padded: where keys differ the key
// order is the byte order, but equal keys do not mean equal strings, so a string row with two adjacent equal keys goes
// to tier 2 whatever its length.  Tier 1 comes from a stable LSD radix sort of W by (row, key); a datetime sorts first
// by its nanoseconds (30 bits), then by its seconds.  Tier 2 runs var_order's pdqsort (its helpers are templated on the
// row) on a thread for rows of at most VO_CTA_MIN entries and on a CTA of vo_cta_kernel's grid for longer ones; its
// comparator is vo_Less over PoVal, which reads a string's bytes as rx_load's aligned 16-byte segments.
//
//   fz_lookup_kernel    the column's checks alone (match_kernel.cuh, as dgx_compare_rows runs it)
//   po_check_kernel     thread per slot: dest and rows strictly ascend, offsets start at 0, do not decrease and end
//                       inside v_cap, dest's length word inside its room; a refused column; the size words
//   po_gather_kernel    thread per value: in dest (IndexOf), its value in the column (a lower bound over uid); a uid
//                       owning more than one value (a list predicate) or a datetime's nanoseconds of 10^9 or more refuse
//   scan_u64_kernel x2  U and W positions (look-back); N's position is U's less W's
//   po_compact_kernel   W (uid, word, extra, row, keys) and N compacted in row order; row offsets of U and W
//   3 x K launches      radix sort of W by key: K = 8 (int64, float64, string); datetime 3 x 4 over the nanoseconds,
//                       po_rekey_kernel, 3 x 8 over the seconds
//   po_rekey_kernel     the sorted entries' rows as the next key (and, for datetime, their seconds after the
//                       nanoseconds' passes)
//   3 x P_r launches    radix sort by row, P_r = ceil(bits(nrows - 1) / 8)
//   po_tier_kernel      adjacent sorted keys tied and NaN: the rows' flags
//   po_rows_kernel      thread per row: its tier, the short tier-2 rows' pdqsort, the long ones listed, page range
//   vo_cta_kernel       fixed grid: the long tier-2 rows, pulled from a counter
//   scan_u64_kernel     page lengths -> output row offsets
//   po_write_kernel     thread per output slot: sorted W, then N; dest positions marked
//   scan_u64_kernel     marks -> new dest positions
//   vo_dest_kernel      the new dest and its length; a refused call writes the length word 0 and nothing else
// Launches: 38 + 3 P_r for int64, float64 and string columns, 51 + 3 P_r for datetime, set by the type and nrows alone.
#pragma once

#include "compare_kernel.cuh"    // the column's lookup (FzParams, fz_lookup_kernel) and rx_span / rx_load
#include "var_order_kernel.cuh"  // the tiers, Go's pdqsort and its cooperative partition

namespace dgx {

constexpr int kLaneErrPredOrder = 16384;  // lane error flag bit: an order-by-predicate input is refused (DGX_ERR_ARG)
constexpr u32 PO_INT = 1, PO_FLOAT = 2, PO_TIME = 5, PO_STR = 6;  // DGX_VAL_*
constexpr int PO_NS_PASSES = 4;            // a datetime's nanoseconds: below 10^9 < 2^30
constexpr u64 PO_NS_MASK = (1ull << 30) - 1;
constexpr u32 PO_NSEC = 1000000000u;

struct PoParams {
    FzParams F;                // the column as fz_lookup_kernel checks it: uid, val_off (byte_off, bytes of strings)
    u32 type;
    int desc;
    const u64* word;           // the column's words (int64, float64 bits, datetime seconds)
    const u32* nsec;           // datetime nanoseconds
    const unsigned char* vbad; // optional, a byte per value: its conversion failed
    const u64* dest;
    const u64* dlen;           // null: dcap values; else a device word whose low 32 bits are |dest|
    u64 dcap;
    const u64* v;
    const u64* v_off;          // nrows + 1
    u64 nrows, v_cap;
    int count, offset;
    u64 tiles;                 // radix tiles over v_cap
    u64* words;                // VO_WORDS, zeroed (var_order's layout; VO_W_NM unused)
    int* bad;
    int* err;
    u32* ticket;               // the CTA grid's row counter, zeroed
    u64 *uf, *ux, *wf, *wx;    // v_cap flags and their scans (v_cap + 1)
    u32* vj;                   // v_cap: column value index of a W value
    u64* N;                    // v_cap: N in row order
    u64 *uoff, *woff;          // nrows + 1
    u64 *wuid, *wword, *wext;  // v_cap: W in row order (word: value or first byte; ext: nanoseconds or end byte)
    u32* wrow;
    u64 *okey, *okey2;         // v_cap: sort keys (datetime: seconds, nanoseconds; otherwise okey2 is 0)
    u64* ek;                   // v_cap: the radix sort's first keys ...
    u32* ep;                   // ... and payloads (W indices)
    const u32* S;              // the radix sort's payload: W indices in (row, key) order
    u32* rflag;                // nrows, zeroed
    u32* longrows;             // nrows
    u32* pairs;                // v_cap: the cooperative partitions' left positions
    u32* pstart;               // nrows: page starts
    u64* plen;                 // nrows: page lengths ...
    u64* po;                   // ... scanned (nrows + 1)
    u64* mark;                 // dcap, zeroed
    u64* mx;                   // dcap + 1
    u64* out;
    u64* out_off;
    u64* dest_out;
    u64* dest_len;
};

__device__ __forceinline__ void po_refuse(const PoParams& P) {
    atomicOr(P.bad, 1);
    atomicOr(P.err, kLaneErrPredOrder);
}

// ---- byValue.Less over one column's type --------------------------------------------------------------------------

// Bytes [q, q + 8) of a span (offsets from sp.seg) as a big-endian word, those at or past sp.hi as 0.
__device__ __forceinline__ u64 po_be8(const RxSpan& sp, u64 q) {
    if (q >= sp.hi) return 0;
    const u64 g = q >> 4, s = q & 15;
    const uint4 A = rx_load(sp, g);
    const uint4 B = s > 8 ? rx_load(sp, g + 1) : make_uint4(0, 0, 0, 0);
    const u64 L0 = A.x | ((u64)A.y << 32), L1 = A.z | ((u64)A.w << 32), L2 = B.x | ((u64)B.y << 32);
    const u64 lo = s < 8 ? L0 : L1, hi = s < 8 ? L1 : L2;
    const u32 sh = (u32)(s & 7) * 8;
    u64 x = sh ? (lo >> sh) | (hi << (64 - sh)) : lo;  // little-endian: byte k at bits 8k
    if (sp.hi - q < 8) x &= (1ull << (8 * (sp.hi - q))) - 1;
    return ((u64)__byte_perm((u32)x, 0, 0x0123) << 32) | __byte_perm((u32)(x >> 32), 0, 0x0123);
}

// One W value: word and extra by type (int64 / float64: the word; datetime: seconds and nanoseconds; string: its
// byte range in the column, whose bytes and length ride along).
struct PoVal {
    u32 type;
    u64 w, x;
    const unsigned char* bytes;
    u64 nbytes;
};

// Bytewise, unsigned, a proper prefix less: -1, 0 or 1.
__device__ __forceinline__ int po_str_cmp(const PoVal& a, const PoVal& b) {
    const RxSpan sa = rx_span(a.bytes, a.nbytes, a.w, a.x - a.w), sb = rx_span(b.bytes, b.nbytes, b.w, b.x - b.w);
    const u64 la = a.x - a.w, lb = b.x - b.w, m = la < lb ? la : lb;
    for (u64 i = 0; i < m; i += 8) {
        u64 ka = po_be8(sa, sa.lo + i), kb = po_be8(sb, sb.lo + i);
        if (m - i < 8) {  // only the bytes both hold
            const u64 keep = ~0ull << (8 * (8 - (m - i)));
            ka &= keep;
            kb &= keep;
        }
        if (ka != kb) return ka < kb ? -1 : 1;
    }
    return la < lb ? -1 : (la > lb ? 1 : 0);
}

// byValue.Less for values of one type: equal is not less; otherwise types.less, negated for desc.  A NaN is neither
// less nor equal (c == 2), so under desc it is less than anything and anything is less than it.
__device__ __forceinline__ bool vo_Less(const PoVal& a, const PoVal& b, bool desc) {
    int c;
    if (a.type == PO_INT) {
        c = (long long)a.w < (long long)b.w ? -1 : (a.w == b.w ? 0 : 1);
    } else if (a.type == PO_FLOAT) {
        const double x = vo_f64(a.w), y = vo_f64(b.w);
        c = x < y ? -1 : (x == y ? 0 : (x > y ? 1 : 2));
    } else if (a.type == PO_TIME) {
        c = a.w != b.w ? ((long long)a.w < (long long)b.w ? -1 : 1) : (a.x < b.x ? -1 : (a.x == b.x ? 0 : 1));
    } else {
        c = po_str_cmp(a, b);
    }
    if (c == 0) return false;
    const bool l = c < 0;
    return desc ? !l : l;
}

// One row of W, indexed from its start.
struct PoRow {
    u64* w;
    u64* x;
    u64* uid;
    u32 type;
    const unsigned char* bytes;
    u64 nbytes;
    bool desc;
    __device__ __forceinline__ PoVal at(long i) const { return PoVal{type, w[i], x[i], bytes, nbytes}; }
    __device__ __forceinline__ bool less(long i, long j) const { return vo_Less(at(i), at(j), desc); }
    __device__ __forceinline__ void swap(long i, long j) const {
        const u64 a = w[i];
        w[i] = w[j];
        w[j] = a;
        const u64 b = x[i];
        x[i] = x[j];
        x[j] = b;
        const u64 u = uid[i];
        uid[i] = uid[j];
        uid[j] = u;
    }
};

// W of row-start b0 as the sort reads it (vo_cta_kernel's overload for this call)
__device__ __forceinline__ PoRow vo_row(const PoParams& P, u64 b0) {
    return PoRow{P.wword + b0, P.wext + b0, P.wuid + b0, P.type, P.F.bytes, P.F.nbytes, P.desc != 0};
}

// ---- kernels -------------------------------------------------------------------------------------------------------

__device__ __forceinline__ u64 po_row_of(const PoParams& P, u64 t) { return lower_bound_g(P.v_off, P.nrows + 1, t + 1) - 1; }

// Grid over max(dcap, nrows + 1, v_cap) threads.
__global__ void __launch_bounds__(256) po_check_kernel(const PoParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    bool dover = false;
    const u64 nd = vo_word_len(P.dlen, P.dcap, dover);
    const u64 m = P.v_off[P.nrows];
    if (t == 0) {
        if (dover || m > P.v_cap || *(volatile u64*)(P.F.words + FZ_W_BAD)) po_refuse(P);
        P.words[VO_W_M] = m > P.v_cap ? 0 : m;
        P.words[VO_W_H] = (u64)GB_RADIX * P.tiles;
        P.words[VO_W_ND] = nd;
        P.words[VO_W_R] = P.nrows;
    }
    if (t > 0 && t < nd && P.dest[t - 1] >= P.dest[t]) po_refuse(P);
    if (t <= P.nrows) {
        const u64 x = P.v_off[t];
        if (t == 0 ? x != 0 : x < P.v_off[t - 1]) po_refuse(P);
    }
    // only a row start may descend; with v_off[0] != 0 (refused above) the row search could land before the array
    if (t > 0 && t < m && m <= P.v_cap && P.v_off[0] == 0 && P.v[t - 1] >= P.v[t]) {
        if (P.v_off[po_row_of(P, t)] != t) po_refuse(P);
    }
}

// Thread per value slot (grid over v_cap): in dest, and its value.  A refused call (a refused column included) reads
// no column array.
__global__ void __launch_bounds__(256) po_gather_kernel(const PoParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= P.words[VO_W_M]) return;
    u64 u = 0, w = 0;
    if (!*(volatile int*)P.bad) {
        const FzParams& F = P.F;
        const u64 x = P.v[t], nd = P.words[VO_W_ND];
        const u64 i = lower_bound_g(P.dest, nd, x);
        if (i < nd && P.dest[i] == x) {
            u = 1;
            const u64 k = lower_bound_g(F.uid, F.n, x);
            if (k < F.n && ld_probe(F.uid + k) == x) {
                const u64 lo = F.val_off[k], hi = F.val_off[k + 1];
                if (hi - lo > 1) {
                    po_refuse(P);  // a list predicate's column: Go refuses to sort by it
                } else if (hi == lo + 1 && !(P.vbad && P.vbad[lo])) {
                    if (P.type == PO_TIME && P.nsec[lo] >= PO_NSEC) po_refuse(P);
                    w = 1;
                    P.vj[t] = (u32)lo;
                }
            }
        }
    }
    P.uf[t] = u;
    P.wf[t] = w;
}

// Grid over max(v_cap, nrows + 1) threads.
__global__ void __launch_bounds__(256) po_compact_kernel(const PoParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) return;
    if (t < P.words[VO_W_M]) {
        const u64 x = P.v[t];
        if (P.wf[t]) {
            const u64 p = P.wx[t];
            const u32 j = P.vj[t];
            u64 w, e = 0, k, k2 = 0;
            if (P.type == PO_STR) {
                w = P.F.byte_off[j];
                e = P.F.byte_off[j + 1];
                const RxSpan sp = rx_span(P.F.bytes, P.F.nbytes, w, e - w);
                k = po_be8(sp, sp.lo);
                if (P.desc) k = ~k;
            } else if (P.type == PO_TIME) {
                w = P.word[j];
                e = P.nsec[j];
                k = vo_order_key(VO_INT, w, P.desc);
                k2 = P.desc ? PO_NS_MASK - e : e;
            } else {
                w = P.word[j];
                k = vo_order_key(P.type, w, P.desc);
            }
            P.wuid[p] = x;
            P.wword[p] = w;
            P.wext[p] = e;
            P.wrow[p] = (u32)po_row_of(P, t);
            P.okey[p] = k;
            P.okey2[p] = k2;
            P.ek[p] = P.type == PO_TIME ? k2 : k;
            P.ep[p] = (u32)p;
        } else if (P.uf[t]) {
            P.N[P.ux[t] - P.wx[t]] = x;
        }
    }
    if (t <= P.nrows) {
        const u64 o = P.v_off[t];
        P.uoff[t] = P.ux[o];
        P.woff[t] = P.wx[o];
    }
}

// Thread per W entry (grid over v_cap): the sorted entries' next key -- the seconds of a datetime (key) or the row
// (key null) -- and payloads into the next sort's buffers.
__global__ void __launch_bounds__(256) po_rekey_kernel(const PoParams P, const u64* key, const u32* ep, u64* rk,
                                                       u32* rp) {
    const u64 k = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || k >= P.words[VO_W_W]) return;
    const u32 p = ep[k];
    rk[k] = key ? key[p] : P.wrow[p];
    rp[k] = p;
}

// Thread per W entry (grid over v_cap): a row is flagged VO_TIE when an entry ties with the one before it in sorted
// order, VO_MIXED (tier 2 whatever its length) for a NaN or a string prefix tie.
__global__ void __launch_bounds__(256) po_tier_kernel(const PoParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || t >= P.words[VO_W_W]) return;
    const u32 p = P.S[t];
    const u32 r = P.wrow[p];
    u32 f = 0;
    if (P.type == PO_FLOAT && vo_is_nan(VO_FLOAT, P.wword[p])) f |= VO_MIXED;
    if (t > P.woff[r] && P.okey[P.S[t - 1]] == P.okey[p] && P.okey2[P.S[t - 1]] == P.okey2[p])
        f |= P.type == PO_STR ? VO_MIXED : VO_TIE;
    if (f) atomicOr(P.rflag + r, f);
}

// Thread per row (grid over nrows): its tier; a short tier-2 row sorted here, a long one listed for the CTAs; the
// page range over |U|.
__global__ void __launch_bounds__(256, 1) po_rows_kernel(const PoParams P) {
    const u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad || r >= P.nrows) return;
    const u64 b = P.woff[r], n = P.woff[r + 1] - b;
    const u32 f = P.rflag[r];
    if (n > 1 && ((f & VO_MIXED) || ((f & VO_TIE) && n > (u64)VO_MAX_INSERTION))) {
        P.rflag[r] = f | VO_TIER2;
        if (n > VO_CTA_MIN) {
            P.longrows[atomicAdd((unsigned long long*)(P.words + VO_W_L), 1ull)] = (u32)r;
        } else {
            vo_sort_thread(vo_row(P, b), (long)n);
        }
    }
    long long s, e;
    cc_page_range(P.count, P.offset, (long long)(P.uoff[r + 1] - P.uoff[r]), s, e);
    P.pstart[r] = (u32)s;
    P.plen[r] = (u64)(e - s);
}

// Grid over max(v_cap, nrows + 1) threads: output slot t of row r is the (pstart + rank)-th entry of sorted W ++ N:
// the sorted W in place for tier 2, through the radix payload for tier 1, then N.
__global__ void __launch_bounds__(256) po_write_kernel(const PoParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*P.bad) return;
    if (t <= P.nrows) P.out_off[t] = P.po[t];
    if (t >= P.po[P.nrows]) return;
    const u64 r = lower_bound_g(P.po, P.nrows + 1, t + 1) - 1;
    const u64 i = P.pstart[r] + (t - P.po[r]), wb = P.woff[r], nw = P.woff[r + 1] - wb;
    u64 x;
    if (i >= nw) x = P.N[P.uoff[r] - wb + (i - nw)];
    else if (P.rflag[r] & VO_TIER2) x = P.wuid[wb + i];
    else x = P.wuid[P.S[wb + i]];
    P.out[t] = x;
    P.mark[lower_bound_g(P.dest, P.words[VO_W_ND], x)] = 1;
}

}  // namespace dgx
