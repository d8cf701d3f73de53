// compare_kernel.cuh -- the compare functions eq / le / lt / ge / gt / between (types.CompareVals / CompareBetween,
// types/compare.go with Less / Equal, types/sort.go) over a typed value column (dgx_val_column), in one call per path.
//
// The value path (handleValuePostings' compareAttrFn branch, worker/task.go:540-575) tests a UidList:
//   fz_lookup_kernel   match_kernel.cuh's lookup and order checks (byte offsets only for a string column)
//   scan_u64_kernel    value counts -> pair offsets: (candidate, value) pairs flattened
//   cmp_pairs_kernel   fixed grid, thread per pair: a bad value refuses the call; otherwise the typed test, and a hit
//                      counts one for the candidate and sets its keep flag
//   cmp_finish_kernel  thread per candidate: a refused call clears every keep flag; otherwise the counts are written
//   compact_kernel     the kept candidates, in order (compressed_kernel.cuh's look-back compaction)
// eq's arguments arrive sorted and deduplicated (NaN dropped, -0 folded to +0, strings in byte order), so a value takes
// one binary search over them instead of Go's loop over every argument.
//
// The index path (handleCompareFunction's filterRow, :1395-1520) filters selected rows of a uid matrix:
//   fz_lookup_kernel   the column's checks alone (no candidate)
//   cmp_rows_kernel    thread per value slot: the v_off checks, then the value's keep flag -- 1 in a row passed
//                      through, otherwise 1 when one of its column values passes against the row's argument
//   scan_u64_kernel    keep flags -> output positions
//   cmp_place_kernel   the kept values and the row offsets; a refused call writes zero offsets only
// A string value is read as aligned 16-byte segments, the column's first and last byte by byte (regex_kernel.cuh's
// rx_load), so no read leaves the caller's column; the argument's bytes are the call's own copy.
#pragma once

#include "regex_kernel.cuh"  // rx_span / rx_load, and through it match_kernel.cuh

namespace dgx {

constexpr int kLaneErrCompare = 8192;  // lane error flag bit: a compare function's input is refused (DGX_ERR_ARG)
constexpr u32 CMP_LE = 0, CMP_GE = 1, CMP_LT = 2, CMP_GT = 3, CMP_EQ = 4, CMP_BETWEEN = 5;  // DGX_SGF_CMP_*
constexpr u32 CMP_INT = 1, CMP_FLOAT = 2, CMP_BOOL = 3, CMP_TIME = 5, CMP_STR = 6;          // DGX_VAL_*
constexpr u32 CMP_NT = 256;
constexpr u32 CMP_NO_ARG = 0xFFFFFFFFu;  // row_arg: the row passes unchanged
constexpr int CMP_W_M = FZ_W_LONG;       // index path: the value slots the scan covers (v_cap)

struct CmpParams {
    FzParams F;  // candidates, column (uid, val_off, byte_off / bytes of a string column) and workspace
    u32 type, op;
    const u64* word;            // the column's words (not for strings)
    const u32* nsec;            // datetime nanoseconds
    const unsigned char* bad;   // optional, a byte per value
    // arguments
    const u64* aword;
    const u32* ansec;
    const unsigned char* abytes;
    const u64* aoff;
    u32 nargs;
    // value path
    u32* hits;   // ccap: matching values per candidate (zeroed)
    u32* counts; // ccap, optional: the caller's
    // index path
    const u64* v;
    const u64* v_off;
    u64 nrows, v_cap;
    const u32* row_arg;
    u64* flag;     // v_cap: keep flags, then (pos) their scan
    u64* pos;      // v_cap + 1
    u64* out;
    u64* out_off;
};

// The value being tested: its words, or its bytes in the column.
struct CmpVal {
    u64 w;
    u32 ns;
    RxSpan sp;
};

// Bytewise order of value bytes (column) against argument k's: -1, 0 or 1.
__device__ __forceinline__ int cmp_bytes(const RxSpan& sp, const unsigned char* a, u64 alen) {
    const u64 len = sp.hi - sp.lo;
    u64 i = 0;
    for (u64 q = sp.lo & ~15ull; q < sp.hi && i < alen; q += 16) {
        const uint4 v = rx_load(sp, q / 16);
        const u32 w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            if (q + k < sp.lo || q + k >= sp.hi || i >= alen) continue;
            const u32 b = (w[k >> 2] >> (8 * (k & 3))) & 0xFFu, c = __ldg(a + i);
            if (b != c) return b < c ? -1 : 1;
            ++i;
        }
    }
    return len < alen ? -1 : (len > alen ? 1 : 0);
}

// Three-way order of the value against argument k for the ordered types; NaN handled by the caller.
__device__ __forceinline__ int cmp_order(const CmpParams& P, const CmpVal& x, u32 k) {
    switch (P.type) {
        case CMP_INT: {
            const long long a = (long long)P.aword[k], b = (long long)x.w;
            return b < a ? -1 : (b > a ? 1 : 0);
        }
        case CMP_FLOAT: {
            const double a = __longlong_as_double((long long)P.aword[k]), b = __longlong_as_double((long long)x.w);
            return b < a ? -1 : (b > a ? 1 : 0);
        }
        case CMP_TIME: {
            const long long a = (long long)P.aword[k], b = (long long)x.w;
            if (b != a) return b < a ? -1 : 1;
            const u32 an = P.ansec[k];
            return x.ns < an ? -1 : (x.ns > an ? 1 : 0);
        }
        default: {  // CMP_STR
            const u64 a0 = P.aoff[k];
            return cmp_bytes(x.sp, P.abytes + a0, P.aoff[k + 1] - a0);
        }
    }
}

__device__ __forceinline__ bool cmp_isnan(const CmpParams& P, u64 w) {
    return P.type == CMP_FLOAT && isnan(__longlong_as_double((long long)w));
}

// ge(v, a): !Less(v, a), false where Less errors (bool).
__device__ __forceinline__ bool cmp_ge(const CmpParams& P, const CmpVal& x, u32 k) {
    if (P.type == CMP_BOOL) return false;
    if (cmp_isnan(P, x.w) || cmp_isnan(P, P.aword[k])) return true;
    return cmp_order(P, x, k) >= 0;
}
__device__ __forceinline__ bool cmp_le(const CmpParams& P, const CmpVal& x, u32 k) {
    if (P.type == CMP_BOOL) return false;
    if (cmp_isnan(P, x.w) || cmp_isnan(P, P.aword[k])) return true;
    return cmp_order(P, x, k) <= 0;
}

// CompareVals(op, v, args[k]) (between: args k and k + 1); eq over arguments [k, k + ne) sorted and deduplicated.
__device__ bool cmp_test(const CmpParams& P, const CmpVal& x, u32 k, u32 ne) {
    switch (P.op) {
        case CMP_GE: return cmp_ge(P, x, k);
        case CMP_LE: return cmp_le(P, x, k);
        case CMP_BETWEEN: return cmp_ge(P, x, k) && cmp_le(P, x, k + 1);
        case CMP_GT:
        case CMP_LT: {
            if (P.type == CMP_BOOL || cmp_isnan(P, x.w) || cmp_isnan(P, P.aword[k])) return false;
            const int c = cmp_order(P, x, k);
            return P.op == CMP_GT ? c > 0 : c < 0;
        }
        default: {  // CMP_EQ
            if (P.type == CMP_BOOL) {
                for (u32 i = k; i < k + ne; ++i)
                    if ((P.aword[i] != 0) == (x.w != 0)) return true;
                return false;
            }
            if (cmp_isnan(P, x.w)) return false;
            u32 lo = k, hi = k + ne;  // first argument not below the value
            while (lo < hi) {
                const u32 mid = (lo + hi) >> 1;
                if (cmp_order(P, x, mid) > 0) lo = mid + 1; else hi = mid;
            }
            return lo < k + ne && !cmp_isnan(P, P.aword[lo]) && cmp_order(P, x, lo) == 0;
        }
    }
}

__device__ __forceinline__ CmpVal cmp_value(const CmpParams& P, u64 j) {
    CmpVal x{};
    if (P.type == CMP_STR) {
        const u64 b0 = P.F.byte_off[j];
        x.sp = rx_span(P.F.bytes, P.F.nbytes, b0, P.F.byte_off[j + 1] - b0);
    } else {
        x.w = P.word[j];
        if (P.type == CMP_TIME) x.ns = P.nsec[j];
    }
    return x;
}

// A value the value path must refuse: a failed conversion, or datetime nanoseconds out of range.
__device__ __forceinline__ bool cmp_bad(const CmpParams& P, u64 j) {
    return (P.bad && P.bad[j]) || (P.type == CMP_TIME && P.nsec[j] >= 1000000000u);
}

// Fixed grid, thread per (candidate, value) pair.
__global__ void __launch_bounds__(CMP_NT) cmp_pairs_kernel(const CmpParams P) {
    const FzParams& F = P.F;
    if (*(volatile u64*)(F.words + FZ_W_BAD)) return;
    const u64 nc = F.words[FZ_W_N], np = F.words[FZ_W_PAIRS];
    const u64 stride = (u64)gridDim.x * blockDim.x;
    const u32 ne = P.op == CMP_EQ ? P.nargs : 1;
    for (u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x; p < np && p < F.nvals; p += stride) {
        const u64 c = lower_bound_g(F.pair_off, nc + 1, p + 1) - 1;  // the candidate owning pair p
        const u64 j = F.vlo[c] + (p - F.pair_off[c]);
        if (cmp_bad(P, j)) { fz_refuse(F); return; }
        if (ne == 0) continue;  // eq whose every argument was NaN
        if (cmp_test(P, cmp_value(P, j), 0, ne)) {
            atomicAdd(P.hits + c, 1u);
            F.keep[c] = 1;
        }
    }
}

// Thread per candidate slot: a refused call keeps nothing and writes no count.
__global__ void __launch_bounds__(CMP_NT) cmp_finish_kernel(const CmpParams P) {
    const FzParams& F = P.F;
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= F.ccap) return;
    if (*(volatile u64*)(F.words + FZ_W_BAD)) { F.keep[t] = 0; return; }
    if (P.counts && t < F.words[FZ_W_N]) P.counts[t] = P.hits[t];
}

// Thread per value slot of the matrix (grid over max(v_cap, nrows + 1)).
__global__ void __launch_bounds__(CMP_NT) cmp_rows_kernel(const CmpParams P) {
    const FzParams& F = P.F;
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (t == 0) {
        F.words[CMP_W_M] = P.v_cap;
        if (P.v_off[0] != 0 || P.v_off[P.nrows] > P.v_cap) fz_refuse(F);
    }
    if (t < P.nrows && P.v_off[t] > P.v_off[t + 1]) fz_refuse(F);
    if (t >= P.v_cap) return;
    // A refused call keeps nothing, and nothing below reads past an array: with v_off[0] != 0 the row search could land
    // before row_arg, and a column fz_lookup_kernel refused may hold offsets past its values.
    const bool ok = P.v_off[0] == 0 && P.v_off[P.nrows] <= P.v_cap && !*(volatile u64*)(F.words + FZ_W_BAD);
    const u64 m = ok ? P.v_off[P.nrows] : 0;
    u64 keep = 0;
    if (t < m) {
        const u64 r = lower_bound_g(P.v_off, P.nrows + 1, t + 1) - 1;  // the row owning value t
        const u32 k = P.row_arg[r];
        if (k == CMP_NO_ARG) {
            keep = 1;
        } else {
            const u64 x = P.v[t];
            const u64 i = lower_bound_g(F.uid, F.n, x);
            if (i < F.n && ld_probe(F.uid + i) == x) {
                const u64 hi = F.val_off[i + 1];
                for (u64 j = F.val_off[i]; j < hi && !keep; ++j) {
                    if (cmp_bad(P, j)) continue;  // filterRow: a value that does not convert never matches
                    keep = cmp_test(P, cmp_value(P, j), k, 1);
                }
            }
        }
    }
    P.flag[t] = keep;
}

// Thread per value slot and row offset (grid over max(v_cap, nrows + 1)).
__global__ void __launch_bounds__(CMP_NT) cmp_place_kernel(const CmpParams P) {
    const FzParams& F = P.F;
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const bool bad = *(volatile u64*)(F.words + FZ_W_BAD) != 0;
    if (t <= P.nrows) P.out_off[t] = bad ? 0 : P.pos[min(P.v_off[t], P.v_cap)];
    if (!bad && t < P.v_cap && P.flag[t]) P.out[P.pos[t]] = P.v[t];
}

}  // namespace dgx
