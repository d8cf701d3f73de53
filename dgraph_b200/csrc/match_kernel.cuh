// match_kernel.cuh -- handleMatchFunction (worker/task.go:1526-1620): match(attr, query, max)'s candidates tested with
// matchFuzzy / levenshteinDistance (worker/match.go:24-67) over a string value column, in one call.
//
// The candidates are the UidList, or uidsForMatch's union of the query's trigram rows (trigram_kernel.cuh with one OR
// node over every leaf).  Every candidate's values are read from a caller-owned column (dgx_str_column), and a
// candidate is kept when one of its values lies within max edits of the query, distances taken over Go's []rune
// conversion (an invalid UTF-8 byte is one U+FFFD).  The device runs:
//   fz_lookup_kernel   thread per candidate: its value range in the column (binary search), the order checks of the
//                      candidates and of the column (uids strictly ascending, offsets ascending and closed; byte
//                      offsets only when the column has them, so compare_kernel.cuh's typed columns share it)
//   scan_u64_kernel    value counts -> pair offsets: the (candidate, value) pairs flattened, so a hub's 10^4 list
//                      values spread over 10^4 threads
//   fz_test_kernel     thread per pair: an empty value fails; a query of more than 64 runes queues the pair for the
//                      long tier; otherwise the short tier decides it on the thread: the exact shortcuts
//                      (|n - m| > max fails, max >= max(n, m) passes), then Myers / Hyyrö bit-parallel edit distance
//                      with the query as the one-word pattern
//   fz_long_kernel     fixed grid, warp per queued pair (a query of 65 to 4096 runes): the value's rune count from a warp-parallel scan of its bytes,
//                      the shortcuts, then blocked Myers over W = ceil(m / 64) words run as a wavefront -- lane l
//                      holds words l and l + 32 in registers, text rune j reaches word w at step j + w, the horizontal
//                      carry and the rune's Peq row travel one lane up per step by shuffle
//   compact_kernel     the kept candidates, in order (compressed_kernel.cuh's look-back compaction)
// Peq (the query's match masks) is built once on the host from the query's decoded runes: a row per ASCII code and a
// row per distinct other rune, those runes sorted for the text's binary search, W words per row.  A malformed input
// sets the call's bad word and the lane's kLaneErrMatch bit: every later stage then keeps nothing, so the call writes
// only a zero length.
#pragma once

#include "compressed_kernel.cuh"
#include "encode_kernel.cuh"  // scan_u64_kernel

namespace dgx {

constexpr int kLaneErrMatch = 4096;  // lane error flag bit: a match() input is malformed (DGX_ERR_ARG at sync)
constexpr int FZ_MAX_WORDS = 64;     // 4096 query runes: lane l holds words l and l + 32
constexpr int FZ_LONG_NT = 256;      // fz_long_kernel: 8 warps per CTA
constexpr u32 FZ_FFFD = 0xFFFDu;

struct FzParams {
    // candidates
    const u64* cand;
    const u64* cand_len;  // device word: the low 32 bits are the candidate count (null: ccap) ...
    u64 ccap;             // ... at most this
    // the column
    const u64* uid;
    const u64* val_off;
    const u64* byte_off;
    const unsigned char* bytes;
    u64 n, nvals, nbytes;
    // the query
    const u64* peq;    // (128 + nd) rows of W words
    const u32* other;  // nd sorted non-ASCII runes; row 128 + k is other[k]
    u32 nd, W, m, max;
    // workspace
    u64* words;  // [0] candidate count, [1] pair count, [2] long-tier pairs, [3] bad
    u64* cnt;    // ccap: values of candidate t
    u64* vlo;    // ccap: its first value
    u64* pair_off;  // ccap + 1
    unsigned char* keep;  // ccap
    u64* longq;  // nvals: (candidate << 32) | value of a queued pair
    int* err;
    int err_bit;  // the lane error bit a refusal raises (kLaneErrMatch for match() and regexp())
};
constexpr int FZ_W_N = 0, FZ_W_PAIRS = 1, FZ_W_LONG = 2, FZ_W_BAD = 3;

__device__ __forceinline__ void fz_refuse(const FzParams& P) {
    atomicExch((unsigned long long*)(P.words + FZ_W_BAD), 1ull);
    atomicOr(P.err, P.err_bit);
}

// utf8.DecodeRuneInString over p[i .. len): the rune and its width; anything Go does not accept is (U+FFFD, 1).
__device__ __forceinline__ u32 fz_decode(const unsigned char* p, u64 len, u64 i, u32* r) {
    const u32 b0 = p[i];
    if (b0 < 0x80) { *r = b0; return 1; }
    *r = FZ_FFFD;
    if (b0 < 0xC2 || b0 > 0xF4) return 1;
    const u32 need = b0 < 0xE0 ? 1 : (b0 < 0xF0 ? 2 : 3);
    if (i + need >= len) return 1;  // truncated
    u32 lo = 0x80, hi = 0xBF;
    if (b0 == 0xE0) lo = 0xA0;
    else if (b0 == 0xED) hi = 0x9F;
    else if (b0 == 0xF0) lo = 0x90;
    else if (b0 == 0xF4) hi = 0x8F;
    const u32 b1 = p[i + 1];
    if (b1 < lo || b1 > hi) return 1;
    if (need == 1) { *r = ((b0 & 0x1F) << 6) | (b1 & 0x3F); return 2; }
    const u32 b2 = p[i + 2];
    if (b2 < 0x80 || b2 > 0xBF) return 1;
    if (need == 2) { *r = ((b0 & 0x0F) << 12) | ((b1 & 0x3F) << 6) | (b2 & 0x3F); return 3; }
    const u32 b3 = p[i + 3];
    if (b3 < 0x80 || b3 > 0xBF) return 1;
    *r = ((b0 & 0x07) << 18) | ((b1 & 0x3F) << 12) | ((b2 & 0x3F) << 6) | (b3 & 0x3F);
    return 4;
}

// The Peq row of a text rune: its ASCII code, 128 + its index among the query's other runes, or rows (no match).
__device__ __forceinline__ u32 fz_row(const FzParams& P, u32 r) {
    if (r < 128) return r;
    u32 lo = 0, hi = P.nd;
    while (lo < hi) {
        const u32 mid = (lo + hi) >> 1;
        if (P.other[mid] < r) lo = mid + 1; else hi = mid;
    }
    return lo < P.nd && P.other[lo] == r ? 128 + lo : 128 + P.nd;
}
__device__ __forceinline__ u64 fz_eq(const FzParams& P, u32 row, u32 w) {
    return row < 128 + P.nd ? __ldg(P.peq + (u64)row * P.W + w) : 0ull;
}

// One word of Hyyrö's blocked Myers step: the vertical deltas (Pv, Mv) of 64 pattern runes advanced by one text rune
// whose match mask is eq, with the horizontal delta hin (-1, 0, +1) entering at the word's lowest row.  Returns the
// horizontal delta leaving at row bit hb.
__device__ __forceinline__ int fz_block(u64& Pv, u64& Mv, u64 eq, int hin, u32 hb) {
    const u64 neg = hin < 0 ? 1ull : 0ull;
    const u64 Xv = eq | Mv;
    eq |= neg;
    const u64 Xh = (((eq & Pv) + Pv) ^ Pv) | eq;
    u64 Ph = Mv | ~(Xh | Pv);
    u64 Mh = Pv & Xh;
    const int hout = (int)((Ph >> hb) & 1ull) - (int)((Mh >> hb) & 1ull);
    Ph = (Ph << 1) | (hin > 0 ? 1ull : 0ull);
    Mh = (Mh << 1) | neg;
    Pv = Mh | ~(Xv | Ph);
    Mv = Ph & Xv;
    return hout;
}

// The shortcuts every pair takes first: 1 passes, 0 fails, -1 needs the distance.  n, m >= 1 here.
__device__ __forceinline__ int fz_shortcut(u64 n, u64 m, u32 max) {
    const u64 d = n > m ? n - m : m - n;
    if (d > max) return 0;
    if ((u64)max >= (n > m ? n : m)) return 1;
    return -1;
}

// Thread per candidate slot (grid over max(ccap, n + 1, nvals + 1)): the value range of candidate t, and the checks.
__global__ void __launch_bounds__(256) fz_lookup_kernel(const FzParams P) {
    const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const u64 raw = P.cand_len ? *P.cand_len & 0xFFFFFFFFull : P.ccap;
    const u64 nc = raw <= P.ccap ? raw : 0;
    if (t == 0) {
        P.words[FZ_W_N] = nc;
        if (raw > P.ccap) fz_refuse(P);
        if (P.val_off[0] != 0 || P.val_off[P.n] != P.nvals ||
            (P.byte_off && (P.byte_off[0] != 0 || P.byte_off[P.nvals] != P.nbytes)))
            fz_refuse(P);
    }
    if (t < P.n) {
        if ((t > 0 && P.uid[t - 1] >= P.uid[t]) || P.val_off[t] > P.val_off[t + 1]) fz_refuse(P);
    }
    if (P.byte_off && t < P.nvals && P.byte_off[t] > P.byte_off[t + 1]) fz_refuse(P);
    if (t < P.ccap) {
        u64 c = 0, lo = 0;
        if (t < nc) {
            const u64 x = P.cand[t];
            if (t > 0 && P.cand[t - 1] >= x) fz_refuse(P);
            const u64 k = lower_bound_g(P.uid, P.n, x);
            if (k < P.n && ld_probe(P.uid + k) == x) {
                lo = P.val_off[k];
                const u64 hi = P.val_off[k + 1];
                c = hi > lo ? hi - lo : 0;
            }
        }
        P.cnt[t] = c;
        P.vlo[t] = lo;
    }
}

// Thread per pair (grid over nvals): a query of at most 64 runes is decided here, the shortcuts first; a longer
// query queues the pair for fz_long_kernel.
__global__ void __launch_bounds__(256) fz_test_kernel(const FzParams P) {
    const u64 p = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (*(volatile u64*)(P.words + FZ_W_BAD)) return;
    const u64 nc = P.words[FZ_W_N], np = P.words[FZ_W_PAIRS];
    if (p >= np || p >= P.nvals) return;
    const u64 c = lower_bound_g(P.pair_off, nc + 1, p + 1) - 1;  // the candidate owning pair p
    const u64 j = P.vlo[c] + (p - P.pair_off[c]);
    const u64 b0 = P.byte_off[j], len = P.byte_off[j + 1] - b0;
    if (len == 0) return;  // matchFuzzy: an empty value never matches
    if (P.W > 1) {  // a query of more than 64 runes: the long tier
        P.longq[atomicAdd((unsigned long long*)(P.words + FZ_W_LONG), 1ull)] = (c << 32) | (j - P.vlo[c]);
        return;
    }
    const unsigned char* s = P.bytes + b0;
    u32 n = 0;
    for (u64 i = 0; i < len; ++n) {
        u32 r;
        i += fz_decode(s, len, i, &r);
    }
    const int sc = fz_shortcut(n, P.m, P.max);
    if (sc == 1) P.keep[c] = 1;
    if (sc >= 0) return;
    u64 Pv = ~0ull, Mv = 0;
    const u32 hb = P.m - 1;
    u32 score = P.m;
    for (u64 i = 0; i < len;) {
        u32 r;
        i += fz_decode(s, len, i, &r);
        score += fz_block(Pv, Mv, fz_eq(P, fz_row(P, r), 0), 1, hb);
    }
    if (score <= P.max) P.keep[c] = 1;
}

// Is byte i of s[0 .. len) the start of a rune?  Every byte outside 80-BF is (an invalid sequence is one byte wide, a
// valid one holds continuation bytes only); a continuation byte is not when the nearest lead byte within three before
// it starts a valid sequence that covers it.
__device__ __forceinline__ bool fz_starts(const unsigned char* s, u64 len, u64 i) {
    if ((s[i] & 0xC0) != 0x80) return true;
    for (u32 k = 1; k <= 3 && k <= i; ++k) {
        if ((s[i - k] & 0xC0) == 0x80) continue;
        u32 r;
        return fz_decode(s, len, i - k, &r) <= k;
    }
    return true;
}

// Fixed grid, warp per queued pair.
__global__ void __launch_bounds__(FZ_LONG_NT) fz_long_kernel(const FzParams P) {
    const int lane = threadIdx.x & 31;
    const u64 nwarps = (u64)gridDim.x * (FZ_LONG_NT / 32);
    if (*(volatile u64*)(P.words + FZ_W_BAD)) return;
    const u64 nq = P.words[FZ_W_LONG];
    const u32 W = P.W, hb_last = (P.m - 1) & 63;
    for (u64 q = (u64)blockIdx.x * (FZ_LONG_NT / 32) + (threadIdx.x >> 5); q < nq; q += nwarps) {
        const u64 e = P.longq[q], c = e >> 32, j = P.vlo[c] + (e & 0xFFFFFFFFull);
        const u64 b0 = P.byte_off[j], len = P.byte_off[j + 1] - b0;
        const unsigned char* s = P.bytes + b0;
        u64 n = 0;
        for (u64 b = 0; b < len; b += 32) {  // every lane takes every round: the ballot is the whole warp's
            const u64 i = b + lane;
            const bool st = i < len && fz_starts(s, len, i);
            n += __popc(__ballot_sync(0xffffffffu, st));
        }
        const int sc = fz_shortcut(n, P.m, P.max);
        if (sc >= 0) {
            if (sc == 1 && lane == 0) P.keep[c] = 1;
            continue;
        }
        // the wavefront: step t, word w = lane + 32 k works on text rune t - w
        u64 Pv0 = ~0ull, Mv0 = 0, Pv1 = ~0ull, Mv1 = 0;
        u32 out0 = 0, out1 = 0;  // (Peq row << 2) | (hout + 1) of each word's last step
        long long score = P.m;
        u64 cur = 0;  // lane 0: the next rune's byte
        const long long steps = (long long)n + W - 1;
        const u32 w0 = lane, w1 = lane + 32;
        for (long long t = 0; t < steps; ++t) {
            const u32 up0 = __shfl_up_sync(0xffffffffu, out0, 1);
            const u32 wrap = __shfl_sync(0xffffffffu, out0, 31);
            u32 up1 = __shfl_up_sync(0xffffffffu, out1, 1);
            if (lane == 0) up1 = wrap;
            const long long j0 = t - (long long)w0;
            if (w0 < W && j0 >= 0 && j0 < (long long)n) {
                u32 row;
                int hin;
                if (w0 == 0) {
                    u32 r;
                    cur += fz_decode(s, len, cur, &r);
                    row = fz_row(P, r);
                    hin = 1;
                } else {
                    row = up0 >> 2;
                    hin = (int)(up0 & 3) - 1;
                }
                const int h = fz_block(Pv0, Mv0, fz_eq(P, row, w0), hin, w0 == W - 1 ? hb_last : 63);
                out0 = (row << 2) | (u32)(h + 1);
                if (w0 == W - 1) score += h;
            }
            const long long j1 = t - (long long)w1;
            if (w1 < W && j1 >= 0 && j1 < (long long)n) {
                const u32 row = up1 >> 2;
                const int h = fz_block(Pv1, Mv1, fz_eq(P, row, w1), (int)(up1 & 3) - 1, w1 == W - 1 ? hb_last : 63);
                out1 = (row << 2) | (u32)(h + 1);
                if (w1 == W - 1) score += h;
            }
        }
        const u32 owner = (W - 1) & 31;
        score = __shfl_sync(0xffffffffu, score, owner);
        if (lane == 0 && score <= (long long)P.max) P.keep[c] = 1;
    }
}

}  // namespace dgx
